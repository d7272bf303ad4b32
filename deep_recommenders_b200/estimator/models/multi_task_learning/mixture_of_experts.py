"""Estimator-side ``MMoE`` (reference estimator/models/multi_task_learning/mixture_of_experts.py:13-93):
``MMoE(feature_columns, num_tasks, num_experts, expert_hidden_units, task_hidden_units, ...)(features)`` returns a list
of ``num_tasks`` raw [B, 1] outputs.

Forward, five calls: the experts' layer-0 Dense (one GEMM on the concatenated kernel), the experts' grouped upper
layers, one gating Dense (no bias) for all T gates, ``dr_moe_mix_fwd`` (every gate's softmax and mixture in one pass,
no stacked copy of the experts), and the grouped task towers (hidden layers with the task activation, last layer
linear).  Each expert is ``dnn(inputs, expert_hidden_units)`` of the reference: its last layer is linear too.

Deviations from the reference (DESIGN section 7):
  * The reference builds ``num_experts`` gates and uses the first ``num_tasks`` (:73 loops over experts, :80-82 indexes
    by task).  Only the T used gates are built; the reference's extra gates are variables nothing reads.  With
    ``num_tasks > num_experts`` the reference fails with IndexError; this raises it at construction.
  * ``batch_normalization=True`` raises (the branch is broken upstream, as in ``dnn()``); dropout other than None
    raises NotImplementedError.
"""
from __future__ import annotations

import math

import torch

from .... import ops
from ....feature_column import NumericColumn, input_layer
from ..feature_interaction.dnn import relu
from .towers import GroupedTowers

MAX_EXPERTS = 32
MAX_TASKS = 16


def check_tower_options(batch_normalization, dropout) -> None:
    if batch_normalization is True:
        raise TypeError("batch_normalization=True is broken in the reference "
                        "(tf.nn.batch_normalization called without mean/variance) and is not supported")
    if dropout is not None:
        raise NotImplementedError("dropout inside the towers is not on the accelerated path")


def input_width(feature_columns) -> int:
    cols = list(feature_columns)
    for c in cols:
        if not isinstance(c, NumericColumn):
            raise NotImplementedError(f"the multi-task models take numeric columns only; got {type(c).__name__}")
    if not cols:
        raise ValueError("feature_columns must not be empty")
    return sum(c.width for c in cols)


class MMoE(object):

    def __init__(self,
                 feature_columns,
                 num_tasks,
                 num_experts,
                 expert_hidden_units,
                 task_hidden_units,
                 task_hidden_activation=relu,
                 task_batch_normalization=False,
                 task_dropout=None,
                 expert_hidden_activation=relu,
                 expert_batch_normalization=False,
                 expert_dropout=None,
                 seed=None, device=None):
        check_tower_options(task_batch_normalization, task_dropout)
        check_tower_options(expert_batch_normalization, expert_dropout)
        num_tasks, num_experts = int(num_tasks), int(num_experts)
        if num_experts < 1 or num_tasks < 1:
            raise ValueError(f"num_experts and num_tasks must be at least 1, got {num_experts} and {num_tasks}")
        if num_tasks > num_experts:
            raise IndexError(f"list index out of range: MMoE builds one gate per expert and gives task t gate t, so "
                             f"num_tasks ({num_tasks}) cannot exceed num_experts ({num_experts})")
        if num_experts > MAX_EXPERTS or num_tasks > MAX_TASKS:
            raise ValueError(f"MMoE serves up to {MAX_EXPERTS} experts and {MAX_TASKS} tasks, got {num_experts} and "
                             f"{num_tasks}")
        if not expert_hidden_units:
            raise ValueError("expert_hidden_units must not be empty")
        self._columns = feature_columns
        self._num_tasks = num_tasks
        self._num_experts = num_experts
        self._expert_hidden_units = list(expert_hidden_units)
        self._task_hidden_units = list(task_hidden_units)
        self._task_hidden_activation = task_hidden_activation
        self._expert_hidden_activation = expert_hidden_activation
        self._device = torch.device(device) if device is not None else torch.device("cuda")
        d = input_width(feature_columns)
        s = (lambda k: None) if seed is None else (lambda k: seed + k)
        self._experts = GroupedTowers(num_experts, d, self._expert_hidden_units, expert_hidden_activation,
                                      shared_input=True, seed=s(0), device=self._device)
        # gate t: its own Dense(num_experts, use_bias=False), glorot over (d, num_experts); block t of [d, T*E]
        gen = torch.Generator().manual_seed(s(1)) if seed is not None else None
        limit = math.sqrt(6.0 / (d + num_experts))
        gk = torch.empty((num_tasks, d, num_experts), dtype=torch.float32).uniform_(-limit, limit, generator=gen)
        self._gate_kernel = torch.nn.Parameter(
            gk.permute(1, 0, 2).reshape(d, num_tasks * num_experts).contiguous().to(self._device))
        self._tasks = GroupedTowers(num_tasks, self._experts.out_dim, self._task_hidden_units + [1],
                                    task_hidden_activation, shared_input=False, seed=s(2), device=self._device)

    def parameters(self):
        """Experts, then gates, then task towers: the reference's creation order."""
        yield from self._experts.parameters()
        yield self._gate_kernel
        yield from self._tasks.parameters()

    def dense_views(self):
        """[(kernel, bias or None)] of every Dense the reference creates and reads, in its creation order (experts,
        the T used gates, task towers), as views of the parameters."""
        E = self._num_experts
        gates = [(self._gate_kernel.data[:, t * E:(t + 1) * E], None) for t in range(self._num_tasks)]
        return self._experts.dense_views() + gates + self._tasks.dense_views()

    def gating_logits(self, inputs):
        """[B, T*E]: every gate's pre-softmax logits from one Dense."""
        return ops.DenseFn.apply(inputs, self._gate_kernel, None, 0)

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        inputs = input_layer(features, self._columns, device=self._device)
        experts = self._experts(inputs)                                       # [B, E*H]
        mixed = ops.MoEMixFn.apply(experts, self.gating_logits(inputs), self._num_tasks)   # [B, T*H]
        out = self._tasks(mixed)                                              # [B, T]
        return [out[:, t:t + 1] for t in range(self._num_tasks)]
