"""DIN's ``ActivationUnit`` and ``Dice`` layers at ``deep_recommenders.keras.models.ranking.din``, and a ``DIN`` model
on them.

``ActivationUnit`` mirrors reference keras/models/ranking/din.py:6-85 (constructor arguments and defaults :9-35, the
two Dense layers of ``build`` :37-57, ``call(x_embeddings, y_embeddings=None)`` :59-71, ``get_config`` keys :73-85).
With a string activation and an interacter of None, ``Subtract()`` or ``Multiply()`` the whole unit -- concat,
hidden Dense, activation, Dense(1) -- is one CUDA kernel (dr_din_attn_fwd, T = 1); any other interacter, or a
``Layer`` activation such as ``Dice``, runs the composition (concat, ``Dense`` on dr_dense, the activation,
``Dense(1)``).  ``call_pooled(keys, query)`` is DIN's target attention over a behaviour sequence with the weighted sum
pooling in the same kernel.

``Dice`` mirrors din.py:88-130 and keeps its arithmetic, including ``sqrt(std + epsilon)`` as the denominator (the
square root of the standard deviation).  Deviations: it serves rank-2 inputs ``[N, U]`` only (other ranks raise
``ValueError``); for a constant row the gradient through the standard deviation is 0 where TensorFlow's gives NaN.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch
from torch import nn

from .... import ops
from ....embedding import EmbeddingCollection
from ...layers.base import (Dense, Layer, Model, get_initializer, get_regularizer, get_registered,
                            register_keras_serializable, regularization_penalty, serialize_initializer)
from ...layers.merge import Multiply, Subtract

_FUSED_INTERACTERS = {Subtract: "subtract", Multiply: "multiply"}


def _as_tensor(x, device):
    if isinstance(x, torch.Tensor):
        return x if x.dtype == torch.float32 else x.float()
    return torch.as_tensor(np.asarray(x, dtype=np.float32), device=device)


def _shape(x):
    return tuple(x.shape) if isinstance(x, torch.Tensor) else tuple(np.shape(x))


def _serialize_layer(layer):
    return None if layer is None else {"class_name": layer.__class__.__name__, "config": layer.get_config()}


def _deserialize_layer(obj):
    if not isinstance(obj, dict):
        return obj
    cls = {"Subtract": Subtract, "Multiply": Multiply, "Dice": Dice}.get(obj["class_name"])
    if cls is None:
        cls = get_registered(obj["class_name"])
    return cls.from_config(obj.get("config", {}))


@register_keras_serializable()
class Dice(Layer):
    """Dice activation (Zhou et al., 2018) on a rank-2 input: y = a > 0 ? p*a : (1 - p)*a with a = PReLU(x) and
    p = sigmoid((x - mean) / sqrt(std + epsilon)) over each row."""

    def __init__(self,
                 epsilon: float = 1e-8,
                 alpha_initializer="zeros",
                 alpha_regularizer=None,
                 **kwargs):
        super().__init__(**kwargs)
        self._epsilon = epsilon
        self._alpha_initializer = alpha_initializer
        self._alpha_regularizer = get_regularizer(alpha_regularizer)
        self.alpha = None

    def build(self, input_shape, device=None):
        if len(input_shape) != 2:
            raise ValueError("`Dice` serves rank-2 inputs [batch, units]. Got rank = {}".format(len(input_shape)))
        dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
        a = torch.empty((int(input_shape[-1]),), dtype=torch.float32, device=dev)
        get_initializer(self._alpha_initializer)(a, None)
        self.alpha = nn.Parameter(a)        # PReLU's alpha, one per column (shared over the batch axis)
        self.built = True

    def forward(self, inputs, **kwargs):
        if not self.built:
            self.build(_shape(inputs), device=inputs.device if isinstance(inputs, torch.Tensor) else None)
        return self.call(inputs, **kwargs)

    def call(self, inputs, **kwargs):
        rank = inputs.dim() if isinstance(inputs, torch.Tensor) else np.ndim(inputs)
        if rank != 2:
            raise ValueError("`Dice` serves rank-2 inputs [batch, units]. Got rank = {}".format(rank))
        x = _as_tensor(inputs, self.alpha.device)
        return ops.DiceFn.apply(x, self.alpha, float(self._epsilon))

    @property
    def losses(self):
        if self.alpha is None or self._alpha_regularizer is None:
            return []
        return [regularization_penalty(self._alpha_regularizer, self.alpha)]

    def get_config(self):
        config = {
            "epsilon": self._epsilon,
            "alpha_initializer": serialize_initializer(self._alpha_initializer),
            "alpha_regularizer": self._alpha_regularizer,
        }
        base_config = super().get_config()
        return {**base_config, **config}


@register_keras_serializable()
class ActivationUnit(Layer):
    """ DIN's activation unit: Dense(1)(act(Dense(units)([x | y | interacter([x, y])]))) """

    def __init__(self,
                 units,
                 interacter=None,
                 use_bias=True,
                 activation="relu",
                 kernel_init="truncated_normal",
                 kernel_regu=None,
                 bias_init="zeros",
                 bias_regu=None,
                 seed: Optional[int] = None,
                 **kwargs):
        super().__init__(**kwargs)
        self._kernel_units = int(units)
        self._interacter = _deserialize_layer(interacter)
        self._use_bias = use_bias
        activation = _deserialize_layer(activation)
        if isinstance(activation, Layer):
            self._kernel_activation = activation
            self._act = None
        elif isinstance(activation, str) or callable(activation):
            self._kernel_activation = activation
            self._act = ops.act_code(activation)
        else:
            self._kernel_activation = None
            self._act = ops.act_code(None)
        self._kernel_init = kernel_init
        self._kernel_regu = get_regularizer(kernel_regu)
        self._bias_init = bias_init
        self._bias_regu = get_regularizer(bias_regu)
        self._seed = seed
        inter = type(self._interacter) if self._interacter is not None else None
        self._fused = self._act is not None and (self._interacter is None or inter in _FUSED_INTERACTERS)
        self._interact = ops.INTERACT_CODES[_FUSED_INTERACTERS.get(inter)] if self._fused else None
        self.dense_kernel = None
        self.dense_output = None

    def build(self, input_shape, device=None):
        seed = self._seed
        layer_act = isinstance(self._kernel_activation, Layer)
        self.dense_kernel = Dense(self._kernel_units, activation=None if layer_act else self._kernel_activation,
                                  use_bias=self._use_bias, kernel_initializer=self._kernel_init,
                                  kernel_regularizer=self._kernel_regu, bias_initializer=self._bias_init,
                                  bias_regularizer=self._bias_regu, seed=seed)
        self.dense_output = Dense(1, activation=None, use_bias=self._use_bias, kernel_initializer=self._kernel_init,
                                  kernel_regularizer=self._kernel_regu, bias_initializer=self._bias_init,
                                  bias_regularizer=self._bias_regu, seed=None if seed is None else seed + 1)
        dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
        self.dense_kernel._device = self.dense_output._device = torch.device(dev)
        if self._fused and input_shape is not None:
            D = int(input_shape[-1])
            self.dense_kernel.build((None, (3 if self._interacter is not None else 2) * D), device=dev)
            self.dense_output.build((None, self._kernel_units), device=dev)
        self.built = True

    def forward(self, x_embeddings, y_embeddings=None, **kwargs):
        if not self.built:
            self.build(_shape(x_embeddings),
                       device=x_embeddings.device if isinstance(x_embeddings, torch.Tensor) else None)
        return self.call(x_embeddings, y_embeddings, **kwargs)

    def _device(self):
        return self.dense_kernel._device

    def _weights(self):
        w2 = self.dense_output.kernel
        return self.dense_kernel.kernel, self.dense_kernel.bias, w2, self.dense_output.bias

    def call(self, x_embeddings, y_embeddings=None, **kwargs):
        dev = self._device()
        x = _as_tensor(x_embeddings, dev)
        y = x if y_embeddings is None else _as_tensor(y_embeddings, dev)
        if self._fused:
            w1, b1, w2, b2 = self._weights()
            _, score = ops.DINAttentionFn.apply(x.unsqueeze(1), y, w1, b1, w2, b2, self._interact, self._act, False)
            return score
        u = [x, y]
        if self._interacter is not None:
            u.append(self._interacter([x, y]))
        h = self.dense_kernel(torch.cat(u, dim=1))
        if isinstance(self._kernel_activation, Layer):
            h = self._kernel_activation(h)
        return self.dense_output(h)

    def call_pooled(self, keys, query):
        """(pooled [B, D], score [B, T]): the unit applied at every position of keys [B, T, D] against query [B, D],
        and DIN's weighted sum pooling sum_t score * keys, in one kernel."""
        if not self._fused:
            raise ValueError("`ActivationUnit.call_pooled` needs a string activation and an interacter of None, "
                             "`Subtract()` or `Multiply()`")
        if not self.built:
            self.build(_shape(keys), device=keys.device if isinstance(keys, torch.Tensor) else None)
        w1, b1, w2, b2 = self._weights()
        return ops.DINAttentionFn.apply(keys, query, w1, b1, w2, b2, self._interact, self._act, True)

    @property
    def losses(self):
        return [l for d in (self.dense_kernel, self.dense_output) if d is not None and d.kernel is not None
                for l in d.losses]

    def get_config(self):
        act = self._kernel_activation
        config = {
            "units": self._kernel_units,
            "interacter": _serialize_layer(self._interacter),
            "use_bias": self._use_bias,
            "activation": _serialize_layer(act) if isinstance(act, Layer) else (
                "linear" if act is None else (act if isinstance(act, str) else getattr(act, "__name__", str(act)))),
            "kernel_init": serialize_initializer(self._kernel_init),
            "kernel_regu": self._kernel_regu,
            "bias_init": serialize_initializer(self._bias_init),
            "bias_regu": self._bias_regu,
        }
        base_config = super().get_config()
        return {**base_config, **config}


_INTERACTERS = {"subtract": Subtract, "multiply": Multiply, None: None, "none": None}


class DIN(Model):
    """Deep Interest Network (Zhou et al., KDD 2018, "Deep Interest Network for Click-Through Rate Prediction"), this
    repo's definition (the reference has only the layers):

        e_item   = item_table[item_ids]                 [B, D]      one table for the target and the history
        keys     = item_table[hist_ids]                 [B, T, D]   id -1 (padding) or out of range: a zero row
        interest = sum_t ActivationUnit(keys_t, e_item) * keys_t    one fused kernel (dr_din_attn_fwd)
        x        = [flatten(context) | e_item | interest]
        prob     = sigmoid(Dense(1)(MLP(x)))            MLP: Dense layers with Dice (or a DR_ACT_* name) between them

    Inputs: (context_ids [B, S] or None, item_ids [B], hist_ids [B, T]), int32 or int64.
    """

    def __init__(self, item_rows: int, dim: int, context_rows: Sequence[int] = (), att_units: int = 36,
                 att_activation="relu", interacter: Optional[str] = "subtract",
                 dnn_units: Sequence[int] = (200, 80), dnn_activation="dice", sparse_lr: Optional[float] = None,
                 seed: Optional[int] = None, device=None, **kwargs):
        super().__init__(**kwargs)
        if dim % 4 != 0 or not (4 <= dim <= 128):
            raise ValueError(f"DIN: embedding dimension must be a multiple of 4 in [4, 128], got {dim}")
        if interacter not in _INTERACTERS:
            raise ValueError(f"DIN: interacter must be one of 'subtract', 'multiply' or None, got {interacter!r}")
        dev = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        self.sparse_lr = sparse_lr
        gen = torch.Generator(device=dev).manual_seed(seed) if seed is not None else None
        std = 1.0 / np.sqrt(dim)
        t = torch.empty((int(item_rows), int(dim)), dtype=torch.float32, device=dev)
        nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)
        self.item_table = nn.Parameter(t)
        context_rows = [int(r) for r in context_rows]
        self.context = (EmbeddingCollection(context_rows, dim, with_linear=False, device=dev, seed=seed,
                                            sparse_lr=sparse_lr) if context_rows else None)
        inter = _INTERACTERS[interacter]
        self.attention = ActivationUnit(att_units, interacter=inter() if inter else None, activation=att_activation,
                                        seed=None if seed is None else seed + 100)
        self.attention.build((None, dim), device=dev)
        dice = dnn_activation == "dice"
        layers, width = [], len(context_rows) * dim + 2 * dim
        for i, u in enumerate(dnn_units):
            dense = Dense(int(u), activation=None if dice else dnn_activation,
                          seed=None if seed is None else seed + 200 + i)
            dense.build((None, width), device=dev)
            layers.append(dense)
            if dice:
                act = Dice()
                act.build((None, int(u)), device=dev)
                layers.append(act)
            width = int(u)
        self.mlp = nn.ModuleList(layers)
        self.head = Dense(1, seed=None if seed is None else seed + 300)
        self.head.build((None, width), device=dev)
        self._cfg = dict(item_rows=int(item_rows), dim=int(dim), context_rows=context_rows, att_units=int(att_units),
                         att_activation=att_activation, interacter=interacter, dnn_units=[int(u) for u in dnn_units],
                         dnn_activation=dnn_activation)
        self.built = True

    def logits(self, inputs) -> torch.Tensor:
        context_ids, item_ids, hist_ids = inputs
        e_item = ops.Gather.apply(self.item_table, item_ids, self.sparse_lr)
        keys = ops.Gather.apply(self.item_table, hist_ids, self.sparse_lr)
        interest, _ = self.attention.call_pooled(keys, e_item)
        parts = [e_item, interest]
        if self.context is not None:
            if context_ids is None:
                raise ValueError("DIN: this model has context slots, so context_ids must be given")
            stack, _ = self.context(context_ids, want_logit=False)
            parts.insert(0, stack.reshape(stack.shape[0], -1))
        x = torch.cat(parts, dim=1)
        for layer in self.mlp:
            x = layer(x)
        return self.head(x)

    def call(self, inputs, **kwargs):
        return torch.sigmoid(self.logits(inputs))

    @property
    def losses(self):
        return list(self.attention.losses) + [l for layer in self.mlp for l in layer.losses] + list(self.head.losses)

    def get_config(self):
        return {**super().get_config(), **self._cfg}
