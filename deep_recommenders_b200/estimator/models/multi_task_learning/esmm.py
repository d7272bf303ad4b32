"""Estimator-side ``ESMM`` (reference estimator/models/multi_task_learning/esmm.py:13-59):
``ESMM(feature_columns, hidden_units, activation=relu, ...)(features)`` returns ``(p_cvr, p_ctr, p_ctcvr)``, each
[B, 1], with ``p_ctcvr = p_ctr * p_cvr``.

The pCVR and pCTR towers (``dnn(inputs, hidden_units + [1])`` each, :38-54) are one grouped pair of towers: layer 0 is
one Dense on the concatenated kernel, the upper layers are grouped Dense calls; tower 0 is pCVR and tower 1 pCTR, the
reference's creation order.  The sigmoids and the product are torch glue on [B, 2].
``batch_normalization=True`` raises (broken upstream, as in ``dnn()``); dropout other than None raises
NotImplementedError; the reference forwards ``**kwargs`` to ``tf.layers.dense``, which is not served.
"""
from __future__ import annotations

import torch

from ....feature_column import input_layer
from ..feature_interaction.dnn import relu
from .mixture_of_experts import check_tower_options, input_width
from .towers import GroupedTowers


class ESMM(object):

    def __init__(self,
                 feature_columns,
                 hidden_units,
                 activation=relu,
                 batch_normalization=False,
                 dropout=None,
                 seed=None, device=None,
                 **kwargs):
        check_tower_options(batch_normalization, dropout)
        if kwargs:
            raise NotImplementedError(f"ESMM: Dense options {sorted(kwargs)} are not served")
        self._columns = feature_columns
        self._hidden_units = list(hidden_units)
        self._activation = activation
        self._device = torch.device(device) if device is not None else torch.device("cuda")
        self._towers = GroupedTowers(2, input_width(feature_columns), self._hidden_units + [1], activation,
                                     shared_input=True, seed=seed, device=self._device)

    def parameters(self):
        return self._towers.parameters()

    def dense_views(self):
        """[(kernel, bias)] of the pCVR tower's Dense layers, then the pCTR tower's (the reference's creation order)."""
        return self._towers.dense_views()

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        logits = self._towers(input_layer(features, self._columns, device=self._device))    # [B, 2]: cvr, ctr
        p_cvr = torch.sigmoid(logits[:, 0:1])
        p_ctr = torch.sigmoid(logits[:, 1:2])
        p_ctcvr = p_ctr * p_cvr
        return p_cvr, p_ctr, p_ctcvr
