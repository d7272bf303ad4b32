"""Estimator-side DeepFM twin (reference estimator/models/ranking/deepfm.py:9-43):
``DeepFM(indicator_columns, embedding_columns, dnn_units, dnn_activation=relu, ...)(features)``
-> sigmoid(fm + dnn(concat(fm.embeddings), dnn_units + [1]))."""
from __future__ import annotations

import torch

from ..feature_interaction import FM
from ..feature_interaction.dnn import DnnTower, relu


class DeepFM(object):

    def __init__(self,
                 indicator_columns,
                 embedding_columns,
                 dnn_units,
                 dnn_activation=relu,
                 dnn_batch_normalization=False,
                 dnn_dropout=None,
                 sparse_lr=None, seed=None, device=None,
                 **dnn_kwargs):
        if dnn_batch_normalization or dnn_dropout is not None:
            raise NotImplementedError("batch normalisation / dropout are not on the accelerated path")
        self._dnn_hidden_units = list(dnn_units)
        self._fm = FM(indicator_columns, embedding_columns, sparse_lr=sparse_lr, seed=seed, device=device)
        self._dnn = DnnTower(self._dnn_hidden_units + [1], activation=dnn_activation, seed=seed)

    def parameters(self):
        yield from self._fm.parameters()
        yield from self._dnn.parameters()

    def embedding_collection(self):
        """The EmbeddingCollection of the FM part's tables and first-order weights (shared with the tower's input)."""
        return self._fm.embedding_collection()

    def dense_variables(self):
        """The trainable variables outside the table arena: the FM bias and the tower's kernels and biases.  A tower
        that no call has built yet is built here, as the first call would build it (same shapes, same seeded
        initialisers), so that an optimizer made before the first step holds every variable."""
        coll = self.embedding_collection()
        width = coll.num_slots * coll.dim
        for layer in self._dnn.layers:
            if not layer.built:
                layer.build((None, width), device=coll.weight.device)
            width = layer.units
        return self._fm.dense_variables() + list(self._dnn.parameters())

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        fm_outputs = self._fm(features)
        stack = self._fm._stack
        concat_embeddings = stack.view(stack.shape[0], -1)
        return torch.sigmoid(fm_outputs + self._dnn(concat_embeddings))
