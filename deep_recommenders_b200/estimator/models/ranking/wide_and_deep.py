"""Estimator-side Wide & Deep (reference estimator/models/ranking/wide_and_deep.py:9-50):
``WDL(indicator_columns, embedding_columns, dnn_units, dnn_activation=relu, ...)(features)``
-> sigmoid(linear_model(indicator_columns) + dnn(concat(embeddings), dnn_units + [1])).

The reference builds the two halves under the variable scopes "wide" and "deep" and trains them with different
optimizers (FTRL and Adam in examples/train_wdl_on_movielens_estimator.py:63-75).  Here the object owns them:
`wide_variables()` is the LinearTable (weights, bias and FTRL's slots in one arena, updated by ops.FtrlOptimizer),
`deep_variables()` the embedding tables and the tower's kernels and biases.
"""
from __future__ import annotations

import torch

from .... import feature_column as fc
from ....embedding import EmbeddingCollection, LinearTable
from ....hashing import ids_and_bags
from ..feature_interaction.dnn import DnnTower, relu


class WDL(object):

    def __init__(self,
                 indicator_columns,
                 embedding_columns,
                 dnn_units,
                 dnn_activation=relu,
                 dnn_batch_normalization=False,
                 dnn_dropout=None,
                 seed=None, device=None,
                 **dnn_kwargs):
        if dnn_batch_normalization or dnn_dropout is not None:
            raise NotImplementedError("batch normalisation / dropout are not on the accelerated path")
        self._indicator_columns = list(indicator_columns)
        self._embedding_columns = list(embedding_columns)
        self._dnn_hidden_units = list(dnn_units)
        dev = torch.device(device if device is not None else "cuda")
        self.linear = LinearTable([c.categorical_column.num_buckets for c in self._indicator_columns], device=dev)
        # slot order = embedding_columns list order (wide_and_deep.py:36-41 concatenates them in that order)
        self._keys = [c.name.replace("_embedding", "") for c in self._embedding_columns]
        self._cat = {c.categorical_column.key: c.categorical_column for c in self._embedding_columns}
        dims = {c.dimension for c in self._embedding_columns}
        if len(dims) != 1:
            raise ValueError(f"all embedding columns must share one dimension, got {sorted(dims)}")
        for c in self._embedding_columns:
            if c.combiner != "mean":
                raise NotImplementedError(f"embedding column {c.name!r}: combiner {c.combiner!r} (mean only)")
        self.embeddings = EmbeddingCollection([self._cat[k].num_buckets for k in self._keys], dims.pop(),
                                              with_linear=False, seed=seed, device=dev)
        self._dnn = DnnTower(self._dnn_hidden_units + [1], activation=dnn_activation, seed=seed, **dnn_kwargs)
        width = len(self._keys) * self.embeddings.dim
        for layer in self._dnn.layers:      # built now so that deep_variables() is complete before the first call
            layer.build((None, width), device=dev)
            width = layer.units

    def wide_variables(self):
        """What the reference's wide optimizer trains: linear_model's weights and bias (with FTRL's slots)."""
        return [self.linear.state]

    def deep_variables(self):
        """The embedding tables and the tower.  The reference's example collects MODEL_VARIABLES under "deep",
        which holds the feature-column tables but, in TensorFlow's source, not tf.layers.dense's kernels and biases;
        the tower is included here so that the deep optimizer trains it (DESIGN.md section 7)."""
        return [self.embeddings.weight] + list(self._dnn.parameters())

    def embedding_collection(self):
        """The EmbeddingCollection of the deep part's tables (no first-order weights)."""
        return self.embeddings

    def dense_variables(self):
        """The deep variables outside the table arena: the tower's kernels and biases."""
        return list(self._dnn.parameters())

    def parameters(self):
        yield from self.wide_variables()
        yield from self.deep_variables()

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        linear_outputs = fc.linear_model(features, self._indicator_columns, self.linear)
        dev = self.embeddings.weight.device
        ids, bags = ids_and_bags(self._keys, self._cat, features, dev)
        stack, _ = self.embeddings(ids, want_logit=False, bags=bags)
        concat_embeddings = stack.reshape(stack.shape[0], -1)
        dnn_outputs = self._dnn(concat_embeddings)
        return torch.sigmoid(linear_outputs + dnn_outputs)
