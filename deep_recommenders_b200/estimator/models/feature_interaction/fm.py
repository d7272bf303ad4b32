"""Estimator-side twins: ``fm(x)`` and ``FM(indicator_columns, embedding_columns)(features)``.

Mirrors reference estimator/models/feature_interaction/fm.py:10-26 (fm, rank-3 check :19-20)
and :29-56 (FM: linear + factorized, exposes ``.embeddings`` after the call).  TF1 graph
mode / variable scopes do not exist here: the object owns its EmbeddingCollection and is
called eagerly; the arithmetic is the same fused CUDA kernel the Keras model uses.
"""
from __future__ import annotations

import torch

from .... import ops
from ....embedding import EmbeddingCollection
from ....hashing import ids_and_bags


def fm(x):
    """
    Second order interaction in Factorization Machine
    :param x:
        type: torch.Tensor (CUDA, float32)
        shape: (batch_size, num_features, embedding_dim)
    :return: torch.Tensor (batch_size, 1)
    """
    if x.dim() != 3:
        raise ValueError("The rank of `x` should be 3. Got rank = {}.".format(x.dim()))
    return ops.FMInteraction.apply(x)


class FM(object):
    """
    Factorization Machine
    """

    def __init__(self, indicator_columns, embedding_columns, sparse_lr=None, seed=None, device=None):
        self._indicator_columns = indicator_columns
        self._embedding_columns = embedding_columns
        # estimator fm.py:48-49: slot order is the embedding_columns list order
        self._keys = [c.name.replace("_embedding", "") for c in embedding_columns]
        self._cat = {c.categorical_column.key: c.categorical_column for c in embedding_columns}
        dims = {c.dimension for c in embedding_columns}
        if len(dims) != 1:
            raise ValueError(f"all embedding columns must share one dimension, got {sorted(dims)}")
        self.collection = EmbeddingCollection([self._cat[k].num_buckets for k in self._keys], dims.pop(),
                                              with_linear=True, sparse_lr=sparse_lr, seed=seed, device=device)
        self.embeddings = []

    def parameters(self):
        return self.collection.parameters()

    def embedding_collection(self):
        """The EmbeddingCollection of the tables and first-order weights (what an optimizers.RowSparseAdam trains)."""
        return self.collection

    def dense_variables(self):
        """The trainable variables outside the table arena: the bias of the first-order term."""
        return [self.collection.bias]

    def export(self, path):
        """Write the trained tables to `path` as one torch.save file of CPU tensors, keyed by feature name like the two
        dicts the reference's FNN reads from an FM SavedModel (fnn.py:32-48) -- what ranking.FNN warm-starts from:

            {"format": 1, "bias": [1], "linear": {key: [rows, 1]}, "factorized": {key: [rows, D]}}

        Loadable with torch.load(path, weights_only=True).  The tensors are copies: the file does not share storage
        with the collection's arena."""
        coll = self.collection
        if coll.row_optimizer is not None:     # the rows' pending Adam steps first: the file holds what dense Adam would
            coll.row_optimizer.flush()

        def cpu(t):
            return t.detach().to("cpu", copy=True).contiguous()

        state = {"format": 1, "bias": cpu(coll.bias).reshape(1), "linear": {}, "factorized": {}}
        for s, key in enumerate(self._keys):
            state["linear"][key] = cpu(coll.linear_of(s)).reshape(-1, 1)
            state["factorized"][key] = cpu(coll.table(s))
        torch.save(state, path)

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        ids, bags = ids_and_bags(self._keys, self._cat, features, self.collection.weight.device)
        stack, logit = self.collection(ids, want_logit=True, bags=bags)
        self.embeddings = [stack[:, s, :] for s in range(stack.shape[1])]
        self._stack = stack
        return logit.unsqueeze(1)          # linear_outputs + factorized_outputs
