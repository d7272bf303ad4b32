"""Estimator-side FNN (reference estimator/models/ranking/fnn.py:9-90): ``FNN(indicator_columns, embedding_columns,
warmup_from_fm, dnn_units, ...)(features)`` -> sigmoid(dnn(concat([bias, w_1..w_S, e_1..e_S]), dnn_units + [1])).

The reference loads an FM SavedModel and initialises per-field copies of its first-order weights (the kernels of
`tf.layers.dense(units=1, use_bias=False)` over each indicator column) and of its factorized tables (new embedding
columns) from it; the FM's bias becomes a tiled constant.  Here the warm start reads the file `FM.export` writes, once,
at construction, and copies it into the FNN's own EmbeddingCollection (first-order weights and embeddings of a field
in one row), so training the FNN leaves the exported FM untouched.  The bias is a non-trainable buffer.

The tower input is written by one kernel (ops.FnnInputFn, dr_fnn_input_fwd) in a padded layout: P = round_up(1 + S, 4)
columns [bias | w_1..w_S | 0..], then the S embeddings, ld = P + S*D columns in all.  That is the reference's concat
with up to three zero columns after the scalars, which keeps ld a multiple of 4 for the tensor-core GEMM of layer 0.
Layer 0's kernel has zero rows at the pad columns; their gradient is exactly zero (the input column is), so SGD and
Adam leave them at zero and the model computes the reference's function.
"""
from __future__ import annotations

import torch
from torch import nn

from .... import ops
from ....embedding import EmbeddingCollection
from ....hashing import ids_and_bags
from ..feature_interaction.dnn import DnnTower, relu

EXPORT_FORMAT = 1


def _read_fm_export(path, keys, rows, dim):
    """Load and check an FM.export file against the FNN's columns; returns (bias [1], {key: [rows]}, {key: [rows, D]})."""
    state = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(state, dict) or state.get("format") != EXPORT_FORMAT:
        fmt = state.get("format") if isinstance(state, dict) else type(state).__name__
        raise ValueError(f"{path}: unknown FM export format {fmt!r} (expected {EXPORT_FORMAT})")
    bias = torch.as_tensor(state["bias"], dtype=torch.float32).reshape(-1)
    if bias.numel() != 1:
        raise ValueError(f"{path}: bias has {bias.numel()} elements, expected 1")
    linear, factorized = {}, {}
    for key, n in zip(keys, rows):
        for part in ("linear", "factorized"):
            if key not in state[part]:
                raise ValueError(f"{path}: no {part!r} table for feature {key!r}")
        lin = torch.as_tensor(state["linear"][key], dtype=torch.float32)
        emb = torch.as_tensor(state["factorized"][key], dtype=torch.float32)
        if lin.dim() != 2 or lin.shape[1] != 1 or lin.shape[0] != n:
            raise ValueError(f"{path}: linear[{key!r}] has shape {tuple(lin.shape)}, the column needs ({n}, 1)")
        if emb.dim() != 2 or emb.shape[0] != n:
            raise ValueError(f"{path}: factorized[{key!r}] has {tuple(emb.shape)}, the column has {n} buckets")
        if emb.shape[1] != dim:
            raise ValueError(f"{path}: factorized[{key!r}] has dimension {emb.shape[1]}, the column has {dim}")
        linear[key], factorized[key] = lin[:, 0], emb
    return bias, linear, factorized


class FNN(object):

    def __init__(self,
                 indicator_columns,
                 embedding_columns,
                 warmup_from_fm,
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
        self._warmup_from_fm = warmup_from_fm
        self._dnn_hidden_units = list(dnn_units)
        ind_keys = [c.categorical_column.key for c in self._indicator_columns]
        self._keys = [c.categorical_column.key for c in self._embedding_columns]
        if ind_keys != self._keys:
            raise NotImplementedError(
                f"indicator columns {ind_keys} and embedding columns {self._keys} must name the same categorical "
                "columns in the same order (one slot per field)")
        for c in self._embedding_columns:
            if c.combiner != "mean":
                raise NotImplementedError(f"embedding column {c.name!r}: combiner {c.combiner!r} (mean only)")
        dims = {c.dimension for c in self._embedding_columns}
        if len(dims) != 1:
            raise ValueError(f"all embedding columns must share one dimension, got {sorted(dims)}")
        dim = dims.pop()
        self._cat = {c.categorical_column.key: c.categorical_column for c in self._embedding_columns}
        rows = [self._cat[k].num_buckets for k in self._keys]
        bias, linear, factorized = _read_fm_export(warmup_from_fm, self._keys, rows, dim)

        dev = torch.device(device if device is not None else "cuda")
        self.embeddings = EmbeddingCollection(rows, dim, with_linear=True, init="zeros", device=dev)
        self.embeddings.bias = None           # FNN's bias is the FM's constant below, not a trainable variable
        with torch.no_grad():
            for s, key in enumerate(self._keys):
                off = int(self.embeddings._offsets[s])
                self.embeddings.emb_view()[off:off + rows[s]].copy_(factorized[key])
                self.embeddings.lin_view()[off:off + rows[s]].copy_(linear[key])
        self.bias = bias.to(dev)

        S = len(self._keys)
        P, self.ld = ops.fnn_layout(S, dim)
        self._dnn = DnnTower(self._dnn_hidden_units + [1], activation=dnn_activation, seed=seed, **dnn_kwargs)
        first = self._dnn.layers[0]
        # layer 0 is initialised as tf.layers.dense initialises it over the reference's 1 + S + S*D inputs, then its
        # rows move to the padded layout with zero rows at the pad columns 1+S .. P-1
        first.build((None, 1 + S + S * dim), device=dev)
        k = torch.zeros((self.ld, first.units), dtype=torch.float32, device=dev)
        k[:1 + S] = first.kernel.detach()[:1 + S]
        k[P:] = first.kernel.detach()[1 + S:]
        first.kernel = nn.Parameter(k)
        width = first.units
        for layer in self._dnn.layers[1:]:    # built now so that parameters() is complete before the first call
            layer.build((None, width), device=dev)
            width = layer.units

    def pad_rows(self):
        """The rows of layer 0's kernel at the zero pad columns of the input (empty when 1 + S is a multiple of 4)."""
        S = len(self._keys)
        P, _ = ops.fnn_layout(S, self.embeddings.dim)
        return self._dnn.layers[0].kernel[1 + S:P]

    def parameters(self):
        """Every trainable variable: the embedding arena (with the first-order weights; plus `linear` in the split
        layout) and the tower's kernels and biases."""
        yield self.embeddings.weight
        if self.embeddings.linear is not None:
            yield self.embeddings.linear
        yield from self._dnn.parameters()

    def embedding_collection(self):
        """The EmbeddingCollection of the embeddings and first-order weights warm-started from the FM."""
        return self.embeddings

    def dense_variables(self):
        """The trainable variables outside the table arena: the tower's kernels and biases (the bias is a constant)."""
        return list(self._dnn.parameters())

    def __call__(self, *args, **kwargs):
        return self.call(*args, **kwargs)

    def call(self, features):
        coll = self.embeddings
        ids, bags = ids_and_bags(self._keys, self._cat, features, coll.weight.device)
        dnn_inputs = ops.FnnInputFn.apply(ids, coll.weight, coll.linear, self.bias, coll, bags)
        outputs = self._dnn(dnn_inputs)
        return torch.sigmoid(outputs)
