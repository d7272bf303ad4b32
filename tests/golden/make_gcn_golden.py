"""Generates tests/golden/gcn_golden.npz and the small Cora-format fixture tests/golden/cora_small/cora/ by EXECUTING THE
REFERENCE'S OWN keras/models/retrieval/gcn.py and datasets/cora.py (read from a checkout of the reference, never
copied) under the numpy-backed `tensorflow` stand-in in oracle/tf_shim.  Nothing calls this script: the files are
committed and the tests read only them.  Run it by hand, on any machine (no GPU):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_gcn_golden.py

The stand-in lacks a few of the names these files use; this script adds them to the imported shim module for its own
process only (TensorFlow's documented semantics, computed in the inputs' dtype), so the shim files and the other golden
vectors are untouched: tf.SparseTensor (indices [nnz, 2], values, dense_shape), tf.sparse.sparse_dense_matmul
(duplicates summed), tf.linalg.matmul, the "softmax" activation of tf.keras.layers.Dense (max subtracted), and the
np.str / np.bool aliases that current numpy no longer has.  Dense draws its kernel from N(0, 0.5^2) and, so that the
biases are exercised, its bias from N(0, 0.1^2).
It writes:
  tests/golden/cora_small/cora/cora.{content,cites}: write_synthetic_cora(seed 5, 210 papers, 60 words, 420
      citations), at least 20 papers per class, plus the reverse of the first citation (a citation in both directions)
      and a self-citation;
  tests/golden/gcn_golden.npz: for each dtype (prefix f32_ / f64_) layer_<case>_{x, adj (dense), rows, cols, vals
      (the COO entries handed to tf.SparseTensor, duplicates included), w, b, out, args}; and (unprefixed) cora_* :
      every loader method's outputs on the fixture after np.random.seed(CORA_SEED), in the order the tests replay.
"""
import os
import shutil
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_gcn_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, ROOT)
from deep_recommenders_b200.datasets.cora import CORA_CLASSES, write_synthetic_cora  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"

RNG = np.random.RandomState(41)
CORA_SEED = 7
FIXTURE = os.path.join(HERE, "cora_small")

# tag, n_out, n_in, F, units, activation, use_bias, residual, sparse, empty rows, duplicate entries
LAYER_CASES = [
    ("ref_sparse", 3, 3, 4, 2, "relu", False, False, True, 0, 0),      # tests/keras/test_gcn.py:19-45
    ("ref_dense", 3, 3, 4, 2, "relu", False, False, False, 0, 0),      # tests/keras/test_gcn.py:47-69
    ("wide_relu_b", 40, 40, 33, 7, "relu", True, False, True, 3, 4),   # F > units
    ("wide_softmax_b", 40, 40, 33, 7, "softmax", True, False, True, 2, 0),
    ("wide_tanh", 30, 30, 17, 5, "tanh", False, False, False, 2, 0),
    ("narrow_sigmoid_b", 40, 40, 5, 12, "sigmoid", True, False, True, 3, 3),   # F < units
    ("narrow_linear", 25, 25, 3, 8, None, False, False, True, 1, 0),
    ("narrow_softmax", 25, 25, 4, 6, "softmax", False, False, False, 0, 0),
    ("tie_residual_b", 30, 30, 9, 9, "relu", True, True, True, 2, 2),       # F == units: the reference's order
    ("tie_residual_tanh", 20, 20, 6, 6, "tanh", False, True, False, 1, 0),
    ("rect_relu_b", 17, 29, 10, 4, "relu", True, False, True, 2, 0),       # rectangular adj
]


def _extend_shim():
    class SparseTensor:
        def __init__(self, indices, values, dense_shape):
            self.indices = np.asarray(indices, np.int64).reshape(-1, 2)
            self.values = np.asarray(values)
            self.dense_shape = tuple(int(d) for d in dense_shape)

    def sparse_dense_matmul(sp_a, b, name=None):
        b = np.asarray(b)
        dense = np.zeros(sp_a.dense_shape, b.dtype)
        np.add.at(dense, (sp_a.indices[:, 0], sp_a.indices[:, 1]), sp_a.values.astype(b.dtype))
        return tf.convert_to_tensor(dense @ b)

    base_call = tf.keras.layers.Dense.call

    def dense_call(self, x):
        if getattr(self.activation, "__name__", self.activation) != "softmax":
            return base_call(self, x)
        x = np.asarray(x)
        z = x @ self.kernel.astype(x.dtype)
        if self.bias is not None:
            z = z + self.bias.astype(x.dtype)
        e = np.exp(z - z.max(axis=-1, keepdims=True))
        return tf.convert_to_tensor(e / e.sum(axis=-1, keepdims=True))

    def dense_build(self, input_shape):
        dt = tf.DEFAULT_DTYPE[0]
        self.kernel = (RNG.standard_normal((int(input_shape[-1]), self.units)) * 0.5).astype(dt)
        self.bias = (RNG.standard_normal(self.units) * 0.1).astype(dt) if self.use_bias else None
        self.built = True

    tf.SparseTensor = SparseTensor
    tf.sparse = types.SimpleNamespace(sparse_dense_matmul=sparse_dense_matmul)
    tf.linalg = types.SimpleNamespace(matmul=lambda a, b, name=None: tf.convert_to_tensor(np.asarray(a) @ np.asarray(b)))
    tf.keras.layers.Dense.call = dense_call
    tf.keras.layers.Dense.build = dense_build
    np.str = str
    np.bool = bool


def _adjacency(rng, n_out, n_in, empty, dups, dtype):
    a = (rng.random((n_out, n_in)) < 0.2) * rng.uniform(0.1, 1.0, (n_out, n_in))
    if empty:
        a[rng.choice(n_out, empty, replace=False)] = 0
    rows, cols = np.nonzero(a)
    vals = a[rows, cols]
    if dups:                      # repeat some entries with other values: TensorFlow sums them
        k = rng.choice(len(rows), dups, replace=False)
        rows, cols = np.concatenate([rows, rows[k]]), np.concatenate([cols, cols[k]])
        vals = np.concatenate([vals, rng.uniform(0.1, 1.0, dups)])
    dense = np.zeros((n_out, n_in))
    np.add.at(dense, (rows, cols), vals)
    return dense.astype(dtype), rows, cols, vals.astype(dtype)


def generate_layers(dtype, out):
    from deep_recommenders.keras.models.retrieval.gcn import GCN
    tf.set_default_dtype(dtype)
    pre = "f32_" if dtype == np.float32 else "f64_"
    rng = np.random.default_rng(43)
    for tag, n_out, n_in, F, units, act, bias, res, sparse, empty, dups in LAYER_CASES:
        k = f"{pre}layer_{tag}"
        if tag.startswith("ref_"):
            dense = np.asarray([[0, 1, 0], [1, 0, 0], [0, 1, 1]], dtype)
            rows, cols = np.nonzero(dense)
            vals = dense[rows, cols]
            x = np.asarray([[0.1, 0.2, 0.3, 0.0], [0.4, 0.5, 0.6, 0.0], [0.7, 0.8, 0.9, 0.0]], dtype)
        else:
            dense, rows, cols, vals = _adjacency(rng, n_out, n_in, empty, dups, dtype)
            x = rng.standard_normal((n_in, F)).astype(dtype)
        layer = GCN(units, residual=res, use_bias=bias, activation=act if act else None)
        adj = tf.SparseTensor(np.stack([rows, cols], 1), vals, dense.shape) if sparse else dense
        y = layer(x, adj)
        out[k + "_x"], out[k + "_adj"] = x, dense
        out[k + "_rows"], out[k + "_cols"], out[k + "_vals"] = rows.astype(np.int64), cols.astype(np.int64), vals
        out[k + "_w"] = np.asarray(layer._kernel.kernel, dtype)
        out[k + "_b"] = np.asarray(layer._kernel.bias if bias else np.zeros(units), dtype)
        out[k + "_out"] = np.asarray(y, dtype)
        out[k + "_args"] = np.asarray([units, int(bias), int(res), int(sparse)])
        out[k + "_act"] = np.asarray(act or "linear")


def write_fixture():
    shutil.rmtree(FIXTURE, ignore_errors=True)
    write_synthetic_cora(FIXTURE, seed=5, num_papers=210, num_words=60, num_cites=420)
    content = os.path.join(FIXTURE, "cora", "cora.content")
    labels = [line.split("\t")[-1].strip() for line in open(content)]
    counts = [labels.count(c) for c in CORA_CLASSES]
    assert min(counts) >= 20, counts
    cites = os.path.join(FIXTURE, "cora", "cora.cites")
    first = open(cites).readline().split()
    with open(cites, "a") as f:
        f.write(f"{first[1]}\t{first[0]}\n")                 # the first citation, reversed: both directions
        f.write(f"{first[0]}\t{first[0]}\n")                 # a self-citation


def generate_cora(out):
    from deep_recommenders.datasets.cora import Cora
    np.random.seed(CORA_SEED)
    cora = Cora(FIXTURE)
    ids, features, labels = cora.load_content()
    _, raw, _ = cora.load_content(normalize=False)
    graph = cora.build_graph(ids)
    sg = cora.spectral_graph(graph)
    train_nodes = cora.sample_train_nodes(labels)
    (trl, trm), (val, vam), (tel, tem) = cora.split_labels(labels, num_valid_nodes=50)
    out["cora_seed"] = np.asarray(CORA_SEED)
    out["cora_num_classes"] = np.asarray(cora.num_classes)
    out["cora_ids"], out["cora_labels"] = ids, labels
    out["cora_features"], out["cora_features_raw"] = features.toarray(), raw.toarray()
    out["cora_graph"] = graph.toarray()
    out["cora_spectral_indptr"], out["cora_spectral_indices"] = sg.indptr, sg.indices
    out["cora_spectral_data"] = sg.data
    out["cora_train_nodes"] = np.asarray(train_nodes)
    out["cora_encoded"] = cora.encode_labels(labels)
    for name, arr in (("train_labels", trl), ("train_mask", trm), ("valid_labels", val), ("valid_mask", vam),
                      ("test_labels", tel), ("test_mask", tem)):
        out["cora_" + name] = arr
    out["cora_valid_order"] = np.flatnonzero(vam)                       # set order is kept in the labels' rows only
    all_index = np.arange(labels.shape[0])
    np.random.seed(CORA_SEED + 1)
    train_again = cora.sample_train_nodes(labels)
    out["cora_split_rest_order"] = np.asarray(list(set(all_index) - set(train_again)))
    out["cora_split_rest_seed"] = np.asarray(CORA_SEED + 1)


if __name__ == "__main__":
    _extend_shim()
    out = {}
    for dt in (np.float32, np.float64):
        generate_layers(dt, out)
    write_fixture()
    generate_cora(out)
    path = os.path.join(HERE, "gcn_golden.npz")
    np.savez(path, **out)
    print(f"wrote {path}: {len(out)} arrays")
