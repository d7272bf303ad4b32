"""Generates tests/golden/mtl_golden.npz by EXECUTING THE REFERENCE'S OWN estimator/models/multi_task_learning/
{mixture_of_experts,esmm}.py, estimator/models/feature_interaction/dnn.py and datasets/synthetic_for_multi_task.py (read
from a checkout of the reference, never copied) under the numpy-backed `tensorflow` stand-in in oracle/tf_shim.  Nothing
calls this script: the .npz file is committed and the tests read only it.  Run it by hand, on any machine (no GPU):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_mtl_golden.py

The stand-in lacks a few of the ops these files use; this script adds them to the imported shim module for its own
process only (TensorFlow's documented semantics, computed in the inputs' dtype), so the shim files and the other golden
vectors are untouched: tf.feature_column.numeric_column, tf.nn.softmax (max subtracted), tf.linalg.matmul, tf.squeeze,
tf.math.multiply, and a tf.layers.dense that honours use_bias and records every layer it creates.  That Dense draws
its kernel glorot-uniform and, so that the biases are exercised, its bias from N(0, 0.1) (TensorFlow's default bias
is zeros).
It writes only tests/golden/mtl_golden.npz: for each dtype (prefix f32_ / f64_)
  mmoe_<case>_*   x [B, D] (column i is feature "C{i}"), the model's arguments, every dense layer's kernel and bias in
                  creation order (w{i}, b{i}; the gates have no bias, the unused gates are included) and out{t};
  esmm_<case>_*   the same for ESMM with p_cvr, p_ctr, p_ctcvr;
and (unprefixed) syn_<case>_{x,y1,y2} with the seed and arguments: synthetic_data under np.random.seed(seed).
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_mtl_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"

LAYERS = []
RNG = np.random.RandomState(29)


def _extend_shim():
    class Numeric:
        def __init__(self, key, shape=(1,), dtype=None):
            self.key = self.name = key
            self.shape = tuple(shape) if isinstance(shape, (tuple, list)) else (int(shape),)

        def _dense(self, features):
            v = np.asarray(features[self.key])
            return v.reshape(v.shape[0], -1).astype(tf.DEFAULT_DTYPE[0])

    class RecordedDense(tf.keras.layers.Dense):
        def build(self, input_shape):
            dt = tf.DEFAULT_DTYPE[0]
            fan_in = int(input_shape[-1])
            lim = np.sqrt(6.0 / (fan_in + self.units))
            self.kernel = RNG.uniform(-lim, lim, size=(fan_in, self.units)).astype(dt)
            self.bias = (RNG.standard_normal(self.units) * 0.1).astype(dt) if self.use_bias else None
            self.built = True

    def dense(x, units, activation=None, use_bias=True, **k):
        layer = RecordedDense(units, activation=activation, use_bias=use_bias)
        LAYERS.append(layer)
        return layer(x)

    def softmax(x, axis=-1, name=None):
        x = np.asarray(x)
        e = np.exp(x - x.max(axis=axis, keepdims=True))
        return tf.convert_to_tensor(e / e.sum(axis=axis, keepdims=True))

    tf.feature_column.numeric_column = Numeric
    tf.layers.dense = dense
    tf.nn.softmax = softmax
    tf.linalg = types.SimpleNamespace(matmul=lambda a, b, name=None: tf.convert_to_tensor(np.matmul(np.asarray(a),
                                                                                                     np.asarray(b))))
    tf.squeeze = lambda x, axis=None, name=None: tf.convert_to_tensor(np.squeeze(np.asarray(x), axis=axis))
    tf.math.multiply = lambda x, y, name=None: tf.convert_to_tensor(np.asarray(x) * np.asarray(y))


MMOE_CASES = [
    # tag, B, D, num_tasks, num_experts, expert units, task units, expert act, task act
    ("ref", 16, 100, 2, 2, [64, 32], [32, 10], "relu", "relu"),          # tests/estimator/test_mixture_of_experts.py
    ("e3t2", 9, 7, 2, 3, [8, 5], [4], "relu", "relu"),                   # E > T: one dead gate
    ("e1t1", 6, 5, 1, 1, [6], [3, 2], "relu", "relu"),                   # E = 1: the gate is exactly 1
    ("e4t1", 11, 12, 1, 4, [10, 10], [], "tanh", "relu"),                # T = 1, a tower of one linear layer
    ("e5t3", 7, 13, 3, 5, [9, 7, 5], [6], "sigmoid", "tanh"),
]
ESMM_CASES = [
    ("ref", 16, 100, [32, 10], "relu"),                                  # tests/estimator/test_esmm.py
    ("small", 5, 6, [4], "tanh"),
    ("linear", 4, 3, [], "relu"),
]
SYN_CASES = [("s0", 0, 64, 100, 0.3, 0.8, 5), ("s3", 3, 40, 17, 0.5, -0.2, 2), ("s11", 11, 33, 256, 0.3, 0.8, 5)]


def generate(dtype, out):
    from deep_recommenders.estimator.models.multi_task_learning import MMoE, ESMM
    tf.set_default_dtype(dtype)
    pre = "f32_" if dtype == np.float32 else "f64_"
    rng = np.random.RandomState(31)

    def record(k, x, first):
        out[k + "_x"] = np.asarray(x, dtype)
        layers = LAYERS[first:]
        out[k + "_nlayers"] = np.asarray(len(layers))
        for i, l in enumerate(layers):
            out[f"{k}_w{i}"] = np.asarray(l.kernel, dtype)
            if l.bias is not None:
                out[f"{k}_b{i}"] = np.asarray(l.bias, dtype)

    for tag, B, D, T, E, eu, tu, eact, tact in MMOE_CASES:
        x = rng.standard_normal((B, D)).astype(dtype)
        cols = [tf.feature_column.numeric_column("C{}".format(i)) for i in range(D)]
        features = {"C{}".format(i): x[:, i:i + 1] for i in range(D)}
        first = len(LAYERS)
        outs = MMoE(cols, num_tasks=T, num_experts=E, expert_hidden_units=eu, task_hidden_units=tu,
                    expert_hidden_activation=eact, task_hidden_activation=tact)(features)
        k = f"{pre}mmoe_{tag}"
        record(k, x, first)
        out[k + "_args"] = np.asarray([T, E])
        out[k + "_expert_units"], out[k + "_task_units"] = np.asarray(eu, np.int64), np.asarray(tu, np.int64)
        out[k + "_acts"] = np.asarray([eact, tact])
        for t, o in enumerate(outs):
            out[f"{k}_out{t}"] = np.asarray(o, dtype)

    for tag, B, D, hu, act in ESMM_CASES:
        x = rng.standard_normal((B, D)).astype(dtype)
        cols = [tf.feature_column.numeric_column("C{}".format(i)) for i in range(D)]
        features = {"C{}".format(i): x[:, i:i + 1] for i in range(D)}
        first = len(LAYERS)
        p_cvr, p_ctr, p_ctcvr = ESMM(cols, hidden_units=hu, activation=act)(features)
        k = f"{pre}esmm_{tag}"
        record(k, x, first)
        out[k + "_hidden_units"], out[k + "_act"] = np.asarray(hu, np.int64), np.asarray(act)
        out[k + "_p_cvr"], out[k + "_p_ctr"], out[k + "_p_ctcvr"] = (np.asarray(p, dtype) for p in (p_cvr, p_ctr, p_ctcvr))


def generate_synthetic(out):
    from deep_recommenders.datasets.synthetic_for_multi_task import synthetic_data
    for tag, seed, n, dim, c, p, m in SYN_CASES:
        np.random.seed(seed)
        x, (y1, y2) = synthetic_data(n, dim, c=c, p=p, m=m)
        k = f"syn_{tag}"
        out[k + "_args"] = np.asarray([seed, n, dim, c, p, m], np.float64)
        out[k + "_x"], out[k + "_y1"], out[k + "_y2"] = x, y1, y2


if __name__ == "__main__":
    _extend_shim()
    out = {}
    for dt in (np.float32, np.float64):
        generate(dt, out)
    generate_synthetic(out)
    path = os.path.join(HERE, "mtl_golden.npz")
    np.savez(path, **out)
    print(f"wrote {path}: {len(out)} arrays")
