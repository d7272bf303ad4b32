"""Generates tests/golden/cin_golden.npz by EXECUTING THE REFERENCE'S OWN keras/models/ranking/xdeepfm.py (read from a
checkout of the reference, never copied) under the numpy-backed `tensorflow` stand-in in oracle/tf_shim.  Nothing calls
this script: the .npz file is committed and the tests read only it.  Run it by hand, on any machine (no GPU needed):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_cin_golden.py

The stand-in lacks a few of the ops CIN.call uses (xdeepfm.py:82-96); this script adds them to the imported shim
module for its own process only (TensorFlow's documented semantics, computed in the inputs' dtype), so the shim files
and the other golden vectors are untouched:
  tf.split, batched tf.matmul(..., transpose_b=True) on lists, tf.nn.conv1d (width 1, VALID), tf.nn.bias_add,
  tf.keras.activations.get by name, Layer.add_weight with an initializer, tf.keras.backend.ndim.
It writes only tests/golden/cin_golden.npz: for each dtype (prefix f32_ / f64_) the reference's two known-answer cases
(tests/keras/test_xdeepfm.py:30-60), random cases (m != h, D in {1, 3, 16}, bias on / off, relu / sigmoid / linear,
one with x is x0), the three ValueError messages and the get_config keys.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_cin_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"


def _extend_shim():
    _matmul = tf.matmul

    def matmul(a, b, transpose_a=False, transpose_b=False, name=None):
        a, b = np.asarray(a), np.asarray(b)
        if a.ndim <= 2 and b.ndim <= 2:
            return _matmul(a, b, transpose_a, transpose_b)
        if transpose_a:
            a = np.swapaxes(a, -1, -2)
        if transpose_b:
            b = np.swapaxes(b, -1, -2)
        return tf.convert_to_tensor(np.matmul(a, b))

    def conv1d(x, filters, stride=1, padding="VALID", name=None):
        f = np.asarray(filters)
        assert f.shape[0] == 1 and stride == 1 and padding == "VALID"
        return tf.convert_to_tensor(np.asarray(x) @ f[0])

    acts = {"relu": lambda z: tf.convert_to_tensor(np.maximum(np.asarray(z), 0)),
            "sigmoid": lambda z: tf.convert_to_tensor(1.0 / (1.0 + np.exp(-np.asarray(z)))),
            "linear": lambda z: tf.convert_to_tensor(np.asarray(z))}
    for k, f in acts.items():
        f.__name__ = k

    def add_weight(self, name=None, shape=(), initializer=None, regularizer=None, trainable=True, dtype=None, **k):
        return initializer(tuple(shape))

    tf.matmul = matmul
    tf.split = lambda x, num, axis=0, name=None: [tf.convert_to_tensor(p) for p in np.split(np.asarray(x), num, axis)]
    tf.nn.conv1d = conv1d
    tf.nn.bias_add = lambda x, b, name=None: tf.convert_to_tensor(np.asarray(x) + np.asarray(b))
    tf.keras.activations.get = lambda a: acts[a] if isinstance(a, str) else a
    tf.keras.activations.serialize = lambda a: getattr(a, "__name__", a)
    tf.keras.backend = types.SimpleNamespace(ndim=lambda x: np.ndim(x))
    tf.keras.layers.Layer.add_weight = add_weight


def generate(dtype, out):
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    tf.set_default_dtype(dtype)
    pre = "f32_" if dtype == np.float32 else "f64_"
    rng = np.random.RandomState(11)

    def run(layer, x0, x):
        layer.build((tf.TensorShape(np.shape(x0)), tf.TensorShape(np.shape(x))))
        return np.asarray(layer.call((x0, x)))

    def store(tag, layer, x0, x, act, y):
        out[f"{pre}{tag}_x0"] = np.asarray(x0, dtype)
        out[f"{pre}{tag}_x"] = np.asarray(x, dtype)
        out[f"{pre}{tag}_kernel"] = np.asarray(layer._kernel, dtype)
        if layer._use_bias:
            out[f"{pre}{tag}_bias"] = np.asarray(layer._bias, dtype)
        out[f"{pre}{tag}_act"] = np.asarray(act)
        out[f"{pre}{tag}_y"] = np.asarray(y, dtype)

    # known answers (test_xdeepfm.py:30-60)
    x = np.asarray([[[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]]], dtype)
    for tag, bias in (("known_outputs", False), ("known_bias", True)):
        layer = CIN(feature_map=2, use_bias=bias, activation="relu", kernel_init="ones", bias_init="ones")
        store(tag, layer, x, x, "relu", run(layer, x, x))

    # random cases: (tag, B, m, h, D, H, bias, activation, x is x0)
    for tag, B, m, h, D, H, bias, act, same in [
            ("r_relu_bias_d1", 6, 5, 7, 1, 6, True, "relu", False),
            ("r_sigmoid_d3", 5, 7, 4, 3, 9, False, "sigmoid", False),
            ("r_linear_bias_d16", 4, 4, 6, 16, 5, True, "linear", False),
            ("r_sigmoid_d16", 3, 26, 13, 16, 12, False, "sigmoid", False),
            ("r_relu_same_d3", 6, 3, 3, 3, 4, True, "relu", True)]:
        x0 = rng.standard_normal((B, m, D)).astype(dtype)
        xx = x0 if same else rng.standard_normal((B, h, D)).astype(dtype)
        layer = CIN(feature_map=H, use_bias=bias, activation=act)
        layer.build((tf.TensorShape(x0.shape), tf.TensorShape(xx.shape)))
        layer._kernel = (rng.standard_normal((1, m * h, H)) * 0.3).astype(dtype)
        if bias:
            layer._bias = rng.standard_normal(H).astype(dtype)
        store(tag, layer, x0, xx, act, np.asarray(layer.call((x0, xx))))

    # the three error messages (xdeepfm.py:41-48, :75-80)
    errs = []
    for fn in (lambda: CIN(feature_map=3).build(list(np.shape(np.zeros((2, 3, 5))))),
               lambda: CIN(feature_map=3).build((tf.TensorShape((2, 3, 5)),) * 3),
               lambda: run(CIN(feature_map=3), np.zeros((2, 15), dtype), np.zeros((2, 15), dtype))):
        try:
            fn()
            raise AssertionError("no ValueError")
        except ValueError as e:
            errs.append(str(e))
    out[f"{pre}errors"] = np.asarray(errs)
    out[f"{pre}config_keys"] = np.asarray(sorted(CIN(feature_map=3).get_config()))


if __name__ == "__main__":
    _extend_shim()
    out = {}
    for dt in (np.float32, np.float64):
        generate(dt, out)
    path = os.path.join(HERE, "cin_golden.npz")
    np.savez(path, **out)
    print(f"wrote {path}: {len(out)} arrays")
