"""Generates tests/golden/din_golden.npz by EXECUTING THE REFERENCE'S OWN keras/models/ranking/din.py (read from a
checkout of the reference, never copied) under the numpy-backed `tensorflow` stand-in in oracle/tf_shim.  Nothing calls
this script: the .npz file is committed and the tests read only it.  Run it by hand, on any machine (no GPU needed):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_din_golden.py

The stand-in lacks a few of the ops din.py uses (:59-71, :104-121); this script adds them to the imported shim module
for its own process only (TensorFlow's documented semantics, computed in the inputs' dtype), so the shim files and the
other golden vectors are untouched:
  tf.keras.layers.PReLU (alpha of shape input_shape[1:]), tf.math.reduce_mean / reduce_std (population), tf.sqrt,
  tf.nn.sigmoid on tensors, tf.keras.layers.Subtract / Multiply, a Dense whose activation is a Layer (called on the
  pre-activation), initializer objects and names in tf.keras.initializers.serialize, tf.keras.activations.serialize.
It writes only tests/golden/din_golden.npz: for each dtype (prefix f32_ / f64_)
  au_*    ActivationUnit cases: the reference's two known answers (tests/keras/test_din.py:17-48) and random cases over
          no interacter / Subtract / Multiply, relu / sigmoid / linear / a Dice activation, bias on / off, D = 5;
  dice_*  Dice cases: the reference's known answer for each epsilon of test_dice (test_din.py:50-64) and random
          inputs with nonzero (also negative) alpha and a constant row;
  au_config_keys, dice_config_keys.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_din_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"


def _extend_shim():
    Layer = tf.keras.layers.Layer
    init_get, init_serialize = tf.keras.initializers.get, tf.keras.initializers.serialize

    class PReLU(Layer):
        def __init__(self, alpha_initializer="zeros", alpha_regularizer=None, **kwargs):
            super().__init__(**kwargs)
            self._init = init_get(alpha_initializer)
            self.alpha = None

        def build(self, input_shape):
            self.alpha = self._init(tuple(int(s) for s in input_shape[1:]))
            self.built = True

        def call(self, x):
            x = np.asarray(x)
            a = np.asarray(self.alpha).astype(x.dtype)
            return tf.convert_to_tensor(np.maximum(x, 0) - a * np.maximum(-x, 0))

    class Subtract(Layer):
        def call(self, inputs):
            return tf.convert_to_tensor(np.asarray(inputs[0]) - np.asarray(inputs[1]))

    class Multiply(Layer):
        def call(self, inputs):
            return tf.convert_to_tensor(np.asarray(inputs[0]) * np.asarray(inputs[1]))

    dense_call = tf.keras.layers.Dense.call

    def call(self, x):
        act = self.activation
        if isinstance(act, Layer):
            self.activation = None
            try:
                z = dense_call(self, x)
            finally:
                self.activation = act
            return act(z)
        return dense_call(self, x)

    tf.keras.layers.Dense.call = call
    tf.keras.layers.PReLU = PReLU
    tf.keras.layers.Subtract = Subtract
    tf.keras.layers.Multiply = Multiply
    tf.math.reduce_mean = lambda x, axis=None, keepdims=False, name=None: tf.convert_to_tensor(
        np.mean(np.asarray(x), axis=axis, keepdims=keepdims))
    tf.math.reduce_std = lambda x, axis=None, keepdims=False, name=None: tf.convert_to_tensor(
        np.std(np.asarray(x), axis=axis, keepdims=keepdims))
    tf.sqrt = lambda x, name=None: tf.convert_to_tensor(np.sqrt(np.asarray(x)))
    tf.keras.initializers.serialize = lambda i: init_serialize(init_get(i))
    tf.keras.activations.serialize = lambda a: getattr(a, "__name__", a)


def generate(dtype, out):
    from deep_recommenders.keras.models.ranking import din
    tf.set_default_dtype(dtype)
    pre = "f32_" if dtype == np.float32 else "f64_"
    rng = np.random.RandomState(13)

    def unit_case(tag, unit, x, y, inter, act, bias, randomise):
        unit(x, y)                                      # builds the two Dense layers (and a Dice's PReLU)
        if randomise:
            dk, do = unit.dense_kernel, unit.dense_output
            dk.kernel = (rng.standard_normal(dk.kernel.shape) * 0.4).astype(dtype)
            do.kernel = (rng.standard_normal(do.kernel.shape) * 0.4).astype(dtype)
            if bias:
                dk.bias = rng.standard_normal(dk.bias.shape).astype(dtype)
                do.bias = rng.standard_normal(do.bias.shape).astype(dtype)
            if act == "dice":
                unit._kernel_activation.prelu.alpha = (rng.standard_normal(dk.units) * 0.5).astype(dtype)
        res = np.asarray(unit(x, y))
        k = f"{pre}au_{tag}"
        out[k + "_x"], out[k + "_y"] = np.asarray(x, dtype), np.asarray(y, dtype)
        out[k + "_w1"] = np.asarray(unit.dense_kernel.kernel, dtype)
        out[k + "_w2"] = np.asarray(unit.dense_output.kernel, dtype)
        if bias:
            out[k + "_b1"] = np.asarray(unit.dense_kernel.bias, dtype)
            out[k + "_b2"] = np.asarray(unit.dense_output.bias, dtype)
        if act == "dice":
            out[k + "_alpha"] = np.asarray(unit._kernel_activation.prelu.alpha, dtype)
        out[k + "_inter"], out[k + "_act"], out[k + "_bias"] = np.asarray(inter), np.asarray(act), np.asarray(bias)
        out[k + "_out"] = np.asarray(res, dtype)

    # known answers (test_din.py:17-48): kernel_init="ones", relu, bias zeros
    x, y = rng.normal(size=(3, 5)).astype(dtype), rng.normal(size=(3, 5)).astype(dtype)
    unit_case("known_noint", din.ActivationUnit(10, kernel_init="ones"), x, y, "none", "relu", True, False)
    unit_case("known_sub", din.ActivationUnit(10, interacter=tf.keras.layers.Subtract(), kernel_init="ones"), x, y,
              "subtract", "relu", True, False)
    # random cases: (tag, N, D, U, interacter, activation, bias)
    inters = {"none": lambda: None, "subtract": tf.keras.layers.Subtract, "multiply": tf.keras.layers.Multiply}
    for tag, N, D, U, inter, act, bias in [
            ("r_none_relu_d5", 7, 5, 9, "none", "relu", True),
            ("r_sub_sigmoid_d5", 6, 5, 12, "subtract", "sigmoid", False),
            ("r_mul_linear_d8", 5, 8, 6, "multiply", "linear", True),
            ("r_sub_relu_nobias_d16", 9, 16, 36, "subtract", "relu", False),
            ("r_mul_sigmoid_d3", 4, 3, 17, "multiply", "sigmoid", True),
            ("r_sub_dice_d5", 8, 5, 10, "subtract", "dice", True),
            ("r_none_dice_nobias_d4", 6, 4, 7, "none", "dice", False)]:
        x = rng.standard_normal((N, D)).astype(dtype)
        y = rng.standard_normal((N, D)).astype(dtype)
        activation = din.Dice() if act == "dice" else act
        unit = din.ActivationUnit(U, interacter=inters[inter](), use_bias=bias, activation=activation)
        unit_case(tag, unit, x, y, inter, act, bias, True)

    def dice_case(tag, x, eps, alpha=None):
        layer = din.Dice(epsilon=eps)
        layer(x)
        if alpha is not None:
            layer.prelu.alpha = np.asarray(alpha, dtype)
        res = np.asarray(layer(x))
        k = f"{pre}dice_{tag}"
        out[k + "_x"] = np.asarray(x, dtype)
        out[k + "_alpha"] = np.asarray(layer.prelu.alpha, dtype)
        out[k + "_eps"] = np.asarray(eps)
        out[k + "_y"] = np.asarray(res, dtype)

    # known answers (test_din.py:50-64)
    inputs = np.asarray([[-0.2, -0.1, 0.1, 0.2]]).astype(dtype)
    for i, eps in enumerate((1e-7, 1e-8, 1e-9, 1e-10)):
        dice_case(f"known_eps{i}", inputs, eps)
    x = rng.standard_normal((9, 13)).astype(dtype)
    x[2] = 0.75                                          # a constant row
    x[5, :6] = 0.0
    dice_case("r_alpha", x, 1e-8, rng.standard_normal(13) * 0.6)
    dice_case("r_alpha_eps3", rng.standard_normal((5, 40)).astype(dtype) * 3, 1e-3, -np.abs(rng.standard_normal(40)))
    dice_case("r_u1", rng.standard_normal((4, 1)).astype(dtype), 1e-8, [-0.3])

    out[f"{pre}au_config_keys"] = np.asarray(sorted(din.ActivationUnit(4).get_config()))
    out[f"{pre}dice_config_keys"] = np.asarray(sorted(din.Dice().get_config()))


if __name__ == "__main__":
    _extend_shim()
    out = {}
    for dt in (np.float32, np.float64):
        generate(dt, out)
    path = os.path.join(HERE, "din_golden.npz")
    np.savez(path, **out)
    print(f"wrote {path}: {len(out)} arrays")
