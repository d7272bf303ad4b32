"""Generates tests/golden/fnn_golden.npz by EXECUTING THE REFERENCE'S OWN estimator/models/ranking/fnn.py and
estimator/models/feature_interaction/dnn.py (read from a checkout of the reference, never copied) under the
numpy-backed `tensorflow` stand-in in oracle/tf_shim, in float64.  Nothing calls this script: the .npz file is
committed and the tests read only it.  Run it by hand, on any machine (no GPU):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_fnn_golden.py

The stand-in lacks what FNN's warm start uses; this script adds it to the imported shim module for its own process
only, so the shim files and the other golden vectors are untouched:
  * tf.Session (a context manager whose run() returns a stand-in variable's value) and a no-op
    tf.saved_model.load: the "SavedModel" is the seeded FM variables of this script;
  * tf.get_collection(MODEL_VARIABLES, "linear" | "factorized"), returning stand-in variables named as TensorFlow's
    linear_model and input_layer name them (linear/linear_model/<key>_indicator/weights:0,
    linear/linear_model/bias_weights:0, factorized/input_layer/<key>_embedding/embedding_weights:0), so that the
    reference's name parsing (fnn.py:36-46) runs;
  * tf.constant_initializer, embedding_column(initializer=...) that takes its table from it, and a tf.layers.dense
    that honours use_bias and kernel_initializer, records every tower layer and draws the tower's biases from
    N(0, 0.1) so that they are exercised (TensorFlow's default bias is zeros);
  * a named tf.nn.relu (the shim's is a lambda, which its Dense cannot name).
Per case c{k}_: B, S, D, rows{s}, ids{s} (one id per example; -1 is out of vocabulary), the FM variables
table{s} [rows, D], lin{s} [rows] and bias, the tower's kernels k{i} (layer 0 over the reference's 1 + S + S*D
inputs) and biases b{i}, the tower input `x` and the model output `out`.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_fnn_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, ROOT)
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"

LAYERS = []
INPUTS = []
RNG = np.random.RandomState(31)
FM_VARS = {}          # scope -> [stand-in variable]: what the "SavedModel" holds


class Var:
    def __init__(self, name, value):
        self.name = name
        self.value = np.asarray(value, dtype=np.float64)


def _extend_shim():
    class Session:
        def __init__(self, graph=None, **k):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def run(self, var):
            return var.value.copy()

    class Constant:
        def __init__(self, value):
            self.value = np.asarray(value, dtype=np.float64)

    class Embedding(tf._Embedding):
        """embedding_column(initializer=constant_initializer(table)).  The columns handed to FNN are only read for
        their categorical column and dimension (fnn.py:70-75): without an initializer the table is zeros."""

        def __init__(self, cat, dimension, initializer=None, **k):
            self.categorical_column = cat
            self.dimension = dimension
            self.name = cat.key + "_embedding"
            self.table = (np.zeros((cat.num_buckets, dimension)) if initializer is None
                          else initializer.value.reshape(cat.num_buckets, dimension))

    class RecordedDense(tf.keras.layers.Dense):
        def __init__(self, units, activation=None, use_bias=True, kernel_initializer=None):
            super().__init__(units, activation=activation, use_bias=use_bias)
            self._const = kernel_initializer

        def build(self, input_shape):
            fan_in = int(input_shape[-1])
            if self._const is not None:
                self.kernel = self._const.value.reshape(fan_in, self.units)
            else:
                lim = np.sqrt(6.0 / (fan_in + self.units))
                self.kernel = RNG.uniform(-lim, lim, size=(fan_in, self.units))
            self.bias = RNG.standard_normal(self.units) * 0.1 if self.use_bias else None
            self.built = True

    def dense(x, units, activation=None, use_bias=True, kernel_initializer=None, **k):
        layer = RecordedDense(units, activation=activation, use_bias=use_bias, kernel_initializer=kernel_initializer)
        if kernel_initializer is None:       # a tower layer (the per-field weights come with their initializer)
            LAYERS.append(layer)
            if len(LAYERS) == 1:
                INPUTS.append(np.asarray(x))
        return layer(x)

    def relu(x, name=None):
        return tf.convert_to_tensor(np.maximum(np.asarray(x), 0))

    tf.Session = Session
    tf.Graph = lambda: None
    tf.saved_model = type("saved_model", (), {"load": staticmethod(lambda sess, tags, path: None)})
    tf.get_collection = lambda key, scope=None: list(FM_VARS.get(scope, []))
    tf.constant_initializer = Constant
    tf.feature_column.embedding_column = Embedding
    tf.layers.dense = dense
    tf.nn.relu = relu


CASES = [
    # tag, B, D, units, rows per field (the reference example's six fields at D = 16, [64, 32]; a small odd case)
    ("ex", 12, 16, [64, 32], [30, 2, 7, 21, 40, 2]),
    ("small", 7, 8, [5], [5, 3, 9, 4, 6]),
]


def main():
    tf.set_default_dtype(np.float64)
    _extend_shim()
    from deep_recommenders.estimator.models.ranking.fnn import FNN
    out = {"n_cases": np.asarray(len(CASES))}
    rng = np.random.RandomState(41)
    for k, (tag, B, D, units, rows) in enumerate(CASES):
        p = f"c{k}_"
        fc = tf.feature_column
        keys = [f"f{s}" for s in range(len(rows))]
        cats = [fc.categorical_column_with_identity(key, n) for key, n in zip(keys, rows)]
        indicators = [fc.indicator_column(c) for c in cats]
        embeddings = [fc.embedding_column(c, D) for c in cats]
        tables = [rng.normal(0, 0.3, (n, D)) for n in rows]
        lins = [rng.normal(0, 0.3, (n, 1)) for n in rows]
        bias = rng.normal(0, 0.3, (1,))
        FM_VARS["linear"] = ([Var(f"linear/linear_model/{key}_indicator/weights:0", w) for key, w in zip(keys, lins)]
                             + [Var("linear/linear_model/bias_weights:0", bias)])
        FM_VARS["factorized"] = [Var(f"factorized/input_layer/{key}_embedding/embedding_weights:0", t)
                                 for key, t in zip(keys, tables)]
        features = {key: rng.randint(-1, n, B) for key, n in zip(keys, rows)}
        del LAYERS[:]
        del INPUTS[:]
        prob = np.asarray(FNN(indicators, embeddings, "FM", units)(features))
        out[p + "B"], out[p + "S"], out[p + "D"] = np.asarray(B), np.asarray(len(rows)), np.asarray(D)
        for s, key in enumerate(keys):
            out[f"{p}rows{s}"] = np.asarray(rows[s])
            out[f"{p}ids{s}"] = features[key].astype(np.int64)
            out[f"{p}table{s}"] = tables[s]
            out[f"{p}lin{s}"] = lins[s][:, 0]
        out[p + "bias"] = bias
        out[p + "nlayers"] = np.asarray(len(LAYERS))
        for i, l in enumerate(LAYERS):
            out[f"{p}k{i}"], out[f"{p}b{i}"] = l.kernel, l.bias
        out[p + "x"] = INPUTS[0]
        out[p + "out"] = prob
    np.savez_compressed(os.path.join(HERE, "fnn_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "fnn_golden.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
