"""Generates tests/golden/wdl_golden.npz by EXECUTING THE REFERENCE'S OWN estimator/models/ranking/wide_and_deep.py and
estimator/models/feature_interaction/dnn.py (read from a checkout of the reference, never copied) under the
numpy-backed `tensorflow` stand-in in oracle/tf_shim, in float64.  Nothing calls this script: the .npz file is
committed and the tests read only it.  Run it by hand, on any machine (no GPU):

    DR_REFERENCE=<checkout of LongmaoTeamTf/deep_recommenders> python tests/golden/make_wdl_golden.py

The stand-in lacks a few things these files use; this script adds them to the imported shim module for its own
process only, so the shim files and the other golden vectors are untouched:
  * tf.feature_column.crossed_column over raw keys (ids from tests/wdl_oracle.py's restatement of TensorFlow's
    HashCrosser), and indicator columns over it that linear_model accepts;
  * a named tf.nn.relu (the shim's is a lambda, which its Dense cannot name);
  * a tf.layers.dense that records every layer it creates and draws its bias from N(0, 0.1) so that the biases are
    exercised (TensorFlow's default bias is zeros).
linear_model's weights and bias are set to seeded N(0, 0.3) values through the shim's `linear_model_weights`.
Per case c{k}_: B, S, the wide slots (rows, offset, flat ids + splits), w (all wide weights, concatenated in column
order) and bias, the deep ids and tables, the tower's kernels / biases, the model output `out`, and the raw
gender / age features with the ids of their 14-bucket cross.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REFERENCE = os.environ.get("DR_REFERENCE")
if not REFERENCE or not os.path.isdir(os.path.join(REFERENCE, "deep_recommenders")):
    raise SystemExit("make_wdl_golden.py: set DR_REFERENCE to a checkout of the reference repository")
sys.path.insert(0, os.path.join(ROOT, "oracle", "tf_shim"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.path.insert(0, REFERENCE)
sys.dont_write_bytecode = True

import tensorflow as tf  # noqa: E402  (the shim)
import wdl_oracle as W  # noqa: E402

assert "tf_shim" in tf.__file__, "real TensorFlow found: use it directly instead of the shim"

LAYERS = []
RNG = np.random.RandomState(17)


def _extend_shim():
    class Crossed:
        def __init__(self, keys, hash_bucket_size, hash_key=None):
            self.keys = list(keys)
            self.num_buckets = int(hash_bucket_size)
            self.key = self.name = "_X_".join(sorted(self.keys))

        def ids(self, features):
            cols = [np.asarray(features[k]).reshape(-1).tolist() for k in self.keys]
            out = []
            for b in range(len(cols[0])):
                c = W.cross_example([[col[b]] for col in cols], self.num_buckets)
                out.append(c[0] if c else -1)
            return np.asarray(out, dtype=np.int64)

    class RecordedDense(tf.keras.layers.Dense):
        def build(self, input_shape):
            fan_in = int(input_shape[-1])
            lim = np.sqrt(6.0 / (fan_in + self.units))
            self.kernel = RNG.uniform(-lim, lim, size=(fan_in, self.units))
            self.bias = RNG.standard_normal(self.units) * 0.1
            self.built = True

    def dense(x, units, activation=None, **k):
        layer = RecordedDense(units, activation=activation)
        LAYERS.append(layer)
        return layer(x)

    def relu(x, name=None):
        return tf.convert_to_tensor(np.maximum(np.asarray(x), 0))

    tf.feature_column.crossed_column = Crossed
    tf.layers.dense = dense
    tf.nn.relu = relu


CASES = [
    # tag, B, D, units
    ("ex", 12, 16, [64, 16]),
    ("small", 7, 4, [5]),
]


def main():
    tf.set_default_dtype(np.float64)
    _extend_shim()
    from deep_recommenders.estimator.models.ranking.wide_and_deep import WDL
    out = {"n_cases": np.asarray(len(CASES))}
    rng = np.random.RandomState(23)
    genders, ages, occs = ["F", "M"], [1, 18, 25, 35, 45, 50, 56], list(range(21))
    for k, (tag, B, D, units) in enumerate(CASES):
        p = f"c{k}_"
        fc = tf.feature_column
        user = fc.categorical_column_with_identity("user_id", 30)
        gender = fc.categorical_column_with_vocabulary_list("user_gender", genders)
        age = fc.categorical_column_with_vocabulary_list("user_age", ages)
        occ = fc.categorical_column_with_vocabulary_list("user_occupation", occs)
        base = [user, gender, age, occ]
        crosses = [fc.crossed_column(["user_gender", "user_age"], 14),
                   fc.crossed_column(["user_gender", "user_occupation"], 40),
                   fc.crossed_column(["user_age", "user_occupation"], 140)]
        indicators = [fc.indicator_column(c) for c in base + crosses]
        embeddings = [fc.embedding_column(c, dimension=D) for c in base]
        features = {"user_id": rng.randint(-1, 33, B), "user_gender": np.asarray(rng.choice(genders + ["X"], B)),
                    "user_age": rng.choice(ages + [2], B), "user_occupation": rng.choice(occs + [99], B)}
        model = WDL(indicators, embeddings, units)
        first = len(LAYERS)
        model(features)                           # creates linear_model's variables
        ws, bias = tf.linear_model_weights(indicators)
        for c in indicators:
            ws[c.name][:] = rng.normal(0, 0.3, ws[c.name].shape)
        bias[:] = rng.normal(0, 0.3, 1)
        del LAYERS[first:]
        prob = np.asarray(model(features))
        layers = LAYERS[first:]
        out[p + "B"], out[p + "S"] = np.asarray(B), np.asarray(len(base))
        out[p + "n_wide"] = np.asarray(len(indicators))
        off = 0
        for s, c in enumerate(indicators):
            ids = c.categorical_column.ids(features)
            out[f"{p}wide{s}_ids"] = ids
            out[f"{p}wide{s}_splits"] = np.arange(B + 1, dtype=np.int64)
            out[f"{p}wide{s}_rows"] = np.asarray(c.categorical_column.num_buckets)
            out[f"{p}wide{s}_off"] = np.asarray(off)
            off += c.categorical_column.num_buckets
        out[p + "w"] = np.concatenate([ws[c.name] for c in indicators])
        out[p + "bias"] = np.asarray(bias[0])
        for s, c in enumerate(embeddings):
            out[f"{p}deep{s}_ids"] = c.categorical_column.ids(features)
            out[f"{p}table{s}"] = c.table
        out[p + "nlayers"] = np.asarray(len(layers))
        for i, l in enumerate(layers):
            out[f"{p}k{i}"], out[f"{p}b{i}"] = l.kernel, l.bias
        out[p + "out"] = prob
        out[p + "gender"] = features["user_gender"].astype("U")
        out[p + "age"] = features["user_age"]
        out[p + "cross_ids"] = indicators[len(base)].categorical_column.ids(features)
    np.savez_compressed(os.path.join(HERE, "wdl_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "wdl_golden.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
