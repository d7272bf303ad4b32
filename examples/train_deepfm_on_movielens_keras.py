#!/usr/bin/env python
"""The reference's Keras example (/root/reference/examples/train_deepfm_on_movielens_keras.py:10-54) on this
framework: same six MovieLens columns, DeepFM(dnn_units_size=[256, 32]), compile(binary cross-entropy, Adam, AUC /
Precision / Recall), fit(..., validation_data, EarlyStopping(patience=3)).  `import tensorflow as tf` becomes the two
import lines below; the rest reads like the reference script.  Data: the real TFRecord reader when a MovieLens
directory is given, else SYNTHETIC MovieLens-1M-shaped batches (no network here).

    python examples/train_deepfm_on_movielens_keras.py [--steps-per-epoch N] [--epochs E] [--data DIR]
                                                        [--optimizer {keras,tf}]
--optimizer keras (the default) compiles with the engine's Adam (torch.optim.Adam); tf compiles with
optimizers.KerasAdam(), TensorFlow's Adam arithmetic with the embedding tables trained row-sparse.
Needs a CUDA device (the layers run in libdeeprec_b200.so; there is no CPU fallback).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200 import feature_column as fc  # noqa: E402     (tf.feature_column)
from deep_recommenders_b200.keras import engine as K  # noqa: E402          (tf.keras.losses / optimizers / metrics / callbacks)
from deep_recommenders.keras.models.ranking import DeepFM  # noqa: E402
from deep_recommenders_b200.optimizers import KerasAdam  # noqa: E402

NUM_USERS, NUM_MOVIES = 6040, 3952
GENDER_VOCAB = ["F", "M"]
AGE_VOCAB = [1, 18, 25, 35, 45, 50, 56]
OCCUPATION_VOCAB = list(range(21))


def build_columns():
    user_id = fc.categorical_column_with_hash_bucket("user_id", NUM_USERS)
    user_gender = fc.categorical_column_with_vocabulary_list("user_gender", GENDER_VOCAB)
    user_age = fc.categorical_column_with_vocabulary_list("user_age", AGE_VOCAB)
    user_occupation = fc.categorical_column_with_vocabulary_list("user_occupation", OCCUPATION_VOCAB)
    movie_id = fc.categorical_column_with_hash_bucket("movie_id", NUM_MOVIES)
    movie_genres = fc.categorical_column_with_vocabulary_list("movie_genres", GENDER_VOCAB)   # sic (reference :22-23)
    base_columns = [user_id, user_gender, user_age, user_occupation, movie_id, movie_genres]
    indicator_columns = [fc.indicator_column(c) for c in base_columns]
    embedding_columns = [fc.embedding_column(c, dimension=16) for c in base_columns]
    return indicator_columns, embedding_columns


def synthetic_input_fn(seed, batch_size=1024):
    """Endless MovieLens-1M-shaped batches; the label depends on the ids so that there is something to learn."""
    rng = np.random.default_rng(seed)
    taste = np.random.default_rng(7).normal(size=(NUM_USERS + 1,)) * 0.8
    appeal = np.random.default_rng(8).normal(size=(NUM_MOVIES + 1,)) * 0.8
    while True:
        u = rng.integers(1, NUM_USERS + 1, batch_size)
        m = rng.integers(1, NUM_MOVIES + 1, batch_size)
        feats = {"user_id": np.asarray([str(x) for x in u]), "user_gender": rng.choice(GENDER_VOCAB, batch_size),
                 "user_age": rng.choice(AGE_VOCAB, batch_size), "user_occupation": rng.choice(OCCUPATION_VOCAB, batch_size),
                 "movie_id": np.asarray([str(x) for x in m]), "movie_genres": rng.choice(["Action", "Comedy"], batch_size)}
        p = 1.0 / (1.0 + np.exp(-(taste[u] + appeal[m])))
        yield feats, (rng.random(batch_size) < p).astype(np.float32)[:, None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--steps-per-epoch", type=int, default=50)
    ap.add_argument("--validation-steps", type=int, default=10)
    ap.add_argument("--data", default=None, help="MovieLens TFRecord directory (datasets.MovielensRanking); default synthetic")
    ap.add_argument("--optimizer", choices=["keras", "tf"], default="keras",
                    help="keras: the engine's Adam (torch.optim.Adam); tf: optimizers.KerasAdam (TensorFlow's Adam)")
    args = ap.parse_args()
    indicator_columns, embedding_columns = build_columns()
    if args.data:
        from deep_recommenders.datasets import MovielensRanking
        movielens = MovielensRanking(args.data)
        train, test = movielens.training_input_fn, movielens.testing_input_fn
        steps, vsteps = movielens.train_steps_per_epoch, movielens.test_steps
    else:
        train, test, steps, vsteps = synthetic_input_fn(1), synthetic_input_fn(2), args.steps_per_epoch, args.validation_steps

    model = DeepFM(indicator_columns, embedding_columns, dnn_units_size=[256, 32], seed=0, device="cuda")
    model.compile(loss=K.binary_crossentropy,
                  optimizer=K.Adam() if args.optimizer == "keras" else KerasAdam(),
                  metrics=[K.AUC(), K.Precision(), K.Recall()])
    history = model.fit(train,
                        epochs=args.epochs,
                        steps_per_epoch=steps,
                        validation_data=test,
                        validation_steps=vsteps,
                        callbacks=[K.EarlyStopping(patience=3)],
                        verbose=1)
    return history


if __name__ == "__main__":
    main()
