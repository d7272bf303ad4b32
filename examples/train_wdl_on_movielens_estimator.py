#!/usr/bin/env python
"""The reference's examples/train_wdl_on_movielens_estimator.py on this framework: the same six MovieLens columns
(movie_genres built on gender_vocab, as the reference does), three crossed columns with 14, 40 and 140 buckets,
WDL(indicator + crossed columns, embedding columns, [64, 16]), tf.losses.log_loss, FTRL(0.01, l1 = 0.5) on the wide
part and TF1 Adam(0.01) on the deep part, AUC on the evaluation batches.

The reference's two `minimize` calls read the same forward pass and update disjoint variable lists, so one forward,
one backward and both updates is the same step.  Data: the TFRecord reader when a MovieLens directory is given, else
seeded synthetic MovieLens-1M-shaped batches.  Exits non-zero if the training loss did not fall.

    python examples/train_wdl_on_movielens_estimator.py [--train-steps N] [--eval-steps N] [--data DIR]
Needs a CUDA device (the model runs in libdeeprec_b200.so; there is no CPU fallback).
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200 import feature_column as fc  # noqa: E402     (tf.feature_column)
from deep_recommenders_b200 import ops  # noqa: E402                      (tf.train.FtrlOptimizer / AdamOptimizer)
from deep_recommenders_b200.keras import engine as K  # noqa: E402        (tf.metrics.auc)
from deep_recommenders.estimator.models.ranking import WDL  # noqa: E402

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


def cross_product_transformation():
    crossed_columns = [
        fc.crossed_column(["user_gender", "user_age"], 14),
        fc.crossed_column(["user_gender", "user_occupation"], 40),
        fc.crossed_column(["user_age", "user_occupation"], 140),
    ]
    return [fc.indicator_column(c) for c in crossed_columns]


def synthetic_input_fn(seed, batch_size=1024):
    """Endless MovieLens-1M-shaped batches (labels [B] float32); the label depends on the ids and on the
    gender x age cross, so that both halves have something to learn."""
    rng = np.random.default_rng(seed)
    taste = np.random.default_rng(7).normal(size=(NUM_USERS + 1,)) * 0.8
    appeal = np.random.default_rng(8).normal(size=(NUM_MOVIES + 1,)) * 0.8
    cross = np.random.default_rng(9).normal(size=(2, len(AGE_VOCAB))) * 0.8
    while True:
        u = rng.integers(1, NUM_USERS + 1, batch_size)
        m = rng.integers(1, NUM_MOVIES + 1, batch_size)
        g = rng.integers(0, 2, batch_size)
        a = rng.integers(0, len(AGE_VOCAB), batch_size)
        feats = {"user_id": np.asarray([str(x) for x in u]), "user_gender": np.asarray(GENDER_VOCAB)[g],
                 "user_age": np.asarray(AGE_VOCAB, dtype=np.int64)[a],
                 "user_occupation": rng.choice(OCCUPATION_VOCAB, batch_size).astype(np.int64),
                 "movie_id": np.asarray([str(x) for x in m]), "movie_genres": rng.choice(["Action", "Comedy"], batch_size)}
        p = 1.0 / (1.0 + np.exp(-(taste[u] + appeal[m] + cross[g, a])))
        yield feats, (rng.random(batch_size) < p).astype(np.float32)


def log_loss(p, y, eps=1e-7):
    """tf.losses.log_loss with its default epsilon and mean reduction."""
    return torch.mean(-y * torch.log(p + eps) - (1 - y) * torch.log(1 - p + eps))


class DeepAdam:
    """tf.train.AdamOptimizer(0.01) on the deep variables: TensorFlow's ApplyAdam (ops.adam_step_), dense over each
    variable, with the bias-corrected rate kept on the device."""

    def __init__(self, params, lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8):
        self.params = [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in params]
        self.clock = ops.AdamClock(lr, beta1, beta2, eps, device=self.params[0][0].device)

    def step(self):
        self.clock.advance()
        c = self.clock
        for p, m, v in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            ops.adam_step_(p.data, p.grad, m, v, 0.0, c.beta1, c.beta2, c.eps, zero_grad=True, lr_t_dev=c.lr_t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train-steps", type=int, default=400)
    ap.add_argument("--eval-steps", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--data", default=None, help="MovieLens TFRecord directory (datasets.MovielensRanking); default synthetic")
    args = ap.parse_args()
    indicator_columns, embedding_columns = build_columns()
    crossed_product_columns = cross_product_transformation()
    if args.data:
        from deep_recommenders.datasets import MovielensRanking
        movielens = MovielensRanking(batch_size=args.batch_size, filename=os.path.join(args.data, "movielens.tfrecords"))
        train, test = movielens.training_input_fn, movielens.testing_input_fn
    else:
        train, test = synthetic_input_fn(1, args.batch_size), synthetic_input_fn(2, args.batch_size)

    model = WDL(indicator_columns + crossed_product_columns, embedding_columns, [64, 16], seed=42, device="cuda")
    wide_optimizer = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    deep_optimizer = DeepAdam(model.deep_variables(), 0.01)
    dev = torch.device("cuda")

    losses = []
    for step in range(args.train_steps):
        try:
            features, labels = next(train)
        except StopIteration:
            break
        outputs = model(features).reshape(-1)
        loss = log_loss(outputs, torch.as_tensor(np.asarray(labels, dtype=np.float32).reshape(-1), device=dev))
        loss.backward()
        wide_optimizer.apply(model.linear)
        deep_optimizer.step()
        losses.append(loss.detach())
        if (step + 1) % 100 == 0:
            print(f"step {step + 1}: loss {float(torch.stack(losses[-100:]).mean()):.4f}")
    h = torch.stack(losses).cpu().numpy()
    w = max(1, min(50, len(h) // 2))
    first, last = float(h[:w].mean()), float(h[-w:].mean())
    auc = K.AUC()
    with torch.no_grad():
        for _ in range(args.eval_steps):
            try:
                features, labels = next(test)
            except StopIteration:
                break
            auc.update_state(torch.as_tensor(np.asarray(labels, dtype=np.float32).reshape(-1, 1), device=dev),
                             model(features))
    print(f"train log loss, first {w} steps: {first:.4f}, last {w} steps: {last:.4f}")
    print(f"eval auc: {auc.result():.4f}")
    if not last < first:
        raise SystemExit("the training loss did not fall")


if __name__ == "__main__":
    main()
