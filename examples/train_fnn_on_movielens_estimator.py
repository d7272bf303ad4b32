#!/usr/bin/env python
"""The reference's examples/train_fnn_on_movielens_estimator.py on this framework, both of its stages in one script:
the same six MovieLens columns (movie_genres built on gender_vocab, as the reference does) as indicator and embedding
columns of dimension 16.

  Stage 1 (the reference's FM example): FM(indicator_columns, embedding_columns) with tf.losses.sigmoid_cross_entropy
          and Adam(0.01), then FM.export(path) -- the file FNN warm-starts from.  --warm-up-from-fm PATH skips it.
  Stage 2: FNN(indicator_columns, embedding_columns, path, [64, 32]) with tf.losses.log_loss and TF1 Adam(0.01) over
          every FNN variable (ops.adam_step_, dense, as the WDL example's deep part), then AUC on evaluation batches.

Data: the TFRecord reader when a MovieLens directory is given, else seeded synthetic MovieLens-1M-shaped batches.
Exits non-zero if stage 2's training loss did not fall.

    python examples/train_fnn_on_movielens_estimator.py [--fm-steps N] [--train-steps N] [--eval-steps N]
                                                        [--warm-up-from-fm PATH] [--export PATH] [--data DIR]
Needs a CUDA device (the model runs in libdeeprec_b200.so; there is no CPU fallback).
"""
import argparse
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200 import feature_column as fc  # noqa: E402     (tf.feature_column)
from deep_recommenders_b200 import ops  # noqa: E402                      (tf.train.AdamOptimizer)
from deep_recommenders_b200.keras import engine as K  # noqa: E402        (tf.metrics.auc)
from deep_recommenders.estimator.models.feature_interaction import FM  # noqa: E402
from deep_recommenders.estimator.models.ranking import FNN  # noqa: E402

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
    """Endless MovieLens-1M-shaped batches (labels [B] float32); the label depends on the user, the movie and the
    gender x age pair, so that both the first-order weights and the embeddings have something to learn."""
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


class Adam:
    """tf.train.AdamOptimizer(lr): TensorFlow's ApplyAdam (ops.adam_step_), dense over each variable, with the
    bias-corrected rate kept on the device."""

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


def _labels(labels, dev):
    return torch.as_tensor(np.asarray(labels, dtype=np.float32).reshape(-1), device=dev)


def train_fm(columns, train, steps, path, dev):
    """Stage 1: the reference's FM example (sigmoid cross-entropy on the FM logit, Adam(0.01)), then FM.export."""
    indicator_columns, embedding_columns = columns
    fm = FM(indicator_columns, embedding_columns, seed=42, device=dev)
    opt = Adam(list(fm.parameters()), 0.01)
    losses = []
    for _ in range(steps):
        features, labels = next(train)
        logits = fm(features).reshape(-1)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, _labels(labels, dev))
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    if losses:
        h = torch.stack(losses).cpu().numpy()
        w = max(1, min(50, len(h) // 2))
        print(f"stage 1 (FM) sigmoid cross-entropy, first {w} steps: {h[:w].mean():.4f}, last {w}: {h[-w:].mean():.4f}")
    fm.export(path)
    print(f"stage 1: exported the FM to {path}")


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--fm-steps", type=int, default=400)
    ap.add_argument("--train-steps", type=int, default=400)
    ap.add_argument("--eval-steps", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--warm-up-from-fm", default=None, help="an FM.export file: skip stage 1")
    ap.add_argument("--export", default=None, help="where stage 1 writes the FM (default: a temporary directory)")
    ap.add_argument("--data", default=None, help="MovieLens TFRecord directory (datasets.MovielensRanking); default synthetic")
    args = ap.parse_args(argv)
    columns = build_columns()
    if args.data:
        from deep_recommenders.datasets import MovielensRanking
        movielens = MovielensRanking(batch_size=args.batch_size, filename=os.path.join(args.data, "movielens.tfrecords"))
        train, test = movielens.training_input_fn, movielens.testing_input_fn
    else:
        train, test = synthetic_input_fn(1, args.batch_size), synthetic_input_fn(2, args.batch_size)
    dev = torch.device("cuda")

    with tempfile.TemporaryDirectory() as tmp:
        path = args.warm_up_from_fm
        if path is None:
            path = args.export or os.path.join(tmp, "fm.pt")
            train_fm(columns, train, args.fm_steps, path, dev)
        model = FNN(*columns, path, [64, 32], seed=42, device=dev)

    optimizer = Adam(list(model.parameters()), 0.01)
    losses = []
    for step in range(args.train_steps):
        try:
            features, labels = next(train)
        except StopIteration:
            break
        outputs = model(features).reshape(-1)
        loss = log_loss(outputs, _labels(labels, dev))
        loss.backward()
        optimizer.step()
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
            auc.update_state(_labels(labels, dev).reshape(-1, 1), model(features))
    print(f"stage 2 (FNN) train log loss, first {w} steps: {first:.4f}, last {w} steps: {last:.4f}")
    print(f"eval auc: {auc.result():.4f}")
    if not last < first:
        raise SystemExit("the training loss did not fall")
    return first, last, float(auc.result())


if __name__ == "__main__":
    main()
