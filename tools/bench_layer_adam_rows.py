"""TF1 Adam on the tables of the layer-API models: dense (ops.adam_step_ over the whole arena, the examples' default)
against optimizers.RowSparseAdam (--embedding-optimizer rows_tf), whole train steps.

    python tools/bench_layer_adam_rows.py [--batch 65536] [--slots 26] [--rows 1048576] [--dim 16] [--reps 20]
                                          [--models fnn,wdl] [--out FILE]

Writes one JSON document to bench_out/bench_layer_adam_rows.json (or --out) and prints it.  Per model and id
distribution the two optimizers train two copies of the model built from one seed, alternating step by step in one
process; times are CUDA-event medians of whole steps (forward, log loss, backward, the updates).  Shapes (DESIGN.md
section 6): B = 65536, 26 identity columns of 2^20 rows, D = 16, ids uniform or Zipf(1.1) on the device.
  * fnn: FNN [64, 32] warm-started from an untrained FM export; dense Adam over the tower (and, dense, the arena).
  * wdl: WDL [256, 32], its wide part over the 26 indicator columns and 13 two-key crosses of 2^22 buckets, FTRL on it
    in both runs (ids (zipf - 1) mod 2^21 as tools/bench_wdl.py: about half fall outside the 2^20 rows and are pruned).
Also reported: the bytes the dense Adam sweep must move each step (p, g, m, v read, p, m, v written, g zeroed: 32 B per
float of the arena) and the distinct rows a batch touches.  The card, its power limit and SM clock are in the JSON.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402
from deep_recommenders_b200.optimizers import HISTORY, RowSparseAdam  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fns, reps):
    """Median ms of each callable, run alternately."""
    times = [[] for _ in fns]
    for f in fns:
        f()
    torch.cuda.synchronize()
    for _ in range(reps):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in times]


class DenseAdam:
    """tf.train.AdamOptimizer(0.01) over each variable (ops.adam_step_), as the examples keep it."""

    def __init__(self, params, history=0):
        self.params = [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in params]
        self.clock = ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device="cuda", history=history)

    def step(self):
        self.clock.advance()
        c = self.clock
        for p, m, v in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            ops.adam_step_(p.data, p.grad, m, v, 0.0, c.beta1, c.beta2, c.eps, zero_grad=True, lr_t_dev=c.lr_t)


def log_loss(p, y):
    return torch.mean(-y * torch.log(p + 1e-7) - (1 - y) * torch.log(1 - p + 1e-7))


def make_ids(dist, B, S, mod, seed):
    g = np.random.default_rng(seed)
    ids = g.integers(0, mod, (B, S)) if dist == "uniform" else (g.zipf(1.1, (B, S)) - 1) % mod
    return torch.from_numpy(ids.astype(np.int64)).cuda()


def _optimizers(model, mode, dense_all):
    if mode == "dense":
        return DenseAdam(dense_all), None
    d = DenseAdam(model.dense_variables(), history=HISTORY)
    return d, RowSparseAdam(model.embedding_collection(), 0.01, clock=d.clock)


def bench_fnn(args, dist, tmp):
    from deep_recommenders.estimator.models.feature_interaction import FM
    from deep_recommenders.estimator.models.ranking import FNN
    B, S, D, R = args.batch, args.slots, args.dim, args.rows
    cols = [fc.categorical_column_with_identity(f"c{s}", R) for s in range(S)]
    ind, emb = [fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols]
    path = os.path.join(tmp, "fm.pt")
    fm = FM(ind, emb, seed=0, device="cuda")
    fm.export(path)
    del fm
    runs = {}
    for mode in ("dense", "rows_tf"):
        model = FNN(ind, emb, path, [64, 32], seed=0, device="cuda")
        runs[mode] = (model,) + _optimizers(model, mode, list(model.parameters()))
    os.remove(path)
    ids = make_ids(dist, B, S, R, 2)
    feats = {f"c{s}": ids[:, s].contiguous() for s in range(S)}
    y = (torch.rand(B, device="cuda") < 0.3).float()
    arena_floats = runs["dense"][0].embeddings.weight.numel()
    return runs, (lambda model: log_loss(model(feats).reshape(-1), y)), ids, arena_floats, None


def bench_wdl(args, dist, tmp):
    from deep_recommenders.estimator.models.ranking import WDL
    B, S, D, R = args.batch, args.slots, args.dim, args.rows
    g = np.random.default_rng(2)
    ids = make_ids(dist, B, S, 2 * R, 2)
    raw = {f"C{i}": ids[:, i].contiguous() for i in range(S)}
    cats = [fc.categorical_column_with_identity(f"C{i}", R) for i in range(S)]
    crosses = [fc.crossed_column([f"C{2 * i}", f"C{2 * i + 1}"], 1 << 22) for i in range(S // 2)]
    runs = {}
    for mode in ("dense", "rows_tf"):
        model = WDL([fc.indicator_column(c) for c in cats + crosses], [fc.embedding_column(c, D) for c in cats],
                    [256, 32], seed=0, device="cuda")
        runs[mode] = (model,) + _optimizers(model, mode, model.deep_variables())
    y = torch.from_numpy(g.integers(0, 2, B).astype(np.float32)).cuda()
    ftrl = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    valid = torch.where(ids < R, ids, torch.full_like(ids, -1))
    arena_floats = runs["dense"][0].embeddings.weight.numel()
    return runs, (lambda model: log_loss(model(raw).reshape(-1), y)), valid, arena_floats, ftrl


def run(args, kind, dist, tmp):
    runs, loss_of, ids, arena_floats, ftrl = (bench_fnn if kind == "fnn" else bench_wdl)(args, dist, tmp)

    def step(mode):
        model, dense, rows = runs[mode]
        loss = loss_of(model)
        loss.backward()
        if ftrl is not None:
            ftrl.apply(model.linear)
        dense.step()
        if rows is not None:
            rows.step()
        return loss

    t_dense, t_rows = timed([lambda: step("dense"), lambda: step("rows_tf")], args.reps)
    S = ids.shape[1]
    offs = torch.arange(S, device="cuda", dtype=torch.int64) * args.rows
    ok = ids >= 0
    distinct = int(torch.unique((ids + offs)[ok]).numel())
    rows_opt = runs["rows_tf"][2]
    rows_opt.flush()
    return {"model": kind, "ids": dist, "B": args.batch, "slots": S, "rows_per_slot": args.rows, "D": args.dim,
            "arena_bytes": arena_floats * 4, "dense_sweep_bytes_per_step": arena_floats * 32,
            "valid_lookups": int(ok.sum()), "distinct_rows": distinct,
            "dense_step_ms": t_dense, "rows_tf_step_ms": t_rows, "speedup": t_dense / t_rows,
            "examples_per_s_dense": args.batch / t_dense * 1e3, "examples_per_s_rows_tf": args.batch / t_rows * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--models", default="fnn,wdl")
    ap.add_argument("--out", default=os.path.join("bench_out", "bench_layer_adam_rows.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_layer_adam_rows.py needs a CUDA device")
    res = {"card": card(), "torch": torch.__version__, "reps": args.reps, "results": []}
    with tempfile.TemporaryDirectory() as tmp:
        for kind in args.models.split(","):
            for dist in ("uniform", "zipf1.1"):
                r = run(args, kind, dist, tmp)
                res["results"].append(r)
                print(json.dumps(r), flush=True)
                torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
