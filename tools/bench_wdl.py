"""Wide & Deep benchmark: the crossing kernel, the wide part (forward + gradient scatter + row-sparse FTRL) against
TensorFlow's dense FTRL semantics written as a torch composition over the same tables, and whole WDL train steps.

    python tools/bench_wdl.py [--batch 65536] [--reps 20] [--out FILE]

Writes one JSON document to bench_out/bench_wdl.json (or --out) and prints it.  Timings are CUDA-event medians; the
row-sparse and the dense FTRL alternate in one process.  Shapes:
  * crossing: B examples, two single-valued int64 keys on the device, 2^22 buckets;
  * wide part, production-like: B = 65536, 26 indicator columns of 2^20 rows plus 13 two-key crosses of 2^22 buckets
    (81.8 M records of 16 B = 1.31 GB of state), Zipf(1.1) ids per column;
  * whole step: the example's columns at B = 1024, and the production-like wide part with a deep part of the 26
    columns at D = 16 and a [256, 32] tower, trained with FTRL + TF1 Adam as the example does.
Bandwidth is on algorithmic bytes: per valid lookup its 8-B id and the 32-B sector of its record (forward read,
gradient atomic, FTRL claim), per distinct touched row one more sector read and written by the update; the dense
pass reads and writes every record once.  Share of peak is against the H100 SXM's 3.35 TB/s.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))

from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402
from deep_recommenders_b200.embedding import LinearTable  # noqa: E402
from deep_recommenders_b200.hashing import wide_ids  # noqa: E402

PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
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


def production_features(B, rng, dev):
    raw = {f"C{i}": torch.from_numpy((rng.zipf(1.1, B) - 1) % (1 << 21)).to(dev) for i in range(26)}
    cats = [fc.categorical_column_with_identity(f"C{i}", 1 << 20) for i in range(26)]
    crosses = [fc.crossed_column([f"C{2 * i}", f"C{2 * i + 1}"], 1 << 22) for i in range(13)]
    return raw, cats, crosses


def dense_ftrl(state, lr, l1, l2):
    """TensorFlow's ApplyFtrl over every record (what linear_model's dense gradient makes TensorFlow run)."""
    w, z, n, g = state[:, 0], state[:, 1], state[:, 2], state[:, 3]
    n_new = n + g * g
    z += g - (n_new.sqrt() - n.sqrt()) / lr * w
    y = n_new.sqrt() / lr + 2 * l2
    w.copy_(torch.where(z.abs() > l1, (l1 * z.sign() - z) / y, torch.zeros_like(z)))
    n.copy_(n_new)
    g.zero_()


def bench_wide(B, reps, dev):
    rng = np.random.default_rng(0)
    raw, cats, crosses = production_features(B, rng, dev)
    cols = cats + crosses
    ids, bags = wide_ids(cols, raw, dev)
    table = LinearTable([c.num_buckets for c in cols], device=dev)
    ftrl = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    g_logit = torch.randn(B, device=dev) / B
    rows = torch.tensor(table.rows_list, device=dev)
    offs = table._offsets
    valid = (ids >= 0) & (ids < rows)
    lookups = int(valid.sum())
    distinct = int(torch.unique((ids + offs)[valid]).numel())
    R = table.total_rows

    def fwd():
        return table(ids, bags)

    def sparse_step():
        logit = table(ids, bags)
        logit.backward(g_logit)
        ftrl.apply(table)

    def dense_step():
        logit = table(ids, bags)
        logit.backward(g_logit)
        with torch.no_grad():
            dense_ftrl(table.state, 0.01, 0.5, 0.0)

    t_fwd, t_sparse, t_dense = timed([fwd, sparse_step, dense_step], reps)
    b_fwd = lookups * 40
    b_sparse = lookups * 40 * 3 + distinct * 64
    b_dense = lookups * 80 + (R + 1) * 16 * 2
    return {"batch": B, "slots": len(cols), "records": R + 1, "state_bytes": (R + 1) * 16,
            "valid_lookups": lookups, "distinct_rows": distinct,
            "fwd_ms": t_fwd, "fwd_GBps": b_fwd / t_fwd / 1e6, "fwd_share_of_3.35TBps": b_fwd / (t_fwd * 1e-3) / PEAK,
            "sparse_fwd_scatter_ftrl_ms": t_sparse, "sparse_algorithmic_bytes": b_sparse,
            "sparse_GBps": b_sparse / t_sparse / 1e6, "sparse_share_of_3.35TBps": b_sparse / (t_sparse * 1e-3) / PEAK,
            "dense_fwd_scatter_ftrl_ms": t_dense, "dense_algorithmic_bytes": b_dense,
            "dense_GBps": b_dense / t_dense / 1e6, "dense_share_of_3.35TBps": b_dense / (t_dense * 1e-3) / PEAK,
            "speedup_sparse_over_dense": t_dense / t_sparse}


def bench_cross(B, reps, dev):
    rng = np.random.default_rng(1)
    a = torch.from_numpy(rng.integers(0, 1 << 20, B)).to(dev)
    b = torch.from_numpy(rng.integers(0, 1 << 20, B)).to(dev)
    t, = timed([lambda: ops.cross_hash([a, b], [None, None], [None, None], B, 1 << 22, 0xDECAFCAFFE)], reps)
    return {"batch": B, "keys": 2, "ms": t, "examples_per_s": B / t * 1e3}


def bench_steps(reps, dev):
    from deep_recommenders.estimator.models.ranking import WDL
    import train_wdl_on_movielens_estimator as ex
    out = {}
    ind, emb = ex.build_columns()
    model = ex.WDL(ind + ex.cross_product_transformation(), emb, [64, 16], seed=0, device=dev)
    wide_opt = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    deep_opt = ex.DeepAdam(model.deep_variables(), 0.01)
    feats, labels = next(ex.synthetic_input_fn(1, 1024))
    y = torch.from_numpy(labels).to(dev)

    def step(model=model, feats=feats, y=y, wide_opt=wide_opt, deep_opt=deep_opt):
        loss = ex.log_loss(model(feats).reshape(-1), y)
        loss.backward()
        wide_opt.apply(model.linear)
        deep_opt.step()

    out["example_B1024_ms"], = timed([step], reps)
    B = 65536
    rng = np.random.default_rng(2)
    raw, cats, crosses = production_features(B, rng, dev)
    model2 = WDL([fc.indicator_column(c) for c in cats + crosses], [fc.embedding_column(c, 16) for c in cats],
                 [256, 32], seed=0, device=dev)
    wide2 = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    deep2 = ex.DeepAdam(model2.deep_variables(), 0.01)
    y2 = torch.from_numpy(rng.integers(0, 2, B).astype(np.float32)).to(dev)
    out["production_B65536_ms"], = timed([lambda: step(model2, raw, y2, wide2, deep2)], max(3, reps // 2))
    out["production_examples_per_s"] = B / out["production_B65536_ms"] * 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out", "bench_wdl.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wdl.py needs a CUDA device")
    dev = torch.device("cuda")
    res = {"card": card(), "crossing": bench_cross(args.batch, args.reps, dev)}
    res["wide"] = bench_wide(args.batch, args.reps, dev)
    torch.cuda.empty_cache()
    res["step"] = bench_steps(args.reps, dev)
    text = json.dumps(res, indent=1)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
