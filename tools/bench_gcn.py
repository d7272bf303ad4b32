"""GCN benchmark: the CSR SpMM forward and transposed backward against torch.sparse.mm (cuSPARSE) on the same CSR, both
computation orders of one GCN layer on each side of the layer's order selection, and the example-shaped train step.

    python tools/bench_gcn.py [--nodes 1048576] [--reps 20] [--out FILE]

Prints one JSON document.  Timings are CUDA-event medians with the library and the baseline alternating in one
process.  SpMM bandwidth is given two ways: on algorithmic bytes (indptr, indices, values and x read once, y written
once) and on gathered bytes (4 * nnz * F, every neighbour row read).  The power-law graph has the uniform graph's nnz
and shows what one owner per row costs on heavy rows.  The train step at Cora's size (2708 nodes) is a few small
kernels: it measures launch overhead, not bandwidth.
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
sys.path.insert(0, os.path.join(ROOT, "examples"))

from deep_recommenders_b200 import ops  # noqa: E402


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


def graph(n, deg, kind, rng):
    """CSR of n nodes, a self-loop plus `deg` neighbours on average: uniform degree, or power-law degrees (Zipf-like,
    rescaled to the same total)."""
    if kind == "uniform":
        d = np.full(n, deg, np.int64)
    else:
        w = 1.0 / np.arange(1, n + 1) ** 0.8
        d = np.floor(w / w.sum() * deg * n).astype(np.int64)
        d[: deg * n - d.sum()] += 1
        rng.shuffle(d)
    d += 1
    indptr = np.concatenate([[0], np.cumsum(d)])
    idx = rng.integers(0, n, indptr[-1]).astype(np.int32)
    idx[indptr[:-1]] = np.arange(n)                                 # self-loop first in each row
    vals = rng.uniform(0.01, 1.0, indptr[-1]).astype(np.float32)
    return ops.CSRAdjacency(indptr, idx, vals, (n, n)), int(d.max())


def bench_spmm(n, reps, rng):
    out = []
    for kind in ("uniform", "powerlaw"):
        adj, dmax = graph(n, 16, kind, rng)
        ref = torch.sparse_csr_tensor(adj.indptr.long(), adj.indices.long(), adj.values, (n, n))
        ref_t = torch.sparse_csr_tensor(adj.t_indptr.long(), adj.t_indices.long(), adj.t_values, (n, n))
        for F in (32, 128):
            x = torch.randn(n, F, device="cuda")
            ms_lib, ms_ref, ms_lib_t, ms_ref_t = timed([lambda: adj.spmm(x), lambda: torch.sparse.mm(ref, x),
                                                        lambda: adj.spmm(x, transpose=True),
                                                        lambda: torch.sparse.mm(ref_t, x)], reps)
            diff = float((adj.spmm(x)[0] - torch.sparse.mm(ref, x)).abs().max())
            diff_t = float((adj.spmm(x, transpose=True)[0] - torch.sparse.mm(ref_t, x)).abs().max())
            algo = 4 * (n + 1) + 8 * adj.nnz + 4 * n * F + 4 * n * F
            gathered = 4 * adj.nnz * F
            row = {"graph": kind, "nodes": n, "nnz": adj.nnz, "max_row": dmax, "F": F}
            for tag, ms, ms_b, d in (("fwd", ms_lib, ms_ref, diff), ("bwd_transposed", ms_lib_t, ms_ref_t, diff_t)):
                row[tag] = {"ms": round(ms, 4), "cusparse_ms": round(ms_b, 4), "speedup": round(ms_b / ms, 3),
                            "GBps_algorithmic": round(algo / ms / 1e6, 1), "GBps_gathered": round(gathered / ms / 1e6, 1),
                            "max_abs_diff_vs_cusparse": d}
            out.append(row)
        del adj, ref, ref_t
        torch.cuda.empty_cache()
    return out


def bench_orders(n, reps, rng):
    """One GCN layer, forward + backward, in both orders: X W first (the layer's choice when F > units) and A X first
    (its choice otherwise)."""
    adj, _ = graph(n, 16, "uniform", rng)
    out = []
    for F, units in ((1433, 32), (32, 256)):
        x = torch.randn(n, F, device="cuda").requires_grad_()
        w = (torch.randn(F, units, device="cuda") * 0.05).requires_grad_()
        b = torch.zeros(units, device="cuda", requires_grad=True)
        g = torch.randn(n, units, device="cuda")

        def xw_first():
            ops.SpMMFn.apply(ops.DenseFn.apply(x, w, None, 0), b, None, adj, 1).backward(g)

        def ax_first():
            ops.DenseFn.apply(ops.SpMMFn.apply(x, None, None, adj, 0), w, b, 1).backward(g)

        ms_xw, ms_ax = timed([xw_first, ax_first], reps)
        chosen = "XW_first" if F > units else "AX_first"
        out.append({"nodes": n, "F": F, "units": units, "layer_order": chosen, "XW_first_ms": round(ms_xw, 3),
                    "AX_first_ms": round(ms_ax, 3)})
        del x, w, b, g
        torch.cuda.empty_cache()
    return out


def bench_train_step(reps):
    import train_gcn_on_cora_keras as ex
    from deep_recommenders.datasets import Cora, write_synthetic_cora
    with tempfile.TemporaryDirectory() as d:
        cora = Cora(write_synthetic_cora(d, seed=0))
        ids, features, labels = cora.load_content()
        sg = cora.spectral_graph(cora.build_graph(ids))
        (train_labels, train_mask), _, _ = cora.split_labels(labels)
    g = ops.CSRAdjacency.from_any(sg)
    feats = torch.from_numpy(np.asarray(features.todense(), np.float32)).cuda()
    from deep_recommenders_b200.keras.engine import Adam
    model = ex.GCNClassifier(cora.num_classes)
    model.compile(optimizer=Adam(0.01), loss="categorical_crossentropy", weighted_metrics=["acc"])
    steps = 50
    step = lambda: model.fit([g, feats], train_labels, sample_weight=train_mask, epochs=steps)
    ms = timed([step], max(3, reps // 4))[0]
    return {"nodes": sg.shape[0], "widths": [features.shape[1], 32, cora.num_classes], "ms_per_step": round(ms / steps, 4),
            "note": "full-batch engine step (forward, weighted loss, backward, Adam) at Cora's size: launch-overhead bound"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1 << 20)
    ap.add_argument("--layer-nodes", type=int, default=1 << 17)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gcn.py needs a CUDA device")
    rng = np.random.default_rng(0)
    res = {"card": card(), "spmm": bench_spmm(a.nodes, a.reps, rng),
           "layer_orders": bench_orders(a.layer_nodes, a.reps, rng), "train_step": bench_train_step(a.reps)}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
