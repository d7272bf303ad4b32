"""FNN benchmark: the fused tower-input gather (dr_fnn_input_fwd / _bwd) against the torch composition it replaces and
against the stack-only embedding gather that reads the same lines; layer 0 of the tower at the reference's input width
and at the padded one; whole FNN train steps.

    python tools/bench_fnn.py [--batch 65536] [--slots 26] [--rows 1048576] [--dim 16] [--reps 20] [--out FILE]

Writes one JSON document to bench_out/bench_fnn.json (or --out) and prints it.  Timings are CUDA-event medians; the
forms compared alternate in one process.  Shapes: B = 65536 examples, S = 26 tables of 2^20 rows, D = 16 (the fused
row layout: [emb | w] in one 128-B line), uniform and Zipf(1.1) ids.
  * input, forward: dr_fnn_input_fwd; the composition (stack-only EmbedFM, a gather of lin_view(), torch.cat with the
    bias column); stack-only dr_embed_fm_fwd on the same ids.  Forward + dense backward for the first two.
    Bandwidth is on algorithmic bytes: per lookup its 8-B id and its 128-B line, per example the 4*ld bytes written.
    Share of peak is against the H100 SXM's 3.35 TB/s.
  * layer 0 (Dense to 256 units, relu) forward + backward through ops.DenseFn at K = 1 + S + S*D and at K = ld, and the
    GEMM kernels each ran, from a torch.profiler run of its own.
  * whole step (forward, log loss, backward, dense TF1 Adam over every variable, as the example): at the shape above
    with identity columns and ids on the device, and at the example's six MovieLens columns, B = 1024.
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

from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders_b200 import ops  # noqa: E402
from deep_recommenders_b200.embedding import EmbeddingCollection  # noqa: E402

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


def make_ids(dist, B, S, rows, seed):
    g = np.random.default_rng(seed)
    if dist == "uniform":
        ids = g.integers(0, rows, (B, S))
    else:
        ids = (g.zipf(1.1, (B, S)) - 1) % rows
    return torch.from_numpy(ids.astype(np.int64)).cuda()


def composition(coll, ids, bias, weight):
    """The torch glue the fused kernel replaces, in the reference's column order [bias | w | e]."""
    B, S = ids.shape
    stack, _ = ops.EmbedFM.apply(ids, weight, None, None, coll, False)
    rows = coll._rows
    ok = (ids >= 0) & (ids < rows)
    r = torch.where(ok, ids + coll._offsets, torch.zeros_like(ids))
    w = torch.where(ok, coll.lin_view(weight)[r], torch.zeros((), device=ids.device))
    return torch.cat([bias.expand(B, 1), w, stack.reshape(B, -1)], dim=1)


def bench_input(args, res):
    B, S, D, R = args.batch, args.slots, args.dim, args.rows
    coll = EmbeddingCollection([R] * S, D, with_linear=True, seed=0, device="cuda")
    bias = torch.tensor([0.1], device="cuda")
    P, ld = ops.fnn_layout(S, D)
    algo = B * S * (8 + 128) + B * 4 * ld
    out = {"shape": {"B": B, "S": S, "rows": R, "D": D, "P": P, "ld": ld, "layout": coll.layout},
           "algorithmic_bytes_fwd": algo}
    for dist in ("uniform", "zipf1.1"):
        ids = make_ids(dist, B, S, R, 1)
        g_fused = torch.randn((B, ld), device="cuda")
        g_comp = torch.randn((B, 1 + S + S * D), device="cuda")
        with torch.no_grad():
            x = ops.FnnInputFn.apply(ids, coll.weight, None, bias, coll, None)
            y = composition(coll, ids, bias, coll.weight)
            same = bool(torch.equal(torch.cat([x[:, :1 + S], x[:, P:]], 1), y))

        def fused_fwd():
            with torch.no_grad():
                ops.FnnInputFn.apply(ids, coll.weight, None, bias, coll, None)

        def comp_fwd():
            with torch.no_grad():
                composition(coll, ids, bias, coll.weight)

        def stack_only():
            with torch.no_grad():
                ops.EmbedFM.apply(ids, coll.weight, None, None, coll, False)

        def fused_fb():
            coll.weight.grad = None
            ops.FnnInputFn.apply(ids, coll.weight, None, bias, coll, None).backward(g_fused)

        def comp_fb():
            coll.weight.grad = None
            composition(coll, ids, bias, coll.weight).backward(g_comp)

        t = timed([fused_fwd, comp_fwd, stack_only], args.reps)
        tb = timed([fused_fb, comp_fb], args.reps)
        coll.weight.grad = None
        out[dist] = {
            "same_values": same,
            "fused_fwd_ms": t[0], "composition_fwd_ms": t[1], "embed_fm_stack_only_ms": t[2],
            "fused_fwd_GBps": algo / t[0] / 1e6, "fused_fwd_share_of_3.35TBps": algo / t[0] / 1e-3 / PEAK,
            "fused_over_stack_only": t[0] / t[2], "composition_over_fused_fwd": t[1] / t[0],
            "fused_fwd_bwd_ms": tb[0], "composition_fwd_bwd_ms": tb[1], "composition_over_fused_fwd_bwd": tb[1] / tb[0],
        }
        print(json.dumps({dist: out[dist]}), flush=True)
    del coll
    torch.cuda.empty_cache()
    res["input"] = out


def bench_layer0(args, res):
    B, S, D = args.batch, args.slots, args.dim
    P, ld = ops.fnn_layout(S, D)
    N = 256
    out = {"N": N, "act": "relu"}
    fns, names = [], []
    for K in (1 + S + S * D, ld):
        x = torch.randn((B, K), device="cuda")
        w = torch.nn.Parameter(torch.randn((K, N), device="cuda") * 0.05)
        b = torch.nn.Parameter(torch.zeros(N, device="cuda"))
        g = torch.randn((B, N), device="cuda")

        def fb(x=x, w=w, b=b, g=g):
            w.grad = b.grad = None
            ops.DenseFn.apply(x, w, b, 1).backward(g)
        fns.append(fb)
        names.append(K)
    t = timed(fns, args.reps)
    for K, ms in zip(names, t):
        flops = 3 * 2 * B * K * N
        out[f"K{K}"] = {"fwd_bwd_ms": ms, "TFLOPs": flops / ms / 1e9}
    # the GEMM kernels each width ran, from a profiler run of its own
    for K, f in zip(names, fns):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        kern = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
        out[f"K{K}"]["kernels"] = kern
        out[f"K{K}"]["wgmma"] = any("gemm_tc" in k for k in kern)
    res["layer0"] = out
    print(json.dumps({"layer0": out}), flush=True)


def _adam(params):
    state = [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in params]
    clock = ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device="cuda")

    def step():
        clock.advance()
        for p, m, v in state:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            ops.adam_step_(p.data, p.grad, m, v, 0.0, 0.9, 0.999, 1e-8, zero_grad=True, lr_t_dev=clock.lr_t)
    return step


def _train_step(model, step, features, y):
    p = model(features).reshape(-1)
    loss = torch.mean(-y * torch.log(p + 1e-7) - (1 - y) * torch.log(1 - p + 1e-7))
    loss.backward()
    step()
    return loss


def bench_steps(args, res):
    from deep_recommenders.estimator.models.feature_interaction import FM
    from deep_recommenders.estimator.models.ranking import FNN
    import train_fnn_on_movielens_estimator as ex
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        # production shape, identity columns, ids on the device
        B, S, D, R = args.batch, args.slots, args.dim, args.rows
        cols = [fc.categorical_column_with_identity(f"c{s}", R) for s in range(S)]
        ind, emb = [fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols]
        path = os.path.join(tmp, "fm_big.pt")
        fm = FM(ind, emb, seed=0, device="cuda")
        fm.export(path)
        del fm
        model = FNN(ind, emb, path, [64, 32], seed=0, device="cuda")
        os.remove(path)
        step = _adam(list(model.parameters()))
        ids = make_ids("zipf1.1", B, S, R, 2)
        feats = {f"c{s}": ids[:, s].contiguous() for s in range(S)}
        y = (torch.rand(B, device="cuda") < 0.3).float()
        t = timed([lambda: _train_step(model, step, feats, y)], max(5, args.reps // 2))[0]
        out["production"] = {"B": B, "S": S, "rows": R, "D": D, "units": [64, 32], "ids": "zipf1.1",
                             "step_ms": t, "examples_per_s": B / t * 1e3}
        del model, step
        torch.cuda.empty_cache()
        # the example's columns and shape, host string features hashed every step
        columns = ex.build_columns()
        path = os.path.join(tmp, "fm_ex.pt")
        FM(*columns, seed=0, device="cuda").export(path)
        model = FNN(*columns, path, [64, 32], seed=42, device="cuda")
        step = _adam(list(model.parameters()))
        gen = ex.synthetic_input_fn(3, 1024)
        batches = [next(gen) for _ in range(4)]
        it = iter(range(1 << 30))

        def ex_step():
            f, lab = batches[next(it) % len(batches)]
            _train_step(model, step, f, torch.as_tensor(lab, device="cuda"))
        t = timed([ex_step], args.reps)[0]
        out["example"] = {"B": 1024, "units": [64, 32], "step_ms": t}
    res["train_step"] = out
    print(json.dumps({"train_step": out}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join("bench_out", "bench_fnn.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fnn.py needs a CUDA device")
    res = {"card": card(), "torch": torch.__version__}
    bench_input(args, res)
    bench_layer0(args, res)
    bench_steps(args, res)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
