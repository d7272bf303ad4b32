"""DIN target attention at B = 65536, D = 32, U = 36 (DIN's default attention width), Subtract, relu:

  per kernel   CUDA-event times of dr_din_attn_fwd (score + pooled) and dr_din_attn_bwd (g_pooled only: the DIN
               model's case) for each --seq-lens T; useful TFLOP/s counted in the reference's form (per position
               2*3D*U for the hidden Dense, 2*U for Dense(1), 2*D for the pooling; the backward as twice the forward,
               the recompute of h not counted) and their share of the 67 TFLOP/s data-sheet fp32 rate of an H100 SXM
  composition  the forward against the torch fp32 composition the reference's form maps to (materialised [k | q | k-q]
               concat, matmul, relu, matmul, weighted sum; TF32 off; chunked over the batch so it fits), alternating in
               one process; the outputs are compared
  din          the whole DIN training step (item table --rows x D, T = the last --seq-lens, 3 context slots, MLP
               [200, 80] with Dice, BCE, row-sparse SGD fused into the gathers' backward, SGD on the rest) through the
               Keras engine (`fit`, one batch per call), median / min / max over the timed steps

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to
<--out-dir>/bench_din.json (default bench_out/, which git ignores).
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_dcn_step import card  # noqa: E402
from deep_recommenders_b200 import _lib  # noqa: E402
from deep_recommenders_b200.keras.models.ranking.din import DIN  # noqa: E402

FP32_PEAK_TFLOPS = 67.0


def summary(ms):
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "n": len(ms)}


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ev = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        ev.append((e0, e1))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=32)
    ap.add_argument("--units", type=int, default=36)
    ap.add_argument("--seq-lens", default="50,200")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--chunk", type=int, default=2048, help="examples per chunk of the torch composition")
    ap.add_argument("--rows", type=int, default=1_000_000, help="item table rows of the DIN step")
    ap.add_argument("--step-batch", type=int, default=8192, help="batch of the DIN step")
    ap.add_argument("--out-dir", default="bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_din.py measures on a GPU; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    lib = _lib.load()
    st = lambda: torch.cuda.current_stream().cuda_stream
    B, D, U = a.batch, a.dim, a.units
    gen = torch.Generator(device="cuda").manual_seed(0)
    out = {"config": f"DIN attention B={B}, D={D}, U={U}, Subtract, relu", "card": card(),
           "fp32_datasheet_tflops": FP32_PEAK_TFLOPS, "warmup": a.warmup, "iters": a.iters, "seq": []}
    w1 = torch.randn((3 * D, U), device="cuda", generator=gen) * (1.0 / (3 * D) ** 0.5)
    b1 = torch.randn((U,), device="cuda", generator=gen) * 0.1
    w2 = torch.randn((U, 1), device="cuda", generator=gen) * (1.0 / U ** 0.5)
    b2 = torch.zeros((1,), device="cuda")
    q = torch.randn((B, D), device="cuda", generator=gen) * 0.3
    for T in [int(v) for v in a.seq_lens.split(",")]:
        keys = torch.randn((B, T, D), device="cuda", generator=gen) * 0.3
        score = torch.empty((B, T), device="cuda")
        pooled = torch.empty((B, D), device="cuda")
        gp = torch.randn((B, D), device="cuda", generator=gen)
        gk, gq = torch.empty_like(keys), torch.empty_like(q)
        gw1, gb1, gw2, gb2 = torch.empty_like(w1), torch.empty_like(b1), torch.empty_like(w2), torch.empty_like(b2)

        def fwd():
            _lib.check(lib.dr_din_attn_fwd(keys.data_ptr(), q.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                           b2.data_ptr(), B, T, D, U, 1, 1, score.data_ptr(), pooled.data_ptr(),
                                           st()), "dr_din_attn_fwd")

        def bwd():
            _lib.check(lib.dr_din_attn_bwd(keys.data_ptr(), q.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                           b2.data_ptr(), gp.data_ptr(), None, B, T, D, U, 1, 1, gk.data_ptr(),
                                           gq.data_ptr(), gw1.data_ptr(), gb1.data_ptr(), gw2.data_ptr(),
                                           gb2.data_ptr(), st()), "dr_din_attn_bwd")

        flops = 2.0 * B * T * (3 * D * U + U + D)
        rec = {"T": T, "fwd_tflop": flops / 1e12, "bwd_tflop": 2 * flops / 1e12}
        for name, fn, fl in (("fwd", fwd, flops), ("bwd", bwd, 2 * flops)):
            s = summary(timed(fn, a.warmup, a.iters))
            s["tflops_useful"] = fl / s["median_ms"] / 1e9
            s["share_of_fp32_datasheet"] = s["tflops_useful"] / FP32_PEAK_TFLOPS
            rec[name] = s

        pooled_t = torch.empty_like(pooled)

        def composition():
            for c0 in range(0, B, a.chunk):
                k = keys[c0:c0 + a.chunk]
                qb = q[c0:c0 + a.chunk, None, :].expand_as(k)
                u = torch.cat([k, qb, k - qb], -1)                                     # [chunk, T, 3D]
                s = torch.relu(u @ w1 + b1) @ w2 + b2                                  # [chunk, T, 1]
                pooled_t[c0:c0 + a.chunk] = (s * k).sum(1)

        for _ in range(a.warmup):
            fwd()
            composition()
        tk, tt = [], []
        for _ in range(a.iters):
            tk += timed(fwd, 0, 1)
            tt += timed(composition, 0, 1)
        rec["fwd_vs_composition"] = {
            "fused": {**summary(tk), "tflops_useful": flops / statistics.median(tk) / 1e9},
            "torch_fp32_composition": {**summary(tt), "tflops_useful": flops / statistics.median(tt) / 1e9,
                                       "chunk_examples": a.chunk},
            "speedup_median": statistics.median(tt) / statistics.median(tk),
            "max_abs_diff_pooled": (pooled - pooled_t).abs().max().item(),
            "max_abs_pooled": pooled_t.abs().max().item(),
        }
        out["seq"].append(rec)
        del keys, gk, score

    # the whole DIN step through the Keras engine
    T = int(a.seq_lens.split(",")[-1])
    Bs, lr = a.step_batch, 0.01
    model = DIN(a.rows, D, context_rows=[1000, 100, 10], att_units=U, dnn_units=(200, 80), sparse_lr=lr, seed=0,
                device="cuda")
    pool = 4
    batches = []
    for _ in range(pool):
        ctx = torch.stack([torch.randint(0, r, (Bs,), device="cuda", generator=gen) for r in (1000, 100, 10)], 1)
        item = torch.randint(0, a.rows, (Bs,), device="cuda", generator=gen)
        hist = torch.randint(0, a.rows, (Bs, T), device="cuda", generator=gen)
        lens = torch.randint(1, T + 1, (Bs, 1), device="cuda", generator=gen)
        hist[torch.arange(T, device="cuda")[None, :] >= lens] = -1                    # padded histories
        batches.append(((ctx, item, hist), torch.randint(0, 2, (Bs,), device="cuda", generator=gen).float()))
    from deep_recommenders_b200.keras.engine import SGD
    model.compile(loss="binary_crossentropy", optimizer=SGD(learning_rate=lr))
    k = [0]
    losses = []

    def din_step():
        x, y = batches[k[0] % pool]
        k[0] += 1
        losses.append(model.fit(x, y, epochs=1, steps_per_epoch=1)["loss"][0])

    ms = timed(din_step, a.warmup, a.iters)
    out["din_step_keras"] = {**summary(ms), "examples_per_s": Bs / statistics.median(ms) * 1e3,
                             "loss_first": losses[0], "loss_last": losses[-1],
                             "model": f"DIN items={a.rows} D={D} T={T} (padded to random lengths), 3 context slots, "
                                      f"att {U} relu Subtract, MLP [200, 80] Dice, B={Bs}, SGD lr={lr}"}
    print(json.dumps(out), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_din.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
