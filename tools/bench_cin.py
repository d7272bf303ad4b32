"""CIN kernels at the xDeepFM shape of BASELINE config C2 (26 fields, D = 16, CIN [128, 128], B = 65536):

  per kernel   CUDA-event times of dr_cin_fwd and dr_cin_bwd for layer 1 (x0, x0: m = h = 26) and layer 2
               (x0, x1: m = 26, h = 128), both with H = 128; useful TFLOP/s (forward 2*B*D*m*h*H flops, backward three
               times that) and their share of the 67 TFLOP/s data-sheet fp32 rate of an H100 SXM
  composition  layer 2's forward against the torch fp32 composition the reference's form maps to (materialised outer
               product + matmul, TF32 off, chunked over the batch so it fits), alternating in one process; the outputs
               are compared
  stack        the two-layer CIN forward + backward through the layer API (autograd), median / min / max
  xdeepfm      the whole XDeepFM training step (C2 tables 26 x 1M rows with first-order weights, CIN [128, 128], DNN
               [256, 32], BCE, row-sparse SGD fused into the embedding backward, SGD on the rest) through the Keras
               engine (`fit`, one batch per call), median / min / max over the timed steps

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to
<--out-dir>/bench_cin.json (default bench_out/, which git ignores).
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_dcn_step import card  # noqa: E402
from deep_recommenders_b200 import _lib, ops  # noqa: E402
from deep_recommenders_b200.keras.models.ranking.xdeepfm import CIN, XDeepFM  # noqa: E402

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
    ap.add_argument("--fields", type=int, default=26)
    ap.add_argument("--dim", type=int, default=16)
    ap.add_argument("--layers", default="128,128")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--chunk", type=int, default=4096, help="batch rows per chunk of the torch composition")
    ap.add_argument("--rows", type=int, default=1_000_000, help="rows per table of the XDeepFM step")
    ap.add_argument("--pool", type=int, default=4, help="id batches the XDeepFM step cycles through")
    ap.add_argument("--out-dir", default="bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cin.py measures on a GPU; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    lib = _lib.load()
    st = lambda: torch.cuda.current_stream().cuda_stream
    B, m, D = a.batch, a.fields, a.dim
    Hs = [int(v) for v in a.layers.split(",")]
    gen = torch.Generator(device="cuda").manual_seed(0)
    x0 = torch.randn((B, m, D), device="cuda", generator=gen) * 0.3
    out = {"config": f"C2 xDeepFM CIN {Hs}, fields={m}, D={D}, B={B}", "card": card(),
           "fp32_datasheet_tflops": FP32_PEAK_TFLOPS, "warmup": a.warmup, "iters": a.iters, "layers": []}

    x, h = x0, m
    ws = []
    for li, H in enumerate(Hs):
        w = torch.randn((1, m * h, H), device="cuda", generator=gen) * (1.0 / (m * h) ** 0.5)
        ws.append(w)
        y = torch.empty((B, H, D), device="cuda")
        pooled = torch.empty((B, H), device="cuda")
        same = li == 0
        top = li == len(Hs) - 1
        fwd = lambda: _lib.check(lib.dr_cin_fwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), None, B, m, h, D, H, 2,
                                                y.data_ptr(), pooled.data_ptr(), st()), "dr_cin_fwd")
        fwd()
        gy = None if top else torch.randn((B, H, D), device="cuda", generator=gen)
        gp = torch.randn((B, H), device="cuda", generator=gen)
        g_ws, gx0, gw = torch.empty_like(y), torch.empty_like(x0), torch.empty_like(w)
        gx = None if same else torch.empty_like(x)
        bwd = lambda: _lib.check(lib.dr_cin_bwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), y.data_ptr(),
                                                None if gy is None else gy.data_ptr(), gp.data_ptr(), B, m, h, D, H,
                                                2, int(same), g_ws.data_ptr(), gx0.data_ptr(),
                                                None if gx is None else gx.data_ptr(), gw.data_ptr(), None, st()),
                                 "dr_cin_bwd")
        flops = 2.0 * B * D * m * h * H
        rec = {"layer": li + 1, "m": m, "h": h, "H": H, "fwd_tflop": flops / 1e12, "bwd_tflop": 3 * flops / 1e12,
               "bwd_grads": "gpool" if top else "gy+gpool"}
        for name, fn, fl in (("fwd", fwd, flops), ("bwd", bwd, 3 * flops)):
            s = summary(timed(fn, a.warmup, a.iters))
            s["tflops_useful"] = fl / s["median_ms"] / 1e9
            s["share_of_fp32_datasheet"] = s["tflops_useful"] / FP32_PEAK_TFLOPS
            rec[name] = s
        out["layers"].append(rec)
        if not top:
            x, h = y.clone(), H

    # layer 2's forward against the materialised composition, alternating
    H = Hs[-1]
    w2 = ws[-1].view(m * h, H)
    y_k = torch.empty((B, H, D), device="cuda")
    y_t = torch.empty((B, H, D), device="cuda")

    def fused():
        _lib.check(lib.dr_cin_fwd(x0.data_ptr(), x.data_ptr(), w2.data_ptr(), None, B, m, h, D, H, 2, y_k.data_ptr(),
                                  None, st()), "dr_cin_fwd")

    def composition():
        for c0 in range(0, B, a.chunk):
            a0, a1 = x0[c0:c0 + a.chunk], x[c0:c0 + a.chunk]
            z = torch.einsum("bid,bjd->bdij", a0, a1).reshape(-1, m * h)         # [b*D, m*h] outer product
            y_t[c0:c0 + a.chunk] = torch.sigmoid(z @ w2).view(-1, D, H).transpose(1, 2)

    for _ in range(a.warmup):
        fused()
        composition()
    tk, tt = [], []
    for _ in range(a.iters):
        tk += timed(fused, 0, 1)
        tt += timed(composition, 0, 1)
    flops = 2.0 * B * D * m * h * H
    out["layer2_fwd_vs_composition"] = {
        "fused": {**summary(tk), "tflops_useful": flops / statistics.median(tk) / 1e9},
        "torch_fp32_composition": {**summary(tt), "tflops_useful": flops / statistics.median(tt) / 1e9,
                                   "chunk_rows": a.chunk},
        "speedup_median": statistics.median(tt) / statistics.median(tk),
        "max_abs_diff": (y_k - y_t).abs().max().item(),
    }

    # the two-layer stack through the layer API: forward (pooled outputs) + backward
    layers = [CIN(feature_map=H, activation="sigmoid", seed=i) for i, H in enumerate(Hs)]
    xin = x0.clone().requires_grad_()

    def stack_step():
        xx = xin
        pools = []
        for i, layer in enumerate(layers):
            xx, p = layer.call_pooled((xin, xx))
            pools.append(p)
        torch.cat(pools, 1).sum().backward()

    out["stack_fwd_bwd"] = summary(timed(stack_step, a.warmup, a.iters))
    del layers, xin

    # the whole XDeepFM step through the Keras engine
    lr = 0.01
    model = XDeepFM([a.rows] * m, D, cin_layers=Hs, dnn_units=(256, 32), sparse_lr=lr, seed=0, device="cuda")
    ids = [torch.randint(0, a.rows, (B, m), device="cuda", generator=gen) for _ in range(a.pool)]
    ys = [torch.randint(0, 2, (B,), device="cuda", generator=gen).float() for _ in range(a.pool)]
    from deep_recommenders_b200.keras.engine import SGD
    model.compile(loss="binary_crossentropy", optimizer=SGD(learning_rate=lr))
    k = [0]
    losses = []

    def xdeepfm_step():
        i = k[0] % a.pool
        k[0] += 1
        losses.append(model.fit(ids[i], ys[i], epochs=1, steps_per_epoch=1)["loss"][0])

    ms = timed(xdeepfm_step, a.warmup, a.iters)
    out["xdeepfm_step_keras"] = {**summary(ms), "examples_per_s": B / statistics.median(ms) * 1e3,
                                 "loss_first": losses[0], "loss_last": losses[-1],
                                 "model": f"XDeepFM {m}x{a.rows} D={D}, CIN {Hs}, DNN [256, 32], SGD lr={lr}"}
    print(json.dumps(out), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_cin.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
