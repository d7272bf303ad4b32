#!/usr/bin/env python
"""Times the three GEMMs of one Dense layer (forward, dX, dW) through the C-ABI at the tower shapes of C2 / C5, per rank
batch M, under the tile-width knob.  Buffers rotate (3 sets) so the operands come from HBM as in a train step.

The 256 -> 32 layer of C2 is timed as the step runs it: its dX is the chained form (dr_dense_bwd_chain), whose epilogue
multiplies by relu'(layer-0 output) (EPI_ACTGRAD).

Then the layer-0 forward (M = 65536, N = 256, 128 x 128 tiles) is swept over K under a plain store (EPI_STORE, through
dr_debug_gemm) and under bias + relu (EPI_BIAS_ACT, through dr_dense_fwd).  Every CTA of the persistent grid owns the
same number of tiles, so time = tiles per CTA x (fixed cost per tile + K / 32 x cost per k-block): the least-squares
line through (k-blocks, time) gives the fixed per-tile cost as its intercept and the per-k-block cost as its slope.

cache=1 times every GEMM as a train step runs it: the plane cache is switched on (and emptied) before each call, so the
forward and dX take B's hi / lo planes from the workspace (gemm_tc_wplanes_kernel) and each call pays for its own split of
B, as the step pays once per layout of each weight.  cache=0 (the default) is the in-kernel split of every call.
usage: bench_gemm_shapes.py [cache=0|1] [KEY=VALUE ...]   -> one JSON line per shape, one per swept epilogue, one for
the card"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from deep_recommenders_b200 import _lib
from deep_recommenders_b200._lib import check

knobs = [a for a in sys.argv[1:] if "=" in a and not a.startswith("cache=")]
CACHE = any(a == "cache=1" for a in sys.argv[1:])
for kv in knobs:
    k, v = kv.split("=")
    _lib.tune(k, int(v))
lib = _lib.load()
if CACHE:
    _lib.set_workspace(256 << 20)
dev = torch.device("cuda", 0)
SHAPES = [(65536, 416, 256), (65536, 256, 32), (8192, 3328, 512), (16384, 3328, 512), (65536, 3328, 512),
          (8192, 512, 256)]
SWEEP_K = [32, 64, 128, 256, 416]
RELU = 1
R = 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.splitlines()[0]
        name, limit, sm = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": limit, "sm_clock": sm}
    except Exception as e:  # noqa: BLE001 -- the card's name still identifies the run
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({type(e).__name__})"}


def timed(fn, iters=6):
    if CACHE:
        fn0 = fn

        def fn(i):
            check(lib.dr_gemm_plane_cache(1), "plane cache")   # empty: this call splits its own B
            fn0(i)
    for i in range(2):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


print(json.dumps({"card": card(), "knobs": knobs, "cache": CACHE}), flush=True)
st = torch.cuda.current_stream().cuda_stream
for M, K, N in SHAPES:
    xs = [torch.randn(M, K, device=dev).relu_() for _ in range(R)]     # a layer's input is the relu output below it
    gys = [torch.randn(M, N, device=dev) for _ in range(R)]
    ys = [torch.empty(M, N, device=dev) for _ in range(R)]
    gxs = [torch.empty(M, K, device=dev) for _ in range(R)]
    w = torch.randn(K, N, device=dev) / K ** 0.5
    b = torch.zeros(N, device=dev)
    gw = torch.empty(K, N, device=dev)
    fwd = lambda i: check(lib.dr_dense_fwd(xs[i % R].data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, RELU,
                                           ys[i % R].data_ptr(), st), "fwd")
    dx = lambda i: check(lib.dr_dense_bwd(xs[i % R].data_ptr(), w.data_ptr(), None, gys[i % R].data_ptr(), M, K, N, 0, None,
                                          gxs[i % R].data_ptr(), None, None, st), "dx")
    dx_chain = lambda i: check(lib.dr_dense_bwd_chain(xs[i % R].data_ptr(), w.data_ptr(), None, gys[i % R].data_ptr(), M,
                                                      K, N, 0, None, gxs[i % R].data_ptr(), None, None,
                                                      xs[i % R].data_ptr(), RELU, st), "dx_chain")
    dw = lambda i: check(lib.dr_dense_bwd(xs[i % R].data_ptr(), w.data_ptr(), None, gys[i % R].data_ptr(), M, K, N, 0, None,
                                          None, gw.data_ptr(), None, st), "dw")
    t = {"fwd_us": timed(fwd), "dx_us": timed(dx), "dx_chain_us": timed(dx_chain), "dw_us": timed(dw)}
    fl = 2.0 * M * K * N
    print(json.dumps({"M": M, "K": K, "N": N, "knobs": knobs, "cache": CACHE, **{k: round(v, 1) for k, v in t.items()},
                      **{k.replace("_us", "_tflops"): round(fl / v / 1e6, 1) for k, v in t.items()}}), flush=True)
    del xs, gys, ys, gxs
    torch.cuda.empty_cache()

# ---- layer-0 forward swept over K: fixed cost per tile against cost per k-block ----
M, N = 65536, 256
sms = torch.cuda.get_device_properties(0).multi_processor_count
tiles = (M // 128) * (N // 128)
tiles_per_cta = -(-tiles // sms)
Kmax = max(SWEEP_K)
xs = [torch.randn(M, Kmax, device=dev) for _ in range(R)]
ys = [torch.empty(M, N, device=dev) for _ in range(R)]
b = torch.randn(N, device=dev)
for epi in ("store", "bias_relu"):
    times = []
    for K in SWEEP_K:
        xk = [x[:, :K].contiguous() for x in xs]
        w = torch.randn(K, N, device=dev) / K ** 0.5
        if epi == "store":
            fn = lambda i: check(lib.dr_debug_gemm(xk[i % R].data_ptr(), w.data_ptr(), ys[i % R].data_ptr(), M, N, K, 0, 0,
                                                   st), "gemm")
        else:
            fn = lambda i: check(lib.dr_dense_fwd(xk[i % R].data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, RELU,
                                                  ys[i % R].data_ptr(), st), "fwd")
        times.append(timed(fn, iters=30))
        del xk
    kb = np.array(SWEEP_K, dtype=np.float64) / 32
    slope, icpt = np.polyfit(kb, np.array(times), 1)
    t_full = times[SWEEP_K.index(416)]
    print(json.dumps({"sweep": "layer0_fwd", "epi": epi, "cache": CACHE, "M": M, "N": N, "K": SWEEP_K,
                      "us": [round(v, 1) for v in times], "tiles_per_cta": tiles_per_cta,
                      "intercept_us": round(icpt, 1), "slope_us_per_kblock": round(slope, 2),
                      "per_tile_fixed_us": round(icpt / tiles_per_cta, 2),
                      "per_kblock_per_tile_us": round(slope / tiles_per_cta, 3),
                      "intercept_share_of_K416": round(icpt / t_full, 3)}), flush=True)
if CACHE:
    check(lib.dr_gemm_plane_cache(0), "plane cache")
