"""Correctness + timing of the wgmma 3xTF32 GEMM variant against the FFMA variant and an fp64
reference, through the public Dense forward/backward (NN, NT and TN operand layouts)."""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200 import _lib, ops  # noqa: E402


def run(M, K, N, variant, act=1, iters=0):
    _lib.tune("gemm_variant", variant)
    g = torch.Generator(device="cuda").manual_seed(M + K + N)
    x = torch.randn(M, K, device="cuda", generator=g).requires_grad_(True)
    w = (torch.randn(K, N, device="cuda", generator=g) / K ** 0.5).requires_grad_(True)
    b = torch.randn(N, device="cuda", generator=g).requires_grad_(True)
    gy = torch.randn(M, N, device="cuda", generator=g)
    y = ops.DenseFn.apply(x, w, b, act)
    y.backward(gy)
    torch.cuda.synchronize()
    res = dict(y=y.detach(), gx=x.grad, gw=w.grad, gb=b.grad, x=x.detach(), w=w.detach(), b=b.detach(), gy=gy)
    if iters:
        lib = _lib.load()
        st = torch.cuda.current_stream().cuda_stream
        yb = torch.empty_like(y)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            lib.dr_dense_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, act, yb.data_ptr(), st)
        e0.record()
        for _ in range(iters):
            lib.dr_dense_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, act, yb.data_ptr(), st)
        e1.record()
        torch.cuda.synchronize()
        res["fwd_ms"] = e0.elapsed_time(e1) / iters
        gz = torch.empty_like(gy)
        gx = torch.empty_like(x)
        gw = torch.empty_like(w)
        gb = torch.empty_like(b)
        e0.record()
        for _ in range(iters):
            lib.dr_dense_bwd(x.data_ptr(), w.data_ptr(), yb.data_ptr(), gy.data_ptr(), M, K, N, act, gz.data_ptr(),
                             gx.data_ptr(), gw.data_ptr(), gb.data_ptr(), st)
        e1.record()
        torch.cuda.synchronize()
        res["bwd_ms"] = e0.elapsed_time(e1) / iters
    return res


def main():
    _lib.enable_tensor_core_gemm(3 << 30)
    out = []
    shapes = [(256, 64, 128), (300, 96, 200), (1000, 416, 256), (4096, 256, 416), (65536, 416, 256), (65536, 256, 256),
              (131072, 832, 832)]
    if os.environ.get("DR_SHAPES") == "big":
        shapes = [(65536, 416, 256), (131072, 832, 832)]
    bns = [int(x) for x in os.environ.get("DR_BN", "0").split(",")]
    for (M, K, N), bn in [(sh, bn) for sh in shapes for bn in bns]:
        _lib.tune("gemm_bn", bn)
        big = M >= 65536
        r0 = run(M, K, N, 0, iters=5 if (big and bn == bns[0]) else 0)
        r1 = run(M, K, N, 1, iters=5 if big else 0)
        x, w, b, gy = (r0[k].double() for k in ("x", "w", "b", "gy"))
        if M <= 65536 and K * N <= 416 * 416:
            z = x @ w + b
            y = torch.relu(z)
            gz = gy * (z > 0)
            ref = dict(y=y, gx=gz @ w.T, gw=x.T @ gz, gb=gz.sum(0))
            sc = dict(y=(x.abs() @ w.abs() + b.abs()), gx=gz.abs() @ w.abs().T, gw=x.abs().T @ gz.abs(), gb=gz.abs().sum(0))
        else:
            ref = None
        line = dict(M=M, K=K, N=N, bn=bn)
        for k in ("y", "gx", "gw", "gb"):
            if ref is not None:
                for name, r in (("ffma", r0), ("tc", r1)):
                    err = ((r[k].double() - ref[k]).abs() / (sc[k] + 1e-30)).max().item()
                    line[f"{k}_{name}_relerr"] = err
            line[f"{k}_tc_vs_ffma"] = ((r1[k] - r0[k]).abs().max() / (r0[k].abs().max() + 1e-30)).item()
        for k in ("fwd_ms", "bwd_ms"):
            if k in r0:
                line[f"{k}_ffma"] = r0[k]
        if "fwd_ms" in r0:
            fl = 2.0 * M * K * N
            line["fwd_tflops_ffma"] = fl / r0["fwd_ms"] / 1e9
            line["bwd_tflops_ffma"] = 2 * fl / r0["bwd_ms"] / 1e9
        if "fwd_ms" in r1:
            fl = 2.0 * M * K * N
            line["fwd_ms_tc"], line["bwd_ms_tc"] = r1["fwd_ms"], r1["bwd_ms"]
            line["fwd_tflops_tc"] = fl / r1["fwd_ms"] / 1e9
            line["bwd_tflops_tc"] = 2 * fl / r1["bwd_ms"] / 1e9
        print(json.dumps(line), flush=True)
        out.append(line)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open("gpurun_out/check_gemm_tc.json", "w"), indent=1)


if __name__ == "__main__":
    main()
