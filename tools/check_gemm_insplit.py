"""Variant 2 of the wgmma GEMM (hi/lo split inside the kernel) against variant 1 (pre-split planes) and fp64,
through the public Dense forward / backward (NN, NT, TN operand layouts, ragged tiles, split-K weight gradient),
plus timing at the C2 layer shapes.  Exit code 1 on any mismatch.  Writes gpurun_out/check_gemm_insplit.json."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200 import _lib  # noqa: E402
from check_gemm_tc import run  # noqa: E402


def main():
    _lib.enable_tensor_core_gemm(3 << 30)
    ok, out = True, []
    shapes = [(256, 64, 128), (300, 96, 200), (1000, 416, 256), (4096, 256, 416), (65536, 416, 256), (65536, 256, 256)]
    for M, K, N in shapes:
        big = M >= 65536
        r1 = run(M, K, N, 1, iters=5 if big else 0)
        r2 = run(M, K, N, 2, iters=5 if big else 0)
        x, w, b, gy = (r1[k].double() for k in ("x", "w", "b", "gy"))
        z = x @ w + b
        gz = gy * (z > 0)
        ref = dict(y=torch.relu(z), gx=gz @ w.T, gw=x.T @ gz, gb=gz.sum(0))
        sc = dict(y=(x.abs() @ w.abs() + b.abs()), gx=gz.abs() @ w.abs().T, gw=x.abs().T @ gz.abs(), gb=gz.abs().sum(0))
        line = dict(M=M, K=K, N=N)
        for k in ("y", "gx", "gw", "gb"):
            e2 = ((r2[k].double() - ref[k]).abs() / (sc[k] + 1e-30)).max().item()
            e1 = ((r1[k].double() - ref[k]).abs() / (sc[k] + 1e-30)).max().item()
            line[f"{k}_v1_relerr"], line[f"{k}_v2_relerr"] = e1, e2
            line[f"{k}_v2_eq_v1"] = bool(torch.equal(r1[k], r2[k]))
            if not (e2 <= 1e-5):
                ok = False
        if big:
            fl = 2.0 * M * K * N
            line.update(fwd_ms_v1=r1["fwd_ms"], fwd_ms_v2=r2["fwd_ms"], bwd_ms_v1=r1["bwd_ms"], bwd_ms_v2=r2["bwd_ms"],
                        fwd_tflops_v2=fl / r2["fwd_ms"] / 1e9, bwd_tflops_v2=2 * fl / r2["bwd_ms"] / 1e9)
        print(json.dumps(line), flush=True)
        out.append(line)
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open("gpurun_out/check_gemm_insplit.json", "w"), indent=1)
    print("INSPLIT_OK" if ok else "INSPLIT_MISMATCH", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
