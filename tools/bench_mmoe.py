"""Multi-gate mixture of experts: the fused gate-softmax + mixture kernel and the whole MMoE train step.

  mix    CUDA-event times of dr_moe_mix_fwd and of the forward + dr_moe_mix_bwd, against the torch fp32 composition of
         the reference graph (tf.stack of the E expert outputs, then per used gate a softmax and a [B,1,E] @ [B,E,H]
         bmm; autograd for the backward), alternating in one process.  Achieved GB/s count the algorithmic bytes
         (every input read once, every output written once) and are given as a share of the 3.35 TB/s HBM3 data-sheet
         bandwidth of an H100 SXM.  The largest output and gradient differences between the two are reported.
  step   the whole MMoE train step (forward, MSE per task, backward, torch Adam) with the fused kernel and with the
         torch composition in its place, alternating, at the reference example's shape (B 512, 256 inputs, E = T = 2,
         experts [64, 32], tasks [32, 10]) and at a production-like shape (B 65536, 512 inputs, E = 8 experts
         [256, 128], T = 2 tasks [64, 32]); with the library's kernel launches per step.

The card's name and power limit are read in the same run.  Prints one JSON line and writes it to
<--out-dir>/bench_mmoe.json (default bench_out/, which git ignores).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from bench_dcn_step import card  # noqa: E402
from bench_din import summary, timed  # noqa: E402
from deep_recommenders_b200 import _lib, ops  # noqa: E402
from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders.estimator.models.multi_task_learning import MMoE  # noqa: E402

HBM_TBS = 3.35


def composition(experts, logits, E, T, H):
    """The reference graph on our layouts: stack the E expert blocks, then per gate softmax + bmm + squeeze."""
    stack = torch.stack([experts[:, e * H:(e + 1) * H] for e in range(E)], dim=1)          # [B, E, H]
    outs = [torch.bmm(torch.softmax(logits[:, t * E:(t + 1) * E], -1).unsqueeze(1), stack).squeeze(1)
            for t in range(T)]
    return torch.cat(outs, dim=1)


def bench_mix(B, E, T, H, iters, reps):
    torch.manual_seed(0)
    ex = torch.randn(B, E * H, device="cuda")
    lg = torch.randn(B, T * E, device="cuda") * 2
    go = torch.randn(B, T * H, device="cuda")
    exg, lgg = ex.clone().requires_grad_(), lg.clone().requires_grad_()

    def ours_fwd():
        return ops.MoEMixFn.apply(ex, lg, T)

    def ours_fb():
        out = ops.MoEMixFn.apply(exg, lgg, T)
        return torch.autograd.grad(out, (exg, lgg), go)

    def ref_fwd():
        return composition(ex, lg, E, T, H)

    def ref_fb():
        out = composition(exg, lgg, E, T, H)
        return torch.autograd.grad(out, (exg, lgg), go)

    res = {k: [] for k in ("ours_fwd", "ours_fwd_bwd", "torch_fwd", "torch_fwd_bwd")}
    for _ in range(reps):
        res["ours_fwd"] += timed(ours_fwd, 3, iters)
        res["torch_fwd"] += timed(ref_fwd, 3, iters)
        res["ours_fwd_bwd"] += timed(ours_fb, 3, iters)
        res["torch_fwd_bwd"] += timed(ref_fb, 3, iters)
    fwd_bytes = 4 * (B * E * H + 2 * B * T * E + B * T * H)
    bwd_bytes = 4 * (2 * B * E * H + 2 * B * T * E + B * T * H)
    out = {"shape": {"B": B, "E": E, "T": T, "H": H}, "fwd_bytes": fwd_bytes, "bwd_bytes": bwd_bytes}
    for k, v in res.items():
        s = summary(v)
        nbytes = fwd_bytes + (bwd_bytes if k.endswith("bwd") else 0)
        s["GB_per_s"] = nbytes / (s["median_ms"] * 1e-3) / 1e9
        s["share_of_hbm_datasheet"] = s["GB_per_s"] / (HBM_TBS * 1e3)
        out[k] = s
    out["speedup_fwd"] = out["torch_fwd"]["median_ms"] / out["ours_fwd"]["median_ms"]
    out["speedup_fwd_bwd"] = out["torch_fwd_bwd"]["median_ms"] / out["ours_fwd_bwd"]["median_ms"]
    a, b = ours_fb(), ref_fb()
    out["max_abs_diff"] = {"out": float((ours_fwd() - ref_fwd()).abs().max()),
                           "g_experts": float((a[0] - b[0]).abs().max()),
                           "g_logits": float((a[1] - b[1]).abs().max())}
    return out


def bench_step(B, D, E, T, eu, tu, iters, reps):
    torch.manual_seed(0)
    cols = [fc.numeric_column("C{}".format(i)) for i in range(D)]
    m = MMoE(cols, num_tasks=T, num_experts=E, expert_hidden_units=eu, task_hidden_units=tu, seed=0)
    opt = torch.optim.Adam(list(m.parameters()), lr=1e-3, eps=1e-8)
    x = torch.randn(B, D, device="cuda")
    y = torch.randn(B, T, device="cuda")
    H = eu[-1]

    def make(fused):
        def step():
            experts = m._experts(x)
            logits = m.gating_logits(x)
            mixed = ops.MoEMixFn.apply(experts, logits, T) if fused else composition(experts, logits, E, T, H)
            out = m._tasks(mixed)
            loss = sum(((out[:, t] - y[:, t]) ** 2).mean() for t in range(T))
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            return loss
        return step

    fused, ref = make(True), make(False)
    res = {"fused": [], "torch_mix": []}
    for _ in range(reps):
        res["fused"] += timed(fused, 3, iters)
        res["torch_mix"] += timed(ref, 3, iters)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fused()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    out = {"shape": {"B": B, "inputs": D, "E": E, "T": T, "experts": eu, "tasks": tu}}
    for k, v in res.items():
        out[k] = summary(v)
    out["speedup"] = out["torch_mix"]["median_ms"] / out["fused"]["median_ms"]
    out["library_launches_per_step"] = launches
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out-dir", default="bench_out")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mmoe.py needs an H100"
    result = {"card": card(),
              "mix": [bench_mix(65536, 8, 2, 128, args.iters, args.reps),
                      bench_mix(512, 2, 2, 32, args.iters, args.reps),
                      bench_mix(65536, 16, 4, 256, args.iters, args.reps)],
              "step": [bench_step(512, 256, 2, 2, [64, 32], [32, 10], args.iters, args.reps),
                       bench_step(65536, 512, 8, 2, [256, 128], [64, 32], max(args.iters // 5, 5), args.reps)]}
    line = json.dumps(result)
    print(line)
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "bench_mmoe.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
