"""BASELINE config C3 (DCN: 26 slots x 1M rows, D = 32 -> d = 832, 3 full-matrix Cross + DNN [512, 256, 128],
B = 131072), one training step two ways in ONE process, alternating step by step:

  autograd   the layer API's autograd graph (the `step_c3` of bench_configs.py: model.logits -> BCE -> backward ->
             dr_sgd_step per parameter, row-sparse SGD fused into the embedding backward)
  trainer    DCNTrainStep, one CUDA-graph replay per step

Both start from the same weights (same seed) and see the same batches, so their losses are compared step by step at
the timed size.  Step times are CUDA-event times of every single step (median, min, max, quartiles); the trainer's
kernel groups come from `profile_kernels` (eager launches, an event between groups).  The card's name and power limit
are read in the same run and written beside the numbers.  Prints one JSON line and writes it to
<--out-dir>/bench_dcn_step.json (default bench_out/, which git ignores).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_configs import dense_sgd  # noqa: E402
from deep_recommenders_b200 import DCNTrainStep, ops  # noqa: E402
from deep_recommenders_b200.keras.layers import DCN  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # the numbers are still worth having; the missing context is stated
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({type(e).__name__})"}


def summary(ms):
    q = statistics.quantiles(ms, n=4)
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "q1_ms": q[0], "q3_ms": q[2],
            "steps": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=131072)
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--pool", type=int, default=4)
    ap.add_argument("--out-dir", default="bench_out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dcn_step.py measures on a GPU; none is visible")
    B, S, D, lr = a.batch, 26, 32, 0.01
    units = [512, 256, 128]
    mk = lambda: DCN([a.rows] * S, D, num_cross=3, dnn_units=units, sparse_lr=lr, seed=0, device="cuda")
    m_ag, m_tr = mk(), mk()
    gen = torch.Generator(device="cuda").manual_seed(0)
    ids = [torch.randint(0, a.rows, (B, S), device="cuda", generator=gen) for _ in range(a.pool)]
    ys = [torch.randint(0, 2, (B, 1), device="cuda", generator=gen).float() for _ in range(a.pool)]
    m_ag.logits(ids[0])                                       # builds the lazily created layers
    dense = [p for n, p in m_ag.named_parameters() if not n.startswith("embeddings.")]
    tr = DCNTrainStep(m_tr, batch_size=B, lr=lr)
    tr.ids.copy_(ids[0])
    tr.capture()

    def step_autograd(k):
        z = m_ag.logits(ids[k % a.pool])
        loss, gz, _ = ops.bce_with_logits(z, ys[k % a.pool])
        z.backward(gz.view_as(z))
        dense_sgd(dense, lr)
        return loss

    def step_trainer(k):
        return tr.step(ids[k % a.pool], ys[k % a.pool])

    paths = {"autograd": step_autograd, "trainer": step_trainer}
    events = {p: [] for p in paths}
    losses = {p: [] for p in paths}
    for k in range(a.warmup + a.steps):
        for p, fn in paths.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loss = fn(k)
            e1.record()
            losses[p].append(loss.clone())
            if k >= a.warmup:
                events[p].append((e0, e1))
    torch.cuda.synchronize()
    ms = {p: [e0.elapsed_time(e1) for e0, e1 in ev] for p, ev in events.items()}
    la = torch.cat(losses["autograd"]).double().cpu()
    lt = torch.cat(losses["trainer"]).double().cpu()
    rel = ((la - lt).abs() / la.abs()).max().item()
    flops = 3 * (3 * 2 * B * 832 * 832 + 2 * B * (832 * units[0] + units[0] * units[1] + units[1] * units[2]))
    out = {"config": f"C3 DCN {S}x{a.rows} D={D} B={B}, 3 Cross(832) + DNN{units}, SGD lr={lr}", "card": card(),
           "warmup_steps_each": a.warmup, "loss_first": [la[0].item(), lt[0].item()],
           "loss_last": [la[-1].item(), lt[-1].item()], "loss_max_rel_diff": rel, "loss_tolerance": 1e-4,
           "launches_per_step_trainer": tr.launches_per_step}
    for p in paths:
        s = summary(ms[p])
        s["examples_per_s"] = B / s["median_ms"] * 1e3
        s["gemm_tflops_useful"] = flops / s["median_ms"] / 1e9
        out[p] = s
    out["speedup_median"] = out["autograd"]["median_ms"] / out["trainer"]["median_ms"]
    _, groups = tr.profile_kernels(ids, ys, iters=10)         # last: these are real steps on the trainer's model only
    out["trainer_kernel_groups_us"] = {k: round(v * 1e3, 1) for k, v in groups.items()}
    out["trainer_kernel_groups_sum_ms"] = sum(groups.values())
    print(json.dumps(out), flush=True)
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "bench_dcn_step.json"), "w") as f:
        json.dump(out, f, indent=1)
    if not rel <= out["loss_tolerance"]:
        sys.exit(f"losses of the two paths differ by {rel:.3g} relative (tolerance {out['loss_tolerance']})")


if __name__ == "__main__":
    main()
