#!/usr/bin/env python
"""What optimizers.KerasAdam costs next to the engine's Adam (torch.optim.Adam), through the Keras engine's fit().

  * Keras DeepFM at the C2 shape (26 tables of 2^20 rows, D = 16, tower [256, 32], B = 65536, [B, S] id tensors,
    uniform ids), three ways: engine.Adam(), KerasAdam(tables="dense") (TF's update swept over every table row) and
    KerasAdam() (the tables row-sparse).  ms per step on a device-synchronised host clock, after a warm-up, as the median
    and range of several repeats of K steps; peak memory allocated (KerasAdam() keeps 64 floats of state per row at
    D = 16; the dense forms keep m, v and a gradient as wide as the 32-float fused row).
  * The reference Transformer example's step (vocabulary 5000, length 128, batch 128, Adam(beta_2=0.98, epsilon=1e-9))
    with engine.Adam and with KerasAdam: ms per step likewise, and the kernels one optimizer step launches, counted by
    torch.profiler in a run of its own.

The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line per measurement.

    python tools/bench_keras_adam.py [--steps K --warmup W --repeats R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))

from deep_recommenders_b200 import feature_column as fc  # noqa: E402
from deep_recommenders_b200.keras import engine as K  # noqa: E402
from deep_recommenders_b200.keras.models.ranking import DeepFM  # noqa: E402
from deep_recommenders_b200.optimizers import KerasAdam  # noqa: E402

S, ROWS, D, UNITS, B = 26, 1 << 20, 16, [256, 32], 65536
PROFILED_STEPS = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_fit(model, batches, steps, warmup, repeats):
    """(median, min, max) ms per step of fit() over `steps` batches, after `warmup` steps."""
    model.fit(batches(warmup), epochs=1, steps_per_epoch=warmup)
    ms = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.fit(batches(steps), epochs=1, steps_per_epoch=steps)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3 / steps)
    return float(np.median(ms)), float(min(ms)), float(max(ms))


def deepfm(a):
    gen = torch.Generator(device="cuda").manual_seed(0)
    pool = [(torch.randint(0, ROWS, (B, S), device="cuda", generator=gen),
             torch.randint(0, 2, (B, 1), device="cuda", generator=gen).float()) for _ in range(8)]
    batches = lambda n: [pool[i % len(pool)] for i in range(n)]
    cats = [fc.categorical_column_with_identity(f"c{s}", ROWS) for s in range(S)]
    for name, make in (("engine.Adam", lambda: K.Adam()), ("KerasAdam(tables='dense')", lambda: KerasAdam(tables="dense")),
                       ("KerasAdam()", lambda: KerasAdam())):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        model = DeepFM([fc.indicator_column(c) for c in cats], [fc.embedding_column(c, D) for c in cats],
                       dnn_units_size=UNITS, seed=0, device="cuda")
        model.compile(loss="binary_crossentropy", optimizer=make())
        med, lo, hi = time_fit(model, batches, a.steps, a.warmup, a.repeats)
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print(json.dumps({"model": "DeepFM C2", "optimizer": name, "ms_per_step": med, "ms_min": lo, "ms_max": hi,
                          "peak_gib": peak, "steps": a.steps, "repeats": a.repeats, "card": card()}), flush=True)
        del model
        torch.cuda.synchronize()


def transformer(a):
    import train_transformer_on_synthetic_keras as ex
    batch = next(ex.synthetic_batches(5000, 128, 128, 0))
    batches = lambda n: [batch] * n
    kw = dict(beta_1=0.9, beta_2=0.98, epsilon=1e-9)
    for name, make in (("engine.Adam", lambda: K.Adam(**kw)), ("KerasAdam", lambda: KerasAdam(**kw))):
        torch.manual_seed(0)
        model = ex.TransformerClassifier(5000, 128, seed=0)
        model.compile(optimizer=make(), loss="categorical_crossentropy")
        med, lo, hi = time_fit(model, batches, a.steps, a.warmup, a.repeats)
        # the gradients of the last step are still set: profile PROFILED_STEPS more optimizer steps on their own
        opt = model._optimizer
        opt.step()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(PROFILED_STEPS):
                opt.step()
            torch.cuda.synchronize()
        kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and not e.name.startswith(("Memcpy", "Memset", "Optimizer."))]   # not the step's annotation
        n_vars = sum(1 for p in model.parameters() if p.requires_grad)
        print(json.dumps({"model": "Transformer example", "optimizer": name, "ms_per_step": med, "ms_min": lo,
                          "ms_max": hi, "variables": n_vars, "optimizer_kernels_per_step": len(kernels) / PROFILED_STEPS,
                          "kernel_names": sorted(set(kernels)), "card": card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", choices=["deepfm", "transformer"], default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keras_adam.py needs a CUDA device")
    if a.only in (None, "deepfm"):
        deepfm(a)
    if a.only in (None, "transformer"):
        transformer(a)


if __name__ == "__main__":
    main()
