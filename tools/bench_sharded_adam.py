"""tf.keras-equal Adam on the row-sharded DeepFM step at the C2 shape (26 slots x 1 M rows, D = 16, batch 65536 per GPU,
DNN [256, 32]), against sharded SGD and the single-GPU adam_rows_tf step.

    python tools/bench_sharded_adam.py [--steps K] [--warmup W]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/bench_sharded_adam.py

One process per GPU; the per-GPU batch stays 65536 (weak scaling).  Per configuration: ms/step from CUDA events around
K CUDA-graph steps after W warm-ups (barrier + synchronize on both sides, MAX over ranks), the per-group profile of
profile_kernels (eager passes, CUDA events between kernel groups: adam_mark / adam_prepare / adam_apply for the sharded
Adam step), and the bytes the sharded Adam kernels must move (computed from the shapes and the touched rows of the id
pool) over their measured time.  The single-GPU step runs on rank 0 only.  Rank 0 prints one JSON line, with the card's
name and power limit beside the numbers.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

S, ROWS, D, B, DNN = 26, 1_000_000, 16, 65536, [256, 32]
NP = 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {type(e).__name__})"


def time_steps(tr, pool, steps, warm, world):
    for i in range(warm):
        tr.step(*pool[i % NP])

    def sync():
        torch.cuda.synchronize()
        if world > 1 or dist.is_initialized():
            dist.barrier()
        torch.cuda.synchronize()

    sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.step(*pool[i % NP])
    e1.record()
    sync()
    t = torch.tensor([e0.elapsed_time(e1) / steps], device=tr.dev)
    if dist.is_initialized():
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def adam_bytes(local_rows, touched, n_lookups, vdim):
    """Bytes the three sharded Adam kernels must move per step on one rank, in whole 32-B sectors where they touch a
    row: mark reads the ids and stores one int32 per lookup; prepare reads the touch array, writes the row list and
    reads + writes the parameter row and the state block's m, v, m_w, v_w, stamp of every touched row (the replay);
    apply reads + writes the parameter row, the gradient row and the same state of every listed row."""
    sec = lambda b: -(-b // 32) * 32
    row = sec(4 * vdim) if vdim <= 32 else 4 * vdim
    state = 2 * sec(4 * D) + 32                   # m, v, and the sector holding m_w v_w count stamp
    mark = n_lookups * (8 + 4)
    prepare = 4 * local_rows + touched * (4 + 2 * (row + state))
    apply = touched * (4 + 2 * (2 * row + state))
    return {"adam_mark": mark, "adam_prepare": prepare, "adam_apply": apply}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-iters", type=int, default=10)
    args = ap.parse_args()
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29541")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200 import shard_plan
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    from deep_recommenders_b200.training import DeepFMTrainStep

    cols = [fc.categorical_column_with_identity(f"C{i}", ROWS) for i in range(S)]
    gen = torch.Generator(device=dev).manual_seed(7 + rank)
    pool = [(torch.randint(0, ROWS, (B, S), device=dev, generator=gen),
             torch.randint(0, 2, (B,), device=dev, generator=gen).float()) for _ in range(NP)]
    ids_pool, lab_pool = [p[0] for p in pool], [p[1] for p in pool]
    total = S * ROWS
    local_rows = shard_plan.local_rows(total, rank, world)
    # rows this rank owns that one step touches (the global batch's distinct rows / world), mean over the pool
    offs = torch.arange(S, device=dev, dtype=torch.int64) * ROWS
    parts = []
    for ids in ids_pool:
        g = (ids + offs).reshape(-1)
        if world > 1:
            allg = [torch.empty_like(g) for _ in range(world)]
            dist.all_gather(allg, g)
            g = torch.cat(allg)
        u = torch.unique(g)
        parts.append(int(((u % world) == rank).sum()))
    touched = sum(parts) / len(parts)

    results = {}
    runs = [("sharded_sgd_p2p", "p2p", "sgd"), ("sharded_adam_p2p", "p2p", "adam_rows_tf"),
            ("sharded_adam_nccl", "nccl", "adam_rows_tf")]
    for name, exchange, opt in runs:
        tr = ShardedDeepFMTrainStep(cols, D, DNN, batch_size=B, lr=0.01, seed=1, device=dev, exchange=exchange,
                                    optimizer=opt).capture()
        ms = time_steps(tr, pool, args.steps, args.warmup, world)
        _, prof = tr.profile_kernels(ids_pool, lab_pool, iters=args.profile_iters)
        r = {"ms_per_step": ms, "examples_per_s": world * B / ms * 1e3, "launches_per_step": tr.launches_per_step,
             "kernel_ms": prof}
        if opt != "sgd":
            nb = adam_bytes(local_rows, touched, B * S if exchange == "p2p" else world * tr.cap, tr.emb.vdim)
            r["adam_bytes"] = nb
            r["adam_GBps"] = {k: (nb[k] / (prof[k] * 1e-3) / 1e9 if prof.get(k) else None) for k in nb}
        results[name] = r
        del tr
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        dist.barrier()
    if rank == 0:
        model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                       dnn_units_size=DNN, seed=1, device=dev, sparse_lr=0.01)
        tr = DeepFMTrainStep(model, batch_size=B, lr=0.01, optimizer="adam_rows_tf").capture()
        ms = time_steps(tr, pool, args.steps, args.warmup, 1)
        _, prof = tr.profile_kernels(ids_pool, lab_pool, iters=args.profile_iters)
        results["single_gpu_adam_rows_tf"] = {"ms_per_step": ms, "examples_per_s": B / ms * 1e3,
                                              "launches_per_step": tr.launches_per_step, "kernel_ms": prof}
        del tr, model
        torch.cuda.empty_cache()
        print(json.dumps({"tool": "bench_sharded_adam", "card": card(), "n_gpus": world, "steps": args.steps,
                          "warmup": args.warmup,
                          "config": f"C2 shape: {S} slots x {ROWS} rows, D={D}, batch {B} per GPU, DNN {DNN}, "
                                    "synthetic uniform ids, CUDA graphs",
                          "touched_rows_per_rank_per_step": touched, "local_rows": local_rows,
                          "results": results}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
