"""BASELINE config C4 (two-tower DSSM / SBCNM: 1 M users, 10 M items, D = 64, in-batch negatives, GLOBAL batch 16384)
on 1..8 GPUs with the row-sharded step (deep_recommenders_b200/sharded_two_tower.py).  One process per GPU:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/bench_two_tower.py

(N = 1: `python tools/bench_two_tower.py`.)  Timing: CUDA events around K steps after W warm-ups, barrier + synchronize
on both sides, MAX over ranks; rank 0 prints one JSON line.  Strong scaling in the batch (b = 16384 / N per GPU).
"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200.sharded_two_tower import ShardedTwoTowerTrainStep  # noqa: E402


def main():
    steps, warm = int(os.environ.get("STEPS", 30)), int(os.environ.get("WARMUP", 5))
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    U, I, D, Bg = 1_000_000, 10_000_000, 64, 16384
    b = Bg // world
    st = ShardedTwoTowerTrainStep(U, I, D, b, lr=0.01, seed=1, device=dev)
    gen = torch.Generator(device=dev).manual_seed(7 + rank)
    pool = [(torch.randint(0, U, (b,), device=dev, generator=gen), torch.randint(0, I, (b,), device=dev, generator=gen))
            for _ in range(8)]

    def barrier():
        dist.barrier()
        torch.cuda.synchronize()

    for i in range(warm):
        st.step(*pool[i % 8])
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        st.step(*pool[i % 8])
    e1.record()
    barrier()
    # per-phase times (eager passes with events between the phases; every rank runs them: the step has collectives)
    runs = []
    for i in range(8):
        st.user_ids.copy_(pool[i % 8][0].reshape(-1, 1)); st.item_ids.copy_(pool[i % 8][1].reshape(-1, 1))
        evs = []

        def mark(label, evs=evs):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            evs.append((label, e))

        st.run(mark)
        runs.append(evs)
    barrier()
    phases = {}
    for evs in runs[2:]:
        for (l0, a), (l1, b_) in zip(evs[:-1], evs[1:]):
            phases[l1] = phases.get(l1, 0.0) + a.elapsed_time(b_) / (len(runs) - 2)
    t = torch.tensor([e0.elapsed_time(e1)], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    loss = st.loss.clone()
    dist.all_reduce(loss)
    if rank == 0:
        ms = float(t) / steps
        print(json.dumps({"metric": "examples/sec (fwd+bwd) two-tower in-batch softmax, global batch 16384", "value": Bg / ms * 1e3,
                          "unit": "examples/s", "n_gpus": world, "steps": steps, "warmup": warm, "ms_per_step": ms,
                          "scaling": "strong", "dtype": "f32", "data": "synthetic",
                          "config": {"workload": f"C4 two-tower: {U} users, {I} items, D={D}, global batch {Bg} ({b} per GPU), "
                                                 "embedding towers, SGD, row-sharded tables",
                                     "softmax_core": "wgmma 3xTF32 (score block in scratch)" if st.scores_ws is not None
                                     else "fused FFMA (scores never materialised)"},
                          "kernel_ms": phases, "global_loss": float(loss)}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
