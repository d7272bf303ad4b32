"""Launched by tests/test_gpu_sharded_adam.py under torchrun (one rank per GPU): optimizer="adam_rows_tf" of the
row-sharded DeepFM step on the global batch equals the unsharded DeepFMTrainStep(optimizer="adam_rows_tf")."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    for exchange, D in (("p2p", 16), ("nccl", 16), ("p2p", 32)):
        run(exchange, rank, world, dev, D)
    dist.barrier()
    if rank == 0:
        print("SHARDED_ADAM_OK")
    dist.destroy_process_group()


def run(exchange, rank, world, dev, D):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, B, lr = [3000, 7, 500, 1000, 21, 64], 1024, 0.01
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    sh = ShardedDeepFMTrainStep(cols, D, [32, 8], batch_size=B, lr=lr, seed=3, device=dev, exchange=exchange,
                                optimizer="adam_rows_tf")
    total = sum(rows)
    g = torch.Generator(device=dev).manual_seed(11)
    arena_e = torch.zeros((total, D), device=dev).normal_(0, 0.25, generator=g)
    arena_l = torch.zeros((total,), device=dev).normal_(0, 0.1, generator=g)
    with torch.no_grad():
        sh.emb.weight[:, :D].copy_(arena_e[rank::world])
        sh.emb.lin_view().copy_(arena_l[rank::world])
    torch.cuda.synchronize()
    dist.barrier()
    sh.capture()
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=[32, 8], seed=3, device=dev, sparse_lr=lr)
    ref = DeepFMTrainStep(model, batch_size=B * world, lr=lr, use_graph=False, optimizer="adam_rows_tf")
    with torch.no_grad():
        model.embeddings.emb_view().copy_(arena_e)
        model.embeddings.lin_view().copy_(arena_l)
        for i in range(len(ref.layers)):
            ref.w[i].copy_(sh.w[i])
            ref.b[i].copy_(sh.b[i])
    g2 = torch.Generator(device=dev).manual_seed(5)
    for it in range(4):
        ids_g = torch.stack([torch.randint(-1, r + 1, (B * world,), device=dev, generator=g2) for r in rows], dim=1)
        if it in (1, 2):
            ids_g[:, it::2] = -1          # rows sit out steps: the replay runs on the owners
        lab_g = torch.randint(0, 2, (B * world,), device=dev, generator=g2).float()
        l = sh.step(ids_g[rank * B:(rank + 1) * B], lab_g[rank * B:(rank + 1) * B]).clone()
        sh.check_overflow()
        dist.all_reduce(l)
        l_sh = float(l) / world
        l_ref = float(ref.step(ids_g, lab_g).item())
        assert abs(l_sh - l_ref) <= 2e-5 * abs(l_ref) + 1e-6, (exchange, D, l_sh, l_ref)
    sh.flush_optimizer()
    ref.flush_optimizer()
    torch.cuda.synchronize()

    def close(a, b, what):
        err = (a - b).abs()
        assert bool((err <= 1e-4 * b.abs() + 1e-6 * max(1.0, float(b.abs().max()))).all()), \
            (exchange, D, what, float(err.max()))

    close(sh.emb.weight[:, :D], model.embeddings.emb_view()[rank::world], "table")
    close(sh.emb.lin_view(), model.embeddings.lin_view()[rank::world], "first-order weights")
    n, st, rst = sh.emb.local_rows, sh.state, ref.state[rank::world]
    close(st[:n, D:3 * D], rst[:, D:3 * D], "m, v")
    close(st[:n, 3 * D + 1:3 * D + 3], rst[:, 3 * D + 1:3 * D + 3], "m_w, v_w")
    for i in range(len(ref.layers)):
        close(sh.w[i], ref.w[i], f"w{i}")
    close(sh.bias, model.embeddings.bias, "bias")
    torch.cuda.synchronize()
    dist.barrier()
    if rank == 0:
        print(f"world {world} sharded Adam ok: exchange={exchange} D={D}", flush=True)


if __name__ == "__main__":
    main()
