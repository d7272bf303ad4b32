"""Row-sharded embedding tables + data-parallel tower: the N>1 path (SURVEY.md section 8e).

One process per GPU (torch.distributed, NCCL over NVLink/NVSwitch).  Global batch = world * B,
each rank trains on its own B examples:

  fwd  ids [B,S] --dr_shard_bucket_ids--> padded per-owner local row ids
       all-to-all (ids out)            -> every owner gathers its rows  (dr_gather_fwd, fused
                                          rows [emb | w | pad]: the first-order weight rides along)
       all-to-all (vectors back)       -> dr_embed_fm_fwd with table = receive buffer, ids = inv:
                                          un-permute + stack + first-order + FM in ONE kernel
       DNN tower (replicated) -> BCE
  bwd  tower backward -> dr_embed_fm_bwd packs per-lookup gradient rows into the send buffer
       all-to-all (gradients out)      -> owners apply the row-sparse SGD update (dr_scatter_add)
       all-reduce of the flat tower gradient (+ the FM bias gradient), then dr_sgd_step.

optimizer="adam_rows_tf" trains with tf.keras Adam instead (what the reference examples use), equal to Adam applied
densely to the unsharded model on the global batch.  Each owner keeps a gradient arena in its shard's layout, a touch
array, per-row state blocks (m, v, step stamp) and an Adam clock; per step every rank marks the rows its lookups touch
in their owners' touch arrays, each owner lists and replays (skipped steps) its touched rows before the forward reads
them, the backward sends the row gradients (scale 1/world) into the owners' gradient arenas, and after the exchange the
owner applies step t to the listed rows (dr_shard_adam_*).  The tower and the FM bias take dr_adam_step on the averaged
flat gradient.

The exchanges are equal-split (fixed capacity, -1 padded) so there is no host round trip for
split sizes; a STICKY overflow flag set by the bucket kernel is checked by train_step_host() / check_overflow().
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

from . import _lib, ops, shard_plan
from ._lib import check
from .keras.layers.base import Dense
from .training import _DeepFMTower


class ShardedEmbedding:
    """This rank's shard of the global row space, fused rows [emb | w | pad].

    exchange="nccl": rows of D+4 floats in ordinary device memory, moved by all-to-all.
    exchange="p2p" : rows padded to whole 128-B lines in SYMMETRIC memory (every rank maps every
                     other rank's shard), read / updated in place over NVLink by the fused kernels.
    """

    def __init__(self, rows: Sequence[int], dim: int, rank: int, world: int, device, seed: Optional[int] = None,
                 exchange: str = "nccl", group=None):
        self.rows_list = [int(r) for r in rows]
        self.dim, self.rank, self.world = int(dim), rank, world
        self.total_rows = sum(self.rows_list)
        self.local_rows = shard_plan.local_rows(self.total_rows, rank, world)
        # p2p: narrow rows (D <= 28) are [emb | w | pad] = ONE 128-B line, the weight rides in the row
        # (flags = LIN_IN_ROW); wide rows (BASELINE C3-C5, D = 32 ... 128) are exactly D floats and the first-order
        # weights a [max_rows] array trailing the shard in the same symmetric allocation (shard_plan.p2p_layout).
        if exchange == "nccl":
            if dim + 4 > 128:
                raise NotImplementedError("exchange='nccl' moves fused rows of D + 4 <= 128 floats; use exchange='p2p' "
                                          "for wider rows")
            self.lin_in_row, self.vdim, self.lin_offset = True, self.dim + 4, 0
        else:
            layout = shard_plan.p2p_layout(self.total_rows, self.dim, world)
            self.lin_in_row, self.vdim, self.lin_offset = layout.lin_in_row, layout.vdim, layout.lin_offset
        self.flags = 1 if self.lin_in_row else 0
        self.device = device
        self.handle = None
        self.peer_ptrs = None
        std = 1.0 / self.dim ** 0.5
        if exchange == "p2p":
            import torch.distributed._symmetric_memory as symm_mem
            max_rows = layout.max_rows
            buf = symm_mem.empty((layout.numel,), dtype=torch.float32, device=device)
            self.handle = symm_mem.rendezvous(buf, group if group is not None else dist.group.WORLD)
            buf.zero_()
            w = buf[:max_rows * self.vdim].view(max_rows, self.vdim)[:self.local_rows]
            self._buf = buf
            self.lin = None if self.lin_in_row else buf[self.lin_offset:self.lin_offset + max_rows][:self.local_rows]
            self.peer_ptrs = torch.tensor([int(p) for p in self.handle.buffer_ptrs], dtype=torch.int64, device=device)
        else:
            w = torch.zeros((self.local_rows, self.vdim), dtype=torch.float32, device=device)
            self.lin = None
        gen = torch.Generator(device=device).manual_seed((seed or 0) * 1000 + rank)
        torch.nn.init.trunc_normal_(w[:, :self.dim], 0.0, std, -2 * std, 2 * std, generator=gen)
        self.weight = w
        self.slot_offsets = torch.tensor(shard_plan.slot_offsets(self.rows_list), dtype=torch.int64, device=device)
        self.rows = torch.tensor(self.rows_list, dtype=torch.int64, device=device)

    def lin_view(self) -> torch.Tensor:
        """[local_rows] first-order weights of this rank's shard (a column of the fused rows or the trailing array)."""
        return self.weight[:, self.dim] if self.lin_in_row else self.lin


class ShardedDeepFMTrainStep(_DeepFMTower):
    def __init__(self, columns, dim: int, dnn_units: Sequence[int], batch_size: int, lr: float = 0.01,
                 seed: int = 0, device=None, group=None, use_graph: bool = True, exchange: str = "p2p",
                 dw_first: bool = False, optimizer: str = "sgd", beta1: float = 0.9, beta2: float = 0.999,
                 eps: float = 1e-7):
        if not dist.is_initialized():
            raise RuntimeError("ShardedDeepFMTrainStep needs an initialised torch.distributed process group")
        self.lib = _lib.load()
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != "cuda":
            raise _lib.DeepRecError("the sharded hot path runs on CUDA only (no CPU fallback)")
        self.dev = dev
        rows = [c.num_buckets for c in columns]
        self.B, self.S, self.D = int(batch_size), len(rows), int(dim)
        self.lr = float(lr)
        if exchange not in ("p2p", "nccl"):
            raise ValueError(f"exchange must be 'p2p' or 'nccl', got {exchange!r}")
        self.exchange = exchange
        if optimizer not in ("sgd", "adam_rows_tf"):
            raise ValueError(f"optimizer must be 'sgd' or 'adam_rows_tf', got {optimizer!r}")
        self.optimizer = optimizer
        self.dw_first = bool(dw_first)
        self.emb = ShardedEmbedding(rows, dim, self.rank, self.world, dev, seed, exchange, group)
        B, S, D, G = self.B, self.S, self.D, self.world
        self.n = B * S
        self.cap = shard_plan.capacity(self.n, G)
        V = self.emb.vdim
        f = dict(device=dev, dtype=torch.float32)
        # tower: identical initialisation on every rank (same seed), kept in one flat buffer; slot 0 = FM bias
        layers: List[Dense] = [Dense(u, activation="relu", seed=seed + i) for i, u in enumerate(dnn_units)]
        layers.append(Dense(1, seed=seed + len(dnn_units)))
        in_dim = S * D
        for l in layers:
            l.build((B, in_dim), device=dev)
            in_dim = l.units
        [(self.bias, self.g_bias)] = self._init_tower(layers, lead=[torch.zeros((1,), **f)])     # bias at 0, tower at 4
        # static buffers
        # warm-up ids spread over the tables (all-zero ids would all hit one owner)
        self.ids = torch.stack([torch.randint(0, max(1, r), (B,), device=dev) for r in rows], dim=1).contiguous()
        self.labels = torch.zeros((B,), **f)
        if exchange == "nccl":
            self.send_counts = torch.zeros((G,), device=dev, dtype=torch.int64)
            self.send_ids = torch.empty((G * self.cap,), device=dev, dtype=torch.int64)
            self.recv_ids = torch.empty((G * self.cap,), device=dev, dtype=torch.int64)
            self.inv = torch.empty((self.n,), device=dev, dtype=torch.int32)
            self.overflow = torch.zeros((1,), device=dev, dtype=torch.int32)
            self.vec_send = torch.empty((G * self.cap, V), **f)      # rows gathered for the requesters
            self.vec_recv = torch.empty((G * self.cap, V), **f)      # rows this rank asked for
            self.grad_send = torch.empty((G * self.cap, V), **f)
            self.grad_recv = torch.empty((G * self.cap, V), **f)
        if exchange == "nccl":
            # "identity tables": the S slots all read the receive buffer (table base = vec_recv, rows = G*cap)
            base = self.vec_recv.data_ptr()
            self.tp = torch.full((S,), base, device=dev, dtype=torch.int64)
            self.lp = torch.full((S,), base + D * 4, device=dev, dtype=torch.int64)
            gbase = self.grad_send.data_ptr()
            self.gtp = torch.full((S,), gbase, device=dev, dtype=torch.int64)
            self.glp = torch.full((S,), gbase + D * 4, device=dev, dtype=torch.int64)
            self.trows = torch.full((S,), G * self.cap, device=dev, dtype=torch.int64)
        if optimizer == "adam_rows_tf":
            self._init_adam(beta1, beta2, eps)
        self.graph = None
        self.use_graph = use_graph
        self.launches_per_step = None
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._side_stream = torch.cuda.Stream(device=dev)
        self._staged = None

    def _init_adam(self, beta1, beta2, eps):
        """Optimizer state of this rank's shard: gradient arena in the shard's layout + int32 touch array (p2p: one
        symmetric allocation, peers add into the arena and mark the touch array), the list of touched rows and its
        device-resident count, per-row state blocks [m | v | m_w v_w | count | stamp] (dr_embed_adam_state_stride), the
        clock, and m / v of the flat tower (FM bias at 0)."""
        emb, dev, D, G = self.emb, self.dev, self.D, self.world
        n = emb.local_rows
        i32 = dict(device=dev, dtype=torch.int32)
        i64 = dict(device=dev, dtype=torch.int64)
        self.clock = ops.AdamClock(self.lr, beta1, beta2, eps, device=dev, history=1 << 16)
        self.m_flat, self.v_flat = torch.zeros_like(self.flat), torch.zeros_like(self.flat)
        self.state = torch.zeros((max(1, n), self.lib.dr_embed_adam_state_stride(D)), device=dev, dtype=torch.float32)
        self.adam_list = torch.zeros((max(1, n),), **i32)
        self.adam_count = torch.zeros((1,), **i32)
        if self.exchange == "p2p":
            import torch.distributed._symmetric_memory as symm_mem
            layout = shard_plan.p2p_layout(emb.total_rows, D, G)
            tw = (layout.max_rows + 3) // 4 * 4
            buf = symm_mem.empty((layout.numel + tw,), dtype=torch.float32, device=dev)
            self._gbuf_handle = symm_mem.rendezvous(buf, self.group if self.group is not None else dist.group.WORLD)
            buf.zero_()
            self._gbuf = buf
            self.g_arena = buf[:layout.numel]
            self.touch = buf[layout.numel:].view(torch.int32)[:max(1, layout.max_rows)]
            ptrs = [int(p) for p in self._gbuf_handle.buffer_ptrs]
            self.g_peer = torch.tensor(ptrs, **i64)
            self.touch_peer = torch.tensor([p + 4 * layout.numel for p in ptrs], **i64)
            self._mark_offs, self._mark_rows = emb.slot_offsets, emb.rows
        else:
            self.g_arena = torch.zeros((max(1, n), emb.vdim), device=dev, dtype=torch.float32)
            self.touch = torch.zeros((max(1, n),), **i32)
            self.touch_peer = torch.tensor([self.touch.data_ptr()], **i64)
            # the received ids are local rows of this owner: one "table" of local_rows rows, world 1
            self._mark_offs, self._mark_rows = torch.zeros((1,), **i64), torch.tensor([n], **i64)
        base = emb.weight.data_ptr()
        self._shard_tp = torch.tensor([base], **i64)
        self._shard_lp = torch.tensor([base + 4 * emb.lin_offset], **i64)
        self._shard_rows, self._shard_offs = torch.tensor([n], **i64), torch.zeros((1,), **i64)

    def _adam_mark(self, ids, id_bytes, n, S, world):
        ck = self.clock
        check(self.lib.dr_shard_adam_mark(ids, id_bytes, n, S, self._mark_offs.data_ptr(), self._mark_rows.data_ptr(),
                                          world, self.touch_peer.data_ptr(), ck.step.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), "dr_shard_adam_mark")

    def _adam_prepare(self):
        emb, ck = self.emb, self.clock
        check(self.lib.dr_shard_adam_prepare(self.touch.data_ptr(), emb.local_rows, self.adam_list.data_ptr(),
                                             self.adam_count.data_ptr(), self.D, emb.vdim, emb.lin_offset, emb.flags,
                                             emb.weight.data_ptr(), self.state.data_ptr(), ck.step.data_ptr(),
                                             ck.lr_hist.data_ptr(), ck.lr_hist.numel(), ck.lr, ck.beta1, ck.beta2, ck.eps,
                                             torch.cuda.current_stream().cuda_stream), "dr_shard_adam_prepare")

    def _adam_apply(self):
        emb, ck = self.emb, self.clock
        check(self.lib.dr_shard_adam_apply(self.adam_list.data_ptr(), self.adam_count.data_ptr(), emb.local_rows, self.D,
                                           emb.vdim, emb.lin_offset, emb.flags, emb.weight.data_ptr(),
                                           self.g_arena.data_ptr(), self.state.data_ptr(), ck.step.data_ptr(),
                                           ck.lr_t.data_ptr(), ck.beta1, ck.beta2, ck.eps,
                                           torch.cuda.current_stream().cuda_stream), "dr_shard_adam_apply")

    def _dense_update(self, st):
        """The flat tower (FM bias at 0) after the all-reduce: SGD on the summed gradient with lr / world, or Adam on the
        averaged one."""
        if self.optimizer == "sgd":
            check(self.lib.dr_sgd_step(self.flat.data_ptr(), self.gflat.data_ptr(), self.flat.numel(), self.lr / self.world,
                                       st), "dr_sgd_step")
            return
        ck = self.clock
        check(self.lib.dr_adam_step(self.flat.data_ptr(), self.gflat.data_ptr(), self.m_flat.data_ptr(),
                                    self.v_flat.data_ptr(), self.flat.numel(), 0.0, ck.beta1, ck.beta2, ck.eps, 0,
                                    ck.lr_t.data_ptr(), st), "dr_adam_step(tower)")

    def _allreduce_dense(self):
        if self.optimizer == "sgd":
            dist.all_reduce(self.gflat, group=self.group)
        else:           # Adam is not linear in g: the mean gradient of the global batch, not a rescaled rate
            dist.all_reduce(self.gflat, op=dist.ReduceOp.AVG, group=self.group)

    def flush_optimizer(self) -> None:
        """optimizer="adam_rows_tf": replay the pending (skipped) Adam steps of every row of this rank's shard up to the
        current step, so the shard equals what tf.keras Adam's dense update would hold.  Call on every rank before the
        tables are read outside the trainer; a no-op for SGD."""
        if self.optimizer != "adam_rows_tf":
            return
        emb, ck = self.emb, self.clock
        check(self.lib.dr_embed_adam_flush(self._shard_rows.data_ptr(), self._shard_offs.data_ptr(), 1, self.D,
                                           emb.local_rows, emb.vdim, 1, emb.flags, self._shard_tp.data_ptr(),
                                           self._shard_lp.data_ptr(), self.state.data_ptr(), ck.step.data_ptr(),
                                           ck.lr_hist.data_ptr(), ck.lr_hist.numel(), ck.lr, ck.beta1, ck.beta2, ck.eps,
                                           torch.cuda.current_stream().cuda_stream), "dr_embed_adam_flush")

    def _moment_rows(self, k):
        """m (k = 1) or v (k = 2) of this rank's rows, shaped like the weights: ([local, vdim] with the first-order moment
        in the row, or None) and ([local] trailing first-order moments, or None)."""
        D, n = self.D, self.emb.local_rows
        st = self.state[:n]
        rows = torch.zeros_like(self.emb.weight)
        rows[:, :D] = st[:, k * D:(k + 1) * D]
        if self.emb.lin_in_row:
            rows[:, D] = st[:, 3 * D + k]
            return rows, None
        return rows, st[:, 3 * D + k].clone()

    # ---- checkpoint: one file per rank + metadata on rank 0; loadable by any number of ranks (checkpoint.py) -------
    def get_config(self) -> dict:
        cfg = {"class": "ShardedDeepFMTrainStep", "rows": list(self.emb.rows_list), "dim": self.D,
               "dnn_units": [l.units for l in self.layers[:-1]], "batch_size": self.B, "lr": self.lr,
               "exchange": self.exchange, "row_width": self.emb.vdim, "lin_in_row": bool(self.emb.lin_in_row)}
        if self.optimizer != "sgd":         # SGD checkpoints keep the config they always had (a missing key reads as SGD)
            cfg["optimizer"] = self.optimizer
        return cfg

    def save(self, prefix: str) -> None:
        from . import checkpoint
        self.flush_optimizer()              # Adam: every row at the current step, so stamps need not be saved
        torch.cuda.synchronize()
        arrays = {"weight": self.emb.weight}
        if not self.emb.lin_in_row:
            arrays["lin"] = self.emb.lin
        replicated = {"flat": self.flat}
        if self.optimizer != "sgd":
            for k, name in ((1, "m"), (2, "v")):
                rows, lin = self._moment_rows(k)
                arrays[name] = rows
                if lin is not None:
                    arrays[name + "_lin"] = lin
            replicated.update({"m_flat": self.m_flat, "v_flat": self.v_flat, "adam_step": self.clock.step})
        # one id per save, the same on every rank and in the meta file, so that files of two saves cannot be mixed
        import time
        sid = torch.tensor([time.time_ns() // 1000 if self.rank == 0 else 0], dtype=torch.int64, device=self.dev)
        dist.broadcast(sid, src=0 if self.group is None else dist.get_global_rank(self.group, 0), group=self.group)
        save_id = int(sid.item())
        checkpoint.save_rows(prefix, self.rank, self.world, self.emb.total_rows, arrays, save_id=save_id)
        dist.barrier(group=self.group)          # every shard is on disk ...
        if self.rank == 0:                      # ... before the meta file, the commit marker, is written
            checkpoint.save_meta(prefix, self.get_config(), replicated, world=self.world, save_id=save_id)
            checkpoint.remove_stale_shards(prefix, self.world)
        dist.barrier(group=self.group)

    def load(self, prefix: str) -> None:
        """Restore from a checkpoint of the same model written by ANY world size (rows are re-sharded while loading)."""
        from . import checkpoint
        meta = checkpoint.load_meta(prefix)
        cfg, mine = meta["config"], self.get_config()
        for k in ("rows", "dim", "dnn_units", "row_width", "lin_in_row"):
            if cfg[k] != mine[k]:
                raise ValueError(f"checkpoint {prefix!r} was written for {k}={cfg[k]}, this model has {k}={mine[k]}")
        saved_opt = cfg.get("optimizer", "sgd")
        if saved_opt != self.optimizer:
            raise ValueError(f"checkpoint {prefix!r} was written with optimizer={saved_opt!r}, this trainer uses "
                             f"optimizer={self.optimizer!r}")
        got = checkpoint.load_rows(prefix, self.rank, self.world)
        rep = meta["replicated"]
        with torch.no_grad():
            self.emb.weight.copy_(got["weight"].to(self.dev))
            if not self.emb.lin_in_row:
                self.emb.lin.copy_(got["lin"].to(self.dev))
            self.flat.copy_(rep["flat"].to(self.dev))
            if self.optimizer != "sgd":
                self._load_adam(got, rep)
        torch.cuda.synchronize()
        dist.barrier(group=self.group)

    def _load_adam(self, got, rep):
        """Moments of the loaded rows into the state blocks, every stamp = the saved step (the writer flushed), gradient
        arena / touch array / row list / counts cleared, clock and tower moments restored."""
        D, n = self.D, self.emb.local_rows
        t = int(rep["adam_step"].reshape(-1)[0])
        self.state.zero_()
        st = self.state[:n]
        for k, name in ((1, "m"), (2, "v")):
            rows = got[name].to(self.dev)
            st[:, k * D:(k + 1) * D] = rows[:, :D]
            st[:, 3 * D + k] = rows[:, D] if self.emb.lin_in_row else got[name + "_lin"].to(self.dev)
        self.state.view(torch.int32)[:n, 3 * D + 4] = t           # the stamp is an int32 in a float slot
        (self._gbuf if self.exchange == "p2p" else self.g_arena).zero_()
        self.touch.zero_()
        self.adam_list.zero_()
        self.adam_count.zero_()
        self.clock.step.fill_(t)
        self.m_flat.copy_(rep["m_flat"].to(self.dev))
        self.v_flat.copy_(rep["v_flat"].to(self.dev))

    def _a2a(self, out, inp):
        dist.all_to_all_single(out, inp, group=self.group)

    # The step is a chain  compute segment -> collective -> compute segment ...  The compute segments
    # are captured as CUDA graphs; the NCCL collectives are issued between the replays.
    def _segments_p2p(self, mark):
        """exchange="p2p": the fused gather+FM kernel reads every owner's shard directly over NVLink
        and the backward's vector atomics land directly in the owner's shard -- no id exchange, no
        owner-side gather/scatter kernels, no all-to-all.  The tower all-reduce separates the step's
        remote reads from its remote updates; a symmetric-memory barrier ends the step."""
        lib = self.lib
        B, S, D, G, V = self.B, self.S, self.D, self.world, self.emb.vdim

        def st():
            return torch.cuda.current_stream().cuda_stream

        def seg_gather():
            check(lib.dr_embed_fm_fwd_sharded(self.emb.peer_ptrs.data_ptr(), G, self.emb.slot_offsets.data_ptr(),
                                              self.emb.rows.data_ptr(), self.ids.data_ptr(), 8, self.bias.data_ptr(),
                                              B, S, D, V, self.emb.flags, self.emb.lin_offset, self.stack.data_ptr(),
                                              self.sum_e.data_ptr(), self.fm_logit.data_ptr(), st()),
                  "dr_embed_fm_fwd_sharded")
            mark("embed_fm_fwd_p2p")

        def col_reads_done():
            # every rank has finished reading every shard: from here on remote updates may land (this barrier, not the
            # tower all-reduce, is what orders a step's remote reads before its remote updates -- so the update can
            # overlap the layer-0 weight gradient and the all-reduce instead of waiting for them)
            self.emb.handle.barrier(channel=1)
            mark("barrier_reads")

        def seg_tower():
            check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")
            self._tower_fwd_bwd(mark)

        adam = self.optimizer != "sgd"
        # SGD: the update itself lands in the owners' shards; Adam: the mean row gradient lands in their gradient arenas
        dst, scale = (self.g_peer, 1.0 / G) if adam else (self.emb.peer_ptrs, -self.lr / G)

        def seg_update():           # replayed on the SIDE stream: remote vector atomics into the owners' shards
            gz = self.g_acts[-1]
            check(lib.dr_embed_fm_bwd_sharded(dst.data_ptr(), G, self.emb.slot_offsets.data_ptr(),
                                              self.emb.rows.data_ptr(), self.ids.data_ptr(), 8, self.stack.data_ptr(),
                                              self.sum_e.data_ptr(), gz.data_ptr(), self.g_stack.data_ptr(), B, S, D,
                                              V, self.emb.flags, self.emb.lin_offset, None, scale, st()),
                  "dr_embed_fm_bwd_sharded")

        def seg_dw():               # ... meanwhile, on the main stream: layer-0 weight gradient + FM bias gradient
            self._tower_dw()
            check(lib.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
            mark("dense_bwd_0_dw")
            torch.sum(self.g_acts[-1].view(-1), dim=0, keepdim=True, out=self.g_bias)      # FM bias gradient (tiny)
            mark("bias_grad")

        def col_allreduce():
            self._allreduce_dense()
            mark("allreduce_dense")

        def seg_sgd():
            self._dense_update(st())
            mark("adam_dense" if adam else "sgd")

        def col_barrier():
            mark("embed_fm_bwd_p2p_tail")               # what was left of the side-stream update after the join
            self.emb.handle.barrier(channel=0)          # all remote atomics of this step have been issued
            mark("barrier")

        if self.dw_first:
            # the persistent weight-gradient GEMM is submitted BEFORE the remote update (both depend only on the layer-0
            # input gradient): it takes its one CTA per SM and the update's CTAs fill what is left (knob tc_dw_share)
            plan = [(seg_gather, "graph"), (col_reads_done, "eager"), (seg_tower, "graph"), (None, "fork"),
                    (seg_dw, "graph"), (seg_update, "graph_side_fork"), (col_allreduce, "eager"), (seg_sgd, "graph"),
                    (None, "join_side"), (col_barrier, "eager")]
        else:
            plan = [(seg_gather, "graph"), (col_reads_done, "eager"), (seg_tower, "graph"), (seg_update, "graph_side"),
                    (seg_dw, "graph"), (col_allreduce, "eager"), (seg_sgd, "graph"), (None, "join_side"),
                    (col_barrier, "eager")]
        if not adam:
            return plan

        def seg_mark():             # t += 1; this rank's lookups mark their rows in the owners' touch arrays
            self.clock.advance()
            self._adam_mark(self.ids.data_ptr(), 8, self.n, S, G)
            mark("adam_mark")

        def col_marked():           # every mark of this step is in place before any owner lists its rows
            self.emb.handle.barrier(channel=1)
            mark("barrier_marks")

        def seg_prepare():          # owners: list the touched rows, replay the steps they sat out
            self._adam_prepare()
            mark("adam_prepare")

        def col_replayed():         # no rank's forward reads a row before its owner has replayed it
            self.emb.handle.barrier(channel=1)
            mark("barrier_replay")

        def seg_apply():            # after the closing barrier every row gradient has landed: owners take step t
            self._adam_apply()
            mark("adam_apply")

        return ([(seg_mark, "graph"), (col_marked, "eager"), (seg_prepare, "graph"), (col_replayed, "eager")] + plan
                + [(seg_apply, "graph")])

    def _segments(self, mark):
        if self.exchange == "p2p":
            return self._segments_p2p(mark)
        lib = self.lib
        B, S, D, G, V = self.B, self.S, self.D, self.world, self.emb.vdim

        def st():
            return torch.cuda.current_stream().cuda_stream

        adam = self.optimizer != "sgd"

        def seg_bucket():
            if adam:
                self.clock.advance()
            check(lib.dr_shard_bucket_ids(self.ids.data_ptr(), 8, self.n, S, self.emb.slot_offsets.data_ptr(),
                                          self.emb.rows.data_ptr(), G, self.cap, self.send_counts.data_ptr(),
                                          self.send_ids.data_ptr(), self.inv.data_ptr(), self.overflow.data_ptr(), st()),
                  "dr_shard_bucket_ids")
            mark("bucket")

        def col_ids():
            self._a2a(self.recv_ids, self.send_ids)
            mark("a2a_ids")

        def seg_gather():
            if adam:                # owners: mark the received rows, list them and replay their skipped steps
                self._adam_mark(self.recv_ids.data_ptr(), 8, G * self.cap, 1, 1)
                mark("adam_mark")
                self._adam_prepare()
                mark("adam_prepare")
            check(lib.dr_gather_fwd(self.emb.weight.data_ptr(), self.emb.local_rows, self.recv_ids.data_ptr(), 8,
                                    G * self.cap, V, self.vec_send.data_ptr(), st()), "dr_gather_fwd")
            mark("owner_gather")

        def col_vec():
            self._a2a(self.vec_recv, self.vec_send)
            mark("a2a_vectors")

        def seg_main():
            check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")
            check(lib.dr_embed_fm_fwd(self.tp.data_ptr(), self.lp.data_ptr(), self.trows.data_ptr(),
                                      self.inv.data_ptr(), 4, self.bias.data_ptr(), B, S, D, V, V, 1,
                                      self.stack.data_ptr(), self.sum_e.data_ptr(), self.fm_logit.data_ptr(), st()),
                  "dr_embed_fm_fwd")
            mark("embed_fm_fwd")
            x, K = self.stack, S * D
            for i, l in enumerate(self.layers):
                check(lib.dr_dense_fwd(x.data_ptr(), self.w[i].data_ptr(), self.b[i].data_ptr(), B, K, l.units,
                                       l._act, self.acts[i].data_ptr(), st()), "dr_dense_fwd")
                x, K = self.acts[i], l.units
                mark(f"dense_fwd_{i}")
            gz = self.g_acts[-1]
            check(lib.dr_bce_logits_fwd_bwd(self.acts[-1].data_ptr(), self.fm_logit.data_ptr(),
                                            self.labels.data_ptr(), B, self.prob.data_ptr(), self.loss.data_ptr(),
                                            gz.data_ptr(), st()), "dr_bce")
            mark("bce")
            for i in range(len(self.layers) - 1, -1, -1):
                l = self.layers[i]
                xin = self.stack if i == 0 else self.acts[i - 1]
                Kin = S * D if i == 0 else self.layers[i - 1].units
                gx = self.g_stack if i == 0 else self.g_acts[i - 1]
                check(lib.dr_dense_bwd(xin.data_ptr(), self.w[i].data_ptr(), self.acts[i].data_ptr(),
                                       self.g_acts[i].data_ptr(), B, Kin, l.units, l._act, ops._ptr(self.gz_ws[i]),
                                       gx.data_ptr(), self.gw[i].data_ptr(), self.gb[i].data_ptr(), st()),
                      "dr_dense_bwd")
                mark(f"dense_bwd_{i}")
            check(lib.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
            # pack per-lookup gradient rows [dE | g_logit | 0 0 0] into the padded send buffer
            self.grad_send.zero_()
            self.g_bias.zero_()
            check(lib.dr_embed_fm_bwd(self.inv.data_ptr(), 4, self.trows.data_ptr(), self.stack.data_ptr(),
                                      self.sum_e.data_ptr(), gz.data_ptr(), self.g_stack.data_ptr(), B, S, D, V, V, 1,
                                      self.gtp.data_ptr(), self.glp.data_ptr(), self.g_bias.data_ptr(), 1.0, st()),
                  "dr_embed_fm_bwd")
            mark("embed_fm_bwd_pack")

        def col_grads():
            self._a2a(self.grad_recv, self.grad_send)
            mark("a2a_grads")

        def seg_scatter():
            if adam:
                # owners: mean row gradient of the GLOBAL batch (1/world) into the gradient arena, then Adam step t
                check(lib.dr_scatter_add(self.g_arena.data_ptr(), self.emb.local_rows, self.recv_ids.data_ptr(), 8,
                                         G * self.cap, V, self.grad_recv.data_ptr(), 1.0 / G, st()), "dr_scatter_add")
                mark("owner_scatter_grad")
                self._adam_apply()
                mark("adam_apply")
                return
            # owners: row-sparse SGD on the fused rows (mean over the GLOBAL batch: 1/world)
            check(lib.dr_scatter_add(self.emb.weight.data_ptr(), self.emb.local_rows, self.recv_ids.data_ptr(), 8,
                                     G * self.cap, V, self.grad_recv.data_ptr(), -self.lr / G, st()), "dr_scatter_add")
            mark("owner_scatter_sgd")

        def col_allreduce():
            self._allreduce_dense()
            mark("allreduce_dense")

        def seg_sgd():
            self._dense_update(st())
            mark("adam_dense" if adam else "sgd")

        return [(seg_bucket, "graph"), (col_ids, "eager"), (seg_gather, "graph"), (col_vec, "eager"), (seg_main, "graph"),
                (col_grads, "eager"), (seg_scatter, "graph"), (col_allreduce, "eager"), (seg_sgd, "graph")]

    # segment kinds: "graph" = compute on the main stream (captured as a CUDA graph), "eager" = a collective issued
    # between replays, "graph_side" = compute replayed on the side stream after it has waited for the main stream
    # (runs concurrently with what follows), "join_side" = the main stream waits for the side stream.
    def _run_plan(self, plan):
        main = torch.cuda.current_stream()
        for fn, kind in plan:
            if kind == "graph_side":
                self._side_stream.wait_stream(main)
                with torch.cuda.stream(self._side_stream):
                    fn()
            elif kind == "fork":
                fork = torch.cuda.Event()
                fork.record(main)
            elif kind == "graph_side_fork":
                self._side_stream.wait_event(fork)
                with torch.cuda.stream(self._side_stream):
                    fn()
            elif kind == "join_side":
                main.wait_stream(self._side_stream)
            else:
                fn()

    def _enqueue(self, mark=None):
        mark = mark or (lambda label: None)
        mark("start")
        self._run_plan(self._segments(mark))

    def _persistent_state(self):
        """Every tensor a step mutates and a later step reads (this rank's shard incl. trailing first-order weights,
        the flat tower; Adam: gradient arena + touch array, row list and count, state blocks, tower moments, clock)."""
        st = [self.emb._buf if self.exchange == "p2p" else self.emb.weight, self.flat]
        if self.optimizer != "sgd":
            st += [self._gbuf if self.exchange == "p2p" else self.g_arena, self.touch, self.adam_list, self.adam_count,
                   self.state, self.m_flat, self.v_flat, self.clock.step, self.clock.lr_t, self.clock.lr_hist]
        return st

    def _barrier(self):
        """`capture` restores the shards after a warm-up step that sent remote atomics into every peer's shard: all ranks
        meet before the restore (every update has landed) and after it (nobody starts a real step before every shard is
        restored)."""
        dist.barrier(group=self.group)

    def _record_graph(self):
        """Record the compute segments into CUDA graphs; the collectives stay eager NCCL calls (capturing the NCCL
        all-to-all itself dead-locked on this torch/NCCL build).  Returns the plan `_replay` runs."""
        plan = []
        for fn, kind in self._segments(lambda label: None):
            if kind in ("graph", "graph_side", "graph_side_fork"):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fn()
                plan.append((g.replay, kind))
            else:
                plan.append((fn, kind))
        return plan

    def _replay(self):
        self._run_plan(self.graph)

    def check_overflow(self):
        """exchange='nccl' only: raise if ANY bucket call since the last check ran out of send slots (the flag is
        sticky on the device; it is cleared here after it has been read).  Called by capture(), train_step_host() (which
        synchronises on the loss anyway) and once at the end of fit_host(); callers of the asynchronous step() / run()
        call it whenever they synchronise."""
        if self.exchange == "p2p":
            return
        if int(self.overflow.item()) != 0:
            self.overflow.zero_()
            raise _lib.DeepRecError(f"shard exchange overflow: a destination needed more than cap={self.cap} slots "
                                    "(low-cardinality or skewed slot): lookups were dropped in a step since the last "
                                    "check; rebuild the trainer with a larger shard_plan.capacity slack")

    def _launch_embed_fwd(self, ids, st):
        """time_embed_fwd's kernel: this rank's fused gather+FM forward (p2p: (G-1)/G of the rows are read from peers
        over NVLink inside the same kernel).  nccl exchange: the local identity-table kernel only (`ids` unused)."""
        B, S, D, G, V = self.B, self.S, self.D, self.world, self.emb.vdim
        if self.exchange == "p2p":
            check(self.lib.dr_embed_fm_fwd_sharded(self.emb.peer_ptrs.data_ptr(), G, self.emb.slot_offsets.data_ptr(),
                                                   self.emb.rows.data_ptr(), ids.data_ptr(), 8, self.bias.data_ptr(),
                                                   B, S, D, V, self.emb.flags, self.emb.lin_offset,
                                                   self.stack.data_ptr(), self.sum_e.data_ptr(),
                                                   self.fm_logit.data_ptr(), st), "dr_embed_fm_fwd_sharded")
        else:
            check(self.lib.dr_embed_fm_fwd(self.tp.data_ptr(), self.lp.data_ptr(), self.trows.data_ptr(),
                                           self.inv.data_ptr(), 4, self.bias.data_ptr(), B, S, D, V, V, 1,
                                           self.stack.data_ptr(), self.sum_e.data_ptr(), self.fm_logit.data_ptr(), st),
                  "dr_embed_fm_fwd")
