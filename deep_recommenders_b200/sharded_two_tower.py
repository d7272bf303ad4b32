"""Row-sharded two-tower (DSSM / SBCNM) train step: BASELINE config C4 at N > 1 (SURVEY.md section 8e).

One process per GPU; the user and item embedding tables live row-sharded (owner = row mod G) in one symmetric
allocation, rows of exactly D floats, and are read / updated in place over NVLink by the same fused kernels the
sharded DeepFM step uses (S = 1, no first-order term).  Global batch = G x b; every rank trains on its own b pairs:

  fwd  q = gather(user rows)  c = gather(item rows)            dr_embed_fm_fwd_sharded (peer-memory gather)
       all-gather c (and the item ids)                        the one real exchange step of the path: [G, b, D]
       own block first (shard_plan.own_first_order)           -> labels eye(b, G*b) hold for the local queries
       loss_r = sum_i (lse_j s_ij - s_ii), s = q c^T / tau     dr_inbatch_softmax_fwd (never materialises [b, G*b])
  bwd  gq [b, D], gc [G*b, D]                                  dr_inbatch_softmax_bwd
       blocks back to rank order, reduce-scatter(sum) gc       every rank receives the gradient of ITS candidates
       user rows += -lr * gq, item rows += -lr * gc_local      dr_embed_fm_bwd_sharded (vector atomics into the owner)
       symmetric-memory barrier                                all remote updates issued before the next step reads

The global loss (reference Retrieval.call, reduction SUM: sbcnm.py:100-102,151) is the sum of the per-rank losses;
the collectives of this step also order every rank's remote reads before any remote update.
Towers are the embedding tables themselves (plain DSSM); MLP towers stay single-GPU (TwoTower) in this round.

Tests: the exchange plan by the world-2 gloo test (tests/test_two_tower_protocol_cpu.py); the CUDA step at world 1 by
tests/test_gpu_zz_next_rows.py and at world 2 by tests/test_gpu_sharded.py (torchrun worker); its gather / update kernel
calls at world sizes up to 64, emulated on one GPU, by tests/test_gpu_sharded_emulated.py.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from . import _lib, shard_plan
from ._lib import check


class ShardedTwoTowerTrainStep:
    def __init__(self, num_users: int, num_items: int, dim: int, batch_size: int, lr: float = 0.01,
                 temperature: Optional[float] = None, remove_accidental_hits: bool = False, seed: int = 0,
                 device=None, group=None):
        if not dist.is_initialized():
            raise RuntimeError("ShardedTwoTowerTrainStep needs an initialised torch.distributed process group")
        if dim % 4 != 0 or not (4 <= dim <= 128):
            raise ValueError(f"embedding dimension must be a multiple of 4 in [4,128], got {dim}")
        self.lib = _lib.load()
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != "cuda":
            raise _lib.DeepRecError("the sharded two-tower step runs on CUDA only (no CPU fallback)")
        self.dev = dev
        self.U, self.I, self.D, self.b = int(num_users), int(num_items), int(dim), int(batch_size)
        self.lr = float(lr)
        self.inv_tau = 1.0 if temperature is None else 1.0 / float(temperature)
        self.remove_accidental_hits = bool(remove_accidental_hits)
        G, D, b = self.world, self.D, self.b
        # one global row space: users first, then items
        total = self.U + self.I
        self.local_rows = shard_plan.local_rows(total, self.rank, G)
        max_rows = shard_plan.local_rows(total, 0, G)
        import torch.distributed._symmetric_memory as symm_mem
        buf = symm_mem.empty((max_rows * D,), dtype=torch.float32, device=dev)
        self.handle = symm_mem.rendezvous(buf, group if group is not None else dist.group.WORLD)
        buf.zero_()
        self._buf = buf
        self.weight = buf.view(max_rows, D)[:self.local_rows]
        std = 1.0 / D ** 0.5
        gen = torch.Generator(device=dev).manual_seed(seed * 1000 + self.rank)
        torch.nn.init.trunc_normal_(self.weight, 0.0, std, -2 * std, 2 * std, generator=gen)
        self.peer_ptrs = torch.tensor([int(p) for p in self.handle.buffer_ptrs], dtype=torch.int64, device=dev)
        i64 = dict(device=dev, dtype=torch.int64)
        self.off_user, self.rows_user = torch.tensor([0], **i64), torch.tensor([self.U], **i64)
        self.off_item, self.rows_item = torch.tensor([self.U], **i64), torch.tensor([self.I], **i64)
        f = dict(device=dev, dtype=torch.float32)
        self.user_ids = torch.zeros((b, 1), **i64)
        self.item_ids = torch.zeros((b, 1), **i64)
        self.q = torch.empty((b, D), **f)
        self.c_local = torch.empty((b, D), **f)
        self.c_all = torch.empty((G, b, D), **f)          # rank order (what the all-gather produces)
        self.c_rot = torch.empty((G * b, D), **f)         # own block first
        self.ids_all = torch.empty((G, b), **i64)
        self.ids_rot = torch.empty((G * b,), **i64)
        self.lse = torch.empty((b,), **f)
        self.loss = torch.zeros((1,), **f)
        self.gloss = torch.ones((1,), **f)
        self.gq = torch.empty((b, D), **f)
        self.gc_rot = torch.empty((G * b, D), **f)
        self.gc_all = torch.empty((G, b, D), **f)
        self.gc_local = torch.empty((b, D), **f)
        # scores of this rank's b queries against all G b candidates: tensor-core form when the block is big enough to pay
        from . import ops as _ops
        big = b * G * b >= _ops.SOFTMAX_TC_MIN_SCORES and D >= 32 and b * G * b * 4 <= _ops.SOFTMAX_TC_WS_BYTES
        self.scores_ws = torch.empty((b, G * b), **f) if big else None
        order = shard_plan.own_first_order(self.rank, G)
        self._order = torch.tensor(order, **i64)
        self._inv_order = torch.tensor(shard_plan.inverse_order(order), **i64)

    # ---- one step on whatever is in self.user_ids / self.item_ids ----------------------------------------------
    def _gather(self, off, rows, ids, out):
        st = torch.cuda.current_stream().cuda_stream
        check(self.lib.dr_embed_fm_fwd_sharded(self.peer_ptrs.data_ptr(), self.world, off.data_ptr(), rows.data_ptr(),
                                               ids.data_ptr(), 8, None, self.b, 1, self.D, self.D, 0, 0,
                                               out.data_ptr(), None, None, st), "dr_embed_fm_fwd_sharded")

    def _update(self, off, rows, ids, grad):
        st = torch.cuda.current_stream().cuda_stream
        check(self.lib.dr_embed_fm_bwd_sharded(self.peer_ptrs.data_ptr(), self.world, off.data_ptr(), rows.data_ptr(),
                                               ids.data_ptr(), 8, None, None, None, grad.data_ptr(), self.b, 1, self.D,
                                               self.D, 0, 0, None, -self.lr, st), "dr_embed_fm_bwd_sharded")

    def run(self, mark=None) -> torch.Tensor:
        """`mark(label)` (optional, profiling): called after each phase, on the launching stream."""
        lib, G, b, D = self.lib, self.world, self.b, self.D
        st = lambda: torch.cuda.current_stream().cuda_stream
        mark = mark or (lambda label: None)
        mark("start")
        self._gather(self.off_user, self.rows_user, self.user_ids, self.q)
        self._gather(self.off_item, self.rows_item, self.item_ids, self.c_local)
        mark("gather_p2p")
        if G > 1:
            dist.all_gather_into_tensor(self.c_all.view(G * b, D), self.c_local, group=self.group)
            torch.index_select(self.c_all, 0, self._order, out=self.c_rot.view(G, b, D))
        else:
            self.c_rot.copy_(self.c_local)
        ids_ptr = None
        if self.remove_accidental_hits:
            if G > 1:
                dist.all_gather_into_tensor(self.ids_all.view(G * b), self.item_ids.view(b), group=self.group)
                torch.index_select(self.ids_all, 0, self._order, out=self.ids_rot.view(G, b))
            else:
                self.ids_rot.copy_(self.item_ids.view(b))
            ids_ptr = self.ids_rot.data_ptr()
        mark("all_gather_candidates")
        if self.scores_ws is not None:     # tensor-core form: the b x (G b) score block lives in a scratch buffer
            check(lib.dr_inbatch_softmax_fwd_ws(self.q.data_ptr(), self.c_rot.data_ptr(), None, None, ids_ptr, self.inv_tau,
                                                b, G * b, D, self.scores_ws.data_ptr(), b, self.lse.data_ptr(),
                                                self.loss.data_ptr(), st()), "dr_inbatch_softmax_fwd_ws")
            check(lib.dr_inbatch_softmax_bwd_ws(self.q.data_ptr(), self.c_rot.data_ptr(), None, None, ids_ptr, self.inv_tau,
                                                b, G * b, D, self.lse.data_ptr(), self.gloss.data_ptr(),
                                                self.scores_ws.data_ptr(), b, 1, self.gq.data_ptr(),
                                                self.gc_rot.data_ptr(), st()), "dr_inbatch_softmax_bwd_ws")
        else:
            check(lib.dr_inbatch_softmax_fwd(self.q.data_ptr(), self.c_rot.data_ptr(), None, None, ids_ptr, self.inv_tau,
                                             b, G * b, D, self.lse.data_ptr(), self.loss.data_ptr(), st()),
                  "dr_inbatch_softmax_fwd")
            check(lib.dr_inbatch_softmax_bwd(self.q.data_ptr(), self.c_rot.data_ptr(), None, None, ids_ptr, self.inv_tau,
                                             b, G * b, D, self.lse.data_ptr(), self.gloss.data_ptr(), self.gq.data_ptr(),
                                             self.gc_rot.data_ptr(), st()), "dr_inbatch_softmax_bwd")
        mark("softmax_fwd_bwd")
        if G > 1:
            torch.index_select(self.gc_rot.view(G, b, D), 0, self._inv_order, out=self.gc_all)
            dist.reduce_scatter_tensor(self.gc_local, self.gc_all.view(G * b, D), group=self.group)
        else:
            self.gc_local.copy_(self.gc_rot)
        mark("reduce_scatter_grads")
        self._update(self.off_user, self.rows_user, self.user_ids, self.gq)
        self._update(self.off_item, self.rows_item, self.item_ids, self.gc_local)
        mark("update_p2p")
        self.handle.barrier(channel=0)
        mark("barrier")
        return self.loss

    def step(self, user_ids: torch.Tensor, item_ids: torch.Tensor) -> torch.Tensor:
        """Device-resident ids [b]; returns this rank's loss[1] (the global loss is the sum over ranks)."""
        self.user_ids.copy_(user_ids.reshape(-1, 1), non_blocking=True)
        self.item_ids.copy_(item_ids.reshape(-1, 1), non_blocking=True)
        return self.run()

    def rows_of(self, global_rows: torch.Tensor) -> torch.Tensor:
        """This rank's copy of the given GLOBAL rows it owns (tests): row r lives at local index r // world."""
        return self.weight[global_rows // self.world]
