"""RowSparseAdam: tf.train.AdamOptimizer on the embedding tables of a layer-API model, at row-sparse cost.

TensorFlow's Adam is dense.  Its sparse apply still decays m and v of every row and moves every row by its decayed
momentum, every step, so `ops.adam_step_` over the whole arena is the exact form -- and at production table sizes that
sweep is the step.  RowSparseAdam gives the same numbers while it touches only the rows a batch reads (csrc/embed_adam.cu):

  * every row keeps one state block [g D | m D | v D | g_w m_w v_w count stamp | pad] (dr_embed_adam_state_stride), the
    stamp being the last step whose update the row has seen;
  * before every forward, in training and under no_grad alike, the rows the batch reads replay the steps they sat out
    with a zero gradient (dr_embed_adam_catch_up), so the forward reads what dense Adam would have left there;
  * the backward keeps the per-lookup gradients and returns no table gradient: no arena is allocated or zeroed;
  * step(), after the clock has advanced to t, sums the gradients of duplicate lookups of a row and applies step t to
    every touched row (dr_embed_adam_count, then dr_embed_fm_bwd_adam_tf for the FM term of single-valued slots or
    dr_embed_adam_rows_tf for gradient rows given with strides: FNN's input row, a stack gradient, a bag's gradient);
  * flush() replays every row up to the current step, for whatever reads the whole arena (FM.export, state_dict()).

The rates of the replayed steps come from the clock's ring of bias-corrected rates (AdamClock(history=1 << 16)), or are
recomputed for steps that fell out of it; steps more than kCatchUpMax = 2048 behind only decay m and v, in closed form.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

from . import _lib, ops
from ._lib import check

HISTORY = 1 << 16          # the lr ring DeepFMTrainStep(optimizer="adam_rows_tf") keeps


class _Rows(NamedTuple):
    """Lookups whose gradient rows are given with strides (see dr_embed_adam_rows_tf).  slot: None for ids [B, S] over
    every slot, else the bag slot of `ids` (flat members, `splits` [B + 1]).  Offsets and strides count floats."""
    ids: torch.Tensor
    B: int
    S: int
    splits: Optional[torch.Tensor]
    slot: Optional[int]
    g: torch.Tensor
    g_off: int
    g_ld: int
    g_slot: int
    gl: Optional[torch.Tensor]
    gl_off: int
    gl_ld: int
    gl_slot: int


class _FM(NamedTuple):
    """Single-valued lookups with the FM term (dr_embed_fm_bwd_adam_tf forms their gradient rows)."""
    ids: torch.Tensor
    stack: torch.Tensor
    sum_e: torch.Tensor
    g_logit: torch.Tensor
    g_stack: Optional[torch.Tensor]


class RowSparseAdam:
    """tf.train.AdamOptimizer(learning_rate, beta1, beta2, epsilon) on the `weight` (and, in the split layout, the
    `linear`) arena of one EmbeddingCollection, equal to dense Adam at row-sparse cost.  The collection's `bias` and the
    towers stay with a dense optimizer.

    clock: the `ops.AdamClock` of the model's dense optimizer, so that the tower and the tables count one step t, as
    TF1's shared beta1_power does.  It must carry the same lr, betas and eps and a rate ring (history > 0); it is advanced
    by its owner, and step() must follow that advance.  Without a clock the optimizer keeps its own (history = 1 << 16)
    and step() advances it.

    Per step: forward, backward, [the dense optimizer's clock.advance() and update], step().  Attaching to a collection
    with `sparse_lr` (fused SGD) raises ValueError; step() without a backward since the last step raises RuntimeError.
    """

    def __init__(self, collection, learning_rate, beta1=0.9, beta2=0.999, epsilon=1e-8, clock=None):
        if collection.sparse_lr is not None:
            raise ValueError("RowSparseAdam: the collection trains with fused SGD (sparse_lr); build it with "
                             "sparse_lr=None to train its tables with Adam")
        if getattr(collection, "row_optimizer", None) is not None:
            raise ValueError("RowSparseAdam: the collection already has a row-sparse optimizer")
        lib = _lib.load()
        self.collection = collection
        self.lr, self.beta1, self.beta2, self.eps = float(learning_rate), float(beta1), float(beta2), float(epsilon)
        dev = collection.weight.device
        if clock is None:
            clock = ops.AdamClock(self.lr, self.beta1, self.beta2, self.eps, device=dev, history=HISTORY)
            self._advances = True
        else:
            if (clock.lr, clock.beta1, clock.beta2, clock.eps) != (self.lr, self.beta1, self.beta2, self.eps):
                raise ValueError(f"RowSparseAdam: the clock runs lr={clock.lr} beta1={clock.beta1} beta2={clock.beta2} "
                                 f"eps={clock.eps}, the optimizer lr={self.lr} beta1={self.beta1} beta2={self.beta2} "
                                 f"eps={self.eps}")
            if clock.lr_hist is None:
                raise ValueError("RowSparseAdam: the clock keeps no rate history; build it with "
                                 "AdamClock(..., history=1 << 16)")
            self._advances = False
        self.clock = clock
        ss = lib.dr_embed_adam_state_stride(collection.dim)
        if ss < 0:
            raise ValueError(f"RowSparseAdam: embedding dimension {collection.dim} unsupported")
        # zero m, v, gradient accumulators, counts and stamps: a row that was never updated has nothing to replay
        self.state = torch.zeros((collection.total_rows, ss), dtype=torch.float32, device=dev)
        self._pending = []
        collection.row_optimizer = self

    # ---- layout of the collection -----------------------------------------------------------------------------------
    def _tables(self):
        """(table_ptrs, lin_ptrs or None, rows, slot_offsets, flags) of the parameter arena."""
        c = self.collection
        tp, lp, rows = c.pointers(c.weight, c.linear)
        split_lin = c.with_linear and c.layout == "split"
        return tp, (lp if split_lin else None), rows, c._offsets, c.flags

    def _hist(self):
        ck = self.clock
        return ck.step.data_ptr(), ck.lr_hist.data_ptr(), ck.lr_hist.numel()

    # ---- forward side -------------------------------------------------------------------------------------------------
    def catch_up(self, ids: torch.Tensor, bags: Optional[dict] = None) -> None:
        """Replay the pending steps of every row that ids [B, S] (columns of bag slots ignored) and the bags read, up to
        the clock's current step.  The forward ops call it before they read the tables."""
        lib = _lib.load()
        c = self.collection
        tp, lp, rows, offs, flags = self._tables()
        step, hist, hist_len = self._hist()
        ck = self.clock

        def launch(ids_, n, S, s):
            check(lib.dr_embed_adam_catch_up(ids_.data_ptr(), ids_.element_size(), n, S, c.dim, rows.data_ptr() + 8 * s,
                                             offs.data_ptr() + 8 * s, c.row_stride, c.lin_stride, flags,
                                             tp.data_ptr() + 8 * s, None if lp is None else lp.data_ptr() + 8 * s,
                                             self.state.data_ptr(), step, hist, hist_len, ck.lr, ck.beta1, ck.beta2,
                                             ck.eps, ops._stream()), "dr_embed_adam_catch_up")

        ids = ops._ids(ids)
        launch(ops._no_lookup(ids, sorted(bags)) if bags else ids, ids.numel(), ids.shape[1], 0)
        for s, (bid, _) in sorted((bags or {}).items()):
            bid = ops._ids(bid, "bag ids")
            launch(bid, bid.numel(), 1, s)

    # ---- backward side ------------------------------------------------------------------------------------------------
    def record_fm(self, ids, stack, sum_e, g_logit, g_stack) -> None:
        """Single-valued lookups with the FM term: their row gradients g_logit (sum_e - e) + g_stack and first-order
        gradients g_logit are formed by dr_embed_fm_bwd_adam_tf in step()."""
        self._pending.append(_FM(ids, stack.detach(), sum_e, g_logit, g_stack))

    def record_rows(self, ids, g, g_off, g_ld, g_slot, gl=None, gl_off=0, gl_ld=0, gl_slot=0) -> None:
        """ids [B, S]: the gradient row of lookup (b, s) at float g_off + b g_ld + s g_slot of g, its first-order
        gradient in gl likewise.  gl is required exactly when the collection has first-order weights."""
        B, S = ids.shape
        self._pending.append(_Rows(ids, B, S, None, None, g, g_off, g_ld, g_slot, gl, gl_off, gl_ld, gl_slot))

    def record_bag(self, slot, ids, splits, g, g_off, g_ld, gl=None, gl_off=0, gl_ld=0) -> None:
        """The members `ids` of B bags (row_splits `splits`) of one slot, mean combiner: bag b's gradient row at float
        g_off + b g_ld of g, its first-order gradient at gl_off + b gl_ld of gl."""
        B = splits.numel() - 1
        self._pending.append(_Rows(ids, B, 1, splits, int(slot), g, g_off, g_ld, 0, gl, gl_off, gl_ld, 0))

    # ---- the update ---------------------------------------------------------------------------------------------------
    def step(self) -> None:
        """Apply step t (the clock's current step, after its advance) to every row the recorded backwards touched."""
        if not self._pending:
            raise RuntimeError("RowSparseAdam.step(): no backward since the last step (nothing to apply)")
        if self._advances:
            self.clock.advance()
        lib = _lib.load()
        c = self.collection
        tp, lp, rows, offs, flags = self._tables()
        step, hist, hist_len = self._hist()
        ck = self.clock
        st = ops._stream()
        pending, self._pending = self._pending, []
        for rec in pending:            # every lookup of the step is counted before any is applied
            bag = isinstance(rec, _Rows) and rec.slot is not None
            s = rec.slot if bag else 0
            n_b, n_s = (rec.ids.numel(), 1) if bag else tuple(rec.ids.shape)
            check(lib.dr_embed_adam_count(rec.ids.data_ptr(), rec.ids.element_size(), n_b, n_s, c.dim,
                                          rows.data_ptr() + 8 * s, offs.data_ptr() + 8 * s, self.state.data_ptr(), st),
                  "dr_embed_adam_count")
        for rec in pending:
            if isinstance(rec, _FM):
                B, S = rec.ids.shape
                check(lib.dr_embed_fm_bwd_adam_tf(rec.ids.data_ptr(), rec.ids.element_size(), rows.data_ptr(),
                                                  offs.data_ptr(), rec.stack.data_ptr(), rec.sum_e.data_ptr(),
                                                  rec.g_logit.data_ptr(), ops._ptr(rec.g_stack), B, S, c.dim,
                                                  c.row_stride, c.lin_stride, flags, tp.data_ptr(), ops._ptr(lp),
                                                  self.state.data_ptr(), None, step, ck.lr_t.data_ptr(), hist, hist_len,
                                                  ck.lr, ck.beta1, ck.beta2, ck.eps, st), "dr_embed_fm_bwd_adam_tf")
                continue
            s = 0 if rec.slot is None else rec.slot
            check(lib.dr_embed_adam_rows_tf(rec.ids.data_ptr(), rec.ids.element_size(), rec.ids.numel(), rec.B, rec.S,
                                            ops._ptr(rec.splits), rows.data_ptr() + 8 * s, offs.data_ptr() + 8 * s,
                                            rec.g.data_ptr() + 4 * rec.g_off, rec.g_ld, rec.g_slot,
                                            None if rec.gl is None else rec.gl.data_ptr() + 4 * rec.gl_off, rec.gl_ld,
                                            rec.gl_slot, c.dim, c.row_stride, c.lin_stride, flags,
                                            tp.data_ptr() + 8 * s, None if lp is None else lp.data_ptr() + 8 * s,
                                            self.state.data_ptr(), step, ck.lr_t.data_ptr(), hist, hist_len, ck.lr,
                                            ck.beta1, ck.beta2, ck.eps, st), "dr_embed_adam_rows_tf")

    def flush(self) -> None:
        """Replay the pending steps of EVERY row up to the clock's current step: after it the arena holds what dense Adam
        would.  Call it before reading the whole arena (FM.export and the collection's state_dict() do)."""
        lib = _lib.load()
        c = self.collection
        tp, lp, rows, offs, flags = self._tables()
        step, hist, hist_len = self._hist()
        ck = self.clock
        check(lib.dr_embed_adam_flush(rows.data_ptr(), offs.data_ptr(), c.num_slots, c.dim, c.total_rows, c.row_stride,
                                      c.lin_stride, flags, tp.data_ptr(), ops._ptr(lp), self.state.data_ptr(), step, hist,
                                      hist_len, ck.lr, ck.beta1, ck.beta2, ck.eps, ops._stream()), "dr_embed_adam_flush")
