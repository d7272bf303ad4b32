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

KerasAdam is tf.keras.optimizers.Adam for a whole Keras model (compile(optimizer=KerasAdam())): a RowSparseAdam per
EmbeddingCollection and every other variable in one multi-tensor dense update (ops.adam_step_multi_), on one clock.
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

    @property
    def has_pending(self) -> bool:
        """Whether a backward recorded lookups since the last step(), i.e. whether step() has anything to apply."""
        return bool(self._pending)

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


class KerasAdam:
    """tf.keras.optimizers.Adam(learning_rate, beta_1, beta_2, epsilon) for a whole Keras model, with TensorFlow's
    arithmetic (ApplyAdam: eps is added to sqrt(v), the bias correction is folded into lr_t), where the engine's `Adam`
    builds torch.optim.Adam.  Use it as `model.compile(optimizer=KerasAdam(...))`; fit() calls build_for_model(model)
    after the first forward.

    The build walks the model.  tables="rows" (the default) puts every EmbeddingCollection's `weight` (and split
    `linear`) arena on a RowSparseAdam, all of them and the dense variables on one AdamClock: the same numbers as dense
    Adam over the tables, at the cost of the rows a batch reads (4 D + 32 floats of state per row, rounded up to 32).
    Every other trainable parameter -- the collections' `bias`, towers, Cross / CIN / attention weights, `Gather` tables
    -- is in the dense group, whose m and v are two flat arenas stepped by one ops.adam_step_multi_.  tables="dense" keeps
    the arenas in the dense group: the same update swept over every row.

    step(): advance the clock with the current learning rate, update the dense variables that have a gradient (as
    Keras's apply_gradients, a variable without one is left alone), then apply the step to the rows of every collection
    that a backward read.  A collection that no forward read this step is not stepped; its rows replay the step when
    they are next read.  param_groups[0]["lr"] (the engine's model.optimizer.lr) takes effect at the next step(), and the
    clock's ring of rates keeps each step's own lr_t for those replays.

    Rejected: amsgrad=True (NotImplementedError); a collection built with sparse_lr, whose backward applies fused SGD,
    and a collection already carrying a RowSparseAdam that the user attached (ValueError).  A RowSparseAdam of an
    earlier KerasAdam build on the same model is flushed and released, so a recompiled model starts from fresh slots at
    step 1, as a new Keras optimizer does.  Slots are not saved by state_dict().
    """

    def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7, amsgrad=False, tables="rows"):
        if amsgrad:
            raise NotImplementedError("KerasAdam: amsgrad=True is not implemented")
        if tables not in ("rows", "dense"):
            raise ValueError(f"KerasAdam: tables={tables!r}; expected 'rows' or 'dense'")
        self.beta_1, self.beta_2, self.epsilon = float(beta_1), float(beta_2), float(epsilon)
        self.tables = tables
        # the engine reads and writes the rate as spec.kw["lr"] before the build and param_groups[0]["lr"] after it
        self.kw = {"lr": float(learning_rate)}
        self.param_groups = [self.kw]
        self.clock = None
        self.dense = []            # (parameter, m, v) of the dense group
        self.row_optimizers = []   # one RowSparseAdam per collection (tables="rows")

    def build_for_model(self, model) -> "KerasAdam":
        from .embedding import EmbeddingCollection
        colls = [mod for mod in model.modules() if isinstance(mod, EmbeddingCollection)]
        for c in colls:
            if c.sparse_lr is not None:
                raise ValueError("KerasAdam: an EmbeddingCollection of the model trains with fused SGD (sparse_lr); "
                                 "build the model with sparse_lr=None")
            if c.row_optimizer is not None and not getattr(c.row_optimizer, "_keras_adam", False):
                raise ValueError("KerasAdam: an EmbeddingCollection of the model already has a RowSparseAdam attached")
        params = [p for p in model.parameters() if p.requires_grad]
        if not params:
            raise ValueError("KerasAdam: the model has no trainable parameters")
        release_row_optimizers(model)
        b1, b2, eps, lr = self.beta_1, self.beta_2, self.epsilon, self.kw["lr"]
        self.clock = ops.AdamClock(lr, b1, b2, eps, device=params[0].device, history=HISTORY)
        self.row_optimizers, on_rows = [], set()
        if self.tables == "rows":
            for c in colls:
                if not c.weight.requires_grad:
                    continue
                ro = RowSparseAdam(c, lr, b1, b2, eps, clock=self.clock)
                ro._keras_adam = True
                self.row_optimizers.append(ro)
                on_rows.update(id(t) for t in (c.weight, c.linear) if t is not None)
        dense = [p for p in params if id(p) not in on_rows]
        offsets, total = [], 0
        for p in dense:
            if not p.is_contiguous():
                raise ValueError(f"KerasAdam: a parameter of shape {tuple(p.shape)} is not contiguous")
            offsets.append(total)
            total += (p.numel() + 3) // 4 * 4          # every variable's m and v start 16-B aligned
        m = torch.zeros((total,), dtype=torch.float32, device=params[0].device)
        v = torch.zeros_like(m)
        self.dense = [(p, m[o:o + p.numel()].view_as(p), v[o:o + p.numel()].view_as(p)) for p, o in zip(dense, offsets)]
        return self

    def zero_grad(self, set_to_none: bool = True) -> None:
        for p, _, _ in self.dense:
            if p.grad is None:
                continue
            if set_to_none:
                p.grad = None
            else:
                p.grad.detach_().zero_()

    def step(self) -> None:
        if self.clock is None:
            raise RuntimeError("KerasAdam.step(): build_for_model(model) first")
        self.clock.lr = float(self.kw["lr"])
        self.clock.advance()
        live = [(p, p.grad, m, v) for p, m, v in self.dense if p.grad is not None]
        if live:
            ps, gs, ms, vs = zip(*live)
            ops.adam_step_multi_(ps, [g.contiguous() for g in gs], ms, vs, self.clock)
        for ro in self.row_optimizers:
            if ro.has_pending:
                ro.step()


def release_row_optimizers(model) -> None:
    """Flush the RowSparseAdam a KerasAdam build attached to each EmbeddingCollection of `model` and detach it: the
    tables then hold what dense Adam would and train with whatever optimizer the model is compiled with next."""
    from .embedding import EmbeddingCollection
    for c in model.modules():
        if isinstance(c, EmbeddingCollection) and getattr(c.row_optimizer, "_keras_adam", False):
            c.row_optimizer.flush()
            c.row_optimizer = None
