"""Whole-step training drivers for the hot path: forward + backward + optimizer of a DeepFM
model (reference: examples/train_deepfm_on_movielens_keras.py:38-54 -- compile(BCE, optimizer)
+ fit) as one CUDA-graph replay of hand-written kernels.

`DeepFMTrainStep(model, lr)` takes a `deep_recommenders.keras.models.ranking.DeepFM` and runs

   ids [B,S] -> dr_embed_fm_fwd -> Dense(relu)... -> Dense(1) -> BCE(fm_logit + dnn_logit)
             -> dr_dense_bwd x L -> dr_embed_fm_bwd (fused sparse SGD, scale = -lr)
             -> dr_sgd_step on the flat dense-parameter buffer

with every buffer preallocated, so the step is capturable in a CUDA graph (no allocator calls,
no host sync).  Optimizers (`optimizer=`):
  "sgd"       (default, the benchmarked step) row-sparse SGD fused into the embedding backward (only the rows
              a batch touches are read-modify-written), dense SGD on the tower;
  "adam"      what the reference examples train with (tf.keras.optimizers.Adam, eps 1e-7): TensorFlow applies
              Adam DENSELY to embedding variables too, so this is dr_adam_step over the whole table arena
              (gradient arena + m + v: 4x the table memory, 7 arena sweeps per step) -- parity-exact, slow;
  "lazy_adam" row-sparse Adam (dr_lazy_adam_rows: tfa LazyAdam semantics, a stated deviation) on the tables,
              dense Adam on the tower.
The Adam step counter and bias-corrected rate live on the device (dr_adam_advance), so all three replay as one
CUDA graph.

`train_step_host` is the end-to-end entry: ids / labels arrive in (pinned) HOST memory, are
copied H2D on a side stream one batch ahead (double buffered), and the loss is read back D2H.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import _lib, ops
from ._lib import check


def flat_params(params, device):
    """Move `params` (entries may be None) into ONE zero-filled flat buffer, every parameter starting on a 16-byte boundary
    (the tensor-core path splits operands with float4), and rebind each `param.data` to its view, so the model keeps
    working on the weights the trainer updates.  Returns (flat, gflat, [(param view, gradient view) or (None, None)])."""
    r4 = lambda n: (n + 3) // 4 * 4
    total = sum(r4(p.numel()) for p in params if p is not None)
    flat = torch.zeros(total, device=device, dtype=torch.float32)
    gflat = torch.zeros(total, device=device, dtype=torch.float32)
    views, o = [], 0
    with torch.no_grad():
        for p in params:
            if p is None:
                views.append((None, None))
                continue
            n = p.numel()
            flat[o:o + n].copy_(p.reshape(-1))
            p.data = flat[o:o + n].view_as(p)
            views.append((p.data, gflat[o:o + n].view_as(p)))
            o += r4(n)
    return flat, gflat, views


class _WholeStepDriver:
    """What every whole-step trainer shares once it has `_enqueue(mark)` (the step as raw C-ABI calls on the current
    stream), `_persistent_state()`, the static `ids` / `labels` buffers, `loss`, `dev`, `use_graph`, `_copy_stream` and
    `_staged`: CUDA-graph capture and replay, the host-batch pipeline and the per-kernel-group profile.

    A multi-process trainer overrides `_barrier` (all ranks meet), `check_overflow` (raise on a sticky device-side error
    flag) and `_record_graph` / `_replay` (a step that is not one graph)."""

    def _barrier(self):
        """Called on both sides of the warm-up restore in `capture`; a no-op for a single process."""

    def check_overflow(self):
        """Raise if a step since the last check hit a device-side capacity limit; a no-op unless a trainer has one."""

    def _record_graph(self):
        """Record one step; `run` hands what this returns to `_replay`."""
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._enqueue()
        return g

    def _replay(self):
        self.graph.replay()

    def profile_kernels(self, ids_pool, labels_pool, iters: int = 10):
        """Eager (non-graph) passes with a CUDA event on the launching stream between kernel groups.
        Returns ({"embed_fm_fwd_ms": ...}, {label: mean ms}) -- the live per-kernel timing bench.py
        reports in `roofline` and `kernel_ms`."""
        runs = []
        for it in range(iters + 2):      # back-to-back, no host sync in between (steady-state clocks / caches)
            self.ids.copy_(ids_pool[it % len(ids_pool)], non_blocking=True)
            self.labels.copy_(labels_pool[it % len(labels_pool)].reshape(-1), non_blocking=True)
            evs = []

            def mark(label, evs=evs):
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                evs.append((label, e))

            self._enqueue(mark)
            runs.append(evs)
        torch.cuda.synchronize()
        sums, count = {}, 0
        for evs in runs[2:]:
            count += 1
            for (l0, e0), (l1, e1) in zip(evs[:-1], evs[1:]):
                sums[l1] = sums.get(l1, 0.0) + e0.elapsed_time(e1)
        shares = {k: v / count for k, v in sums.items()}
        return {"embed_fm_fwd_ms": shares.get("embed_fm_fwd", shares.get("embed_fm_fwd_p2p"))}, shares

    def capture(self):
        """Warm up (sets kernel attributes) then record the step into a CUDA graph.

        Side-effect free: the warm-up launch is a real step on whatever the static id / label buffers hold, so every
        parameter and every piece of optimizer state (Adam clock, m, v, stamps) is snapshotted before it and restored
        after it -- `capture()` leaves the trainer bit-identical to how it found it."""
        n0 = _lib.launch_count()
        with torch.no_grad():
            state = self._persistent_state()
            saved = [t.clone() for t in state]
            s = torch.cuda.Stream(device=self.dev)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self._enqueue()
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            self._barrier()          # every peer's remote updates of the warm-up step have landed
            for t, keep in zip(state, saved):
                t.copy_(keep)
            del saved
            torch.cuda.synchronize()
            self._barrier()          # nobody starts a real step before every peer has restored its state
        self.launches_per_step = _lib.launch_count() - n0
        self.check_overflow()
        if self.use_graph:
            self.graph = self._record_graph()
        return self

    def run(self):
        """One step on whatever is in self.ids / self.labels (device resident)."""
        if self.graph is not None:
            self._replay()
        else:
            self._enqueue()

    def step(self, ids: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """Device-resident inputs: copy into the static buffers (D2D) and run. Returns loss[1]."""
        self.ids.copy_(ids, non_blocking=True)
        self.labels.copy_(labels.reshape(-1), non_blocking=True)
        self.run()
        return self.loss

    # ---- end-to-end: host buffers in, loss out ---------------------------------------------------
    def stage_host(self, ids_host: torch.Tensor, labels_host: torch.Tensor):
        """Start the H2D copy of the NEXT batch on the copy stream into the spare device buffers."""
        if not hasattr(self, "_spare"):
            self._spare = (torch.empty_like(self.ids), torch.empty_like(self.labels))
        with torch.cuda.stream(self._copy_stream):
            self._spare[0].copy_(ids_host, non_blocking=True)
            self._spare[1].copy_(labels_host.reshape(-1), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        self._staged = ev

    def train_step_host(self, ids_host, labels_host, next_ids_host=None, next_labels_host=None) -> float:
        """Public end-to-end step.  ids/labels are HOST tensors (pinned for async copies).  If the
        caller passes the next batch too, its H2D copy overlaps this step's kernels."""
        cur = torch.cuda.current_stream()
        if self._staged is None:
            self.stage_host(ids_host, labels_host)
        cur.wait_event(self._staged)
        # swap staged buffers into the static ones the graph reads (D2D, 13.6 MB at C2)
        self.ids.copy_(self._spare[0], non_blocking=True)
        self.labels.copy_(self._spare[1], non_blocking=True)
        done = torch.cuda.Event()
        done.record(cur)
        self._staged = None
        if next_ids_host is not None:
            self._copy_stream.wait_event(done)
            self.stage_host(next_ids_host, next_labels_host)
        self.run()
        loss = float(self.loss.item())          # D2H read of the step's result (synchronises)
        self.check_overflow()
        return loss

    def fit_host(self, batches, depth: int = 2) -> List[float]:
        """Pipelined epoch loop over HOST batches: the public end-to-end call.

        `batches`: sequence of (ids_host, labels_host) HOST tensors (pinned for asynchronous copies).  Per step, inside
        this call: the H2D copy of the batch (copy stream, overlapping the previous step's kernels), the D2D swap into the
        static buffers the CUDA graph reads, the step, and an asynchronous D2H copy of the step's loss into a pinned ring.
        The host reads the loss of step k - depth while step k is being enqueued, i.e. it never idles the GPU waiting for
        a scalar (train_step_host blocks on `loss.item()` every step); returns every step's loss, in order.
        `check_overflow` runs once at the end."""
        batches = list(batches)
        if not batches:
            self.check_overflow()
            return []
        cur = torch.cuda.current_stream()
        ring = getattr(self, "_loss_ring", None)
        if ring is None or ring.numel() < depth + 1:
            ring = self._loss_ring = torch.empty((depth + 1,), dtype=torch.float32).pin_memory()
        events: List[Optional[torch.cuda.Event]] = [None] * (depth + 1)
        losses: List[float] = []
        self._copy_stream.wait_stream(cur)          # whatever still reads the spare buffers has been enqueued on `cur`
        self.stage_host(*batches[0])
        for k, _ in enumerate(batches):
            cur.wait_event(self._staged)
            self.ids.copy_(self._spare[0], non_blocking=True)            # D2D swap into the graph's static buffers
            self.labels.copy_(self._spare[1], non_blocking=True)
            done = torch.cuda.Event()
            done.record(cur)
            self._staged = None
            if k + 1 < len(batches):
                self._copy_stream.wait_event(done)                       # the spare buffers are free again
                self.stage_host(*batches[k + 1])
            self.run()
            slot = k % (depth + 1)
            if events[slot] is not None:                                 # the loss that lived in this slot: step k-depth-1
                events[slot].synchronize()
                losses.append(float(ring[slot]))
            ring[slot:slot + 1].copy_(self.loss.reshape(-1)[:1], non_blocking=True)     # D2H read of this step's result
            ev = torch.cuda.Event()
            ev.record(cur)
            events[slot] = ev
        n = len(batches)
        for k in range(max(0, n - (depth + 1)), n):                      # drain, in step order
            slot = k % (depth + 1)
            events[slot].synchronize()
            losses.append(float(ring[slot]))
        self.check_overflow()
        return losses


class _DeepFMTower(_WholeStepDriver):
    """The DeepFM tower as both DeepFM trainers run it: from the stacked embeddings `stack` [B, S*D] and `fm_logit` to
    the BCE loss, the tower gradients in `gflat` and the input gradient `g_stack` the embedding update reads.  The
    trainer owns the gather, the embedding update, the optimizers, the streams and `dr_gemm_plane_cache`."""

    def _init_tower(self, layers, lead=()):
        """Move `lead` and every Dense parameter of `layers` (built) into `flat`, allocate the tower's buffers and size
        the GEMM workspace for them.  Returns the (parameter, gradient) views of `lead`."""
        self.layers = layers
        B, S, D, dev = self.B, self.S, self.D, self.dev
        lead = list(lead)
        self.flat, self.gflat, views = flat_params(lead + [p for l in layers for p in (l.kernel, l.bias)], dev)
        tower = views[len(lead):]
        self.w, self.gw = [p for p, _ in tower[0::2]], [g for _, g in tower[0::2]]
        self.b, self.gb = [p for p, _ in tower[1::2]], [g for _, g in tower[1::2]]
        f = dict(device=dev, dtype=torch.float32)
        self.stack = torch.empty((B, S, D), **f)
        self.sum_e = torch.empty((B, D), **f)
        self.fm_logit = torch.empty((B,), **f)
        self.acts = [torch.empty((B, l.units), **f) for l in layers]
        self.g_acts = [torch.empty((B, l.units), **f) for l in layers]       # dL/d(output of layer i)
        self.gz_ws = [torch.empty((B, l.units), **f) if l._act != 0 else None for l in layers]
        self.g_stack = torch.empty((B, S, D), **f)
        self.loss = torch.zeros((1,), **f)
        self.prob = torch.empty((B,), **f)
        # the skinny end (final Dense(1) + BCE + their backward) is ONE kernel when the layer below is <= 256 wide
        L = len(layers)
        self._fused_head = (L >= 2 and layers[-1].units == 1 and layers[-1]._act == 0 and layers[-2].units <= 256
                            and self.b[-1] is not None and self.b[-2] is not None)
        widths = [S * D] + [l.units for l in layers]
        _lib.ensure_gemm_workspace(B, max(widths), max(widths), dev)
        # plane cache: x, every activation, every upstream gradient and every kernel, hi + lo
        cache_bytes = 8 * (B * (widths[0] + 2 * sum(widths[1:])) + sum(a * b for a, b in zip(widths[:-1], widths[1:])))
        _lib.set_workspace(max(cache_bytes * 5 // 4 + (1 << 20), _lib._workspace.numel() if _lib._workspace is not None else 0), dev)
        return views[:len(lead)]

    def _tower_fwd_bwd(self, mark, first: int = 0):
        """Dense forwards from layer `first` (the layers below it have run already), the loss head, the chained backward
        and the layer-0 input gradient into `g_stack`, on the current stream."""
        lib, st = self.lib, torch.cuda.current_stream().cuda_stream
        B, S, D = self.B, self.S, self.D
        L = len(self.layers)
        head = self._fused_head
        gz = self.g_acts[-1]                                   # [B,1]: dL/dlogit
        x, K = (self.stack, S * D) if first == 0 else (self.acts[first - 1], self.layers[first - 1].units)
        for i in range(first, L - 1 if head else L):
            l = self.layers[i]
            check(lib.dr_dense_fwd(x.data_ptr(), self.w[i].data_ptr(), ops._ptr(self.b[i]), B, K, l.units, l._act,
                                   self.acts[i].data_ptr(), st), "dr_dense_fwd")
            mark(f"dense_fwd_{i}")
            x, K = self.acts[i], l.units
        if head:
            check(lib.dr_dense_head_bce_fwd_bwd(self.acts[L - 2].data_ptr(), self.w[L - 1].data_ptr(),
                                                self.b[L - 1].data_ptr(), self.fm_logit.data_ptr(), self.labels.data_ptr(),
                                                B, self.layers[L - 2].units, self.layers[L - 2]._act,
                                                self.acts[L - 1].data_ptr(), self.prob.data_ptr(), self.loss.data_ptr(),
                                                gz.data_ptr(), self.g_acts[L - 2].data_ptr(), self.gw[L - 1].data_ptr(),
                                                self.gb[L - 1].data_ptr(), self.gb[L - 2].data_ptr(), st),
                  "dr_dense_head_bce_fwd_bwd")
            mark("head_bce")
        else:
            check(lib.dr_bce_logits_fwd_bwd(self.acts[-1].data_ptr(), self.fm_logit.data_ptr(), self.labels.data_ptr(), B,
                                            self.prob.data_ptr(), self.loss.data_ptr(), gz.data_ptr(), st), "dr_bce")
            mark("bce")
        # Chained backward: layer i's input gradient leaves its GEMM already multiplied by act'(output of layer i-1)
        # (dr_dense_bwd_chain), so g_acts[i-1] IS the pre-activation gradient of layer i-1 and no layer below the top
        # needs its own activation-gradient pass (only the column sums for the bias gradient; the layer right below the
        # fused head got those from the head kernel too).
        first_bwd = L - 2 if head else L - 1                  # highest layer that still needs its backward here
        for i in range(first_bwd, 0, -1):
            l = self.layers[i]
            top = (i == L - 1)                                # only without the fused head: gy is dL/d(output), not gz
            have_gb = head and i == L - 2
            xin, Kin, gx = self.acts[i - 1], self.layers[i - 1].units, self.g_acts[i - 1]
            check(lib.dr_dense_bwd_chain(xin.data_ptr(), self.w[i].data_ptr(), self.acts[i].data_ptr() if top else None,
                                         self.g_acts[i].data_ptr(), B, Kin, l.units, l._act if top else 0,
                                         ops._ptr(self.gz_ws[i]) if top else None, gx.data_ptr(), self.gw[i].data_ptr(),
                                         None if have_gb else ops._ptr(self.gb[i]), xin.data_ptr(),
                                         self.layers[i - 1]._act, st),
                  "dr_dense_bwd_chain")
            mark(f"dense_bwd_{i}")
        # layer 0: the input gradient only (the embedding update needs it); its weight gradient is `_tower_dw`
        l = self.layers[0]
        top0 = L == 1
        gb0 = None if (head and L == 2) else ops._ptr(self.gb[0])
        check(lib.dr_dense_bwd(self.stack.data_ptr(), self.w[0].data_ptr(), self.acts[0].data_ptr() if top0 else None,
                               self.g_acts[0].data_ptr(), B, S * D, l.units, l._act if top0 else 0,
                               ops._ptr(self.gz_ws[0]) if top0 else None,
                               self.g_stack.data_ptr(), None, gb0, st), "dr_dense_bwd(dx)")
        mark("dense_bwd_0_dx")

    def _tower_dw(self):
        """The layer-0 weight gradient, on the current stream (after `_tower_fwd_bwd`)."""
        l = self.layers[0]
        gz0 = (self.gz_ws[0] if l._act != 0 else self.g_acts[0]) if len(self.layers) == 1 else self.g_acts[0]
        check(self.lib.dr_dense_bwd(self.stack.data_ptr(), self.w[0].data_ptr(), None, gz0.data_ptr(), self.B,
                                    self.S * self.D, l.units, 0, None, None, self.gw[0].data_ptr(), None,
                                    torch.cuda.current_stream().cuda_stream), "dr_dense_bwd(dw)")

    def time_embed_fwd(self, ids_pool, iters: int = 30) -> float:
        """Mean duration (ms) of the fused gather+FM forward alone: `iters` back-to-back launches on the
        launching stream between two CUDA events, cycling through the id pool (tables >> L2)."""
        st = torch.cuda.current_stream().cuda_stream
        for k in range(5):
            self._launch_embed_fwd(ids_pool[k % len(ids_pool)], st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(iters):
            self._launch_embed_fwd(ids_pool[k % len(ids_pool)], st)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters


class DeepFMTrainStep(_DeepFMTower):
    def __init__(self, model, batch_size: int, lr: float = 0.01, id_dtype=torch.int64, use_graph: bool = True,
                 optimizer: str = "sgd", beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-7,
                 embed_fwd: str = "ldg", fwd_chunks: int = 1, dw_first: bool = False):
        self.lib = _lib.load()
        # fwd_chunks > 1: the gather and the first tower GEMM run as `fwd_chunks` alternating launches over slices of the
        # batch (gather slice k -> GEMM slice k -> gather slice k+1 ...): a slice's stacked rows are still dirty in L2 when
        # its GEMM reads them, and their write-back drains behind the (shared-memory-bound) GEMM instead of inside the
        # DRAM-bound gather.  Same kernels, same results (examples are independent in both).
        self.fwd_chunks = max(1, int(fwd_chunks))
        # dw_first: enqueue the layer-0 weight-gradient GEMM BEFORE the embedding update of the side stream (both depend
        # only on the layer-0 input gradient), so the persistent GEMM owns one CTA slot per SM and the update co-resides
        self.dw_first = bool(dw_first)
        if optimizer not in ("sgd", "adam", "lazy_adam", "adam_rows", "adam_rows_tf"):
            raise ValueError(f"optimizer must be 'sgd', 'adam', 'lazy_adam', 'adam_rows' or 'adam_rows_tf', got {optimizer!r}")
        self.optimizer = optimizer
        if embed_fwd not in ("ldg", "tma"):
            raise ValueError(f"embed_fwd must be 'ldg' (register loads, default) or 'tma' (gather4 staging), got {embed_fwd!r}")
        self.embed_fwd = embed_fwd
        self.model = model
        coll = model.embeddings
        self.coll = coll
        self.B, self.S, self.D = int(batch_size), coll.num_slots, coll.dim
        self.lr = float(lr)
        dev = coll.weight.device
        if dev.type != "cuda":
            raise _lib.DeepRecError("DeepFMTrainStep needs the model on a CUDA device (no CPU fallback)")
        self.dev = dev
        # make sure the lazily built Dense layers exist, then move the tower into ONE flat buffer
        layers = list(model._dnn.layers)
        in_dim = self.S * self.D
        for l in layers:
            if not l.built:
                l.build((self.B, in_dim), device=dev)
            in_dim = l.units
        self._init_tower(layers)
        B, S, D = self.B, self.S, self.D
        f = dict(device=dev, dtype=torch.float32)
        self.ids = torch.zeros((B, S), device=dev, dtype=id_dtype)
        self.labels = torch.zeros((B,), **f)
        self.tp, self.lp, self.rows = coll.pointers(coll.weight, coll.linear)
        if optimizer != "sgd":
            # optimizer state: gradient arena (all-zero between steps), m, v in the tables' own layout
            self.clock = ops.AdamClock(lr, beta1, beta2, eps, device=dev,
                                       history=(1 << 16) if optimizer == "adam_rows_tf" else 0)
            z = lambda t: None if (t is None or optimizer in ("adam_rows", "adam_rows_tf")) else torch.zeros_like(t)
            self.g_arena, self.m_arena, self.v_arena = z(coll.weight.data), z(coll.weight.data), z(coll.weight.data)
            self.g_lin, self.m_lin, self.v_lin = z(coll.linear), z(coll.linear), z(coll.linear)
            self.g_bias, self.m_bias, self.v_bias = (torch.zeros((1,), **f) for _ in range(3))
            self.m_flat, self.v_flat = torch.zeros_like(self.flat), torch.zeros_like(self.flat)
            if optimizer not in ("adam_rows", "adam_rows_tf"):
                self.gtp, self.glp, _ = coll.pointers(self.g_arena, self.g_lin, cache=False)
            self.stamp = (torch.zeros((coll.total_rows,), device=dev, dtype=torch.int32)
                          if optimizer == "lazy_adam" else None)
            self.state = None
            if optimizer in ("adam_rows", "adam_rows_tf"):
                # row-sparse Adam fused into the backward: ONE state block per row [g | m | v | g_w m_w v_w count]
                # replaces the three table-shaped arenas (dr_embed_fm_bwd_adam)
                ss = self.lib.dr_embed_adam_state_stride(D)
                self.state = torch.zeros((coll.total_rows, ss), **f)
                self.g_arena = self.m_arena = self.v_arena = self.g_lin = self.m_lin = self.v_lin = None
        self.graph = None
        self.use_graph = use_graph
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._side_stream = torch.cuda.Stream(device=dev)
        self._staged = None
        self.launches_per_step = None

    # ---- the step, as raw C-ABI calls on the current stream ------------------------------------
    def _enqueue(self, mark=None):
        """`mark(label)` (optional) is called after each kernel group; profile_kernels uses it to
        drop a CUDA event on the launching stream between groups."""
        lib, st = self.lib, torch.cuda.current_stream().cuda_stream
        B, S, D = self.B, self.S, self.D
        c = self.coll
        mark = mark or (lambda label: None)
        check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")   # one split per tensor per step
        if self.optimizer != "sgd":
            self.clock.advance()                                  # t += 1, lr_t (device scalars)
        mark("start")
        if self.optimizer == "adam_rows_tf":
            # tf.keras Adam is dense: rows move in the steps that do not touch them.  Before the forward reads them, the
            # rows of THIS batch replay their pending steps (and the batch's per-row lookup counts are taken)
            ck = self.clock
            check(lib.dr_embed_adam_prepare(self.ids.data_ptr(), self.ids.element_size(), B, S, D, self.rows.data_ptr(),
                                            c._offsets.data_ptr(), c.row_stride, c.lin_stride, c.flags, self.tp.data_ptr(),
                                            self.lp.data_ptr(), self.state.data_ptr(), ck.step.data_ptr(),
                                            ck.lr_hist.data_ptr(), ck.lr_hist.numel(), ck.lr, ck.beta1, ck.beta2, ck.eps, st),
                  "dr_embed_adam_prepare")
            mark("adam_prepare")
        nch = self.fwd_chunks if self.embed_fwd == "ldg" else 1
        if nch > 1:
            # slices on 128-row boundaries (the GEMM's tile height)
            per = (((B + nch - 1) // nch) + 127) // 128 * 128
            bounds = [(b0, min(B, b0 + per)) for b0 in range(0, B, per)]
        else:
            bounds = [(0, B)]
        l0 = self.layers[0]
        chunk_l0 = len(bounds) > 1
        esz = self.ids.element_size()
        for (b0, b1) in bounds:
            if self.embed_fwd == "tma":      # opt-in: rows staged through TMA (tile::gather4) into shared memory
                check(lib.dr_embed_fm_fwd_tma(c.weight.data_ptr(), c.total_rows, c._offsets.data_ptr(), self.rows.data_ptr(),
                                              self.ids.data_ptr(), esz, c.bias.data_ptr(), B, S, D,
                                              c.row_stride, self.stack.data_ptr(), self.sum_e.data_ptr(),
                                              self.fm_logit.data_ptr(), st), "dr_embed_fm_fwd_tma")
            else:
                check(lib.dr_embed_fm_fwd(self.tp.data_ptr(), self.lp.data_ptr(), self.rows.data_ptr(),
                                          self.ids.data_ptr() + b0 * S * esz, esz, c.bias.data_ptr(), b1 - b0, S, D,
                                          c.row_stride, c.lin_stride, c.flags, self.stack.data_ptr() + b0 * S * D * 4,
                                          self.sum_e.data_ptr() + b0 * D * 4, self.fm_logit.data_ptr() + b0 * 4, st),
                      "dr_embed_fm_fwd")
            mark("embed_fm_fwd")
            if chunk_l0:
                check(lib.dr_dense_fwd(self.stack.data_ptr() + b0 * S * D * 4, self.w[0].data_ptr(), ops._ptr(self.b[0]),
                                       b1 - b0, S * D, l0.units, l0._act, self.acts[0].data_ptr() + b0 * l0.units * 4, st),
                      "dr_dense_fwd")
                mark("dense_fwd_0")
        if self.optimizer == "adam_rows":     # per-row lookup counts of this batch: on the side stream, behind the GEMMs
            self._side_stream.wait_stream(torch.cuda.current_stream())   # (not behind the gather: both are DRAM-bound)
            with torch.cuda.stream(self._side_stream):
                check(lib.dr_embed_adam_count(self.ids.data_ptr(), self.ids.element_size(), B, S, D, self.rows.data_ptr(),
                                              c._offsets.data_ptr(), self.state.data_ptr(), self._side_stream.cuda_stream),
                      "dr_embed_adam_count")
        self._tower_fwd_bwd(mark, first=1 if chunk_l0 else 0)
        # layer 0's weight gradient (tensor cores) runs CONCURRENTLY with the HBM-bound embedding update on a side stream
        gz = self.g_acts[-1]
        main = torch.cuda.current_stream()
        side = self._side_stream
        adam = self.optimizer != "sgd"
        fork = torch.cuda.Event()
        fork.record(main)                                  # layer-0 input gradient done: both branches may start
        if self.dw_first:                                  # the persistent GEMM takes its one CTA per SM first; the update's
            self._tower_dw()                               # CTAs fill what is left of every SM (knob tc_dw_share)
        side.wait_event(fork)
        with torch.cuda.stream(side):
            sst = side.cuda_stream
            if self.optimizer == "adam_rows_tf":  # the same, equal to tf.keras Adam: skipped steps of a row are replayed
                ck = self.clock
                check(lib.dr_embed_fm_bwd_adam_tf(self.ids.data_ptr(), self.ids.element_size(), self.rows.data_ptr(),
                                                  c._offsets.data_ptr(), self.stack.data_ptr(), self.sum_e.data_ptr(),
                                                  gz.data_ptr(), self.g_stack.data_ptr(), B, S, D, c.row_stride,
                                                  c.lin_stride, c.flags, self.tp.data_ptr(), self.lp.data_ptr(),
                                                  self.state.data_ptr(), self.g_bias.data_ptr(), ck.step.data_ptr(),
                                                  ck.lr_t.data_ptr(), ck.lr_hist.data_ptr(), ck.lr_hist.numel(), ck.lr,
                                                  ck.beta1, ck.beta2, ck.eps, sst), "dr_embed_fm_bwd_adam_tf")
                check(lib.dr_adam_step(c.bias.data_ptr(), self.g_bias.data_ptr(), self.m_bias.data_ptr(),
                                       self.v_bias.data_ptr(), 1, 0.0, ck.beta1, ck.beta2, ck.eps, 1, ck.lr_t.data_ptr(), sst),
                      "dr_adam_step(bias)")
            elif self.optimizer == "adam_rows":     # Adam of the touched rows inside the backward scatter (one kernel)
                ck = self.clock
                check(lib.dr_embed_fm_bwd_adam(self.ids.data_ptr(), self.ids.element_size(), self.rows.data_ptr(),
                                               c._offsets.data_ptr(), self.stack.data_ptr(), self.sum_e.data_ptr(),
                                               gz.data_ptr(), self.g_stack.data_ptr(), B, S, D, c.row_stride, c.lin_stride,
                                               c.flags, self.tp.data_ptr(), self.lp.data_ptr(), self.state.data_ptr(),
                                               self.g_bias.data_ptr(), ck.lr_t.data_ptr(), ck.beta1, ck.beta2, ck.eps, sst),
                      "dr_embed_fm_bwd_adam")
                check(lib.dr_adam_step(c.bias.data_ptr(), self.g_bias.data_ptr(), self.m_bias.data_ptr(),
                                       self.v_bias.data_ptr(), 1, 0.0, ck.beta1, ck.beta2, ck.eps, 1, ck.lr_t.data_ptr(), sst),
                      "dr_adam_step(bias)")
            elif not adam:     # fused row-sparse SGD: the backward updates the parameter arena in place
                check(lib.dr_embed_fm_bwd(self.ids.data_ptr(), self.ids.element_size(), self.rows.data_ptr(),
                                          self.stack.data_ptr(), self.sum_e.data_ptr(), gz.data_ptr(),
                                          self.g_stack.data_ptr(), B, S, D, c.row_stride, c.lin_stride, c.flags,
                                          self.tp.data_ptr(), self.lp.data_ptr(), c.bias.data_ptr(), -self.lr,
                                          sst), "dr_embed_fm_bwd")
            else:            # Adam is not linear in g: accumulate the row gradients first (scale = 1), then update
                ck = self.clock
                check(lib.dr_embed_fm_bwd(self.ids.data_ptr(), self.ids.element_size(), self.rows.data_ptr(),
                                          self.stack.data_ptr(), self.sum_e.data_ptr(), gz.data_ptr(),
                                          self.g_stack.data_ptr(), B, S, D, c.row_stride, c.lin_stride, c.flags,
                                          self.gtp.data_ptr(), self.glp.data_ptr(), self.g_bias.data_ptr(), 1.0,
                                          sst), "dr_embed_fm_bwd")
                lt = ck.lr_t.data_ptr()
                if self.optimizer == "adam":
                    w = c.weight.data
                    check(lib.dr_adam_step(w.data_ptr(), self.g_arena.data_ptr(), self.m_arena.data_ptr(),
                                           self.v_arena.data_ptr(), w.numel(), 0.0, ck.beta1, ck.beta2, ck.eps, 1, lt,
                                           sst), "dr_adam_step(tables)")
                    if c.linear is not None:
                        check(lib.dr_adam_step(c.linear.data_ptr(), self.g_lin.data_ptr(), self.m_lin.data_ptr(),
                                               self.v_lin.data_ptr(), c.linear.numel(), 0.0, ck.beta1, ck.beta2,
                                               ck.eps, 1, lt, sst), "dr_adam_step(first order)")
                else:
                    has_lin = c.linear is not None
                    check(lib.dr_lazy_adam_rows(self.ids.data_ptr(), self.ids.element_size(), B, S, D,
                                                self.rows.data_ptr(), c._offsets.data_ptr(), c.weight.data_ptr(),
                                                self.g_arena.data_ptr(), self.m_arena.data_ptr(),
                                                self.v_arena.data_ptr(), c.row_stride, c.flags,
                                                c.linear.data_ptr() if has_lin else None,
                                                self.g_lin.data_ptr() if has_lin else None,
                                                self.m_lin.data_ptr() if has_lin else None,
                                                self.v_lin.data_ptr() if has_lin else None, self.stamp.data_ptr(),
                                                ck.step.data_ptr(), lt, ck.beta1, ck.beta2, ck.eps, sst),
                          "dr_lazy_adam_rows")
                check(lib.dr_adam_step(c.bias.data_ptr(), self.g_bias.data_ptr(), self.m_bias.data_ptr(),
                                       self.v_bias.data_ptr(), 1, 0.0, ck.beta1, ck.beta2, ck.eps, 1, lt, sst),
                      "dr_adam_step(bias)")
        if not self.dw_first:
            self._tower_dw()
        main.wait_stream(side)
        mark("dense_bwd_0_dw+embed_fm_bwd")
        if not adam:
            check(lib.dr_sgd_step(self.flat.data_ptr(), self.gflat.data_ptr(), self.flat.numel(), self.lr, st), "dr_sgd_step")
        else:
            ck = self.clock
            check(lib.dr_adam_step(self.flat.data_ptr(), self.gflat.data_ptr(), self.m_flat.data_ptr(),
                                   self.v_flat.data_ptr(), self.flat.numel(), 0.0, ck.beta1, ck.beta2, ck.eps, 0,
                                   ck.lr_t.data_ptr(), st), "dr_adam_step(tower)")
        check(lib.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
        mark("sgd")

    def _launch_embed_fwd(self, ids, st):
        c = self.coll
        check(self.lib.dr_embed_fm_fwd(self.tp.data_ptr(), self.lp.data_ptr(), self.rows.data_ptr(), ids.data_ptr(),
                                       ids.element_size(), c.bias.data_ptr(), self.B, self.S, self.D, c.row_stride,
                                       c.lin_stride, c.flags, self.stack.data_ptr(), self.sum_e.data_ptr(),
                                       self.fm_logit.data_ptr(), st), "dr_embed_fm_fwd")

    def _persistent_state(self) -> List[torch.Tensor]:
        """Every tensor a step mutates AND a later step reads: parameters and optimizer state."""
        c = self.coll
        st = [c.weight.data, self.flat]
        st += [t.data for t in (c.linear, c.bias) if t is not None]
        if self.optimizer != "sgd":
            st += [t for t in (self.g_arena, self.m_arena, self.v_arena, self.g_lin, self.m_lin, self.v_lin, self.g_bias,
                               self.m_bias, self.v_bias, self.m_flat, self.v_flat, self.stamp, self.state, self.clock.step,
                               self.clock.lr_t, self.clock.lr_hist) if t is not None]
        return st

    def flush_optimizer(self) -> None:
        """optimizer="adam_rows_tf": replay the pending (skipped) Adam steps of EVERY table row up to the current step, so
        that the tables equal what tf.keras Adam's dense update would hold.  Call before reading the tables outside the
        trainer (evaluation, checkpoint); a no-op for the other optimizers."""
        if self.optimizer != "adam_rows_tf":
            return
        c, ck = self.coll, self.clock
        check(self.lib.dr_embed_adam_flush(self.rows.data_ptr(), c._offsets.data_ptr(), self.S, self.D, c.total_rows,
                                           c.row_stride, c.lin_stride, c.flags, self.tp.data_ptr(), self.lp.data_ptr(),
                                           self.state.data_ptr(), ck.step.data_ptr(), ck.lr_hist.data_ptr(),
                                           ck.lr_hist.numel(), ck.lr, ck.beta1, ck.beta2, ck.eps,
                                           torch.cuda.current_stream().cuda_stream), "dr_embed_adam_flush")
