"""Whole-step training driver for the DCN model (`deep_recommenders.keras.layers.DCN`: embedding lookup -> [Cross stack ||
DNN tower] -> concat -> Dense(1) -> sigmoid; the stacking of the reference's tests/keras/test_dcn.py:27-32 on
keras/models/ranking/dcn.py:70-88): forward + backward + SGD as one CUDA-graph replay of hand-written kernels.

   ids [B,S] -> dr_embed_fm_fwd (pure gather)                     -> x0 [B, S*D]
             -> dr_cross_fwd x L (layer 0 with x = x0)            -> y_l, u_l saved
             -> dr_dense_fwd x n on x0                            -> deep
             -> dr_dcn_head_bce_fwd_bwd (no concat)               -> loss, prob, g_xc, g_deep, head gradients
             -> dr_dense_bwd_chain down the tower; the layer-0 input-gradient GEMM STORES into g_x0 (initialises it)
             -> dr_cross_bwd_acc top to bottom: every layer adds its x0 gradient into g_x0, the bottom layer (x is x0)
                its input gradient too -- the gradient of x0 is never assembled by element-wise passes
             -> dr_embed_fm_bwd (fused row-sparse SGD, scale = -lr) beside the layer-0 weight-gradient GEMM
             -> dr_sgd_step on the flat buffer of every Cross / DNN / head parameter

Every buffer is preallocated, so the step is capturable in a CUDA graph.  The model's parameters alias the flat buffer:
`model.logits`, `model.save` and the Keras engine keep working on the weights the trainer updates.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import _lib, ops
from ._lib import check
from .training import _WholeStepDriver, flat_params

HEAD_MAX_WIDTH = 4096      # dr_dcn_head_bce_fwd_bwd serves d + n up to this


class DCNTrainStep(_WholeStepDriver):
    def __init__(self, model, batch_size: int, lr: float = 0.01, id_dtype=torch.int64, use_graph: bool = True):
        self.lib = _lib.load()
        self.model = model
        coll = model.embeddings
        self.coll = coll
        self.B, self.S, self.D = int(batch_size), coll.num_slots, coll.dim
        self.d = self.S * self.D
        self.lr = float(lr)
        dev = coll.weight.device
        if dev.type != "cuda":
            raise _lib.DeepRecError("DCNTrainStep needs the model on a CUDA device (no CPU fallback)")
        self.dev = dev
        self.cross = list(model.cross)
        self.layers = list(model.dnn.layers)
        if not self.cross:
            raise ValueError("DCNTrainStep needs at least one Cross layer")
        if not self.layers:
            raise ValueError("DCNTrainStep needs at least one DNN layer (the head kernel reads the deep tower's output)")
        for c in self.cross:
            if c._kernel_regu is not None or c._bias_regu is not None:
                raise ValueError("DCNTrainStep has no penalty term: Cross layers with a regulariser are not served")
        B, d = self.B, self.d
        self.n = self.layers[-1].units
        if d + self.n > HEAD_MAX_WIDTH:
            raise ValueError(f"DCNTrainStep: head width d + n = {d + self.n} exceeds the {HEAD_MAX_WIDTH} the head kernel serves")
        # make sure the lazily built layers exist, then move every dense parameter into ONE flat buffer
        for c in self.cross:
            if not c.built:
                c.build((B, d), device=dev)
        in_dim = d
        for l in self.layers:
            if not l.built:
                l.build((B, in_dim), device=dev)
            in_dim = l.units
        if not model.head.built:
            model.head.build((B, d + self.n), device=dev)
        params = []
        for c in self.cross:
            params += [c.kernel, c.kernel_u, c.kernel_v, c.bias]
        for l in self.layers + [model.head]:
            params += [l.kernel, l.bias]
        self.flat, self.gflat, views = flat_params(params, dev)
        L, nl = len(self.cross), len(self.layers)
        self.cw = views[:4 * L]                                   # per Cross layer: kernel, kernel_u, kernel_v, bias
        self.w = [views[4 * L + 2 * i] for i in range(nl)]        # (parameter, gradient) pairs
        self.b = [views[4 * L + 2 * i + 1] for i in range(nl)]
        self.hw, self.hb = views[-2], views[-1]
        self.rank = [0 if c.kernel is not None else int(c.kernel_u.shape[1]) for c in self.cross]
        self.alpha = [float(c._diag_scale or 0.0) for c in self.cross]
        f = dict(device=dev, dtype=torch.float32)
        self.ids = torch.zeros((B, self.S), device=dev, dtype=id_dtype)
        self.labels = torch.zeros((B,), **f)
        self.x0 = torch.empty((B, d), **f)
        self.ys = [torch.empty((B, d), **f) for _ in self.cross]
        self.us = [torch.empty((B, d), **f) for _ in self.cross]
        self.xus = [torch.empty((B, r), **f) if r else None for r in self.rank]
        self.h_ws = torch.empty((B, d), **f)
        self.t_ws = torch.empty((B, max(self.rank)), **f) if max(self.rank) else None
        self.g_pp = [torch.empty((B, d), **f) for _ in range(min(2, L))]      # dL/dy of the Cross layers, ping-pong
        self.g_x0 = torch.empty((B, d), **f)
        self.acts = [torch.empty((B, l.units), **f) for l in self.layers]
        self.g_acts = [torch.empty((B, l.units), **f) for l in self.layers]  # PRE-activation gradient of layer i
        self.logit = torch.empty((B,), **f)
        self.prob = torch.empty((B,), **f)
        self.g_logit = torch.empty((B,), **f)
        self.loss = torch.zeros((1,), **f)
        self.tp, _, self.rows = coll.pointers(coll.weight, coll.linear)
        kmax = max([d] + [l.units for l in self.layers])
        _lib.ensure_gemm_workspace(B, kmax, kmax, dev)
        self.graph = None
        self.use_graph = use_graph
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._side_stream = torch.cuda.Stream(device=dev)
        self._staged = None
        self.launches_per_step = None

    def _enqueue(self, mark=None):
        """`mark(label)` (optional) is called after each kernel group (profile_kernels)."""
        lib, st = self.lib, torch.cuda.current_stream().cuda_stream
        B, S, D, d, n = self.B, self.S, self.D, self.d, self.n
        c = self.coll
        mark = mark or (lambda label: None)
        P = ops._ptr
        mark("start")
        check(lib.dr_embed_fm_fwd(self.tp.data_ptr(), None, self.rows.data_ptr(), self.ids.data_ptr(),
                                  self.ids.element_size(), None, B, S, D, c.row_stride, c.lin_stride, 0,
                                  self.x0.data_ptr(), None, None, st), "dr_embed_fm_fwd")
        mark("embed_fm_fwd")
        L, nl = len(self.cross), len(self.layers)
        x = self.x0
        for i in range(L):
            (w, _), (uk, _), (vk, _), (b, _) = self.cw[4 * i:4 * i + 4]
            check(lib.dr_cross_fwd(self.x0.data_ptr(), x.data_ptr(), P(w), P(uk), P(vk), P(b), self.alpha[i], B, d,
                                   self.rank[i], P(self.xus[i]), self.us[i].data_ptr(), self.ys[i].data_ptr(), st),
                  "dr_cross_fwd")
            mark(f"cross_fwd_{i}")
            x = self.ys[i]
        x, K = self.x0, d
        for i, l in enumerate(self.layers):
            check(lib.dr_dense_fwd(x.data_ptr(), self.w[i][0].data_ptr(), P(self.b[i][0]), B, K, l.units, l._act,
                                   self.acts[i].data_ptr(), st), "dr_dense_fwd")
            mark(f"dense_fwd_{i}")
            x, K = self.acts[i], l.units
        g = self.g_pp[0]
        check(lib.dr_dcn_head_bce_fwd_bwd(self.ys[-1].data_ptr(), self.acts[-1].data_ptr(), self.hw[0].data_ptr(),
                                          P(self.hb[0]), self.labels.data_ptr(), B, d, n, self.layers[-1]._act,
                                          self.logit.data_ptr(), self.prob.data_ptr(), self.loss.data_ptr(),
                                          self.g_logit.data_ptr(), g.data_ptr(), self.g_acts[-1].data_ptr(),
                                          self.hw[1].data_ptr(), P(self.hb[1]), P(self.b[-1][1]), st),
              "dr_dcn_head_bce_fwd_bwd")
        mark("head_bce")
        # DNN backward first: its layer-0 input-gradient GEMM stores into g_x0, which initialises the buffer every Cross
        # layer then accumulates into.  g_acts[i] is a pre-activation gradient throughout (dr_dense_bwd_chain), so only
        # the layers below the top still need their bias column sums here (the top one's came from the head kernel).
        for i in range(nl - 1, 0, -1):
            l = self.layers[i]
            xin = self.acts[i - 1]
            check(lib.dr_dense_bwd_chain(xin.data_ptr(), self.w[i][0].data_ptr(), None, self.g_acts[i].data_ptr(), B,
                                         self.layers[i - 1].units, l.units, 0, None, self.g_acts[i - 1].data_ptr(),
                                         self.w[i][1].data_ptr(), None if i == nl - 1 else P(self.b[i][1]),
                                         xin.data_ptr(), self.layers[i - 1]._act, st), "dr_dense_bwd_chain")
            mark(f"dense_bwd_{i}")
        l0 = self.layers[0]
        check(lib.dr_dense_bwd(self.x0.data_ptr(), self.w[0][0].data_ptr(), None, self.g_acts[0].data_ptr(), B, d,
                               l0.units, 0, None, self.g_x0.data_ptr(), None, None if nl == 1 else P(self.b[0][1]), st),
              "dr_dense_bwd(dx)")
        mark("dense_bwd_0_dx")
        for i in range(L - 1, -1, -1):
            (w, gw), (uk, guk), (vk, gvk), (_, gb) = self.cw[4 * i:4 * i + 4]
            bottom = i == 0
            xin = self.x0 if bottom else self.ys[i - 1]
            gx = None if bottom else self.g_pp[1] if g is self.g_pp[0] else self.g_pp[0]
            check(lib.dr_cross_bwd_acc(self.x0.data_ptr(), xin.data_ptr(), P(w), P(uk), P(vk), self.alpha[i],
                                       self.us[i].data_ptr(), P(self.xus[i]), g.data_ptr(), B, d, self.rank[i],
                                       self.h_ws.data_ptr(), P(self.t_ws), self.g_x0.data_ptr(), P(gx), P(gw), P(guk),
                                       P(gvk), P(gb), 1 if bottom else 0, st), "dr_cross_bwd_acc")
            mark(f"cross_bwd_{i}")
            g = gx
        # g_x0 is complete: the HBM-bound embedding update runs on a side stream beside the layer-0 weight-gradient GEMM
        main, side = torch.cuda.current_stream(), self._side_stream
        fork = torch.cuda.Event()
        fork.record(main)
        side.wait_event(fork)
        with torch.cuda.stream(side):
            check(lib.dr_embed_fm_bwd(self.ids.data_ptr(), self.ids.element_size(), self.rows.data_ptr(),
                                      self.x0.data_ptr(), None, None, self.g_x0.data_ptr(), B, S, D, c.row_stride,
                                      c.lin_stride, 0, self.tp.data_ptr(), None, None, -self.lr, side.cuda_stream),
                  "dr_embed_fm_bwd")
        check(lib.dr_dense_bwd(self.x0.data_ptr(), self.w[0][0].data_ptr(), None, self.g_acts[0].data_ptr(), B, d,
                               l0.units, 0, None, None, self.w[0][1].data_ptr(), None, st), "dr_dense_bwd(dw)")
        main.wait_stream(side)
        mark("dense_bwd_0_dw+embed_fm_bwd")
        check(lib.dr_sgd_step(self.flat.data_ptr(), self.gflat.data_ptr(), self.flat.numel(), self.lr, st), "dr_sgd_step")
        mark("sgd")

    def _persistent_state(self) -> List[torch.Tensor]:
        """Every tensor a step mutates AND a later step reads: the tables and the flat parameter buffer."""
        return [self.coll.weight.data, self.flat]
