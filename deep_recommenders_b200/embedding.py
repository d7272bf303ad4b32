"""EmbeddingCollection: the S embedding tables + first-order weights of a ranking model, laid
out for HBM as ONE arena per kind so a batch is served by ONE fused kernel launch.

Replaces the per-column ``tf.keras.layers.DenseFeatures(embedding_column)`` /
``DenseFeatures(indicator_columns) -> Dense(1)`` objects the reference builds
(keras/models/ranking/fm.py:47-51, deepfm.py:24-28; estimator/.../fm.py:43-52).

Layout in HBM (layout="fused", the default when the first-order term exists and D <= 28)
  weight : [sum_s rows_s, 32] fp32   row = [ D embedding floats | w | pad ] in ONE 128-byte,
           128-byte-aligned line: the first-order weight w of an id (the
           Dense(1, kernel_initializer="zeros") kernel entry of the reference's multi-hot linear
           term) travels in the same HBM line as its embedding vector: a separate 4-B first-order
           gather would touch a second random DRAM line per lookup; fusing them halves the random
           lines per lookup.
  bias   : [1]                       that Dense's bias.
layout="split": weight [sum rows, D] and linear [sum rows] as two arrays (two random lines per
lookup; used for D >= 32 where the row already fills whole lines).  Table s occupies rows
[off_s, off_s + rows_s) in either layout.
The reference densifies the indicator columns into a [B, sum_s N_s] multi-hot and multiplies
by a [sum N, 1] kernel (fm.py:16-20,26); the sparse gather-sum here is the same number.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
from torch import nn

from . import ops


def _flush_row_optimizer(module, prefix, keep_vars):
    if module.row_optimizer is not None:
        module.row_optimizer.flush()


class EmbeddingCollection(nn.Module):
    def __init__(self, rows: Sequence[int], dim: int, with_linear: bool = True, device=None,
                 init_stddev: Optional[float] = None, seed: Optional[int] = None,
                 sparse_lr: Optional[float] = None, init: str = "truncated_normal",
                 layout: Optional[str] = None):
        super().__init__()
        if dim % 4 != 0 or not (4 <= dim <= 128):
            raise ValueError(f"embedding dimension must be a multiple of 4 in [4,128], got {dim}")
        self.rows_list = [int(r) for r in rows]
        self.dim = int(dim)
        self.num_slots = len(self.rows_list)
        self.sparse_lr = sparse_lr           # None: dense .grad via autograd; float: fused sparse SGD
        dev = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        offs = [0]
        for r in self.rows_list:
            offs.append(offs[-1] + r)
        self.total_rows = offs[-1]
        self.with_linear = bool(with_linear)
        self.layout = layout or ("fused" if (with_linear and self.dim + 1 <= 32) else "split")
        if self.layout not in ("fused", "split"):
            raise ValueError(f"unknown layout {self.layout!r}")
        if self.layout == "fused" and not with_linear:
            raise ValueError("layout='fused' needs with_linear=True")
        if self.layout == "fused" and self.dim + 1 > 32:
            raise ValueError("layout='fused' packs [emb | w] into one 128-B line: needs D <= 28")
        self.row_stride = 32 if self.layout == "fused" else self.dim
        self.lin_stride = self.row_stride if self.layout == "fused" else 1
        self.flags = 1 if self.layout == "fused" else 0      # DR_EMBED_LIN_IN_ROW
        std = init_stddev if init_stddev is not None else 1.0 / math.sqrt(self.dim)
        w = torch.zeros((self.total_rows, self.row_stride), dtype=torch.float32, device=dev)
        if init == "truncated_normal":
            # TF embedding_column default: truncated_normal_initializer(mean=0, stddev=1/sqrt(D))
            gen = None
            if seed is not None:
                gen = torch.Generator(device=dev).manual_seed(seed)
            nn.init.trunc_normal_(w[:, :self.dim], mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)
        elif init not in ("zeros", "empty"):
            raise ValueError(f"unknown init {init!r}")
        self.weight = nn.Parameter(w)
        self.linear = (nn.Parameter(torch.zeros((self.total_rows,), dtype=torch.float32, device=dev))
                       if (with_linear and self.layout == "split") else None)
        self.bias = nn.Parameter(torch.zeros((1,), dtype=torch.float32, device=dev)) if with_linear else None
        self.register_buffer("_offsets", torch.tensor(offs[:-1], dtype=torch.int64, device=dev), persistent=False)
        self.register_buffer("_rows", torch.tensor(self.rows_list, dtype=torch.int64, device=dev), persistent=False)
        self._ptr_cache = {}
        # optimizers.RowSparseAdam, once one trains the tables: the forward ops replay the rows' pending steps first,
        # and the arena is flushed before state_dict() reads it
        self.row_optimizer = None
        self.register_state_dict_pre_hook(_flush_row_optimizer)

    # device pointer arrays for the kernel (computed on device: no host sync)
    def pointers(self, weight: torch.Tensor, linear: Optional[torch.Tensor], cache: bool = True):
        key = (weight.data_ptr(), None if linear is None else linear.data_ptr())
        if cache and key in self._ptr_cache:
            return self._ptr_cache[key]
        offs = self._offsets.to(weight.device)
        tp = offs * (self.row_stride * 4) + weight.data_ptr()
        if self.layout == "fused":
            lp = tp + self.dim * 4
        else:
            lp = (offs * 4 + linear.data_ptr()) if linear is not None else tp
        out = (tp, lp, self._rows.to(weight.device))
        if cache:
            self._ptr_cache = {key: out}
        return out

    # ---- logical views (independent of the physical layout) --------------------------------
    def emb_view(self, t: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[total_rows, D] view of the embedding vectors of `t` (default: the parameters)."""
        t = self.weight if t is None else t
        return t[:, :self.dim]

    def lin_view(self, t: Optional[torch.Tensor] = None, lin: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[total_rows] view of the first-order weights."""
        if self.layout == "fused":
            return (self.weight if t is None else t)[:, self.dim]
        return self.linear if lin is None else lin

    def grads(self):
        """(d/d embeddings [R,D], d/d first-order [R], d/d bias [1]) after a dense-mode backward."""
        gw = self.weight.grad
        gl = gw[:, self.dim] if self.layout == "fused" else (None if self.linear is None else self.linear.grad)
        return gw[:, :self.dim], gl, (None if self.bias is None else self.bias.grad)

    def table(self, s: int) -> torch.Tensor:
        o = int(self._offsets[s])
        return self.emb_view()[o:o + self.rows_list[s]]

    def linear_of(self, s: int) -> torch.Tensor:
        o = int(self._offsets[s])
        return self.lin_view()[o:o + self.rows_list[s]]

    def forward(self, ids: torch.Tensor, want_logit: bool = True, bags: Optional[dict] = None,
                second_order: bool = True):
        """ids [B, S] int64/int32 -> (stack [B,S,D], logit [B] = bias + linear + FM 2nd order).

        second_order=False: logit = bias + linear only (xDeepFM's linear unit), from the same fused kernel.

        bags: {slot: (flat_ids [nnz], row_splits [B+1])} for multi-valued slots (mean-combined embedding,
        summed first-order weights); the matching columns of `ids` are ignored.  A collection without first-order
        weights serves bags with want_logit=False.
        """
        if ids.dim() != 2 or ids.shape[1] != self.num_slots:
            raise ValueError(f"ids must be [B, {self.num_slots}], got {tuple(ids.shape)}")
        if bags:
            if not second_order:
                raise ValueError("second_order=False is not served with multi-valued slots (bags)")
            if want_logit and not self.with_linear:
                raise ValueError("a logit over multi-valued slots (bags) needs a collection with the first-order term "
                                 "(with_linear=True)")
            bad = [s for s in bags if not (0 <= s < self.num_slots)]
            if bad:
                raise ValueError(f"bags: slot indices {bad} outside [0, {self.num_slots})")
        stack, logit = ops.EmbedFM.apply(ids, self.weight, self.linear, self.bias, self, want_logit,
                                         bool(second_order), bags)
        return stack, (logit if want_logit else None)


class LinearTable(nn.Module):
    """The variables of tf.feature_column.linear_model over S indicator / crossed columns (estimator
    wide_and_deep.py:31-33): one scalar weight per row of each column and one bias, with the two slots
    tf.train.FtrlOptimizer keeps for them.

    state [total_rows + 1, 4] fp32: row r = {w, z, n, g} -- weight, FTRL linear slot, FTRL accumulator and the
    gradient of the current batch -- in ONE 16-byte record, so a lookup, its gradient atomic and the update of a row
    touch one 32-B sector (csrc/wide.cu).  Record total_rows is the bias.  Column s owns rows [off_s, off_s + rows_s).
    w, z and g start at zero, as linear_model's zeros initializer and FTRL's linear slot do; n starts at
    initial_accumulator_value, the FTRL optimizer's setting, which ops.FtrlOptimizer checks it matches.  The slots
    live in the table, so they are saved with it and a new optimizer continues from them.
    """

    def __init__(self, rows: Sequence[int], device=None, initial_accumulator_value: float = 0.1):
        super().__init__()
        self.rows_list = [int(r) for r in rows]
        if not self.rows_list or any(r < 1 for r in self.rows_list):
            raise ValueError(f"LinearTable needs at least one column and rows >= 1 per column, got {self.rows_list}")
        self.num_slots = len(self.rows_list)
        dev = torch.device(device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu"))
        offs = [0]
        for r in self.rows_list:
            offs.append(offs[-1] + r)
        self.total_rows = offs[-1]
        # a Parameter so that autograd runs the backward that accumulates g in place; its .grad stays None
        if not initial_accumulator_value >= 0.0:
            raise ValueError(f"initial_accumulator_value {initial_accumulator_value} needs to be positive or zero")
        self.initial_accumulator_value = float(initial_accumulator_value)
        state = torch.zeros((self.total_rows + 1, 4), dtype=torch.float32, device=dev)
        state[:, 2] = self.initial_accumulator_value
        self.state = nn.Parameter(state)
        self.register_buffer("_offsets", torch.tensor(offs[:-1], dtype=torch.int64, device=dev), persistent=False)
        self.register_buffer("_rows", torch.tensor(self.rows_list, dtype=torch.int64, device=dev), persistent=False)
        self.lookups = None        # (ids, bags) of the last forward: the rows the optimizer updates

    @property
    def weights(self) -> torch.Tensor:
        """[total_rows] view of the weights (column s at [off_s, off_s + rows_s))."""
        return self.state.detach()[:self.total_rows, 0]

    @property
    def bias(self) -> torch.Tensor:
        return self.state.detach()[self.total_rows:, 0]

    def weights_of(self, s: int) -> torch.Tensor:
        o = int(self._offsets[s])
        return self.weights[o:o + self.rows_list[s]]

    def forward(self, ids: torch.Tensor, bags: Optional[dict] = None) -> torch.Tensor:
        """ids [B, S] int64 (columns of multi-valued slots ignored), bags {slot: (flat ids, row_splits)} -> logit [B]."""
        if ids.dim() != 2 or ids.shape[1] != self.num_slots:
            raise ValueError(f"ids must be [B, {self.num_slots}], got {tuple(ids.shape)}")
        self.lookups = (ids, bags)
        return ops.WideLinearFn.apply(self.state, self, ids, bags)
