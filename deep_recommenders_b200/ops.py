"""torch.autograd.Function wrappers over the C-ABI (include/deeprec_b200.h).

PyTorch is plumbing here: it owns device memory and streams and gives the layers an autograd
graph.  All arithmetic happens in libdeeprec_b200.so.  Every function raises if its inputs are
not CUDA fp32 tensors -- there is no CPU or eager-PyTorch fallback on this path.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import check

ACT_CODES = {None: 0, "linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3}
_DR_EMBED_NO_FM = 2


def act_code(act) -> int:
    if callable(act):
        act = getattr(act, "__name__", str(act))
    if act not in ACT_CODES:
        raise ValueError(f"unsupported activation {act!r}; supported: {sorted(k for k in ACT_CODES if k)}")
    return ACT_CODES[act]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise _lib.DeepRecError(f"{name} is on {t.device}: the hot path runs on CUDA only (no CPU fallback)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: expected float32, got {t.dtype}")
    return t.contiguous()


def _ids(t: torch.Tensor, name: str = "ids") -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.DeepRecError(f"{name} is on {t.device}: the hot path runs on CUDA only (no CPU fallback)")
    if t.dtype not in (torch.int64, torch.int32):
        raise TypeError(f"{name}: expected int64 or int32 ids, got {t.dtype}")
    return t.contiguous()


# ------------------------------------------------------------------------------------------
# Rows E + L + F: fused multi-slot gather + linear + FM
# ------------------------------------------------------------------------------------------
class EmbedFM(torch.autograd.Function):
    """stack, logit = EmbedFM(ids, weight_arena, linear_arena, bias, meta, want_logit, second_order).

    `meta` carries the device pointer arrays (table_ptrs, lin_ptrs, rows) of the collection.
    Backward either scatter-adds into dense .grad buffers (meta.sparse_lr is None) or applies
    the fused sparse SGD update in place (meta.sparse_lr = lr) and returns no table gradient.
    second_order=False (DR_EMBED_NO_FM): the logit is bias + first order only (xDeepFM's linear unit).
    """

    @staticmethod
    def forward(ctx, ids, weight, linear, bias, meta, want_logit: bool, second_order: bool = True):
        lib = _lib.load()
        ids = _ids(ids)
        B, S = ids.shape
        D = meta.dim
        stack = torch.empty((B, S, D), device=weight.device, dtype=torch.float32)
        sum_e = torch.empty((B, D), device=weight.device, dtype=torch.float32) if want_logit else None
        logit = torch.empty((B,), device=weight.device, dtype=torch.float32) if want_logit else None
        tp, lp, rows = meta.pointers(weight, linear)
        has_lin = want_logit and meta.with_linear
        no_fm = 0 if (second_order or not want_logit) else _DR_EMBED_NO_FM
        check(lib.dr_embed_fm_fwd(tp.data_ptr(), lp.data_ptr() if has_lin else None,
                                  rows.data_ptr(), ids.data_ptr(), ids.element_size(),
                                  _ptr(bias) if want_logit else None, B, S, D, meta.row_stride, meta.lin_stride,
                                  (meta.flags if has_lin else 0) | no_fm, stack.data_ptr(), _ptr(sum_e), _ptr(logit),
                                  _stream()), "dr_embed_fm_fwd")
        ctx.meta = meta
        ctx.no_fm = no_fm
        ctx.want_logit = want_logit
        ctx.has_lin = has_lin
        ctx.has_bias = bias is not None
        ctx.save_for_backward(ids, stack, sum_e, weight, linear, bias)
        if want_logit:
            return stack, logit
        dummy = stack.new_zeros((0,))
        ctx.mark_non_differentiable(dummy)
        return stack, dummy

    @staticmethod
    def backward(ctx, g_stack, g_logit):
        lib = _lib.load()
        ids, stack, sum_e, weight, linear, bias = ctx.saved_tensors
        meta = ctx.meta
        B, S = ids.shape
        D = meta.dim
        want_logit = ctx.want_logit
        g_stack = None if g_stack is None else _f32(g_stack, "g_stack")
        g_logit = _f32(g_logit, "g_logit") if (want_logit and g_logit is not None) else None
        if g_stack is None and g_logit is None:
            return None, None, None, None, None, None, None
        fused = meta.sparse_lr is not None
        if fused:
            gw, gl, gb = weight, linear, bias
            scale = -float(meta.sparse_lr)
            tp, lp, rows = meta.pointers(weight, linear)
        else:
            gw = torch.zeros_like(weight)
            gl = torch.zeros_like(linear) if (linear is not None and g_logit is not None) else None
            gb = torch.zeros_like(bias) if (bias is not None and g_logit is not None) else None
            scale = 1.0
            tp, lp, rows = meta.pointers(gw, gl, cache=False)
        lin_grad = ctx.has_lin and g_logit is not None
        with torch.no_grad():
            check(lib.dr_embed_fm_bwd(ids.data_ptr(), ids.element_size(), rows.data_ptr(),
                                      stack.data_ptr(), _ptr(sum_e), _ptr(g_logit), _ptr(g_stack),
                                      B, S, D, meta.row_stride, meta.lin_stride,
                                      (meta.flags if lin_grad else 0) | (ctx.no_fm if g_logit is not None else 0),
                                      tp.data_ptr(),
                                      lp.data_ptr() if lin_grad else None,
                                      _ptr(gb) if g_logit is not None else None, scale, _stream()),
                  "dr_embed_fm_bwd")
        if fused:
            return None, None, None, None, None, None, None
        return None, gw, gl, gb, None, None, None


class Gather(torch.autograd.Function):
    """rows = table[ids] for one table (two-tower user / item tower); OOV id -> zero row."""

    @staticmethod
    def forward(ctx, table, ids, sparse_lr):
        lib = _lib.load()
        table = _f32(table, "table")
        ids = _ids(ids)
        n = ids.numel()
        D = table.shape[1]
        out = torch.empty((n, D), device=table.device, dtype=torch.float32)
        check(lib.dr_gather_fwd(table.data_ptr(), table.shape[0], ids.data_ptr(), ids.element_size(), n, D,
                                out.data_ptr(), _stream()), "dr_gather_fwd")
        ctx.save_for_backward(table, ids)
        ctx.sparse_lr = sparse_lr
        return out.view(*ids.shape, D)

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        table, ids = ctx.saved_tensors
        g = _f32(g, "g").view(-1, table.shape[1])
        fused = ctx.sparse_lr is not None
        tgt = table if fused else torch.zeros_like(table)
        with torch.no_grad():
            check(lib.dr_scatter_add(tgt.data_ptr(), table.shape[0], ids.data_ptr(), ids.element_size(),
                                     ids.numel(), table.shape[1], g.data_ptr(),
                                     -float(ctx.sparse_lr) if fused else 1.0, _stream()), "dr_scatter_add")
        return (None if fused else tgt), None, None


# ------------------------------------------------------------------------------------------
# Row F standalone
# ------------------------------------------------------------------------------------------
class FMInteraction(torch.autograd.Function):
    """0.5 * sum_d((sum_s x)^2 - sum_s x^2), keepdims -> [B, 1]."""

    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        x = _f32(x, "x")
        if x.dim() != 3:
            raise ValueError("The rank of `x` should be 3. Got rank = {}.".format(x.dim()))
        B, S, D = x.shape
        out = torch.empty((B,), device=x.device, dtype=torch.float32)
        check(lib.dr_fm_fwd(x.data_ptr(), B, S, D, out.data_ptr(), _stream()), "dr_fm_fwd")
        ctx.save_for_backward(x)
        return out.view(B, 1)

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        (x,) = ctx.saved_tensors
        B, S, D = x.shape
        g = _f32(g, "g").reshape(B)
        gx = torch.empty_like(x)
        check(lib.dr_fm_bwd(x.data_ptr(), g.data_ptr(), B, S, D, gx.data_ptr(), _stream()), "dr_fm_bwd")
        return gx


# ------------------------------------------------------------------------------------------
# Row D: Dense
# ------------------------------------------------------------------------------------------
class DenseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act: int):
        lib = _lib.load()
        x = _f32(x, "x")
        w = _f32(w, "kernel")
        b = None if b is None else _f32(b, "bias")
        lead = x.shape[:-1]
        K = x.shape[-1]
        x2 = x.reshape(-1, K)
        M = x2.shape[0]
        if w.shape[0] != K:
            raise ValueError(f"Dense: input dim {K} does not match kernel {tuple(w.shape)}")
        N = w.shape[1]
        _lib.ensure_gemm_workspace(M, K, N, x.device)
        y = torch.empty((M, N), device=x.device, dtype=torch.float32)
        check(lib.dr_dense_fwd(x2.data_ptr(), w.data_ptr(), _ptr(b), M, K, N, act, y.data_ptr(), _stream()),
              "dr_dense_fwd")
        ctx.act = act
        ctx.has_bias = b is not None
        ctx.save_for_backward(x2, w, y)
        ctx.lead = lead
        return y.view(*lead, N)

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x2, w, y = ctx.saved_tensors
        M, K = x2.shape
        N = w.shape[1]
        gy = _f32(gy, "gy").reshape(M, N)
        need_x = ctx.needs_input_grad[0]
        gz_ws = torch.empty_like(gy) if ctx.act != 0 else None
        gx = torch.empty((M, K), device=gy.device, dtype=torch.float32) if need_x else None
        gw = torch.empty_like(w)
        gb = torch.empty((N,), device=gy.device, dtype=torch.float32) if ctx.has_bias else None
        check(lib.dr_dense_bwd(x2.data_ptr(), w.data_ptr(), y.data_ptr(), gy.data_ptr(), M, K, N, ctx.act,
                               _ptr(gz_ws), _ptr(gx), gw.data_ptr(), _ptr(gb), _stream()), "dr_dense_bwd")
        return (gx.view(*ctx.lead, K) if need_x else None), gw, gb, None


class GroupedDenseFn(torch.autograd.Function):
    """y [M, G*N] = GroupedDenseFn(x [M, G*K], w [G, K, N], b [G, N] or None, act): G Dense layers of one shape on
    column blocks (dr_dense_grouped_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x, w, b, act: int):
        lib = _lib.load()
        x = _f32(x, "x")
        w = _f32(w, "kernel")
        b = None if b is None else _f32(b, "bias")
        if w.dim() != 3 or x.dim() != 2 or x.shape[1] != w.shape[0] * w.shape[1] or (
                b is not None and tuple(b.shape) != (w.shape[0], w.shape[2])):
            raise ValueError(f"grouped Dense: x [M, G*K], kernel [G, K, N], bias [G, N] expected, got {tuple(x.shape)}, "
                             f"{tuple(w.shape)}, {None if b is None else tuple(b.shape)}")
        G, K, N = w.shape
        M = x.shape[0]
        _lib.ensure_gemm_workspace(M, G * K, G * N, x.device)
        y = torch.empty((M, G * N), device=x.device, dtype=torch.float32)
        check(lib.dr_dense_grouped_fwd(x.data_ptr(), w.data_ptr(), _ptr(b), M, G, K, N, act, y.data_ptr(), _stream()),
              "dr_dense_grouped_fwd")
        ctx.act = act
        ctx.has_bias = b is not None
        ctx.save_for_backward(x, w, y)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x, w, y = ctx.saved_tensors
        G, K, N = w.shape
        M = x.shape[0]
        gy = _f32(gy, "gy")
        gz_ws = torch.empty_like(gy) if ctx.act != 0 else None
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = torch.empty_like(w)
        gb = torch.empty((G, N), device=gy.device, dtype=torch.float32) if ctx.has_bias else None
        check(lib.dr_dense_grouped_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), gy.data_ptr(), M, G, K, N, ctx.act,
                                       _ptr(gz_ws), _ptr(gx), gw.data_ptr(), _ptr(gb), _stream()),
              "dr_dense_grouped_bwd")
        return gx, gw, gb, None


class MoEMixFn(torch.autograd.Function):
    """out [B, T*H] = MoEMixFn(experts [B, E*H], logits [B, T*E], T): per task t, softmax(logits[:, t*E:(t+1)*E]) mixes
    the E expert blocks (dr_moe_mix_fwd / _bwd).  Saves the gates."""

    @staticmethod
    def forward(ctx, experts, logits, T: int):
        lib = _lib.load()
        experts, logits = _f32(experts, "experts"), _f32(logits, "logits")
        T = int(T)
        if experts.dim() != 2 or logits.dim() != 2 or logits.shape[0] != experts.shape[0] or T < 1 or \
                logits.shape[1] < T or logits.shape[1] % T or experts.shape[1] % (logits.shape[1] // T) or \
                experts.shape[1] == 0:
            raise ValueError(f"mixture of experts: experts [B, E*H] and logits [B, T*E] with T = {T} expected, got "
                             f"{tuple(experts.shape)} and {tuple(logits.shape)}")
        B = experts.shape[0]
        E = logits.shape[1] // T
        H = experts.shape[1] // E
        gates = torch.empty_like(logits)
        out = torch.empty((B, T * H), device=experts.device, dtype=torch.float32)
        check(lib.dr_moe_mix_fwd(experts.data_ptr(), logits.data_ptr(), B, E, T, H, gates.data_ptr(), out.data_ptr(),
                                 _stream()), "dr_moe_mix_fwd")
        ctx.shape = (E, T, H)
        ctx.save_for_backward(experts, gates)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        experts, gates = ctx.saved_tensors
        E, T, H = ctx.shape
        g = _f32(g, "g_out")
        g_experts, g_logits = torch.empty_like(experts), torch.empty_like(gates)
        check(lib.dr_moe_mix_bwd(experts.data_ptr(), gates.data_ptr(), g.data_ptr(), experts.shape[0], E, T, H,
                                 g_experts.data_ptr(), g_logits.data_ptr(), _stream()), "dr_moe_mix_bwd")
        return g_experts, g_logits, None


# ------------------------------------------------------------------------------------------
# GCN: CSR sparse x dense product (dr_spmm_csr_fwd)
# ------------------------------------------------------------------------------------------
ACT_SOFTMAX = 4          # DR_ACT_SOFTMAX: served by the SpMM epilogue only
SPMM_SOFTMAX_MAX_F = 1024


class CSRAdjacency:
    """A constant sparse matrix A [n_rows, n_cols] prepared once on the device: the int32 CSR of A and of A^T.

    Build it from a scipy sparse matrix (anything with ``tocsr()``), a torch sparse COO or CSR tensor, or CSR arrays.
    The arrays are validated once on the host (``ValueError`` for a malformed ``indptr``, an index out of range or
    non-float values).  Entries keep their stored order: duplicates are summed where they stand, and a COO tensor is
    grouped by row without coalescing.  A^T is a stable sort of the entries by column, so each transposed row lists
    its entries in ascending original row, and the backward sums in a fixed order.  The values are an input, not a
    parameter: no gradient reaches them (TensorFlow would give a SparseTensor's values one)."""

    def __init__(self, indptr, indices, values, shape, device=None):
        import numpy as np
        indptr = np.asarray(indptr)
        indices = np.asarray(indices)
        values = np.asarray(values)
        n_rows, n_cols = int(shape[0]), int(shape[1])
        if n_rows < 0 or n_cols < 0 or indptr.ndim != 1 or indptr.shape[0] != n_rows + 1:
            raise ValueError(f"CSR: indptr must have n_rows + 1 = {n_rows + 1} entries, got shape {indptr.shape}")
        if indices.ndim != 1 or values.shape != indices.shape:
            raise ValueError(f"CSR: indices {indices.shape} and values {values.shape} must be 1-D of one length")
        if not (np.issubdtype(indptr.dtype, np.integer) and np.issubdtype(indices.dtype, np.integer)):
            raise ValueError("CSR: indptr and indices must be integers")
        if not np.issubdtype(values.dtype, np.floating):
            raise ValueError(f"CSR: values must be floating point, got {values.dtype}")
        nnz = indices.shape[0]
        if max(n_rows, n_cols, nnz) >= 2 ** 31:
            raise ValueError(f"CSR: n_rows, n_cols and nnz must stay below 2^31, got {n_rows}, {n_cols}, {nnz}")
        if indptr[0] != 0 or indptr[-1] != nnz or (n_rows and np.any(np.diff(indptr) < 0)):
            raise ValueError(f"CSR: indptr must start at 0, never decrease and end at nnz = {nnz}")
        if nnz and (indices.min() < 0 or indices.max() >= n_cols):
            raise ValueError(f"CSR: column index out of range [0, {n_cols})")
        dev = torch.device(device if device is not None else "cuda")
        self.shape = (n_rows, n_cols)
        self.nnz = nnz
        self.indptr = torch.from_numpy(indptr.astype(np.int32)).to(dev)
        self.indices = torch.from_numpy(indices.astype(np.int32)).to(dev)
        self.values = torch.from_numpy(values.astype(np.float32)).to(dev)
        rows = torch.repeat_interleave(torch.arange(n_rows, device=dev, dtype=torch.int32),
                                       (self.indptr[1:] - self.indptr[:-1]).long())
        order = torch.sort(self.indices, stable=True).indices
        counts = torch.bincount(self.indices.long(), minlength=n_cols)
        self.t_indptr = torch.zeros(n_cols + 1, dtype=torch.int32, device=dev)
        self.t_indptr[1:] = torch.cumsum(counts, 0).to(torch.int32)
        self.t_indices = rows[order].contiguous()
        self.t_values = self.values[order].contiguous()

    @classmethod
    def from_any(cls, adj, device=None) -> "CSRAdjacency":
        """A prepared adjacency from a scipy sparse matrix (duck-typed through ``tocsr()``) or a torch sparse tensor."""
        if isinstance(adj, CSRAdjacency):
            return adj
        if isinstance(adj, torch.Tensor):
            if adj.layout == torch.sparse_csr:
                return cls(adj.crow_indices().cpu().numpy(), adj.col_indices().cpu().numpy(),
                           adj.values().detach().cpu().numpy(), adj.shape, device or adj.device)
            if adj.layout == torch.sparse_coo:
                idx = adj._indices().cpu()
                vals = adj._values().detach().cpu()
                order = torch.sort(idx[0], stable=True).indices
                counts = torch.bincount(idx[0], minlength=adj.shape[0])
                indptr = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(counts, 0)])
                return cls(indptr.numpy(), idx[1][order].numpy(), vals[order].numpy(), adj.shape,
                           device or (adj.device if adj.is_cuda else None))
            raise ValueError(f"CSRAdjacency: a torch tensor must be sparse COO or CSR, got layout {adj.layout}")
        if hasattr(adj, "tocsr"):
            csr = adj.tocsr()
            return cls(csr.indptr, csr.indices, csr.data, csr.shape, device)
        raise TypeError(f"CSRAdjacency: expected a scipy sparse matrix or a torch sparse tensor, got {type(adj).__name__}")

    def spmm(self, x, bias=None, residual=None, act: int = 0, transpose: bool = False):
        """act(A @ x + bias) (+ residual), or A^T @ x with transpose=True, as raw tensors (no autograd)."""
        lib = _lib.load()
        n_rows, n_cols = self.shape[::-1] if transpose else self.shape
        indptr, indices, values = ((self.t_indptr, self.t_indices, self.t_values) if transpose
                                   else (self.indptr, self.indices, self.values))
        if x.dim() != 2 or x.shape[0] != n_cols or x.shape[1] < 1:
            raise ValueError(f"SpMM: x must be [{n_cols}, F], got {tuple(x.shape)}")
        F = x.shape[1]
        if bias is not None and tuple(bias.shape) != (F,):
            raise ValueError(f"SpMM: bias must be [{F}], got {tuple(bias.shape)}")
        if residual is not None and tuple(residual.shape) != (n_rows, F):
            raise ValueError(f"SpMM: residual must be [{n_rows}, {F}], got {tuple(residual.shape)}")
        y = torch.empty((n_rows, F), device=x.device, dtype=torch.float32)
        out = torch.empty_like(y) if residual is not None else None
        check(lib.dr_spmm_csr_fwd(indptr.data_ptr(), indices.data_ptr(), values.data_ptr(), n_rows, n_cols,
                                  self.nnz, x.data_ptr(), F, _ptr(bias), _ptr(residual), act, y.data_ptr(),
                                  _ptr(out), _stream()), "dr_spmm_csr_fwd")
        return y, out


class SpMMFn(torch.autograd.Function):
    """SpMMFn(x [n_cols, F], bias [F] or None, residual [n_rows, F] or None, adj: CSRAdjacency, act) =
    act(A @ x + bias) (+ residual): the plain product with bias None, residual None and act 0, else the fused epilogue
    (dr_spmm_csr_fwd).  act is a DR_ACT_* code or ACT_SOFTMAX.  Backward: the activation gradient from the saved
    output (dr_act_bwd_colsum, after dr_softmax_rows_bwd for the softmax), then gx = A^T @ gz on the transposed CSR."""

    @staticmethod
    def forward(ctx, x, bias, residual, adj, act: int):
        x = _f32(x, "x")
        bias = None if bias is None else _f32(bias, "bias")
        residual = None if residual is None else _f32(residual, "residual")
        y, out = adj.spmm(x, bias, residual, act)
        ctx.adj, ctx.act = adj, act
        ctx.has_bias, ctx.has_res = bias is not None, residual is not None
        ctx.save_for_backward(y)
        return out if residual is not None else y

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        (y,) = ctx.saved_tensors
        g = _f32(g, "g")
        M, F = y.shape
        act = ctx.act
        gb = torch.empty((F,), device=g.device, dtype=torch.float32) if ctx.has_bias else None
        gz = g
        if act == ACT_SOFTMAX:
            gz = torch.empty_like(y)
            check(lib.dr_softmax_rows_bwd(y.data_ptr(), g.data_ptr(), M, F, gz.data_ptr(), _stream()),
                  "dr_softmax_rows_bwd")
            act = 0
        elif act != 0:
            gz = torch.empty_like(y)
        if act != 0 or gb is not None:
            check(lib.dr_act_bwd_colsum(_ptr(y) if act else None, gz.data_ptr() if act == 0 else g.data_ptr(), M, F,
                                        act, gz.data_ptr() if act else None, _ptr(gb), _stream()),
                  "dr_act_bwd_colsum")
        gx = ctx.adj.spmm(gz, transpose=True)[0] if ctx.needs_input_grad[0] else None
        return gx, gb, (g if ctx.has_res else None), None, None


# ------------------------------------------------------------------------------------------
# Row X: Cross
# ------------------------------------------------------------------------------------------
class CrossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, x, w, uk, vk, b, alpha: float, same: bool):
        lib = _lib.load()
        x0 = _f32(x0, "x0")
        x = x0 if same else _f32(x, "x")
        d = x0.shape[-1]
        lead = x0.shape[:-1]
        x0_2 = x0.reshape(-1, d)
        x_2 = x.reshape(-1, d)
        B = x0_2.shape[0]
        r = 0 if w is not None else uk.shape[1]
        _lib.ensure_gemm_workspace(B, d, d, x0.device)
        y = torch.empty((B, d), device=x0.device, dtype=torch.float32)
        u = torch.empty((B, d), device=x0.device, dtype=torch.float32)
        xu = torch.empty((B, r), device=x0.device, dtype=torch.float32) if r else None
        check(lib.dr_cross_fwd(x0_2.data_ptr(), x_2.data_ptr(), _ptr(w), _ptr(uk), _ptr(vk), _ptr(b),
                               float(alpha), B, d, r, _ptr(xu), u.data_ptr(), y.data_ptr(), _stream()),
              "dr_cross_fwd")
        ctx.alpha = float(alpha)
        ctx.same = same
        ctx.r = r
        ctx.lead = lead
        ctx.save_for_backward(x0_2, x_2, w, uk, vk, b, u, xu)
        return y.view(*lead, d)

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        x0, x, w, uk, vk, b, u, xu = ctx.saved_tensors
        B, d = x0.shape
        r = ctx.r
        g = _f32(g, "g").reshape(B, d)
        dev = g.device
        h = torch.empty((B, d), device=dev, dtype=torch.float32)
        t = torch.empty((B, r), device=dev, dtype=torch.float32) if r else None
        gx0 = torch.empty((B, d), device=dev, dtype=torch.float32)
        gx = torch.empty((B, d), device=dev, dtype=torch.float32)
        gw = torch.empty_like(w) if w is not None else None
        guk = torch.empty_like(uk) if uk is not None else None
        gvk = torch.empty_like(vk) if vk is not None else None
        gb = torch.empty_like(b) if b is not None else None
        check(lib.dr_cross_bwd(x0.data_ptr(), x.data_ptr(), _ptr(w), _ptr(uk), _ptr(vk), ctx.alpha,
                               u.data_ptr(), _ptr(xu), g.data_ptr(), B, d, r, h.data_ptr(), _ptr(t),
                               gx0.data_ptr(), gx.data_ptr(), _ptr(gw), _ptr(guk), _ptr(gvk), _ptr(gb),
                               _stream()), "dr_cross_bwd")
        if ctx.same:
            gx0 = gx0 + gx
            gx = None
        else:
            gx = gx.view(*ctx.lead, d)
        return gx0.view(*ctx.lead, d), gx, gw, guk, gvk, gb, None, None


# ------------------------------------------------------------------------------------------
# Row C: CIN (xDeepFM)
# ------------------------------------------------------------------------------------------
class CINFn(torch.autograd.Function):
    """y [B, H, D], pooled [B, H] = CINFn(x0 [B, m, D], x [B, h, D], kernel [1, m*h, H], bias, act, same, pool).

    `same` is the first layer's call on (x0, x0): one input gradient.  With `pool` False the second output is an empty
    tensor without gradient."""

    @staticmethod
    def forward(ctx, x0, x, w, b, act: int, same: bool, pool: bool):
        lib = _lib.load()
        x0 = _f32(x0, "x0")
        x = x0 if same else _f32(x, "x")
        w = _f32(w, "kernel")
        b = None if b is None else _f32(b, "bias")
        B, m, D = x0.shape
        h = x.shape[1]
        H = w.shape[-1]
        if x.shape[0] != B or x.shape[2] != D or w.numel() != m * h * H:
            raise ValueError(f"CIN: x0 {tuple(x0.shape)}, x {tuple(x.shape)} and kernel {tuple(w.shape)} do not match")
        y = torch.empty((B, H, D), device=x0.device, dtype=torch.float32)
        pooled = torch.empty((B, H) if pool else (0,), device=x0.device, dtype=torch.float32)
        check(lib.dr_cin_fwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), _ptr(b), B, m, h, D, H, act, y.data_ptr(),
                             pooled.data_ptr() if pool else None, _stream()), "dr_cin_fwd")
        ctx.act = act
        ctx.same = same
        ctx.set_materialize_grads(False)      # an unused output reaches backward as None, not as zeros to read
        ctx.save_for_backward(x0, x, w, b, y)
        if not pool:
            ctx.mark_non_differentiable(pooled)
        return y, pooled

    @staticmethod
    def backward(ctx, gy, gpool):
        lib = _lib.load()
        x0, x, w, b, y = ctx.saved_tensors
        B, m, D = x0.shape
        h = x.shape[1]
        H = y.shape[1]
        gy = None if gy is None else _f32(gy, "gy")
        gpool = None if (gpool is None or gpool.numel() == 0) else _f32(gpool, "gpool")
        if gy is None and gpool is None:
            return None, None, None, None, None, None, None
        g_ws = torch.empty_like(y)
        gx0 = torch.empty_like(x0)
        gx = None if ctx.same else torch.empty_like(x)
        gw = torch.empty_like(w)
        gb = None if b is None else torch.empty_like(b)
        check(lib.dr_cin_bwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), y.data_ptr(), _ptr(gy), _ptr(gpool),
                             B, m, h, D, H, ctx.act, int(ctx.same), g_ws.data_ptr(), gx0.data_ptr(), _ptr(gx),
                             gw.data_ptr(), _ptr(gb), _stream()), "dr_cin_bwd")
        return gx0, gx, gw, gb, None, None, None


# ------------------------------------------------------------------------------------------
# Row A: DIN's activation unit (target attention + pooling) and Dice
# ------------------------------------------------------------------------------------------
INTERACT_CODES = {None: 0, "none": 0, "subtract": 1, "multiply": 2}


class DINAttentionFn(torch.autograd.Function):
    """pooled [B, D], score [B, T] = DINAttentionFn(keys [B, T, D], query [B, D], W1 [(2|3)D, U], b1, w2 [U, 1] or
    [U], b2, interact, act, pool): score = act([k | q | f(k, q)] W1 + b1) w2 + b2, pooled = sum_t score * k.

    With `pool` False the first output is an empty tensor without gradient.  An unused output reaches the backward as
    None, not as zeros to read."""

    @staticmethod
    def forward(ctx, keys, query, w1, b1, w2, b2, interact: int, act: int, pool: bool):
        lib = _lib.load()
        keys = _f32(keys, "keys")
        query = _f32(query, "query")
        w1 = _f32(w1, "W1")
        w2 = _f32(w2, "w2")
        b1 = None if b1 is None else _f32(b1, "b1")
        b2 = None if b2 is None else _f32(b2, "b2")
        if keys.dim() != 3 or query.dim() != 2:
            raise ValueError(f"DIN attention: keys must be [B, T, D] and query [B, D], got {tuple(keys.shape)} "
                             f"and {tuple(query.shape)}")
        B, T, D = keys.shape
        U = w1.shape[-1]
        blocks = 3 if interact else 2
        if query.shape != (B, D) or w1.shape != (blocks * D, U) or w2.numel() != U:
            raise ValueError(f"DIN attention: keys {tuple(keys.shape)}, query {tuple(query.shape)}, W1 "
                             f"{tuple(w1.shape)} and w2 {tuple(w2.shape)} do not match")
        score = torch.empty((B, T), device=keys.device, dtype=torch.float32)
        pooled = torch.empty((B, D) if pool else (0,), device=keys.device, dtype=torch.float32)
        check(lib.dr_din_attn_fwd(keys.data_ptr(), query.data_ptr(), w1.data_ptr(), _ptr(b1), w2.data_ptr(), _ptr(b2),
                                  B, T, D, U, interact, act, score.data_ptr(), pooled.data_ptr() if pool else None,
                                  _stream()), "dr_din_attn_fwd")
        ctx.interact, ctx.act = interact, act
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(keys, query, w1, b1, w2, b2)
        if not pool:
            ctx.mark_non_differentiable(pooled)
        return pooled, score

    @staticmethod
    def backward(ctx, g_pooled, g_score):
        lib = _lib.load()
        keys, query, w1, b1, w2, b2 = ctx.saved_tensors
        B, T, D = keys.shape
        U = w1.shape[-1]
        g_pooled = None if (g_pooled is None or g_pooled.numel() == 0) else _f32(g_pooled, "g_pooled")
        g_score = None if g_score is None else _f32(g_score, "g_score")
        if g_pooled is None and g_score is None:
            return (None,) * 9
        g_keys = torch.empty_like(keys)
        g_query = torch.empty_like(query)
        gw1 = torch.empty_like(w1)
        gw2 = torch.empty_like(w2)
        gb1 = None if b1 is None else torch.empty_like(b1)
        gb2 = None if b2 is None else torch.empty_like(b2)
        check(lib.dr_din_attn_bwd(keys.data_ptr(), query.data_ptr(), w1.data_ptr(), _ptr(b1), w2.data_ptr(), _ptr(b2),
                                  _ptr(g_pooled), _ptr(g_score), B, T, D, U, ctx.interact, ctx.act,
                                  g_keys.data_ptr(), g_query.data_ptr(), gw1.data_ptr(), _ptr(gb1), gw2.data_ptr(),
                                  _ptr(gb2), _stream()), "dr_din_attn_bwd")
        return g_keys, g_query, gw1, gb1, gw2, gb2, None, None, None


class DiceFn(torch.autograd.Function):
    """y [N, U] = Dice(x [N, U]; alpha [U], epsilon): see dr_dice_fwd."""

    @staticmethod
    def forward(ctx, x, alpha, eps: float):
        lib = _lib.load()
        x = _f32(x, "x")
        alpha = _f32(alpha, "alpha")
        if x.dim() != 2 or alpha.numel() != x.shape[1]:
            raise ValueError(f"Dice: x must be [N, U] with alpha [U], got {tuple(x.shape)} and {tuple(alpha.shape)}")
        N, U = x.shape
        y = torch.empty_like(x)
        check(lib.dr_dice_fwd(x.data_ptr(), alpha.data_ptr(), N, U, float(eps), y.data_ptr(), _stream()),
              "dr_dice_fwd")
        ctx.eps = float(eps)
        ctx.save_for_backward(x, alpha)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x, alpha = ctx.saved_tensors
        N, U = x.shape
        gy = _f32(gy, "gy")
        gx = torch.empty_like(x)
        galpha = torch.empty_like(alpha)
        check(lib.dr_dice_bwd(x.data_ptr(), alpha.data_ptr(), gy.data_ptr(), N, U, ctx.eps, gx.data_ptr(),
                              galpha.data_ptr(), _stream()), "dr_dice_bwd")
        return gx, galpha, None


# ------------------------------------------------------------------------------------------
# Row T: multi-head attention, LayerNorm of a sum, row softmax
# ------------------------------------------------------------------------------------------
class MHAttentionFn(torch.autograd.Function):
    """out [B, Lq, H*dh] = MHAttentionFn(q [B, Lq, H*dh], k, v [B, Lk, H*dh], mask [Bm, Lk] or None, H, causal, rate,
    seed): scaled dot-product attention per head (see dr_mha_attn_fwd).  Saves out and the float64 log-sum-exp; the
    backward regenerates the dropout mask from (seed, rate)."""

    @staticmethod
    def forward(ctx, q, k, v, mask, H: int, causal: bool, rate: float, seed: int):
        lib = _lib.load()
        q, k, v = _f32(q, "queries"), _f32(k, "keys"), _f32(v, "values")
        mask = None if mask is None else _f32(mask, "masks")
        if q.dim() != 3 or k.dim() != 3 or v.shape != k.shape or q.shape[0] != k.shape[0] or q.shape[2] != k.shape[2]:
            raise ValueError(f"attention: queries [B, Lq, H*dh], keys and values [B, Lk, H*dh] expected, got "
                             f"{tuple(q.shape)}, {tuple(k.shape)}, {tuple(v.shape)}")
        B, Lq, HD = q.shape
        Lk = k.shape[1]
        if HD % H:
            raise ValueError(f"attention: width {HD} is not a multiple of {H} heads")
        Bm = 0
        if mask is not None:
            if mask.dim() != 2 or mask.shape[1] != Lk or mask.shape[0] == 0 or (H * B) % mask.shape[0]:
                raise ValueError(f"attention: masks must be [Bm, {Lk}] with Bm dividing {H * B}, got "
                                 f"{tuple(mask.shape)}")
            Bm = mask.shape[0]
        out = torch.empty_like(q)
        lse = torch.empty((H * B, Lq), device=q.device, dtype=torch.float64)
        seed = int(seed) % (1 << 64)
        check(lib.dr_mha_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), _ptr(mask), B, H, Lq, Lk, HD // H, Bm,
                                  int(bool(causal)), float(rate), seed, out.data_ptr(), lse.data_ptr(), _stream()),
              "dr_mha_attn_fwd")
        ctx.meta = (H, bool(causal), float(rate), seed, Bm)
        ctx.save_for_backward(q, k, v, mask, out, lse)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        q, k, v, mask, out, lse = ctx.saved_tensors
        H, causal, rate, seed, Bm = ctx.meta
        B, Lq, HD = q.shape
        Lk = k.shape[1]
        g = _f32(g, "g_out")
        gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        check(lib.dr_mha_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), _ptr(mask), out.data_ptr(), lse.data_ptr(),
                                  g.data_ptr(), B, H, Lq, Lk, HD // H, Bm, int(causal), rate, seed, gq.data_ptr(),
                                  gk.data_ptr(), gv.data_ptr(), _stream()), "dr_mha_attn_bwd")
        return gq, gk, gv, None, None, None, None, None


class AddLayerNormFn(torch.autograd.Function):
    """y [..., C] = gamma * normalize(x + residual) + beta (residual may be None): see dr_add_layernorm_fwd."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps: float):
        lib = _lib.load()
        x = _f32(x, "inputs")
        residual = None if residual is None else _f32(residual, "residual")
        gamma, beta = _f32(gamma, "gamma"), _f32(beta, "beta")
        C = x.shape[-1]
        if (residual is not None and residual.shape != x.shape) or gamma.numel() != C or beta.numel() != C:
            raise ValueError(f"LayerNormalization: inputs {tuple(x.shape)}, residual "
                             f"{None if residual is None else tuple(residual.shape)}, gamma {tuple(gamma.shape)} and "
                             f"beta {tuple(beta.shape)} do not match")
        N = x.numel() // C
        y = torch.empty_like(x)
        check(lib.dr_add_layernorm_fwd(x.data_ptr(), _ptr(residual), gamma.data_ptr(), beta.data_ptr(), N, C,
                                       float(eps), y.data_ptr(), _stream()), "dr_add_layernorm_fwd")
        ctx.eps = float(eps)
        ctx.has_res = residual is not None
        ctx.save_for_backward(x, residual, gamma)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        x, residual, gamma = ctx.saved_tensors
        C = x.shape[-1]
        gy = _f32(gy, "gy")
        gx = torch.empty_like(x)
        ggamma, gbeta = torch.empty_like(gamma), torch.empty_like(gamma)
        check(lib.dr_add_layernorm_bwd(x.data_ptr(), _ptr(residual), gamma.data_ptr(), gy.data_ptr(), x.numel() // C,
                                       C, ctx.eps, gx.data_ptr(), ggamma.data_ptr(), gbeta.data_ptr(), _stream()),
              "dr_add_layernorm_bwd")
        return gx, (gx if ctx.has_res else None), ggamma, gbeta, None


class SoftmaxRowsFn(torch.autograd.Function):
    """softmax over the last axis (dr_softmax_rows_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        x = _f32(x, "inputs")
        V = x.shape[-1]
        y = torch.empty_like(x)
        check(lib.dr_softmax_rows_fwd(x.data_ptr(), x.numel() // V, V, y.data_ptr(), _stream()), "dr_softmax_rows_fwd")
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, gy):
        lib = _lib.load()
        (y,) = ctx.saved_tensors
        V = y.shape[-1]
        gy = _f32(gy, "gy")
        gx = torch.empty_like(y)
        check(lib.dr_softmax_rows_bwd(y.data_ptr(), gy.data_ptr(), y.numel() // V, V, gx.data_ptr(), _stream()),
              "dr_softmax_rows_bwd")
        return gx


class TiedProjectionFn(torch.autograd.Function):
    """logits [M, V] = x [M, d] @ table [V, d]^T without a transposed copy of the table:
    forward dr_scores_fwd(x, table); gx = G @ table (dr_dense_fwd, table as a [V, d] weight);
    gtable = G^T @ x (the weight-gradient half of dr_dense_bwd, act NONE)."""

    @staticmethod
    def forward(ctx, x, table):
        lib = _lib.load()
        x, table = _f32(x, "inputs"), _f32(table, "embeddings")
        if x.dim() != 2 or table.dim() != 2 or x.shape[1] != table.shape[1]:
            raise ValueError(f"tied projection: x [M, d] and table [V, d] expected, got {tuple(x.shape)}, "
                             f"{tuple(table.shape)}")
        M, d = x.shape
        V = table.shape[0]
        _lib.ensure_gemm_workspace(M, d, V, x.device)
        out = torch.empty((M, V), device=x.device, dtype=torch.float32)
        check(lib.dr_scores_fwd(x.data_ptr(), table.data_ptr(), None, None, M, V, d, out.data_ptr(), _stream()),
              "dr_scores_fwd")
        ctx.save_for_backward(x, table)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        x, table = ctx.saved_tensors
        M, d = x.shape
        V = table.shape[0]
        g = _f32(g, "g")
        gx = torch.empty_like(x)
        gt = torch.empty_like(table)
        _lib.ensure_gemm_workspace(M, V, d, x.device)
        check(lib.dr_dense_fwd(g.data_ptr(), table.data_ptr(), None, M, V, d, 0, gx.data_ptr(), _stream()),
              "dr_dense_fwd")
        check(lib.dr_dense_bwd(g.data_ptr(), table.data_ptr(), None, x.data_ptr(), M, V, d, 0, None, None,
                               gt.data_ptr(), None, _stream()), "dr_dense_bwd")
        return gx, gt


# ------------------------------------------------------------------------------------------
# Row R: in-batch softmax
# ------------------------------------------------------------------------------------------
# Retrieval losses with at least this many scores (nq * nc) run the tensor-core form (score blocks materialised in a
# scratch buffer of at most SOFTMAX_TC_WS_BYTES); smaller ones the fused FFMA kernels that never materialise scores.
SOFTMAX_TC_MIN_SCORES = 1 << 22
SOFTMAX_TC_WS_BYTES = 2 << 30


class InBatchSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, c, sample_weight, sampling_prob, cand_ids, inv_tau: float):
        lib = _lib.load()
        q = _f32(q, "query_embeddings")
        c = _f32(c, "candidate_embeddings")
        if q.dim() != 2 or c.dim() != 2 or q.shape[1] != c.shape[1]:
            raise ValueError(f"Retrieval: embeddings must be [nq,D] and [nc,D], got {tuple(q.shape)} {tuple(c.shape)}")
        nq, D = q.shape
        nc = c.shape[0]
        w = None if sample_weight is None else _f32(sample_weight, "sample_weight").reshape(nq)
        p = None if sampling_prob is None else _f32(sampling_prob, "candidate_sampling_probability").reshape(nc)
        ids = None
        if cand_ids is not None:
            ids = cand_ids.to(torch.int64).contiguous().reshape(nc)
        lse = torch.empty((nq,), device=q.device, dtype=torch.float32)
        loss = torch.empty((1,), device=q.device, dtype=torch.float32)
        ws = None
        if nq * nc >= SOFTMAX_TC_MIN_SCORES and D >= 32:
            # tensor-core form: score blocks through the wgmma GEMM, kept in a scratch buffer for the backward
            rows = min(nq, max(128, SOFTMAX_TC_WS_BYTES // (4 * nc) // 128 * 128))
            ws = torch.empty((rows, nc), device=q.device, dtype=torch.float32)
            check(lib.dr_inbatch_softmax_fwd_ws(q.data_ptr(), c.data_ptr(), _ptr(w), _ptr(p), _ptr(ids), float(inv_tau),
                                                nq, nc, D, ws.data_ptr(), rows, lse.data_ptr(), loss.data_ptr(), _stream()),
                  "dr_inbatch_softmax_fwd_ws")
        else:
            check(lib.dr_inbatch_softmax_fwd(q.data_ptr(), c.data_ptr(), _ptr(w), _ptr(p), _ptr(ids), float(inv_tau),
                                             nq, nc, D, lse.data_ptr(), loss.data_ptr(), _stream()),
                  "dr_inbatch_softmax_fwd")
        ctx.inv_tau = float(inv_tau)
        ctx.ws = ws
        ctx.save_for_backward(q, c, w, p, ids, lse)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gloss):
        lib = _lib.load()
        q, c, w, p, ids, lse = ctx.saved_tensors
        nq, D = q.shape
        nc = c.shape[0]
        gl = _f32(gloss, "gloss").reshape(1)
        gq = torch.empty_like(q)
        gc = torch.empty_like(c)
        ws = ctx.ws
        if ws is not None:
            ctx.ws = None          # consumed (overwritten with the gradient factor) by this call
            check(lib.dr_inbatch_softmax_bwd_ws(q.data_ptr(), c.data_ptr(), _ptr(w), _ptr(p), _ptr(ids), ctx.inv_tau,
                                                nq, nc, D, lse.data_ptr(), gl.data_ptr(), ws.data_ptr(), ws.shape[0], 1,
                                                gq.data_ptr(), gc.data_ptr(), _stream()), "dr_inbatch_softmax_bwd_ws")
        else:
            check(lib.dr_inbatch_softmax_bwd(q.data_ptr(), c.data_ptr(), _ptr(w), _ptr(p), _ptr(ids), ctx.inv_tau,
                                             nq, nc, D, lse.data_ptr(), gl.data_ptr(), gq.data_ptr(), gc.data_ptr(),
                                             _stream()), "dr_inbatch_softmax_bwd")
        return gq, gc, None, None, None, None


def scores(q, c, sampling_prob=None, cand_ids=None) -> torch.Tensor:
    """Materialised [nq, nc] logits with R1/R2 corrections (no temperature); not differentiable."""
    lib = _lib.load()
    q = _f32(q, "q")
    c = _f32(c, "c")
    nq, D = q.shape
    nc = c.shape[0]
    p = None if sampling_prob is None else _f32(sampling_prob, "p").reshape(nc)
    ids = None if cand_ids is None else cand_ids.to(torch.int64).contiguous().reshape(nc)
    _lib.ensure_gemm_workspace(nq, D, nc, q.device)
    out = torch.empty((nq, nc), device=q.device, dtype=torch.float32)
    check(lib.dr_scores_fwd(q.data_ptr(), c.data_ptr(), _ptr(p), _ptr(ids), nq, nc, D, out.data_ptr(), _stream()),
          "dr_scores_fwd")
    return out


def hard_negative_topk(logits: torch.Tensor, k: int):
    lib = _lib.load()
    logits = _f32(logits, "logits")
    nq, nc = logits.shape
    out_l = torch.empty((nq, k), device=logits.device, dtype=torch.float32)
    out_y = torch.empty((nq, k), device=logits.device, dtype=torch.float32)
    out_i = torch.empty((nq, k), device=logits.device, dtype=torch.int32)
    check(lib.dr_hard_negative_topk(logits.data_ptr(), nq, nc, k, out_l.data_ptr(), out_y.data_ptr(),
                                    out_i.data_ptr(), _stream()), "dr_hard_negative_topk")
    return out_l, out_y, out_i


def bce_with_logits(z: torch.Tensor, y: torch.Tensor, z_add: torch.Tensor = None):
    """(loss[1], grad_z[B], prob[B]) of mean binary cross-entropy on logits z (+ z_add), one kernel."""
    lib = _lib.load()
    z = _f32(z, "logits").reshape(-1)
    z_add = None if z_add is None else _f32(z_add, "z_add").reshape(-1)
    y = _f32(y, "labels").reshape(-1)
    B = z.numel()
    prob = torch.empty_like(z)
    gz = torch.empty_like(z)
    loss = torch.empty((1,), device=z.device, dtype=torch.float32)
    check(lib.dr_bce_logits_fwd_bwd(z.data_ptr(), _ptr(z_add), y.data_ptr(), B, prob.data_ptr(), loss.data_ptr(), gz.data_ptr(),
                                    _stream()), "dr_bce_logits_fwd_bwd")
    return loss, gz, prob


def sgd_step_(p: torch.Tensor, g: torch.Tensor, lr: float) -> None:
    lib = _lib.load()
    check(lib.dr_sgd_step(p.data_ptr(), g.data_ptr(), p.numel(), float(lr), _stream()), "dr_sgd_step")


# ------------------------------------------------------------------------------------------
# SURVEY 8(f) "next" rows: Adam, id pipeline on the device, multi-valued slots, row top-k
# ------------------------------------------------------------------------------------------
COMBINER_CODES = {"sum": 0, "mean": 1, "sqrtn": 2}


def adam_step_(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, lr_t: float,
               beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-7, zero_grad: bool = True,
               lr_t_dev: torch.Tensor = None) -> None:
    """In-place dense Adam over a flat fp32 buffer (TensorFlow's ApplyAdam arithmetic; lr_t carries the bias
    correction, or lr_t_dev -- a 1-element CUDA float kept by `AdamClock` -- overrides it)."""
    lib = _lib.load()
    for name, t in (("p", p), ("g", g), ("m", m), ("v", v)):
        _f32(t, name)
        if not t.is_contiguous() or t.numel() != p.numel():
            raise ValueError(f"adam_step_: {name} must be contiguous with {p.numel()} elements")
    check(lib.dr_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), float(lr_t),
                           float(beta1), float(beta2), float(eps), int(bool(zero_grad)), _ptr(lr_t_dev), _stream()),
          "dr_adam_step")


class AdamClock:
    """Device-resident step counter t and bias-corrected rate lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t)
    (Keras optimizer_v2 Adam._prepare_local), advanced by one kernel so a captured train step needs no host scalar."""

    def __init__(self, lr: float, beta1: float = 0.9, beta2: float = 0.999, eps: float = 1e-7, device="cuda",
                 history: int = 0):
        self.lr, self.beta1, self.beta2, self.eps = float(lr), float(beta1), float(beta2), float(eps)
        self.step = torch.zeros((1,), dtype=torch.int64, device=device)
        self.lr_t = torch.zeros((1,), dtype=torch.float32, device=device)
        # ring of the last `history` bias-corrected rates (dr_adam_advance_hist): what the row-sparse TF-equal Adam
        # replays the skipped steps of a row with
        self.lr_hist = torch.zeros((history,), dtype=torch.float32, device=device) if history else None

    def advance(self) -> None:
        lib = _lib.load()
        if self.lr_hist is not None:
            check(lib.dr_adam_advance_hist(self.step.data_ptr(), self.lr, self.beta1, self.beta2, self.lr_t.data_ptr(),
                                           self.lr_hist.data_ptr(), self.lr_hist.numel(), _stream()), "dr_adam_advance_hist")
            return
        check(lib.dr_adam_advance(self.step.data_ptr(), self.lr, self.beta1, self.beta2, self.lr_t.data_ptr(),
                                  _stream()), "dr_adam_advance")


def lazy_adam_rows_(ids: torch.Tensor, rows: torch.Tensor, slot_offsets: torch.Tensor, D: int, row_stride: int,
                    flags: int, p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor,
                    stamp: torch.Tensor, clock: AdamClock, lin=None) -> None:
    """Row-sparse Adam over the rows `ids` [B, S] touch (see dr_lazy_adam_rows).  lin = (p, g, m, v) first-order
    arrays for the split layout, None when the weight rides in the row."""
    lib = _lib.load()
    ids = _ids(ids)
    B, S = ids.shape
    if stamp.dtype != torch.int32 or not stamp.is_cuda:
        raise TypeError("lazy_adam_rows_: stamp must be a CUDA int32 tensor [total rows]")
    lp = [None] * 4 if lin is None else [_f32(t, "lin").data_ptr() for t in lin]
    check(lib.dr_lazy_adam_rows(ids.data_ptr(), ids.element_size(), B, S, int(D), rows.data_ptr(),
                                slot_offsets.data_ptr(), p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(),
                                int(row_stride), int(flags), lp[0], lp[1], lp[2], lp[3], stamp.data_ptr(),
                                clock.step.data_ptr(), clock.lr_t.data_ptr(), clock.beta1, clock.beta2, clock.eps,
                                _stream()), "dr_lazy_adam_rows")


def _wide_bags(bags, B: int):
    """{slot: (flat ids, row_splits)} -> (n, host arrays of slots / id pointers / split pointers, kept tensors)."""
    import ctypes as C
    slots = sorted(bags) if bags else []
    keep = []
    for s in slots:
        bid, bsp = _ids(bags[s][0], "bag ids").to(torch.int64), _splits(bags[s][1])
        if bsp.numel() != B + 1:
            raise ValueError(f"slot {s}: row_splits has {bsp.numel()} entries, expected B+1 = {B + 1}")
        keep.append((bid, bsp))
    n = len(slots)
    return (n, (C.c_int * max(n, 1))(*slots), (C.c_void_p * max(n, 1))(*[k[0].data_ptr() for k in keep]),
            (C.c_void_p * max(n, 1))(*[k[1].data_ptr() for k in keep]), keep)


def _wide_args(table, ids, bags):
    ids = _ids(ids).to(torch.int64).contiguous()
    B, S = ids.shape
    n, bs, bi, bp, keep = _wide_bags(bags, B)
    return (table.state.data_ptr(), table.total_rows, table._rows.data_ptr(), table._offsets.data_ptr(), ids.data_ptr(),
            B, S, n, bs, bi, bp), (ids, keep)


class WideLinearFn(torch.autograd.Function):
    """logit [B] = tf.feature_column.linear_model over the LinearTable's columns (dr_wide_fwd).  Backward accumulates
    the row gradients into the table's records (dr_wide_bwd) for FtrlOptimizer.apply and returns no tensor gradient."""

    @staticmethod
    def forward(ctx, state, table, ids, bags):
        lib = _lib.load()
        _f32(state, "state")
        args, keep = _wide_args(table, ids, bags)
        logit = torch.empty((args[5],), device=state.device, dtype=torch.float32)
        check(lib.dr_wide_fwd(*args, logit.data_ptr(), _stream()), "dr_wide_fwd")
        ctx.table, ctx.args, ctx.keep = table, args, keep
        return logit

    @staticmethod
    def backward(ctx, g_logit):
        lib = _lib.load()
        g_logit = _f32(g_logit, "g_logit")
        with torch.no_grad():
            check(lib.dr_wide_bwd(*ctx.args, g_logit.data_ptr(), _stream()), "dr_wide_bwd")
        return None, None, None, None


class FtrlOptimizer:
    """tf.train.FtrlOptimizer(learning_rate, learning_rate_power=-0.5, initial_accumulator_value=0.1,
    l1_regularization_strength=0.0, l2_regularization_strength=0.0) for the wide part of a model: `apply(table)`
    updates the rows of a LinearTable the last forward touched, and its bias, with TensorFlow's ApplyFtrl arithmetic
    (dr_wide_ftrl), after the backward has accumulated their gradients.  Rows the batch did not touch keep their
    values, which is what TensorFlow's dense update leaves in them (see csrc/wide.cu).
    Served: learning_rate_power = -0.5 and no l2 shrinkage."""

    def __init__(self, learning_rate, learning_rate_power=-0.5, initial_accumulator_value=0.1,
                 l1_regularization_strength=0.0, l2_regularization_strength=0.0,
                 l2_shrinkage_regularization_strength=0.0):
        if not learning_rate > 0:
            raise ValueError(f"learning_rate {learning_rate} must be positive")
        if initial_accumulator_value < 0.0:
            raise ValueError(f"initial_accumulator_value {initial_accumulator_value} needs to be positive or zero")
        if learning_rate_power > 0.0:
            raise ValueError(f"learning_rate_power {learning_rate_power} needs to be negative or zero")
        if l1_regularization_strength < 0.0:
            raise ValueError(f"l1_regularization_strength {l1_regularization_strength} needs to be positive or zero")
        if l2_regularization_strength < 0.0:
            raise ValueError(f"l2_regularization_strength {l2_regularization_strength} needs to be positive or zero")
        if l2_shrinkage_regularization_strength < 0.0:
            raise ValueError("l2_shrinkage_regularization_strength needs to be positive or zero")
        if learning_rate_power != -0.5:
            raise NotImplementedError("FtrlOptimizer serves learning_rate_power = -0.5 only")
        if l2_shrinkage_regularization_strength != 0.0:
            raise NotImplementedError("FtrlOptimizer does not serve l2_shrinkage_regularization_strength")
        self.learning_rate = float(learning_rate)
        self.initial_accumulator_value = float(initial_accumulator_value)
        self.l1 = float(l1_regularization_strength)
        self.l2 = float(l2_regularization_strength)

    def apply(self, table) -> None:
        if table.lookups is None:
            raise RuntimeError("FtrlOptimizer.apply: the table has not run a forward pass")
        # the accumulator slot lives in the table (it is initialised there, and saved with it)
        if table.initial_accumulator_value != self.initial_accumulator_value:
            raise ValueError(f"FtrlOptimizer.apply: the table's accumulators start at "
                             f"{table.initial_accumulator_value}, this optimizer's initial_accumulator_value is "
                             f"{self.initial_accumulator_value}: build the LinearTable with the optimizer's value")
        lib = _lib.load()
        args, keep = _wide_args(table, *table.lookups)
        with torch.no_grad():
            check(lib.dr_wide_ftrl(*args, self.learning_rate, self.l1, self.l2, _stream()), "dr_wide_ftrl")


def cross_hash(values, value_offsets, row_splits, B: int, num_buckets: int, hash_key: int):
    """crossed_column on the device (dr_cross_hash).  values[k]: CUDA int64 values, or uint8 bytes of strings with
    value_offsets[k] (CUDA int64 [n+1]); row_splits[k]: CUDA int64 [B+1] or None (one value per example).
    -> ids [B] (-1: no cross) when every key is single-valued, else (flat ids, row_splits [B+1])."""
    import ctypes as C
    lib = _lib.load()
    K = len(values)
    dev = values[0].device
    for t in list(values) + [t for t in value_offsets if t is not None] + [t for t in row_splits if t is not None]:
        if not t.is_cuda or not t.is_contiguous():
            raise _lib.DeepRecError("cross_hash: every input must be a contiguous CUDA tensor")
    # the kernel reads B values (or B + 1 splits) of every key: check the lengths before it runs
    n = [v.numel() if o is None else o.numel() - 1 for v, o in zip(values, value_offsets)]
    for k, (nk, s) in enumerate(zip(n, row_splits)):
        if s is None and nk != B:
            raise ValueError(f"cross_hash: key {k} is single-valued with {nk} values for a batch of {B}")
        if s is not None and s.numel() != B + 1:
            raise ValueError(f"cross_hash: key {k} has {s.numel()} row splits for a batch of {B}")
    ragged = [k for k, s in enumerate(row_splits) if s is not None]
    if ragged and B > 0:
        ends = torch.stack([row_splits[k][-1] for k in ragged]).tolist()
        for k, e in zip(ragged, ends):
            if e > n[k]:
                raise ValueError(f"cross_hash: key {k}'s row splits end at {e}, past its {n[k]} values")
    # an empty values tensor has no storage; the kernel reads none of it but needs a non-null pointer
    values = [v if v.numel() else v.new_zeros((1,)) for v in values]
    vp = (C.c_void_p * K)(*[v.data_ptr() for v in values])
    op = (C.c_void_p * K)(*[None if o is None else o.data_ptr() for o in value_offsets])
    sp = (C.c_void_p * K)(*[None if s is None else s.data_ptr() for s in row_splits])
    hk = int(hash_key) & 0xFFFFFFFFFFFFFFFF
    if all(s is None for s in row_splits):
        out = torch.empty((B,), dtype=torch.int64, device=dev)
        check(lib.dr_cross_hash(K, vp, op, sp, B, hk, int(num_buckets), None, out.data_ptr(), _stream()),
              "dr_cross_hash")
        return out
    splits = torch.empty((B + 1,), dtype=torch.int64, device=dev)
    check(lib.dr_cross_hash(K, vp, op, sp, B, hk, int(num_buckets), splits.data_ptr(), None, _stream()),
          "dr_cross_hash")
    splits = torch.cumsum(splits, 0)
    out = torch.empty((int(splits[-1]),), dtype=torch.int64, device=dev)
    if out.numel() == 0:
        return out, splits
    check(lib.dr_cross_hash(K, vp, op, sp, B, hk, int(num_buckets), splits.data_ptr(), out.data_ptr(), _stream()),
          "dr_cross_hash")
    return out, splits


def hash_bucket_i64(values: torch.Tensor, num_buckets: int) -> torch.Tensor:
    """tf.strings.to_hash_bucket_fast(tf.as_string(values), num_buckets) for a CUDA int64 tensor."""
    lib = _lib.load()
    if not values.is_cuda:
        raise _lib.DeepRecError("hash_bucket_i64: values must be a CUDA tensor (host features use hashing.hash_bucket)")
    v = values.to(torch.int64).contiguous()
    out = torch.empty_like(v)
    check(lib.dr_hash_bucket_i64(v.data_ptr(), v.numel(), int(num_buckets), out.data_ptr(), _stream()),
          "dr_hash_bucket_i64")
    return out


def hash_bucket_bytes(data: torch.Tensor, offsets: torch.Tensor, num_buckets: int) -> torch.Tensor:
    """Strings shipped as one uint8 CUDA buffer + int64 offsets [n+1] -> bucket ids [n]."""
    lib = _lib.load()
    if not (data.is_cuda and offsets.is_cuda):
        raise _lib.DeepRecError("hash_bucket_bytes: data / offsets must be CUDA tensors")
    if data.dtype != torch.uint8 or offsets.dtype != torch.int64:
        raise TypeError("hash_bucket_bytes: data must be uint8 and offsets int64")
    data, offsets = data.contiguous(), offsets.contiguous()
    n = offsets.numel() - 1
    out = torch.empty((max(n, 0),), device=data.device, dtype=torch.int64)
    check(lib.dr_hash_bucket_bytes(data.data_ptr(), offsets.data_ptr(), n, int(num_buckets), out.data_ptr(), _stream()),
          "dr_hash_bucket_bytes")
    return out


def vocab_lookup_i64(values: torch.Tensor, keys_sorted: torch.Tensor, vocab_index: torch.Tensor,
                     default_id: int = -1) -> torch.Tensor:
    lib = _lib.load()
    if not values.is_cuda:
        raise _lib.DeepRecError("vocab_lookup_i64: values must be a CUDA tensor")
    v = values.to(torch.int64).contiguous()
    out = torch.empty_like(v)
    check(lib.dr_vocab_lookup_i64(v.data_ptr(), v.numel(), keys_sorted.data_ptr(), vocab_index.data_ptr(),
                                  keys_sorted.numel(), int(default_id), out.data_ptr(), _stream()),
          "dr_vocab_lookup_i64")
    return out


def _bag_fwd(lib, table_ptr, rows, row_stride, ids, splits, B, D, combiner, out_ptr, out_stride):
    check(lib.dr_embed_bag_fwd(table_ptr, rows, row_stride, ids.data_ptr(), ids.element_size(), splits.data_ptr(),
                               B, D, COMBINER_CODES[combiner], out_ptr, out_stride, _stream()), "dr_embed_bag_fwd")


def _bag_bwd(lib, ids, splits, B, D, combiner, g_ptr, g_stride, rows, row_stride, grad_ptr, scale):
    check(lib.dr_embed_bag_bwd(ids.data_ptr(), ids.element_size(), splits.data_ptr(), B, D, COMBINER_CODES[combiner],
                               g_ptr, g_stride, rows, row_stride, grad_ptr, float(scale), _stream()),
          "dr_embed_bag_bwd")


def _splits(row_splits: torch.Tensor) -> torch.Tensor:
    if not isinstance(row_splits, torch.Tensor) or row_splits.dtype != torch.int64 or not row_splits.is_cuda:
        raise TypeError("row_splits must be a CUDA int64 tensor [B+1]")
    return row_splits.contiguous()


class EmbedBag(torch.autograd.Function):
    """out[B, D] = combine over the valid ids of each ragged bag (multi-valued slot); see dr_embed_bag_fwd.

    `table` is a contiguous [rows, row_stride] fp32 tensor; the D embedding columns start at `col_offset`
    (row_stride == D, col_offset == 0 for a plain table).  sparse_lr: None -> dense gradient for `table`;
    a float -> fused sparse SGD in backward.
    """

    @staticmethod
    def forward(ctx, table, ids, row_splits, D: int, combiner: str, sparse_lr, col_offset: int = 0):
        lib = _lib.load()
        table = _f32(table, "table")
        ids = _ids(ids)
        row_splits = _splits(row_splits)
        B = row_splits.numel() - 1
        rows, stride = table.shape
        if col_offset + D > stride:
            raise ValueError(f"EmbedBag: columns [{col_offset}, {col_offset + D}) exceed the row pitch {stride}")
        out = torch.empty((B, D), device=table.device, dtype=torch.float32)
        _bag_fwd(lib, table.data_ptr() + 4 * col_offset, rows, stride, ids, row_splits, B, D, combiner, out.data_ptr(), D)
        ctx.save_for_backward(table, ids, row_splits)
        ctx.D, ctx.combiner, ctx.sparse_lr, ctx.col_offset = D, combiner, sparse_lr, col_offset
        return out

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        table, ids, row_splits = ctx.saved_tensors
        g = _f32(g, "g")
        fused = ctx.sparse_lr is not None
        tgt = table if fused else torch.zeros_like(table)
        B = row_splits.numel() - 1
        with torch.no_grad():
            _bag_bwd(lib, ids, row_splits, B, ctx.D, ctx.combiner, g.data_ptr(), ctx.D, table.shape[0], table.shape[1],
                     tgt.data_ptr() + 4 * ctx.col_offset, -float(ctx.sparse_lr) if fused else 1.0)
        return (None if fused else tgt), None, None, None, None, None, None


class EmbedFMMixed(torch.autograd.Function):
    """EmbedFM for a collection in which some slots are multi-valued (SURVEY 8f #2).

    Each ragged slot r is first reduced into a per-batch scratch "table" of B rows in the collection's own row
    layout (embedding columns = mean of the bag's valid rows, first-order entry = SUM of their weights: the
    indicator column is a multi-hot count vector); the fused gather + FM kernel then reads slot r from that
    scratch with ids 0..B-1, so the whole model is still ONE dr_embed_fm_fwd launch.  Backward mirrors it: the
    fused backward accumulates slot r's per-example gradient in a scratch grad table, dr_embed_bag_bwd spreads
    it over the bag's rows (embedding / count, first-order x 1).

    ids [B, S]: columns of ragged slots are ignored.  bags: {slot: (flat_ids, row_splits[B+1])}.
    """

    @staticmethod
    def forward(ctx, ids, weight, linear, bias, meta, bags):
        lib = _lib.load()
        if not meta.with_linear:
            return EmbedFMMixed._forward_no_linear(ctx, ids, weight, meta, bags)
        if bias is None:
            raise ValueError("EmbedFMMixed needs a collection with the first-order term (with_linear=True)")
        ids = _ids(ids).clone()
        B, S = ids.shape
        D, RS = meta.dim, meta.row_stride
        dev = weight.device
        fused_rows = meta.layout == "fused"
        tp, lp, rows = meta.pointers(weight, linear)
        tp, lp, rows = tp.clone(), lp.clone(), rows.clone()
        slots = sorted(bags)
        scratch = torch.zeros((len(slots), B, RS), device=dev, dtype=torch.float32)
        scratch_lin = None if fused_rows else torch.zeros((len(slots), B), device=dev, dtype=torch.float32)
        ar = torch.arange(B, device=dev, dtype=ids.dtype)
        saved_bags = []
        for k, s in enumerate(slots):
            bid, bsp = bags[s]
            bid, bsp = _ids(bid, "bag ids"), _splits(bsp)
            if bsp.numel() != B + 1:
                raise ValueError(f"slot {s}: row_splits has {bsp.numel()} entries, expected B+1 = {B + 1}")
            off, n_rows = int(meta._offsets[s]), meta.rows_list[s]
            base = weight.data_ptr() + 4 * off * RS
            _bag_fwd(lib, base, n_rows, RS, bid, bsp, B, D, "mean", scratch[k].data_ptr(), RS)
            if fused_rows:
                _bag_fwd(lib, base + 4 * D, n_rows, RS, bid, bsp, B, 1, "sum", scratch[k].data_ptr() + 4 * D, RS)
                lin_ptr = scratch[k].data_ptr() + 4 * D
            else:
                _bag_fwd(lib, linear.data_ptr() + 4 * off, n_rows, 1, bid, bsp, B, 1, "sum",
                         scratch_lin[k].data_ptr(), 1)
                lin_ptr = scratch_lin[k].data_ptr()
            tp[s] = scratch[k].data_ptr()
            lp[s] = lin_ptr
            rows[s] = B
            ids[:, s] = ar
            saved_bags.append((s, bid, bsp))
        stack = torch.empty((B, S, D), device=dev, dtype=torch.float32)
        sum_e = torch.empty((B, D), device=dev, dtype=torch.float32)
        logit = torch.empty((B,), device=dev, dtype=torch.float32)
        check(lib.dr_embed_fm_fwd(tp.data_ptr(), lp.data_ptr(), rows.data_ptr(), ids.data_ptr(), ids.element_size(),
                                  _ptr(bias), B, S, D, RS, meta.lin_stride, meta.flags, stack.data_ptr(),
                                  sum_e.data_ptr(), logit.data_ptr(), _stream()), "dr_embed_fm_fwd")
        ctx.meta, ctx.saved_bags = meta, saved_bags
        ctx.save_for_backward(ids, stack, sum_e, weight, linear, bias, rows)
        return stack, logit

    @staticmethod
    def _forward_no_linear(ctx, ids, weight, meta, bags):
        """Embeddings only (a collection without first-order weights, e.g. WDL's deep half): the bags are
        mean-reduced into scratch tables and one dr_embed_fm_fwd without a logit gathers the stack."""
        lib = _lib.load()
        ids = _ids(ids).clone()
        B, S = ids.shape
        D, RS = meta.dim, meta.row_stride
        dev = weight.device
        tp, _, rows = meta.pointers(weight, None)
        tp, rows = tp.clone(), rows.clone()
        slots = sorted(bags)
        scratch = torch.empty((len(slots), B, RS), device=dev, dtype=torch.float32)
        ar = torch.arange(B, device=dev, dtype=ids.dtype)
        saved_bags = []
        for k, s in enumerate(slots):
            bid, bsp = bags[s]
            bid, bsp = _ids(bid, "bag ids"), _splits(bsp)
            if bsp.numel() != B + 1:
                raise ValueError(f"slot {s}: row_splits has {bsp.numel()} entries, expected B+1 = {B + 1}")
            off, n_rows = int(meta._offsets[s]), meta.rows_list[s]
            _bag_fwd(lib, weight.data_ptr() + 4 * off * RS, n_rows, RS, bid, bsp, B, D, "mean", scratch[k].data_ptr(),
                     RS)
            tp[s] = scratch[k].data_ptr()
            rows[s] = B
            ids[:, s] = ar
            saved_bags.append((s, bid, bsp))
        stack = torch.empty((B, S, D), device=dev, dtype=torch.float32)
        check(lib.dr_embed_fm_fwd(tp.data_ptr(), None, rows.data_ptr(), ids.data_ptr(), ids.element_size(), None,
                                  B, S, D, RS, meta.lin_stride, 0, stack.data_ptr(), None, None, _stream()),
              "dr_embed_fm_fwd")
        ctx.meta, ctx.saved_bags = meta, saved_bags
        ctx.save_for_backward(ids, stack, None, weight, None, None, rows)
        dummy = stack.new_zeros((0,))
        ctx.mark_non_differentiable(dummy)
        return stack, dummy

    @staticmethod
    def _backward_no_linear(ctx, g_stack):
        lib = _lib.load()
        ids, stack, _, weight, _, _, rows = ctx.saved_tensors
        meta = ctx.meta
        if g_stack is None:
            return None, None, None, None, None, None
        g_stack = _f32(g_stack, "g_stack")
        B, S = ids.shape
        D, RS = meta.dim, meta.row_stride
        fused_sgd = meta.sparse_lr is not None
        gw, scale = (weight, -float(meta.sparse_lr)) if fused_sgd else (torch.zeros_like(weight), 1.0)
        tp, _, _ = meta.pointers(gw, None, cache=False)
        tp = tp.clone()
        gscratch = torch.zeros((len(ctx.saved_bags), B, RS), device=weight.device, dtype=torch.float32)
        for k, (s, _, _) in enumerate(ctx.saved_bags):
            tp[s] = gscratch[k].data_ptr()
        with torch.no_grad():
            check(lib.dr_embed_fm_bwd(ids.data_ptr(), ids.element_size(), rows.data_ptr(), stack.data_ptr(), None, None,
                                      g_stack.data_ptr(), B, S, D, RS, meta.lin_stride, 0, tp.data_ptr(), None, None,
                                      scale, _stream()), "dr_embed_fm_bwd")
            for k, (s, bid, bsp) in enumerate(ctx.saved_bags):
                off, n_rows = int(meta._offsets[s]), meta.rows_list[s]
                _bag_bwd(lib, bid, bsp, B, D, "mean", gscratch[k].data_ptr(), RS, n_rows, RS,
                         gw.data_ptr() + 4 * off * RS, 1.0)
        return None, (None if fused_sgd else gw), None, None, None, None

    @staticmethod
    def backward(ctx, g_stack, g_logit):
        if not ctx.meta.with_linear:
            return EmbedFMMixed._backward_no_linear(ctx, g_stack)
        lib = _lib.load()
        ids, stack, sum_e, weight, linear, bias, rows = ctx.saved_tensors
        meta = ctx.meta
        B, S = ids.shape
        D, RS = meta.dim, meta.row_stride
        dev = weight.device
        fused_rows = meta.layout == "fused"
        g_stack = None if g_stack is None else _f32(g_stack, "g_stack")
        g_logit = None if g_logit is None else _f32(g_logit, "g_logit")
        if g_stack is None and g_logit is None:
            return None, None, None, None, None, None
        if g_logit is None:
            g_logit = torch.zeros((B,), device=dev, dtype=torch.float32)
        fused_sgd = meta.sparse_lr is not None
        if fused_sgd:
            gw, gl, gb, scale = weight, linear, bias, -float(meta.sparse_lr)
        else:
            gw = torch.zeros_like(weight)
            gl = None if linear is None else torch.zeros_like(linear)
            gb = None if bias is None else torch.zeros_like(bias)
            scale = 1.0
        tp, lp, _ = meta.pointers(gw, gl, cache=False)
        tp, lp = tp.clone(), lp.clone()
        nb = len(ctx.saved_bags)
        gscratch = torch.zeros((nb, B, RS), device=dev, dtype=torch.float32)
        gscratch_lin = None if fused_rows else torch.zeros((nb, B), device=dev, dtype=torch.float32)
        for k, (s, _, _) in enumerate(ctx.saved_bags):
            tp[s] = gscratch[k].data_ptr()
            lp[s] = gscratch[k].data_ptr() + 4 * D if fused_rows else gscratch_lin[k].data_ptr()
        with torch.no_grad():
            check(lib.dr_embed_fm_bwd(ids.data_ptr(), ids.element_size(), rows.data_ptr(), stack.data_ptr(),
                                      sum_e.data_ptr(), g_logit.data_ptr(), _ptr(g_stack), B, S, D, RS,
                                      meta.lin_stride, meta.flags, tp.data_ptr(), lp.data_ptr(), _ptr(gb), scale,
                                      _stream()), "dr_embed_fm_bwd")
            for k, (s, bid, bsp) in enumerate(ctx.saved_bags):
                off, n_rows = int(meta._offsets[s]), meta.rows_list[s]
                base = gw.data_ptr() + 4 * off * RS
                # the scratch already carries `scale`: spread it with scale = 1
                _bag_bwd(lib, bid, bsp, B, D, "mean", gscratch[k].data_ptr(), RS, n_rows, RS, base, 1.0)
                if fused_rows:
                    _bag_bwd(lib, bid, bsp, B, 1, "sum", gscratch[k].data_ptr() + 4 * D, RS, n_rows, RS, base + 4 * D, 1.0)
                else:
                    _bag_bwd(lib, bid, bsp, B, 1, "sum", gscratch_lin[k].data_ptr(), 1, n_rows, 1,
                             gl.data_ptr() + 4 * off, 1.0)
        if fused_sgd:
            return None, None, None, None, None, None
        return None, gw, gl, gb, None, None


def topk_rows(scores_: torch.Tensor, k: int):
    """tf.math.top_k(scores, k) on a CUDA [nq, nc] matrix: (values [nq,k] descending, int32 indices [nq,k])."""
    lib = _lib.load()
    s = _f32(scores_, "scores")
    if s.dim() != 2:
        raise ValueError(f"topk_rows: expected a 2-D score matrix, got shape {tuple(s.shape)}")
    nq, nc = s.shape
    if k > nc or k < 1:
        raise ValueError(f"input must have at least k columns. Had {nc}, needed {k}")
    vals = torch.empty((nq, k), device=s.device, dtype=torch.float32)
    idx = torch.empty((nq, k), device=s.device, dtype=torch.int32)
    check(lib.dr_topk_rows(s.data_ptr(), nq, nc, nc, k, vals.data_ptr(), idx.data_ptr(), _stream()), "dr_topk_rows")
    return vals, idx


def _idx32(indices: torch.Tensor) -> torch.Tensor:
    if not indices.is_cuda:
        raise _lib.DeepRecError("indices must be a CUDA tensor (no CPU fallback)")
    if indices.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"indices: expected int32 / int64, got {indices.dtype}")
    return indices.to(torch.int32).contiguous()


def take_long_axis(arr: torch.Tensor, indices: torch.Tensor) -> torch.Tensor:
    """out[i, j] = arr[i, indices[i, j]] (factorized_top_k.py:26-41) for any 4- or 8-byte dtype; a 1-D `arr` is one
    shared row: tf.gather(identifiers, indices)."""
    lib = _lib.load()
    if not arr.is_cuda:
        raise _lib.DeepRecError("take_long_axis: arr must be a CUDA tensor (no CPU fallback)")
    if arr.element_size() not in (4, 8):
        raise TypeError(f"take_long_axis: 4- or 8-byte elements only, got {arr.dtype}")
    idx = _idx32(indices)
    if idx.dim() != 2:
        raise ValueError(f"take_long_axis: indices must be 2-D, got shape {tuple(idx.shape)}")
    arr = arr.contiguous()
    nq, k = idx.shape
    if arr.dim() == 1:
        ncols, ld = arr.shape[0], 0
    elif arr.dim() == 2 and arr.shape[0] == nq:
        ncols, ld = arr.shape[1], arr.shape[1]
    else:
        raise ValueError(f"take_long_axis: arr {tuple(arr.shape)} does not match indices {tuple(idx.shape)}")
    out = torch.empty((nq, k), device=arr.device, dtype=arr.dtype)
    if nq and k:
        check(lib.dr_take_long_axis(arr.data_ptr(), arr.element_size(), nq, ncols, ld, idx.data_ptr(), k, out.data_ptr(),
                                    _stream()), "dr_take_long_axis")
    return out


def exclude_adjust(scores_: torch.Tensor, identifiers: torch.Tensor, exclude: torch.Tensor,
                   penalty: float = 1.0e5) -> torch.Tensor:
    """scores - isin(identifiers, exclude) * 1e5 (factorized_top_k.py:58-62), integer identifiers."""
    lib = _lib.load()
    s = _f32(scores_, "scores")
    ident = _ids(identifiers, "identifiers").to(torch.int64).contiguous()
    ex = _ids(exclude, "exclude").to(torch.int64).contiguous()
    if s.dim() != 2 or ident.shape != s.shape or ex.dim() != 2 or ex.shape[0] != s.shape[0]:
        raise ValueError(f"exclude_adjust: scores {tuple(s.shape)}, identifiers {tuple(ident.shape)}, "
                         f"exclude {tuple(ex.shape)} do not line up")
    out = torch.empty_like(s)
    check(lib.dr_exclude_adjust(s.data_ptr(), ident.data_ptr(), ex.data_ptr(), s.shape[0], s.shape[1], ex.shape[1],
                                float(penalty), out.data_ptr(), _stream()), "dr_exclude_adjust")
    return out


def rowwise_dot(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """[n, 1] = reduce_sum(a * b, axis=1, keepdims=True)."""
    lib = _lib.load()
    a, b = _f32(a, "a"), _f32(b, "b")
    if a.shape != b.shape or a.dim() != 2:
        raise ValueError(f"rowwise_dot: shapes {tuple(a.shape)} vs {tuple(b.shape)}")
    out = torch.empty((a.shape[0], 1), device=a.device, dtype=torch.float32)
    check(lib.dr_rowwise_dot(a.data_ptr(), b.data_ptr(), a.shape[0], a.shape[1], out.data_ptr(), _stream()),
          "dr_rowwise_dot")
    return out


def column_rank(positive: torch.Tensor, others: torch.Tensor) -> torch.Tensor:
    """rank[i] = number of entries of others[i, :] strictly above positive[i] (int32)."""
    lib = _lib.load()
    p, o = _f32(positive, "positive").reshape(-1), _f32(others, "others")
    if o.dim() != 2 or o.shape[0] != p.shape[0]:
        raise ValueError(f"column_rank: positive {tuple(p.shape)} vs others {tuple(o.shape)}")
    rank = torch.empty((p.shape[0],), device=p.device, dtype=torch.int32)
    check(lib.dr_column_rank(p.data_ptr(), o.data_ptr(), p.shape[0], o.shape[1], o.shape[1], rank.data_ptr(), _stream()),
          "dr_column_rank")
    return rank
