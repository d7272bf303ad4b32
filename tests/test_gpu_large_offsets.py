"""The embedding, Adam and sharded-row kernels on arenas past 2^31 and 2^32 elements, against the float64 oracle.

A production table -- bench.py's C5 workload keeps 26 x 3.8 M rows x 128 floats in one arena of 12.8 G floats -- puts
row offsets far past what a 32-bit product can hold, while every other test of these kernels uses arenas of at most a
few hundred million elements.  Each case here allocates one arena (table, state blocks, Adam buffers or owner shards)
past 2^31 or 2^32 elements and touches rows whose element offset (row x row stride, or global row x state stride) lies

  * just below 2^31, on 2^31, on 2^32 (a row that straddles each boundary when the stride is not a power of two),
  * in [2^32, 2^32 + 2^31), and the last row of the arena,

plus a few low rows, each looked up several times (the accumulation paths run at the high offsets too), with int32
and int64 ids.

Arenas are never copied to the host.  Every float is a deterministic function of (row, column) (`pattern`), written
on the device chunk by chunk, so the oracle's inputs are regenerated for the touched rows only and "every row the call
must not write is unchanged" is a chunked on-device comparison against the same function.  A truncated offset
(row x stride mod 2^32) lands on a low row inside the allocation: the touched rows then come out wrong, and the low row
it hit shows up as a changed row; the low rows at the same offsets modulo 2^32 are kept out of the touched set.

Gathers and copies are checked bit for bit; everything else at the bounds of the small-shape test of the same entry
(test_gpu_embed.py, test_gpu_adam_replay.py, test_gpu_sharded_emulated.py).  Each test states the memory it needs and
skips, naming it and what was free, when the (shared) GPU has less than need x 1.1 + 2 GiB free; it prints its peak
allocation and wall time.
"""
import functools
import gc
import time
import traceback

import numpy as np
import pytest
import torch

from adam_oracle import (K_CATCH_UP_MAX, U, Entry, check_bound, functor, moments, replay, update_slack)
from adam_oracle import C_FUNCTOR, C_MOMENT, U64
from oracle import reference_np as R

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
GiB = 1 << 30
TWO31, TWO32 = 1 << 31, 1 << 32
CHUNK = 1 << 24                 # elements per fill / compare pass
SENT = -7777.25                 # around every output: must survive
PAD = 64
LIN_IN_ROW = 1


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L


def _st():
    return torch.cuda.current_stream().cuda_stream


def _call(name, *args):
    L = _lib()
    L.check(getattr(L.load(), name)(*args), name)


def _ptr(t):
    return None if t is None else t.data_ptr()


def need(nbytes, what):
    free, _ = torch.cuda.mem_get_info()
    want = int(nbytes * 1.1) + 2 * GiB
    if free < want:
        pytest.skip(f"{what} needs {nbytes / GiB:.1f} GiB ({want / GiB:.1f} GiB with the margin); "
                    f"{free / GiB:.1f} GiB free on this shared GPU")


@pytest.fixture(autouse=True)
def _memory_and_time(request):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    free0 = torch.cuda.mem_get_info()[0]
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[{request.node.name}] peak allocated {torch.cuda.max_memory_allocated() / GiB:.2f} GiB, "
          f"{time.perf_counter() - t0:.1f} s, {free0 / GiB:.1f} GiB free at start")
    gc.collect()
    torch.cuda.empty_cache()


def releases_memory(fn):
    """Runs the test body so that a failure keeps no reference to its frames: a traceback would hold tens of GB of
    arenas alive and make every later test skip."""
    @functools.wraps(fn)
    def wrapper(*a, **kw):
        msg = None
        try:
            fn(*a, **kw)
        except Exception:           # noqa: BLE001  (pytest's skip / fail outcomes are BaseExceptions and pass through)
            msg = traceback.format_exc()
        if msg is not None:
            pytest.fail(msg, pytrace=False)
    return wrapper


# ---- the pattern: every float a function of (global row, column, salt) ------------------------------------------------
def _key(r, c, salt):
    return (r * 131 + c * 7 + salt) % 8191


def pattern_np(rows, ncols, salt, scale):
    r = np.asarray(rows, np.int64)[:, None]
    c = np.arange(ncols, dtype=np.int64)[None, :]
    return ((_key(r, c, salt) - 4095).astype(F64) * scale).astype(F32)


def pattern_dev(r0, r1, ncols, salt, scale, mul=1, add=0):
    """Rows r0 .. r1 of a [*, ncols] buffer whose local row L holds global row L * mul + add."""
    r = torch.arange(r0, r1, dtype=torch.int64, device="cuda")[:, None] * mul + add
    c = torch.arange(ncols, dtype=torch.int64, device="cuda")[None, :]
    return (_key(r, c, salt) - 4095).to(torch.float32) * scale


def _chunks(nrows, ncols):
    step = max(1, CHUNK // ncols)
    for r0 in range(0, nrows, step):
        yield r0, min(nrows, r0 + step)


def fill(t2d, gen):
    """t2d [rows, cols] (a view into an arena) <- gen(r0, r1) chunk by chunk."""
    for r0, r1 in _chunks(t2d.shape[0], t2d.shape[1]):
        t2d[r0:r1].copy_(gen(r0, r1))


def changed_rows(t2d, gen):
    """Local rows of t2d whose bits differ from gen (NaN-safe: compared as int32)."""
    out = []
    for r0, r1 in _chunks(t2d.shape[0], t2d.shape[1]):
        diff = (t2d[r0:r1].view(torch.int32) != gen(r0, r1).view(torch.int32)).any(1)
        idx = diff.nonzero().flatten()
        if idx.numel():
            out.append(idx.cpu().numpy() + r0)
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def assert_only(changed, allowed, what):
    bad = np.setdiff1d(changed, allowed)
    assert bad.size == 0, f"{what}: {bad.size} rows outside the touched set changed, e.g. {bad[:8].tolist()}"


class Guarded:
    def __init__(self, n):
        self.n = n
        self.full = torch.full((n + 2 * PAD,), SENT, device="cuda")
        self.t = self.full[PAD:PAD + n]

    def get(self):
        f = self.full.cpu().numpy()
        assert (f[:PAD] == SENT).all() and (f[PAD + self.n:] == SENT).all(), "store outside the output"
        return f[PAD:PAD + self.n].copy()


# ---- row placement -----------------------------------------------------------------------------------------------------
def placed_rows(total, stride, low=(3, 777)):
    """Rows whose element offset row * stride is just below 2^31, on / across 2^31 and 2^32, inside
    [2^32, 2^32 + 2^31), and the last row; plus low rows.  Returns (touched, aliases): the rows holding the same offsets
    modulo 2^32, which must stay untouched."""
    want = set(low)
    for edge in (TWO31, TWO32):
        r = edge // stride
        want |= {r - 1, (edge - 1) // stride, r, r + 1}
    mid = (TWO32 + TWO31 // 2) // stride + 17
    if mid >= total:                     # an arena that ends before 2^32 + 2^31: halfway from 2^32 to its end
        mid = (TWO32 // stride + total) // 2
    want |= {mid, total - 2, total - 1}
    touched = np.array(sorted(r for r in want if 0 <= r < total), np.int64)
    aliases = []
    for r in touched:
        for off in (r * stride, (r + 1) * stride - 1):
            if off >= TWO32:
                aliases.append((off - TWO32) // stride)
    aliases = np.unique(np.array(aliases, np.int64))
    assert not np.intersect1d(touched, aliases).size
    return touched, aliases


def slot_plan(total, edge=8):
    """Three slots: [the bulk | edge rows | edge rows], so slot 0's local ids times the stride reach past 2^32 and
    the other slots' table pointers sit at the end of the arena."""
    rows = [total - 2 * edge, edge, edge]
    offs = np.array([0, total - 2 * edge, total - edge], np.int64)
    return rows, offs


def make_ids(touched, rows, offs, seed, dup=(1, 2, 3)):
    """[B, S] local ids: every touched row looked up 1-3 times (round robin), OOV ids -1 and rows[s], the rest -1."""
    rng = np.random.default_rng(seed)
    S = len(rows)
    cols = [[] for _ in range(S)]
    for k, r in enumerate(touched):
        s = int(np.searchsorted(offs, r, side="right") - 1)
        cols[s] += [int(r - offs[s])] * dup[k % len(dup)]
    for s in range(S):
        cols[s] += [-1, rows[s], -1]
    B = max(len(c) for c in cols) + 5
    ids = np.full((B, S), -1, np.int64)
    for s, c in enumerate(cols):
        ids[:, s] = rng.permutation(c + [-1] * (B - len(c)))
    return ids


class Compact:
    """The oracle's view of the lookups: per slot a table holding only the rows the ids name, ids remapped to it."""

    def __init__(self, ids, rows, offs, emb_of, lin_of):
        self.ids = np.full(ids.shape, -1, np.int64)
        self.tables, self.lins, self.uniq = [], [], []
        for s in range(ids.shape[1]):
            col = ids[:, s]
            ok = (col >= 0) & (col < rows[s])
            u = np.unique(col[ok])
            self.uniq.append(u + offs[s])
            self.tables.append(emb_of(u + offs[s]))
            self.lins.append(lin_of(u + offs[s]))
            self.ids[ok, s] = np.searchsorted(u, col[ok])
        self.rows = [t.shape[0] for t in self.tables]

    def global_rows(self):
        return np.concatenate(self.uniq)


def check_forward(comp, bias, stack, sum_e, logit, what):
    ref_stack = R.stack_embeddings(comp.tables, comp.ids)
    assert np.array_equal(stack.view(np.uint32), ref_stack.reshape(-1).view(np.uint32)), f"{what}: stack not a copy"
    st64 = ref_stack.astype(F64)
    if sum_e is not None:
        err = np.abs(sum_e.astype(F64) - st64.sum(1).reshape(-1))
        assert (err <= 1e-5 * np.abs(st64).sum(1).reshape(-1) + 1e-7).all(), f"{what}: sum_e max err {err.max()}"
    if logit is not None:
        ref, _ = R.fm_logit(comp.tables, comp.lins, bias, comp.ids, F64)
        lin = np.abs(R.linear_term(comp.lins, 0.0, comp.ids, F64)).reshape(-1) + abs(float(bias))
        scale = lin + 0.5 * ((st64.sum(1) ** 2).sum(1) + (st64 ** 2).sum((1, 2)))
        err = np.abs(logit.astype(F64) - ref.reshape(-1))
        assert (err <= 1e-5 * scale + 1e-6).all(), f"{what}: logit max err {err.max()}"


def fm_grads(comp, stack, gl, gs):
    """Row gradients of the FM backward (float64), their scales (test_gpu_embed's bound) and per-lookup |terms|."""
    st64 = stack.astype(F64)
    gts, gls, gb = R.embed_fm_grad(comp.rows, comp.ids, st64, gl, gs, F64)
    absdE = np.abs(gl)[:, None, None] * (np.abs(st64.sum(1, keepdims=True)) + np.abs(st64)) + np.abs(gs)
    sct, _, _ = R.embed_fm_grad(comp.rows, comp.ids, st64 * 0, None, absdE, F64)
    _, scl, _ = R.embed_fm_grad(comp.rows, comp.ids, st64, np.abs(gl), None, F64)
    d_e = gl[:, None, None] * (st64.sum(1, keepdims=True) - st64) + gs
    tt, tl, _ = R.embed_fm_grad(comp.rows, comp.ids, st64 * 0, np.abs(gl), np.abs(d_e), F64)
    hits = [np.bincount(comp.ids[:, s][comp.ids[:, s] >= 0], minlength=comp.rows[s]) for s in range(len(comp.rows))]
    cat = lambda xs: np.concatenate(xs, 0)
    return dict(g=cat(gts), gl=cat(gls), sc=cat(sct), scl=cat(scl), tt=cat(tt), tl=cat(tl), hits=cat(hits), gb=gb)


# ---- 1-2. the embedding kernels on one arena ---------------------------------------------------------------------------
EMB_SALT, LIN_SALT = 11, 5
EMB_SCALE, LIN_SCALE = 2.0 ** -13, 2.0 ** -16

LAYOUTS = {
    # name: D, row_stride, total rows, first-order weight in the row
    "fused_D16": (16, 32, (1 << 27) + 1024, True),       # 2^32 + 32768 floats, 17.2 GB
    "split_D128": (128, 128, (1 << 25) + 64, False),     # 2^32 + 8192 floats + 134 MB of first-order weights
    "split_D12": (12, 12, (TWO32 + (1 << 28)) // 12 + 3, False),   # rows straddle 2^31 and 2^32; 18.3 + 1.5 GB
}


class Table:
    def __init__(self, D, rs, total, fused):
        self.D, self.rs, self.total, self.fused = D, rs, total, fused
        self.rows, self.offs = slot_plan(total)
        self.arena = torch.empty((total, rs), device="cuda")
        self.lin = None if fused else torch.empty(total, device="cuda")
        self.reset()
        base = self.arena.data_ptr()
        self.d_rows = torch.tensor(self.rows, dtype=torch.int64, device="cuda")
        self.d_offs = torch.from_numpy(self.offs).cuda()
        self.tp = torch.tensor([base + int(o) * rs * 4 for o in self.offs], dtype=torch.int64, device="cuda")
        self.lp = self.tp if fused else torch.tensor([self.lin.data_ptr() + int(o) * 4 for o in self.offs],
                                                     dtype=torch.int64, device="cuda")
        self.flags = LIN_IN_ROW if fused else 0
        self.lin_stride = rs if fused else 1

    def gen(self, r0, r1):
        return pattern_dev(r0, r1, self.rs, EMB_SALT, EMB_SCALE)

    def gen_lin(self, r0, r1):
        return pattern_dev(r0, r1, 1, LIN_SALT, LIN_SCALE)

    def reset(self):
        fill(self.arena, self.gen)
        if self.lin is not None:
            fill(self.lin.view(-1, 1), self.gen_lin)

    def emb_of(self, g):
        return pattern_np(g, self.rs, EMB_SALT, EMB_SCALE)[:, :self.D]

    def lin_of(self, g):
        if self.fused:
            return pattern_np(g, self.rs, EMB_SALT, EMB_SCALE)[:, self.D]
        return pattern_np(g, 1, LIN_SALT, LIN_SCALE)[:, 0]

    def rows_now(self, g):
        """(emb [n, D], lin [n]) of global rows g as the arena holds them now."""
        gi = torch.from_numpy(np.asarray(g, np.int64)).cuda()
        w = self.arena.index_select(0, gi).cpu().numpy()
        lin = w[:, self.D] if self.fused else self.lin.index_select(0, gi).cpu().numpy()
        return w[:, :self.D], lin

    def changed(self, zero=False):
        gen = (lambda a, b: torch.zeros((b - a, self.rs), device="cuda")) if zero else self.gen
        ch = changed_rows(self.arena, gen)
        if self.lin is not None:
            genl = (lambda a, b: torch.zeros((b - a, 1), device="cuda")) if zero else self.gen_lin
            ch = np.union1d(ch, changed_rows(self.lin.view(-1, 1), genl))
        return ch

    def nbytes(self):
        return self.total * (self.rs + (0 if self.fused else 1)) * 4


def _fwd(tab, ids_t, B, bias):
    S, D = len(tab.rows), tab.D
    outs = Guarded(B * S * D), Guarded(B * D), Guarded(B)
    _call("dr_embed_fm_fwd", tab.tp.data_ptr(), tab.lp.data_ptr(), tab.d_rows.data_ptr(), ids_t.data_ptr(),
          ids_t.element_size(), bias.data_ptr(), B, S, D, tab.rs, tab.lin_stride, tab.flags,
          *(o.t.data_ptr() for o in outs), _st())
    torch.cuda.synchronize()
    return [o.get() for o in outs]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@releases_memory
def test_embedding_kernels_past_2_32(layout):
    D, rs, total, fused = LAYOUTS[layout]
    need(total * (rs + (0 if fused else 1)) * 4, f"the {layout} arena ({total} rows x {rs} floats)")
    tab = Table(D, rs, total, fused)
    assert tab.total * rs > TWO32
    touched, aliases = placed_rows(total, rs)
    rows, offs = tab.rows, tab.offs
    ids = make_ids(touched, rows, offs, seed=D)
    B, S = ids.shape
    comp = Compact(ids, rows, offs, tab.emb_of, tab.lin_of)
    assert np.array_equal(comp.global_rows(), touched)
    bias = torch.tensor([0.375], device="cuda")

    # forward: dr_embed_fm_fwd with int64 and int32 ids
    for dt in (torch.int64, torch.int32):
        ids_t = torch.from_numpy(ids).cuda().to(dt)
        stack, sum_e, logit = _fwd(tab, ids_t, B, bias)
        check_forward(comp, 0.375, stack, sum_e, logit, f"dr_embed_fm_fwd {dt}")
    ids64 = torch.from_numpy(ids).cuda()
    ids32 = ids64.to(torch.int32)

    # dr_embed_fm_fwd_tma (fused D = 16 only; it addresses the one arena with slot offsets)
    if fused and D == 16:
        outs = Guarded(B * S * D), Guarded(B * D), Guarded(B)
        _call("dr_embed_fm_fwd_tma", tab.arena.data_ptr(), total, tab.d_offs.data_ptr(), tab.d_rows.data_ptr(),
              ids32.data_ptr(), 4, bias.data_ptr(), B, S, D, rs, *(o.t.data_ptr() for o in outs), _st())
        torch.cuda.synchronize()
        check_forward(comp, 0.375, *(o.get() for o in outs), "dr_embed_fm_fwd_tma")

    # dr_gather_fwd: the arena as one [total, rs] table, global ids (and OOV), bit for bit
    gids = np.concatenate([touched, touched[::-1], [-1, total, total + 5]]).astype(np.int64)
    out = Guarded(gids.size * rs)
    gt = torch.from_numpy(gids).cuda().to(torch.int32)
    _call("dr_gather_fwd", tab.arena.data_ptr(), total, gt.data_ptr(), 4, gids.size, rs, out.t.data_ptr(), _st())
    torch.cuda.synchronize()
    want = np.zeros((gids.size, rs), F32)
    ok = (gids >= 0) & (gids < total)
    want[ok] = pattern_np(gids[ok], rs, EMB_SALT, EMB_SCALE)
    assert np.array_equal(out.get().view(np.uint32), want.reshape(-1).view(np.uint32)), "dr_gather_fwd"

    # dr_embed_bag_fwd (mean and sum) on the arena, global ids; dr_fnn_input_fwd on the slots
    nb = 6
    splits = np.array([0, 5, 5, 12, 17, 21, gids.size], np.int64)
    ids_b = torch.from_numpy(gids).cuda()
    sp = torch.from_numpy(splits).cuda()
    for comb, name in ((1, "mean"), (0, "sum")):
        out = Guarded(nb * D)
        _call("dr_embed_bag_fwd", tab.arena.data_ptr(), total, rs, ids_b.data_ptr(), 8, sp.data_ptr(), nb, D, comb,
              out.t.data_ptr(), D, _st())
        torch.cuda.synchronize()
        u = np.unique(gids[ok])
        bag_tab = tab.emb_of(u)
        cid = np.where(ok, np.searchsorted(u, np.where(ok, gids, 0)), -1)
        ref = R.embedding_bag(bag_tab.astype(F64), cid, splits, name, F64)
        sc = R.embedding_bag(np.abs(bag_tab.astype(F64)), cid, splits, name, F64)
        err = np.abs(out.get().reshape(nb, D) - ref)
        assert (err <= 1e-5 * sc + 1e-7).all(), f"dr_embed_bag_fwd {name}: max err {err.max()}"
    P = (1 + S + 3) // 4 * 4
    ld = P + S * D
    out = Guarded(B * ld)
    _call("dr_fnn_input_fwd", tab.tp.data_ptr(), tab.lp.data_ptr(), tab.d_rows.data_ptr(), ids64.data_ptr(), 8, rs,
          tab.lin_stride, tab.flags, bias.data_ptr(), B, S, D, ld, out.t.data_ptr(), _st())
    torch.cuda.synchronize()
    x = out.get().reshape(B, ld)
    want = np.zeros((B, ld), F32)
    want[:, 0] = 0.375
    for s in range(S):
        hit = comp.ids[:, s] >= 0
        want[hit, 1 + s] = comp.lins[s][comp.ids[hit, s]]
    want[:, P:] = R.stack_embeddings(comp.tables, comp.ids).reshape(B, S * D)
    assert np.array_equal(x.view(np.uint32), want.view(np.uint32)), "dr_fnn_input_fwd"
    assert not tab.changed().size, "a forward wrote the arena"

    # backward fused with sparse SGD (scale = -lr, gradient pointers = the parameters), int64 ids
    rng = np.random.default_rng(D + 1)
    stack = R.stack_embeddings(comp.tables, comp.ids)
    gl = (rng.standard_normal(B) * 0.5).astype(F32)
    gs = (rng.standard_normal((B, S, D)) * 0.1).astype(F32)
    d_stack, d_gl, d_gs = (torch.from_numpy(a).cuda() for a in (stack, gl, gs))
    lr = 0.05
    emb0, lin0 = tab.rows_now(touched)
    _call("dr_embed_fm_bwd", ids64.data_ptr(), 8, tab.d_rows.data_ptr(), d_stack.data_ptr(), None, d_gl.data_ptr(),
          d_gs.data_ptr(), B, S, D, rs, tab.lin_stride, tab.flags, tab.tp.data_ptr(), tab.lp.data_ptr(), None, -lr,
          _st())
    torch.cuda.synchronize()
    gr = fm_grads(comp, stack, gl.astype(F64), gs.astype(F64))
    emb1, lin1 = tab.rows_now(touched)
    for name, p0, p1, g, sc, terms in (("table", emb0, emb1, gr["g"], gr["sc"], gr["tt"]),
                                       ("first-order", lin0, lin1, gr["gl"], gr["scl"], gr["tl"])):
        hits = gr["hits"].reshape((-1,) + (1,) * (g.ndim - 1))
        rec = (p0.astype(F64) - p1.astype(F64)) / lr
        bound = 1e-5 * sc + 1e-7 + update_slack(p0, p1, lr, hits, terms)
        check_bound(f"fused SGD {name} rows", rec, g, bound)
    assert_only(tab.changed(), touched, "fused SGD")
    if fused:
        pad = tab.arena.index_select(0, torch.from_numpy(touched).cuda())[:, D + 1:].cpu().numpy()
        assert np.array_equal(pad, pattern_np(touched, rs, EMB_SALT, EMB_SCALE)[:, D + 1:]), "row padding changed"

    # dense gradient arena: the same arena zeroed, scale = 1, int32 ids
    tab.arena.zero_()
    if tab.lin is not None:
        tab.lin.zero_()
    _call("dr_embed_fm_bwd", ids32.data_ptr(), 4, tab.d_rows.data_ptr(), d_stack.data_ptr(), None, d_gl.data_ptr(),
          d_gs.data_ptr(), B, S, D, rs, tab.lin_stride, tab.flags, tab.tp.data_ptr(), tab.lp.data_ptr(), None, 1.0,
          _st())
    torch.cuda.synchronize()
    g1, l1 = tab.rows_now(touched)
    check_bound("dense gradient rows", g1, gr["g"], 1e-5 * gr["sc"] + 1e-7)
    check_bound("dense first-order gradient", l1, gr["gl"], 1e-5 * gr["scl"] + 1e-7)
    assert_only(tab.changed(zero=True), touched, "dense gradient")

    # dr_fnn_input_bwd into the zeroed arena (scale = 1), int64 ids
    tab.arena.zero_()
    if tab.lin is not None:
        tab.lin.zero_()
    gx = (rng.standard_normal((B, ld)) * 0.1).astype(F32)
    d_gx = torch.from_numpy(gx).cuda()
    _call("dr_fnn_input_bwd", ids64.data_ptr(), 8, tab.d_rows.data_ptr(), d_gx.data_ptr(), B, S, D, ld, rs,
          tab.lin_stride, tab.flags, tab.tp.data_ptr(), tab.lp.data_ptr(), 1.0, _st())
    torch.cuda.synchronize()
    g_e = gx[:, P:].reshape(B, S, D).astype(F64)
    g_w = gx[:, 1:1 + S].astype(F64)
    gts, _, _ = R.embed_fm_grad(comp.rows, comp.ids, np.zeros((B, S, D)), None, g_e, F64)
    sct, _, _ = R.embed_fm_grad(comp.rows, comp.ids, np.zeros((B, S, D)), None, np.abs(g_e), F64)
    gw = np.concatenate([np.bincount(comp.ids[:, s][comp.ids[:, s] >= 0], g_w[:, s][comp.ids[:, s] >= 0],
                                     minlength=comp.rows[s]) for s in range(S)])
    sw = np.concatenate([np.bincount(comp.ids[:, s][comp.ids[:, s] >= 0], np.abs(g_w[:, s])[comp.ids[:, s] >= 0],
                                     minlength=comp.rows[s]) for s in range(S)])
    g1, l1 = tab.rows_now(touched)
    check_bound("dr_fnn_input_bwd rows", g1, np.concatenate(gts), 1e-5 * np.concatenate(sct) + 1e-7)
    check_bound("dr_fnn_input_bwd first-order", l1, gw, 1e-5 * sw + 1e-7)
    assert_only(tab.changed(zero=True), touched, "dr_fnn_input_bwd")

    # dr_scatter_add (scale 0.5) and dr_embed_bag_bwd (mean, then sum) on the zeroed arena, global ids
    for step in ("scatter", "bag_mean", "bag_sum"):
        tab.arena.zero_()
        if step == "scatter":
            g = (rng.standard_normal((gids.size, rs)) * 0.1).astype(F32)
            d_g = torch.from_numpy(g).cuda()
            _call("dr_scatter_add", tab.arena.data_ptr(), total, gt.data_ptr(), 4, gids.size, rs, d_g.data_ptr(), 0.5,
                  _st())
            ref = np.zeros((touched.size, rs))
            sc = np.zeros((touched.size, rs))
            pos = np.searchsorted(touched, gids[ok])
            np.add.at(ref, pos, 0.5 * g[ok].astype(F64))
            np.add.at(sc, pos, 0.5 * np.abs(g[ok].astype(F64)))
            cols = rs
        else:
            comb, name = (1, "mean") if step == "bag_mean" else (0, "sum")
            g = (rng.standard_normal((nb, D)) * 0.1).astype(F32)
            d_g = torch.from_numpy(g).cuda()
            _call("dr_embed_bag_bwd", ids_b.data_ptr(), 8, sp.data_ptr(), nb, D, comb, d_g.data_ptr(), D, total, rs,
                  tab.arena.data_ptr(), 1.0, _st())
            cid = np.where(ok, np.searchsorted(touched, np.where(ok, gids, 0)), -1)
            ref = R.embedding_bag_grad(touched.size, cid, splits, g.astype(F64), name)
            sc = R.embedding_bag_grad(touched.size, cid, splits, np.abs(g.astype(F64)), name)
            cols = D
        torch.cuda.synchronize()
        got = tab.arena.index_select(0, torch.from_numpy(touched).cuda()).cpu().numpy()
        check_bound(step, got[:, :cols], ref, 1e-5 * sc + 1e-7)
        assert not got[:, cols:].any(), f"{step}: wrote past D"
        ch = changed_rows(tab.arena, lambda a, b: torch.zeros((b - a, rs), device="cuda"))
        assert_only(ch, touched, step)
    assert aliases.size and not np.intersect1d(aliases, touched).size


# ---- 4. dense Adam over 2^31 + 1027 floats -------------------------------------------------------------------------------
N_DENSE = TWO31 + 1027           # odd tail: the scalar loop runs after the float4 one
LR_T, B1, B2, EPS = 1.5e-3, 0.9, 0.999, 1e-7
DENSE_GEN = {  # buffer: (salt, scale); v is made positive below
    "p": (1, 2.0 ** -8), "g": (2, 2.0 ** -10), "m": (3, 2.0 ** -14), "v": (4, 2.0 ** -30)}


def _dense_gen(name, e0, e1):
    salt, scale = DENSE_GEN[name]
    x = pattern_dev(e0, e1, 1, salt, scale).view(-1)
    return (x.abs() + 2.0 ** -30) if name == "v" else x


def _check_dense_adam(bufs, off, n, lr_t_, zero_grad, what):
    """Elements [off, off + n) of each buffer after one ApplyAdam from the pattern, chunk by chunk against float64."""
    o1, o2 = F64(F32(1.0) - F32(B1)), F64(F32(1.0) - F32(B2))
    worst = 0.0
    for e0 in range(0, n, CHUNK // 4):
        e1 = min(n, e0 + CHUNK // 4)
        p0, g0, m0, v0 = (_dense_gen(k, e0, e1).double() for k in "pgmv")
        p1, g1, m1, v1 = (bufs[k][off + e0:off + e1].double() for k in "pgmv")
        rm = m0 + (g0 - m0) * o1
        rv = v0 + (g0 * g0 - v0) * o2
        bm = C_MOMENT * U * (m0.abs() + rm.abs())
        bv = C_MOMENT * U * (v0.abs() + rv.abs())
        dp = F64(F32(lr_t_)) * m1 / (v1.sqrt() + F64(F32(EPS)))
        rp = p0 - dp
        bp = C_FUNCTOR * U * dp.abs() + torch.minimum(U * rp.abs(), dp.abs()) + U64 * rp.abs()
        for name, got, ref, b in (("m", m1, rm, bm), ("v", v1, rv, bv), ("p", p1, rp, bp)):
            err = (got - ref).abs()
            bad = ~(err <= b)
            if bool(bad.any()):
                i = int(bad.nonzero()[0])
                raise AssertionError(f"{what} {name}: {int(bad.sum())} elements outside the bound in [{off + e0}, "
                                     f"{off + e1}); first at {off + e0 + i}: got {float(got[i])!r} want "
                                     f"{float(ref[i])!r} bound {float(b[i])!r}")
            worst = max(worst, float((err / b.clamp_min(1e-300)).max()))
        if zero_grad:
            assert not bool(g1.any()), f"{what}: gradient not cleared in [{off + e0}, {off + e1})"
        else:
            assert torch.equal(g1, g0), f"{what}: gradient changed in [{off + e0}, {off + e1})"
    return worst


@releases_memory
def test_dense_adam_past_2_31():
    """dr_adam_step on n = 2^31 + 1027 (aligned, then a view one float in: scalar path throughout) and
    dr_adam_step_multi with that tensor between small ones.  The largest test (~34.4 GB): the first to skip on a
    busy GPU."""
    need(4 * (N_DENSE + 4) * 4, "four Adam buffers of 2^31 + 1031 floats (the largest test here)")
    bufs = {k: torch.empty(N_DENSE + 4, device="cuda") for k in "pgmv"}

    def refill(off):
        for k in "pgmv":
            fill(bufs[k][off:off + N_DENSE].view(-1, 1), lambda a, b, k=k: _dense_gen(k, a, b).view(-1, 1))
            bufs[k][:off].fill_(SENT)
            bufs[k][off + N_DENSE:].fill_(SENT)

    def guards(off):
        for k in "pgmv":
            rest = torch.cat([bufs[k][:off], bufs[k][off + N_DENSE:]])
            assert bool((rest == SENT).all()), f"{k}: a store outside the tensor"

    report = {}
    for off, zero in ((0, 1), (1, 0)):      # off = 1: no pointer is 16-B aligned
        refill(off)
        _call("dr_adam_step", *(bufs[k].data_ptr() + 4 * off for k in "pgmv"), N_DENSE, LR_T, B1, B2, EPS, zero, None,
              _st())
        torch.cuda.synchronize()
        report[f"adam_step off {off}"] = _check_dense_adam(bufs, off, N_DENSE, LR_T, zero, f"dr_adam_step off={off}")
        guards(off)

    import ctypes as C
    refill(0)
    smalls = [[torch.randn(5, device="cuda") for _ in range(4)], [torch.randn(1028, device="cuda")[1:] for _ in range(4)]]
    for s4 in smalls:
        s4[3].abs_()
    want = [[x.clone() for x in s4] for s4 in smalls]
    for s4 in want:
        _call("dr_adam_step", *(x.data_ptr() for x in s4), s4[0].numel(), LR_T, B1, B2, EPS, 0, None, _st())
    tensors = [smalls[0], [bufs[k][:N_DENSE] for k in "pgmv"], smalls[1]]
    arr = lambda j: (C.c_void_p * 3)(*[t4[j].data_ptr() for t4 in tensors])
    ns = (C.c_int64 * 3)(*[t4[0].numel() for t4 in tensors])
    _call("dr_adam_step_multi", 3, arr(0), arr(1), arr(2), arr(3), ns, LR_T, B1, B2, EPS, None, _st())
    torch.cuda.synchronize()
    report["adam_step_multi"] = _check_dense_adam(bufs, 0, N_DENSE, LR_T, False, "dr_adam_step_multi")
    guards(0)
    for s4, w4 in zip(smalls, want):
        for x, y in zip(s4, w4):
            assert torch.equal(x, y), "dr_adam_step_multi: a small tensor differs from dr_adam_step"
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- 3. row-sparse, TensorFlow-exact Adam on state blocks past 2^32 floats ------------------------------------------------
ADAM_D, ADAM_ROWS, HIST, LR = 16, 67_200_000, 16, 0.01
GAPS = (1, 3, K_CATCH_UP_MAX + 52, 0, 17)     # steps a touched row sat out (0: never updated, stamp 0)


def state_gen(D, SS, r0, r1):
    """State blocks [g D | m D | v D | g_w m_w v_w count stamp | pad] of rows r0 .. r1: m ~ 2^-13 and v ~ m^2 (so every
    replayed step moves p by about lr_j); g, count and stamp zero."""
    r = torch.arange(r0, r1, dtype=torch.int64, device="cuda")[:, None]
    c = torch.arange(SS, device="cuda")[None, :]
    k = _key(r, c, 3)
    m = (k - 4095).to(torch.float32) * 2.0 ** -24
    v = ((k % 97) + 32).to(torch.float32) * 2.0 ** -34
    zero = (c < D) | (c == 3 * D) | (c == 3 * D + 3) | (c == 3 * D + 4)
    is_v = ((c >= 2 * D) & (c < 3 * D)) | (c == 3 * D + 2)
    return torch.where(zero, torch.zeros_like(m), torch.where(is_v, v, m))


class AdamState:
    """The fused D = 16 table (row stride 32: 2^31 + 6.4 M floats) and its state blocks (stride 64: 2^32 + 12.8 M)."""

    def __init__(self):
        D = ADAM_D
        self.tab = Table(D, 32, ADAM_ROWS, True)
        self.SS = SS = _lib().load().dr_embed_adam_state_stride(D)
        assert SS == 64 and ADAM_ROWS * SS > TWO32
        self.state = torch.empty((ADAM_ROWS, SS), device="cuda")
        fill(self.state, self.gen)
        self.step = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.lr_t = torch.zeros(1, device="cuda")
        self.hist = torch.zeros(HIST, device="cuda")

    def gen(self, r0, r1):
        return state_gen(ADAM_D, self.SS, r0, r1)

    def advance(self, n=1):
        for _ in range(n):
            _call("dr_adam_advance_hist", self.step.data_ptr(), LR, B1, B2, self.lr_t.data_ptr(), self.hist.data_ptr(),
                  HIST, _st())
        torch.cuda.synchronize()
        return int(self.step)

    def set_stamps(self, rows, stamps):
        gi = torch.from_numpy(rows).cuda()
        self.state.view(torch.int32)[gi, 3 * ADAM_D + 4] = torch.from_numpy(np.asarray(stamps, np.int32)).cuda()

    def snap(self, rows):
        D = ADAM_D
        gi = torch.from_numpy(rows).cuda()
        w = self.tab.arena.index_select(0, gi).cpu().numpy()
        st = self.state.index_select(0, gi).cpu().numpy()
        cat = lambda a, b: np.concatenate([a, b], 1).astype(F64)
        return dict(p=cat(w[:, :D], w[:, D:D + 1]), m=cat(st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]),
                    v=cat(st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]), g=cat(st[:, :D], st[:, 3 * D:3 * D + 1]),
                    stamp=st[:, 3 * D + 4].view(np.int32).astype(np.int64), count=st[:, 3 * D + 3].view(np.int32))

    def common(self, lin_ptrs=True):
        """The layer API's entries take no first-order pointers when the weight is in the row."""
        t = self.tab
        return (t.d_rows.data_ptr(), t.d_offs.data_ptr(), t.rs, t.lin_stride, t.flags, t.tp.data_ptr(),
                t.lp.data_ptr() if lin_ptrs else None, self.state.data_ptr())

    def untouched(self, touched, what):
        assert_only(changed_rows(self.tab.arena, self.tab.gen), touched, f"{what}: table")
        assert_only(changed_rows(self.state, self.gen), touched, f"{what}: state")


def _replayed(name, h0, h1, upto, t_now, report):
    rp, rm, rv, bp, bm, bv = replay(h0["p"], h0["m"], h0["v"], h0["stamp"], upto, LR, B1, B2, EPS, t_now=t_now,
                                    hist_len=HIST)
    for k, ref, b in (("p", rp, bp), ("m", rm, bm), ("v", rv, bv)):
        report[f"{name} {k}"] = check_bound(f"{name} {k}", h1[k], ref, b)


def _stepped(name, h0, h1, e, hits, lr_t_, report):
    extra = U * e.terms + update_slack(0, 0, 1, hits[:, None], e.terms)
    m1, bm, v1, bv = moments(h0["m"], h0["v"], e, extra, B1, B2)
    report[f"{name} m"] = check_bound(f"{name} m", h1["m"], m1, bm)
    report[f"{name} v"] = check_bound(f"{name} v", h1["v"], v1, bv)
    p1, bp = functor(h0["p"], h1["m"], h1["v"], F64(lr_t_), EPS)
    report[f"{name} p"] = check_bound(f"{name} p", h1["p"], p1, bp)
    assert not h1["g"].any() and not h1["count"].any(), f"{name}: gradient slots or countdowns not cleared"


@releases_memory
def test_row_sparse_adam_state_past_2_32():
    """dr_embed_adam_prepare + dr_embed_fm_bwd_adam_tf (the trainer's step), dr_embed_adam_catch_up +
    dr_embed_adam_count + dr_embed_adam_rows_tf (the layer API's step) and dr_embed_adam_flush, on rows that sat out
    1, 3, kCatchUpMax + 52 and 17 steps or were never updated, at state offsets across 2^31 and 2^32."""
    need(ADAM_ROWS * (32 + 64) * 4, f"a {ADAM_ROWS}-row D = 16 table with its Adam state blocks")
    D = ADAM_D
    a = AdamState()
    touched = np.union1d(placed_rows(ADAM_ROWS, a.SS)[0], placed_rows(ADAM_ROWS, 32)[0])
    rows, offs = a.tab.rows, a.tab.offs
    gaps = np.array([GAPS[k % len(GAPS)] for k in range(touched.size)])
    report = {}

    # the trainer's step t0: prepare (replay to t0 - 1, count), backward with the update; int32 then int64 ids
    a.step.fill_(3000 - HIST)
    a.advance(HIST - 1)
    for k, dt in enumerate((torch.int32, torch.int64)):
        t0 = a.advance()
        a.set_stamps(touched, np.where(gaps > 0, t0 - 1 - gaps, 0))          # prepare replays `gaps` steps
        ids = make_ids(touched, rows, offs, seed=k + 1)
        B, S = ids.shape
        comp = Compact(ids, rows, offs, a.tab.emb_of, a.tab.lin_of)
        ids_t = torch.from_numpy(ids).cuda().to(dt)
        h0 = a.snap(touched)
        _call("dr_embed_adam_prepare", ids_t.data_ptr(), ids_t.element_size(), B, S, D, *a.common(), a.step.data_ptr(), a.hist.data_ptr(),
              HIST, LR, B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h1 = a.snap(touched)
        _replayed("prepare", h0, h1, t0 - 1, t0, report)
        hits = np.concatenate([np.bincount(comp.ids[:, s][comp.ids[:, s] >= 0], minlength=comp.rows[s]) for s in range(S)])
        assert np.array_equal(h1["count"], hits), "dr_embed_adam_prepare: count != lookups per row"
        a.untouched(touched, "dr_embed_adam_prepare")

        rng = np.random.default_rng(7 + k)
        ok = comp.ids >= 0
        stack = (np.round(rng.uniform(-1, 1, (B, S, D)) * 256) / 256 * ok[:, :, None]).astype(F32)
        gl = (np.round(rng.uniform(-1, 1, B) * 2 ** 8) / 2 ** 14).astype(F32)
        gs = (rng.standard_normal((B, S, D)) * 1e-2).astype(F32)
        sum_e = stack.sum(1, dtype=F32)
        dev = [torch.from_numpy(x).cuda() for x in (stack, sum_e, gl, gs)]
        g_bias = torch.zeros(1, device="cuda")
        _call("dr_embed_fm_bwd_adam_tf", ids_t.data_ptr(), ids_t.element_size(), a.tab.d_rows.data_ptr(), a.tab.d_offs.data_ptr(),
              *(x.data_ptr() for x in dev), B, S, D, a.tab.rs, a.tab.lin_stride, a.tab.flags, a.tab.tp.data_ptr(),
              a.tab.lp.data_ptr(), a.state.data_ptr(), g_bias.data_ptr(), a.step.data_ptr(), a.lr_t.data_ptr(),
              a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h2 = a.snap(touched)
        gr = fm_grads(comp, stack, gl.astype(F64), gs.astype(F64))
        e = Entry(np.concatenate([gr["g"], gr["gl"][:, None]], 1), 0.0, 0.0,
                  np.concatenate([gr["tt"], gr["tl"][:, None]], 1))
        _stepped("bwd_adam_tf", h1, h2, e, hits, float(a.lr_t), report)
        assert (h2["stamp"] == t0).all()
        a.untouched(touched, "dr_embed_fm_bwd_adam_tf")

    # the layer API two steps later: catch up to the last completed step, then step t with per-lookup gradient rows; int64 then int32 ids
    for k, dt in enumerate((torch.int64, torch.int32)):
        t_last = a.advance(2)
        a.set_stamps(touched, np.where(gaps > 0, t_last - gaps + 1, 0))
        ids = make_ids(touched, rows, offs, seed=k + 3, dup=(3, 1, 2))
        B, S = ids.shape
        comp = Compact(ids, rows, offs, a.tab.emb_of, a.tab.lin_of)
        ids_t = torch.from_numpy(ids).cuda().to(dt)
        h0 = a.snap(touched)
        _call("dr_embed_adam_catch_up", ids_t.data_ptr(), ids_t.element_size(), B * S, S, D, *a.common(lin_ptrs=False), a.step.data_ptr(),
              a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h1 = a.snap(touched)
        _replayed("catch_up", h0, h1, t_last, t_last, report)
        t = a.advance()
        _call("dr_embed_adam_count", ids_t.data_ptr(), ids_t.element_size(), B, S, D, a.tab.d_rows.data_ptr(), a.tab.d_offs.data_ptr(),
              a.state.data_ptr(), _st())
        ge = (rng.standard_normal((B, S, D)) * 1e-2).astype(F32)
        gw = (rng.standard_normal((B, S)) * 1e-2).astype(F32)
        d_ge, d_gw = torch.from_numpy(ge).cuda(), torch.from_numpy(gw).cuda()
        _call("dr_embed_adam_rows_tf", ids_t.data_ptr(), ids_t.element_size(), B * S, B, S, None, a.tab.d_rows.data_ptr(),
              a.tab.d_offs.data_ptr(), d_ge.data_ptr(), S * D, D, d_gw.data_ptr(), S, 1, D, a.tab.rs, a.tab.lin_stride,
              a.tab.flags, a.tab.tp.data_ptr(), None, a.state.data_ptr(), a.step.data_ptr(),
              a.lr_t.data_ptr(), a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h2 = a.snap(touched)
        z = np.zeros((B, S, D))
        gts, _, _ = R.embed_fm_grad(comp.rows, comp.ids, z, None, ge.astype(F64), F64)
        tts, _, _ = R.embed_fm_grad(comp.rows, comp.ids, z, None, np.abs(ge.astype(F64)), F64)
        per_w = lambda w: np.concatenate([np.bincount(comp.ids[:, s][comp.ids[:, s] >= 0], w[:, s][comp.ids[:, s] >= 0],
                                                      minlength=comp.rows[s]) for s in range(S)])
        e = Entry(np.concatenate([np.concatenate(gts), per_w(gw.astype(F64))[:, None]], 1), 0.0, 0.0,
                  np.concatenate([np.concatenate(tts), per_w(np.abs(gw.astype(F64)))[:, None]], 1))
        hits = per_w(np.ones((B, S))).astype(np.int64)
        _stepped("rows_tf", h1, h2, e, hits, float(a.lr_t), report)
        assert (h2["stamp"] == t).all()
        a.untouched(touched, "dr_embed_adam_rows_tf")

    # flush three steps on: every row with a stamp in (0, t) replays up to t -- only the touched rows have one
    t = a.advance(3)
    a.set_stamps(touched, np.where(gaps > 0, t - gaps, 0))
    h0 = a.snap(touched)
    _call("dr_embed_adam_flush", a.tab.d_rows.data_ptr(), a.tab.d_offs.data_ptr(), S, D, ADAM_ROWS, a.tab.rs,
          a.tab.lin_stride, a.tab.flags, a.tab.tp.data_ptr(), a.tab.lp.data_ptr(), a.state.data_ptr(),
          a.step.data_ptr(), a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _st())
    torch.cuda.synchronize()
    h1 = a.snap(touched)
    _replayed("flush", h0, h1, t, t, report)
    assert (h1["stamp"][gaps > 0] == t).all() and (h1["stamp"][gaps == 0] == 0).all()
    a.untouched(touched, "dr_embed_adam_flush")
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- 5. the row-sharded owner arenas (emulated worlds on one GPU, as test_gpu_sharded_emulated.py) -----------------------
SHARD_D = 128
SHARD_WORLDS = {1: (1 << 25) + 64,              # one owner of 2^32 + 8192 floats (+ its first-order weights)
                2: 2 * ((1 << 24) + 64) + 1}    # two owners of 2^31 + 8320 floats and more: owner = row mod 2


class Shards:
    """`world` owner allocations in the p2p layout (shard_plan.p2p_layout: wide rows of D floats, then the [max_rows]
    first-order weights); global row r lives on owner r % world at local row r // world and holds pattern(r)."""

    def __init__(self, total, world):
        from deep_recommenders_b200 import shard_plan
        D = SHARD_D
        self.total, self.world = total, world
        self.lay = lay = shard_plan.p2p_layout(total, D, world)
        assert lay.vdim == D and not lay.lin_in_row and lay.max_rows * D > (TWO32 if world == 1 else TWO31)
        self.nloc = [shard_plan.local_rows(total, g, world) for g in range(world)]
        self.bufs = [torch.empty(lay.numel, device="cuda") for _ in range(world)]
        for g in range(world):
            fill(self.emb(g), functools.partial(self.gen, g))
            fill(self.lin(g), functools.partial(self.gen_lin, g))
        self.peer = torch.tensor([b.data_ptr() for b in self.bufs], dtype=torch.int64, device="cuda")
        self.rows, self.offs = slot_plan(total)
        self.d_rows = torch.tensor(self.rows, dtype=torch.int64, device="cuda")
        self.d_offs = torch.from_numpy(self.offs).cuda()

    def emb(self, g):
        return self.bufs[g][:self.lay.max_rows * SHARD_D].view(-1, SHARD_D)

    def lin(self, g):
        return self.bufs[g][self.lay.lin_offset:self.lay.lin_offset + self.lay.max_rows].view(-1, 1)

    def gen(self, g, r0, r1):
        return pattern_dev(r0, r1, SHARD_D, EMB_SALT, EMB_SCALE, mul=self.world, add=g)

    def gen_lin(self, g, r0, r1):
        return pattern_dev(r0, r1, 1, LIN_SALT, LIN_SCALE, mul=self.world, add=g)

    def rows_now(self, rows):
        emb = np.empty((rows.size, SHARD_D), F32)
        lin = np.empty(rows.size, F32)
        for g in range(self.world):
            sel = rows % self.world == g
            li = torch.from_numpy(rows[sel] // self.world).cuda()
            emb[sel] = self.emb(g).index_select(0, li).cpu().numpy()
            lin[sel] = self.lin(g).index_select(0, li).cpu().numpy()[:, 0]
        return emb, lin

    def changed(self):
        out = []
        for g in range(self.world):
            for view, gen in ((self.emb(g), self.gen), (self.lin(g), self.gen_lin)):
                out.append(changed_rows(view, functools.partial(gen, g)) * self.world + g)
        return np.unique(np.concatenate(out))


@pytest.mark.parametrize("world", list(SHARD_WORLDS), ids=[f"w{w}" for w in SHARD_WORLDS])
@releases_memory
def test_sharded_owner_arenas_past_2_31(world):
    """dr_shard_bucket_ids, dr_embed_fm_fwd_sharded and dr_embed_fm_bwd_sharded (fused SGD into the owners) at D = 128
    with the first-order weights trailing each owner's rows."""
    from deep_recommenders_b200 import shard_plan
    total = SHARD_WORLDS[world]
    D = SHARD_D
    lay = shard_plan.p2p_layout(total, D, world)
    need(world * lay.numel * 4, f"{world} owner arena(s) of {lay.numel} floats")
    sh = Shards(total, world)
    touched = np.unique(np.concatenate([
        placed_rows(lay.max_rows, D)[0] * world + g for g in range(world)]))
    touched = touched[touched < total]
    assert touched.max() == total - 1 or world > 1
    ids = make_ids(touched, sh.rows, sh.offs, seed=world)
    B, S = ids.shape
    comp = Compact(ids, sh.rows, sh.offs, lambda r: pattern_np(r, D, EMB_SALT, EMB_SCALE),
                   lambda r: pattern_np(r, 1, LIN_SALT, LIN_SCALE)[:, 0])
    assert np.array_equal(comp.global_rows(), touched)
    bias = torch.tensor([0.375], device="cuda")

    # bucketing: every valid lookup goes to owner row % world as local row row // world
    ids32 = torch.from_numpy(ids).cuda().to(torch.int32)
    n, cap = B * S, B * S
    counts = torch.zeros(world, dtype=torch.int64, device="cuda")
    send = torch.full((world * cap,), -7, dtype=torch.int64, device="cuda")
    inv = torch.zeros(n, dtype=torch.int32, device="cuda")
    over = torch.zeros(1, dtype=torch.int32, device="cuda")
    _call("dr_shard_bucket_ids", ids32.data_ptr(), 4, n, S, sh.d_offs.data_ptr(), sh.d_rows.data_ptr(), world, cap,
          counts.data_ptr(), send.data_ptr(), inv.data_ptr(), over.data_ptr(), _st())
    torch.cuda.synchronize()
    from oracle import shard_np
    o_send, o_inv, o_counts, o_over = shard_np.bucket_ids(ids, sh.offs, sh.rows, world, cap)
    inv_h, send_h = inv.cpu().numpy().astype(np.int64), send.cpu().numpy()
    assert int(over) == int(o_over) == 0 and np.array_equal(counts.cpu().numpy(), o_counts)
    sent = o_inv >= 0                    # order inside a segment is unspecified: compare owner and local row per lookup
    assert np.array_equal(inv_h < 0, ~sent), "OOV lookups must send nothing"
    assert np.array_equal(inv_h[sent] // cap, o_inv[sent] // cap), "lookup sent to the wrong owner"
    assert np.array_equal(send_h[inv_h[sent]], o_send[o_inv[sent]]), "wrong local row in the send buffer"

    # forward, int64 and int32 ids
    for ids_t in (torch.from_numpy(ids).cuda(), ids32):
        outs = Guarded(B * S * D), Guarded(B * D), Guarded(B)
        _call("dr_embed_fm_fwd_sharded", sh.peer.data_ptr(), world, sh.d_offs.data_ptr(), sh.d_rows.data_ptr(),
              ids_t.data_ptr(), ids_t.element_size(), bias.data_ptr(), B, S, D, lay.vdim, 0, lay.lin_offset,
              *(o.t.data_ptr() for o in outs), _st())
        torch.cuda.synchronize()
        check_forward(comp, 0.375, *(o.get() for o in outs), f"dr_embed_fm_fwd_sharded {ids_t.dtype}")
    assert not sh.changed().size, "the forward wrote an owner arena"

    # backward fused with SGD into the owners' rows and first-order weights
    rng = np.random.default_rng(world)
    stack = R.stack_embeddings(comp.tables, comp.ids)
    gl = (rng.standard_normal(B) * 0.5).astype(F32)
    gs = (rng.standard_normal((B, S, D)) * 0.1).astype(F32)
    d_stack, d_gl, d_gs = (torch.from_numpy(a).cuda() for a in (stack, gl, gs))
    lr = 0.05
    emb0, lin0 = sh.rows_now(touched)
    _call("dr_embed_fm_bwd_sharded", sh.peer.data_ptr(), world, sh.d_offs.data_ptr(), sh.d_rows.data_ptr(),
          ids32.data_ptr(), 4, d_stack.data_ptr(), None, d_gl.data_ptr(), d_gs.data_ptr(), B, S, D, lay.vdim, 0,
          lay.lin_offset, None, -lr, _st())
    torch.cuda.synchronize()
    gr = fm_grads(comp, stack, gl.astype(F64), gs.astype(F64))
    emb1, lin1 = sh.rows_now(touched)
    for name, p0, p1, g, sc, terms in (("table", emb0, emb1, gr["g"], gr["sc"], gr["tt"]),
                                       ("first-order", lin0, lin1, gr["gl"], gr["scl"], gr["tl"])):
        hits = gr["hits"].reshape((-1,) + (1,) * (g.ndim - 1))
        rec = (p0.astype(F64) - p1.astype(F64)) / lr
        check_bound(f"sharded SGD {name} rows", rec, g, 1e-5 * sc + 1e-7 + update_slack(p0, p1, lr, hits, terms))
    assert_only(sh.changed(), touched, "dr_embed_fm_bwd_sharded")


# ---- 3b. dr_lazy_adam_rows: four arenas of just past 2^31 floats ---------------------------------------------------------
LAZY_D, LAZY_RS, LAZY_ROWS = 16, 20, 107_400_000        # [emb 16 | w | pad 3]: 2^31 + 0.5 M floats per arena


def _lazy_gen(name, r0, r1):
    k = _key(torch.arange(r0, r1, dtype=torch.int64, device="cuda")[:, None],
             torch.arange(LAZY_RS, device="cuda")[None, :], {"p": EMB_SALT, "m": 3, "v": 4}[name])
    if name == "p":
        return (k - 4095).to(torch.float32) * EMB_SCALE
    if name == "m":
        return (k - 4095).to(torch.float32) * 2.0 ** -24
    return ((k % 97) + 32).to(torch.float32) * 2.0 ** -34


@releases_memory
def test_lazy_adam_rows_past_2_31():
    """Two steps (int64, then int32 ids) of dr_lazy_adam_rows on p, g, m, v arenas of 107.4 M rows x 20 floats."""
    D, rs, total = LAZY_D, LAZY_RS, LAZY_ROWS
    assert total * rs > TWO31
    need(4 * total * rs * 4 + total * 4, "four lazy-Adam arenas of 2^31 + 0.5 M floats and the stamps")
    ar = {k: torch.empty((total, rs), device="cuda") for k in "pgmv"}
    for k in "pmv":
        fill(ar[k], functools.partial(_lazy_gen, k))
    ar["g"].zero_()
    stamp = torch.zeros(total, dtype=torch.int32, device="cuda")
    touched = placed_rows(total, rs)[0]
    rows, offs = slot_plan(total)
    d_rows, d_offs = torch.tensor(rows, dtype=torch.int64, device="cuda"), torch.from_numpy(offs).cuda()
    gi = torch.from_numpy(touched).cuda()
    step, lr_dev = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, device="cuda")
    rng = np.random.default_rng(11)
    report = {}
    for k, dt in enumerate((torch.int64, torch.int32)):
        _call("dr_adam_advance", step.data_ptr(), LR, B1, B2, lr_dev.data_ptr(), _st())
        ids = make_ids(touched, rows, offs, seed=20 + k)
        ids_t = torch.from_numpy(ids).cuda().to(dt)
        # the gradient arena holds the batch's row gradients (summed over duplicates) and zeros elsewhere
        g = np.zeros((touched.size, rs), F32)
        g[:, :D + 1] = rng.standard_normal((touched.size, D + 1)) * 1e-2
        ar["g"].index_copy_(0, gi, torch.from_numpy(g).cuda())
        snap = lambda: {n: ar[n].index_select(0, gi).cpu().numpy().astype(F64) for n in "pmv"}
        h0 = snap()
        _call("dr_lazy_adam_rows", ids_t.data_ptr(), ids_t.element_size(), ids.shape[0], len(rows), D,
              d_rows.data_ptr(), d_offs.data_ptr(), *(ar[n].data_ptr() for n in "pgmv"), rs, LIN_IN_ROW, None, None,
              None, None, stamp.data_ptr(), step.data_ptr(), lr_dev.data_ptr(), B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h1 = snap()
        c = slice(0, D + 1)
        m1, bm, v1, bv = moments(h0["m"][:, c], h0["v"][:, c], Entry(g[:, c].astype(F64), 0.0, 0.0), 0.0, B1, B2)
        report[f"m {dt}"] = check_bound("lazy m", h1["m"][:, c], m1, bm)
        report[f"v {dt}"] = check_bound("lazy v", h1["v"][:, c], v1, bv)
        p1, bp = functor(h0["p"][:, c], h1["m"][:, c], h1["v"][:, c], F64(float(lr_dev)), EPS)
        report[f"p {dt}"] = check_bound("lazy p", h1["p"][:, c], p1, bp)
        for n in "pmv":
            assert np.array_equal(h1[n][:, D + 1:], h0[n][:, D + 1:]), f"row padding of {n} changed"
        assert not bool(ar["g"].any()), "gradient arena not cleared"
        st = stamp.cpu().numpy()
        assert (st[touched] == int(step)).all() and np.count_nonzero(st) == touched.size, "stamps"
        # the touched rows' p, m, v are now the kernel's: regenerate the rest from the pattern
        for n in "pmv":
            assert_only(changed_rows(ar[n], functools.partial(_lazy_gen, n)), touched, f"dr_lazy_adam_rows: {n}")
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- 5b. the sharded TensorFlow-exact Adam: mark, prepare (list + replay), apply -----------------------------------------
@releases_memory
def test_sharded_adam_owner_state_past_2_32():
    """dr_shard_adam_mark / _prepare / _apply at world 1 (owner = 0, local row = global row) on a D = 16 shard of
    67.2 M rows x 20 floats ([emb | w | pad], first-order weight in the row) whose state blocks pass 2^32 floats.  Two
    steps, int32 then int64 ids; the touched rows sat out 1, 3, 17 and kCatchUpMax + 52 steps or were never updated."""
    D, rs, total, W = ADAM_D, 20, ADAM_ROWS, 1
    SS = _lib().load().dr_embed_adam_state_stride(D)
    need(total * (2 * rs + SS + 2) * 4, f"a {total}-row D = 16 owner shard, its gradient arena and state blocks")
    shard = torch.empty((total, rs), device="cuda")
    gen_p = lambda r0, r1: pattern_dev(r0, r1, rs, EMB_SALT, EMB_SCALE)
    fill(shard, gen_p)
    grad = torch.zeros((total, rs), device="cuda")
    gen_st = functools.partial(state_gen, D, SS)
    state = torch.empty((total, SS), device="cuda")
    fill(state, gen_st)
    i32 = dict(dtype=torch.int32, device="cuda")
    touch, lst, count = torch.zeros(total, **i32), torch.zeros(total, **i32), torch.zeros(1, **i32)
    touch_peer = torch.tensor([touch.data_ptr()], dtype=torch.int64, device="cuda")
    step, lr_t_ = torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, device="cuda")
    hist = torch.zeros(HIST, device="cuda")
    step.fill_(3000 - HIST)
    for _ in range(HIST - 1):
        _call("dr_adam_advance_hist", step.data_ptr(), LR, B1, B2, lr_t_.data_ptr(), hist.data_ptr(), HIST, _st())
    touched = np.union1d(placed_rows(total, SS)[0], placed_rows(total, rs)[0])
    gi = torch.from_numpy(touched).cuda()
    gaps = np.array([GAPS[k % len(GAPS)] for k in range(touched.size)])
    rows, offs = slot_plan(total)
    d_rows, d_offs = torch.tensor(rows, dtype=torch.int64, device="cuda"), torch.from_numpy(offs).cuda()

    def snap():
        w = shard.index_select(0, gi).cpu().numpy()
        st = state.index_select(0, gi).cpu().numpy()
        cat = lambda x, y: np.concatenate([x, y], 1).astype(F64)
        return dict(p=cat(w[:, :D], w[:, D:D + 1]), m=cat(st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]),
                    v=cat(st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]), g=cat(st[:, :D], st[:, 3 * D:3 * D + 1]),
                    stamp=st[:, 3 * D + 4].view(np.int32).astype(np.int64), count=st[:, 3 * D + 3].view(np.int32),
                    pad=w[:, D + 1:])

    rng = np.random.default_rng(13)
    report = {}
    for k, dt in enumerate((torch.int32, torch.int64)):
        _call("dr_adam_advance_hist", step.data_ptr(), LR, B1, B2, lr_t_.data_ptr(), hist.data_ptr(), HIST, _st())
        torch.cuda.synchronize()
        t = int(step)
        state.view(torch.int32)[gi, 3 * D + 4] = torch.from_numpy(np.where(gaps > 0, t - 1 - gaps, 0).astype(
            np.int32)).cuda()
        ids = make_ids(touched, rows, offs, seed=30 + k)
        ids_t = torch.from_numpy(ids).cuda().to(dt)
        h0 = snap()
        _call("dr_shard_adam_mark", ids_t.data_ptr(), ids_t.element_size(), ids.size, len(rows), d_offs.data_ptr(),
              d_rows.data_ptr(), W, touch_peer.data_ptr(), step.data_ptr(), _st())
        torch.cuda.synchronize()
        assert np.array_equal((touch == t).nonzero().flatten().cpu().numpy(), touched), "mark: wrong touch marks"
        count.zero_()
        _call("dr_shard_adam_prepare", touch.data_ptr(), total, lst.data_ptr(), count.data_ptr(), D, rs, 0,
              LIN_IN_ROW, shard.data_ptr(), state.data_ptr(), step.data_ptr(), hist.data_ptr(), HIST, LR, B1, B2, EPS,
              _st())
        torch.cuda.synchronize()
        n = int(count)
        assert np.array_equal(np.sort(lst[:n].cpu().numpy()), touched), "prepare listed other rows than the marked ones"
        h1 = snap()
        _replayed(f"shard prepare {dt}", h0, h1, t - 1, t, report)
        assert_only(changed_rows(shard, gen_p), touched, "dr_shard_adam_prepare: shard")
        assert_only(changed_rows(state, gen_st), touched, "dr_shard_adam_prepare: state")
        # the backward's red.add into the owner's gradient arena, stood in for by the row gradients themselves
        g = np.zeros((touched.size, rs), F32)
        g[:, :D + 1] = rng.standard_normal((touched.size, D + 1)) * 1e-2
        grad.index_copy_(0, gi, torch.from_numpy(g).cuda())
        _call("dr_shard_adam_apply", lst.data_ptr(), count.data_ptr(), total, D, rs, 0, LIN_IN_ROW, shard.data_ptr(),
              grad.data_ptr(), state.data_ptr(), step.data_ptr(), lr_t_.data_ptr(), B1, B2, EPS, _st())
        torch.cuda.synchronize()
        h2 = snap()
        _stepped(f"shard apply {dt}", h1, h2, Entry(g[:, :D + 1].astype(F64), 0.0, 0.0), np.ones(touched.size),
                 float(lr_t_), report)
        assert (h2["stamp"] == t).all() and np.array_equal(h2["pad"], h0["pad"])
        assert not bool(grad.any()), "apply left a gradient row behind"
        assert_only(changed_rows(shard, gen_p), touched, "dr_shard_adam_apply: shard")
        assert_only(changed_rows(state, gen_st), touched, "dr_shard_adam_apply: state")
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- 6. one whole DeepFMTrainStep on tables past 2^32 floats --------------------------------------------------------------
C5_SLOTS, C5_ROWS, C5_B = 26, 1_291_000, 2048         # 26 x 1.291 M rows x 128 floats = 2^32 + 1.5 M floats


def _steered_ids(rng, rows, offs, touched, B):
    """[B, S] ids: the placed rows (by slot), the top 2000 rows of every slot and the last slot's last rows, with OOV
    ids of both kinds; the placed rows several times each."""
    S = len(rows)
    ids = np.stack([rng.integers(max(0, r - 2000), r + 1, B) for r in rows], 1).astype(np.int64)
    ids[rng.random((B, S)) < 0.03] = -1
    ids[:, S - 1] = np.where(rng.random(B) < 0.5, rows[-1] - 1 - rng.integers(0, 3, B), ids[:, S - 1])
    b = 0
    for r in touched:
        s = int(np.searchsorted(offs, r, side="right") - 1)
        for _ in range(3):
            ids[b % B, s] = r - offs[s]
            b += 1
    return ids


@pytest.mark.parametrize("case", ["sgd_graph", "sgd_eager", "adam_rows_tf"])
@releases_memory
def test_train_step_on_tables_past_2_32(case):
    """sgd_*: split D = 128, 26 slots of 1.291 M rows (C5's tower [512, 256], B = 2048), lr = 1, the step as captured
    graph and eagerly; loss, forward values, tower gradients and updates and every touched row held to
    tests/deepfm_oracle.py at the bounds of test_gpu_deepfm_train_step.py.  adam_rows_tf: one step (t = 1) on the fused
    D = 16 table of 67.2 M rows, whose state blocks pass 2^32 floats; the touched rows' m, v and p held to adam_oracle."""
    from deepfm_oracle import check, deepfm_step
    from test_gpu_deepfm_train_step import _trainer, npy
    adam = case == "adam_rows_tf"
    if adam:
        D, rows, units, B = ADAM_D, slot_plan(ADAM_ROWS)[0], [64, 32], 512
        need(2 * ADAM_ROWS * (32 + 64) * 4 + GiB, "a 67.2 M-row D = 16 table, its Adam state and capture()'s snapshot of both")
    else:
        D, rows, units, B = 128, [C5_ROWS] * C5_SLOTS, [512, 256], C5_B
        need(2 * sum(rows) * 129 * 4 + GiB, "a C5-shaped split D = 128 table of 2^32 + 1.5 M floats and capture()'s snapshot of it")
    lr = 0.01 if adam else 1.0
    opts = dict(optimizer="adam_rows_tf") if adam else {}
    tr = _trainer(units, "relu", D, B, rows, lr, use_graph=(case != "sgd_eager"), **opts)
    c = tr.coll
    total = c.total_rows
    assert total * c.row_stride > TWO32 or (adam and total * tr.state.shape[1] > TWO32)
    offs = np.array([int(o) for o in c._offsets.cpu()], np.int64)
    rs = c.row_stride
    gen = lambda r0, r1: pattern_dev(r0, r1, rs, EMB_SALT, EMB_SCALE)
    gen_lin = lambda r0, r1: pattern_dev(r0, r1, 1, LIN_SALT, LIN_SCALE)
    with torch.no_grad():
        fill(c.weight.data.view(total, rs), gen)
        if c.linear is not None:
            fill(c.linear.data.view(-1, 1), gen_lin)
    emb_of = lambda g: pattern_np(g, rs, EMB_SALT, EMB_SCALE)[:, :D]
    lin_of = ((lambda g: pattern_np(g, rs, EMB_SALT, EMB_SCALE)[:, D]) if c.linear is None
              else (lambda g: pattern_np(g, 1, LIN_SALT, LIN_SCALE)[:, 0]))
    rng = np.random.default_rng(17)
    touched = placed_rows(total, tr.state.shape[1] if adam else rs)[0]
    ids = _steered_ids(rng, rows, offs, touched, B)
    labels = rng.integers(0, 2, B).astype(np.float32)
    comp = Compact(ids, rows, offs, emb_of, lin_of)
    rows_g = comp.global_rows()
    assert np.isin(touched, rows_g).all()
    ws0, bs0 = [npy(w) for w in tr.w], [npy(b) for b in tr.b]
    bias0 = float(c.bias.detach())
    o = deepfm_step(comp.tables, comp.lins, bias0, ws0, bs0, "relu", comp.ids, labels)
    tr.step(torch.from_numpy(ids).cuda(), torch.from_numpy(labels).cuda())
    torch.cuda.synchronize()
    report = {}
    got = lambda k, t, e, extra=0.0: report.__setitem__(k, check(k, t, e, extra=extra))
    got("loss", float(tr.loss), o["loss"])
    got("prob", npy(tr.prob), o["prob"])
    got("fm_logit", npy(tr.fm_logit), o["fm_logit"])
    got("stack", npy(tr.stack), o["stack"])
    for i in range(len(ws0)):
        got(f"acts.{i}", npy(tr.acts[i]), o[f"acts.{i}"])
        if not adam:
            for k, buf, p0, p1 in ((f"w.{i}", tr.gw[i], ws0[i], tr.w[i]), (f"b.{i}", tr.gb[i], bs0[i], tr.b[i])):
                got("grad buffer " + k, npy(buf), o[k])
                after = npy(p1)
                got("update " + k, (p0 - after) / lr, o[k], update_slack(p0, after, lr, 1, o[k].terms))
    gi = torch.from_numpy(rows_g).cuda()
    w1 = c.weight.detach().view(total, rs).index_select(0, gi).cpu().numpy().astype(F64)
    emb1 = w1[:, :D]
    lin1 = w1[:, D] if c.linear is None else c.linear.detach().index_select(0, gi).cpu().numpy().astype(F64)
    hits = np.concatenate([o[f"hits.{s}"] for s in range(len(rows))])
    emb0 = np.concatenate(comp.tables).astype(F64)
    lin0 = np.concatenate(comp.lins).astype(F64)
    fields = lambda key: [np.concatenate([np.broadcast_to(np.asarray(getattr(o[f"{key}.{s}"], f), F64),
                                                          np.shape(o[f"{key}.{s}"].ref))
                                          for s in range(len(rows))], 0) for f in Entry._fields]
    e_t, e_l = Entry(*fields("table")), Entry(*fields("lin"))
    if adam:
        SS = tr.state.shape[1]
        st = tr.state.index_select(0, gi).cpu().numpy().astype(F64)
        m = np.concatenate([st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]], 1)
        v = np.concatenate([st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]], 1)
        e = Entry(np.concatenate([e_t.ref, e_l.ref[:, None]], 1), np.concatenate([e_t.scale, e_l.scale[:, None]], 1),
                  np.concatenate([e_t.slack + np.zeros_like(e_t.ref), (e_l.slack + np.zeros_like(e_l.ref))[:, None]], 1),
                  np.concatenate([e_t.terms, e_l.terms[:, None]], 1))
        extra = U * e.terms + update_slack(0, 0, 1, hits[:, None], e.terms)
        m1, bm, v1, bv = moments(np.zeros_like(m), np.zeros_like(v), e, extra, B1, B2)
        report["m"] = check_bound("adam_rows_tf m", m, m1, bm)
        report["v"] = check_bound("adam_rows_tf v", v, v1, bv)
        p1, bp = functor(np.concatenate([emb0, lin0[:, None]], 1), m, v, F64(float(tr.clock.lr_t)), EPS)
        report["p"] = check_bound("adam_rows_tf p", np.concatenate([emb1, lin1[:, None]], 1), p1, bp)
        assert_only(changed_rows(tr.state, lambda r0, r1: torch.zeros((r1 - r0, SS), device="cuda")), rows_g,
                    "adam_rows_tf: state")
    else:
        got("update table rows", (emb0 - emb1) / lr, e_t, update_slack(emb0, emb1, lr, hits[:, None], e_t.terms))
        got("update first-order", (lin0 - lin1) / lr, e_l, update_slack(lin0, lin1, lr, hits, e_l.terms))
    assert_only(changed_rows(c.weight.detach().view(total, rs), gen), rows_g, f"{case}: table")
    if c.linear is not None:
        assert_only(changed_rows(c.linear.detach().view(-1, 1), gen_lin), rows_g, f"{case}: first-order weights")
    print("max err/scale:", {k: f"{v:.1e}" for k, v in report.items() if v > 0})
