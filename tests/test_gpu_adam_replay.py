"""The row-sparse Adam kernels of embed_adam.cu and optim.cu called directly through the C-ABI on constructed state,
held per element to the float64 model of tests/adam_oracle.py.

The arena has two tables whose rows carry hand-set step stamps -- 0 (never updated), t-1, t-2, t-15, t-16, t-17, and
at t = 5000 also t-2047, t-2048, t-2049 and 1, and t itself -- with non-zero m, v, m_w, v_w, and a rate ring of
hist_len = 16 that dr_adam_advance_hist fills.  So the replay (adam_catch_up / adam_lr_at) takes every branch:

  ring hit: stamps t-2 .. t-16 (stamp t-16 starts at j = t-15, still in the ring);
  t_now - j == hist_len (the first rate that is recomputed): t-17, whose first replayed step is j = t-16;
  recompute: t-17, 1 (and every stamp at t = 40 below t-16, where powf's error is amplified most);
  kCatchUpMax: t-2049 in the prepare (2048 steps, exactly the cap), t-2048 in the flush; above it (closed-form decay of
  m and v): t-2049 in the flush, 1 in both.

Every launch instantiation is named by a case (LPR = lanes per row, from D):
  embed_adam_prepare / embed_adam_flush / embed_fm_bwd_adam (EXACT and not, int32 and int64 ids):
      LPR 1: D4 (either layout), 2: fused D8, 4: fused D16, 8: fused D28 and split D32, 16: split D64, 32: split D128;
  lazy_adam_rows (the fused layout's [w | pad] chunk counts as a lane): LPR 1: split D4, 2: fused D4, 4: fused D8,
      8: fused D16 / D28 and split D32, 16: split D64, 32: split D128;
  embed_adam_count: int32 and int64 ids.
"""
import numpy as np
import pytest
import torch

from adam_oracle import (K_CATCH_UP_MAX, U, Entry, adam_bias_additions, check_bound, f32, functor, lr_t, moments,
                         replay, update_slack)
from oracle import reference_np as R

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-7
HIST = 16
ROWS = [40, 27]
DR_EINVAL, DR_EALIGN = -1, -2

LAYOUTS = [pytest.param(D, lay, id=f"{lay}_D{D}") for D, lay in
           [(4, "fused"), (8, "fused"), (16, "fused"), (28, "fused"), (4, "split"), (32, "split"), (64, "split"),
            (128, "split")]]
T_NOW = [pytest.param(40, id="t40"), pytest.param(5000, id="t5000")]
IDS = [pytest.param(torch.int64, id="i64"), pytest.param(torch.int32, id="i32")]


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _stamp_classes(t):
    return sorted({s for s in (0, t - 1, t - 2, t - 15, t - 16, t - 17, t - 2047, t - 2048, t - 2049, 1, t) if s >= 0})


class Arena:
    """Two tables of the given layout with per-row Adam state blocks [g D | m D | v D | g_w m_w v_w count stamp | pad]."""

    def __init__(self, D, layout, t, seed):
        rng = np.random.default_rng(seed)
        self.D, self.layout, self.t = D, layout, t
        self.fused = layout == "fused"
        self.rs = 32 if self.fused else D
        self.R = sum(ROWS)
        self.offs = np.concatenate([[0], np.cumsum(ROWS)[:-1]]).astype(np.int64)
        w = np.zeros((self.R, self.rs), F32)
        w[:] = rng.standard_normal(w.shape) * 0.05         # padding too: it must come back bit for bit
        lin = (rng.standard_normal(self.R) * 0.05).astype(F32)
        self.SS = _lib().dr_embed_adam_state_stride(D)
        st = np.zeros((self.R, self.SS), F32)
        m = rng.standard_normal((self.R, D + 1)) * 1e-3
        v = m ** 2 * rng.uniform(0.5, 2.0, m.shape)        # |m| / sqrt(v) ~ 1: every replayed step moves p by ~lr_j
        st[:, D:2 * D], st[:, 2 * D:3 * D] = m[:, :D], v[:, :D]
        st[:, 3 * D + 1], st[:, 3 * D + 2] = m[:, D], v[:, D]
        classes = _stamp_classes(t)
        stamps = np.array([classes[(r // 2) % len(classes)] for r in range(self.R)], np.int32)   # odd and even rows
        st[:, 3 * D + 4] = stamps.view(F32)
        self.w = torch.from_numpy(w).cuda()
        self.lin = None if self.fused else torch.from_numpy(lin).cuda()
        self.state = torch.from_numpy(st).cuda()
        self.rows = torch.tensor(ROWS, dtype=torch.int64, device="cuda")
        self.slot_offsets = torch.from_numpy(self.offs).cuda()
        base = self.w.data_ptr()
        self.tp = torch.tensor([base + int(o) * self.rs * 4 for o in self.offs], dtype=torch.int64, device="cuda")
        lbase = self.tp if self.fused else torch.tensor([self.lin.data_ptr() + int(o) * 4 for o in self.offs],
                                                         dtype=torch.int64, device="cuda")
        self.lp = lbase
        self.flags = 1 if self.fused else 0
        self.lin_stride = self.rs if self.fused else 1
        # the clock at step t, its last HIST rates in the ring (dr_adam_advance_hist fills it: set t - HIST, advance)
        self.step = torch.tensor([t - HIST], dtype=torch.int64, device="cuda")
        self.lr_t = torch.zeros(1, device="cuda")
        self.hist = torch.zeros(HIST, device="cuda")
        for _ in range(HIST):
            rc = _lib().dr_adam_advance_hist(self.step.data_ptr(), LR, B1, B2, self.lr_t.data_ptr(), self.hist.data_ptr(),
                                             HIST, _stream())
            assert rc == 0
        torch.cuda.synchronize()
        assert int(self.step) == t

    # ---- host views (float64) ----
    def host(self):
        D = self.D
        w = self.w.cpu().numpy()
        st = self.state.cpu().numpy()
        lin = w[:, D] if self.fused else self.lin.cpu().numpy()
        p = np.concatenate([w[:, :D], lin[:, None]], 1).astype(F64)          # [emb | w]
        m = np.concatenate([st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]], 1).astype(F64)
        v = np.concatenate([st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]], 1).astype(F64)
        return dict(p=p, m=m, v=v, w=w.copy(), lin=lin.copy(), st=st.copy(),
                    stamp=st[:, 3 * D + 4].view(np.int32).astype(np.int64), count=st[:, 3 * D + 3].view(np.int32).copy(),
                    g=np.concatenate([st[:, :D], st[:, 3 * D:3 * D + 1]], 1))


def _ids(seed, id_dtype):
    """Every even local row of each table once, local row 2 seven more times, OOV ids of both kinds; columns shuffled."""
    rng = np.random.default_rng(seed)
    cols = []
    for r in ROWS:
        c = list(range(0, r, 2)) + [2] * 7 + [-1, r, -1, r]
        cols.append(c)
    B = max(len(c) for c in cols)
    ids = np.full((B, len(ROWS)), -1, np.int64)
    for s, c in enumerate(cols):
        c = c + [ROWS[s] if k % 2 else -1 for k in range(B - len(c))]
        ids[:, s] = rng.permutation(c)
    return ids, torch.from_numpy(ids).cuda().to(id_dtype)


def _touched(a, ids):
    hits = np.zeros(a.R, np.int64)
    for s, r in enumerate(ROWS):
        col = ids[:, s]
        ok = col[(col >= 0) & (col < r)]
        np.add.at(hits, a.offs[s] + ok, 1)
    return hits


def _lr_checks(a):
    """The ring holds float32(lr_j) for the last HIST steps within 1 ulp, and lr_t is lr_t(t); dr_adam_advance gives
    the same bits as dr_adam_advance_hist."""
    ring = a.hist.cpu().numpy()
    for j in range(a.t - HIST + 1, a.t + 1):
        want = lr_t(j)
        assert abs(F64(ring[j % HIST]) - want) <= 2 * U * want, j
    assert float(a.lr_t) == ring[a.t % HIST]
    step, out = torch.tensor([a.t - 1], dtype=torch.int64, device="cuda"), torch.zeros(1, device="cuda")
    assert _lib().dr_adam_advance(step.data_ptr(), LR, B1, B2, out.data_ptr(), _stream()) == 0
    assert int(step) == a.t and torch.equal(out.view(torch.int32), a.lr_t.view(torch.int32))


def _same_bits(name, got, want):
    assert np.array_equal(np.asarray(got).view(np.int32), np.asarray(want).view(np.int32)), name


def _check_replayed(name, a, h0, h1, sel, upto, report):
    """Rows `sel`: p, m, v (table and first-order) per `replay` of the snapshot h0 up to `upto`."""
    rp, rm, rv, bp, bm, bv = replay(h0["p"][sel], h0["m"][sel], h0["v"][sel], h0["stamp"][sel], upto, LR, B1, B2, EPS,
                                    t_now=a.t, hist_len=HIST)
    for k, ref, b in (("p", rp, bp), ("m", rm, bm), ("v", rv, bv)):
        report[f"{name} {k}"] = max(report.get(f"{name} {k}", 0.0), check_bound(f"{name} {k}", h1[k][sel], ref, b))
    return rp, rm, rv, bp, bm, bv


def _untouched_bits(a, h0, h1, keep):
    _same_bits("untouched rows: parameters", h1["w"][keep], h0["w"][keep])
    _same_bits("untouched rows: first-order weights", h1["lin"][keep], h0["lin"][keep])
    _same_bits("untouched rows: state", h1["st"][keep], h0["st"][keep])
    if a.fused:
        _same_bits("row padding", h1["w"][:, a.D + 1:], h0["w"][:, a.D + 1:])


# ---- dr_embed_adam_prepare ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("id_dtype", IDS)
@pytest.mark.parametrize("t", T_NOW)
@pytest.mark.parametrize("D,layout", LAYOUTS)
def test_prepare_replays_touched_rows_up_to_t_minus_1(D, layout, t, id_dtype):
    a = Arena(D, layout, t, seed=D + t)
    _lr_checks(a)
    ids, tids = _ids(D, id_dtype)
    h0 = a.host()
    rc = _lib().dr_embed_adam_prepare(tids.data_ptr(), tids.element_size(), ids.shape[0], len(ROWS), D,
                                      a.rows.data_ptr(), a.slot_offsets.data_ptr(), a.rs, a.lin_stride, a.flags,
                                      a.tp.data_ptr(), a.lp.data_ptr(), a.state.data_ptr(), a.step.data_ptr(),
                                      a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    h1 = a.host()
    hits = _touched(a, ids)
    sel = hits > 0
    report = {}
    _check_replayed("prepare", a, h0, h1, sel, t - 1, report)
    s0 = h0["stamp"]
    moved = sel & (s0 > 0) & (s0 < t - 1)
    assert moved.sum() >= 3
    assert (h1["stamp"][moved] == t - 1).all() and (h1["stamp"][~moved] == s0[~moved]).all()
    assert np.array_equal(h1["count"], hits), "count column != lookups per row"
    assert not h1["g"].any()
    _untouched_bits(a, h0, h1, ~sel)
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- dr_embed_adam_flush --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", T_NOW)
@pytest.mark.parametrize("D,layout", LAYOUTS)
def test_flush_replays_every_stale_row_up_to_t(D, layout, t):
    a = Arena(D, layout, t, seed=3 * D + t)
    h0 = a.host()
    rc = _lib().dr_embed_adam_flush(a.rows.data_ptr(), a.slot_offsets.data_ptr(), len(ROWS), D, a.R, a.rs, a.lin_stride,
                                    a.flags, a.tp.data_ptr(), a.lp.data_ptr(), a.state.data_ptr(), a.step.data_ptr(),
                                    a.hist.data_ptr(), HIST, LR, B1, B2, EPS, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    h1 = a.host()
    s0 = h0["stamp"]
    stale = (s0 > 0) & (s0 < t)
    report = {}
    _check_replayed("flush", a, h0, h1, stale, t, report)
    assert (h1["stamp"][stale] == t).all()
    _untouched_bits(a, h0, h1, ~stale)
    if t > K_CATCH_UP_MAX + 1:            # the steps beyond the cap move a row by less than half an ulp
        far = stale & (t - s0 > K_CATCH_UP_MAX)
        full = replay(h0["p"][far], h0["m"][far], h0["v"][far], s0[far], t)[0]
        capped = replay(h0["p"][far], h0["m"][far], h0["v"][far], s0[far], s0[far] + K_CATCH_UP_MAX)[0]
        assert far.any() and (np.abs(full - capped) < U * np.abs(capped)).all()
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- the Adam backward: dr_embed_fm_bwd_adam (non-EXACT) and dr_embed_fm_bwd_adam_tf without a prepare ----------------
def _bwd_inputs(a, ids, seed):
    """stack on a 2^-8 grid (float32 sums of it are exact), dL/dlogit on a 2^-14 grid, g_stack arbitrary."""
    rng = np.random.default_rng(seed)
    B, S, D = ids.shape[0], len(ROWS), a.D
    ok = np.stack([(ids[:, s] >= 0) & (ids[:, s] < ROWS[s]) for s in range(S)], 1)
    stack = (np.round(rng.uniform(-1, 1, (B, S, D)) * 256) / 256 * ok[:, :, None]).astype(F32)
    gl = (np.round(rng.uniform(-1, 1, B) * 2 ** 8) / 2 ** 14).astype(F32)
    gs = (rng.standard_normal((B, S, D)) * 1e-2).astype(F32)
    sum_e = stack.sum(1, dtype=F32)
    return stack, gl, gs, sum_e


def _grad_entries(a, ids, stack, gl, gs):
    """Row gradients (float64) with the rounding of the kernel: one FMA per lookup (sum - e and gl * (.) are exact on
    these grids) and `hits` float32 additions into the zeroed gradient slots."""
    gt, glin, gbias = R.embed_fm_grad(ROWS, ids, stack.astype(F64), gl.astype(F64), gs.astype(F64))
    d = gl[:, None, None].astype(F64) * (stack.sum(1, keepdims=True).astype(F64) - stack) + gs
    tt, tl, _ = R.embed_fm_grad(ROWS, ids, np.zeros(stack.shape), np.abs(gl.astype(F64)), np.abs(d), F64)
    ref = np.concatenate([np.concatenate([g, l[:, None]], 1) for g, l in zip(gt, glin)], 0)
    terms = np.concatenate([np.concatenate([g, l[:, None]], 1) for g, l in zip(tt, tl)], 0)
    return Entry(ref, 0.0, 0.0, terms), float(gbias), float(np.abs(gl.astype(F64)).sum())


def _count(a, tids, B):
    rc = _lib().dr_embed_adam_count(tids.data_ptr(), tids.element_size(), B, len(ROWS), a.D, a.rows.data_ptr(),
                                    a.slot_offsets.data_ptr(), a.state.data_ptr(), _stream())
    assert rc == 0


@pytest.mark.parametrize("exact", [pytest.param(False, id="bwd_adam"), pytest.param(True, id="bwd_adam_tf")])
@pytest.mark.parametrize("id_dtype", IDS)
@pytest.mark.parametrize("t", T_NOW)
@pytest.mark.parametrize("D,layout", LAYOUTS)
def test_adam_backward_on_constructed_state(D, layout, t, id_dtype, exact):
    """Counts from dr_embed_adam_count, then one backward.  EXACT without a prepare: every touched row replays
    (stamp, t-1] inside the backward, then takes step t's update, and is stamped t."""
    a = Arena(D, layout, t, seed=5 * D + t + exact)
    ids, tids = _ids(D + 1, id_dtype)
    B, S = ids.shape
    stack, gl, gs, sum_e = _bwd_inputs(a, ids, D + t)
    d_stack, d_gl, d_gs, d_sum = (torch.from_numpy(x).cuda() for x in (stack, gl, gs, sum_e))
    g_bias = torch.zeros(1, device="cuda")
    h0 = a.host()
    _count(a, tids, B)
    torch.cuda.synchronize()
    hits = _touched(a, ids)
    assert np.array_equal(a.host()["count"], hits), "dr_embed_adam_count: count column != lookups per row"
    lib = _lib()
    args = (tids.data_ptr(), tids.element_size(), a.rows.data_ptr(), a.slot_offsets.data_ptr(), d_stack.data_ptr(),
            d_sum.data_ptr(), d_gl.data_ptr(), d_gs.data_ptr(), B, S, D, a.rs, a.lin_stride, a.flags, a.tp.data_ptr(),
            a.lp.data_ptr(), a.state.data_ptr(), g_bias.data_ptr())
    if exact:
        rc = lib.dr_embed_fm_bwd_adam_tf(*args, a.step.data_ptr(), a.lr_t.data_ptr(), a.hist.data_ptr(), HIST, LR, B1,
                                         B2, EPS, _stream())
    else:
        rc = lib.dr_embed_fm_bwd_adam(*args, a.lr_t.data_ptr(), B1, B2, EPS, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    h1 = a.host()
    sel = hits > 0
    e, gbias, gbias_terms = _grad_entries(a, ids, stack, gl, gs)
    e = Entry(e.ref[sel], 0.0, 0.0, e.terms[sel])
    extra = U * e.terms + update_slack(0, 0, 1, hits[sel][:, None], e.terms)
    s0 = h0["stamp"][sel]
    p0, m0, v0 = h0["p"][sel], h0["m"][sel], h0["v"][sel]
    bp0 = bm0 = bv0 = 0.0
    if exact:
        p0, m0, v0, bp0, bm0, bv0 = replay(p0, m0, v0, s0, t - 1, LR, B1, B2, EPS, t_now=t, hist_len=HIST)
    report = {}
    m1, bm, v1, bv = moments(m0, v0, e, extra, B1, B2, m0_err=bm0, v0_err=bv0)
    report["m"] = check_bound("m", h1["m"][sel], m1, bm)
    report["v"] = check_bound("v", h1["v"][sel], v1, bv)
    p1, bp = functor(p0, h1["m"][sel], h1["v"][sel], F64(float(a.lr_t)), EPS, p0_err=bp0)
    report["p"] = check_bound("p", h1["p"][sel], p1, bp)
    from test_gpu_deepfm_train_step import _sms
    bb = update_slack(0, 0, 1, adam_bias_additions(B, _sms()), gbias_terms)
    report["g_bias"] = check_bound("g_bias", float(g_bias), gbias, bb)
    assert not h1["g"].any(), "gradient slots not cleared"
    assert not h1["count"].any(), "countdowns not back to zero"
    if exact:
        assert (h1["stamp"][sel] == t).all()
        replayed = (s0 > 0) & (s0 < t - 1)
        assert replayed.sum() >= 3
    else:
        assert np.array_equal(h1["stamp"], h0["stamp"])
    _untouched_bits(a, h0, h1, ~sel)
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- dr_lazy_adam_rows ------------------------------------------------------------------------------------------------
LAZY = LAYOUTS + [pytest.param(12, "fused", id="fused_D12")]


@pytest.mark.parametrize("id_dtype", IDS)
@pytest.mark.parametrize("D,layout", LAZY)
def test_lazy_adam_rows_on_constructed_arenas(D, layout, id_dtype):
    rng = np.random.default_rng(D)
    fused = layout == "fused"
    rs = 32 if fused else D
    Rt = sum(ROWS)
    offs = np.concatenate([[0], np.cumsum(ROWS)[:-1]]).astype(np.int64)
    ids, tids = _ids(2 * D, id_dtype)
    hits = np.zeros(Rt, np.int64)
    for s, r in enumerate(ROWS):
        col = ids[:, s]
        np.add.at(hits, offs[s] + col[(col >= 0) & (col < r)], 1)
    sel = hits > 0
    ncol = D + 1 if fused else D
    p = (rng.standard_normal((Rt, rs)) * 0.05).astype(F32)
    m = (rng.standard_normal((Rt, rs)) * 1e-3).astype(F32)
    v = (m.astype(F64) ** 2 * rng.uniform(0.5, 2.0, m.shape)).astype(F32)
    g = np.zeros((Rt, rs), F32)
    g[sel, :ncol] = rng.standard_normal((int(sel.sum()), ncol)) * 1e-2
    lin = [(rng.standard_normal(Rt) * s).astype(F32) for s in (0.05, 0, 1e-3, 1e-6)] if not fused else None
    if lin is not None:
        lin[1][sel] = rng.standard_normal(int(sel.sum())) * 1e-2
        lin[3] = np.abs(lin[3])
    t = 7
    stamp0 = rng.integers(1, t, Rt).astype(np.int32)
    dev = lambda x: torch.from_numpy(x.copy()).cuda()
    tp, tg, tm, tv, tst = dev(p), dev(g), dev(m), dev(v), dev(stamp0)
    tl = [dev(x) for x in lin] if lin is not None else None
    step = torch.tensor([t], dtype=torch.int64, device="cuda")
    lr_dev = torch.tensor([lr_t(t)], dtype=torch.float32, device="cuda")
    ptr = lambda x: None if x is None else x.data_ptr()
    d_rows, d_offs = torch.tensor(ROWS, device="cuda"), dev(offs)      # held: the kernel reads them after this line
    rc = _lib().dr_lazy_adam_rows(tids.data_ptr(), tids.element_size(), ids.shape[0], len(ROWS), D,
                                  d_rows.data_ptr(), d_offs.data_ptr(), tp.data_ptr(),
                                  tg.data_ptr(), tm.data_ptr(), tv.data_ptr(), rs, 1 if fused else 0,
                                  *(ptr(x) for x in (tl or [None] * 4)), tst.data_ptr(), step.data_ptr(),
                                  lr_dev.data_ptr(), B1, B2, EPS, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    host = lambda x: x.cpu().numpy()
    P, G, M, V, ST = host(tp), host(tg), host(tm), host(tv), host(tst)
    cols = [(p[:, :ncol], g[:, :ncol], m[:, :ncol], v[:, :ncol], P[:, :ncol], M[:, :ncol], V[:, :ncol])]
    if lin is not None:
        L1 = [host(x) for x in tl]
        cols.append((lin[0][:, None], lin[1][:, None], lin[2][:, None], lin[3][:, None], L1[0][:, None],
                     L1[2][:, None], L1[3][:, None]))
        assert not L1[1].any() and np.array_equal(L1[0][~sel], lin[0][~sel])
    report = {}
    lr_ = F64(float(lr_dev))
    for k, (p0, g0, m0, v0, p1, m1g, v1g) in enumerate(cols):
        e = Entry(g0[sel].astype(F64), 0.0, 0.0)
        m1, bm, v1, bv = moments(m0[sel], v0[sel], e, 0.0, B1, B2)
        report[f"m{k}"] = check_bound("m", m1g[sel], m1, bm)
        report[f"v{k}"] = check_bound("v", v1g[sel], v1, bv)
        pr, bp = functor(p0[sel], m1g[sel], v1g[sel], lr_, EPS)
        report[f"p{k}"] = check_bound("p", p1[sel], pr, bp)
    assert not G.any(), "gradient arena not cleared"
    for name, got, want in (("p", P, p), ("m", M, m), ("v", V, v)):
        _same_bits(f"untouched rows: {name}", got[~sel], want[~sel])
        _same_bits(f"padding: {name}", got[:, ncol:], want[:, ncol:])
    assert (ST[sel] == t).all() and np.array_equal(ST[~sel], stamp0[~sel])
    print("max err/bound:", {k: f"{v:.1e}" for k, v in report.items()})


# ---- argument checks: the entries refuse without launching ------------------------------------------------------------
def test_adam_entries_reject_bad_arguments_without_launching():
    from deep_recommenders_b200 import _lib as L
    lib = _lib()
    a = Arena(16, "fused", 40, seed=0)
    ids, tids = _ids(0, torch.int64)
    B, S, D = ids.shape[0], len(ROWS), 16
    stack = torch.zeros((B, S, D), device="cuda")
    gl = torch.zeros(B, device="cuda")
    st = _stream()
    n0 = L.launch_count()
    ab = (a.rows.data_ptr(), a.slot_offsets.data_ptr())
    bwd = lambda state, d=D, idb=8: lib.dr_embed_fm_bwd_adam(
        tids.data_ptr(), idb, *ab, stack.data_ptr(), None, gl.data_ptr(), None, B, S, d, a.rs, a.lin_stride, a.flags,
        a.tp.data_ptr(), a.lp.data_ptr(), state, None, a.lr_t.data_ptr(), B1, B2, EPS, st)
    assert bwd(a.state.data_ptr() + 4) == DR_EALIGN
    assert bwd(a.state.data_ptr(), d=6) == DR_EINVAL
    assert bwd(a.state.data_ptr(), idb=2) == DR_EINVAL
    assert lib.dr_embed_fm_bwd_adam_tf(tids.data_ptr(), 8, *ab, stack.data_ptr(), None, gl.data_ptr(), None, B, S, D,
                                       a.rs, a.lin_stride, a.flags, a.tp.data_ptr(), a.lp.data_ptr(), a.state.data_ptr(),
                                       None, None, a.lr_t.data_ptr(), a.hist.data_ptr(), HIST, LR, B1, B2, EPS,
                                       st) == DR_EINVAL                                   # no step counter
    assert lib.dr_embed_fm_bwd_adam_tf(tids.data_ptr(), 8, *ab, stack.data_ptr(), None, gl.data_ptr(), None, B, S, D,
                                       a.rs, a.lin_stride, a.flags, a.tp.data_ptr(), a.lp.data_ptr(), a.state.data_ptr(),
                                       None, a.step.data_ptr(), a.lr_t.data_ptr(), None, HIST, LR, B1, B2, EPS,
                                       st) == DR_EINVAL                                   # ring length without a ring
    assert lib.dr_embed_adam_count(tids.data_ptr(), 8, B, S, 130, *ab, a.state.data_ptr(), st) == DR_EINVAL
    assert lib.dr_embed_adam_count(tids.data_ptr(), 8, B, 0, D, *ab, a.state.data_ptr(), st) == DR_EINVAL
    assert lib.dr_embed_adam_prepare(tids.data_ptr(), 8, B, S, D, *ab, a.rs, a.lin_stride, a.flags, a.tp.data_ptr(),
                                     a.lp.data_ptr(), a.state.data_ptr(), None, a.hist.data_ptr(), HIST, LR, B1, B2,
                                     EPS, st) == DR_EINVAL
    assert lib.dr_embed_adam_flush(*ab, S, 10, a.R, a.rs, a.lin_stride, a.flags, a.tp.data_ptr(), a.lp.data_ptr(),
                                   a.state.data_ptr(), a.step.data_ptr(), a.hist.data_ptr(), HIST, LR, B1, B2, EPS,
                                   st) == DR_EINVAL
    assert lib.dr_adam_advance_hist(a.step.data_ptr(), LR, 1.0, B2, a.lr_t.data_ptr(), a.hist.data_ptr(), HIST,
                                    st) == DR_EINVAL
    assert lib.dr_adam_advance_hist(a.step.data_ptr(), LR, B1, B2, a.lr_t.data_ptr(), a.hist.data_ptr(), -1,
                                    st) == DR_EINVAL
    arena = torch.zeros((a.R + 1, 32), device="cuda")
    lz = lambda p, d=D, rs=32, flags=1: lib.dr_lazy_adam_rows(
        tids.data_ptr(), 8, B, S, d, *ab, p, arena.data_ptr(), arena.data_ptr(), arena.data_ptr(), rs, flags, None, None,
        None, None, torch.zeros(a.R, dtype=torch.int32, device="cuda").data_ptr(), a.step.data_ptr(), a.lr_t.data_ptr(),
        B1, B2, EPS, st)
    assert lz(arena.data_ptr() + 4) == DR_EALIGN
    assert lz(arena.data_ptr(), d=128, rs=132) == DR_EINVAL          # [w | pad] chunk needs D <= 124
    assert lz(arena.data_ptr(), rs=16) == DR_EINVAL                  # row stride below D + 4
    assert L.launch_count() == n0, "a rejected call launched a kernel"
    torch.cuda.synchronize()
