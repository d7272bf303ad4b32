"""The float64 Adam model of tests/adam_oracle.py against a plain float64 torch restatement, and its bounds: they accept
float32 results a few ulps off (a float32 emulation of the kernels' arithmetic) and reject each modelled kernel bug."""
import numpy as np
import pytest
import torch

from adam_oracle import (K_CATCH_UP_MAX, U, adam_bias_additions, f32, functor, lr_err, lr_t, moments, omb, outside,
                         replay)
from deepfm_oracle import RTOL, Entry, deepfm_step, update_slack
from oracle import reference_np as R
from test_cpu_deepfm_oracle import _problem

F32, F64 = np.float32, np.float64
LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-7
HIST = 16


# ---- the model against a float64 torch restatement ------------------------------------------------------------------
def _torch_adam(p, g, m, v, lr_t_, b1=B1, b2=B2, eps=EPS):
    p, g, m, v = (torch.tensor(np.asarray(a, F64)) for a in (p, g, m, v))
    o1, o2 = float(omb(b1)), float(omb(b2))
    m = m * (1 - o1) + g * o1
    v = v * (1 - o2) + g * g * o2
    p = p - lr_t_ * m / (v.sqrt() + float(F32(eps)))
    return p.numpy(), m.numpy(), v.numpy()


def _close(a, b):
    a, b = np.asarray(a, F64), np.asarray(b, F64)
    return np.abs(a - b).max(initial=0.0) <= 1e-12 * max(1.0, np.abs(b).max(initial=0.0))


def test_lr_t_is_keras_bias_corrected_rate():
    for t in (1, 2, 3, 17, 1000, 5000):
        b1, b2 = F64(F32(B1)), F64(F32(B2))
        want = float(F32(LR)) * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        assert abs(lr_t(t) - want) <= 1e-15 * want and abs(lr_t(t) - R.adam_lr_t(LR, t)) <= 1e-15 * want


def test_moments_functor_and_replay_equal_torch_restatement():
    rng = np.random.default_rng(0)
    p, g = f32(rng.standard_normal((5, 6))), rng.standard_normal((5, 6)) * 1e-2
    m, v = f32(rng.standard_normal((5, 6)) * 1e-3), f32(rng.random((5, 6)) * 1e-5)
    e = Entry(g, np.zeros_like(g), 0.0)
    m1, _, v1, _ = moments(m, v, e)
    p1, _ = functor(p, m1, v1, lr_t(7))
    tp, tm, tv = _torch_adam(p, g, m, v, lr_t(7))
    assert _close(m1, tm) and _close(v1, tv) and _close(p1, tp)
    # replay: dense Adam with g = 0 for every step after the stamp, per row, uncapped
    stamp, upto = np.array([0, 3, 6, 7, 1]), 7
    rp, rm, rv, *_ = replay(p, m, v, stamp, upto)
    for r in range(5):
        tp, tm, tv = p[r], m[r], v[r]
        for j in range(stamp[r] + 1, upto + 1) if stamp[r] > 0 else ():
            tp, tm, tv = _torch_adam(tp, np.zeros(6), tm, tv, lr_t(j))
        assert _close(rp[r], tp) and _close(rm[r], tm) and _close(rv[r], tv), r
    # beyond kCatchUpMax too: the model is not capped
    rp, rm, rv, bp, *_ = replay(p[:1], m[:1], v[:1], [1], K_CATCH_UP_MAX + 11)
    tp, tm, tv = p[0], m[0], v[0]
    for j in range(2, K_CATCH_UP_MAX + 12):
        tp, tm, tv = _torch_adam(tp, np.zeros(6), tm, tv, lr_t(j))
    assert _close(rp[0], tp) and _close(rm[0], tm) and _close(rv[0], tv)


def test_adam_bias_additions_is_one_per_cta_of_the_adam_backward():
    assert adam_bias_additions(1, 132) == 1 and adam_bias_additions(96, 132) == 12
    assert adam_bias_additions(8448, 132) == 1056 and adam_bias_additions(9000, 132) == 1056


# ---- a float32 emulation of the kernels' arithmetic ----------------------------------------------------------------
def _ring(t_now):
    """The ring dr_adam_advance_hist leaves at step t_now: float32(lr_j) at j % HIST for the last HIST steps."""
    ring = np.zeros(HIST, F32)
    for j in range(max(1, t_now - HIST + 1), t_now + 1):
        ring[j % HIST] = F32(lr_t(j))
    return ring


def _powf(b, j):
    return F32(F64(F32(b)) ** j)


def _catch_up_f32(p, m, v, stamp, upto, t_now, bug=None):
    """adam_catch_up in float32 over rows [p | w] (the last column is the first-order weight), with modelled bugs."""
    p, m, v = (np.array(a, F32, copy=True) for a in (p, m, v))
    o1, o2 = F32(1) - F32(B1), F32(1) - F32(B2)
    ring = _ring(t_now)
    for r, s in enumerate(np.asarray(stamp, np.int64)):
        if s <= 0 or upto <= s:
            continue
        gap = upto - s
        n = min(gap, K_CATCH_UP_MAX)
        cols = slice(0, p.shape[1] - 1) if bug == "w_not_replayed" else slice(None)
        for k in range(1, n + 1):
            j = s + k
            if bug == "skip_step" and k == n:
                continue
            hit = (t_now - j <= HIST) if bug == "boundary_le" else (t_now - j < HIST)
            if bug == "lr_now":
                lj = F32(lr_t(t_now))
            elif hit:
                lj = ring[(j - 1) % HIST] if bug == "ring_prev" else ring[j % HIST]
            else:
                lj = F32(F32(LR) * np.sqrt(F32(1) - _powf(B2, j), dtype=F32) / (F32(1) - _powf(B1, j)))
            mm, vv = m[r, cols], v[r, cols]
            if bug != "no_m_decay":
                mm = F32(F64(mm) - F64(mm) * F64(o1))
            vv = F32(F64(vv) - F64(vv) * F64(o2))
            p[r, cols] = p[r, cols] - F32(F32(mm * lj) / (np.sqrt(vv, dtype=F32) + F32(EPS)))
            m[r, cols], v[r, cols] = mm, vv
        if gap > n:
            dm, dv = _powf(F32(1) - o1, gap - n), _powf(F32(1) - o2, gap - n)
            m[r] = m[r] * dm
            if bug != "closed_form_m_only":
                v[r] = v[r] * dv
    return p, m, v


def _replay_state(t_now, rng, n=5):
    """Rows [emb(n) | w] of every stamp class the kernels distinguish at t_now, with non-zero m and v."""
    stamps = [s for s in (1, t_now - 1, t_now - 2, t_now - 15, t_now - 16, t_now - 17, t_now - 2047, t_now - 2048,
                          t_now - 2049) if s >= 1]
    R_ = len(stamps)
    p = f32(rng.standard_normal((R_, n + 1)) * 0.05)
    m = f32(rng.standard_normal((R_, n + 1)) * 1e-3)
    v = f32(m ** 2 * rng.uniform(0.5, 2.0, m.shape))          # |m| / sqrt(v) ~ 1: every replayed step moves p by ~lr_j
    return p, m, v, np.array(stamps)


def _replay_rejects(bug, t_now, upto, seed=0):
    rng = np.random.default_rng(seed)
    p, m, v, stamp = _replay_state(t_now, rng)
    rp, rm, rv, bp, bm, bv = replay(p, m, v, stamp, upto, t_now=t_now, hist_len=HIST)
    gp, gm, gv = _catch_up_f32(p, m, v, stamp, upto, t_now, bug)
    return outside(gp, rp, bp).any() or outside(gm, rm, bm).any() or outside(gv, rv, bv).any()


@pytest.mark.parametrize("t_now", [40, 5000])
@pytest.mark.parametrize("upto", ["prepare", "flush"])
def test_replay_bound_accepts_the_float32_kernel_arithmetic(t_now, upto):
    """Every stamp class -- ring hit, t_now - j == hist_len, recompute, below / at / above kCatchUpMax, closed-form
    decay -- of the float32 arithmetic of adam_catch_up is inside the bound, with room to spare."""
    up = t_now - 1 if upto == "prepare" else t_now
    rng = np.random.default_rng(t_now)
    p, m, v, stamp = _replay_state(t_now, rng)
    rp, rm, rv, bp, bm, bv = replay(p, m, v, stamp, up, t_now=t_now, hist_len=HIST)
    gp, gm, gv = _catch_up_f32(p, m, v, stamp, up, t_now)
    for got, want, b in ((gp, rp, bp), (gm, rm, bm), (gv, rv, bv)):
        assert not outside(got, want, b).any()
    # and the steps beyond the cap really move p by less than half an ulp, as the cap claims
    far = stamp == 1
    if up - 1 > K_CATCH_UP_MAX:
        capped = replay(p[far], m[far], v[far], [1], 1 + K_CATCH_UP_MAX)[0]
        assert (np.abs(rp[far] - capped) < U * np.abs(capped)).all()


@pytest.mark.parametrize("bug,t_now,upto", [
    ("skip_step", 40, 39), ("skip_step", 5000, 4999),
    ("lr_now", 40, 39), ("lr_now", 5000, 4999),
    ("ring_prev", 40, 39), ("ring_prev", 5000, 4999),
    ("boundary_le", 40, 39), ("boundary_le", 5000, 4999),
    ("w_not_replayed", 40, 39),
    ("no_m_decay", 40, 39), ("no_m_decay", 5000, 4999),
    ("closed_form_m_only", 5000, 5000),
])
def test_replay_bound_rejects_modelled_bugs(bug, t_now, upto):
    assert _replay_rejects(bug, t_now, upto)


def test_replay_bound_rejects_a_stamp_left_unchanged():
    """A stamp that is not advanced makes the next replay take the same steps again."""
    rng = np.random.default_rng(3)
    p, m, v, stamp = _replay_state(40, rng)
    rp, rm, rv, bp, bm, bv = replay(p, m, v, stamp, 39, t_now=40, hist_len=HIST)
    gp, gm, gv = _catch_up_f32(p, m, v, stamp, 39, 40)
    gp, gm, gv = _catch_up_f32(gp, gm, gv, stamp, 39, 40)          # replayed again from the stale stamp
    moved = (stamp > 0) & (stamp < 39)
    assert outside(gp, rp, bp)[moved].any(axis=1).all()


def test_recompute_rate_error_bound_holds_for_float32_powf():
    """lr_err's recompute branch covers a float32 evaluation whose powf is off by 4 ulps, at every j up to 5000."""
    j = np.arange(1, 5001)
    exact = lr_t(j)
    worst = np.zeros(j.shape)
    for sgn in (-1, 1):
        for b, other in ((B1, B2), (B2, B1)):
            pw = F32(F64(F32(b)) ** j)
            for _ in range(4):
                pw = np.nextafter(pw, F32(sgn * 2.0))
            po = F32(F64(F32(other)) ** j)
            p1, p2 = (pw, po) if b == B1 else (po, pw)
            got = F32(F32(LR) * np.sqrt(F32(1) - p2, dtype=F32) / (F32(1) - p1))
            worst = np.maximum(worst, np.abs(got - exact) / exact)
    assert (worst <= lr_err(j, 10 ** 9, HIST)).all()


# ---- the one-step bounds: gradient through m and v, update through the functor ------------------------------------
def _adam_f32(p, g, m, v, lr_t_, eps=EPS):
    """ApplyAdam in float32: the arithmetic of adam_elem / adam_functor."""
    p, g, m, v = (np.asarray(a, F32) for a in (p, g, m, v))
    o1, o2 = F32(1) - F32(B1), F32(1) - F32(B2)
    m = m + (g - m) * o1
    v = v + (g * g - v) * o2
    p = p - (m * F32(lr_t_)) / (np.sqrt(v) + F32(eps))
    return p.astype(F64), m.astype(F64), v.astype(F64)


def _hot_problem():
    p = _problem([12], "tanh", 1200, hot=True)
    return p, deepfm_step(*p)


def test_one_step_bounds_accept_float32_adam():
    (tables, *_), o = _hot_problem()
    rng = np.random.default_rng(5)
    e, hits = o["table.0"], o["hits.0"]
    extra = update_slack(0, 0, 1, hits[:, None], e.terms)
    m0 = f32(rng.standard_normal(e.ref.shape) * 1e-3)
    v0 = f32(rng.random(e.ref.shape) * 1e-6)
    for t, (mm, vv) in ((1, (np.zeros_like(m0), np.zeros_like(v0))), (4, (m0, v0))):
        g32 = f32(e.ref + rng.uniform(-1, 1, e.ref.shape) * 4 * 2 * U * e.scale)   # a few ulps of the scale off
        gp, gm, gv = _adam_f32(tables[0], g32, mm, vv, F32(lr_t(t)))
        m1, bm, v1, bv = moments(mm, vv, e, extra)
        assert not outside(gm, m1, bm).any() and not outside(gv, v1, bv).any()
        p1, bp = functor(tables[0], gm, gv, F64(F32(lr_t(t))))
        assert not outside(gp, p1, bp).any()


def test_one_step_bounds_reject_modelled_bugs():
    p, o = _hot_problem()
    tables, lins, bias, ws, bs, act, ids, labels = p
    e, hits = o["table.0"], o["hits.0"]
    extra = update_slack(0, 0, 1, hits[:, None], e.terms)
    zero = np.zeros_like(e.ref)
    # one of ~1000 duplicate contributions to the hot row lost at t = 1: invisible in p (Adam moves it by ~lr sign(g)),
    # outside the bound on m and v
    hot = int(np.flatnonzero(ids[:, 0] == 5)[0])
    single = deepfm_step(tables, lins, bias, ws, bs, act, ids[hot:hot + 1], labels[hot:hot + 1])
    lost = e.ref.copy()
    lost[5] -= single["table.0"].ref[5] / len(ids)
    gp_ok, gm_ok, gv_ok = _adam_f32(tables[0], e.ref, zero, zero, F32(lr_t(1)))
    gp, gm, gv = _adam_f32(tables[0], lost, zero, zero, F32(lr_t(1)))
    m1, bm, v1, bv = moments(zero, zero, e, extra)
    assert not outside(gm_ok, m1, bm).any() and not outside(gv_ok, v1, bv).any()
    assert outside(gm, m1, bm)[5].any() and outside(gv, v1, bv)[5].any()
    assert np.abs(gp - gp_ok).max() < 3e-2 * LR                  # what the parameter check of 3e-2 * lr could not see
    # lr_t of step t - 1, and eps inside the sqrt, against the functor recomputed from the kernel's own m, v, lr_t
    rng = np.random.default_rng(9)
    m0, v0 = f32(rng.standard_normal(e.ref.shape) * 1e-3), f32(rng.random(e.ref.shape) * 1e-6)
    _, gm, gv = _adam_f32(tables[0], e.ref, m0, v0, F32(lr_t(3)))
    p_ref, bp = functor(tables[0], gm, gv, F64(F32(lr_t(3))))
    stale = f32(tables[0] - F64(F32(lr_t(2))) * gm / (np.sqrt(gv) + F64(F32(EPS))))
    assert outside(stale, p_ref, bp).mean() > 0.9
    inside = f32(tables[0] - F64(F32(lr_t(3))) * gm / np.sqrt(gv + F64(F32(EPS))))
    assert outside(inside, p_ref, bp).mean() > 0.9
    # the betas swapped in the moment update
    swapped_m = f32(m0 + (e.ref - m0) * omb(B2))
    assert outside(swapped_m, *moments(m0, v0, e, extra)[:2]).mean() > 0.9
    # dense adam: m of a row the batch did not touch is not decayed (its gradient is exactly 0)
    untouched = hits == 0
    assert untouched.any()
    e0 = e._replace(ref=np.zeros_like(e.ref), scale=np.zeros_like(e.ref), slack=0.0)
    m1, bm, v1, bv = moments(m0, v0, e0)
    assert outside(m0, m1, bm)[untouched].all(axis=1).all()
    assert outside(v0, v1, bv)[untouched].all(axis=1).all()


def test_gradient_bound_of_the_global_bias_rejects_a_missing_contribution():
    """The Adam backward adds the global bias's gradient once per CTA: the bound with that many additions still
    rejects the gradient of one missing CTA's examples."""
    p = _problem([32], "relu", 4099, rows=(97, 7, 300), D=16, seed=2)
    e = deepfm_step(*p)["bias"]
    extra = update_slack(0, 0, 1, adam_bias_additions(4099, 132), e.terms)
    gl = (deepfm_step(*p)["prob"].ref - p[-1]) / 4099
    m1, bm, _, _ = moments(0.0, 0.0, e, extra)
    assert not outside(f32(omb(B1) * f32(gl.sum())), m1, bm)
    assert outside(f32(omb(B1) * f32(gl[8:].sum())), m1, bm)
    assert RTOL * e.scale + extra < abs(e.ref)
