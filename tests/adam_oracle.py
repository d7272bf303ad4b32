"""float64 model of the Adam optimizers of DeepFMTrainStep ("adam", "lazy_adam", "adam_rows", "adam_rows_tf") and the
per-element bounds the Adam tests hold the kernels to.

Adam is checked in parts that each have a tight bound, not through its final output (at t = 1 Adam moves a parameter
by about lr * sign(g), whatever |g| is, so the parameters alone cannot show a gradient that is a few percent off):

  * the gradient, read through m and v, which are linear in g and g^2 (`moments`);
  * the update, recomputed from the kernel's own m, v and lr_t (`functor`): a wrong lr_t, eps inside the sqrt, the
    betas swapped or a stale m show here, independently of the gradient;
  * the replay of the steps a row sat out under "adam_rows_tf" (`replay`), as a float64 step-by-step model of dense
    Adam with a zero gradient that is not capped at kCatchUpMax, so the cap itself is tested.

Every function returns float64 values and a bound on |float32 result - value|.  Gradients come as `Entry`s of
tests/deepfm_oracle.py (ref, scale, slack, terms); their own bound is RTOL * scale + slack + `extra`.
"""
import numpy as np

from deepfm_oracle import RTOL, U, Entry, update_slack  # noqa: F401  (Entry, update_slack: for the tests)

F32, F64 = np.float32, np.float64
K_CATCH_UP_MAX = 2048        # embed_adam.cu: steps replayed one by one; later ones only decay m and v in closed form
TINY = 2.0 ** -150           # half the smallest float32 subnormal: the absolute rounding of a result that underflows
# The model's own rounding: p0 - dp in float64 is off by up to 2^-53 |p1|.  Where |dp| is below an ulp of the float32 p
# (a gradient far below eps), the kernel's p1 is p0 and the bound is |dp| itself, so this term matters there.
U64 = 2.0 ** -53

# |float32 result - exact| of the ApplyAdam moment update m + (g - m)(1 - b), per unit of U * (|m0| + |m1|): the
# subtraction, the product and the sum round once each (twice when the compiler contracts them into an FMA); the first
# two are relative to |g - m0| * omb = |m1 - m0| <= |m0| + |m1|, the last to |m1|.  For v the square g*g rounds too,
# relative to omb * g^2 <= |v1| + 2 |v0|.  So 3 suffices for m and 4 for v; 4 covers both.
C_MOMENT = 4
# |float32 result - exact| of lr_t * m / (sqrt(v) + eps) relative to itself: m * lr_t, sqrtf, + eps and / round once each
# (IEEE sqrtf and division: the library is built without fast math), plus the second-order terms.
C_FUNCTOR = 5
# The same quotient in the replay, which divides with __fdividef (at most 2 ulps = 4 U inside [2^-126, 2^126]): 7 U.
C_REPLAY_STEP = 7


def f32(x):
    """float32 value of x, as float64."""
    return np.asarray(x, F32).astype(F64)


def omb(beta):
    """1 - beta formed in float32, as the kernels (and TF's functor, `T(1) - beta()`) form it."""
    return F64(F32(1.0) - F32(beta))


def lr_t(t, lr=0.01, b1=0.9, b2=0.999):
    """Keras Adam's bias-corrected rate lr * sqrt(1 - b2^t) / (1 - b1^t) at step t (t >= 1), float64, with lr and the
    betas as the float32 values the kernels receive."""
    t = np.asarray(t, F64)
    b1, b2 = F64(F32(b1)), F64(F32(b2))
    return F64(F32(lr)) * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)


def adam_bias_additions(B, num_sms):
    """Float32 additions dr_embed_fm_bwd_adam(_tf) makes to the global bias's gradient: one per CTA, and it launches
    one CTA per 8 examples (8 warps of 256 threads, a warp per example), at most 8 per SM."""
    return min(-(-B // 8), 8 * num_sms)


def grad_bound(e: Entry, extra=0.0, rtol=RTOL):
    """The bound of a float32 gradient against its Entry: rtol * scale + slack + extra."""
    return rtol * np.asarray(e.scale, F64) + e.slack + extra


def moments(m0, v0, e: Entry, extra=0.0, b1=0.9, b2=0.999, m0_err=0.0, v0_err=0.0, rtol=RTOL):
    """m1, v1 of the ApplyAdam functor from the kernel's pre-step moments m0, v0 and the oracle gradient e.ref.

    `extra` is the gradient's rounding beyond RTOL * scale + slack (for a row gradient summed by `hits` separate float32
    additions into a zeroed buffer: update_slack(0, 0, 1, hits, e.terms)); `m0_err`, `v0_err` bound m0, v0 when they
    are themselves modelled (the replayed moments of "adam_rows_tf").  Returns (m1, m1 bound, v1, v1 bound)."""
    m0, v0, g = (np.asarray(a, F64) for a in (m0, v0, e.ref))
    o1, o2 = omb(b1), omb(b2)
    m1 = m0 + (g - m0) * o1
    v1 = v0 + (g * g - v0) * o2
    eg = grad_bound(e, extra, rtol)
    bm = o1 * eg + (1 - o1) * m0_err + C_MOMENT * U * (np.abs(m0) + np.abs(m1))
    bv = o2 * (2 * np.abs(g) * eg + eg * eg) + (1 - o2) * v0_err + C_MOMENT * U * (np.abs(v0) + np.abs(v1))
    return m1, bm, v1, bv


def functor(p0, m1, v1, lr_t_, eps=1e-7, p0_err=0.0):
    """p1 = p0 - lr_t * m1 / (sqrt(v1) + eps) in float64 from the kernel's own m1, v1 and lr_t (clock.lr_t).

    Bound: C_FUNCTOR U of |dp| for the quotient, plus U |p1| for the final subtraction (never more than |dp| itself:
    p0 is one of the candidates the subtraction rounds to), plus `p0_err` when p0 is modelled, plus the float64
    rounding of p1 itself (U64 |p1|).  Returns (p1, bound)."""
    p0, m1, v1 = (np.asarray(a, F64) for a in (p0, m1, v1))
    dp = F64(lr_t_) * m1 / (np.sqrt(v1) + F64(F32(eps)))
    p1 = p0 - dp
    b = C_FUNCTOR * U * np.abs(dp) + np.minimum(U * np.abs(p1), np.abs(dp)) + p0_err + U64 * np.abs(p1)
    return p1, b


def lr_err(j, t_now, hist_len, b1=0.9, b2=0.999):
    """Relative error of the rate adam_lr_at gives the replay of step j at step t_now.

    Ring hit (t_now - j < hist_len): the ring holds float32(lr_j) of a double-precision formula (dr_adam_advance_hist):
    U, doubled for the double pow.  Recompute: lr * sqrtf(1 - powf(b2, j)) / (1 - powf(b1, j)) in float32.  powf is
    within 4 ulps (<= 8 U relative) of b^j, and 1 - b^j cancels: its relative error is 8 U b^j / (1 - b^j) + U.  The
    sqrt halves its argument's error and rounds (U); the division and the product with lr round once each:
        8 U (b2^j / (2 (1 - b2^j)) + b1^j / (1 - b1^j)) + 5 U   (U/2 + U + U + U + U, rounded up)."""
    j = np.asarray(j, F64)
    b1, b2 = F64(F32(b1)), F64(F32(b2))
    p1, p2 = b1 ** j, b2 ** j
    rec = 8 * U * (p2 / (2 * (1 - p2)) + p1 / (1 - p1)) + 5 * U
    hit = (t_now - j < hist_len) if hist_len else np.zeros(np.shape(j), bool)
    return np.where(hit, 2 * U, rec)


def replay(p, m, v, stamp, upto, lr=0.01, b1=0.9, b2=0.999, eps=1e-7, t_now=None, hist_len=0):
    """Dense Adam with a zero gradient for every step j in (stamp, upto] -- what tf.keras Adam does to a row in the
    steps that do not touch it -- in float64, NOT capped at kCatchUpMax.

    p, m, v: [rows, n] (float32 values), stamp: [rows] (<= 0: never updated, nothing to replay).  t_now / hist_len say
    which rates came from the ring (see `lr_err`).  Returns (p, m, v, bound p, bound m, bound v), float64.

    Bound, summed per replayed step j (the k-th of the row):
      * m and v decay by one FMA each, so their relative error grows by U per step (plus TINY absolute once they
        underflow);
      * the step's |dp_j| carries lr_err(j) + C_REPLAY_STEP U + m's relative error + half of v's, and the subtraction
        rounds by at most min(U |p_j|, |dp_j|) (plus U64 |p_j| for the model's own float64 rounding);
      * beyond kCatchUpMax steps the kernel no longer moves p: the bound takes the float64 |dp_j| of every such step
        (that sum is what the cap's claim "cannot move the row any more" is checked against), and m, v decay in closed
        form by powf(1 - omb, gap - 2048): 8 U for powf, U for the product, and (gap - 2048) times the relative
        error of 1 - omb itself, which is 0 for the default betas (1 - (1 - b) is exact there)."""
    p, m, v = (np.array(a, F64, copy=True) for a in (p, m, v))
    stamp = np.asarray(stamp, np.int64).reshape(-1)
    rows = p.shape[0]
    bp, bm, bv = np.zeros_like(p), np.zeros_like(m), np.zeros_like(v)
    o1, o2 = omb(b1), omb(b2)
    gap = np.where(stamp > 0, np.maximum(np.asarray(upto, np.int64) - stamp, 0), 0)
    t_now = upto if t_now is None else t_now
    e32 = F64(F32(eps))
    rm = np.zeros_like(m)                # relative error of m (v) so far
    rv = np.zeros_like(v)
    am = np.zeros_like(m)                # absolute floor from underflow
    av = np.zeros_like(v)
    for k in range(1, int(gap.max(initial=0)) + 1):
        act = (gap >= k).reshape(rows, *([1] * (p.ndim - 1)))
        j = (stamp + k).astype(F64).reshape(act.shape)
        m_new = m - m * o1
        v_new = v - v * o2
        lj = lr_t(j, lr, b1, b2)
        dp = lj * m_new / (np.sqrt(v_new) + e32)
        capped = k > K_CATCH_UP_MAX
        if not capped:
            rm_new, rv_new = rm + U, rv + U
            am_new, av_new = am + TINY, av + TINY
            rel = lr_err(j, t_now, hist_len, b1, b2) + C_REPLAY_STEP * U + rm_new + 0.5 * rv_new
            err_dp = np.abs(dp) * rel + lj * am_new / e32
            p_new = p - dp
            bp = np.where(act, bp + err_dp + np.minimum(U * np.abs(p_new), np.abs(dp) + err_dp) + U64 * np.abs(p_new),
                          bp)
            rm, rv = np.where(act, rm_new, rm), np.where(act, rv_new, rv)
            am, av = np.where(act, am_new, am), np.where(act, av_new, av)
        else:
            p_new = p - dp
            bp = np.where(act, bp + np.abs(dp), bp)
        p = np.where(act, p_new, p)
        m = np.where(act, m_new, m)
        v = np.where(act, v_new, v)
    bm = rm * np.abs(m) + am
    bv = rv * np.abs(v) + av
    over = (gap > K_CATCH_UP_MAX).reshape(rows, *([1] * (p.ndim - 1)))
    if over.any():
        extra_steps = (gap - K_CATCH_UP_MAX).reshape(over.shape).astype(F64)
        for o, mm, b in ((o1, m, bm), (o2, v, bv)):
            base = F64(F32(1.0) - F32(o))
            d_base = abs(base - (1.0 - o)) / (1.0 - o)
            b += np.where(over, (9 * U + extra_steps * d_base) * np.abs(mm) + TINY, 0.0)
    return p, m, v, bp, bm, bv


def check_bound(name, got, ref, bound):
    """Assert |got - ref| <= bound per element (NaN is outside); the message names the worst element.  Returns the
    largest err / bound (the share of its bound the result used; 0 where the bound is 0 and the result exact)."""
    got, ref = np.asarray(got, F64), np.asarray(ref, F64)
    bound = np.broadcast_to(np.asarray(bound, F64), ref.shape)
    got = got.reshape(ref.shape)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    if bad.any():
        idx = np.unravel_index(np.argmax(np.where(bad, np.nan_to_num(err - bound, nan=np.inf), -np.inf)), ref.shape)
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.size} elements outside the bound; worst at {idx}: "
                             f"got {got[idx]!r} want {ref[idx]!r} bound {bound[idx]!r}")
    nz = bound > 0
    return float((err[nz] / bound[nz]).max()) if nz.any() else 0.0


def outside(got, ref, bound):
    """Boolean mask of the elements outside |got - ref| <= bound."""
    return ~(np.abs(np.asarray(got, F64) - np.asarray(ref, F64)) <= np.asarray(bound, F64))
