"""float64 restatement of tf.keras.optimizers.Adam with a learning rate per step -- the oracle optimizers.KerasAdam is held
to -- built on the per-element bounds of tests/adam_oracle.py.

Keras (optimizer_v2/adam.py, ApplyAdam) folds the bias correction into the rate and adds eps to sqrt(v):
    lr_t = lr_t_step * sqrt(1 - b2^t) / (1 - b1^t),  m += (g - m)(1 - b1),  v += (g^2 - v)(1 - b2),
    p -= lr_t m / (sqrt(v) + eps)
torch.optim.Adam divides by sqrt(v / (1 - b2^t)) + eps instead, i.e. its effective eps is eps * sqrt(1 - b2^t)."""
import numpy as np

from adam_oracle import C_REPLAY_STEP, TINY, U, U64, lr_t, omb

F32, F64 = np.float32, np.float64


def keras_adam(p, grads, lrs, b1=0.9, b2=0.999, eps=1e-7):
    """Dense Keras Adam from p over the gradients grads[t - 1] at the rates lrs[t - 1], t = 1, 2, ...; float64 (p, m, v)."""
    p = np.array(p, F64, copy=True)
    m, v = np.zeros_like(p), np.zeros_like(p)
    for t, (g, lr) in enumerate(zip(grads, lrs), 1):
        g = np.asarray(g, F64)
        lt = lr * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
        m = m + (g - m) * (1.0 - b1)
        v = v + (g * g - v) * (1.0 - b2)
        p = p - lt * m / (np.sqrt(v) + eps)
    return p, m, v


def replay_sched(p, m, v, stamp, upto, lrs, b1=0.9, b2=0.999, eps=1e-7):
    """adam_oracle.replay for rows whose skipped steps j in (stamp, upto] take the rate of their own step, lrs[j - 1],
    every one of them from the clock's ring (float32 of a double-precision formula: 2 U).  Gaps stay below kCatchUpMax.
    Returns (p, m, v, bound p, bound m, bound v), float64."""
    p, m, v = (np.array(a, F64, copy=True) for a in (p, m, v))
    stamp = np.asarray(stamp, np.int64).reshape(-1)
    rows = p.shape[0]
    bp = np.zeros_like(p)
    o1, o2 = omb(b1), omb(b2)
    gap = np.where(stamp > 0, np.maximum(int(upto) - stamp, 0), 0)
    e32 = F64(F32(eps))
    rm, rv, am, av = (np.zeros_like(m) for _ in range(4))
    sched = np.asarray([lr_t(j, lrs[j - 1], b1, b2) for j in range(1, int(upto) + 1)], F64)
    for k in range(1, int(gap.max(initial=0)) + 1):
        act = (gap >= k).reshape(rows, *([1] * (p.ndim - 1)))
        j = np.clip(stamp + k, 1, max(int(upto), 1)).reshape(act.shape)
        lj = sched[j - 1]
        m_new = m - m * o1
        v_new = v - v * o2
        dp = lj * m_new / (np.sqrt(v_new) + e32)
        rm_new, rv_new = rm + U, rv + U
        am_new, av_new = am + TINY, av + TINY
        err_dp = np.abs(dp) * (2 * U + C_REPLAY_STEP * U + rm_new + 0.5 * rv_new) + lj * am_new / e32
        p_new = p - dp
        bp = np.where(act, bp + err_dp + np.minimum(U * np.abs(p_new), np.abs(dp) + err_dp) + U64 * np.abs(p_new), bp)
        rm, rv = np.where(act, rm_new, rm), np.where(act, rv_new, rv)
        am, av = np.where(act, am_new, am), np.where(act, av_new, av)
        p, m, v = np.where(act, p_new, p), np.where(act, m_new, m), np.where(act, v_new, v)
    return p, m, v, bp, rm * np.abs(m) + am, rv * np.abs(v) + av
