"""float64 / float32 numpy oracle of DIN's layers (reference keras/models/ranking/din.py): `activation_unit`
(ActivationUnit.call, :59-71), `dice` (Dice.call, :110-121), the target attention `din_attention` (the unit at every
position of a sequence plus the weighted sum pooling), their gradients (TensorFlow autodiff of those calls) and the
DIN model forward composed from them.  Shared by the CPU and the GPU tests; the golden vectors in
tests/golden/din_golden.npz pin `activation_unit` and `dice` to the reference's own code."""
import numpy as np

_ACTS = {
    None: lambda z: z, "linear": lambda z: z,
    "relu": lambda z: np.maximum(z, 0),
    "sigmoid": lambda z: 1.0 / (1.0 + np.exp(-z)),
    "tanh": np.tanh,
}


def act_grad_from_y(y, act):
    if act == "relu":
        return (y > 0).astype(y.dtype)
    if act == "sigmoid":
        return y * (1 - y)
    if act == "tanh":
        return 1 - y * y
    return np.ones_like(y)


def interaction(k, q, interact):
    if interact in (None, "none"):
        return None
    return k - q if interact == "subtract" else k * q


def unit_input(k, q, interact):
    """[k | q | f(k, q)] along the last axis (q broadcast over the positions of k)."""
    q = np.broadcast_to(q, k.shape)
    f = interaction(k, q, interact)
    return np.concatenate([k, q] if f is None else [k, q, f], axis=-1)


def dice(x, alpha, eps=1e-8, dtype=np.float64):
    """din.py:112-121 on a rank-2 x: p = sigmoid((x - mean) / sqrt(std + eps)), a = PReLU(x), where(a > 0, p*a,
    (1-p)*a)."""
    x, alpha = np.asarray(x, dtype), np.asarray(alpha, dtype)
    mu = x.mean(axis=1, keepdims=True)
    sd = np.sqrt(((x - mu) ** 2).mean(axis=1, keepdims=True))
    p = 1.0 / (1.0 + np.exp(-((x - mu) / np.sqrt(sd + dtype(eps)))))
    a = np.where(x > 0, x, alpha * x)
    return np.where(a > 0, p * a, (1 - p) * a).astype(dtype)


def dice_grad(x, alpha, gy, eps=1e-8, dtype=np.float64):
    """(gx, galpha) of `dice`; a constant row (std = 0) gets no gradient through the std (TensorFlow: NaN)."""
    x, alpha, gy = (np.asarray(a, dtype) for a in (x, alpha, gy))
    U = x.shape[1]
    mu = x.mean(axis=1, keepdims=True)
    c = x - mu
    sd = np.sqrt((c ** 2).mean(axis=1, keepdims=True))
    den = np.sqrt(sd + eps)
    p = 1.0 / (1.0 + np.exp(-(c / den)))
    a = np.where(x > 0, x, alpha * x)
    pos = a > 0
    ga = gy * np.where(pos, p, 1 - p)
    gz = gy * np.where(pos, a, -a) * p * (1 - p)
    s1 = gz.sum(axis=1, keepdims=True)
    s2 = (gz * c).sum(axis=1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        coef = np.where(sd > 0, (-s2 / den ** 2) / (2 * den * U * sd), 0.0)
    da = np.where(x > 0, 1.0, np.where(x < 0, alpha, 0.0))
    gx = ga * da + gz / den - s1 / den / U + coef * c
    galpha = (ga * np.where(x < 0, x, 0.0)).sum(axis=0)
    return gx.astype(dtype), galpha.astype(dtype)


def activation_unit(x, y, w1, b1, w2, b2, act="relu", interact=None, dtype=np.float64, layer_act=None):
    """din.py:59-71: Dense(1)(act(Dense(U)([x | y | f(x, y)]))) -> [N, 1].  `layer_act` (a callable on [N, U]) replaces
    the named activation (a Layer activation such as Dice)."""
    x, y = np.asarray(x, dtype), np.asarray(y, dtype)
    u = unit_input(x, y, interact)
    z = u @ np.asarray(w1, dtype) + (0 if b1 is None else np.asarray(b1, dtype))
    h = layer_act(z) if layer_act is not None else _ACTS[act](z)
    return (h @ np.asarray(w2, dtype).reshape(-1, 1) + (0 if b2 is None else np.asarray(b2, dtype))).astype(dtype)


def din_attention(keys, query, w1, b1, w2, b2, act="relu", interact="subtract", dtype=np.float64):
    """(pooled [B, D], score [B, T], h [B, T, U]): the unit at every position of keys against query, and
    sum_t score * keys."""
    keys, query = np.asarray(keys, dtype), np.asarray(query, dtype)
    u = unit_input(keys, query[:, None, :], interact)
    z = u @ np.asarray(w1, dtype) + (0 if b1 is None else np.asarray(b1, dtype))
    h = _ACTS[act](z)
    score = h @ np.asarray(w2, dtype).reshape(-1) + (0 if b2 is None else np.asarray(b2, dtype).reshape(()))
    pooled = (score[:, :, None] * keys).sum(axis=1)
    return pooled.astype(dtype), score.astype(dtype), h


def din_attention_abs(keys, query, w1, b1, w2, b2, act="relu", interact="subtract"):
    """(score_abs [B, T], pooled_abs [B, D]): sums of |terms|, the scale the fp32 tolerance is measured against (the
    reference's own terms |k||Wk| + |q||Wq| + |f(k, q)||Wi| + |b1|, carried through |w2| (every activation here is
    1-Lipschitz), plus |h||w2| + |b2|, then (|score| + that) |k| summed over t)."""
    keys, query = np.asarray(keys, np.float64), np.asarray(query, np.float64)
    aw1, aw2 = np.abs(np.asarray(w1, np.float64)), np.abs(np.asarray(w2, np.float64)).reshape(-1)
    z_abs = np.abs(unit_input(keys, query[:, None, :], interact)) @ aw1
    if b1 is not None:
        z_abs = z_abs + np.abs(np.asarray(b1, np.float64))
    _, score, h = din_attention(keys, query, w1, b1, w2, b2, act, interact)
    s_abs = z_abs @ aw2 + np.abs(h) @ aw2 + (0 if b2 is None else abs(float(np.asarray(b2).reshape(()))))
    p_abs = ((s_abs + np.abs(score))[:, :, None] * np.abs(keys)).sum(axis=1)
    return s_abs, p_abs


def din_attention_grad(keys, query, w1, b1, w2, b2, g_pooled=None, g_score=None, act="relu", interact="subtract",
                       dtype=np.float64):
    """(g_keys, g_query, gw1, gb1, gw2, gb2) of `din_attention` given the gradients of pooled and of score."""
    keys, query, w1, w2 = (np.asarray(a, dtype) for a in (keys, query, w1, w2))
    B, T, D = keys.shape
    pooled, score, h = din_attention(keys, query, w1, b1, w2, b2, act, interact, dtype)
    ds = np.zeros((B, T), dtype)
    gk = np.zeros_like(keys)
    if g_score is not None:
        ds = ds + np.asarray(g_score, dtype)
    if g_pooled is not None:
        gp = np.asarray(g_pooled, dtype)
        ds = ds + np.einsum("btd,bd->bt", keys, gp)
        gk = gk + score[:, :, None] * gp[:, None, :]
    w2v = w2.reshape(-1)
    gz = ds[:, :, None] * w2v[None, None, :] * act_grad_from_y(h, act)
    gu = gz @ w1.T                                   # [B, T, (2|3)D]
    qb = np.broadcast_to(query[:, None, :], keys.shape)
    gk = gk + gu[..., :D]
    gq = gu[..., D:2 * D].sum(axis=1)
    if interact == "subtract":
        gk = gk + gu[..., 2 * D:]
        gq = gq - gu[..., 2 * D:].sum(axis=1)
    elif interact == "multiply":
        gk = gk + gu[..., 2 * D:] * qb
        gq = gq + (gu[..., 2 * D:] * keys).sum(axis=1)
    u = unit_input(keys, query[:, None, :], interact)
    gw1 = np.einsum("btk,btu->ku", u, gz)
    gb1 = None if b1 is None else gz.sum(axis=(0, 1))
    gw2 = np.einsum("btu,bt->u", h, ds).reshape(np.shape(w2))
    gb2 = None if b2 is None else np.asarray(ds.sum()).reshape(np.shape(b2))
    return gk, gq, gw1, gb1, gw2, gb2


def din_forward(item_table, ctx_tables, ctx_ids, item_ids, hist_ids, att, mlp, head_w, head_b, dtype=np.float64):
    """The DIN model (Zhou et al., 2018) on `din_attention`: e_item = item_table[item_ids], keys = item_table[hist_ids]
    (an id outside [0, rows) is a zero row), interest = sum_t score * keys, x = [ctx | e_item | interest], an MLP of
    (w, b, act) layers (act "dice" = Dice with its alpha), prob = sigmoid(x @ head_w + head_b).
    att = (w1, b1, w2, b2, act, interact).  Returns (prob, logit)."""
    tab = np.asarray(item_table, dtype)

    def gather(t, ids):
        ids = np.asarray(ids)
        ok = (ids >= 0) & (ids < t.shape[0])
        out = np.zeros(ids.shape + (t.shape[1],), dtype)
        out[ok] = t[ids[ok]]
        return out

    e_item = gather(tab, item_ids)
    keys = gather(tab, hist_ids)
    w1, b1, w2, b2, act, interact = att
    interest, _, _ = din_attention(keys, e_item, w1, b1, w2, b2, act, interact, dtype)
    parts = [e_item, interest]
    if ctx_tables:
        ctx = np.concatenate([gather(np.asarray(t, dtype), np.asarray(ctx_ids)[:, s])
                              for s, t in enumerate(ctx_tables)], axis=1)
        parts.insert(0, ctx)
    x = np.concatenate(parts, axis=1)
    for w, b, a in mlp:
        z = x @ np.asarray(w, dtype) + np.asarray(b, dtype)
        x = dice(z, a, dtype=dtype) if not isinstance(a, str) else _ACTS[a](z)
    logit = (x @ np.asarray(head_w, dtype)).reshape(-1) + np.asarray(head_b, dtype).reshape(())
    return 1.0 / (1.0 + np.exp(-logit)), logit
