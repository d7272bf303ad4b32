"""Float64 numpy restatement of the Wide & Deep train step of examples/train_wdl_on_movielens_estimator.py, written
from TensorFlow's documented semantics (independent of the CUDA code):

  crosses       tf.feature_column.crossed_column: FingerprintCat64 chain from hash_key over Fingerprint64(string) /
                raw int64 per key, mod N; a dense key drops empty strings and -1, a multi-valued (sparse) key keeps
                them; cartesian product, last key fastest
  wide          linear_model: bias + sum of w over the example's ids (indicator multi-hot counts duplicates)
  deep          mean-combined embeddings concatenated, dense tower (activation on all but the last layer)
  loss          tf.losses.log_loss: mean(-y log(p + 1e-7) - (1 - y) log(1 - p + 1e-7)), p = sigmoid(wide + deep)
  ftrl          ApplyFtrl (learning_rate_power = -0.5) over WHOLE tables, as TensorFlow applies it to the dense
                gradient of linear_model's weights
  adam          tf.train.AdamOptimizer (TF1 form: lr_t = lr sqrt(1 - b2^t) / (1 - b1^t), eps outside the sqrt)
"""
import numpy as np

from oracle.farmhash_py import fingerprint64

M64 = (1 << 64) - 1
K_MUL = 0xC6A4A7935BD1E995
DEFAULT_HASH_KEY = 0xDECAFCAFFE


def _shift_mix(v):
    return v ^ (v >> 47)


def fingerprint_cat64(a, b):
    r = a ^ K_MUL
    r ^= (_shift_mix((b * K_MUL) & M64) * K_MUL) & M64
    r = (r * K_MUL) & M64
    r = (_shift_mix(r) * K_MUL) & M64
    return _shift_mix(r)


def _value_hash(v):
    if isinstance(v, (bytes, str)):
        return fingerprint64(v.encode() if isinstance(v, str) else v)
    return int(v) & M64


def _kept(v):
    if isinstance(v, (bytes, str)):
        return len(v) > 0
    return int(v) != -1


def cross_example(values_per_key, num_buckets, hash_key=DEFAULT_HASH_KEY, ragged=None):
    """values_per_key: one list of raw values per key, for ONE example -> list of crossed ids (TF order).
    ragged[k]: key k is multi-valued (a SparseTensor in TensorFlow), which keeps '' and -1; a dense key drops them."""
    ragged = ragged or [False] * len(values_per_key)
    kept = [[_value_hash(v) for v in vals if r or _kept(v)] for vals, r in zip(values_per_key, ragged)]
    out = [hash_key]
    for fs in kept:          # cartesian product, last key fastest
        out = [fingerprint_cat64(h, f) for h in out for f in fs]
    return [h % num_buckets for h in out]


def cross_batch(key_lists, num_buckets, hash_key=DEFAULT_HASH_KEY, ragged=None):
    """key_lists: per key, a per-example list of value lists -> (flat ids, row_splits).  ragged as in cross_example
    (default: a key is multi-valued when some example does not have exactly one value)."""
    B = len(key_lists[0])
    if ragged is None:
        ragged = [any(len(v) != 1 for v in k) for k in key_lists]
    ids, splits = [], [0]
    for b in range(B):
        ids += cross_example([k[b] for k in key_lists], num_buckets, hash_key, ragged)
        splits.append(len(ids))
    return np.asarray(ids, dtype=np.int64), np.asarray(splits, dtype=np.int64)


def wide_lookups(slots, B):
    """slots: per slot (rows, offset, per-example id lists) -> list per example of global rows (OOV dropped)."""
    out = [[] for _ in range(B)]
    for rows, off, per_ex in slots:
        for b in range(B):
            out[b] += [off + int(i) for i in per_ex[b] if 0 <= int(i) < rows]
    return out


def wide_forward(w, bias, lookups):
    return np.asarray([bias + sum(w[r] for r in rs) for rs in lookups], dtype=np.float64)


def wide_grad(total_rows, lookups, g_logit):
    g = np.zeros(total_rows, dtype=np.float64)
    for b, rs in enumerate(lookups):
        for r in rs:
            g[r] += g_logit[b]
    return g, float(np.sum(g_logit))


def ftrl_dense(w, z, n, g, lr, l1, l2):
    """ApplyFtrl with learning_rate_power = -0.5 on whole arrays (returns new w, z, n)."""
    n_new = n + g * g
    z = z + g - (np.sqrt(n_new) - np.sqrt(n)) / lr * w
    x = l1 * np.sign(z) - z
    y = np.sqrt(n_new) / lr + 2.0 * l2
    w = np.where(np.abs(z) > l1, x / y, 0.0)
    return w, z, n_new


def ftrl_rows(w, z, n, g, rows, lr, l1, l2):
    """The same update applied only to `rows` (the row-sparse form)."""
    w, z, n = w.copy(), z.copy(), n.copy()
    rows = np.asarray(sorted(set(rows)), dtype=np.int64)
    if rows.size:
        w[rows], z[rows], n[rows] = ftrl_dense(w[rows], z[rows], n[rows], g[rows], lr, l1, l2)
    return w, z, n


def _act(x, act):
    if act == "relu":
        return np.maximum(x, 0.0)
    if act == "sigmoid":
        return 1.0 / (1.0 + np.exp(-x))
    if act == "tanh":
        return np.tanh(x)
    return x


def _act_grad(y, act):
    if act == "relu":
        return (y > 0).astype(np.float64)
    if act == "sigmoid":
        return y * (1.0 - y)
    if act == "tanh":
        return 1.0 - y * y
    return np.ones_like(y)


def deep_embed(tables, per_slot_ids):
    """tables [S] of [rows, D]; per_slot_ids [S] per-example id lists -> [B, S*D] mean-combined (OOV pruned)."""
    B = len(per_slot_ids[0])
    out = []
    for t, per_ex in zip(tables, per_slot_ids):
        e = np.zeros((B, t.shape[1]))
        for b in range(B):
            ok = [int(i) for i in per_ex[b] if 0 <= int(i) < t.shape[0]]
            if ok:
                e[b] = t[ok].mean(axis=0)
        out.append(e)
    return np.concatenate(out, axis=1)


def tower_forward(x, ws, bs, act):
    hs = [x]
    for i, (w, b) in enumerate(zip(ws, bs)):
        z = hs[-1] @ w + b
        hs.append(_act(z, act) if i < len(ws) - 1 else z)
    return hs


def log_loss(p, y, eps=1e-7):
    return float(np.mean(-y * np.log(p + eps) - (1 - y) * np.log(1 - p + eps)))


def step(state, batch, act="relu", lr_ftrl=0.01, l1=0.5, l2=0.0, lr_adam=0.01, eps_adam=1e-8):
    """One WDL train step in float64.  state: dict(w, z, n, bias_wzn [3], tables [S], ws, bs, adam dict or None, t).
    batch: dict(wide_slots = [(rows, offset, per-example id lists)], deep_ids = per-slot per-example id lists,
    y [B]).  Returns (loss, prob) and updates state in place."""
    B = len(batch["y"])
    y = np.asarray(batch["y"], dtype=np.float64)
    look = wide_lookups(batch["wide_slots"], B)
    wide = wide_forward(state["w"], state["bias_wzn"][0], look)
    x = deep_embed(state["tables"], batch["deep_ids"])
    hs = tower_forward(x, state["ws"], state["bs"], act)
    logit = wide + hs[-1][:, 0]
    p = 1.0 / (1.0 + np.exp(-logit))
    loss = log_loss(p, y)
    eps = 1e-7
    g_p = (-y / (p + eps) + (1 - y) / (1 - p + eps)) / B
    g_logit = g_p * p * (1 - p)
    # wide gradients and FTRL over the whole table (+ bias)
    g_w, g_b = wide_grad(state["w"].size, look, g_logit)
    state["w"], state["z"], state["n"] = ftrl_dense(state["w"], state["z"], state["n"], g_w, lr_ftrl, l1, l2)
    bw, bz, bn = ftrl_dense(*(np.asarray([v]) for v in state["bias_wzn"]), np.asarray([g_b]), lr_ftrl, l1, l2)
    state["bias_wzn"] = np.asarray([bw[0], bz[0], bn[0]])
    # deep gradients
    g = g_logit[:, None]
    gws, gbs = [], []
    for i in range(len(state["ws"]) - 1, -1, -1):
        if i < len(state["ws"]) - 1:
            g = g * _act_grad(hs[i + 1], act)
        gws.insert(0, hs[i].T @ g)
        gbs.insert(0, g.sum(axis=0))
        g = g @ state["ws"][i].T
    D = state["tables"][0].shape[1]
    g_tables = [np.zeros_like(t) for t in state["tables"]]
    for s, (t, per_ex) in enumerate(zip(state["tables"], batch["deep_ids"])):
        for b in range(B):
            ok = [int(i) for i in per_ex[b] if 0 <= int(i) < t.shape[0]]
            for i in ok:
                g_tables[s][i] += g[b, s * D:(s + 1) * D] / len(ok)
    # TF1 Adam on every deep variable (dense: untouched embedding rows decay too)
    params = state["tables"] + state["ws"] + state["bs"]
    grads = g_tables + gws + gbs
    if state.get("adam") is None:
        state["adam"] = {"m": [np.zeros_like(q) for q in params], "v": [np.zeros_like(q) for q in params]}
    state["t"] = state.get("t", 0) + 1
    t = state["t"]
    lr_t = lr_adam * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    new = []
    for q, gq, m, v in zip(params, grads, state["adam"]["m"], state["adam"]["v"]):
        m += (gq - m) * (1 - 0.9)
        v += (gq * gq - v) * (1 - 0.999)
        new.append(q - lr_t * m / (np.sqrt(v) + eps_adam))
    S, L = len(state["tables"]), len(state["ws"])
    state["tables"], state["ws"], state["bs"] = new[:S], new[S:S + L], new[S + L:]
    return loss, p
