"""Float64 restatement of the reference's FNN (estimator/models/ranking/fnn.py:50-90, dnn.py) and of its training
step with tf.losses.log_loss and tf.train.AdamOptimizer (examples/train_fnn_on_movielens_estimator.py:36-53).

Fields are given as per-slot, per-example id lists (a single-valued field has one id per example): the embedding is
the mean of the valid rows (embedding_column's default combiner; ids < 0 or >= rows are pruned, an empty bag gives
zeros) and w is the SUM of their first-order weights (the indicator column is a multi-hot count vector times the
field's [rows, 1] kernel).  The tower input is concat([bias, w_1..w_S, e_1..e_S]); `pad_row` / `pad_kernel` move it
and layer 0's kernel to the padded layout dr_fnn_input_fwd writes (P = round_up(1 + S, 4), zeros at 1+S..P-1).
"""
import numpy as np


def layout(S, D):
    P = (1 + S + 3) // 4 * 4
    return P, P + S * D


def _valid(ids, n):
    return [int(i) for i in ids if 0 <= int(i) < n]


def input_row(tables, lins, bias, per_slot_ids):
    """-> x [B, 1 + S + S*D] in the reference's column order."""
    S, D = len(tables), tables[0].shape[1]
    B = len(per_slot_ids[0])
    w = np.zeros((B, S))
    e = np.zeros((B, S * D))
    for s, (t, l, per_ex) in enumerate(zip(tables, lins, per_slot_ids)):
        for b in range(B):
            ok = _valid(per_ex[b], t.shape[0])
            if ok:
                w[b, s] = np.sum(np.asarray(l, dtype=np.float64)[ok])
                e[b, s * D:(s + 1) * D] = np.asarray(t, dtype=np.float64)[ok].mean(axis=0)
    return np.concatenate([np.full((B, 1), float(np.asarray(bias).reshape(-1)[0])), w, e], axis=1)


def pad_row(x, S, D):
    P, ld = layout(S, D)
    out = np.zeros((x.shape[0], ld))
    out[:, :1 + S] = x[:, :1 + S]
    out[:, P:] = x[:, 1 + S:]
    return out


def unpad_row(xp, S, D):
    P, _ = layout(S, D)
    return np.concatenate([xp[:, :1 + S], xp[:, P:]], axis=1)


def pad_kernel(k0, S, D):
    P, ld = layout(S, D)
    out = np.zeros((ld, k0.shape[1]))
    out[:1 + S] = k0[:1 + S]
    out[P:] = k0[1 + S:]
    return out


def input_grad(g_x, rows, D, per_slot_ids, scale=1.0):
    """Backward of input_row: g_x [B, 1 + S + S*D] (reference order) -> (d tables [S] of [rows, D], d lins [S] of
    [rows]).  The bias column gets no gradient (a constant of the model)."""
    S = len(rows)
    B = g_x.shape[0]
    gt = [np.zeros((n, D)) for n in rows]
    gl = [np.zeros(n) for n in rows]
    for s in range(S):
        for b in range(B):
            ok = _valid(per_slot_ids[s][b], rows[s])
            for i in ok:
                gt[s][i] += scale * g_x[b, 1 + S + s * D:1 + S + (s + 1) * D] / len(ok)
                gl[s][i] += scale * g_x[b, 1 + s]
    return gt, gl


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


def tower_forward(x, ws, bs, act="relu"):
    """dnn(x, units + [1]): activation on every layer but the last.  Returns the activations [x, h_1, .., z]."""
    hs = [x]
    for i, (w, b) in enumerate(zip(ws, bs)):
        z = hs[-1] @ w + b
        hs.append(_act(z, act) if i < len(ws) - 1 else z)
    return hs


def forward(state, per_slot_ids, act="relu"):
    """state: dict(tables, lins, bias, ws, bs) (layer 0 over the reference's 1 + S + S*D inputs) -> (x, hs, p [B])."""
    x = input_row(state["tables"], state["lins"], state["bias"], per_slot_ids)
    hs = tower_forward(x, state["ws"], state["bs"], act)
    return x, hs, 1.0 / (1.0 + np.exp(-hs[-1][:, 0]))


def log_loss(p, y, eps=1e-7):
    """tf.losses.log_loss with its default epsilon and mean reduction."""
    return float(np.mean(-y * np.log(p + eps) - (1 - y) * np.log(1 - p + eps)))


def grads(state, per_slot_ids, y, act="relu", eps=1e-7):
    """-> (loss, p, d tables, d lins, d ws, d bs) of the log loss of sigmoid(tower(x))."""
    y = np.asarray(y, dtype=np.float64)
    B = len(y)
    x, hs, p = forward(state, per_slot_ids, act)
    loss = log_loss(p, y, eps)
    g_p = (-y / (p + eps) + (1 - y) / (1 - p + eps)) / B
    g = (g_p * p * (1 - p))[:, None]
    gws, gbs = [], []
    for i in range(len(state["ws"]) - 1, -1, -1):
        if i < len(state["ws"]) - 1:
            g = g * _act_grad(hs[i + 1], act)
        gws.insert(0, hs[i].T @ g)
        gbs.insert(0, g.sum(axis=0))
        g = g @ state["ws"][i].T
    rows = [t.shape[0] for t in state["tables"]]
    gt, gl = input_grad(g, rows, state["tables"][0].shape[1], per_slot_ids)
    return loss, p, gt, gl, gws, gbs


def adam_step(state, per_slot_ids, y, lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8, act="relu"):
    """One step of TF1 ApplyAdam over every FNN variable (whole tables: untouched rows decay with their moments).
    Updates state in place (state["adam"], state["t"]) and returns (loss, p)."""
    loss, p, gt, gl, gws, gbs = grads(state, per_slot_ids, y, act)
    params = state["tables"] + state["lins"] + state["ws"] + state["bs"]
    gq = gt + gl + gws + gbs
    if state.get("adam") is None:
        state["adam"] = {"m": [np.zeros_like(q) for q in params], "v": [np.zeros_like(q) for q in params]}
    state["t"] = state.get("t", 0) + 1
    t = state["t"]
    lr_t = lr * np.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
    new = []
    for q, g, m, v in zip(params, gq, state["adam"]["m"], state["adam"]["v"]):
        m += (g - m) * (1 - beta1)
        v += (g * g - v) * (1 - beta2)
        new.append(q - lr_t * m / (np.sqrt(v) + eps))
    S, L = len(state["tables"]), len(state["ws"])
    state["tables"], state["lins"] = new[:S], new[S:2 * S]
    state["ws"], state["bs"] = new[2 * S:2 * S + L], new[2 * S + L:]
    return loss, p
