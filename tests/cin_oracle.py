"""float64 / float32 numpy oracle of xDeepFM's CIN layer (reference keras/models/ranking/xdeepfm.py:71-96) and of its
gradient (TensorFlow autodiff of that call), and the xDeepFM forward composed from it.  Shared by the CPU and the GPU
tests; the golden vectors in tests/golden/cin_golden.npz pin `cin` to the reference's own code."""
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


def cin(x0, x, w, b=None, act="sigmoid", dtype=np.float64):
    """y [B, H, D] = act(sum_{i,j} w[0, i*h+j, k] * x0[b,i,d] * x[b,j,d] + b[k]): xdeepfm.py:82-96 (the outer product
    in its reshape order i*h + j, the width-1 VALID conv1d, bias_add, activation, final transpose)."""
    x0, x, w = (np.asarray(a, dtype) for a in (x0, x, w))
    m, h = x0.shape[1], x.shape[1]
    wk = w.reshape(m, h, -1)
    z = np.einsum("bid,bjd,ijk->bkd", x0, x, wk, optimize=True)
    if b is not None:
        z = z + np.asarray(b, dtype)[None, :, None]
    return _ACTS[act](z).astype(dtype)


def cin_grad(x0, x, w, y, gy=None, gpool=None, act="sigmoid", dtype=np.float64):
    """(gx0, gx, gw [1, m*h, H], gb) of the CIN call given its output y and the gradients of y and of sum_d y."""
    x0, x, w, y = (np.asarray(a, dtype) for a in (x0, x, w, y))
    m, h = x0.shape[1], x.shape[1]
    wk = w.reshape(m, h, -1)
    g = np.zeros_like(y)
    if gy is not None:
        g = g + np.asarray(gy, dtype)
    if gpool is not None:
        g = g + np.asarray(gpool, dtype)[:, :, None]
    g = g * act_grad_from_y(y, act)
    gx0 = np.einsum("ijk,bjd,bkd->bid", wk, x, g, optimize=True)
    gx = np.einsum("ijk,bid,bkd->bjd", wk, x0, g, optimize=True)
    gw = np.einsum("bid,bjd,bkd->ijk", x0, x, g, optimize=True).reshape(1, m * h, -1)
    gb = g.sum(axis=(0, 2))
    return gx0, gx, gw, gb, g



def xdeepfm_forward(tables, lins, bias, ids, cin_ws, cin_act, dnn_ws, dnn_bs, dnn_act, head_w, head_b,
                    dtype=np.float64):
    """The XDeepFM model (Lian et al., 2018) on `cin`: linear = bias + sum_s lins[s][id], x0 = the [B, S, D] stack
    (an id outside [0, rows) is a zero row with a zero weight), x_k = cin((x0, x_{k-1})) sum-pooled over d, a DNN on
    flatten(x0), prob = sigmoid(Dense(1)([pools | deep]) + linear).  Returns (prob, logit)."""
    ids = np.asarray(ids)
    B, S = ids.shape
    D = np.asarray(tables[0]).shape[1]
    x0 = np.zeros((B, S, D), dtype)
    lin = np.full(B, float(bias), dtype)
    for s in range(S):
        t, l = np.asarray(tables[s], dtype), np.asarray(lins[s], dtype)
        ok = (ids[:, s] >= 0) & (ids[:, s] < t.shape[0])
        x0[ok, s] = t[ids[ok, s]]
        lin[ok] += l[ids[ok, s]]
    x, pools = x0, []
    for w in cin_ws:
        x = cin(x0, x, w, None, cin_act, dtype)
        pools.append(x.sum(axis=2))
    h = x0.reshape(B, -1)
    for w, b in zip(dnn_ws, dnn_bs):
        h = _ACTS[dnn_act](h @ np.asarray(w, dtype) + np.asarray(b, dtype))
    feat = np.concatenate(pools + [h], axis=1)
    logit = (feat @ np.asarray(head_w, dtype)).reshape(-1) + np.asarray(head_b, dtype).reshape(()) + lin
    return 1.0 / (1.0 + np.exp(-logit)), logit
