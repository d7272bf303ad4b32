"""Float64 restatement of the GCN layer (reference keras/models/retrieval/gcn.py:43-55), forward and backward.

forward:  S = A @ X;  Z = S @ W + b;  Y = act(Z);  out = Y + X when residual
backward: gZ = act'(Y) * g (softmax: Y * (g - sum(g * Y)) per row);  gb = colsum(gZ);  gW = S^T gZ;
          gX = A^T (gZ W^T) (+ g when residual).  No gradient reaches A.
"""
import numpy as np

ACTS = ("linear", "relu", "sigmoid", "tanh", "softmax")


def act_fwd(z, act):
    if act in (None, "linear"):
        return z
    if act == "relu":
        return np.maximum(z, 0)
    if act == "sigmoid":
        return 1 / (1 + np.exp(-z))
    if act == "tanh":
        return np.tanh(z)
    if act == "softmax":
        e = np.exp(z - z.max(axis=-1, keepdims=True))
        return e / e.sum(axis=-1, keepdims=True)
    raise ValueError(act)


def act_bwd(y, g, act):
    if act in (None, "linear"):
        return g
    if act == "relu":
        return g * (y > 0)
    if act == "sigmoid":
        return g * y * (1 - y)
    if act == "tanh":
        return g * (1 - y * y)
    if act == "softmax":
        return y * (g - (g * y).sum(axis=-1, keepdims=True))
    raise ValueError(act)


def gcn_forward(adj, x, w, b, act, residual):
    adj, x, w = (np.asarray(t, np.float64) for t in (adj, x, w))
    s = adj @ x
    z = s @ w
    if b is not None:
        z = z + np.asarray(b, np.float64)
    y = act_fwd(z, act)
    return (y + x if residual else y), (s, y)


def gcn_backward(adj, x, w, act, residual, saved, g):
    s, y = saved
    adj, w, g = (np.asarray(t, np.float64) for t in (adj, w, g))
    gz = act_bwd(y, g, act)
    gx = adj.T @ (gz @ w.T)
    if residual:
        gx = gx + g
    return gx, s.T @ gz, gz.sum(axis=0)


def spmm_fwd(indptr, indices, values, n_cols, x, bias=None, residual=None, act="linear"):
    """act(A @ x + bias) (+ residual) from CSR arrays, in float64: duplicates summed, out-of-range columns dropped."""
    x = np.asarray(x, np.float64)
    n_rows = len(indptr) - 1
    a = np.zeros((n_rows, n_cols))
    rows = np.repeat(np.arange(n_rows), np.diff(indptr))
    ok = (indices >= 0) & (indices < n_cols)
    np.add.at(a, (rows[ok], np.asarray(indices)[ok]), np.asarray(values, np.float64)[ok])
    z = a @ x
    if bias is not None:
        z = z + np.asarray(bias, np.float64)
    y = act_fwd(z, act)
    return y, (None if residual is None else y + np.asarray(residual, np.float64))
