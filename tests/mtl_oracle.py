"""numpy float64 restatement of the multi-task models (reference estimator/models/multi_task_learning/
mixture_of_experts.py, esmm.py on estimator/models/feature_interaction/dnn.py), forward and analytic backward.

Weights are lists in the reference's creation order: for MMoE every expert tower (bottom layer first), then all
num_experts gates (kernel only; the first num_tasks are used), then every task tower; for ESMM the pCVR tower, then the
pCTR tower.  A tower's hidden layers use the activation, its last layer is linear.  The tests pin this file to
tests/golden/mtl_golden.npz (the reference run under the numpy TensorFlow stand-in) and to torch float64 autograd.
"""
import numpy as np


def input_order(dim):
    """Column order of tf.feature_column.input_layer over numeric columns C0..C{dim-1}: sorted by name."""
    return sorted(range(dim), key=lambda i: "C{}".format(i))


def _act(z, act):
    if act in (None, "linear"):
        return z
    if act == "relu":
        return np.maximum(z, 0)
    if act == "sigmoid":
        return 1 / (1 + np.exp(-z))
    if act == "tanh":
        return np.tanh(z)
    raise ValueError(act)


def _act_grad(y, act):
    if act in (None, "linear"):
        return np.ones_like(y)
    if act == "relu":
        return (y > 0).astype(y.dtype)
    if act == "sigmoid":
        return y * (1 - y)
    if act == "tanh":
        return 1 - y * y
    raise ValueError(act)


def tower_fwd(x, ws, bs, act):
    """-> list of layer inputs/outputs [x, y0, y1, ...]."""
    ys = [x]
    for i, (w, b) in enumerate(zip(ws, bs)):
        z = ys[-1] @ w + (0 if b is None else b)
        ys.append(_act(z, act if i < len(ws) - 1 else None))
    return ys


def tower_bwd(ys, ws, bs, act, g):
    """-> (gx, [gw], [gb]) for upstream gradient g of the tower output."""
    gws, gbs = [None] * len(ws), [None] * len(ws)
    for i in reversed(range(len(ws))):
        gz = g * _act_grad(ys[i + 1], act if i < len(ws) - 1 else None)
        gws[i] = ys[i].T @ gz
        gbs[i] = None if bs[i] is None else gz.sum(0)
        g = gz @ ws[i].T
    return g, gws, gbs


def softmax(x):
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def mix_fwd(experts, logits):
    """experts [B, E, H], logits [B, T, E] -> gates [B, T, E], out [B, T, H]."""
    gates = softmax(logits)
    return gates, np.einsum("bte,beh->bth", gates, experts)


def mix_bwd(experts, gates, g_out):
    """-> g_experts [B, E, H], g_logits [B, T, E]."""
    g_experts = np.einsum("bte,bth->beh", gates, g_out)
    dg = np.einsum("bth,beh->bte", g_out, experts)
    g_logits = gates * (dg - (gates * dg).sum(-1, keepdims=True))
    return g_experts, g_logits


def mmoe_layout(E, T, n_expert_layers, n_task_layers):
    """Index ranges of the weight list: experts[e], gates (all E), tasks[t]."""
    experts = [list(range(e * n_expert_layers, (e + 1) * n_expert_layers)) for e in range(E)]
    g0 = E * n_expert_layers
    gates = list(range(g0, g0 + E))
    t0 = g0 + E
    tasks = [list(range(t0 + t * n_task_layers, t0 + (t + 1) * n_task_layers)) for t in range(T)]
    return experts, gates, tasks


def mmoe_forward(inputs, ws, bs, E, T, expert_units, task_units, expert_act="relu", task_act="relu"):
    """inputs [B, D] (already in input_layer order) -> (list of T [B, 1] outputs, cache)."""
    ex_idx, gate_idx, task_idx = mmoe_layout(E, T, len(expert_units), len(task_units) + 1)
    ex_ys = [tower_fwd(inputs, [ws[i] for i in ix], [bs[i] for i in ix], expert_act) for ix in ex_idx]
    experts = np.stack([ys[-1] for ys in ex_ys], axis=1)                                   # [B, E, H]
    logits = np.stack([inputs @ ws[gate_idx[t]] for t in range(T)], axis=1)                 # [B, T, E]
    gates, mixed = mix_fwd(experts, logits)
    task_ys = [tower_fwd(mixed[:, t], [ws[i] for i in ix], [bs[i] for i in ix], task_act)
               for t, ix in enumerate(task_idx)]
    cache = dict(inputs=inputs, ws=ws, bs=bs, idx=(ex_idx, gate_idx, task_idx), ex_ys=ex_ys, experts=experts,
                 gates=gates, acts=(expert_act, task_act), T=T)
    return [ys[-1] for ys in task_ys], dict(cache, task_ys=task_ys)


def mmoe_backward(cache, g_outs):
    """g_outs: T arrays [B, 1] -> (g_inputs, gws, gbs) in creation order (unused gates get zero gradients)."""
    ws, bs, T = cache["ws"], cache["bs"], cache["T"]
    ex_idx, gate_idx, task_idx = cache["idx"]
    expert_act, task_act = cache["acts"]
    inputs = cache["inputs"]
    gws = [np.zeros_like(w) for w in ws]
    gbs = [None if b is None else np.zeros_like(b) for b in bs]
    g_mixed = []
    for t, ix in enumerate(task_idx):
        gm, gw, gb = tower_bwd(cache["task_ys"][t], [ws[i] for i in ix], [bs[i] for i in ix], task_act, g_outs[t])
        g_mixed.append(gm)
        for j, i in enumerate(ix):
            gws[i], gbs[i] = gw[j], gb[j]
    g_experts, g_logits = mix_bwd(cache["experts"], cache["gates"], np.stack(g_mixed, axis=1))
    g_in = np.zeros_like(inputs)
    for t in range(T):
        gws[gate_idx[t]] = inputs.T @ g_logits[:, t]
        g_in += g_logits[:, t] @ ws[gate_idx[t]].T
    for e, ix in enumerate(ex_idx):
        gx, gw, gb = tower_bwd(cache["ex_ys"][e], [ws[i] for i in ix], [bs[i] for i in ix], expert_act,
                               g_experts[:, e])
        g_in += gx
        for j, i in enumerate(ix):
            gws[i], gbs[i] = gw[j], gb[j]
    return g_in, gws, gbs


def esmm_forward(inputs, ws, bs, hidden_units, act="relu"):
    """-> ((p_cvr, p_ctr, p_ctcvr), cache); towers: ws[:L] pCVR, ws[L:] pCTR."""
    L = len(hidden_units) + 1
    cvr_ys = tower_fwd(inputs, ws[:L], bs[:L], act)
    ctr_ys = tower_fwd(inputs, ws[L:], bs[L:], act)
    p_cvr, p_ctr = _act(cvr_ys[-1], "sigmoid"), _act(ctr_ys[-1], "sigmoid")
    return (p_cvr, p_ctr, p_ctr * p_cvr), dict(ws=ws, bs=bs, L=L, ys=(cvr_ys, ctr_ys), p=(p_cvr, p_ctr), act=act)


def esmm_backward(cache, g_cvr, g_ctr, g_ctcvr):
    """-> (g_inputs, gws, gbs) in creation order."""
    ws, bs, L, act = cache["ws"], cache["bs"], cache["L"], cache["act"]
    p_cvr, p_ctr = cache["p"]
    gz_cvr = (g_cvr + g_ctcvr * p_ctr) * p_cvr * (1 - p_cvr)
    gz_ctr = (g_ctr + g_ctcvr * p_cvr) * p_ctr * (1 - p_ctr)
    gx0, gw0, gb0 = tower_bwd(cache["ys"][0], ws[:L], bs[:L], act, gz_cvr)
    gx1, gw1, gb1 = tower_bwd(cache["ys"][1], ws[L:], bs[L:], act, gz_ctr)
    return gx0 + gx1, gw0 + gw1, gb0 + gb1


def golden_weights(z, key):
    """(ws, bs) of a golden case in creation order (bs[i] None for the bias-free gates)."""
    n = int(z[key + "_nlayers"])
    ws = [z[f"{key}_w{i}"] for i in range(n)]
    bs = [z[f"{key}_b{i}"] if f"{key}_b{i}" in z.files else None for i in range(n)]
    return ws, bs
