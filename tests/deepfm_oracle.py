"""float64 oracle of one DeepFM training step (reference keras/models/ranking/deepfm.py:36-47 trained on the mean
binary cross-entropy), composed from oracle/reference_np.py, and the per-element check the DeepFM step tests share.

`deepfm_step` returns every value the step computes -- loss, probabilities, FM logit, stacked embeddings, tower
activations -- and the gradient of every parameter, each as an `Entry(ref, scale, slack, terms)`:

  * `scale` is the sum of |terms| behind the value, carried through the whole composition: the same formulas run on
    absolute values, with every input's own scale in place of its magnitude, so a kernel whose every sum is
    accurate to `RTOL` relative to its terms stays within `RTOL * scale`;
  * `slack` is what relu' decisions on pre-activations within `RTOL * scale` of zero can move the value: a correct
    kernel may land on either side of 0 there, and the term it then keeps or drops is allowed, nothing more;
  * `terms` (gradients only) is the sum of |what the update adds|: per lookup for a table row or a first-order
    weight, per example for the global bias, the gradient itself for a tower parameter.  It bounds the running
    value of an update applied as separate float32 additions (`update_slack`).

`_cpu_deepfm_grads` is the float64 torch-autograd restatement of the same step; the CPU tests hold the numpy
composition to it.
"""
from collections import namedtuple

import numpy as np
import torch

from oracle import reference_np as R

F64 = np.float64
U = 2.0 ** -24            # unit roundoff of float32

# Per-element bound of every DeepFM step test: |got - ref| <= RTOL * scale + slack (+ update rounding, below).
# 1e-5 is about 80 float32 ulps of the scale.  Every sum in the step is a float32 sum (FFMA, or 3xTF32 wgmma whose
# dropped lo*lo product is ~2^-22 of a term) of at most 65536 terms whose rounding errors are not all of one sign;
# the DCN step's test uses 1e-4.  The accept case of tests/test_cpu_deepfm_oracle.py (float32-rounded values, a few
# ulps of the scale off) passes with 10x to spare, and every modelled kernel bug there is rejected.  On an H100 80GB
# HBM3 (700 W) the largest err / scale of tests/test_gpu_deepfm_train_step.py was 1.6e-6 (layer 0's activations at
# S = 120, K = 1920, 3xTF32); the GPU tests print theirs.
RTOL = 1e-5

Entry = namedtuple("Entry", "ref scale slack terms", defaults=(0.0,))

_LIP = {"relu": 1.0, "tanh": 1.0, "sigmoid": 0.25, None: 1.0, "linear": 1.0}       # max |act'|
_CURV = {"relu": 0.0, "tanh": 2.0, "sigmoid": 1.0, None: 0.0, "linear": 0.0}       # max |d act'(y) / dy|


def deepfm_step(tables, lins, bias, ws, bs, activation, ids, labels, rtol=RTOL):
    """tables[s] [rows_s, D], lins[s] [rows_s], bias scalar, tower kernels ws[i] [in, out] and biases bs[i] (the last
    layer is Dense(1) with no activation), ids [B, S] (< 0 or >= rows_s: OOV, a zero row), labels [B] in {0, 1}.

    Returns {name: Entry}: "loss", "prob", "fm_logit", "stack" [B,S,D], "acts.i" [B, units_i], "w.i", "b.i",
    "table.s" [rows_s, D], "lin.s" [rows_s], "bias"; and "hits.s": the number of valid lookups of every row of slot s
    (how many separate additions its update takes)."""
    ids = np.asarray(ids, dtype=np.int64)
    y = np.asarray(labels, F64).reshape(-1)
    B, S = ids.shape
    tables = [np.asarray(t, F64) for t in tables]
    lins = [np.asarray(l, F64) for l in lins]
    ws = [np.asarray(w, F64) for w in ws]
    bs = [np.asarray(b, F64) for b in bs]
    acts = [activation] * (len(ws) - 1) + [None]
    L = len(ws)
    out = {}

    # ---- forward ----
    prob, logit, stack, hs = R.deepfm_forward(tables, lins, bias, ws, bs, ids, activation, F64)
    prob, logit = prob.reshape(-1), logit.reshape(-1)
    fm = (R.fm_logit(tables, lins, bias, ids, F64)[0]).reshape(-1)
    a = np.abs(stack)
    fm_s = (abs(bias) + R.linear_term([np.abs(l) for l in lins], 0.0, ids, F64).reshape(-1)
            + 0.5 * ((a.sum(1) ** 2).sum(1) + (a * a).sum((1, 2))))
    out["stack"] = Entry(stack, np.zeros_like(stack), 0.0)
    out["fm_logit"] = Entry(fm, fm_s, 0.0)
    x = stack.reshape(B, -1)
    hsc = [np.abs(x)]                     # scale of every tower input / activation
    zs, zsc = [], []
    for i in range(L):
        z = hs[i] @ ws[i] + bs[i]
        zsc.append(hsc[i] @ np.abs(ws[i]) + np.abs(bs[i]))
        zs.append(z)
        hsc.append(np.abs(hs[i + 1]) + _LIP[acts[i]] * zsc[i])
        out[f"acts.{i}"] = Entry(hs[i + 1], hsc[i + 1], 0.0)
    logit_s = fm_s + zsc[-1].reshape(-1)
    out["prob"] = Entry(prob, prob + 0.25 * logit_s, 0.0)
    per = np.maximum(logit, 0) - logit * y + np.log1p(np.exp(-np.abs(logit)))
    out["loss"] = Entry(float(per.mean()), float((per + logit_s).mean()), 0.0)

    # ---- backward ----
    gl = (prob - y) / B                                       # d mean-BCE / d logit
    gl_s = (prob + y + 0.25 * logit_s) / B
    g, g_s, g_f = gl.reshape(B, 1), gl_s.reshape(B, 1), np.zeros((B, 1))
    for i in range(L - 1, -1, -1):
        act = acts[i]
        gx, gw, gb = R.dense_grad(hs[i], ws[i], hs[i + 1], g, act, F64)
        d = {"relu": (hs[i + 1] > 0).astype(F64), "sigmoid": hs[i + 1] * (1 - hs[i + 1]),
             "tanh": 1 - hs[i + 1] ** 2}.get(act, 1.0)
        gz = g * d
        gz_s = g_s * _LIP[act] + np.abs(g) * _CURV[act] * (hsc[i + 1] - np.abs(hs[i + 1]))
        gz_f = g_f * np.abs(d) if act != "relu" else g_f * ((zs[i] > 0) | (np.abs(zs[i]) <= 2 * rtol * zsc[i]))
        if act == "relu":
            gz_f = gz_f + np.abs(g) * (np.abs(zs[i]) <= 2 * rtol * zsc[i])
        out[f"w.{i}"] = Entry(gw, hsc[i].T @ gz_s, np.abs(hs[i]).T @ gz_f, np.abs(gw))
        out[f"b.{i}"] = Entry(gb, gz_s.sum(0), gz_f.sum(0), np.abs(gb))
        g, g_s, g_f = gx, gz_s @ np.abs(ws[i]).T, gz_f @ np.abs(ws[i]).T
    shape = stack.shape
    rows = [t.shape[0] for t in tables]
    gt, glin, gbias = R.embed_fm_grad(rows, ids, stack, gl, g.reshape(shape), F64)
    st, sl, _ = R.embed_fm_grad(rows, ids, np.abs(stack), gl_s, g_s.reshape(shape), F64)
    ft, _, _ = R.embed_fm_grad(rows, ids, np.zeros(shape), None, g_f.reshape(shape), F64)
    d_e = gl[:, None, None] * (stack.sum(1, keepdims=True) - stack) + g.reshape(shape)      # what each lookup adds
    tt, tl, _ = R.embed_fm_grad(rows, ids, np.zeros(shape), np.abs(gl), np.abs(d_e), F64)
    for s in range(S):
        col = ids[:, s]
        ok = (col >= 0) & (col < rows[s])
        out[f"table.{s}"] = Entry(gt[s], st[s], ft[s], tt[s])
        out[f"lin.{s}"] = Entry(glin[s], sl[s], 0.0, tl[s])
        out[f"hits.{s}"] = np.bincount(col[ok], minlength=rows[s])
    out["bias"] = Entry(float(gbias), float(gl_s.sum()), 0.0, float(np.abs(gl).sum()))
    return out


def update_slack(before, after, lr, adds, terms):
    """What float32 rounding can move the gradient recovered as (before - after) / lr from an update applied as
    `adds` separate float32 additions whose |values| sum to lr * `terms` (Entry.terms): each addition rounds by at
    most U times the running value, which never exceeds max(|before|, |after|) + lr * terms.

    This is the worst case.  Where it reaches |gradient| -- about 3e4 lookups of one row onto |p| ~ 0.25 at lr =
    0.01 -- the recovered gradient cannot tell a correct update from none; `resolved` names the elements where it
    can, and the tests check the others another way."""
    run = np.maximum(np.abs(np.asarray(before, F64)), np.abs(np.asarray(after, F64))) + lr * np.asarray(terms, F64)
    return np.asarray(adds, F64) * U * run / lr


def resolved(e: Entry, extra, rtol=RTOL):
    """Elements whose bound is below |ref|: there a zero or a sign-flipped result is outside it."""
    return rtol * np.asarray(e.scale, F64) + e.slack + extra < np.abs(np.asarray(e.ref, F64))


def bias_additions(B, num_sms):
    """Float32 additions the embedding backward makes to the global bias (or its gradient): one per CTA, and
    dr_embed_fm_bwd launches at most one CTA per 4 examples (>= 4 warps, >= 1 example each) and 16 per SM."""
    return min(-(-B // 4), 16 * num_sms)


def violations(got, e: Entry, rtol=RTOL, extra=0.0):
    """Boolean mask of the elements outside |got - ref| <= rtol * scale + slack + extra (NaN is outside)."""
    got = np.asarray(got, F64).reshape(np.shape(e.ref))
    err = np.abs(got - e.ref)
    return ~(err <= rtol * e.scale + e.slack + extra)


def check(name, got, e: Entry, rtol=RTOL, extra=0.0):
    """Assert the per-element bound; the message names the worst element.  Returns max(err / scale) over the
    elements with a non-zero scale (the share of RTOL a run used)."""
    got = np.asarray(got, F64).reshape(np.shape(e.ref))
    bad = violations(got, e, rtol, extra)
    err = np.abs(got - np.asarray(e.ref, F64))
    if bad.any():
        idx = np.unravel_index(np.argmax(np.where(bad, err - rtol * np.asarray(e.scale) - e.slack, -np.inf)),
                               np.shape(e.ref)) if np.ndim(e.ref) else ()
        pick = lambda v: np.broadcast_to(np.asarray(v, F64), np.shape(e.ref))[idx]
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.size} elements outside the bound; worst at {idx}: "
                             f"got {pick(got)!r} want {pick(e.ref)!r} scale {pick(e.scale)!r} "
                             f"slack {pick(e.slack)!r} extra {pick(extra)!r}")
    sc = np.broadcast_to(np.asarray(e.scale, F64), err.shape)
    nz = sc > 0
    return float((err[nz] / sc[nz]).max()) if nz.any() else 0.0


def _cpu_deepfm_grads(tables, lins, bias, ws, bs, ids, labels, activation="relu"):
    """float64 torch-CPU autograd of the reference composition (deepfm.py:36-47 + BCE mean): dense gradients."""
    act = {"relu": torch.relu, "tanh": torch.tanh, "sigmoid": torch.sigmoid}[activation]
    tt = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in tables]
    tl = [torch.tensor(l, dtype=torch.float64, requires_grad=True) for l in lins]
    tb = torch.tensor([bias], dtype=torch.float64, requires_grad=True)
    tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in ws]
    tbi = [torch.tensor(b, dtype=torch.float64, requires_grad=True) for b in bs]
    B = ids.shape[0]
    cols, lin = [], tb.expand(B)
    for s, t in enumerate(tt):
        ok = torch.from_numpy((ids[:, s] >= 0) & (ids[:, s] < t.shape[0]))
        idx = torch.from_numpy(np.clip(ids[:, s], 0, t.shape[0] - 1))
        cols.append(t[idx] * ok[:, None])
        lin = lin + tl[s][idx] * ok
    st = torch.stack(cols, 1)
    fm = 0.5 * ((st.sum(1) ** 2) - (st ** 2).sum(1)).sum(1)
    h = st.reshape(B, -1)
    for i, (w, b) in enumerate(zip(tw, tbi)):
        h = h @ w + b
        if i < len(tw) - 1:
            h = act(h)
    z = lin + fm + h[:, 0]
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z, torch.from_numpy(labels).double())
    loss.backward()
    g = lambda xs: [x.grad.numpy() for x in xs]
    return float(loss.detach()), g(tt), g(tl), tb.grad.numpy(), g(tw), g(tbi)
