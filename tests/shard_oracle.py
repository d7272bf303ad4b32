"""float64 oracle of the row-sharded embedding path: the FM forward and the row-sparse SGD step on one GLOBAL
table (all S slot tables stacked, row = slot_offset[s] + id), whatever the world size that holds it."""
import numpy as np

from oracle import reference_np as R


def split(table, lin, rows):
    """Global [total, D] table and [total] first-order weights -> per-slot lists."""
    cuts = np.cumsum(rows)[:-1]
    return np.split(table, cuts), np.split(lin, cuts)


def global_rows(ids, rows):
    """Global row of every lookup of ids [B, S], -1 where the id is out of vocabulary."""
    ids = np.asarray(ids, np.int64)
    rws = np.asarray(rows, np.int64)[None, :]
    offs = np.concatenate([[0], np.cumsum(rows)[:-1]]).astype(np.int64)[None, :]
    return np.where((ids >= 0) & (ids < rws), offs + ids, -1)


def fm_forward(table, lin, bias, rows, ids):
    """(stack fp32 [B,S,D], sum_e float64 [B,D], its |.| scale, logit float64 [B], its cancellation-aware scale)."""
    tables, lins = split(table, lin, rows)
    logit, stack = R.fm_logit(tables, lins, bias, ids, np.float64)
    st = stack.astype(np.float64)
    lin_abs = np.abs(R.linear_term(lins, 0.0, ids, np.float64)).reshape(-1) + abs(float(bias))
    scale = lin_abs + 0.5 * ((st.sum(1) ** 2).sum(1) + (st ** 2).sum((1, 2)))
    return stack, st.sum(1), np.abs(st).sum(1), logit.reshape(-1), scale


def sgd_step(table, lin, rows, ids, g_logit, g_stack, scale):
    """One row-sparse SGD step w += scale * dL/dw over the lookups ids [N, S] (g_logit [N] and g_stack [N,S,D] may
    each be None).  Returns (table, lin, table bound, lin bound, touched rows): the bounds are 1e-5 of the running
    magnitude of each fp32 sum, |w0| + |scale| * sum of |gradient terms|, the FM term's |sum_e| taken as
    sum_s |e_s| because sum_e is itself an fp32 sum."""
    tables, _ = split(table, lin, rows)
    stack = R.stack_embeddings(tables, ids)
    st = stack.astype(np.float64)
    total, D = table.shape
    gts, gls, _ = R.embed_fm_grad(rows, ids, stack, g_logit, g_stack, np.float64)
    gl_abs = None if g_logit is None else np.abs(np.asarray(g_logit, np.float64))
    terms = np.zeros_like(st)
    if g_logit is not None:
        terms += gl_abs[:, None, None] * (np.abs(st).sum(1, keepdims=True) + np.abs(st))
    if g_stack is not None:
        terms += np.abs(np.asarray(g_stack, np.float64))
    ats, _, _ = R.embed_fm_grad(rows, ids, st * 0, None, terms, np.float64)
    _, als, _ = R.embed_fm_grad(rows, ids, st * 0, gl_abs, None, np.float64)
    t0, l0 = table.astype(np.float64), lin.astype(np.float64)
    new_t = t0 + scale * np.concatenate(gts, 0)
    new_l = l0 + scale * np.concatenate(gls, 0)
    bound_t = 1e-5 * (np.abs(t0) + abs(scale) * np.concatenate(ats, 0)) + 1e-7
    bound_l = 1e-5 * (np.abs(l0) + abs(scale) * np.concatenate(als, 0)) + 1e-7
    gr = global_rows(ids, rows).reshape(-1)
    touched = np.zeros(total, bool)
    touched[gr[gr >= 0]] = True
    return new_t, new_l, bound_t, bound_l, touched
