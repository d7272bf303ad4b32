"""The float64 oracle of one DeepFM step (tests/deepfm_oracle.py) against torch autograd, and the per-element check
the GPU step tests use: it accepts float32 results a few ulps off and rejects each modelled kernel bug."""
import numpy as np
import pytest

from deepfm_oracle import (RTOL, U, _cpu_deepfm_grads, bias_additions, check, deepfm_step, resolved, update_slack,
                           violations)

F32 = np.float32


def _problem(units, act, B, rows=(97, 7, 300, 41), D=8, hot=False, seed=0):
    rng = np.random.default_rng(seed)
    tables = [rng.standard_normal((r, D)) * 0.3 for r in rows]
    lins = [rng.standard_normal(r) * 0.1 for r in rows]
    dims = [len(rows) * D] + list(units) + [1]
    ws = [rng.standard_normal((a, b)) / np.sqrt(a) for a, b in zip(dims[:-1], dims[1:])]
    bs = [rng.standard_normal(b) * 0.1 for b in dims[1:]]
    ids = np.stack([rng.integers(-1, r + 1, B) for r in rows], 1).astype(np.int64)   # -1 and == rows: OOV
    if hot:
        ids[:1000, 0] = 5
    labels = rng.integers(0, 2, B).astype(F32)
    f32 = lambda xs: [x.astype(F32).astype(np.float64) for x in xs]         # parameters a float32 kernel can hold
    return f32(tables), f32(lins), 0.2, f32(ws), f32(bs), act, ids, labels


@pytest.mark.parametrize("units,act,B,hot", [
    ([16, 8], "relu", 64, False),
    ([16, 8], "tanh", 64, False),
    ([16, 8], "sigmoid", 64, False),
    ([], "relu", 64, False),                   # one Dense(1)
    ([12], "tanh", 1200, True),                 # one id looked up 1000 times
])
def test_oracle_gradients_equal_torch_autograd(units, act, B, hot):
    p = _problem(units, act, B, hot=hot)
    tables, lins, bias, ws, bs, _, ids, labels = p
    o = deepfm_step(*p)
    loss, gt, gl, gb, gw, gbi = _cpu_deepfm_grads(tables, lins, bias, ws, bs, ids, labels, act)
    close = lambda a, b: np.abs(np.asarray(a) - np.asarray(b)).max() <= 1e-12 * max(1.0, np.abs(b).max())
    assert close(o["loss"].ref, loss)
    assert close(o["bias"].ref, gb[0])
    for s in range(len(tables)):
        assert close(o[f"table.{s}"].ref, gt[s]) and close(o[f"lin.{s}"].ref, gl[s])
    for i in range(len(ws)):
        assert close(o[f"w.{i}"].ref, gw[i]) and close(o[f"b.{i}"].ref, gbi[i])
    if hot:
        assert o["hits.0"][5] >= 1000 and np.abs(o["table.0"].ref[5]).sum() > 0
    # OOV ids of both kinds contribute nothing: a table whose every id is OOV has an all-zero gradient
    ids_oov = ids.copy()
    ids_oov[:, 1] = np.where(np.arange(B) % 2 == 0, -1, len(tables[1]))
    o2 = deepfm_step(tables, lins, bias, ws, bs, act, ids_oov, labels)
    assert not o2["table.1"].ref.any() and not o2["lin.1"].ref.any() and not o2["hits.1"].any()
    assert not o2["stack"].ref[:, 1].any()


# ---- the check has teeth ------------------------------------------------------------------------------------------
def _perturbed(e, rng, ulps=4):
    """The oracle's value rounded to float32, then moved by up to `ulps` float32 ulps of its scale."""
    ref = np.asarray(e.ref, np.float64)
    sc = np.broadcast_to(np.asarray(e.scale, np.float64), ref.shape)
    return ref.astype(F32).astype(np.float64) + rng.uniform(-1, 1, ref.shape) * ulps * 2 * U * sc


def _tower_bias_problem():
    # [32, 32]: two layers of one width, so one bias gradient can stand in for the other; B = 129: a ragged 128-row tile
    return _problem([32, 32], "relu", 129, seed=3)


def test_check_accepts_float32_results_a_few_ulps_off():
    rng = np.random.default_rng(1)
    for p in (_tower_bias_problem(), _problem([12], "tanh", 1200, hot=True), _problem([16, 8], "sigmoid", 64)):
        o = deepfm_step(*p)
        for k, e in o.items():
            if k.startswith("hits."):
                continue
            if k == "stack":
                check(k, np.asarray(e.ref, F32), e)          # the gather is a copy: bit-exact
                continue
            worst = check(k, _perturbed(e, rng), e)
            assert worst <= RTOL / 10, (k, worst)


def _applied(before, g, lr=1.0):
    """p - lr * g in float32 and the gradient recovered from it."""
    after = (before.astype(F32) - F32(lr) * g.astype(F32)).astype(np.float64)
    return (before - after) / lr, after


def test_check_rejects_modelled_kernel_bugs():
    p = _tower_bias_problem()
    tables, lins, bias, ws, bs, act, ids, labels = p
    o = deepfm_step(*p)
    rejected = lambda got, e, extra=0.0: violations(got, e, extra=extra).any()

    # the last example of the ragged tile (row 128) dropped from layer 0's weight gradient
    B = ids.shape[0]
    o_drop = deepfm_step(tables, lins, bias, ws, bs, act, ids[:B - 1], labels[:B - 1])
    gz_last = (o["w.0"].ref - o_drop["w.0"].ref * (B - 1) / B)      # the mean's 1/B: undo to isolate the example
    assert rejected(o["w.0"].ref - gz_last, o["w.0"])
    # the bias gradient of layer 1 written where layer 0's belongs
    assert not np.allclose(o["b.0"].ref, o["b.1"].ref)
    assert rejected(o["b.1"].ref, o["b.0"])
    # relu' taken on the wrong side of 0 for one column of layer 0: that column's terms flip in or out
    x = o["stack"].ref.reshape(B, -1)
    z0 = x @ ws[0] + bs[0]
    j = int(np.argmax(np.abs(o["b.0"].ref)))
    mask = (z0[:, j] > 0)
    # the gradient w.r.t. layer 0's output, column j, from layer 1's weights and pre-activation gradients
    h1 = np.maximum(x @ ws[0] + bs[0], 0)
    z1 = h1 @ ws[1] + bs[1]
    prob = o["prob"].ref
    gl = (prob - labels) / B
    gz2 = gl[:, None] * ws[2].T * (z1 > 0)                          # [B, 32]: gradient at layer 1's pre-activation
    gy0 = gz2 @ ws[1].T                                              # [B, 32]: at layer 0's output
    assert np.isclose((gy0[:, j] * mask).sum(), o["b.0"].ref[j], rtol=1e-12, atol=1e-15)
    flipped_b0 = o["b.0"].ref.copy()
    flipped_b0[j] = (gy0[:, j] * ~mask).sum()
    assert rejected(flipped_b0, o["b.0"])
    flipped_w0 = o["w.0"].ref.copy()
    flipped_w0[:, j] = x.T @ (gy0[:, j] * ~mask)
    assert rejected(flipped_w0, o["w.0"])

    # the update of one slot scaled by +lr: the recovered gradient is -g
    lr = 1.0
    for s in range(len(tables)):
        e = o[f"table.{s}"]
        got, after = _applied(tables[s], -e.ref, lr)
        extra = update_slack(tables[s], after, lr, o[f"hits.{s}"][:, None], e.terms)
        assert rejected(got, e, extra), s
        got_ok, after_ok = _applied(tables[s], e.ref, lr)
        assert not rejected(got_ok, e, update_slack(tables[s], after_ok, lr, o[f"hits.{s}"][:, None], e.terms))

    # relu' on the wrong side of 0 for one example far from 0: its term is outside the relu slack
    b = int(np.argmax(np.abs(gy0[:, j]) * (np.abs(z0[:, j]) > 0.1 * np.abs(z0[:, j]).max())))
    sign = 1.0 if not mask[b] else -1.0
    one = o["b.0"].ref.copy()
    one[j] += sign * gy0[b, j]
    assert rejected(one, o["b.0"])
    one_w = o["w.0"].ref.copy()
    one_w[:, j] += sign * x[b] * gy0[b, j]
    assert rejected(one_w, o["w.0"])


def test_check_rejects_one_lost_duplicate_contribution():
    """One id looked up 1000 times: losing any single lookup's contribution from its row is outside the bound, even
    with the rounding allowance of 1000 separate float32 additions at lr = 1."""
    p = _problem([12], "tanh", 1200, hot=True)
    tables, lins, bias, ws, bs, act, ids, labels = p
    o = deepfm_step(*p)
    e, hits = o["table.0"], o["hits.0"]
    hot = np.flatnonzero(ids[:, 0] == 5)
    assert hits[5] == len(hot) >= 1000
    for drop in (hot[0], hot[len(hot) // 2], hot[-1]):
        # that lookup's contribution alone (examples are independent; the batch mean's 1/B undone)
        single = deepfm_step(tables, lins, bias, ws, bs, act, ids[drop:drop + 1], labels[drop:drop + 1])
        contrib = single["table.0"].ref[5] / len(ids)                 # single's mean is over 1 example
        got = e.ref.copy()
        got[5] -= contrib
        after = tables[0] - got
        extra = update_slack(tables[0], after, 1.0, hits[:, None], e.terms)
        assert violations(got, e, extra=extra)[5].any(), drop

H100_SMS = 132


@pytest.mark.parametrize("B,lr", [(1200, 1.0), (4099, 1.0), (65536, 0.01)])
def test_missing_global_bias_gradient_is_rejected_under_the_gpu_bound(B, lr):
    """The global bias's update is checked with the rounding allowance of one float32 addition per CTA of the
    embedding backward.  At the batch sizes and rates the GPU tests run, a missing gradient is outside that bound in
    every one of 10 draws, and a correct update inside it (every GPU case also asserts the first for its own batch)."""
    for seed in range(10):
        tables, lins, bias, ws, bs, act, ids, labels = _problem([32], "relu", B, rows=(97, 7, 300), D=16, seed=seed)
        e = deepfm_step(tables, lins, bias, ws, bs, act, ids, labels)["bias"]
        after = float(np.float32(bias - lr * e.ref))
        extra = update_slack(bias, after, lr, bias_additions(B, H100_SMS), e.terms)
        assert violations(0.0, e, extra=extra).any(), seed
        assert not violations((bias - after) / lr, e, extra=extra).any(), seed


def test_hot_row_at_c2_magnitudes():
    """C2's zipf batch at lr = 0.01: one row looked up ~3e4 times, tables of std 1/sqrt(D).  Through the update most of
    its gradient is not resolvable (a zero update passes the worst-case rounding bound there); through a replay into a zeroed
    gradient arena a zero or sign-flipped gradient is rejected; one lost lookup is resolved by neither."""
    rng = np.random.default_rng(100)
    B, D, R_, lr = 65536, 16, 1_000_000, 0.01
    raw = np.minimum(rng.zipf(1.05, size=(B, 4)) - 1, R_ - 1)
    uniq = [np.unique(raw[:, s]) for s in range(4)]
    ids = np.stack([np.searchsorted(uniq[s], raw[:, s]) for s in range(4)], 1)
    f32 = lambda a: a.astype(F32).astype(np.float64)
    tables = [f32(np.clip(rng.standard_normal((len(u), D)), -2, 2) / np.sqrt(D)) for u in uniq]
    lins = [f32(rng.standard_normal(len(u)) * 0.01) for u in uniq]
    ws = [f32(rng.standard_normal((4 * D, 32)) / np.sqrt(4 * D)), f32(rng.standard_normal((32, 1)) / np.sqrt(32))]
    bs = [np.zeros(32), np.zeros(1)]
    labels = rng.integers(0, 2, B).astype(F32)
    o = deepfm_step(tables, lins, 0.0, ws, bs, "relu", ids, labels)
    e, hits = o["table.0"], o["hits.0"]
    r = int(np.argmax(hits))
    assert hits[r] > 20000
    row = e._replace(ref=e.ref[r], scale=e.scale[r], slack=e.slack[r], terms=e.terms[r])
    p0 = tables[0][r]
    after = f32(p0 - lr * row.ref)
    upd = update_slack(p0, after, lr, hits[r], row.terms)
    un = ~resolved(row, upd)                                      # elements the update cannot resolve: most of them
    assert un.sum() >= D // 2 and not violations(np.zeros(D), row, extra=upd)[un].any()
    rep = update_slack(0.0, 0.0, 1.0, hits[r], row.terms)
    assert resolved(row, rep).all()
    assert violations(np.zeros(D), row, extra=rep).all() and violations(-row.ref, row, extra=rep).all()
    one = row.terms / hits[r]                                     # one lookup's mean |contribution|
    assert not violations(row.ref - one, row, extra=rep).any()    # below the rounding of the row's own sum
