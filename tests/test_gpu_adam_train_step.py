"""DeepFMTrainStep with the four Adam optimizers ("adam", "lazy_adam", "adam_rows", "adam_rows_tf") per element against
the float64 models of tests/deepfm_oracle.py (the step's values and gradients) and tests/adam_oracle.py (Adam).

Every step snapshots the parameters and all optimizer state on the host, runs, and checks:
  * every forward value (loss, prob, fm_logit, stack, activations) against the parameters the forward read;
  * the gradients through m and v (`moments`), per element, for the tower, every table row the step moves, every
    first-order weight and the global bias; and the tower's gradient buffer directly;
  * the updates through `functor`, recomputed from the kernels' own m, v and lr_t: under "adam" every arena element
    (untouched rows move by their decayed m; the fused rows' padding stays bit-identical with m = v = 0), under the
    row-sparse optimizers the touched rows, with the untouched ones bit-identical;
  * the invariants between steps: gradient buffers and countdowns zero, stamps, the clock;
  * under "adam_rows_tf", the rows dr_embed_adam_prepare replayed before the forward read them, against `replay` of the
    pre-step snapshot (the float32 values the forward used are in tr.stack), and after the last step every row
    flush_optimizer() brings up to date.

lr = 0.01 and eps = 1e-7 as the reference examples train; batches of 96 over tables of 7 to 300 rows leave rows
untouched for one to several steps, so the prepare replays rows at every step after the second.
"""
import time

import numpy as np
import pytest
import torch

from adam_oracle import (U, adam_bias_additions, check_bound, functor, lr_t, moments, replay)
from deepfm_oracle import RTOL, Entry, bias_additions, check, deepfm_step, resolved, update_slack
from test_gpu_deepfm_train_step import C2, _batch, _bench_ids, _sms, knobs, npy  # noqa: F401  (knobs: fixture)

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-7
ROWS = [97, 7, 300, 41]
UNITS = [32, 16]


def _trainer(optimizer, D, B, id_dtype=torch.int64, use_graph=True, seed=5, rows=ROWS, **opts):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=UNITS, dnn_activation="relu", seed=seed, device="cuda")
    tr = DeepFMTrainStep(model, batch_size=B, lr=LR, id_dtype=id_dtype, use_graph=use_graph, optimizer=optimizer,
                         beta1=B1, beta2=B2, eps=EPS, **opts)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        model.embeddings.lin_view().normal_(0, 0.1, generator=gen)
        model.embeddings.bias.fill_(0.2)
        for b in tr.b:
            b.normal_(0, 0.1, generator=gen)
    before = [t.clone() for t in tr._persistent_state()]
    tr.capture()
    # capture() is side-effect free: every parameter and every piece of optimizer state comes back bit for bit
    for a, b in zip(before, tr._persistent_state()):
        assert torch.equal(a.view(torch.int32) if a.is_floating_point() else a,
                           b.view(torch.int32) if b.is_floating_point() else b), "capture() left state behind"
    assert int(tr.clock.step) == 0
    return tr


def _snap(tr):
    """Host copies (numpy) of every parameter and optimizer state tensor of the trainer, by name."""
    names = ("g_arena", "m_arena", "v_arena", "g_lin", "m_lin", "v_lin", "g_bias", "m_bias", "v_bias", "m_flat",
             "v_flat", "stamp", "state", "flat", "gflat")
    h = {k: getattr(tr, k).detach().cpu().numpy().copy() for k in names if getattr(tr, k) is not None}
    c = tr.coll
    h["arena"] = c.weight.detach().cpu().numpy().copy()
    h["linear"] = None if c.linear is None else c.linear.detach().cpu().numpy().copy()
    h["bias"] = c.bias.detach().cpu().numpy().copy()
    D = tr.D
    h["p"] = np.concatenate([h["arena"][:, :D], (h["arena"][:, D] if c.layout == "fused" else h["linear"])[:, None]],
                            1).astype(F64)                      # [emb | w] per global row
    if "state" in h:
        st = h["state"]
        h["m"] = np.concatenate([st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]], 1).astype(F64)
        h["v"] = np.concatenate([st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]], 1).astype(F64)
        h["row_stamp"] = st[:, 3 * D + 4].view(np.int32).astype(np.int64)
    else:
        lin = lambda a, l: (a[:, D] if c.layout == "fused" else l)[:, None]
        h["m"] = np.concatenate([h["m_arena"][:, :D], lin(h["m_arena"], h.get("m_lin"))], 1).astype(F64)
        h["v"] = np.concatenate([h["v_arena"][:, :D], lin(h["v_arena"], h.get("v_lin"))], 1).astype(F64)
    h["step"], h["lr_t"] = int(tr.clock.step), float(tr.clock.lr_t)
    return h


def _tower(tr):
    """(name, slice of the flat buffer, shape) of every tower parameter."""
    base = tr.flat.data_ptr()
    out = []
    for i, (w, b) in enumerate(zip(tr.w, tr.b)):
        for k, t in ((f"w.{i}", w), (f"b.{i}", b)):
            if t is not None:
                o = (t.data_ptr() - base) // 4
                out.append((k, slice(o, o + t.numel()), tuple(t.shape)))
    return out


def _hits(tr, ids):
    hits = np.zeros(tr.coll.total_rows, np.int64)
    offs = tr.coll._offsets.cpu().numpy()
    for s, r in enumerate(tr.coll.rows_list):
        col = ids[:, s]
        np.add.at(hits, offs[s] + col[(col >= 0) & (col < r)], 1)
    return hits


def _rows_entry(o, S):
    """The gradient of every global row [emb | w] as one Entry (float64 arrays)."""
    cat = lambda f: np.concatenate([np.concatenate([np.broadcast_to(f(o[f"table.{s}"]), o[f"table.{s}"].ref.shape),
                                                    np.broadcast_to(f(o[f"lin.{s}"]), o[f"lin.{s}"].ref.shape)[:, None]],
                                                   1) for s in range(S)], 0).astype(F64)
    return Entry(cat(lambda e: e.ref), cat(lambda e: e.scale), cat(lambda e: e.slack), cat(lambda e: e.terms))


def _same_bits(name, got, want):
    assert np.array_equal(np.asarray(got).view(np.int32), np.asarray(want).view(np.int32)), name


class Report(dict):
    def got(self, k, share):
        self[k] = max(self.get(k, 0.0), share)


def _check_tower_and_bias(tr, opt, o, h0, h1, lr_gpu, rtol, rep):
    """The tower (gradient buffer, moments, functor) and the global bias (moments, functor) of one step."""
    B = tr.B
    # ---- the tower: gradient buffer, moments, functor ----
    flat0, tw = h0["flat"].astype(F64), _tower(tr)
    flat1, mf0, vf0, mf1, vf1 = h1["flat"], h0["m_flat"], h0["v_flat"], h1["m_flat"], h1["v_flat"]
    gflat = h1["gflat"]
    for k, sl, sh in tw:
        e = o[k]
        rep.got("grad buffer " + k, check("grad buffer " + k, gflat[sl].reshape(sh), e, rtol=rtol))
        m1, bm_, v1, bv_ = moments(mf0[sl].reshape(sh), vf0[sl].reshape(sh), e, 0.0, B1, B2, rtol=rtol)
        rep.got("m tower", check_bound(f"m {k}", mf1[sl].reshape(sh), m1, bm_))
        rep.got("v tower", check_bound(f"v {k}", vf1[sl].reshape(sh), v1, bv_))
        p1, bp_ = functor(flat0[sl], mf1[sl], vf1[sl], lr_gpu, EPS)
        rep.got("p tower", check_bound(f"p {k}", flat1[sl], p1, bp_))
    # ---- the global bias ----
    e = o["bias"]
    adds = adam_bias_additions(B, _sms()) if opt in ("adam_rows", "adam_rows_tf") else bias_additions(B, _sms())
    m1, bm_, v1, bv_ = moments(h0["m_bias"], h0["v_bias"], e, update_slack(0, 0, 1, adds, e.terms), B1, B2, rtol=rtol)
    rep.got("m bias", check_bound("m bias", h1["m_bias"], m1, bm_))
    rep.got("v bias", check_bound("v bias", h1["v_bias"], v1, bv_))
    p1, bp_ = functor(h0["bias"], h1["m_bias"], h1["v_bias"], lr_gpu, EPS)
    rep.got("p bias", check_bound("p bias", h1["bias"], p1, bp_))
    assert not h1["g_bias"].any()


def _step_and_check(tr, opt, ids, labels, t, rep: Report):
    c, D, S, B = tr.coll, tr.D, tr.S, tr.B
    offs = c._offsets.cpu().numpy()
    split = lambda a: [a[o:o + r] for o, r in zip(offs, c.rows_list)]
    h0 = _snap(tr)
    hits = _hits(tr, ids)
    touched = hits > 0
    tr.step(torch.from_numpy(ids).cuda().to(tr.ids.dtype), torch.from_numpy(labels).cuda())
    torch.cuda.synchronize()
    h1 = _snap(tr)
    lr_gpu = F64(h1["lr_t"])
    # ---- the clock ----
    assert h1["step"] == t
    assert abs(lr_gpu - lr_t(t, LR, B1, B2)) <= 2 * U * lr_t(t, LR, B1, B2)
    # ---- what the forward read ----
    p_fwd, p_err = h0["p"].copy(), np.zeros_like(h0["p"])
    m_pre, v_pre, m_err, v_err = h0["m"], h0["v"], 0.0, 0.0
    rtol = RTOL
    if opt == "adam_rows_tf":
        s0 = h0["row_stamp"]
        rp, rm, rv, bp, bm, bv = replay(h0["p"], h0["m"], h0["v"], np.where(touched, s0, 0), t - 1, LR, B1, B2, EPS,
                                        t_now=t, hist_len=tr.clock.lr_hist.numel())
        stack = npy(tr.stack)
        ok = np.stack([(ids[:, s] >= 0) & (ids[:, s] < c.rows_list[s]) for s in range(S)], 1)
        grow = np.where(ok, ids + offs[None, :], 0)
        seen = stack[ok]                                        # [lookups, D]: the rows the forward read
        rep.got("prepare replay (stack)", check_bound("prepare replay of the rows the forward read", seen,
                                                      rp[grow[ok], :D], bp[grow[ok], :D]))
        p_fwd[grow[ok], :D] = seen                              # the float32 values the forward used
        first = np.zeros(c.total_rows, np.int64)
        first[grow[ok]] = np.arange(int(ok.sum()))
        assert np.array_equal(seen, seen[first[grow[ok]]]), "two lookups of one row read different values"
        p_fwd[touched, D] = rp[touched, D]
        p_err[touched, D] = bp[touched, D]
        m_pre, v_pre, m_err, v_err = rm, rv, bm, bv
        rep["rows replayed"] = rep.get("rows replayed", 0) + int((touched & (s0 > 0) & (s0 < t - 1)).sum())
    tables = split(p_fwd[:, :D])
    lins = split(p_fwd[:, D])
    flat0 = h0["flat"].astype(F64)
    tw = _tower(tr)
    ws = [flat0[sl].reshape(sh) for k, sl, sh in tw if k.startswith("w.")]
    bs = [flat0[sl].reshape(sh) for k, sl, sh in tw if k.startswith("b.")]
    o = deepfm_step(tables, lins, float(h0["bias"][0]), ws, bs, "relu", ids, labels)
    # first-order weights the forward read through a replay: their bound moves every logit; below 1 % of RTOL of the
    # logit's scale (asserted), so the gradients, whose scales carry the logit's, keep 1.01 RTOL
    d_logit = np.zeros(B)
    if opt == "adam_rows_tf":
        d_logit = np.where(ok, p_err[grow, D], 0.0).sum(1)
        logit_s = 4 * (o["prob"].scale - o["prob"].ref)
        assert (d_logit <= 0.01 * RTOL * logit_s).all()
        rtol = 1.01 * RTOL
    rep.got("loss", check("loss", float(tr.loss), o["loss"], extra=float(d_logit.mean())))
    rep.got("prob", check("prob", npy(tr.prob), o["prob"], extra=0.25 * d_logit))
    rep.got("fm_logit", check("fm_logit", npy(tr.fm_logit), o["fm_logit"], extra=d_logit))
    rep.got("stack", check("stack", npy(tr.stack), o["stack"]))
    for i in range(len(tr.w)):
        rep.got(f"acts.{i}", check(f"acts.{i}", npy(tr.acts[i]), o[f"acts.{i}"]))
    _check_tower_and_bias(tr, opt, o, h0, h1, lr_gpu, rtol, rep)
    # ---- table rows and first-order weights ----
    E = _rows_entry(o, S)
    rows = np.arange(c.total_rows) if opt == "adam" else np.flatnonzero(touched)
    e = Entry(E.ref[rows], E.scale[rows], E.slack[rows], E.terms[rows])
    extra = update_slack(0, 0, 1, hits[rows][:, None], e.terms)
    pick = lambda x: x[rows] if np.ndim(x) else x
    m1, bm_, v1, bv_ = moments(m_pre[rows], v_pre[rows], e, extra, B1, B2, pick(m_err), pick(v_err), rtol=rtol)
    rep.got("m rows", check_bound("m of the table rows [emb | w]", h1["m"][rows], m1, bm_))
    rep.got("v rows", check_bound("v of the table rows [emb | w]", h1["v"][rows], v1, bv_))
    p1, bp_ = functor(p_fwd[rows], h1["m"][rows], h1["v"][rows], lr_gpu, EPS, p0_err=p_err[rows])
    rep.got("p rows", check_bound("p of the table rows [emb | w]", h1["p"][rows], p1, bp_))
    keep = ~touched
    if c.layout == "fused":
        _same_bits("fused row padding", h1["arena"][:, D + 1:], h0["arena"][:, D + 1:])
    if opt == "adam":
        if c.layout == "fused":
            assert not h1["m_arena"][:, D + 1:].any() and not h1["v_arena"][:, D + 1:].any()
        assert not h1["g_arena"].any() and (h1.get("g_lin") is None or not h1["g_lin"].any())
    else:
        for k in ("p", "m", "v"):
            _same_bits(f"untouched rows: {k}", h1[k][keep], h0[k][keep])
    if opt == "lazy_adam":
        assert not h1["g_arena"].any() and (h1.get("g_lin") is None or not h1["g_lin"].any())
        assert np.array_equal(h1["stamp"] == t, touched) and np.array_equal(h1["stamp"][keep], h0["stamp"][keep])
    if opt in ("adam_rows", "adam_rows_tf"):
        st = h1["state"]
        assert not st[:, :D].any() and not st[:, 3 * D].any(), "gradient slots not zero between steps"
        assert not st[:, 3 * D + 3].view(np.int32).any(), "countdowns not zero between steps"
        _same_bits("untouched rows: state", st[keep], h0["state"][keep])
    if opt == "adam_rows_tf":
        assert (h1["row_stamp"][touched] == t).all()
    return h1


def _flush_and_check(tr, rep):
    h0 = _snap(tr)
    t = h0["step"]
    tr.flush_optimizer()
    torch.cuda.synchronize()
    h1 = _snap(tr)
    s0 = h0["row_stamp"]
    stale = (s0 > 0) & (s0 < t)
    rp, rm, rv, bp, bm, bv = replay(h0["p"][stale], h0["m"][stale], h0["v"][stale], s0[stale], t, LR, B1, B2, EPS,
                                    t_now=t, hist_len=tr.clock.lr_hist.numel())
    for k, ref, b in (("p", rp, bp), ("m", rm, bm), ("v", rv, bv)):
        rep.got(f"flush {k}", check_bound(f"flush {k}", h1[k][stale], ref, b))
    assert (h1["row_stamp"][s0 > 0] == t).all()
    _same_bits("flush: rows with stamp 0 or t", h1["state"][~stale], h0["state"][~stale])
    _same_bits("flush: parameters of rows with stamp 0 or t", h1["p"][~stale], h0["p"][~stale])
    return int(stale.sum())


def _case(name, opt, D=16, B=96, id_dtype=torch.int64, use_graph=True, steps=4, **opts):
    return pytest.param(dict(opt=opt, D=D, B=B, id_dtype=id_dtype, use_graph=use_graph, steps=steps, opts=opts), id=name)


OPTS = ["adam", "lazy_adam", "adam_rows", "adam_rows_tf"]
CASES = [_case(f"{o}_base", o) for o in OPTS]
# D: fused 4, 8, 12, 16, 28 and split 32, 64, 128 (LPR of the row-sparse kernels: 1, 2, 4, 4, 8, 8, 16, 32; of
# lazy_adam_rows with the [w | pad] chunk: 2, 4, 4, 8, 8, 8, 16, 32)
CASES += [_case(f"{o}_D{D}", o, D=D) for o in ("lazy_adam", "adam_rows", "adam_rows_tf") for D in (4, 8, 12, 28, 32, 64, 128)]
CASES += [_case("adam_D32", "adam", D=32), _case("adam_D4", "adam", D=4)]
CASES += [_case(f"{o}_int32", o, id_dtype=torch.int32) for o in OPTS]
CASES += [_case(f"{o}_eager", o, use_graph=False) for o in OPTS]
CASES += [_case(f"{o}_B{B}", o, B=B, steps=3) for o in ("adam_rows", "adam_rows_tf") for B in (1, 4099, 9000)]
CASES += [_case("lazy_adam_B4099", "lazy_adam", B=4099, steps=3), _case("adam_B1", "adam", B=1, steps=3)]
CASES += [_case(f"{o}_{k}", o, **{k: v}) for o in ("adam_rows", "adam_rows_tf")
          for k, v in (("fwd_chunks", 3), ("embed_fwd", "tma"), ("dw_first", True))]
CASES += [                                              # the risky ones stacked
    _case("adam_rows_tf_split_D64_int32_B9000_eager", "adam_rows_tf", D=64, id_dtype=torch.int32, B=9000,
          use_graph=False, steps=3),
    _case("adam_rows_fused_D4_int32_B9000_chunks3", "adam_rows", D=4, id_dtype=torch.int32, B=9000, steps=3,
          fwd_chunks=3),
    _case("adam_rows_tf_fused_D8_int32_dw_first", "adam_rows_tf", D=8, id_dtype=torch.int32, dw_first=True),
    _case("adam_rows_tf_tma_int32_eager", "adam_rows_tf", id_dtype=torch.int32, use_graph=False, embed_fwd="tma"),
    _case("lazy_adam_split_D128_int32_eager", "lazy_adam", D=128, id_dtype=torch.int32, use_graph=False),
]


@pytest.mark.parametrize("cfg", CASES)
def test_adam_steps_match_oracle(knobs, cfg):
    knobs(tc_dw_share=int(cfg["opts"].get("dw_first", False)))
    t0 = time.perf_counter()
    opt, B = cfg["opt"], cfg["B"]
    tr = _trainer(opt, cfg["D"], B, cfg["id_dtype"], cfg["use_graph"], **cfg["opts"])
    assert (tr.graph is not None) == cfg["use_graph"]
    rng = np.random.default_rng(B + cfg["D"])
    rep = Report()
    for t in range(1, cfg["steps"] + 1):
        ids, labels = _batch(rng, ROWS, B)
        _step_and_check(tr, opt, ids, labels, t, rep)
    if opt == "adam_rows_tf":
        if 96 <= B < 1000:                  # from B = 1000 on every row of these tables is touched at every step
            assert rep["rows replayed"] > 0, "no step replayed a row: pick other batches"
        rep["rows flushed"] = _flush_and_check(tr, rep)
    print(f"{time.perf_counter() - t0:.1f} s; max err/bound (err/scale for forward values and the grad buffer):",
          {k: (f"{v:.1e}" if isinstance(v, float) else v) for k, v in rep.items()})



# ---- the benchmark's shape at full size ------------------------------------------------------------------------------
def _small(tr):
    """Host copies of the tower, the global bias and their Adam state (the table state stays on the device)."""
    h = {k: getattr(tr, k).detach().cpu().numpy().copy() for k in ("flat", "gflat", "m_flat", "v_flat", "m_bias",
                                                                   "v_bias", "g_bias")}
    h["bias"] = tr.coll.bias.detach().cpu().numpy().copy()
    return h


def _row_mv(st, D):
    """[emb | w] views of m and v in gathered state blocks."""
    m = np.concatenate([st[:, D:2 * D], st[:, 3 * D + 1:3 * D + 2]], 1).astype(F64)
    v = np.concatenate([st[:, 2 * D:3 * D], st[:, 3 * D + 2:3 * D + 3]], 1).astype(F64)
    return m, v


@pytest.mark.parametrize("opt", ["adam_rows", "adam_rows_tf"])
def test_full_size_step(opt):
    """C2 as bench.py builds it (26 tables of 1 M rows, D = 16, B = 65536, DNN [256, 32], DeepFM seed 1, CUDA graph)
    under the fused row-sparse Adam: one step on a batch of uniform ids, then one on Zipf(1.05) ids, where row 0 and
    the clipped last row of every slot collect tens of thousands of lookups, all counted down by one atomic each in the
    backward.  The state blocks span 6.7 GB (64 floats per row), so rows sit at byte offsets beyond 4 GB.

    The oracle sees only the rows a batch touches, gathered on the device; every other row of the arena and of the
    state is compared bit for bit on the device.  Under "adam_rows_tf" the second step replays nothing (every touched
    row was last updated at step 0 or 1 = t - 1: asserted), so the forward reads the gathered rows as they were.

    Resolution: at lr = 0.01 the update alone says little about the gradient (Adam's first step moves a parameter by
    about lr * sign(g)); the gradient is read through m and v, whose bound carries the worst-case rounding of `hits`
    float32 additions into the zeroed gradient slot, hits * U * (sum of |contributions|).  That rules out a zero
    gradient for most touched elements (the printed counts), but not one lookup lost from a row looked up ~3e4 times:
    one lookup is ~1/3e4 of the row's terms, below the 3e4 * U ~ 1.8e-3 of them the rounding may take."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    t_start = time.perf_counter()
    dev = torch.device("cuda", 0)
    B, S, D, R_ = C2["batch"], C2["slots"], C2["dim"], C2["rows"]
    cols = [fc.categorical_column_with_identity(f"C{i}", R_) for i in range(S)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=C2["dnn"], seed=1, device=dev, sparse_lr=LR)
    tr = DeepFMTrainStep(model, batch_size=B, lr=LR, optimizer=opt, beta1=B1, beta2=B2, eps=EPS).capture()
    c = tr.coll
    assert c.layout == "fused" and tr.graph is not None and tr.state.shape[1] == 64
    gen = torch.Generator(device=dev).manual_seed(7)
    rep = Report()
    for t, kind in enumerate(("uniform", "zipf"), start=1):
        ids = _bench_ids(kind, dev)
        labels = torch.randint(0, 2, (B,), device=dev, generator=gen).float()
        ids_np = ids.cpu().numpy()
        uniq = [np.unique(ids_np[:, s]) for s in range(S)]
        cids = np.stack([np.searchsorted(uniq[s], ids_np[:, s]) for s in range(S)], 1)
        offs = c._offsets.cpu().numpy()
        grow = torch.from_numpy(np.concatenate([uniq[s] + offs[s] for s in range(S)])).to(dev)
        split = np.cumsum([len(u) for u in uniq])[:-1]
        rows0, st0, h0 = npy(c.weight.detach()[grow]), tr.state[grow].cpu().numpy(), _small(tr)
        stamp0 = st0[:, 3 * D + 4].view(np.int32)
        assert ((stamp0 == 0) | (stamp0 == t - 1)).all()
        tables, lins = np.split(rows0[:, :D], split), np.split(rows0[:, D], split)
        flat0 = h0["flat"].astype(F64)
        tw = _tower(tr)
        ws = [flat0[sl].reshape(sh) for k, sl, sh in tw if k.startswith("w.")]
        bs = [flat0[sl].reshape(sh) for k, sl, sh in tw if k.startswith("b.")]
        t0 = time.perf_counter()
        o = deepfm_step(tables, lins, float(h0["bias"][0]), ws, bs, "relu", cids, labels.cpu().numpy())
        t_oracle = time.perf_counter() - t0
        snap_w, snap_s = c.weight.detach().clone(), tr.state.clone()
        tr.step(ids, labels)
        torch.cuda.synchronize()
        for name, now, was in (("arena", c.weight.detach(), snap_w), ("state", tr.state, snap_s)):
            changed = (now.view(torch.int32) != was.view(torch.int32)).any(1)
            changed[grow] = False
            assert not bool(changed.any()), f"{kind}: {name} of a row the batch did not touch changed"
            del changed
        del snap_w, snap_s
        rows1, st1, h1 = npy(c.weight.detach()[grow]), tr.state[grow].cpu().numpy(), _small(tr)
        lr_gpu = F64(float(tr.clock.lr_t))
        assert int(tr.clock.step) == t and abs(lr_gpu - lr_t(t, LR, B1, B2)) <= 2 * U * lr_t(t, LR, B1, B2)
        got = lambda k, v: rep.got(k, v)
        got("loss", check("loss", float(tr.loss), o["loss"]))
        got("prob", check("prob", npy(tr.prob), o["prob"]))
        got("fm_logit", check("fm_logit", npy(tr.fm_logit), o["fm_logit"]))
        for i in range(len(tr.w)):
            got(f"acts.{i}", check(f"acts.{i}", npy(tr.acts[i]), o[f"acts.{i}"]))
        _check_tower_and_bias(tr, opt, o, h0, h1, lr_gpu, RTOL, rep)
        # the touched rows: gradient through m and v, update through the functor, invariants of the state blocks
        hits = np.concatenate([o[f"hits.{s}"] for s in range(S)])
        e = _rows_entry(o, S)
        extra = update_slack(0, 0, 1, hits[:, None], e.terms)
        (m0, v0), (mg, vg) = _row_mv(st0, D), _row_mv(st1, D)
        m1, bm_, v1, bv_ = moments(m0, v0, e, extra, B1, B2)
        got("m rows", check_bound(f"{kind}: m of the touched rows [emb | w]", mg, m1, bm_))
        got("v rows", check_bound(f"{kind}: v of the touched rows [emb | w]", vg, v1, bv_))
        p0 = np.concatenate([rows0[:, :D], rows0[:, D:D + 1]], 1)
        p1g = np.concatenate([rows1[:, :D], rows1[:, D:D + 1]], 1)
        p1, bp_ = functor(p0, mg, vg, lr_gpu, EPS)
        got("p rows", check_bound(f"{kind}: p of the touched rows [emb | w]", p1g, p1, bp_))
        assert np.array_equal(rows1[:, D + 1:].view(np.int32), rows0[:, D + 1:].view(np.int32)), "row padding changed"
        assert not st1[:, :D].any() and not st1[:, 3 * D].any(), "gradient slots not zero after the step"
        assert not st1[:, 3 * D + 3].view(np.int32).any(), "countdowns not zero after the step"
        stamp1 = st1[:, 3 * D + 4].view(np.int32)
        assert (stamp1 == t).all() if opt == "adam_rows_tf" else (stamp1 == 0).all()
        hot = int(np.argmax(hits))
        one = e.terms[hot] / hits[hot]                       # one lookup's mean |contribution| to the hot row
        eg = RTOL * e.scale[hot] + e.slack[hot] + extra[hot]
        zero_ok = resolved(e, extra)
        print(f"{kind}: float64 oracle {t_oracle:.1f} s on the host; most lookups of one row {int(hits[hot])}; "
              f"of {zero_ok.size} touched table and first-order elements, the m/v bound rules out a zero gradient "
              f"for {int(zero_ok.sum())}; on the hottest row one lost lookup is outside the bound for "
              f"{int((one > eg).sum())} of {D + 1} elements")
    print(f"{time.perf_counter() - t_start:.1f} s; max err/bound (err/scale for forward values and the grad buffer):",
          {k: f"{v:.1e}" for k, v in rep.items()})
