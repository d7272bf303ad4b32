"""optimizers.RowSparseAdam on the estimator models FM, DeepFM, WDL (deep part) and FNN, held to TensorFlow's dense Adam.

Each model trains T = 22 steps twice from the same seed: once with dense Adam over every variable (ops.adam_step_ over
the whole arena, what the examples run by default) and once with the tables on RowSparseAdam and the other variables on
dense Adam sharing its clock, whose rate ring is 16 steps long here.  The batches make rows sit out 1 step, 3 steps and
18 steps (outside the ring), or every step after the first (replayed by the final flush), and carry duplicate ids,
pruned ids (-1 and >= rows) and, where a model has one, a bag slot with empty bags, duplicate and pruned members.

Checked, per element, against the float64 model of tests/adam_oracle.py: every step is dense ApplyAdam from the arena the
kernels left at the end of the previous step -- the steps a row sat out replayed with a zero gradient (`replay`), then the
step's update (`moments`, `functor`) from a float64 row gradient formed from the per-lookup gradients the backward kept --
and rows the step did not read keep every bit.  After the last step, flush() must bring every row, m and v to the
replayed dense values.  Against the dense run: the per-step losses, an evaluation forward under no_grad between steps,
the flushed tables and FM.export's file.
"""
import numpy as np
import pytest
import torch

from adam_oracle import U, Entry, check_bound, functor, moments, replay

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
LR, B1, B2, EPS = 0.01, 0.9, 0.999, 1e-8
HIST = 16
T = 22
ROWS = {"a": 40, "b": 24, "c": 16}
BATCH = 24


def _columns(D, bags):
    from deep_recommenders_b200 import feature_column as fc
    keys = ["a", "b"] + (["c"] if bags else [])
    cats = [fc.categorical_column_with_identity(k, ROWS[k]) for k in keys]
    return [fc.indicator_column(c) for c in cats], [fc.embedding_column(c, dimension=D) for c in cats]


def _batch(t, bags):
    """Step t's features (and labels): column a carries the skip pattern, b random ids, c the bags."""
    from deep_recommenders_b200.feature_column import RaggedFeature
    rng = np.random.default_rng(1000 + t)
    a = [0, 0, 0, 1, 2, 3, -1, 40]                       # every step; row 0 three times; pruned
    if t % 2:
        a += [4, 5, 6, 7]                                # sit out 1 step
    if t % 4 == 1:
        a += [8, 9, 10, 11]                              # sit out 3 steps
    if t in (1, 20):
        a += [12, 13, 14, 15]                            # sit out 18 steps: beyond the 16-step ring
    if t == 1:
        a += [16, 17, 18, 19]                            # only the first step: the flush replays 21 steps
    a += list(rng.integers(20, 40, BATCH - len(a)))
    a = rng.permutation(np.asarray(a, np.int64))
    feats = {"a": a, "b": rng.integers(-1, ROWS["b"] + 1, BATCH).astype(np.int64)}
    if bags:
        vals, splits = [], [0]
        for b in range(BATCH):
            n = int(rng.integers(0, 4)) if b % 5 else 0                     # every fifth bag empty
            members = list(rng.integers(-1, ROWS["c"] + 1, n))             # pruned members at both ends
            if b == 1:
                members += [0, 0]                                           # a duplicate member
            if t in (1, 20) and b == 2:
                members += [4, 5]
            vals += members
            splits.append(len(vals))
        feats["c"] = RaggedFeature(np.asarray(vals, np.int64), np.asarray(splits, np.int64))
    return feats, (rng.random(BATCH) < 0.5).astype(np.float32)


class DenseAdam:
    """tf.train.AdamOptimizer over each variable (ops.adam_step_), as the examples keep it."""

    def __init__(self, params, history=0):
        from deep_recommenders_b200 import ops
        self.ops = ops
        self.params = [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in params]
        self.clock = ops.AdamClock(LR, B1, B2, EPS, device="cuda", history=history)

    def step(self):
        self.clock.advance()
        c = self.clock
        for p, m, v in self.params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            self.ops.adam_step_(p.data, p.grad, m, v, 0.0, c.beta1, c.beta2, c.eps, zero_grad=True, lr_t_dev=c.lr_t)


def _model(kind, D, bags, fm_path):
    from deep_recommenders.estimator.models.feature_interaction import FM
    from deep_recommenders.estimator.models.ranking import FNN, WDL, DeepFM
    cols = _columns(D, bags)
    if kind == "fm":
        return FM(*cols, seed=3, device="cuda")
    if kind == "deepfm":
        return DeepFM(*cols, [16, 8], seed=3, device="cuda")
    if kind == "wdl":
        return WDL(*cols, [16, 8], seed=3, device="cuda")
    return FNN(*cols, fm_path, [16, 8], seed=3, device="cuda")


def _loss(kind, model, feats, y):
    out = model(feats).reshape(-1)
    y = torch.from_numpy(y).cuda()
    if kind == "fm":
        return torch.nn.functional.binary_cross_entropy_with_logits(out, y)
    return torch.mean(-y * torch.log(out + 1e-7) - (1 - y) * torch.log(1 - out + 1e-7))


def _optimizers(model, rows_tf):
    from deep_recommenders_b200.optimizers import RowSparseAdam
    dense_vars = model.dense_variables()
    if not rows_tf:
        params = model.deep_variables() if hasattr(model, "deep_variables") else list(model.parameters())
        return DenseAdam(params), None
    dense = DenseAdam(dense_vars, history=HIST)
    return dense, RowSparseAdam(model.embedding_collection(), LR, B1, B2, EPS, clock=dense.clock)


def _host(coll, opt):
    """Float64 (p, m, v) [rows, D (+1 first-order)], the raw arena and the stamps."""
    D = coll.dim
    w = coll.weight.detach().cpu().numpy().copy()
    st = opt.state.detach().cpu().numpy().copy()
    p, m, v = w[:, :D], st[:, D:2 * D], st[:, 2 * D:3 * D]
    lin = None
    if coll.with_linear:
        lin = w[:, D] if coll.layout == "fused" else coll.linear.detach().cpu().numpy().copy()
        p = np.concatenate([p, lin[:, None]], 1)
        m = np.concatenate([m, st[:, 3 * D + 1:3 * D + 2]], 1)
        v = np.concatenate([v, st[:, 3 * D + 2:3 * D + 3]], 1)
    return dict(p=p.astype(F64), m=m.astype(F64), v=v.astype(F64), w=w, lin=lin,
                stamp=st[:, 3 * D + 4].view(np.int32).astype(np.int64), st=st)


def _grads64(opt, coll):
    """Float64 row gradients of the recorded backward [rows, D (+1)], their bound and the lookups per row."""
    from deep_recommenders_b200.optimizers import _FM
    R, D = coll.total_rows, coll.dim
    W = D + (1 if coll.with_linear else 0)
    G, A, SL = np.zeros((R, W)), np.zeros((R, W)), np.zeros((R, W))     # gradient, sum |contribution|, slack
    hits = np.zeros(R, np.int64)
    offs, nrows = coll._offsets.detach().cpu().numpy(), coll.rows_list

    def add(r, row, lin, slack):
        G[r, :D] += row
        A[r, :D] += np.abs(row)
        SL[r, :D] += slack
        if coll.with_linear:
            G[r, D] += lin
            A[r, D] += abs(lin)
        hits[r] += 1

    for rec in opt._pending:
        ids = rec.ids.detach().cpu().numpy()
        if isinstance(rec, _FM):
            stack = rec.stack.detach().cpu().numpy().astype(F64)
            sum_e = rec.sum_e.detach().cpu().numpy().astype(F64)
            gl = rec.g_logit.detach().cpu().numpy().astype(F64)
            gs = np.zeros_like(stack) if rec.g_stack is None else rec.g_stack.detach().cpu().numpy().astype(F64)
            for b, s in np.ndindex(*ids.shape):
                if 0 <= ids[b, s] < nrows[s]:
                    diff = sum_e[b] - stack[b, s]
                    d = gl[b] * diff + gs[b, s]
                    add(offs[s] + ids[b, s], d, gl[b], U * (2 * abs(gl[b]) * np.abs(diff) + np.abs(d)))
            continue
        g = rec.g.detach().cpu().numpy().reshape(-1).astype(F64)
        gl = None if rec.gl is None else rec.gl.detach().cpu().numpy().reshape(-1).astype(F64)
        lin_of = lambda b, s: 0.0 if gl is None else gl[rec.gl_off + b * rec.gl_ld + s * rec.gl_slot]
        row_of = lambda b, s: g[rec.g_off + b * rec.g_ld + s * rec.g_slot:][:D]
        if rec.slot is None:
            for b, s in np.ndindex(*ids.shape):
                if 0 <= ids[b, s] < nrows[s]:
                    add(offs[s] + ids[b, s], row_of(b, s), lin_of(b, s), 0.0)
            continue
        s, splits = rec.slot, rec.splits.detach().cpu().numpy()
        for b in range(rec.B):
            members = [q for q in ids[splits[b]:splits[b + 1]] if 0 <= q < nrows[s]]
            for q in members:
                row = row_of(b, 0) / len(members)
                add(offs[s] + q, row, lin_of(b, 0), U * np.abs(row))
    return Entry(G, 0.0, SL + hits[:, None] * U * A), hits


def _check_replay(name, before, after, rows, upto, t_now):
    """Rows `rows` of `after` are `before` replayed up to step `upto` (zero-gradient dense Adam)."""
    p, m, v, bp, bm, bv = replay(before["p"][rows], before["m"][rows], before["v"][rows], before["stamp"][rows], upto,
                                 LR, B1, B2, EPS, t_now=t_now, hist_len=HIST)
    check_bound(f"{name} p", after["p"][rows], p, bp)
    check_bound(f"{name} m", after["m"][rows], m, bm)
    check_bound(f"{name} v", after["v"][rows], v, bv)


def _check_step(name, s0, s1, entry, hits, t, lr_t_):
    """Step t: touched rows = s0 replayed to t-1, then ApplyAdam with the float64 gradient; the others unchanged."""
    hit = hits > 0
    p, m, v, bp, bm, bv = replay(s0["p"][hit], s0["m"][hit], s0["v"][hit], s0["stamp"][hit], t - 1, LR, B1, B2, EPS,
                                 t_now=t - 1, hist_len=HIST)
    e = Entry(entry.ref[hit], 0.0, entry.slack[hit])
    m1, bm1, v1, bv1 = moments(m, v, e, 0.0, B1, B2, m0_err=bm, v0_err=bv)
    check_bound(f"{name} m", s1["m"][hit], m1, bm1)
    check_bound(f"{name} v", s1["v"][hit], v1, bv1)
    p1, bp1 = functor(p, s1["m"][hit], s1["v"][hit], lr_t_, EPS, p0_err=bp)
    check_bound(f"{name} p", s1["p"][hit], p1, bp1)
    assert (s1["stamp"][hit] == t).all(), f"{name}: stamps of the touched rows"
    assert np.array_equal(s1["w"][~hit], s0["w"][~hit]), f"{name}: an untouched row moved"
    assert np.array_equal(s1["st"][~hit], s0["st"][~hit]), f"{name}: the state of an untouched row changed"


CASES = [pytest.param("fm", 8, False, id="fm_fused"), pytest.param("fm", 32, True, id="fm_split_bags"),
         pytest.param("deepfm", 8, False, id="deepfm"), pytest.param("deepfm", 8, True, id="deepfm_bags"),
         pytest.param("wdl", 8, False, id="wdl"), pytest.param("wdl", 8, True, id="wdl_bags"),
         pytest.param("fnn", 8, False, id="fnn"), pytest.param("fnn", 8, True, id="fnn_bags")]


@pytest.mark.parametrize("kind,D,bags", CASES)
def test_rows_tf_equals_dense_adam(tmp_path, kind, D, bags):
    from deep_recommenders.estimator.models.feature_interaction import FM
    fm_path = str(tmp_path / "fm.pt")
    if kind == "fnn":
        FM(*_columns(D, bags), seed=5, device="cuda").export(fm_path)
    dense_model, rows_model = _model(kind, D, bags, fm_path), _model(kind, D, bags, fm_path)
    dense_opt, _ = _optimizers(dense_model, False)
    tower_opt, rows_opt = _optimizers(rows_model, True)
    coll = rows_model.embedding_collection()
    dense_losses, rows_losses = [], []
    for t in range(1, T + 1):
        feats, y = _batch(t, bags)
        loss = _loss(kind, dense_model, feats, y)
        loss.backward()
        dense_opt.step()
        dense_losses.append(float(loss.detach()))

        s0 = _host(coll, rows_opt)
        loss = _loss(kind, rows_model, feats, y)
        loss.backward()
        entry, hits = _grads64(rows_opt, coll)
        tower_opt.step()
        rows_opt.step()
        rows_losses.append(float(loss.detach()))
        s1 = _host(coll, rows_opt)
        _check_step(f"{kind} step {t}", s0, s1, entry, hits, t, float(rows_opt.clock.lr_t))

        if t in (9, 21):         # evaluation between steps reads what dense Adam left
            ev, _ = _batch(100 + t, bags)
            e0 = _host(coll, rows_opt)
            with torch.no_grad():
                want, got = dense_model(ev), rows_model(ev)
            torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
            e1 = _host(coll, rows_opt)
            moved = (e1["stamp"] != e0["stamp"])
            assert (e1["stamp"][moved] == t).all()
            _check_replay(f"{kind} evaluation at {t}", e0, e1, moved, t, t)

    np.testing.assert_allclose(rows_losses, dense_losses, rtol=1e-4, atol=1e-5)
    assert not rows_opt._pending
    with pytest.raises(RuntimeError, match="no backward"):
        rows_opt.step()

    before = _host(coll, rows_opt)
    rows_opt.flush()
    after = _host(coll, rows_opt)
    _check_replay(f"{kind} flush", before, after, np.ones(coll.total_rows, bool), T, T)
    assert (after["stamp"][before["stamp"] > 0] == T).all()

    dcoll = dense_model.embedding_collection()
    torch.testing.assert_close(coll.emb_view().detach(), dcoll.emb_view().detach(), rtol=1e-4, atol=1e-5)
    if coll.with_linear:
        torch.testing.assert_close(coll.lin_view().detach(), dcoll.lin_view().detach(), rtol=1e-4, atol=1e-5)
    # the arena is flushed before state_dict() reads it
    sd = coll.state_dict()
    assert torch.equal(sd["weight"], coll.weight.detach())


def test_fm_export_and_fnn_warm_start_match_the_dense_run(tmp_path):
    from deep_recommenders.estimator.models.ranking import FNN
    paths = {}
    for rows_tf in (False, True):
        model = _model("fm", 8, True, None)
        dense, rows = _optimizers(model, rows_tf)
        for t in range(1, 12):
            feats, y = _batch(t, True)
            _loss("fm", model, feats, y).backward()
            dense.step()
            if rows is not None:
                rows.step()
        paths[rows_tf] = str(tmp_path / f"fm_{rows_tf}.pt")
        model.export(paths[rows_tf])     # flushes first under rows_tf: rows 16..19 sat out 10 steps
    want = torch.load(paths[False], weights_only=True)
    got = torch.load(paths[True], weights_only=True)
    torch.testing.assert_close(got["bias"], want["bias"], rtol=1e-4, atol=1e-6)
    for part in ("linear", "factorized"):
        assert got[part].keys() == want[part].keys()
        for k in want[part]:
            torch.testing.assert_close(got[part][k], want[part][k], rtol=1e-4, atol=1e-5)
    fnn = FNN(*_columns(8, True), paths[True], [16, 8], seed=3, device="cuda")
    for s, k in enumerate(["a", "b", "c"]):
        assert torch.equal(fnn.embeddings.table(s).cpu(), got["factorized"][k])


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L.load()


@pytest.mark.parametrize("layout", ["fused", "split_nolin"])
@pytest.mark.parametrize("bag", [False, True], ids=["dense", "bag"])
def test_kernels_write_between_sentinels(layout, bag):
    """dr_embed_adam_catch_up / dr_embed_adam_rows_tf called through the C-ABI on an arena and state blocks framed by
    sentinel rows: nothing outside the touched rows' p, m, v, first-order slot and stamp changes; the pad columns of a
    fused row keep their bits, and so do a no-first-order table's state floats 3D..3D+2."""
    lib = _lib()
    D, rows = 8, [10, 6]
    fused = layout == "fused"
    rs = 32 if fused else D
    R, G = sum(rows), 4                                              # G sentinel rows on each side
    SS = lib.dr_embed_adam_state_stride(D)
    sentinel = float(np.frombuffer(np.uint32(0x5EBADBAD).tobytes(), F32)[0])
    arena = torch.full((R + 2 * G, rs), sentinel, device="cuda")
    state = torch.full((R + 2 * G, SS), sentinel, device="cuda")
    rng = np.random.default_rng(0)
    arena[G:G + R, :D] = torch.from_numpy(rng.standard_normal((R, D)).astype(F32)).cuda()
    if fused:
        arena[G:G + R, D] = torch.from_numpy(rng.standard_normal(R).astype(F32)).cuda()
    st = np.zeros((R, SS), F32)
    st[:, D:3 * D] = np.abs(rng.standard_normal((R, 2 * D))) * 1e-3
    st[:, 3 * D + 1:3 * D + 3] = np.abs(rng.standard_normal((R, 2))) * 1e-3
    st[:, 3 * D + 4] = np.array([3] * R, np.int32).view(F32)          # every row last updated at step 3
    st[:, 3 * D + 5:] = sentinel                                      # the block's padding
    if not fused:
        st[:, 3 * D:3 * D + 3] = sentinel                             # no first-order slot: must stay as it is
    state[G:G + R] = torch.from_numpy(st).cuda()
    offs = torch.tensor([0, rows[0]], dtype=torch.int64, device="cuda")
    nrows = torch.tensor(rows, dtype=torch.int64, device="cuda")
    base = arena[G:].data_ptr()
    tp = torch.tensor([base + 4 * rs * 0, base + 4 * rs * rows[0]], dtype=torch.int64, device="cuda")
    flags = 1 if fused else 0
    step = torch.tensor([8], dtype=torch.int64, device="cuda")
    lr_t = torch.zeros(1, device="cuda")
    hist = torch.zeros(HIST, device="cuda")
    for _ in range(2):                                                # steps 9, 10 in the ring
        assert lib.dr_adam_advance_hist(step.data_ptr(), LR, B1, B2, lr_t.data_ptr(), hist.data_ptr(), HIST, None) == 0
    step.fill_(9)                                                     # the forward of step 10 runs at t = 9
    stp = state[G:].data_ptr()
    if bag:
        ids = torch.tensor([1, 1, -1, 6, 3, 2], dtype=torch.int64, device="cuda")    # slot 1 (6 rows): 6 is pruned
        splits = torch.tensor([0, 3, 3, 6], dtype=torch.int64, device="cuda")
        n, B, S, s = 6, 3, 1, 1
    else:
        ids = torch.tensor([[0, 5], [9, 5], [-1, 6], [2, 0]], dtype=torch.int64, device="cuda")
        splits, n, B, S, s = None, 8, 4, 2, 0
    g = torch.from_numpy(rng.standard_normal((B, S * D)).astype(F32)).cuda()
    gl = torch.from_numpy(rng.standard_normal((B, S)).astype(F32)).cuda() if fused else None
    sub = lambda t: t.data_ptr() + 8 * s
    rc = lib.dr_embed_adam_catch_up(ids.data_ptr(), 8, n, S, D, sub(nrows), sub(offs), rs, 1 if not fused else rs, flags,
                                    sub(tp), None, stp, step.data_ptr(), hist.data_ptr(), HIST, LR, B1, B2, EPS, None)
    assert rc == 0
    step.fill_(10)
    assert lib.dr_embed_adam_count(ids.data_ptr(), 8, n // S, S, D, sub(nrows), sub(offs), stp, None) == 0
    rc = lib.dr_embed_adam_rows_tf(ids.data_ptr(), 8, n, B, S, None if splits is None else splits.data_ptr(), sub(nrows),
                                   sub(offs), g.data_ptr(), S * D, D if S > 1 else 0,
                                   None if gl is None else gl.data_ptr(), S, 1, D, rs, rs if fused else 1, flags,
                                   sub(tp), None, stp, step.data_ptr(), lr_t.data_ptr(), hist.data_ptr(), HIST, LR, B1,
                                   B2, EPS, None)
    assert rc == 0
    torch.cuda.synchronize()
    a, sta = arena.detach().cpu().numpy(), state.detach().cpu().numpy()
    sbits = np.uint32(0x5EBADBAD)
    for name, x in (("arena", a), ("state", sta)):
        assert (x[:G].view(np.uint32) == sbits).all() and (x[G + R:].view(np.uint32) == sbits).all(), name
    if fused:
        assert (a[G:G + R, D + 1:].view(np.uint32) == sbits).all(), "pad columns of a fused row"
    else:
        assert (sta[G:G + R, 3 * D:3 * D + 3].view(np.uint32) == sbits).all(), "first-order state of a table without"
    assert (sta[G:G + R, 3 * D + 5:].view(np.uint32) == sbits).all(), "state padding"
    touched = sta[G:G + R, 3 * D + 4].view(np.int32) == 10
    assert touched.sum() == (3 if bag else 5)                        # distinct valid rows of the lookups
    assert (sta[G:G + R][touched][:, :D] == 0).all(), "gradient accumulators are cleared"
    assert (sta[G:G + R][touched][:, 3 * D + 3].view(np.int32) == 0).all(), "counts are back to zero"
