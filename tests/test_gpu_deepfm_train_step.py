"""DeepFMTrainStep with optimizer="sgd" (the step bench.py measures) against the float64 oracle of one DeepFM step
(tests/deepfm_oracle.py): every value the step computes and every parameter's gradient, per element, within
RTOL * (sum of |terms|), plus the relu' slack and the float32 rounding of the update the oracle names.

One step runs at lr = 1, so (before - after) / lr recovers the gradient the update applied; the tower's gradient is
also read from the trainer's gradient buffer, which shows the update used that buffer.  First-order weights, the
global bias and every tower bias start non-zero, so a bias read or written in the wrong place shows on step 1.

The one-step cases vary one axis at a time from a base case, then stack the risky ones; each `_enqueue` branch has
a case that takes it:
  fused head (last hidden layer <= 256 wide): base ([64, 32]);  no head: "tower_260";
  head with L = 2 (the head writes layer 0's bias gradient, gb0 = None): "tower_32";
  one Dense(1) (top0): "tower_1";  chunk_l0 (fwd_chunks > 1): "chunks_2", "chunks_3", "B4099_chunks3_tc";
  embed_fwd="tma": "tma";  dw_first with tc_dw_share = 1: "dw_first".
"""
import os
import time

import numpy as np
import pytest
import torch

from deepfm_oracle import RTOL, U, Entry, bias_additions, check, deepfm_step, resolved, update_slack

pytestmark = pytest.mark.gpu

F64 = np.float64
ROWS = [97, 7, 300, 1000, 41, 13]


@pytest.fixture
def knobs():
    """knobs(gemm_variant=, embed_bwd=(mode, agg), tc_dw_share=) for one test; everything goes back afterwards."""
    from deep_recommenders_b200 import _lib
    _lib.load()
    saved_variant, saved_share = _lib.tune_get("gemm_variant"), _lib.tune_get("tc_dw_share")
    saved_py = (_lib._tc_enabled, _lib._tc_variant, _lib._tc_applied)

    def set_(gemm_variant=2, embed_bwd=(0, 1), tc_dw_share=0):
        if gemm_variant == 0:
            _lib.disable_tensor_core_gemm()
        else:
            _lib.enable_tensor_core_gemm(variant=gemm_variant)
        _lib.tune("embed_bwd_mode", embed_bwd[0])
        _lib.tune("embed_bwd_agg", embed_bwd[1])
        _lib.tune("tc_dw_share", tc_dw_share)

    yield set_
    _lib.tune("embed_bwd_mode", 0)              # the library's defaults (write-only knobs)
    _lib.tune("embed_bwd_agg", 1)
    _lib.tune("tc_dw_share", saved_share)
    _lib.tune("gemm_variant", saved_variant)
    _lib._tc_enabled, _lib._tc_variant, _lib._tc_applied = saved_py


def npy(t):
    return t.detach().cpu().numpy().astype(F64)


def _trainer(units, act, D, B, rows, lr, id_dtype=torch.int64, seed=5, **opts):
    """A DeepFM step whose first-order weights, global bias and tower biases are all non-zero."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=list(units), dnn_activation=act, seed=seed, device="cuda")
    tr = DeepFMTrainStep(model, batch_size=B, lr=lr, id_dtype=id_dtype, **opts)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        model.embeddings.lin_view().normal_(0, 0.1, generator=gen)
        model.embeddings.bias.fill_(0.2)
        for b in tr.b:
            b.normal_(0, 0.1, generator=gen)
    return tr.capture()


def _batch(rng, rows, B):
    """ids with OOV of both kinds (-1 and == rows); from B = 1000 on, one id of slot 0 looked up 1000 times."""
    ids = np.stack([rng.integers(-1, r + 1, B) for r in rows], 1).astype(np.int64)
    if B >= 1000:
        ids[:1000, 0] = 5
    return ids, rng.integers(0, 2, B).astype(np.float32)


def _params(tr):
    c = tr.coll
    return ([npy(c.table(s)) for s in range(tr.S)], [npy(c.linear_of(s)) for s in range(tr.S)], float(c.bias.detach()),
            [npy(w) for w in tr.w], [npy(b) for b in tr.b])


def _check_step(tr, o, before, lr, B, report):
    """Every forward value, the gradient buffer and the gradients recovered from the update."""
    tables, lins, bias, ws, bs = before
    got = lambda k, t, e, extra=0.0: report.__setitem__(k, max(report.get(k, 0.0), check(k, t, e, extra=extra)))
    got("loss", float(tr.loss), o["loss"])
    got("prob", npy(tr.prob), o["prob"])
    got("fm_logit", npy(tr.fm_logit), o["fm_logit"])
    got("stack", npy(tr.stack), o["stack"])
    for i in range(len(ws)):
        got(f"acts.{i}", npy(tr.acts[i]), o[f"acts.{i}"])
        for k, buf, p0, p1 in ((f"w.{i}", tr.gw[i], ws[i], tr.w[i]), (f"b.{i}", tr.gb[i], bs[i], tr.b[i])):
            e = o[k]
            got("grad buffer " + k, npy(buf), e)
            after = npy(p1)
            got("update " + k, (p0 - after) / lr, e, update_slack(p0, after, lr, 1, e.terms))
    c = tr.coll
    for s in range(tr.S):
        hits = o[f"hits.{s}"]
        for k, p0, p1, h in ((f"table.{s}", tables[s], c.table(s), hits[:, None]), (f"lin.{s}", lins[s], c.linear_of(s), hits)):
            e = o[k]
            after = npy(p1)
            got("update " + k, (p0 - after) / lr, e, update_slack(p0, after, lr, h, e.terms))
    _check_bias(float(c.bias.detach()), bias, o["bias"], lr, B, got)


def _check_bias(after, before, e, lr, B, got):
    """The global bias's update; this batch's bound is below |gradient|, so a missing gradient would fail it."""
    extra = update_slack(before, after, lr, bias_additions(B, _sms()), e.terms)
    assert resolved(e, extra), "this batch cannot tell a missing global-bias gradient: pick other data"
    got("update bias", (before - after) / lr, e, extra)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _touched_rows(tr, ids):
    c = tr.coll
    mask = torch.zeros(c.total_rows, dtype=torch.bool, device="cuda")
    for s, r in enumerate(c.rows_list):
        col = ids[:, s]
        ok = col[(col >= 0) & (col < r)]
        mask[int(c._offsets[s]) + torch.from_numpy(ok).cuda()] = True
    return mask


def _check_bits(tr, arena0, lin0, touched):
    """Rows the batch did not touch are bit-unchanged; so is the padding of every fused row."""
    c = tr.coll
    bits = lambda t: t.detach().view(torch.int32)
    assert torch.equal(bits(c.weight)[~touched], bits(arena0)[~touched]), "an untouched row changed"
    if c.linear is not None:
        assert torch.equal(bits(c.linear)[~touched], bits(lin0)[~touched]), "an untouched first-order weight changed"
    if c.layout == "fused":
        assert torch.equal(bits(c.weight)[:, c.dim + 1:], bits(arena0)[:, c.dim + 1:]), "row padding changed"


def _case(name, units=(64, 32), act="relu", D=16, B=1200, id_dtype=torch.int64, S=None, use_graph=True,
          fwd_chunks=1, embed_fwd="ldg", dw_first=False, gemm_variant=2, embed_bwd=(0, 1)):
    return pytest.param(dict(units=list(units), act=act, D=D, B=B, id_dtype=id_dtype, S=S, use_graph=use_graph,
                             fwd_chunks=fwd_chunks, embed_fwd=embed_fwd, dw_first=dw_first,
                             gemm_variant=gemm_variant, embed_bwd=embed_bwd), id=name)


CASES = [
    _case("base"),                                            # [64, 32] relu, fused D = 16, fused head with L = 3
    # tower
    _case("tower_32", units=[32]),                            # head with L = 2: gb0 = None
    _case("tower_1", units=[]),                               # one Dense(1): top0
    _case("tower_256", units=[256]),                          # head at its 256 limit
    _case("tower_260", units=[260]),                          # no head: dr_bce + the chained top layer
    _case("tower_128_64_32", units=[128, 64, 32]),
    _case("tower_100_33", units=[100, 33]),                   # widths not a multiple of 4: the FFMA fallback
    # activation (the chain and the head take _act of the layer below)
    _case("tanh", act="tanh"),
    _case("sigmoid", act="sigmoid"),
    # layout / D
    _case("fused_D4", D=4), _case("fused_D12", D=12), _case("fused_D28", D=28),
    _case("split_D32", D=32), _case("split_D64", D=64), _case("split_D128", D=128),
    # B: ragged 128-row tiles
    _case("B1", B=1), _case("B127", B=127), _case("B129", B=129), _case("B4099", B=4099),
    # ids
    _case("int32", id_dtype=torch.int32),
    # step options
    _case("eager", use_graph=False),
    _case("chunks_2", fwd_chunks=2), _case("chunks_3", fwd_chunks=3),
    _case("tma", embed_fwd="tma"),                            # serves fused D = 16 with S <= 32 only
    _case("dw_first", dw_first=True),                         # run with tc_dw_share = 1
    # knobs
    _case("ffma", gemm_variant=0), _case("tc", gemm_variant=1),
    _case("bwd_example_parallel", embed_bwd=(1, 0)), _case("bwd_example_parallel_agg", embed_bwd=(1, 1)),
    _case("S120", S=120, B=257),                              # opt-in shared memory in the forward
    # the risky ones stacked
    _case("B4099_chunks3_tc", B=4099, fwd_chunks=3, gemm_variant=1),
    _case("B129_chunks2_tanh", B=129, fwd_chunks=2, act="tanh"),
    _case("split_D64_int32_sigmoid_eager", D=64, id_dtype=torch.int32, act="sigmoid", use_graph=False),
    _case("tower_1_split_D32_chunks2", units=[], D=32, fwd_chunks=2),
    _case("tower_260_tanh_B129_agg_ffma", units=[260], act="tanh", B=129, embed_bwd=(1, 1), gemm_variant=0),
    _case("tower_100_33_tc_B4099", units=[100, 33], gemm_variant=1, B=4099),
    _case("tower_32_sigmoid_dw_first_tc", units=[32], act="sigmoid", dw_first=True, gemm_variant=1),
    _case("tma_int32_eager", embed_fwd="tma", id_dtype=torch.int32, use_graph=False),
]


@pytest.mark.parametrize("cfg", CASES)
def test_one_step_matches_oracle(knobs, cfg):
    knobs(gemm_variant=cfg["gemm_variant"], embed_bwd=cfg["embed_bwd"], tc_dw_share=int(cfg["dw_first"]))
    rows = ROWS if cfg["S"] is None else [37] * cfg["S"]
    B, lr = cfg["B"], 1.0                   # one step: p - g keeps every bit of g that float32 can hold next to p
    tr = _trainer(cfg["units"], cfg["act"], cfg["D"], B, rows, lr, cfg["id_dtype"], use_graph=cfg["use_graph"],
                  fwd_chunks=cfg["fwd_chunks"], embed_fwd=cfg["embed_fwd"], dw_first=cfg["dw_first"])
    assert (tr.graph is not None) == cfg["use_graph"]
    ids, labels = _batch(np.random.default_rng(B + len(rows)), rows, B)
    before = _params(tr)
    o = deepfm_step(*before, cfg["act"], ids, labels)
    arena0 = tr.coll.weight.detach().clone()
    lin0 = None if tr.coll.linear is None else tr.coll.linear.detach().clone()
    tr.step(torch.from_numpy(ids).cuda().to(cfg["id_dtype"]), torch.from_numpy(labels).cuda())
    torch.cuda.synchronize()
    report = {}
    _check_step(tr, o, before, lr, B, report)
    _check_bits(tr, arena0, lin0, _touched_rows(tr, ids))
    print("max err/scale:", {k: f"{v:.1e}" for k, v in report.items() if v > 0})


# ---- three steps against the float64 SGD recursion ---------------------------------------------------------------
@pytest.mark.parametrize("gemm_variant", [1, 2])
@pytest.mark.parametrize("use_graph", [True, False])
def test_three_steps_match_float64_sgd(knobs, use_graph, gemm_variant):
    """State carried between steps: a tower gradient added onto the previous step's, planes cached from the previous
    step's weights, a graph holding a stale pointer.  The oracle applies its own gradients in float64; the bound on
    every parameter is the sum of the per-step bounds."""
    knobs(gemm_variant=gemm_variant)
    units, act, D, B, lr = [64, 32], "relu", 16, 1200, 0.05
    tr = _trainer(units, act, D, B, ROWS, lr, use_graph=use_graph)
    tables, lins, bias, ws, bs = _params(tr)
    tol = {}                                    # accumulated per-step bounds, in parameter units
    gtol = {}                                   # and in gradient units
    rng = np.random.default_rng(17)
    for k in range(3):
        ids, labels = _batch(rng, ROWS, B)
        o = deepfm_step(tables, lins, bias, ws, bs, act, ids, labels)
        tr.step(torch.from_numpy(ids).cuda(), torch.from_numpy(labels).cuda())
        torch.cuda.synchronize()
        for i in range(len(ws)):
            for name, buf in ((f"w.{i}", tr.gw[i]), (f"b.{i}", tr.gb[i])):
                e = o[name]
                gtol[name] = gtol.get(name, 0.0) + RTOL * e.scale + e.slack
                check(f"step {k + 1} grad buffer {name}", npy(buf), e._replace(scale=0.0, slack=gtol[name]))

        def apply(name, p, adds):
            e = o[name]
            tol[name] = tol.get(name, 0.0) + lr * (RTOL * e.scale + e.slack) + adds * U * (np.abs(p) + lr * e.terms)
            return p - lr * e.ref

        for s in range(len(ROWS)):
            hits = o[f"hits.{s}"]
            tables[s] = apply(f"table.{s}", tables[s], hits[:, None])
            lins[s] = apply(f"lin.{s}", lins[s], hits)
        bias = apply("bias", bias, bias_additions(B, _sms()))
        ws = [apply(f"w.{i}", w, 1) for i, w in enumerate(ws)]
        bs = [apply(f"b.{i}", b, 1) for i, b in enumerate(bs)]
    got = _params(tr)
    pairs = [(f"table.{s}", got[0][s], tables[s]) for s in range(len(ROWS))]
    pairs += [(f"lin.{s}", got[1][s], lins[s]) for s in range(len(ROWS))]
    pairs += [("bias", got[2], bias)]
    pairs += [(f"w.{i}", got[3][i], ws[i]) for i in range(len(ws))] + [(f"b.{i}", got[4][i], bs[i]) for i in range(len(bs))]
    for name, have, want in pairs:
        check(f"after 3 steps {name}", have, Entry(want, 0.0, tol[name]))


# ---- the benchmark's own step at full size ---------------------------------------------------------------------------
C2 = dict(slots=26, rows=1_000_000, dim=16, batch=65536, dnn=[256, 32])


def _bench_ids(kind, dev):
    """The id expressions of bench.py (first batch of its pool; seed 100 + rank at rank 0)."""
    B, S = C2["batch"], C2["slots"]
    if kind == "zipf":
        rng = np.random.default_rng(100)
        return torch.from_numpy(np.minimum(rng.zipf(1.05, size=(B, S)) - 1, C2["rows"] - 1).astype(np.int64)).to(dev)
    gen = torch.Generator(device=dev).manual_seed(100)
    return torch.randint(0, C2["rows"], (B, S), device=dev, generator=gen)


def test_bench_step_at_full_size():
    """C2 built as bench.py builds it (DeepFM seed 1, lr 0.01, CUDA graph), one step on a batch of uniform ids, then
    one on a batch of Zipf(1.05) ids, where row 0 and the clipped last row of every slot collect tens of thousands of
    lookups.  The oracle sees only the rows the batch touches (gathered on the device); the other rows of the 3.3 GB
    arena are compared bit for bit on the device.

    At lr = 0.01 the update of a row looked up ~3e4 times is not resolvable through (before - after) / lr: the worst
    case of that many float32 additions onto |p| ~ 0.25 exceeds the gradient.  Such rows are still held to that bound,
    and their gradient is checked through a replay of the same backward into a zeroed arena; the printed line counts
    the elements each way resolves and those neither does.  Neither resolves one lookup's contribution lost from a
    row looked up ~3e4 times: that is below the worst-case rounding of the row's own sum.  The float64 oracle of one
    such step took 12-13 s of host time beside an H100 80GB HBM3 (700 W); the whole test 31 s.  Both are printed."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    dev = torch.device("cuda", 0)
    B, S, D, R_ = C2["batch"], C2["slots"], C2["dim"], C2["rows"]
    cols = [fc.categorical_column_with_identity(f"C{i}", R_) for i in range(S)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=C2["dnn"], seed=1, device=dev, sparse_lr=0.01)
    lr = 0.01
    tr = DeepFMTrainStep(model, batch_size=B, lr=lr).capture()
    c = tr.coll
    assert c.layout == "fused" and tr.graph is not None
    gen = torch.Generator(device=dev).manual_seed(7)
    for kind in ("uniform", "zipf"):           # the second step starts from the first one's non-zero biases
        ids = _bench_ids(kind, dev)
        labels = torch.randint(0, 2, (B,), device=dev, generator=gen).float()
        ids_np = ids.cpu().numpy()
        # compact every slot to the rows this batch touches
        uniq = [np.unique(ids_np[:, s]) for s in range(S)]
        cids = np.stack([np.searchsorted(uniq[s], ids_np[:, s]) for s in range(S)], 1)
        offs = c._offsets.cpu().numpy()
        grow = torch.from_numpy(np.concatenate([uniq[s] + offs[s] for s in range(S)])).to(dev)
        split = np.cumsum([len(u) for u in uniq])[:-1]
        rows0 = npy(c.weight.detach()[grow])
        tables = np.split(rows0[:, :D], split)
        lins = np.split(rows0[:, D], split)
        bias, ws, bs = float(c.bias.detach()), [npy(w) for w in tr.w], [npy(b) for b in tr.b]
        t0 = time.perf_counter()
        o = deepfm_step(tables, lins, bias, ws, bs, "relu", cids, labels.cpu().numpy())
        t_oracle = time.perf_counter() - t0
        snap = c.weight.detach().clone()
        tr.step(ids, labels)
        torch.cuda.synchronize()
        changed = (c.weight.detach().view(torch.int32) != snap.view(torch.int32)).any(1)
        changed[grow] = False
        assert not bool(changed.any()), f"{kind}: a row the batch did not touch changed"
        del snap, changed
        rows1 = npy(c.weight.detach()[grow])
        assert np.array_equal(rows1[:, D + 1:], rows0[:, D + 1:]), "row padding changed"
        report = {}
        got = lambda k, t, e, extra=0.0: report.__setitem__(k, check(f"{kind} {k}", t, e, extra=extra))
        got("loss", float(tr.loss), o["loss"])
        got("prob", npy(tr.prob), o["prob"])
        got("fm_logit", npy(tr.fm_logit), o["fm_logit"])
        for i in range(len(ws)):
            got(f"acts.{i}", npy(tr.acts[i]), o[f"acts.{i}"])
            for k, buf, p0, p1 in ((f"w.{i}", tr.gw[i], ws[i], tr.w[i]), (f"b.{i}", tr.gb[i], bs[i], tr.b[i])):
                e = o[k]
                got("grad buffer " + k, npy(buf), e)
                after = npy(p1)
                got("update " + k, (p0 - after) / lr, e, update_slack(p0, after, lr, 1, e.terms))
        _check_bias(float(c.bias.detach()), bias, o["bias"], lr, B, got)
        # The same backward replayed on this step's buffers (ids, stack, sum_e, dL/dlogit, g_stack) with scale 1 into
        # a zeroed gradient arena: its running values start at 0 instead of |p|, so rows whose update is too small
        # to resolve through (before - after) / lr are checked here.
        g_arena, g_bias = torch.zeros_like(c.weight.detach()), torch.zeros(1, device=dev)
        gtp, glp, _ = c.pointers(g_arena, None, cache=False)
        from deep_recommenders_b200._lib import check as rc
        rc(tr.lib.dr_embed_fm_bwd(tr.ids.data_ptr(), tr.ids.element_size(), tr.rows.data_ptr(), tr.stack.data_ptr(),
                                  tr.sum_e.data_ptr(), tr.g_acts[-1].data_ptr(), tr.g_stack.data_ptr(), B, S, D,
                                  c.row_stride, c.lin_stride, c.flags, gtp.data_ptr(), glp.data_ptr(), g_bias.data_ptr(),
                                  1.0, torch.cuda.current_stream().cuda_stream), "dr_embed_fm_bwd")
        grad = npy(g_arena[grow])
        del g_arena
        rows1 = np.split(rows1, split)
        grad = np.split(grad, split)
        count = dict(update=0, replay=0, neither=0, all=0)
        for s in range(S):
            hits = o[f"hits.{s}"]
            for k, col, h in ((f"table.{s}", slice(0, D), hits[:, None]), (f"lin.{s}", D, hits)):
                e, p0 = o[k], (tables[s] if col != D else lins[s])
                p1 = rows1[s][:, col]
                upd = update_slack(p0, p1, lr, h, e.terms)
                got("update " + k, (p0 - p1) / lr, e, upd)
                rep = update_slack(0.0, 0.0, 1.0, h, e.terms)
                got("replay " + k, grad[s][:, col], e, rep)
                a, b = resolved(e, upd), resolved(e, rep)
                count["update"] += int(a.sum())
                count["replay"] += int((b & ~a).sum())
                count["neither"] += int((~a & ~b).sum())
                count["all"] += a.size
        got("replay bias", float(g_bias), o["bias"], update_slack(0.0, 0.0, 1.0, bias_additions(B, _sms()), o["bias"].terms))
        print(f"{kind}: float64 oracle {t_oracle:.1f} s on the host, most lookups of one row "
              f"{max(int(o[f'hits.{s}'].max()) for s in range(S))}; of {count['all']} touched table and first-order "
              f"elements, a zero update is ruled out through the update for {count['update']}, only through the "
              f"replay for {count['replay']}, by neither for {count['neither']}; max err/scale:",
              {k: f"{v:.1e}" for k, v in report.items() if v > 0 and not k.startswith(("update t", "update l", "replay"))})


# ---- the sharded trainer at world size 1 -----------------------------------------------------------------------------
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_world1_sharded_step_matches_oracle(exchange):
    import torch.distributed as dist
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    from test_gpu_sharded import _free_port
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(_free_port())
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        D, rows, B, lr = 16, [300, 7, 50, 1000, 21], 1100, 1.0
        cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
        sh = ShardedDeepFMTrainStep(cols, D, [32, 8], batch_size=B, lr=lr, seed=3, device="cuda", exchange=exchange)
        gen = torch.Generator(device="cuda").manual_seed(3)
        with torch.no_grad():
            sh.emb.lin_view().normal_(0, 0.1, generator=gen)
            sh.bias.fill_(0.2)
            for b in sh.b:
                b.normal_(0, 0.1, generator=gen)
        offs = np.concatenate([[0], np.cumsum(rows)[:-1]])
        emb = lambda: npy(sh.emb.weight[:, :D])
        lin = lambda: npy(sh.emb.lin_view())
        e0, l0 = emb(), lin()
        tables = [e0[o:o + r] for o, r in zip(offs, rows)]
        lins = [l0[o:o + r] for o, r in zip(offs, rows)]
        bias, ws, bs = float(sh.bias), [npy(w) for w in sh.w], [npy(b) for b in sh.b]
        ids, labels = _batch(np.random.default_rng(4), rows, B)
        o = deepfm_step(tables, lins, bias, ws, bs, "relu", ids, labels)
        sh.step(torch.from_numpy(ids).cuda(), torch.from_numpy(labels).cuda())
        torch.cuda.synchronize()
        sh.check_overflow()
        check("loss", float(sh.loss), o["loss"])
        check("prob", npy(sh.prob), o["prob"])
        check("stack", npy(sh.stack), o["stack"])
        for i in range(len(ws)):
            for k, buf, p0, p1 in ((f"w.{i}", sh.gw[i], ws[i], sh.w[i]), (f"b.{i}", sh.gb[i], bs[i], sh.b[i])):
                e = o[k]
                check("grad buffer " + k, npy(buf), e)
                after = npy(p1)
                check("update " + k, (p0 - after) / lr, e, extra=update_slack(p0, after, lr, 1, e.terms))
        e1, l1 = emb(), lin()
        for s, (off, r) in enumerate(zip(offs, rows)):
            hits = o[f"hits.{s}"]
            for k, p0, p1, h in ((f"table.{s}", tables[s], e1[off:off + r], hits[:, None]),
                                 (f"lin.{s}", lins[s], l1[off:off + r], hits)):
                check("update " + k, (p0 - p1) / lr, o[k], extra=update_slack(p0, p1, lr, h, o[k].terms))
        _check_bias(float(sh.bias), bias, o["bias"], lr, B, lambda k, t, e, extra: check(k, t, e, extra=extra))
    finally:
        dist.destroy_process_group()
