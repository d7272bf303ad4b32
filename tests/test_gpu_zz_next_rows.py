"""SURVEY 8(f) "next" rows on the GPU through the C-ABI, against the oracle: device id pipeline (FarmHash bucket,
vocabulary lookup: bit-exact), multi-valued slot bags (mean / sum / sqrtn, OOV pruning), mixed single- and
multi-valued collections through the fused gather, dense Adam (TF ApplyAdam arithmetic), row top-k (tf.math.top_k
order incl. ties).  (File name sorts after the hot-path suites on purpose: rows (a)-(e) run first.)"""
import numpy as np
import pytest
import torch

from oracle import farmhash_py as F
from oracle import reference_np as R
from deepfm_oracle import _cpu_deepfm_grads

pytestmark = pytest.mark.gpu


# ---- id pipeline ---------------------------------------------------------------------------------------
def test_device_hash_bucket_i64_bit_exact():
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(0)
    vals = np.concatenate([np.array([0, 1, -1, 9, 10, 6040, -2 ** 63, 2 ** 63 - 1], dtype=np.int64),
                           rng.integers(-10 ** 12, 10 ** 12, size=5000), rng.integers(0, 7000, size=5000)])
    for nb in (1, 100, 1_000_000, 2 ** 40 + 9):
        got = ops.hash_bucket_i64(torch.from_numpy(vals).cuda(), nb).cpu().numpy()
        assert got.tolist() == F.hash_bucket_py(vals.tolist(), nb)


def test_device_hash_bucket_bytes_bit_exact_all_length_branches():
    from deep_recommenders_b200 import ops
    from deep_recommenders_b200.hashing import pack_strings, hash_bucket
    rng = np.random.default_rng(1)
    lengths = list(range(0, 70)) + [127, 128, 129, 192, 193, 500]
    strings = [bytes(rng.integers(0, 256, size=n, dtype=np.uint8)) for n in lengths for _ in range(2)]
    data, offs = pack_strings(strings)
    got = ops.hash_bucket_bytes(torch.from_numpy(data.copy()).cuda(), torch.from_numpy(offs).cuda(), 1_000_003)
    assert got.cpu().tolist() == F.hash_bucket_py(strings, 1_000_003)
    assert got.cpu().tolist() == hash_bucket(strings, 1_000_003).tolist()      # host twin, same source
    empty = ops.hash_bucket_bytes(torch.zeros(1, dtype=torch.uint8, device="cuda"),
                                  torch.zeros(1, dtype=torch.int64, device="cuda"), 10)
    assert empty.numel() == 0


def test_device_vocab_lookup_bit_exact():
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.hashing import flat_ids, vocabulary_ids
    vocab = [56, 1, 18, 25, 35, 45, 50]                           # deliberately unsorted
    col = fc.categorical_column_with_vocabulary_list("age", vocab)
    rng = np.random.default_rng(2)
    vals = rng.integers(-5, 70, size=4000).astype(np.int64)
    got = flat_ids(col, torch.from_numpy(vals).cuda(), torch.device("cuda"))
    want = np.array([vocab.index(v) if v in vocab else -1 for v in vals.tolist()])
    assert np.array_equal(got.cpu().numpy(), want)
    assert np.array_equal(vocabulary_ids(col, vals.tolist()), want)


def test_device_and_host_id_paths_agree_for_hash_columns():
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.hashing import flat_ids
    col = fc.categorical_column_with_hash_bucket("user_id", 6040, dtype="int64")
    vals = np.random.default_rng(3).integers(1, 6041, size=3000).astype(np.int64)
    on_dev = flat_ids(col, torch.from_numpy(vals).cuda(), torch.device("cuda")).cpu().numpy()
    on_host = flat_ids(col, vals, torch.device("cuda")).cpu().numpy()
    assert np.array_equal(on_dev, on_host)
    assert on_dev.min() >= 0 and on_dev.max() < 6040


# ---- multi-valued slots -----------------------------------------------------------------------------------
def make_bags(B, rows, seed, max_len=6, oov_frac=0.15, empty_frac=0.2):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 1, size=B)
    lens[rng.random(B) < empty_frac] = 0
    splits = np.zeros(B + 1, dtype=np.int64)
    np.cumsum(lens, out=splits[1:])
    ids = rng.integers(0, rows, size=int(splits[-1])).astype(np.int64)
    oov = rng.random(ids.shape) < oov_frac
    ids = np.where(oov, np.where(rng.random(ids.shape) < 0.5, -1, rows + 5), ids)
    return ids, splits


@pytest.mark.parametrize("D", [1, 3, 4, 16, 20, 64, 128])
@pytest.mark.parametrize("combiner", ["mean", "sum", "sqrtn"])
def test_embed_bag_forward_and_backward(D, combiner):
    from deep_recommenders_b200 import ops
    rows, B = 37, 301
    rng = np.random.default_rng(D)
    table = rng.standard_normal((rows, D)).astype(np.float32)
    ids, splits = make_bags(B, rows, seed=D + 1)
    t = torch.from_numpy(table).cuda().requires_grad_(True)
    out = ops.EmbedBag.apply(t, torch.from_numpy(ids).cuda(), torch.from_numpy(splits).cuda(), D, combiner, None)
    ref64 = R.embedding_bag(table, ids, splits, combiner, np.float64)
    scale = R.embedding_bag(np.abs(table), ids, splits, "sum", np.float64)
    assert (np.abs(out.detach().cpu().numpy() - ref64) <= 1e-6 * scale + 1e-7).all()
    if combiner == "sum":       # same accumulation order as the sequential oracle: bit-exact
        assert np.array_equal(out.detach().cpu().numpy(), R.embedding_bag(table, ids, splits, "sum", np.float32))
    g = rng.standard_normal((B, D)).astype(np.float32)
    out.backward(torch.from_numpy(g).cuda())
    gref = R.embedding_bag_grad(rows, ids, splits, g, combiner, np.float64)
    gabs = R.embedding_bag_grad(rows, ids, splits, np.abs(g), combiner, np.float64)
    assert (np.abs(t.grad.cpu().numpy() - gref) <= 1e-5 * gabs + 1e-7).all()


def test_embed_bag_int32_ids_empty_batch_and_fused_sgd():
    from deep_recommenders_b200 import ops
    rows, B, D = 11, 40, 8
    rng = np.random.default_rng(5)
    table = rng.standard_normal((rows, D)).astype(np.float32)
    ids, splits = make_bags(B, rows, seed=6)
    t = torch.from_numpy(table).cuda().requires_grad_(True)
    out = ops.EmbedBag.apply(t, torch.from_numpy(ids.astype(np.int32)).cuda(), torch.from_numpy(splits).cuda(), D,
                             "mean", 0.5)
    assert np.allclose(out.detach().cpu().numpy(), R.embedding_bag(table, ids, splits, "mean"), rtol=1e-6, atol=1e-7)
    g = rng.standard_normal((B, D)).astype(np.float32)
    out.backward(torch.from_numpy(g).cuda())
    assert t.grad is None                                           # fused: the table itself moved
    want = table - 0.5 * R.embedding_bag_grad(rows, ids, splits, g, "mean", np.float64)
    assert np.allclose(t.detach().cpu().numpy(), want, rtol=1e-5, atol=1e-6)
    z = ops.EmbedBag.apply(t.detach(), torch.zeros(0, dtype=torch.int64, device="cuda"),
                           torch.zeros(1, dtype=torch.int64, device="cuda"), D, "mean", None)
    assert tuple(z.shape) == (0, D)


@pytest.mark.parametrize("D,layout", [(16, "fused"), (16, "split"), (32, "split")])
def test_mixed_collection_forward_backward_vs_oracle(D, layout):
    """DeepFM-style collection where slot 1 is multi-valued (the MovieLens "Genres" shape): the stack row of that
    slot is the mean of the bag, its first-order term the SUM of the bag's weights (multi-hot indicator)."""
    from deep_recommenders_b200.embedding import EmbeddingCollection
    rows, B = [13, 9, 21], 130
    S = len(rows)
    rng = np.random.default_rng(D)
    tables = [rng.standard_normal((r, D)).astype(np.float32) / 4 for r in rows]
    lins = [rng.standard_normal((r,)).astype(np.float32) / 4 for r in rows]
    ids = np.stack([rng.integers(-1, r, size=B) for r in rows], axis=1).astype(np.int64)
    bag_ids, bag_splits = make_bags(B, rows[1], seed=9)
    coll = EmbeddingCollection(rows, D, device="cuda", init="empty", layout=layout)
    with torch.no_grad():
        coll.emb_view().copy_(torch.from_numpy(np.concatenate(tables, 0)))
        coll.lin_view().copy_(torch.from_numpy(np.concatenate(lins, 0)))
        coll.bias.fill_(0.25)
    bags = {1: (torch.from_numpy(bag_ids).cuda(), torch.from_numpy(bag_splits).cuda())}
    stack, logit = coll(torch.from_numpy(ids).cuda(), want_logit=True, bags=bags)

    # oracle: the reference's composition (deepfm.py:39-45) with the ragged slot combined TF's way
    ref_stack = R.stack_embeddings(tables, ids).astype(np.float64)
    ref_stack[:, 1, :] = R.embedding_bag(tables[1], bag_ids, bag_splits, "mean", np.float64)
    ids_lin = ids.copy()
    ids_lin[:, 1] = -1
    lin = R.linear_term(lins, 0.25, ids_lin, np.float64).reshape(-1)
    lin = lin + R.embedding_bag(lins[1].reshape(-1, 1), bag_ids, bag_splits, "sum", np.float64).reshape(-1)
    ref_logit = lin + R.fm_second_order(ref_stack, np.float64).reshape(-1)
    scale = np.abs(lin) + 0.5 * ((ref_stack.sum(1) ** 2).sum(1) + (ref_stack ** 2).sum((1, 2))) + 1.0
    assert np.allclose(stack.detach().cpu().numpy(), ref_stack, rtol=1e-6, atol=1e-7)
    assert (np.abs(logit.detach().cpu().numpy() - ref_logit) <= 1e-5 * scale).all()

    # backward: torch-CPU autograd of the same composition in float64 is the checker
    g_stack = rng.standard_normal((B, S, D)).astype(np.float32)
    g_logit = rng.standard_normal((B,)).astype(np.float32)
    (stack * torch.from_numpy(g_stack).cuda()).sum().add((logit * torch.from_numpy(g_logit).cuda()).sum()).backward()
    tt = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in tables]
    tl = [torch.tensor(l, dtype=torch.float64, requires_grad=True) for l in lins]
    cols, lin_t = [], torch.zeros(B, dtype=torch.float64)
    for s in range(S):
        if s == 1:
            e = torch.zeros(B, D, dtype=torch.float64)
            rowsb, lw = [], []
            for b in range(B):
                seg = bag_ids[bag_splits[b]:bag_splits[b + 1]]
                seg = seg[(seg >= 0) & (seg < rows[1])]
                if len(seg):
                    rowsb.append(tt[1][torch.from_numpy(seg)].mean(0))
                    lw.append(tl[1][torch.from_numpy(seg)].sum())
                else:
                    rowsb.append(torch.zeros(D, dtype=torch.float64))
                    lw.append(torch.zeros((), dtype=torch.float64))
            e = torch.stack(rowsb)
            lin_t = lin_t + torch.stack(lw)
        else:
            ok = torch.from_numpy((ids[:, s] >= 0) & (ids[:, s] < rows[s]))
            idx = torch.from_numpy(np.clip(ids[:, s], 0, rows[s] - 1))
            e = tt[s][idx] * ok[:, None]
            lin_t = lin_t + tl[s][idx] * ok
        cols.append(e)
    st = torch.stack(cols, 1)
    lg = lin_t + 0.5 * ((st.sum(1) ** 2) - (st ** 2).sum(1)).sum(1)
    ((st * torch.from_numpy(g_stack).double()).sum() + (lg * torch.from_numpy(g_logit).double()).sum()).backward()
    gw_t, gl_t, gb_t = coll.grads()
    gw, gl = gw_t.cpu().numpy(), gl_t.cpu().numpy().reshape(-1)
    assert abs(float(gb_t) - float(g_logit.astype(np.float64).sum())) <= 1e-4 * (np.abs(g_logit).sum() + 1)
    ref_gw = np.concatenate([t.grad.numpy() for t in tt], 0)
    ref_gl = np.concatenate([l.grad.numpy() for l in tl], 0)
    tol_w = 1e-5 * (np.abs(ref_gw).max() + 1) * 8
    assert np.abs(gw - ref_gw).max() <= tol_w, np.abs(gw - ref_gw).max()
    assert np.abs(gl - ref_gl).max() <= 1e-5 * (np.abs(ref_gl).max() + 1) * 8


# ---- Adam ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4, 1000, 4099, 1 << 20])
def test_adam_step_matches_apply_adam(n):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(n)
    p, g = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    m, v = (rng.standard_normal(n) * 0.1).astype(np.float32), (rng.random(n) * 0.1).astype(np.float32)
    tp, tg, tm, tv = (torch.from_numpy(a.copy()).cuda() for a in (p, g, m, v))
    pn, mn, vn = p, m, v
    for t in range(1, 4):
        lr_t = float(R.adam_lr_t(0.01, t))
        ops.adam_step_(tp, tg, tm, tv, lr_t, zero_grad=False)
        pn, mn, vn = R.adam_dense(pn, g, mn, vn, lr_t, dtype=np.float64)
    assert np.allclose(tm.cpu().numpy(), mn, rtol=1e-5, atol=1e-7)
    assert np.allclose(tv.cpu().numpy(), vn, rtol=1e-5, atol=1e-9)
    assert np.allclose(tp.cpu().numpy(), pn, rtol=1e-5, atol=1e-6)
    ops.adam_step_(tp, tg, tm, tv, 0.01, zero_grad=True)
    assert float(tg.abs().max()) == 0.0


def test_adam_step_unaligned_views_use_the_scalar_path():
    from deep_recommenders_b200 import ops
    base = [torch.randn(1030, device="cuda") for _ in range(4)]
    base[3].abs_()
    p, g, m, v = (b[1:1026] for b in base)                          # 4-byte aligned only
    ref = R.adam_dense(p.cpu().numpy(), g.cpu().numpy(), m.cpu().numpy(), v.cpu().numpy(), 0.01, dtype=np.float64)
    ops.adam_step_(p, g, m, v, 0.01, zero_grad=False)
    assert np.allclose(base[0][1:1026].cpu().numpy(), ref[0], rtol=1e-5, atol=1e-6)
    assert np.allclose(base[2][1:1026].cpu().numpy(), ref[1], rtol=1e-5, atol=1e-7)


# ---- row top-k ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nq,nc,k", [(1, 1, 1), (7, 5, 5), (33, 100, 10), (64, 1000, 100), (3, 4097, 17)])
def test_topk_rows_matches_tf_top_k_order(nq, nc, k):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(nq + nc)
    s = rng.standard_normal((nq, nc)).astype(np.float32)
    s[:, ::3] = np.round(s[:, ::3])                                 # plenty of exact ties
    vals, idx = ops.topk_rows(torch.from_numpy(s).cuda(), k)
    rv, ri = R.top_k(s, k)
    assert np.array_equal(idx.cpu().numpy(), ri)
    assert np.array_equal(vals.cpu().numpy(), rv)


def test_topk_rows_rejects_k_larger_than_row():
    from deep_recommenders_b200 import ops
    with pytest.raises(ValueError, match="at least k columns"):
        ops.topk_rows(torch.zeros(2, 3, device="cuda"), 4)


# ---- Adam inside the train step (SURVEY 8f #1) ------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["adam", "lazy_adam", "adam_rows"])
@pytest.mark.parametrize("D", [16, 32])                   # fused 128-B rows / split layout
@pytest.mark.parametrize("use_graph", [False, True])
def test_train_step_adam_matches_apply_adam_oracle(optimizer, D, use_graph):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, B, lr = [50, 7, 30], 96, 0.01
    S = len(rows)
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=[16, 8], seed=5, device="cuda")
    coll = model.embeddings
    with torch.no_grad():
        coll.lin_view().normal_(0, 0.1)
    tr = DeepFMTrainStep(model, batch_size=B, lr=lr, use_graph=use_graph, optimizer=optimizer)
    snap = [p.detach().clone() for p in (coll.weight, tr.flat, coll.bias)] + ([coll.linear.detach().clone()] if coll.linear is not None else [])
    if use_graph:
        tr.capture()                  # must be side-effect free (round-1 advisor finding): parameters, Adam clock, m, v
        assert all(torch.equal(a, b) for a, b in zip(snap, (coll.weight, tr.flat, coll.bias) + ((coll.linear,) if coll.linear is not None else ())))
        if optimizer != "sgd":
            for t in (tr.m_arena, tr.v_arena, tr.g_arena, tr.m_flat, tr.v_flat, tr.m_bias, tr.v_bias, tr.g_bias,
                      tr.m_lin, tr.v_lin, tr.g_lin, tr.stamp, tr.state, tr.clock.step):
                assert t is None or not bool(t.any()), "capture() left optimizer state behind"
    tables = [coll.table(s).detach().cpu().numpy().astype(np.float64) for s in range(S)]
    lins = [coll.linear_of(s).detach().cpu().numpy().astype(np.float64) for s in range(S)]
    bias = float(coll.bias.detach())
    ws = [w.detach().cpu().numpy().astype(np.float64) for w in tr.w]
    bs = [b.detach().cpu().numpy().astype(np.float64) for b in tr.b]
    state = lambda xs: ([np.zeros_like(x) for x in xs], [np.zeros_like(x) for x in xs])
    (mt, vt), (ml, vl), (mw, vw), (mb, vb) = state(tables), state(lins), state(ws), state(bs)
    mbias = vbias = np.zeros(1)
    rng = np.random.default_rng(11)
    for t in range(1, 4):
        ids = np.stack([rng.integers(-1, r + 1, size=B) for r in rows], axis=1).astype(np.int64)
        ids[: B // 3] = ids[0]                                    # heavy duplicates
        labels = rng.integers(0, 2, size=B).astype(np.float32)
        loss_gpu = float(tr.step(torch.from_numpy(ids).cuda(), torch.from_numpy(labels).cuda()).item())
        loss, gt, gl, gb, gw, gbi = _cpu_deepfm_grads(tables, lins, bias, ws, bs, ids, labels)
        assert abs(loss_gpu - loss) <= (1e-5 if t == 1 else 2e-4) * abs(loss) + 1e-6
        lr_t = R.adam_lr_t(lr, t)
        for s in range(S):
            if optimizer == "adam":
                tables[s], mt[s], vt[s] = R.adam_dense(tables[s], gt[s], mt[s], vt[s], lr_t, dtype=np.float64)
                lins[s], ml[s], vl[s] = R.adam_dense(lins[s], gl[s], ml[s], vl[s], lr_t, dtype=np.float64)
            else:
                tables[s], mt[s], vt[s] = R.adam_rows_lazy(tables[s], gt[s], mt[s], vt[s], ids[:, s], lr_t, dtype=np.float64)
                lins[s], ml[s], vl[s] = R.adam_rows_lazy(lins[s], gl[s], ml[s], vl[s], ids[:, s], lr_t, dtype=np.float64)
        b_, mbias, vbias = R.adam_dense(np.array([bias]), gb, mbias, vbias, lr_t, dtype=np.float64)
        bias = float(b_[0])
        for i in range(len(ws)):
            ws[i], mw[i], vw[i] = R.adam_dense(ws[i], gw[i], mw[i], vw[i], lr_t, dtype=np.float64)
            bs[i], mb[i], vb[i] = R.adam_dense(bs[i], gbi[i], mb[i], vb[i], lr_t, dtype=np.float64)
    torch.cuda.synchronize()
    assert int(tr.clock.step) == 3
    assert abs(float(tr.clock.lr_t) - R.adam_lr_t(lr, 3)) <= 1e-6 * R.adam_lr_t(lr, 3)
    # first moments are linear in the gradients: tight; parameters: Adam divides by sqrt(v) + eps, loose
    RS = coll.row_stride
    if optimizer == "adam_rows":         # fused form: one state block per row [g D | m D | v D | g_w m_w v_w count | pad]
        st = tr.state.cpu().numpy()
        m_emb = st[:, D:2 * D]
        assert np.abs(st[:, 3 * D + 1] - np.concatenate(ml, 0)).max() <= 1e-4 * np.abs(np.concatenate(ml, 0)).max() + 1e-9
        assert not st[:, :D].any() and not st[:, 3 * D].any(), "gradient accumulators must be zero between steps"
        assert not tr.state[:, 3 * D + 3].view(torch.int32).any(), "row countdowns must be zero between steps"
    else:
        m_emb = tr.m_arena.view(-1, RS)[:, :D].cpu().numpy()
    ref_m = np.concatenate(mt, 0)
    assert np.abs(m_emb - ref_m).max() <= 1e-4 * np.abs(ref_m).max() + 1e-9
    got_tables = np.concatenate([coll.table(s).detach().cpu().numpy() for s in range(S)], 0)
    got_lins = np.concatenate([coll.linear_of(s).detach().cpu().numpy() for s in range(S)], 0)
    assert np.abs(got_tables - np.concatenate(tables, 0)).max() <= 3e-2 * lr
    assert np.abs(got_lins - np.concatenate(lins, 0)).max() <= 3e-2 * lr
    assert abs(float(coll.bias) - bias) <= 3e-2 * lr
    for i in range(len(ws)):
        assert np.abs(tr.w[i].cpu().numpy() - ws[i]).max() <= 3e-2 * lr
        assert np.abs(tr.b[i].cpu().numpy() - bs[i]).max() <= 3e-2 * lr
    # the gradient arena is all-zero again after every step (both variants clear what they consumed)
    assert (tr.g_arena is None or float(tr.g_arena.abs().max()) == 0.0) and float(tr.g_bias.abs().max()) == 0.0
    # and the parameters really moved by about lr per step where a gradient flowed
    assert np.abs(got_tables - snap[0].view(-1, RS)[:, :D].cpu().numpy()).max() > 0.5 * lr


def test_lazy_adam_rows_updates_each_touched_row_exactly_once():
    """Standalone dr_lazy_adam_rows: a gradient arena with known rows, ids with many duplicates and OOV entries."""
    from deep_recommenders_b200 import ops
    rows, D, RS, B = [40, 9], 16, 32, 257
    total = sum(rows)
    rng = np.random.default_rng(3)
    p = rng.standard_normal((total, RS)).astype(np.float32)
    m = (rng.standard_normal((total, RS)) * 0.01).astype(np.float32)
    v = (rng.random((total, RS)) * 0.01).astype(np.float32)
    ids = np.stack([rng.integers(-2, r + 2, size=B) for r in rows], axis=1).astype(np.int64)
    ids[:100, 0] = 3
    offs = np.array([0, rows[0]], dtype=np.int64)
    touched = np.unique(np.concatenate([offs[s] + ids[:, s][(ids[:, s] >= 0) & (ids[:, s] < rows[s])] for s in range(2)]))
    g = np.zeros((total, RS), dtype=np.float32)
    g[touched, :D + 1] = rng.standard_normal((touched.size, D + 1)).astype(np.float32)
    tp, tg, tm, tv = (torch.from_numpy(a.copy()).cuda() for a in (p, g, m, v))
    stamp = torch.zeros(total, dtype=torch.int32, device="cuda")
    clock = ops.AdamClock(0.01, device="cuda")
    clock.advance()
    ops.lazy_adam_rows_(torch.from_numpy(ids).cuda(), torch.tensor(rows, device="cuda"), torch.from_numpy(offs).cuda(),
                        D, RS, 1, tp, tg, tm, tv, stamp, clock)
    torch.cuda.synchronize()
    lr_t = R.adam_lr_t(0.01, 1)
    rp, rm, rv = R.adam_rows_lazy(p[:, :D + 1], g[:, :D + 1], m[:, :D + 1], v[:, :D + 1], touched, lr_t, dtype=np.float64)
    assert np.allclose(tp.cpu().numpy()[:, :D + 1], rp, rtol=1e-5, atol=1e-6)
    assert np.allclose(tm.cpu().numpy()[:, :D + 1], rm, rtol=1e-5, atol=1e-8)
    assert np.allclose(tv.cpu().numpy()[:, :D + 1], rv, rtol=1e-5, atol=1e-9)
    assert np.array_equal(tp.cpu().numpy()[:, D + 1:], p[:, D + 1:])          # padding untouched
    untouched = np.setdiff1d(np.arange(total), touched)
    assert np.array_equal(tp.cpu().numpy()[untouched], p[untouched])
    assert float(tg.abs().max()) == 0.0
    assert np.array_equal(stamp.cpu().numpy() == 1, np.isin(np.arange(total), touched))


# ---- top-k retrieval and the FactorizedTopK metric (SURVEY 8f #3) ------------------------------------------------
@pytest.fixture
def topk_variant():
    from deep_recommenders_b200 import _lib
    yield lambda v: _lib.tune("topk_variant", v)
    _lib.tune("topk_variant", 0)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("nq,nc,k", [(5, 40, 1), (9, 33, 33), (17, 2000, 50), (3, 70000, 128), (2, 5000, 1000)])
def test_topk_variants_agree_with_oracle(topk_variant, variant, nq, nc, k):
    from deep_recommenders_b200 import ops
    if variant == 1 and k * nc > 10 ** 7:
        pytest.skip("k-pass variant: quadratic, covered at smaller sizes")
    topk_variant(variant)
    rng = np.random.default_rng(nc + k)
    s = rng.standard_normal((nq, nc)).astype(np.float32)
    s[:, ::2] = np.round(s[:, ::2] * 2) / 2                        # exact ties across the row
    s[0, :] = np.sort(s[0, :])                                      # ascending: every column is an insertion
    s[-1, :] = 1.0                                                  # one value: index order decides
    vals, idx = ops.topk_rows(torch.from_numpy(s).cuda(), k)
    rv, ri = R.top_k(s, k)
    assert np.array_equal(idx.cpu().numpy(), ri)
    assert np.array_equal(vals.cpu().numpy(), rv)


def test_take_long_axis_kat():                                     # reference tests/keras/test_factorized_top_k.py:17-23
    from deep_recommenders.keras.models.retrieval import factorized_top_k
    arr = torch.tensor([[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]], device="cuda")
    indices = torch.tensor([[0, 1], [2, 1]], device="cuda")
    out = factorized_top_k._take_long_axis(arr, indices)
    assert torch.equal(out.cpu(), torch.tensor([[0.1, 0.2], [0.6, 0.5]]))


def test_exclude_kat():                                            # reference tests/keras/test_factorized_top_k.py:25-34
    from deep_recommenders.keras.models.retrieval import factorized_top_k
    scores = torch.tensor([[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]], device="cuda")
    identifiers = torch.tensor([[0, 1, 2], [3, 4, 5]], device="cuda")
    exclude = torch.tensor([[1, 2], [3, 5]], device="cuda")
    x, y = factorized_top_k._exclude(scores, identifiers, exclude, 1)
    assert torch.equal(x.cpu(), torch.tensor([[0.1], [0.5]])) and y.cpu().tolist() == [[0], [4]]


@pytest.mark.parametrize("layer", ["streaming", "brute_force", "brute_force_blocked", None])
def test_factorized_topk_metrics(layer, monkeypatch):              # reference tests/keras/test_factorized_top_k.py:86-130
    from deep_recommenders.keras.models.retrieval import FactorizedTopK, factorized_top_k
    rng = np.random.RandomState(42)
    num_candidates, num_queries, dim = 100, 10, 4
    candidates = rng.normal(size=(num_candidates, dim)).astype(np.float32)
    queries = rng.normal(size=(num_queries, dim)).astype(np.float32)
    true_candidates = rng.normal(size=(num_queries, dim)).astype(np.float32)
    positive = (queries * true_candidates).sum(axis=1, keepdims=True)
    all_scores = np.concatenate([positive, queries @ candidates.T], axis=1)
    ks = [1, 5, 10, 50]
    batches = [torch.from_numpy(candidates[i:i + 32]).cuda() for i in range(0, num_candidates, 32)]   # .batch(32)
    if layer == "streaming":
        cand = factorized_top_k.Streaming().index(batches)
    elif layer == "brute_force":
        cand = factorized_top_k.BruteForce().index(batches)
    elif layer == "brute_force_blocked":
        monkeypatch.setattr(factorized_top_k, "_SCORE_BLOCK_BYTES", 4 * num_queries * 55)   # blocks of 55 candidates
        cand = factorized_top_k.BruteForce().index(torch.from_numpy(candidates).cuda())
    else:
        cand = batches                                              # a raw dataset -> Streaming(k) inside the metric
    metric = FactorizedTopK(candidates=cand,
                            metrics=[factorized_top_k.TopKCategoricalAccuracy(k=x, name=f"top_{x}_categorical_accuracy")
                                     for x in ks], k=max(ks))
    metric.update_state(query_embeddings=torch.from_numpy(queries).cuda(),
                        true_candidate_embeddings=torch.from_numpy(true_candidates).cuda())
    for k, value in zip(ks, metric.result()):
        in_top_k = ((all_scores > all_scores[:, :1]).sum(axis=1) < k)
        assert value == pytest.approx(in_top_k.mean())


@pytest.mark.parametrize("ident_dtype", [None, torch.int32, torch.int64, torch.float32, torch.float64])
def test_streaming_and_brute_force_retrieve_the_oracles_candidates(ident_dtype):
    from deep_recommenders.keras.models.retrieval import factorized_top_k
    rng = np.random.default_rng(5)
    nc, nq, dim, k = 1000, 37, 8, 10
    cands = rng.standard_normal((nc, dim)).astype(np.float32)
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    names = None if ident_dtype is None else (torch.arange(nc) * 3 + 7).to(ident_dtype)
    ref_names = np.arange(nc) if names is None else names.numpy()
    rs, ri = R.brute_force_topk(q, cands, ref_names, k, np.float64)
    batches = [torch.from_numpy(cands[i:i + 96]).cuda() for i in range(0, nc, 96)]         # last batch has 40 rows
    ident_batches = None if names is None else [names[i:i + 96] for i in range(0, nc, 96)]
    tq = torch.from_numpy(q).cuda()
    for index in (factorized_top_k.Streaming(k=k).index(batches, ident_batches),
                  factorized_top_k.BruteForce(k=k).index(torch.from_numpy(cands).cuda(), names)):
        s, i = index(tq)
        assert np.array_equal(i.cpu().numpy(), ri)
        assert np.allclose(s.cpu().numpy(), rs, rtol=1e-5, atol=1e-5)
        s2, i2 = index(tq, k=3)
        assert np.array_equal(i2.cpu().numpy(), ri[:, :3])


def test_query_with_exclusions_and_error_paths():
    from deep_recommenders.keras.models.retrieval import factorized_top_k
    rng = np.random.default_rng(6)
    cands = rng.standard_normal((200, 8)).astype(np.float32)
    q = rng.standard_normal((11, 8)).astype(np.float32)
    bf = factorized_top_k.BruteForce(k=5).index(torch.from_numpy(cands).cuda())
    s, i = bf(torch.from_numpy(q).cuda())
    excl = i[:, [0, 2]].to(torch.int64).contiguous()                 # ban the 1st and 3rd hit of every query
    s2, i2 = bf.query_with_exclusions(torch.from_numpy(q).cuda(), excl, k=5)
    full_s, full_i = R.brute_force_topk(q, cands, None, 7, np.float64)
    xs, xi = R.exclude(full_s.astype(np.float32), full_i, excl.cpu().numpy(), 7)
    assert np.array_equal(i2.cpu().numpy(), xi)
    got, ban = i2.cpu().numpy(), excl.cpu().numpy()
    assert not any(np.isin(got[r, :5], ban[r]).any() for r in range(got.shape[0]))     # per query
    with pytest.raises(ValueError, match="index"):
        factorized_top_k.BruteForce()(torch.from_numpy(q).cuda())
    with pytest.raises(ValueError, match="ndim should be 2"):
        factorized_top_k.BruteForce().index(torch.zeros(4, device="cuda"))
    small = [torch.from_numpy(cands[:4]).cuda()]
    with pytest.raises(ValueError, match="candidate batch too small"):
        factorized_top_k.Streaming(k=10, handle_incomplete_batches=False).index(small)(torch.from_numpy(q).cuda())
    with pytest.raises(NotImplementedError):
        factorized_top_k.Faiss(k=10)


# ---- the real input path: TFRecord file -> dataset classes -> columns -> FM (SURVEY 8f #4, BASELINE config C1) ------
def test_c1_tfrecord_pipeline_matches_oracle(tmp_path):
    import importlib.util
    import pathlib
    spec = importlib.util.spec_from_file_location(
        "c1_tfrecords_example", pathlib.Path(__file__).resolve().parent.parent / "examples" / "train_fm_on_movielens_tfrecords.py")
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    from deep_recommenders.datasets.movielens import MovielensRanking, serialize_tfrecords
    from deep_recommenders.estimator.models.feature_interaction import FM
    d = ex.write_synthetic_ml1m(str(tmp_path / "ml-1m"), n_users=80, n_movies=60, n_ratings=700, seed=3)
    rec = str(tmp_path / "movielens.tfrecords")
    serialize_tfrecords(rec, datadir=d, seed=0)
    ml = MovielensRanking(epochs=2, batch_size=256, filename=rec)
    for fix in (False, True):           # the reference's always-OOV genre slot, and the genre vocabulary proper
        ind, emb = ex.build_columns(ml, fix_genre_vocab=fix)
        model = FM(ind, emb, seed=1, device="cuda")
        coll = model.collection
        with torch.no_grad():
            coll.lin_view().normal_(0, 0.1)
            coll.bias.fill_(-0.2)
        feats, labels = next(iter(ml.input_fn()))
        logits = model(feats)
        assert logits.shape == (256, 1) and labels.shape == (256, 1)
        # oracle ids from the raw strings with the Python FarmHash restatement and list.index
        uid, mid = feats["user_id"].tolist(), feats["movie_id"].tolist()
        gender = [s.decode() for s in feats["user_gender"].tolist()]
        ids = np.stack([
            np.asarray(F.hash_bucket_py(uid, ml.num_users)),
            np.asarray([ml.gender_vocab.index(g) for g in gender]),
            np.asarray([ml.age_vocab.index(int(a)) for a in feats["user_age"]]),
            np.asarray([ml.occupation_vocab.index(int(o)) for o in feats["user_occupation"]]),
            np.asarray(F.hash_bucket_py(mid, ml.num_movies)),
            np.full(256, -1),
        ], axis=1).astype(np.int64)
        S = 6
        tables = [coll.table(s).detach().cpu().numpy() for s in range(S)]
        lins = [coll.linear_of(s).detach().cpu().numpy() for s in range(S)]
        g = feats["movie_genres"]
        gvocab = ml.genres_vocab if fix else ml.gender_vocab
        gid = np.asarray([gvocab.index(s.decode()) if s.decode() in gvocab else -1 for s in g.values.tolist()])
        stack = R.stack_embeddings(tables, ids).astype(np.float64)
        stack[:, 5, :] = R.embedding_bag(tables[5], gid, g.row_splits, "mean", np.float64)
        lin = R.linear_term(lins, float(coll.bias), ids, np.float64).reshape(-1)
        lin = lin + R.embedding_bag(lins[5].reshape(-1, 1), gid, g.row_splits, "sum", np.float64).reshape(-1)
        ref = lin + R.fm_second_order(stack, np.float64).reshape(-1)
        assert np.allclose(logits.detach().cpu().numpy().reshape(-1), ref, rtol=1e-5, atol=2e-5)
        if not fix:
            assert float(np.abs(stack[:, 5]).max()) == 0.0
        else:
            assert float(np.abs(stack[:, 5]).max()) > 0.0
        opt = torch.optim.Adam(model.parameters(), lr=0.01)
        y = torch.from_numpy(labels).cuda()
        first = None
        for _ in range(10):
            loss = torch.nn.functional.binary_cross_entropy_with_logits(model(feats), y)
            opt.zero_grad()
            loss.backward()
            opt.step()
            first = first if first is not None else float(loss)
        assert float(loss) < first


# ---- row-sharded wide rows (BASELINE configs C3-C5: D = 32 ... 128), world 1 ---------------------------------------
@pytest.mark.parametrize("D", [32, 128])
def test_world1_sharded_wide_rows_equal_single_gpu_step(D):
    """The p2p sharded kernels with rows of exactly D floats and the first-order weights trailing the shard
    (lin_offset addressing) against the single-GPU split-layout step; world 2 / 8 runs are the bench's job."""
    import os
    import socket
    import torch.distributed as dist
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    from deep_recommenders_b200.training import DeepFMTrainStep
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        rows, B = [300, 7, 50, 1000, 21], 384
        cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
        sh = ShardedDeepFMTrainStep(cols, D, [32, 8], batch_size=B, lr=0.05, seed=3, device="cuda", exchange="p2p")
        assert sh.emb.vdim == D and sh.emb.flags == 0 and sh.emb.lin_offset == sum(rows) * D
        model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                       dnn_units_size=[32, 8], seed=3, device="cuda", sparse_lr=0.05)
        ref = DeepFMTrainStep(model, batch_size=B, lr=0.05, use_graph=False)
        with torch.no_grad():
            sh.emb.lin_view().normal_(0, 0.1)
            model.embeddings.emb_view().copy_(sh.emb.weight[:, :D])
            model.embeddings.lin_view().copy_(sh.emb.lin_view())
            for i in range(len(ref.layers)):
                ref.w[i].copy_(sh.w[i])
                ref.b[i].copy_(sh.b[i])
        gen = torch.Generator(device="cuda").manual_seed(0)
        ids = torch.stack([torch.randint(-1, r + 1, (B,), device="cuda", generator=gen) for r in rows], dim=1)
        lab = torch.randint(0, 2, (B,), device="cuda", generator=gen).float()
        for it in range(3):
            l_sh = float(sh.step(ids, lab).item())
            l_ref = float(ref.step(ids, lab).item())
            assert abs(l_sh - l_ref) <= 1e-5 * abs(l_ref) + 1e-6
            if it == 0:
                assert torch.equal(sh.stack, ref.stack)                   # gathered rows bit-exact
                assert torch.allclose(sh.fm_logit, ref.fm_logit, rtol=1e-5, atol=1e-5)
            else:
                assert torch.allclose(sh.stack, ref.stack, rtol=1e-5, atol=1e-6)
        assert torch.allclose(sh.emb.weight[:, :D], model.embeddings.emb_view(), rtol=1e-5, atol=1e-6)
        assert torch.allclose(sh.emb.lin_view(), model.embeddings.lin_view(), rtol=1e-5, atol=1e-6)
        assert torch.allclose(sh.bias, model.embeddings.bias, rtol=1e-5, atol=1e-6)
    finally:
        dist.destroy_process_group()


# ---- scheduling variants of the headline forward kernel: identical results required -------------------------------
@pytest.fixture
def embed_knobs():
    from deep_recommenders_b200 import _lib

    def set_(**kw):
        for k, v in kw.items():
            _lib.tune(k, v)
    yield set_
    for k in ("embed_fwd_minblocks", "embed_fwd_unroll", "embed_ctas_per_sm"):
        _lib.tune(k, 0)
    _lib.tune("embed_fwd_linx", 1)          # the library default


@pytest.mark.parametrize("linx", [0, 1])
@pytest.mark.parametrize("minb", [0, 3, 4])
@pytest.mark.parametrize("unroll", [8, 13])
@pytest.mark.parametrize("B,rows,D", [(257, [50, 60, 70, 2, 7, 21], 16), (1000, [1000] * 26, 16), (99, [64] * 4, 12),
                                      (33, [19] * 2, 20), (65, [31] * 3, 28), (40, [9] * 5, 8), (7, [5] * 2, 4)])
def test_forward_variants_bit_identical_to_default(embed_knobs, linx, minb, unroll, B, rows, D):
    import importlib.util
    import pathlib
    spec = importlib.util.spec_from_file_location("t_embed", pathlib.Path(__file__).resolve().parent / "test_gpu_embed.py")
    te = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(te)
    tables, lins, bias, ids = te.make_problem(B, rows, D, seed=B + D, oov_frac=0.1)
    coll = te.to_collection(tables, lins, bias, layout="fused")
    idt = torch.from_numpy(ids).cuda()
    with torch.no_grad():
        embed_knobs(embed_fwd_linx=0)                       # the round-1 mapping (lin lane inside an 8-lane group)
        stack0, logit0 = coll(idt)
        embed_knobs(embed_fwd_minblocks=minb, embed_fwd_linx=linx, embed_fwd_unroll=unroll)
        stack1, logit1 = coll(idt)
        stack_only, _ = coll(idt, want_logit=False)
    torch.cuda.synchronize()
    assert torch.equal(stack0, stack1) and torch.equal(logit0, logit1) and torch.equal(stack0, stack_only)
    ref_stack = R.stack_embeddings(tables, ids)
    assert np.array_equal(stack1.cpu().numpy().view(np.uint32), ref_stack.view(np.uint32))
    ref_logit, _ = R.fm_logit(tables, lins, bias, ids, np.float64)
    err = np.abs(logit1.cpu().numpy().astype(np.float64) - ref_logit.reshape(-1))
    assert (err <= 1e-5 * te.logit_scale(tables, lins, bias, ids) + 1e-6).all()


@pytest.mark.parametrize("linx", [0, 1])
@pytest.mark.parametrize("S", [120, 400])
def test_forward_many_slots_needs_opt_in_shared_memory(embed_knobs, linx, S):
    """Per-warp id staging grows with S: beyond 48 KB of dynamic shared memory the launch must opt in (both mappings)."""
    import importlib.util
    import pathlib
    spec = importlib.util.spec_from_file_location("t_embed", pathlib.Path(__file__).resolve().parent / "test_gpu_embed.py")
    te = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(te)
    B, D = 333, 16
    tables, lins, bias, ids = te.make_problem(B, [37] * S, D, seed=S, oov_frac=0.05)
    coll = te.to_collection(tables, lins, bias, layout="fused")
    embed_knobs(embed_fwd_linx=linx)
    with torch.no_grad():
        stack, logit = coll(torch.from_numpy(ids).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(stack.cpu().numpy().view(np.uint32), R.stack_embeddings(tables, ids).view(np.uint32))
    ref_logit, _ = R.fm_logit(tables, lins, bias, ids, np.float64)
    err = np.abs(logit.cpu().numpy().astype(np.float64) - ref_logit.reshape(-1))
    assert (err <= 1e-5 * te.logit_scale(tables, lins, bias, ids) + 1e-6).all()


def test_world1_sharded_forward_linx_mapping_equals_default(embed_knobs):
    """Knob embed_fwd_linx_shard (off by default until measured at N > 1): the LINX lane mapping in the peer-memory
    forward must give the same bits as the default sharded forward."""
    import os
    import socket
    import torch.distributed as dist
    from deep_recommenders_b200 import _lib, feature_column as fc
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        rows, B, D = [300, 7, 50, 1000, 21], 384, 16
        cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
        sh = ShardedDeepFMTrainStep(cols, D, [32, 8], batch_size=B, lr=0.0, seed=3, device="cuda", exchange="p2p",
                                    use_graph=False)
        with torch.no_grad():
            sh.emb.lin_view().normal_(0, 0.1)
        gen = torch.Generator(device="cuda").manual_seed(0)
        ids = torch.stack([torch.randint(-1, r + 1, (B,), device="cuda", generator=gen) for r in rows], dim=1)
        lab = torch.randint(0, 2, (B,), device="cuda", generator=gen).float()
        sh.step(ids, lab)
        torch.cuda.synchronize()
        ref = (sh.stack.clone(), sh.fm_logit.clone(), sh.sum_e.clone())
        _lib.tune("embed_fwd_linx_shard", 1)
        sh.step(ids, lab)                       # lr = 0: parameters unchanged, forward must reproduce itself
        torch.cuda.synchronize()
        assert torch.equal(sh.stack, ref[0]) and torch.equal(sh.fm_logit, ref[1]) and torch.equal(sh.sum_e, ref[2])
    finally:
        _lib.tune("embed_fwd_linx_shard", 0)
        dist.destroy_process_group()


def test_retrieval_classes_reproduce_the_reference_source_golden():
    """tests/golden/retrieval_golden.npz = the reference's own factorized_top_k.py executed under the TF stand-in
    (tests/golden/make_golden.py): identifiers must match exactly, scores to 1e-5."""
    import os
    from deep_recommenders.keras.models.retrieval import FactorizedTopK, factorized_top_k as ftk
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "retrieval_golden.npz"))
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = ftk._take_long_axis(cu(g["tla_arr"]), cu(g["tla_idx"]))
    assert np.array_equal(out.cpu().numpy(), g["tla_out"])
    for k in (5, 40, 60):
        xs, xi = ftk._exclude(cu(g["exclude_scores"]), cu(g["exclude_ident"]), cu(g["exclude_excl"]), k)
        assert np.array_equal(xi.cpu().numpy(), g[f"exclude_k{k}_ids"])
        assert np.array_equal(xs.cpu().numpy(), g[f"exclude_k{k}_scores"])
    q, c, names = cu(g["idx_queries"]), g["idx_candidates"], g["idx_names"]
    batches = [cu(c[i:i + 32]) for i in range(0, 100, 32)]
    nbatches = [torch.from_numpy(names[i:i + 32]) for i in range(0, 100, 32)]
    for tag, nb in (("noid", None), ("id", nbatches)):
        for cls, key in ((ftk.Streaming, "streaming"), (ftk.BruteForce, "brute")):
            s, i = cls(k=10).index(batches, nb)(q)
            assert np.array_equal(i.cpu().numpy(), g[f"{key}_{tag}_ids"])
            assert np.allclose(s.cpu().numpy(), g[f"{key}_{tag}_scores"], rtol=1e-5, atol=1e-6)
        s3, i3 = ftk.BruteForce(k=10).index(batches, nb)(q, k=3)
        assert np.array_equal(i3.cpu().numpy(), g[f"brute_{tag}_k3_ids"])
    bf = ftk.BruteForce(k=5).index(cu(c), torch.from_numpy(names))
    xs, xi = bf.query_with_exclusions(q, cu(g["qwe_ban"]), k=5)
    assert np.array_equal(xi.cpu().numpy(), g["qwe_ids"])
    assert np.allclose(xs.cpu().numpy(), g["qwe_scores"], rtol=1e-5, atol=1e-6)
    s, i = ftk.Streaming(k=50).index([cu(c[:32]), cu(c[32:40])])(q)
    assert np.array_equal(i.cpu().numpy(), g["streaming_small_ids"])
    with pytest.raises(ValueError) as ei:
        ftk.Streaming(k=50, handle_incomplete_batches=False).index([cu(c[:32]), cu(c[32:40])])(q)
    assert str(ei.value) == str(g["streaming_small_error"])
    ks = g["metric_ks"].tolist()
    for tag, cand in (("streaming", ftk.Streaming().index(batches)), ("brute", ftk.BruteForce().index(batches)),
                      ("dataset", batches)):
        m = FactorizedTopK(candidates=cand, metrics=[ftk.TopKCategoricalAccuracy(k=x) for x in ks], k=max(ks))
        m.update_state(q, cu(g["idx_true"]))
        assert np.allclose(m.result(), g[f"metric_{tag}"], rtol=1e-6)


import os as _os

@pytest.mark.parametrize("temperature,accidental", [(None, False), (0.5, True)])
def test_world1_sharded_two_tower_step_matches_oracle(temperature, accidental):
    import socket
    import torch.distributed as dist
    from deep_recommenders_b200.sharded_two_tower import ShardedTwoTowerTrainStep
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    _os.environ["MASTER_ADDR"], _os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        U, I, D, b, lr = 300, 500, 64, 256, 0.05
        st = ShardedTwoTowerTrainStep(U, I, D, b, lr=lr, temperature=temperature, remove_accidental_hits=accidental,
                                      seed=2, device="cuda")
        arena = st.weight.detach().cpu().numpy().astype(np.float64)          # world 1: local index == global row
        rng = np.random.default_rng(0)
        for it in range(3):
            uid = rng.integers(0, U, b)
            iid = rng.integers(0, I, b)
            iid[: b // 8] = iid[0]                                           # accidental hits / duplicate rows
            loss = float(st.step(torch.from_numpy(uid).cuda(), torch.from_numpy(iid).cuda()).item())
            Q, C = arena[uid], arena[U + iid]
            ids = iid if accidental else None
            ref_loss, _, _ = R.retrieval_loss(Q, C, candidate_ids=ids, temperature=temperature, dtype=np.float64)
            gq, gc = R.retrieval_grad(Q, C, candidate_ids=ids, temperature=temperature, dtype=np.float64)
            assert abs(loss - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)) + 1e-4
            if it == 0:
                assert np.array_equal(st.q.cpu().numpy(), Q.astype(np.float32))   # gathered rows bit-exact
            np.add.at(arena, uid, -lr * gq)
            np.add.at(arena, U + iid, -lr * gc)
            got = st.weight.detach().cpu().numpy()
            assert np.abs(got - arena).max() <= 1e-5 * (np.abs(arena).max() + lr * (np.abs(gq).max() + np.abs(gc).max()) * b / 8)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("B,rows,D", [(257, [50, 60, 70, 2, 7, 21], 16), (1000, [1000] * 26, 16), (99, [64] * 4, 12),
                                      (65, [31] * 3, 28), (40, [9] * 5, 8)])
def test_backward_linx_mapping_matches_default(B, rows, D):
    """Knob embed_bwd_linx: same gradients as the default slot-parallel backward (up to the order of the atomics)."""
    import importlib.util
    import pathlib
    from deep_recommenders_b200 import _lib
    spec = importlib.util.spec_from_file_location("t_embed", pathlib.Path(__file__).resolve().parent / "test_gpu_embed.py")
    te = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(te)
    tables, lins, bias, ids = te.make_problem(B, rows, D, seed=B + D, oov_frac=0.1)
    idt = torch.from_numpy(ids).cuda()
    S = len(rows)
    gs = torch.randn(B, S, D, device="cuda")
    gl = torch.randn(B, device="cuda")
    grads = []
    try:
        for linx in (0, 1):
            _lib.tune("embed_bwd_linx", linx)
            coll = te.to_collection(tables, lins, bias, layout="fused")
            stack, logit = coll(idt)
            ((stack * gs).sum() + (logit * gl).sum()).backward()
            grads.append([g.detach().clone() for g in coll.grads()])
    finally:
        _lib.tune("embed_bwd_linx", 0)
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(a.abs().max()) + 1e-7)


@pytest.mark.parametrize("D", [16, 128])
def test_world1_sharded_trainer_checkpoint_round_trip(tmp_path, D):
    import socket
    import torch.distributed as dist
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    _os.environ["MASTER_ADDR"], _os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    try:
        rows, B = [300, 7, 50], 128
        cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
        mk = lambda seed: ShardedDeepFMTrainStep(cols, D, [32, 8], batch_size=B, lr=0.05, seed=seed, device="cuda",
                                                 exchange="p2p", use_graph=False)
        a = mk(3)
        with torch.no_grad():
            a.emb.lin_view().normal_(0, 0.1)
        ids = torch.stack([torch.randint(0, r, (B,), device="cuda") for r in rows], dim=1)
        lab = torch.randint(0, 2, (B,), device="cuda").float()
        a.step(ids, lab)
        prefix = str(tmp_path / "ckpt")
        a.save(prefix)
        b = mk(99)                                     # different initialisation, then restored
        b.load(prefix)
        assert torch.equal(a.emb.weight, b.emb.weight) and torch.equal(a.flat, b.flat)
        assert torch.equal(a.emb.lin_view(), b.emb.lin_view())
        assert a.get_config() == b.get_config()
        la, lb = float(a.step(ids, lab).item()), float(b.step(ids, lab).item())
        assert abs(la - lb) <= 1e-6 * abs(la)       # same state, same batch; the loss is summed with float atomics (order)
        with pytest.raises(ValueError, match="was written for"):
            ShardedDeepFMTrainStep(cols, D, [16, 8], batch_size=B, lr=0.05, seed=1, device="cuda", exchange="p2p",
                                   use_graph=False).load(prefix)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("D", [16, 32])                   # fused 128-B rows / split layout
@pytest.mark.parametrize("use_graph", [False, True])
def test_train_step_adam_rows_tf_equals_dense_tf_adam(D, use_graph):
    """optimizer="adam_rows_tf": the row-sparse Adam fused into the backward, with per-row step stamps and replay of the
    steps a row sat out, must give what tf.keras Adam's DENSE update gives (examples/train_deepfm_on_movielens_keras.py:44):
    the float64 ApplyAdam oracle applied to every row every step.  Sparse batches over 8 steps: most rows are untouched
    in most steps, some are touched twice with several steps in between, some never again (flushed at the end)."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, B, lr = [300, 7, 120], 16, 0.01
    S = len(rows)
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=[16, 8], seed=5, device="cuda")
    coll = model.embeddings
    with torch.no_grad():
        coll.lin_view().normal_(0, 0.1)
    tr = DeepFMTrainStep(model, batch_size=B, lr=lr, use_graph=use_graph, optimizer="adam_rows_tf")
    if use_graph:
        tr.capture()
    tables = [coll.table(s).detach().cpu().numpy().astype(np.float64) for s in range(S)]
    lins = [coll.linear_of(s).detach().cpu().numpy().astype(np.float64) for s in range(S)]
    bias = float(coll.bias.detach())
    ws = [w.detach().cpu().numpy().astype(np.float64) for w in tr.w]
    bs = [b.detach().cpu().numpy().astype(np.float64) for b in tr.b]
    state = lambda xs: ([np.zeros_like(x) for x in xs], [np.zeros_like(x) for x in xs])
    (mt, vt), (ml, vl), (mw, vw), (mb, vb) = state(tables), state(lins), state(ws), state(bs)
    lazy_t = [t.copy() for t in tables]                       # what the LAZY semantics would give (must differ: see below)
    lazy_m, lazy_v = [np.zeros_like(t) for t in tables], [np.zeros_like(t) for t in tables]
    mbias = vbias = np.zeros(1)
    rng = np.random.default_rng(23)
    for t in range(1, 9):
        ids = np.stack([rng.integers(-1, r + 1, size=B) for r in rows], axis=1).astype(np.int64)
        ids[:4] = [5, 3, 7]                                   # duplicates; row 5 / 7 of the big tables touched EVERY step
        if t in (1, 6):
            ids[4:8] = [11, 1, 13]                            # rows 11 / 13: touched at steps 1 and 6 only (gap of 4 steps)
        labels = rng.integers(0, 2, size=B).astype(np.float32)
        tr.step(torch.from_numpy(ids).cuda(), torch.from_numpy(labels).cuda())
        loss, gt, gl, gb, gw, gbi = _cpu_deepfm_grads(tables, lins, bias, ws, bs, ids, labels)
        lr_t = R.adam_lr_t(lr, t)
        for s in range(S):
            lazy_t[s], lazy_m[s], lazy_v[s] = R.adam_rows_lazy(lazy_t[s], gt[s], lazy_m[s], lazy_v[s], ids[:, s], lr_t, dtype=np.float64)
            tables[s], mt[s], vt[s] = R.adam_dense(tables[s], gt[s], mt[s], vt[s], lr_t, dtype=np.float64)   # TF: dense
            lins[s], ml[s], vl[s] = R.adam_dense(lins[s], gl[s], ml[s], vl[s], lr_t, dtype=np.float64)
        b_, mbias, vbias = R.adam_dense(np.array([bias]), gb, mbias, vbias, lr_t, dtype=np.float64)
        bias = float(b_[0])
        for i in range(len(ws)):
            ws[i], mw[i], vw[i] = R.adam_dense(ws[i], gw[i], mw[i], vw[i], lr_t, dtype=np.float64)
            bs[i], mb[i], vb[i] = R.adam_dense(bs[i], gbi[i], mb[i], vb[i], lr_t, dtype=np.float64)
    tr.flush_optimizer()                                      # rows not touched by the last steps catch up here
    torch.cuda.synchronize()
    got_tables = np.concatenate([coll.table(s).detach().cpu().numpy() for s in range(S)], 0)
    got_lins = np.concatenate([coll.linear_of(s).detach().cpu().numpy() for s in range(S)], 0)
    ref_tables, ref_lazy = np.concatenate(tables, 0), np.concatenate(lazy_t, 0)
    # the test discriminates: under lazy semantics the tables would be off by many times the tolerance
    assert np.abs(ref_lazy - ref_tables).max() > 1.0 * lr
    assert np.abs(got_tables - ref_tables).max() <= 3e-2 * lr, np.abs(got_tables - ref_tables).max() / lr
    assert np.abs(got_lins - np.concatenate(lins, 0)).max() <= 3e-2 * lr
    # moments too (linear in the gradients: tight), read from the per-row state blocks after the flush
    st = tr.state.cpu().numpy()
    ref_m = np.concatenate(mt, 0)
    assert np.abs(st[:, D:2 * D] - ref_m).max() <= 1e-4 * np.abs(ref_m).max() + 1e-9
    ref_v = np.concatenate(vt, 0)
    assert np.abs(st[:, 2 * D:3 * D] - ref_v).max() <= 1e-4 * np.abs(ref_v).max() + 1e-12
    assert (st[:, 3 * D + 4].view(np.int32)[np.abs(ref_m).sum(1) > 0] == 8).all()      # every updated row is stamped with the last step
