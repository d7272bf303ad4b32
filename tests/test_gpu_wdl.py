"""Wide & Deep on the GPU (-m gpu): the device crossing against its host twin, the wide forward / gradient and the
row-sparse FTRL kernel against the float64 oracle (tests/wdl_oracle.py), and whole WDL train steps against it."""
import numpy as np
import pytest
import torch

import wdl_oracle as W

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def _ragged(per_ex):
    from deep_recommenders_b200.feature_column import RaggedFeature
    flat = [v for vals in per_ex for v in vals]
    return RaggedFeature(flat, np.cumsum([0] + [len(v) for v in per_ex]))


@pytest.mark.parametrize("ragged", [False, True])
def test_device_crossing_is_bit_identical_to_the_host_twin(ragged):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.hashing import cross_ids
    rng = np.random.default_rng(11)
    B = 3000
    ints = rng.integers(-3, 50, B).astype(np.int64)
    ints[:5] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, -1]
    strs = np.asarray([["", "F", "M", "Zürich", "x" * 70][k] for k in rng.integers(0, 5, B)], dtype=object)
    col = fc.crossed_column(["a", "s", "i2"], 1 << 33)
    i2 = rng.integers(0, 1 << 40, B).astype(np.int64)
    if ragged:
        per_ex = [[int(x) for x in rng.integers(-2, 9, int(rng.integers(0, 4)))] for _ in range(B)]
        host = {"a": _ragged(per_ex), "s": strs, "i2": i2}
        dev = {"a": _ragged(per_ex), "s": strs, "i2": torch.from_numpy(i2).to(DEV)}
        dev["a"].values = torch.tensor(dev["a"].values, dtype=torch.int64, device=DEV)
    else:
        host = {"a": ints, "s": strs, "i2": i2}
        dev = {"a": torch.from_numpy(ints).to(DEV), "s": strs, "i2": torch.from_numpy(i2).to(DEV)}
    h = cross_ids(col, host, DEV)
    d = cross_ids(col, dev, DEV)
    torch.cuda.synchronize()
    if ragged:
        assert torch.equal(h[1], d[1]) and torch.equal(h[0], d[0])
        assert h[0].numel() > B // 2
    else:
        assert torch.equal(h, d)
        assert (h == -1).any() and (h >= 0).any()
    # and the Python restatement on a sample of examples
    keys = [[[v] for v in ints[:50].tolist()] if not ragged else [list(x) for x in per_ex[:50]],
            [[v] for v in strs[:50].tolist()], [[int(v)] for v in i2[:50]]]
    want, want_splits = W.cross_batch(keys, 1 << 33, ragged=[ragged, False, False])
    if ragged:
        assert h[0][:int(want_splits[-1])].cpu().tolist() == want.tolist()
    else:
        per = [want[want_splits[b]:want_splits[b + 1]].tolist() for b in range(50)]
        assert h[:50].cpu().tolist() == [p[0] if p else -1 for p in per]


def test_device_crossing_with_a_host_string_key_first():
    """A host string key (multi-byte strings, copied to the device as bytes + offsets) ahead of a CUDA int key: the
    batch size comes from the string offsets, not the byte count, and the ids equal the host twin's."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.hashing import cross_ids
    s = np.asarray(["Zurich", "F", "", "hello"], dtype=object)
    i = np.asarray([3, -1, 7, 12], dtype=np.int64)
    col = fc.crossed_column(["s", "i"], 1000)
    d = cross_ids(col, {"s": s, "i": torch.from_numpy(i).to(DEV)}, DEV)
    h = cross_ids(col, {"s": s, "i": i}, DEV)
    assert d.shape == (4,) and torch.equal(d, h)
    want, splits = W.cross_batch([[[v] for v in s.tolist()], [[int(v)] for v in i]], 1000)
    assert d.cpu().tolist() == [want[splits[b]] if splits[b + 1] > splits[b] else -1 for b in range(4)]


def test_device_crossing_with_an_empty_ragged_key_and_bad_lengths():
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200 import ops
    from deep_recommenders_b200.feature_column import RaggedFeature
    from deep_recommenders_b200.hashing import cross_ids
    col = fc.crossed_column(["a", "b"], 97)
    empty = RaggedFeature(torch.zeros((0,), dtype=torch.int64, device=DEV),
                          torch.zeros((4,), dtype=torch.int64, device=DEV))
    ids, splits = cross_ids(col, {"a": empty, "b": torch.arange(3, device=DEV)}, DEV)
    assert ids.numel() == 0 and splits.cpu().tolist() == [0, 0, 0, 0]
    v = torch.arange(4, device=DEV)
    with pytest.raises(ValueError):
        ops.cross_hash([v, v[:3]], [None, None], [None, None], 4, 97, 0)
    with pytest.raises(ValueError):
        ops.cross_hash([v, v[:2]], [None, None], [torch.tensor([0, 1, 5], device=DEV), None], 2, 97, 0)


def _wide_batch(rng, B, rows, n_bags, zipf=1.2):
    """ids [B, S] with Zipf-heavy duplicates and OOV ids, plus bags for the last n_bags slots."""
    S = len(rows)
    ids = np.stack([(rng.zipf(zipf, B) - 1) % (r + 3) - 1 for r in rows], axis=1).astype(np.int64)  # -1 and >= r: OOV
    bags, per_slot = {}, []
    for s in range(S):
        if s >= S - n_bags:
            per_ex = [list((rng.zipf(zipf, int(rng.integers(0, 5))) - 1) % (rows[s] + 2) - 1) for _ in range(B)]
            bags[s] = (torch.tensor([v for p in per_ex for v in p], dtype=torch.int64, device=DEV),
                       torch.tensor(np.cumsum([0] + [len(p) for p in per_ex]), dtype=torch.int64, device=DEV))
            per_slot.append(per_ex)
        else:
            per_slot.append([[int(v)] for v in ids[:, s]])
    return torch.from_numpy(ids).to(DEV), (bags or None), per_slot


def test_wide_forward_and_gradient_match_the_oracle():
    from deep_recommenders_b200.embedding import LinearTable
    rng = np.random.default_rng(2)
    rows = [50, 7, 1000, 3, 200]
    B = 777
    t = LinearTable(rows, device=DEV)
    with torch.no_grad():
        t.state[:, 0].copy_(torch.from_numpy(rng.normal(0, 1, t.total_rows + 1)))
    ids, bags, per_slot = _wide_batch(rng, B, rows, 2)
    offs = np.cumsum([0] + rows)[:-1]
    slots = [(r, int(o), p) for r, o, p in zip(rows, offs, per_slot)]
    look = W.wide_lookups(slots, B)
    w = t.state[:, 0].detach().double().cpu().numpy()
    logit = t(ids, bags)
    want = W.wide_forward(w[:-1], w[-1], look)
    np.testing.assert_allclose(logit.detach().cpu().numpy(), want, rtol=1e-5, atol=1e-5)
    g_logit = torch.from_numpy(rng.normal(0, 1, B).astype(np.float32)).to(DEV)
    logit.backward(g_logit)
    g_rows, g_bias = W.wide_grad(t.total_rows, look, g_logit.double().cpu().numpy())
    g = t.state[:, 3].detach().double().cpu().numpy()
    np.testing.assert_allclose(g[:-1], g_rows, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(g[-1], g_bias, rtol=1e-5, atol=1e-4)
    assert t.state.grad is None


@pytest.mark.parametrize("l1,l2", [(0.05, 0.0), (0.0, 0.2)])
def test_ftrl_kernel_matches_the_dense_oracle_over_steps(l1, l2):
    """Zipf-heavy duplicates, OOV ids and multi-valued slots; after every step the whole table equals TensorFlow's
    dense ApplyFtrl in float64 and the rows no batch touched are bit-for-bit what they were."""
    from deep_recommenders_b200.embedding import LinearTable
    from deep_recommenders_b200.ops import FtrlOptimizer
    rng = np.random.default_rng(7)
    rows = [300, 11, 5000, 64]
    B, lr = 2048, 0.05
    t = LinearTable(rows, device=DEV)
    opt = FtrlOptimizer(lr, initial_accumulator_value=0.1, l1_regularization_strength=l1,
                        l2_regularization_strength=l2)
    R = t.total_rows
    ref = [np.zeros(R + 1), np.zeros(R + 1), np.full(R + 1, 0.1)]
    offs = np.cumsum([0] + rows)[:-1]
    touched = np.zeros(R + 1, dtype=bool)
    touched[R] = True
    for step in range(4):
        before = t.state.detach().clone()
        ids, bags, per_slot = _wide_batch(rng, B, rows, 1)
        look = W.wide_lookups([(r, int(o), p) for r, o, p in zip(rows, offs, per_slot)], B)
        logit = t(ids, bags)
        g_logit = torch.from_numpy(rng.normal(0, 0.5, B).astype(np.float32)).to(DEV)
        logit.backward(g_logit)
        g_rows, g_bias = W.wide_grad(R, look, g_logit.double().cpu().numpy())
        opt.apply(t)
        ref = list(W.ftrl_dense(*ref, np.append(g_rows, g_bias), lr, l1, l2))
        st = t.state.detach().double().cpu().numpy()
        step_rows = np.zeros(R + 1, dtype=bool)
        step_rows[sorted({r for rs in look for r in rs})] = True
        step_rows[R] = True
        touched |= step_rows
        for k, name in enumerate("wzn"):
            np.testing.assert_allclose(st[:, k], ref[k], rtol=2e-4, atol=2e-6, err_msg=f"step {step} {name}")
        assert (st[:, 3] == 0).all()
        # rows this batch did not touch: bitwise unchanged
        same = torch.from_numpy(~step_rows).to(DEV)
        assert torch.equal(t.state.detach()[same, :3], before[same, :3])
    assert touched[:-1].sum() < R           # some rows were never touched ...
    never = ~touched
    assert (t.state.detach()[torch.from_numpy(never).to(DEV), :2] == 0).all()   # ... and stayed at their start
    if l1 > 0:
        assert ((st[:, 0] == 0) & (st[:, 1] != 0)).any()    # L1 holds some touched weights at zero


def _adam_tf(params, clock):
    from deep_recommenders_b200 import ops
    clock.advance()
    for p, st in params:
        if p.grad is None:
            p.grad = torch.zeros_like(p)
        ops.adam_step_(p.data, p.grad, st[0], st[1], 0.0, 0.9, 0.999, 1e-8, zero_grad=True, lr_t_dev=clock.lr_t)


def wdl_train_step(model, ftrl, params, clock, features, labels):
    """One step of the example: log loss, one backward, FTRL on the wide part and TF1 Adam on the deep part."""
    p = model(features).reshape(-1)
    y = labels.reshape(-1)
    loss = torch.mean(-y * torch.log(p + 1e-7) - (1 - y) * torch.log(1 - p + 1e-7))
    loss.backward()
    ftrl.apply(model.linear)
    _adam_tf(params, clock)
    return loss, p


def _run_steps(indicator_columns, embedding_columns, units, batches):
    from deep_recommenders_b200 import ops
    from deep_recommenders.estimator.models.ranking import WDL
    from deep_recommenders_b200.hashing import wide_ids, ids_and_bags
    model = WDL(indicator_columns, embedding_columns, units, seed=3, device=DEV)
    ftrl = ops.FtrlOptimizer(0.01, l1_regularization_strength=0.5)
    params = [(p, (torch.zeros_like(p), torch.zeros_like(p))) for p in model.deep_variables()]
    clock = ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device=DEV)
    coll = model.embeddings
    state = {"w": np.zeros(model.linear.total_rows), "z": np.zeros(model.linear.total_rows),
             "n": np.full(model.linear.total_rows, 0.1), "bias_wzn": np.asarray([0.0, 0.0, 0.1]),
             "tables": [coll.table(s).detach().double().cpu().numpy() for s in range(coll.num_slots)],
             "ws": [l.kernel.detach().double().cpu().numpy() for l in model._dnn.layers],
             "bs": [l.bias.detach().double().cpu().numpy() for l in model._dnn.layers]}
    cats = [c.categorical_column for c in indicator_columns]
    offs = np.cumsum([0] + model.linear.rows_list)[:-1]
    for features, labels in batches:
        B = len(labels)
        ids, bags = wide_ids(cats, features, DEV)
        wide_slots = []
        for s, c in enumerate(cats):
            if bags and s in bags:
                fl, sp = (x.cpu().numpy() for x in bags[s])
                per = [fl[sp[b]:sp[b + 1]].tolist() for b in range(B)]
            else:
                per = [[int(v)] for v in ids[:, s].cpu().numpy()]
            wide_slots.append((c.num_buckets, int(offs[s]), per))
        dids, dbags = ids_and_bags(model._keys, model._cat, features, DEV)
        deep_ids = []
        for s in range(len(model._keys)):
            if dbags and s in dbags:
                fl, sp = (x.cpu().numpy() for x in dbags[s])
                deep_ids.append([fl[sp[b]:sp[b + 1]].tolist() for b in range(B)])
            else:
                deep_ids.append([[int(v)] for v in dids[:, s].cpu().numpy()])
        loss, p = wdl_train_step(model, ftrl, params, clock, features, torch.from_numpy(labels).to(DEV))
        ref_loss, ref_p = W.step(state, {"wide_slots": wide_slots, "deep_ids": deep_ids, "y": labels})
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref_p, rtol=1e-5, atol=1e-6)
        assert abs(float(loss.detach()) - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss))
        st = model.linear.state.detach().double().cpu().numpy()
        np.testing.assert_allclose(st[:-1, 0], state["w"], rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(st[-1, :3], state["bias_wzn"], rtol=1e-4, atol=1e-6)
        for s in range(coll.num_slots):
            np.testing.assert_allclose(coll.table(s).detach().cpu().numpy(), state["tables"][s], rtol=1e-4,
                                       atol=2e-6)
        for l, w_ref, b_ref in zip(model._dnn.layers, state["ws"], state["bs"]):
            np.testing.assert_allclose(l.kernel.detach().cpu().numpy(), w_ref, rtol=1e-4, atol=2e-6)
            np.testing.assert_allclose(l.bias.detach().cpu().numpy(), b_ref, rtol=1e-4, atol=2e-6)
    return model


def test_wdl_train_steps_match_the_oracle_small():
    from deep_recommenders_b200 import feature_column as fc
    rng = np.random.default_rng(4)
    a = fc.categorical_column_with_identity("a", 40)
    b = fc.categorical_column_with_vocabulary_list("b", ["x", "y", "z"])
    m = fc.categorical_column_with_identity("m", 9)
    ind = [fc.indicator_column(c) for c in (a, b, m)] + [fc.indicator_column(fc.crossed_column(["a", "b"], 23))]
    emb = [fc.embedding_column(c, dimension=8) for c in (a, b, m)]
    batches = []
    for _ in range(3):
        B = 64
        feats = {"a": rng.integers(-1, 45, B), "b": rng.choice(["x", "y", "z", "w"], B),
                 "m": _ragged([list(rng.integers(0, 9, int(rng.integers(0, 4)))) for _ in range(B)])}
        batches.append((feats, rng.integers(0, 2, B).astype(np.float32)))
    _run_steps(ind, emb, [16, 8], batches)


def test_wdl_train_steps_match_the_oracle_example_columns():
    import importlib.util
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("wdl_example",
                                                  os.path.join(root, "examples", "train_wdl_on_movielens_estimator.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    indicator_columns, embedding_columns = ex.build_columns()
    gen = ex.synthetic_input_fn(5, batch_size=256)
    _run_steps(indicator_columns + ex.cross_product_transformation(), embedding_columns, [64, 16],
               [next(gen) for _ in range(3)])
