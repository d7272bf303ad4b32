"""FNN on the GPU: dr_fnn_input_fwd / _bwd against the float64 oracle (tests/fnn_oracle.py) and the arena itself, and
the ranking.FNN model against the reference's own fnn.py (tests/golden/fnn_golden.npz) and against TF1 Adam steps."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import fnn_oracle as O
from test_cpu_fnn import golden_cases

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _collection(rows, D, layout, seed=0, sparse_lr=None):
    from deep_recommenders_b200.embedding import EmbeddingCollection
    coll = EmbeddingCollection(rows, D, with_linear=True, layout=layout, seed=seed, device=DEV, sparse_lr=sparse_lr)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    with torch.no_grad():
        coll.lin_view().copy_(torch.randn(coll.total_rows, device=DEV, generator=g))
    return coll


def _ids(rng, B, rows, dtype):
    """[B, S] ids with duplicates, -1 and out-of-range entries."""
    ids = np.stack([rng.integers(-1, n + 3, B) for n in rows], axis=1)
    ids[::7, 0] = -5
    return torch.from_numpy(ids.astype(np.int64)).to(DEV).to(dtype)


def _bags(rng, B, n, slot):
    """A multi-valued slot: 0..3 ids per example (empty bags, an out-of-range id, duplicates)."""
    per = [list(rng.integers(-1, n + 2, int(rng.integers(0, 4)))) for _ in range(B)]
    per[0] = []
    per[1] = [0, 0, n + 1]
    flat = torch.tensor([v for p in per for v in p], dtype=torch.int64, device=DEV)
    splits = torch.tensor(np.cumsum([0] + [len(p) for p in per]), dtype=torch.int64, device=DEV)
    return {slot: (flat, splits)}, per


def _np_state(coll):
    S = coll.num_slots
    return ([coll.table(s).detach().double().cpu().numpy() for s in range(S)],
            [coll.linear_of(s).detach().double().cpu().numpy() for s in range(S)])


def _per_slot(ids, per_bag=None, bag_slot=None):
    cols = ids.long().cpu().numpy().T
    out = [[[int(v)] for v in col] for col in cols]
    if per_bag is not None:
        out[bag_slot] = [[int(v) for v in p] for p in per_bag]
    return out


CASES = [(S, D, layout, dt) for S in (4, 5, 6, 7) for D, layout in ((16, "fused"), (32, "split"))
         for dt in (torch.int64, torch.int32)]


@pytest.mark.parametrize("S,D,layout,dtype", CASES)
def test_forward_is_an_exact_copy_of_the_arena(S, D, layout, dtype):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(S * 100 + D)
    rows = [int(rng.integers(5, 60)) for _ in range(S)]
    coll = _collection(rows, D, layout, seed=S)
    B = 301
    ids = _ids(rng, B, rows, dtype)
    bias = torch.tensor([0.375], device=DEV)
    x = ops.FnnInputFn.apply(ids, coll.weight, coll.linear, bias, coll, None)
    P, ld = ops.fnn_layout(S, D)
    assert x.shape == (B, ld) and ld % 4 == 0
    x = x.detach().cpu()
    tables, lins = _np_state(coll)
    emb, lin = coll.emb_view().detach().cpu(), coll.lin_view().detach().cpu()
    want = torch.zeros((B, ld))
    want[:, 0] = 0.375
    idn = ids.long().cpu()
    offs = coll._offsets.cpu()
    for s in range(S):
        ok = (idn[:, s] >= 0) & (idn[:, s] < rows[s])
        r = (offs[s] + idn[:, s].clamp(0, rows[s] - 1))
        want[ok, 1 + s] = lin[r[ok]]
        want[ok, P + s * D:P + (s + 1) * D] = emb[r[ok]]
    assert torch.equal(x, want)          # bias, w, zero pad and embeddings: bit for bit
    np.testing.assert_array_equal(x.double().numpy(), O.pad_row(O.input_row(tables, lins, 0.375, _per_slot(ids)), S, D)
                                  .astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("S,D,layout", [(5, 16, "fused"), (6, 32, "split"), (7, 8, "fused")])
def test_bags_forward_and_backward_match_the_oracle(S, D, layout):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(7 + S)
    rows = [int(rng.integers(5, 40)) for _ in range(S)]
    coll = _collection(rows, D, layout, seed=S)
    B = 97
    ids = _ids(rng, B, rows, torch.int64)
    bags, per = _bags(rng, B, rows[2], 2)
    bias = torch.tensor([-0.5], device=DEV)
    x = ops.FnnInputFn.apply(ids, coll.weight, coll.linear, bias, coll, bags)
    tables, lins = _np_state(coll)
    per_slot = _per_slot(ids, per, 2)
    ref = O.pad_row(O.input_row(tables, lins, -0.5, per_slot), S, D)
    np.testing.assert_allclose(x.detach().cpu().numpy(), ref, rtol=1e-5, atol=1e-6)
    g = torch.randn(x.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    x.backward(g)
    gt, gl = O.input_grad(O.unpad_row(g.double().cpu().numpy(), S, D), rows, D, per_slot)
    gw, glin, _ = coll.grads()
    offs = coll._offsets.cpu().tolist()
    for s in range(S):
        np.testing.assert_allclose(gw[offs[s]:offs[s] + rows[s]].cpu().numpy(), gt[s], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(glin[offs[s]:offs[s] + rows[s]].cpu().numpy(), gl[s], rtol=1e-5, atol=1e-5)
    if layout == "fused":     # the pad floats of the arena's lines get no gradient
        assert torch.count_nonzero(coll.weight.grad[:, D + 1:]) == 0


@pytest.mark.parametrize("S,D,layout,dtype", [c for c in CASES if c[3] == torch.int64 or c[0] == 6])
def test_backward_matches_the_oracle(S, D, layout, dtype):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(S * 10 + D)
    rows = [int(rng.integers(3, 30)) for _ in range(S)]        # few rows: many duplicate ids per row
    coll = _collection(rows, D, layout, seed=S)
    B = 257
    ids = _ids(rng, B, rows, dtype)
    x = ops.FnnInputFn.apply(ids, coll.weight, coll.linear, torch.zeros(1, device=DEV), coll, None)
    g = torch.randn(x.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(S))
    x.backward(g)
    gt, gl = O.input_grad(O.unpad_row(g.double().cpu().numpy(), S, D), rows, D, _per_slot(ids))
    gw, glin, _ = coll.grads()
    offs = coll._offsets.cpu().tolist()
    for s in range(S):
        np.testing.assert_allclose(gw[offs[s]:offs[s] + rows[s], :D].cpu().numpy(), gt[s], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(glin[offs[s]:offs[s] + rows[s]].cpu().numpy(), gl[s], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("layout,D,bag", [("fused", 16, False), ("split", 32, False), ("fused", 16, True),
                                          ("split", 32, True)])
def test_sparse_sgd_equals_dense_gradient_plus_sgd(layout, D, bag):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(11)
    S, B, lr = 6, 199, 0.05
    rows = [int(rng.integers(5, 30)) for _ in range(S)]
    ids = _ids(rng, B, rows, torch.int64)
    bags = _bags(rng, B, rows[1], 1)[0] if bag else None
    dense = _collection(rows, D, layout, seed=5)
    fused = _collection(rows, D, layout, seed=5, sparse_lr=lr)
    g = torch.randn((B, ops.fnn_layout(S, D)[1]), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    bias = torch.zeros(1, device=DEV)
    ops.FnnInputFn.apply(ids, dense.weight, dense.linear, bias, dense, bags).backward(g)
    ops.FnnInputFn.apply(ids, fused.weight, fused.linear, bias, fused, bags).backward(g)
    assert fused.weight.grad is None
    with torch.no_grad():
        want_w = dense.weight - lr * dense.weight.grad
        torch.testing.assert_close(fused.weight, want_w, rtol=1e-6, atol=1e-6)
        if layout == "split":
            torch.testing.assert_close(fused.linear, dense.linear - lr * dense.linear.grad, rtol=1e-6, atol=1e-6)


def test_bad_arguments_are_refused():
    from deep_recommenders_b200 import _lib, ops
    lib = _lib.load()
    coll = _collection([10, 10, 10], 16, "fused")
    tp, lp, rows = coll.pointers(coll.weight, None)
    S, D = 3, 16
    P, ld = ops.fnn_layout(S, D)
    ids = torch.zeros((8, S), dtype=torch.int64, device=DEV)
    bias = torch.zeros(1, device=DEV)
    out = torch.zeros((8 * ld + 4,), device=DEV)
    g = torch.zeros_like(out)
    st = torch.cuda.current_stream().cuda_stream
    fl = coll.flags

    def fwd(tp_=tp.data_ptr(), ids_=ids.data_ptr(), bias_=bias.data_ptr(), D_=D, ld_=ld, out_=out.data_ptr(),
            flags=fl, lp_=None):
        return lib.dr_fnn_input_fwd(tp_, lp_, rows.data_ptr(), ids_, 8, coll.row_stride, coll.lin_stride, flags,
                                    bias_, 8, S, D_, ld_, out_, st)

    def bwd(tp_=tp.data_ptr(), ids_=ids.data_ptr(), D_=D, ld_=ld, g_=g.data_ptr(), flags=fl):
        return lib.dr_fnn_input_bwd(ids_, 8, rows.data_ptr(), g_, 8, S, D_, ld_, coll.row_stride, coll.lin_stride,
                                    flags, tp_, None, 1.0, st)

    DR_EINVAL, DR_EALIGN = -1, -2
    assert fwd() == 0 and bwd() == 0
    assert fwd(tp_=None) == DR_EINVAL and fwd(ids_=None) == DR_EINVAL and fwd(bias_=None) == DR_EINVAL
    assert fwd(out_=None) == DR_EINVAL and bwd(g_=None) == DR_EINVAL and bwd(tp_=None) == DR_EINVAL
    assert fwd(D_=6) == DR_EINVAL and bwd(D_=6) == DR_EINVAL
    assert fwd(ld_=ld - 4) == DR_EINVAL and fwd(ld_=ld + 1) == DR_EINVAL and bwd(ld_=ld + 4) == DR_EINVAL
    assert fwd(flags=0) == DR_EINVAL        # the split layout needs lin_ptrs
    assert fwd(out_=out.data_ptr() + 4) == DR_EALIGN and bwd(g_=g.data_ptr() + 8) == DR_EALIGN
    torch.cuda.synchronize()
    assert "dr_fnn_input_bwd" in lib.dr_last_error().decode()
    with pytest.raises(ValueError, match="dr_fnn_input_fwd"):
        _lib.check(fwd(ld_=ld + 1), "dr_fnn_input_fwd")


# ---- model level ---------------------------------------------------------------------------------------------------
def _golden_export(c, path):
    torch.save({"format": 1, "bias": torch.tensor(c["bias"], dtype=torch.float32),
                "linear": {f"f{s}": torch.tensor(c["lins"][s], dtype=torch.float32).reshape(-1, 1) for s in range(c["S"])},
                "factorized": {f"f{s}": torch.tensor(c["tables"][s], dtype=torch.float32) for s in range(c["S"])}}, path)


def _golden_model(c, path):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders.estimator.models.ranking import FNN
    cols = [fc.categorical_column_with_identity(f"f{s}", c["rows"][s]) for s in range(c["S"])]
    units = [w.shape[1] for w in c["ws"][:-1]]
    model = FNN([fc.indicator_column(x) for x in cols], [fc.embedding_column(x, c["D"]) for x in cols], path, units,
                seed=0, device=DEV)
    with torch.no_grad():
        for i, l in enumerate(model._dnn.layers):
            k = O.pad_kernel(c["ws"][0], c["S"], c["D"]) if i == 0 else c["ws"][i]
            l.kernel.copy_(torch.tensor(k, dtype=torch.float32))
            l.bias.copy_(torch.tensor(c["bs"][i], dtype=torch.float32))
    return model


@pytest.mark.parametrize("k", [0, 1])
def test_fnn_matches_the_reference_golden(k, tmp_path):
    c = golden_cases()[k]
    path = tmp_path / "fm.pt"
    _golden_export(c, path)
    model = _golden_model(c, path)
    features = {f"f{s}": torch.tensor(c["ids"][s], device=DEV) for s in range(c["S"])}
    out = model(features)
    assert out.shape == (c["B"], 1)
    np.testing.assert_allclose(out.detach().cpu().numpy(), c["out"].reshape(-1, 1), rtol=1e-5, atol=1e-6)


def _fm_and_columns(rows, D):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders.estimator.models.feature_interaction import FM
    cols = [fc.categorical_column_with_identity(f"f{s}", n) for s, n in enumerate(rows)]
    ind, emb = [fc.indicator_column(x) for x in cols], [fc.embedding_column(x, D) for x in cols]
    fm = FM(ind, emb, seed=1, device=DEV)
    with torch.no_grad():
        fm.collection.lin_view().normal_(0, 0.2)
        fm.collection.bias.fill_(-0.3)
    return ind, emb, fm


def _adam(params):
    from deep_recommenders_b200 import ops
    state = [(p, torch.zeros_like(p), torch.zeros_like(p)) for p in params]
    clock = ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device=DEV)

    def step():
        clock.advance()
        for p, m, v in state:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            ops.adam_step_(p.data, p.grad, m, v, 0.0, 0.9, 0.999, 1e-8, zero_grad=True, lr_t_dev=clock.lr_t)
    return step


@pytest.mark.parametrize("rows,D,units,layout", [([40, 3, 9, 25, 7], 8, [16, 8], "fused"),
                                                 ([30, 5, 12, 6, 9, 4], 16, [64, 32], "fused"),
                                                 ([20, 6, 11], 32, [8], "split")])
def test_warm_start_and_adam_steps_match_the_oracle(rows, D, units, layout, tmp_path):
    from deep_recommenders.estimator.models.ranking import FNN
    ind, emb, fm = _fm_and_columns(rows, D)
    assert fm.collection.layout == layout
    path = tmp_path / "fm.pt"
    fm.export(path)
    fm_before = [t.detach().clone() for t in fm.parameters()]
    model = FNN(ind, emb, path, units, seed=2, device=DEV)
    coll = model.embeddings
    S = len(rows)
    for s in range(S):      # warm start: the FM's tables, bit for bit
        assert torch.equal(coll.table(s), fm.collection.table(s))
        assert torch.equal(coll.linear_of(s), fm.collection.linear_of(s))
    assert torch.equal(model.bias, fm.collection.bias.detach())
    P, ld = O.layout(S, D)
    assert model._dnn.layers[0].kernel.shape == (ld, units[0])
    assert torch.count_nonzero(model.pad_rows()) == 0
    tables, lins = _np_state(coll)
    k0 = model._dnn.layers[0].kernel.detach().double().cpu().numpy()
    state = {"tables": tables, "lins": lins, "bias": float(model.bias),
             "ws": [np.concatenate([k0[:1 + S], k0[P:]])] +
                   [l.kernel.detach().double().cpu().numpy() for l in model._dnn.layers[1:]],
             "bs": [l.bias.detach().double().cpu().numpy() for l in model._dnn.layers]}
    step = _adam(list(model.parameters()))
    rng = np.random.default_rng(len(rows))
    B = 128
    for it in range(5):
        ids = np.stack([rng.integers(-1, n, B) for n in rows], axis=1)
        y = rng.integers(0, 2, B).astype(np.float64)
        features = {f"f{s}": torch.from_numpy(ids[:, s]).to(DEV) for s in range(S)}
        p = model(features).reshape(-1)
        yt = torch.from_numpy(y.astype(np.float32)).to(DEV)
        loss = torch.mean(-yt * torch.log(p + 1e-7) - (1 - yt) * torch.log(1 - p + 1e-7))
        loss.backward()
        step()
        ref_loss, ref_p = O.adam_step(state, [[[int(v)] for v in ids[:, s]] for s in range(S)], y)
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref_p, rtol=1e-5, atol=1e-6, err_msg=f"step {it}")
        assert abs(float(loss) - ref_loss) <= 1e-5 * max(1.0, abs(ref_loss)), (it, float(loss), ref_loss)
        assert torch.count_nonzero(model.pad_rows()) == 0, f"pad rows of layer 0 moved at step {it}"
    tables, lins = _np_state(coll)
    for s in range(S):
        np.testing.assert_allclose(tables[s], state["tables"][s], rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(lins[s], state["lins"][s], rtol=1e-4, atol=2e-6)
    k0 = model._dnn.layers[0].kernel.detach().double().cpu().numpy()
    np.testing.assert_allclose(np.concatenate([k0[:1 + S], k0[P:]]), state["ws"][0], rtol=1e-4, atol=2e-6)
    for l, w_ref, b_ref in zip(model._dnn.layers, [None] + state["ws"][1:], state["bs"]):
        if w_ref is not None:
            np.testing.assert_allclose(l.kernel.detach().cpu().numpy(), w_ref, rtol=1e-4, atol=2e-6)
        np.testing.assert_allclose(l.bias.detach().cpu().numpy(), b_ref, rtol=1e-4, atol=2e-6)
    # training the FNN left the FM (and its file) alone
    for a, b in zip(fm_before, fm.parameters()):
        assert torch.equal(a, b.detach())
    saved = torch.load(path, weights_only=True)
    for s in range(S):
        assert torch.equal(saved["factorized"][f"f{s}"], fm.collection.table(s).detach().cpu())


def test_example_runs_both_stages(tmp_path):
    spec = importlib.util.spec_from_file_location(
        "fnn_example", os.path.join(ROOT, "examples", "train_fnn_on_movielens_estimator.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    path = str(tmp_path / "fm.pt")
    first, last, auc = ex.main(["--fm-steps", "20", "--train-steps", "60", "--eval-steps", "2", "--batch-size", "512",
                                "--export", path])
    assert last < first and 0.0 <= auc <= 1.0
    assert os.path.exists(path)
    first2, last2, _ = ex.main(["--warm-up-from-fm", path, "--train-steps", "60", "--eval-steps", "1",
                                "--batch-size", "512"])
    assert last2 < first2
