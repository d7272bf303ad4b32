"""CPU tests of the multi-task package: the float64 oracle against the golden vectors of the reference and against
torch autograd, the SyntheticForMultiTask port, input_layer, constructor errors, and C-ABI argument validation."""
import os

import numpy as np
import pytest
import torch

import mtl_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mtl_golden.npz")
MMOE_CASES = ["ref", "e3t2", "e1t1", "e4t1", "e5t3"]
ESMM_CASES = ["ref", "small", "linear"]


@pytest.fixture(scope="module")
def z():
    return np.load(GOLDEN)


def _mmoe_args(z, k):
    T, E = (int(v) for v in z[k + "_args"])
    eact, tact = (str(a) for a in z[k + "_acts"])
    return E, T, [int(u) for u in z[k + "_expert_units"]], [int(u) for u in z[k + "_task_units"]], eact, tact


@pytest.mark.parametrize("pre,tol", [("f64_", 1e-12), ("f32_", 1e-5)])
@pytest.mark.parametrize("case", MMOE_CASES)
def test_mmoe_oracle_matches_golden(z, pre, tol, case):
    k = f"{pre}mmoe_{case}"
    E, T, eu, tu, eact, tact = _mmoe_args(z, k)
    x = z[k + "_x"].astype(np.float64)
    ws, bs = O.golden_weights(z, k)
    ws = [w.astype(np.float64) for w in ws]
    bs = [None if b is None else b.astype(np.float64) for b in bs]
    assert len(ws) == E * len(eu) + E + T * (len(tu) + 1)
    outs, _ = O.mmoe_forward(x[:, O.input_order(x.shape[1])], ws, bs, E, T, eu, tu, eact, tact)
    assert len(outs) == T
    for t in range(T):
        ref = z[f"{k}_out{t}"]
        assert ref.shape == (x.shape[0], 1)
        np.testing.assert_allclose(outs[t], ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("pre,tol", [("f64_", 1e-12), ("f32_", 1e-5)])
@pytest.mark.parametrize("case", ESMM_CASES)
def test_esmm_oracle_matches_golden(z, pre, tol, case):
    k = f"{pre}esmm_{case}"
    x = z[k + "_x"].astype(np.float64)
    ws, bs = O.golden_weights(z, k)
    hu = [int(u) for u in z[k + "_hidden_units"]]
    (p_cvr, p_ctr, p_ctcvr), _ = O.esmm_forward(x[:, O.input_order(x.shape[1])], [w.astype(np.float64) for w in ws],
                                                [b.astype(np.float64) for b in bs], hu, str(z[k + "_act"]))
    for name, v in (("p_cvr", p_cvr), ("p_ctr", p_ctr), ("p_ctcvr", p_ctcvr)):
        np.testing.assert_allclose(v, z[f"{k}_{name}"], rtol=tol, atol=tol)


_TORCH_ACT = {"relu": torch.relu, "tanh": torch.tanh, "sigmoid": torch.sigmoid}


def _torch_tower(x, ws, bs, act):
    for i, (w, b) in enumerate(zip(ws, bs)):
        x = x @ w + (0 if b is None else b)
        if i < len(ws) - 1:
            x = _TORCH_ACT[act](x)
    return x


@pytest.mark.parametrize("case", MMOE_CASES)
def test_mmoe_oracle_backward_matches_autograd(z, case):
    k = f"f64_mmoe_{case}"
    E, T, eu, tu, eact, tact = _mmoe_args(z, k)
    x = z[k + "_x"][:, O.input_order(z[k + "_x"].shape[1])]
    ws, bs = O.golden_weights(z, k)
    rng = np.random.default_rng(5)
    g = [rng.standard_normal((x.shape[0], 1)) for _ in range(T)]
    outs, cache = O.mmoe_forward(x, ws, bs, E, T, eu, tu, eact, tact)
    gx, gws, gbs = O.mmoe_backward(cache, g)

    tx = torch.tensor(x, requires_grad=True)
    tw = [torch.tensor(w, requires_grad=True) for w in ws]
    tb = [None if b is None else torch.tensor(b, requires_grad=True) for b in bs]
    ex_idx, gate_idx, task_idx = O.mmoe_layout(E, T, len(eu), len(tu) + 1)
    experts = torch.stack([_torch_tower(tx, [tw[i] for i in ix], [tb[i] for i in ix], eact) for ix in ex_idx], 1)
    loss = 0
    for t in range(T):
        gate = torch.softmax(tx @ tw[gate_idx[t]], dim=-1)
        mixed = torch.bmm(gate.unsqueeze(1), experts).squeeze(1)
        out = _torch_tower(mixed, [tw[i] for i in task_idx[t]], [tb[i] for i in task_idx[t]], tact)
        np.testing.assert_allclose(out.detach().numpy(), outs[t], rtol=1e-12, atol=1e-12)
        loss = loss + (out * torch.tensor(g[t])).sum()
    loss.backward()
    np.testing.assert_allclose(gx, tx.grad.numpy(), rtol=1e-10, atol=1e-12)
    for i in range(len(ws)):
        ref = tw[i].grad.numpy() if tw[i].grad is not None else np.zeros_like(ws[i])   # unused gates: no gradient
        np.testing.assert_allclose(gws[i], ref, rtol=1e-10, atol=1e-12, err_msg=f"w{i}")
        if bs[i] is not None:
            np.testing.assert_allclose(gbs[i], tb[i].grad.numpy(), rtol=1e-10, atol=1e-12, err_msg=f"b{i}")


@pytest.mark.parametrize("case", ESMM_CASES)
def test_esmm_oracle_backward_matches_autograd(z, case):
    k = f"f64_esmm_{case}"
    x = z[k + "_x"][:, O.input_order(z[k + "_x"].shape[1])]
    ws, bs = O.golden_weights(z, k)
    hu, act = [int(u) for u in z[k + "_hidden_units"]], str(z[k + "_act"])
    rng = np.random.default_rng(6)
    g = [rng.standard_normal((x.shape[0], 1)) for _ in range(3)]
    _, cache = O.esmm_forward(x, ws, bs, hu, act)
    gx, gws, gbs = O.esmm_backward(cache, *g)
    tx = torch.tensor(x, requires_grad=True)
    tw = [torch.tensor(w, requires_grad=True) for w in ws]
    tb = [torch.tensor(b, requires_grad=True) for b in bs]
    L = len(hu) + 1
    p_cvr = torch.sigmoid(_torch_tower(tx, tw[:L], tb[:L], act))
    p_ctr = torch.sigmoid(_torch_tower(tx, tw[L:], tb[L:], act))
    sum(((p * torch.tensor(gg)).sum() for p, gg in zip((p_cvr, p_ctr, p_ctr * p_cvr), g))).backward()
    np.testing.assert_allclose(gx, tx.grad.numpy(), rtol=1e-10, atol=1e-12)
    for i in range(len(ws)):
        np.testing.assert_allclose(gws[i], tw[i].grad.numpy(), rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(gbs[i], tb[i].grad.numpy(), rtol=1e-10, atol=1e-12)


def test_oracle_mix_softmax_extremes():
    experts = np.arange(2 * 3 * 4, dtype=np.float64).reshape(2, 3, 4)
    logits = np.array([[[1e4, -1e4, 0.0]], [[5.0, 5.0, 5.0]]])
    gates, out = O.mix_fwd(experts, logits)
    assert np.isfinite(gates).all()
    np.testing.assert_array_equal(gates[0, 0], [1.0, 0.0, 0.0])
    np.testing.assert_allclose(gates[1, 0], [1 / 3] * 3)
    np.testing.assert_allclose(out[1, 0], experts[1].mean(0))


# ---- SyntheticForMultiTask ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["s0", "s3", "s11"])
def test_synthetic_data_bit_identical_to_reference(z, case):
    from deep_recommenders.datasets.synthetic_for_multi_task import synthetic_data
    seed, n, dim, c, p, m = z[f"syn_{case}_args"]
    np.random.seed(int(seed))
    x, (y1, y2) = synthetic_data(int(n), int(dim), c=c, p=p, m=int(m))
    for got, name in ((x, "x"), (y1, "y1"), (y2, "y2")):
        ref = z[f"syn_{case}_{name}"]
        assert got.dtype == np.float32 and got.shape == ref.shape
        assert got.tobytes() == ref.tobytes(), name


def test_input_fn_batches_repeat_and_remainder():
    from deep_recommenders.datasets import SyntheticForMultiTask
    ds = SyntheticForMultiTask(10, example_dim=3)
    np.random.seed(4)
    batches = list(ds.input_fn(epochs=2, batch_size=4))
    assert [b[0]["C0"].shape for b in batches] == [(4, 1)] * 5
    np.random.seed(4)
    batches = list(ds.input_fn(epochs=3, batch_size=7))
    assert [len(b[1]["labels0"]) for b in batches] == [7, 7, 7, 7, 2]        # remainder kept
    f, lab = batches[1]
    assert sorted(f) == ["C0", "C1", "C2"] and sorted(lab) == ["labels0", "labels1"]
    assert f["C1"].dtype == np.float32 and lab["labels1"].shape == (7,)
    # the same draw, unbatched: rows repeat across the epoch boundary in order
    from deep_recommenders.datasets.synthetic_for_multi_task import synthetic_data
    np.random.seed(4)
    x, (y1, _) = synthetic_data(10, 3)
    rows = np.concatenate([b[0]["C2"][:, 0] for b in batches])
    np.testing.assert_array_equal(rows, np.tile(x[:, 2], 3))
    np.testing.assert_array_equal(np.concatenate([b[1]["labels0"] for b in batches]), np.tile(y1, 3))


def test_input_fn_take_skip_and_new_draw_per_call():
    from deep_recommenders.datasets import SyntheticForMultiTask
    ds = SyntheticForMultiTask(100, example_dim=4)
    np.random.seed(0)
    a = ds.input_fn(batch_size=8)
    b = ds.input_fn(batch_size=8)
    assert len(a) == 13 and len(a.take(5)) == 5 and len(a.skip(10)) == 3 and len(a.skip(3).take(20)) == 10
    first_a, first_b = next(iter(a))[0]["C0"], next(iter(b))[0]["C0"]
    assert not np.array_equal(first_a, first_b)                         # each call draws a new dataset
    np.testing.assert_array_equal(next(iter(a.skip(2)))[0]["C3"], list(a)[2][0]["C3"])


# ---- feature columns --------------------------------------------------------------------------------------------------
def test_input_layer_sorts_by_name_and_copies_once(monkeypatch):
    from deep_recommenders_b200 import feature_column as fc
    cols = [fc.numeric_column("C{}".format(i)) for i in range(12)]
    x = np.arange(3 * 12, dtype=np.float64).reshape(3, 12)
    feats = {"C{}".format(i): x[:, i:i + 1] for i in range(12)}
    copies = []
    real_to = torch.Tensor.to
    monkeypatch.setattr(torch.Tensor, "to", lambda self, *a, **k: copies.append(1) or real_to(self, *a, **k))
    out = fc.input_layer(feats, cols, device="cpu")
    assert len(copies) == 1
    order = [0, 1, 10, 11, 2, 3, 4, 5, 6, 7, 8, 9]
    assert out.dtype == torch.float32
    np.testing.assert_array_equal(out.numpy(), x[:, order].astype(np.float32))
    assert [c for c in sorted(["C{}".format(i) for i in range(100)])][:4] == ["C0", "C1", "C10", "C11"]


def test_input_layer_shapes_and_errors():
    from deep_recommenders_b200 import feature_column as fc
    wide = fc.numeric_column("a", shape=(2, 3))
    assert wide.width == 6 and fc.numeric_column("b", shape=4).shape == (4,)
    out = fc.input_layer({"a": np.ones((2, 2, 3)), "b": np.zeros((2, 4))}, [fc.numeric_column("b", 4), wide], "cpu")
    assert out.shape == (2, 10) and out[:, :6].sum() == 12
    with pytest.raises(KeyError, match="missing"):
        fc.input_layer({"a": np.ones((2, 6))}, [wide, fc.numeric_column("z")], "cpu")
    with pytest.raises(ValueError, match="expects"):
        fc.input_layer({"a": np.ones((2, 5))}, [wide], "cpu")
    with pytest.raises(NotImplementedError, match="numeric columns only"):
        fc.input_layer({}, [fc.indicator_column(fc.categorical_column_with_identity("c", 3))], "cpu")
    with pytest.raises(ValueError, match="greater than 0"):
        fc.numeric_column("x", shape=(0,))


# ---- constructors ---------------------------------------------------------------------------------------------------
def test_constructor_errors_before_any_cuda_call(monkeypatch):
    from deep_recommenders_b200 import _lib
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders.estimator.models.multi_task_learning import ESMM, MMoE
    monkeypatch.setattr(_lib, "load", lambda: pytest.fail("C-ABI reached"))
    cols = [fc.numeric_column("C{}".format(i)) for i in range(4)]
    kw = dict(expert_hidden_units=[4], task_hidden_units=[3])
    with pytest.raises(IndexError, match="num_tasks"):
        MMoE(cols, num_tasks=3, num_experts=2, **kw)
    with pytest.raises(TypeError, match="batch_normalization"):
        MMoE(cols, 2, 2, task_batch_normalization=True, **kw)
    with pytest.raises(TypeError, match="batch_normalization"):
        MMoE(cols, 2, 2, expert_batch_normalization=True, **kw)
    with pytest.raises(NotImplementedError, match="dropout"):
        MMoE(cols, 2, 2, expert_dropout=0.1, **kw)
    with pytest.raises(NotImplementedError, match="dropout"):
        MMoE(cols, 2, 2, task_dropout=0.5, **kw)
    with pytest.raises(ValueError, match="serves up to"):
        MMoE(cols, 2, 33, **kw)
    with pytest.raises(ValueError, match="unsupported activation"):
        MMoE(cols, 2, 2, expert_hidden_activation="gelu", device="cpu", **kw)
    with pytest.raises(NotImplementedError, match="numeric"):
        MMoE([fc.indicator_column(fc.categorical_column_with_identity("c", 3))], 1, 1, **kw)
    with pytest.raises(TypeError, match="batch_normalization"):
        ESMM(cols, [4], batch_normalization=True)
    with pytest.raises(NotImplementedError, match="dropout"):
        ESMM(cols, [4], dropout=0.2)
    with pytest.raises(NotImplementedError, match="not served"):
        ESMM(cols, [4], kernel_initializer="ones")


def test_parameter_order_and_independent_towers():
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders.estimator.models.multi_task_learning import ESMM, MMoE
    cols = [fc.numeric_column("C{}".format(i)) for i in range(6)]
    m = MMoE(cols, num_tasks=2, num_experts=3, expert_hidden_units=[5, 4], task_hidden_units=[3], seed=1, device="cpu")
    shapes = [tuple(k.shape) for k, _ in m.dense_views()]
    assert shapes == [(6, 5), (5, 4)] * 3 + [(6, 3)] * 2 + [(4, 3), (3, 1)] * 2
    assert [b is None for _, b in m.dense_views()] == [False] * 6 + [True] * 2 + [False] * 4
    # every parameter element belongs to exactly one reference variable: writing one view changes no other
    views = m.dense_views()
    params = list(m.parameters())
    total = sum(p.numel() for p in params)
    assert total == sum(k.numel() + (0 if b is None else b.numel()) for k, b in views)
    with torch.no_grad():
        for p in params:
            p.zero_()
        views[0][0].fill_(1.0)                                 # expert 0, layer 0 kernel
    assert sum(float(p.detach().sum()) for p in params) == views[0][0].numel()
    assert float(views[2][0].abs().sum()) == 0.0              # expert 1 untouched
    # expert towers initialised independently (not one cached tower)
    m2 = MMoE(cols, num_tasks=2, num_experts=2, expert_hidden_units=[5], task_hidden_units=[], seed=3, device="cpu")
    v = m2.dense_views()
    assert not torch.equal(v[0][0], v[1][0]) and not torch.equal(v[4][0], v[5][0])
    e = ESMM(cols, [4, 3], seed=2, device="cpu")
    v = e.dense_views()
    assert [tuple(k.shape) for k, _ in v] == [(6, 4), (4, 3), (3, 1)] * 2
    assert not torch.equal(v[0][0], v[3][0]) and not torch.equal(v[1][0], v[4][0])
    # glorot limit of each block uses that tower's own fan_out
    big = MMoE([fc.numeric_column("x", shape=400)], 1, 8, expert_hidden_units=[100], task_hidden_units=[],
               seed=0, device="cpu")
    lim = np.sqrt(6.0 / (400 + 100))
    k0 = big.dense_views()[0][0]
    assert float(k0.abs().max()) <= lim and float(k0.abs().max()) > 0.9 * lim


def test_reference_import_paths():
    from deep_recommenders.estimator.models.multi_task_learning import MMoE, ESMM
    from deep_recommenders.estimator.models.multi_task_learning.mixture_of_experts import MMoE as M2
    from deep_recommenders.estimator.models.multi_task_learning.esmm import ESMM as E2
    from deep_recommenders.datasets import SyntheticForMultiTask
    from deep_recommenders.datasets.synthetic_for_multi_task import SyntheticForMultiTask as S2, synthetic_data
    assert MMoE is M2 and ESMM is E2 and SyntheticForMultiTask is S2 and callable(synthetic_data)


# ---- C-ABI ----------------------------------------------------------------------------------------------------------
def test_c_abi_host_validation(lib):
    p = 256
    #                    experts logits B  E  T  H  gates out stream
    assert lib.dr_moe_mix_fwd(None, p, 2, 2, 2, 4, p, p, None) == -1
    assert b"null pointer" in lib.dr_last_error()
    assert lib.dr_moe_mix_fwd(p, p, 2, 2, 2, 4, p, None, None) == -1
    assert lib.dr_moe_mix_fwd(p, p, -1, 2, 2, 4, p, p, None) == -1
    assert lib.dr_moe_mix_fwd(p, p, 2, 0, 2, 4, p, p, None) == -1
    assert lib.dr_moe_mix_fwd(p, p, 2, 2, 0, 4, p, p, None) == -1
    assert lib.dr_moe_mix_fwd(p, p, 2, 2, 2, 0, p, p, None) == -1
    assert lib.dr_moe_mix_fwd(p, p, 2, 33, 2, 4, p, p, None) == -3            # DR_ENOTSUP just outside
    assert b"served" in lib.dr_last_error()
    assert lib.dr_moe_mix_fwd(p, p, 2, 2, 17, 4, p, p, None) == -3
    assert lib.dr_moe_mix_fwd(p, p, 2, 32, 16, 1 << 26, p, p, None) == -3
    assert lib.dr_moe_mix_fwd(p, p, 0, 32, 16, 1024, p, p, None) == 0          # B = 0: no-op, no launch
    #                    experts gates g_out B  E  T  H  g_experts g_logits stream
    assert lib.dr_moe_mix_bwd(p, p, None, 2, 2, 2, 4, p, p, None) == -1
    assert lib.dr_moe_mix_bwd(p, p, p, 2, 2, 2, 4, p, None, None) == -1
    assert lib.dr_moe_mix_bwd(p, p, p, 2, 33, 2, 4, p, p, None) == -3
    assert lib.dr_moe_mix_bwd(p, p, p, 2, 1, 17, 4, p, p, None) == -3
    assert lib.dr_moe_mix_bwd(p, p, p, 0, 1, 1, 1, p, p, None) == 0
    #                          x  w  b  M  G  K  N  act y stream
    assert lib.dr_dense_grouped_fwd(None, p, p, 4, 2, 3, 3, 0, p, None) == -1
    assert lib.dr_dense_grouped_fwd(p, p, p, 4, 0, 3, 3, 0, p, None) == -1
    assert lib.dr_dense_grouped_fwd(p, p, p, 4, 2, 0, 3, 0, p, None) == -1
    assert lib.dr_dense_grouped_fwd(p, p, p, -1, 2, 3, 3, 0, p, None) == -1
    assert lib.dr_dense_grouped_fwd(p, p, p, 4, 2, 3, 3, 7, p, None) == -1
    assert b"activation" in lib.dr_last_error()
    assert lib.dr_dense_grouped_fwd(p, p, p, 4, 1 << 20, 1 << 12, 3, 0, p, None) == -1
    assert b"2^31" in lib.dr_last_error()
    #                          x  w  y  gy M  G  K  N  act gz gx gw gb stream
    assert lib.dr_dense_grouped_bwd(p, p, p, None, 4, 2, 3, 3, 0, None, p, p, None, None) == -1
    assert lib.dr_dense_grouped_bwd(p, p, p, p, 4, 2, 3, 3, 0, None, None, None, None, None) == -1
    assert lib.dr_dense_grouped_bwd(p, p, None, p, 4, 2, 3, 3, 1, p, p, p, None, None) == -1
    assert b"activation needs" in lib.dr_last_error()
    assert lib.dr_dense_grouped_bwd(p, p, p, p, 4, 2, 3, 3, 1, None, p, p, None, None) == -1
    assert lib.dr_dense_grouped_bwd(p, p, p, p, 4, 2, 3, 0, 0, None, p, p, None, None) == -1
