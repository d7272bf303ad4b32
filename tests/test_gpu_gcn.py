"""GPU checks of the GCN feature: dr_spmm_csr_fwd against float64 with guard words around every output, bit-identical
reruns, the transposed CSR, out-of-range indices, the layer's gradients in both computation orders against the float64
oracle, the reference's golden outputs and its three tests (tests/keras/test_gcn.py), and a training run on the
synthetic Cora."""
import os
import tempfile

import numpy as np
import pytest
import torch

from gcn_oracle import gcn_backward, gcn_forward, spmm_fwd

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ACT = {"linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3, "softmax": 4}
SENTINEL = 12345.0
PAD = 4


def _graph(rng, n_rows, n_cols, empty=3, dup=True, unsorted=True, bad=0):
    """CSR with empty rows, duplicate and unsorted column indices, and `bad` out-of-range indices."""
    deg = rng.integers(0, 9, n_rows)
    deg[rng.choice(n_rows, min(empty, n_rows), replace=False)] = 0
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    idx = rng.integers(0, n_cols, indptr[-1]).astype(np.int32)
    for r in range(n_rows):
        seg = idx[indptr[r]:indptr[r + 1]]
        seg.sort()
        if unsorted and r % 2:
            seg[:] = seg[::-1]
        if dup and len(seg) > 2 and r % 3 == 0:
            seg[1] = seg[0]
    if bad:
        pos = rng.choice(len(idx), bad, replace=False)
        idx[pos] = np.where(np.arange(bad) % 2, -1, n_cols + 5)
    vals = rng.uniform(-1, 1, len(idx)).astype(np.float32)
    return indptr, idx, vals


def _guarded(n, misalign=0):
    buf = torch.full((n + 2 * PAD + misalign,), SENTINEL, device="cuda")
    return buf, buf[PAD + misalign:PAD + misalign + n]


def _check_guards(buf, n, misalign=0):
    b = buf.cpu().numpy()
    assert (b[:PAD + misalign] == SENTINEL).all() and (b[PAD + misalign + n:] == SENTINEL).all()


def _spmm_raw(lib, indptr, idx, vals, n_rows, n_cols, x, F, bias, res, act, misalign=0):
    dev = lambda a: torch.from_numpy(a).cuda() if a is not None else None
    t_ip, t_ix, t_v = dev(indptr), dev(idx), dev(vals)
    ybuf, y = _guarded(n_rows * F, misalign)
    obuf, out = _guarded(n_rows * F, misalign) if res is not None else (None, None)
    xt, bt, rt = dev(x), dev(bias), dev(res)
    p = lambda t: None if t is None else t.data_ptr()
    rc = lib.dr_spmm_csr_fwd(p(t_ip), p(t_ix), p(t_v), n_rows, n_cols, len(idx), p(xt), F, p(bt), p(rt), act, p(y),
                             p(out), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, ybuf, y, obuf, out


@pytest.mark.parametrize("F", [1, 3, 4, 7, 32, 33, 128, 1433])
@pytest.mark.parametrize("act", list(ACT))
@pytest.mark.parametrize("bias,residual", [(False, False), (True, False), (True, True)])
def test_spmm_kernel_against_float64(lib, F, act, bias, residual):
    rng = np.random.default_rng(F * 31 + ACT[act])
    n_rows, n_cols = 37, 53                                     # rectangular
    indptr, idx, vals = _graph(rng, n_rows, n_cols)
    x = rng.standard_normal((n_cols, F)).astype(np.float32)
    b = rng.standard_normal(F).astype(np.float32) if bias else None
    r = rng.standard_normal((n_rows, F)).astype(np.float32) if residual else None
    misalign = 1 if F % 4 == 0 and residual else 0             # also the scalar path for a 4-multiple width
    rc, ybuf, y, obuf, out = _spmm_raw(lib, indptr, idx, vals, n_rows, n_cols, x, F, b, r, ACT[act], misalign)
    if act == "softmax" and F > 1024:
        assert rc == -3 and b"1024" in lib.dr_last_error()
        return
    assert rc == 0, lib.dr_last_error()
    ry, rout = spmm_fwd(indptr, idx, vals, n_cols, x, b, r, act)
    np.testing.assert_allclose(y.cpu().numpy().reshape(n_rows, F), ry, rtol=2e-5, atol=2e-5)
    _check_guards(ybuf, n_rows * F, misalign)
    if residual:
        np.testing.assert_allclose(out.cpu().numpy().reshape(n_rows, F), rout, rtol=2e-5, atol=2e-5)
        _check_guards(obuf, n_rows * F, misalign)
    empty = np.flatnonzero(np.diff(indptr) == 0)
    assert len(empty) and np.allclose(ry[empty], spmm_fwd(np.zeros(2, np.int32), np.zeros(0, np.int32),
                                                           np.zeros(0, np.float32), n_cols, x, b, None, act)[0][0])


def test_spmm_zero_rows_and_out_of_range_indices(lib):
    rng = np.random.default_rng(2)
    x = rng.standard_normal((10, 8)).astype(np.float32)
    rc, ybuf, _, _, _ = _spmm_raw(lib, np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32), 0, 10,
                                  x, 8, None, None, 0)
    assert rc == 0
    _check_guards(ybuf, 0)
    indptr, idx, vals = _graph(rng, 20, 10, bad=6)
    for F in (8, 7):
        xf = rng.standard_normal((10, F)).astype(np.float32)
        rc, ybuf, y, _, _ = _spmm_raw(lib, indptr, idx, vals, 20, 10, xf, F, None, None, 1)
        assert rc == 0
        np.testing.assert_allclose(y.cpu().numpy().reshape(20, F), spmm_fwd(indptr, idx, vals, 10, xf, act="relu")[0],
                                   rtol=2e-5, atol=2e-5)
        _check_guards(ybuf, 20 * F)
    from deep_recommenders_b200.ops import CSRAdjacency
    with pytest.raises(ValueError):
        CSRAdjacency(indptr, idx, vals, (20, 10))
    assert lib.dr_spmm_csr_fwd(None, None, None, 1 << 31, 4, 0, None, 4, None, None, 0, None, None, None) == -3
    assert lib.dr_spmm_csr_fwd(None, None, None, 4, 4, 0, None, 4, None, None, 9, None, None, None) == -1


def _adj(rng, n_rows, n_cols):
    import scipy.sparse as sp
    from deep_recommenders_b200.ops import CSRAdjacency
    indptr, idx, vals = _graph(rng, n_rows, n_cols)
    return CSRAdjacency(indptr, idx, vals, (n_rows, n_cols)), sp.csr_matrix((vals, idx, indptr), (n_rows, n_cols))


def test_transpose_against_scipy():
    a, m = _adj(np.random.default_rng(4), 300, 211)
    t = m.T.tocsr()                     # scipy's transpose lists each transposed row in ascending original row
    assert np.array_equal(a.t_indptr.cpu().numpy(), t.indptr)
    assert np.array_equal(a.t_indices.cpu().numpy(), t.indices) and np.array_equal(a.t_values.cpu().numpy(), t.data)


@pytest.mark.parametrize("F", [7, 128])
def test_bit_identical_reruns_forward_and_transposed_backward(F):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(5)
    a, _ = _adj(rng, 5000, 4000)
    x = torch.from_numpy(rng.standard_normal((4000, F)).astype(np.float32)).cuda()
    g = torch.from_numpy(rng.standard_normal((5000, F)).astype(np.float32)).cuda()
    runs = []
    for _ in range(3):
        xr = x.clone().requires_grad_()
        y = ops.SpMMFn.apply(xr, None, None, a, 1)
        y.backward(g)
        runs.append((y.detach().clone(), xr.grad.clone()))
    for y, gx in runs[1:]:
        assert torch.equal(y, runs[0][0]) and torch.equal(gx, runs[0][1])


def _layer_case(rng, F, units, act, bias, residual, sparse):
    from deep_recommenders.keras.models.retrieval import GCN
    n = 60
    a, m = _adj(rng, n, n)
    x = rng.standard_normal((n, F)).astype(np.float32)
    layer = GCN(units, residual=residual, use_bias=bias, activation=None if act == "linear" else act)
    xt = torch.from_numpy(x).cuda().requires_grad_()
    layer(xt, a if sparse else torch.from_numpy(m.toarray()).cuda())        # builds
    with torch.no_grad():
        layer.kernel.copy_(torch.from_numpy(rng.standard_normal((F, units)).astype(np.float32) * 0.5))
        if bias:
            layer.bias.copy_(torch.from_numpy(rng.standard_normal(units).astype(np.float32)))
    return layer, a, m, x, xt


@pytest.mark.parametrize("F,units", [(40, 6), (5, 24), (9, 9)])           # F > units, F < units, tie
@pytest.mark.parametrize("act", list(ACT))
@pytest.mark.parametrize("sparse", [True, False])
def test_layer_gradients_both_orders_against_oracle(F, units, act, sparse):
    rng = np.random.default_rng(F * 7 + units + ACT[act])
    residual = F == units
    layer, a, m, x, xt = _layer_case(rng, F, units, act, True, residual, sparse)
    adj = a if sparse else torch.from_numpy(m.toarray()).cuda()
    out = layer(xt, adj)
    g = rng.standard_normal(out.shape).astype(np.float32)
    out.backward(torch.from_numpy(g).cuda())
    w, b = layer.kernel.detach().cpu().numpy(), layer.bias.detach().cpu().numpy()
    ref, saved = gcn_forward(m.toarray(), x, w, b, act, residual)
    gx, gw, gb = gcn_backward(m.toarray(), x, w, act, residual, saved, g)
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref, rtol=1e-4, atol=1e-5)
    for got, want in ((xt.grad, gx), (layer.kernel.grad, gw), (layer.bias.grad, gb)):
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-4, atol=1e-4)


def test_layer_reproduces_reference_golden():
    import scipy.sparse as sp
    from deep_recommenders.keras.models.retrieval import GCN
    gold = np.load(os.path.join(HERE, "golden", "gcn_golden.npz"))
    tags = sorted({k[len("f32_layer_"):-len("_out")] for k in gold.files if k.startswith("f32_layer_") and k.endswith("_out")})
    for tag in tags:
        k = f"f32_layer_{tag}"
        units, bias, res, sparse = gold[k + "_args"].tolist()
        act = str(gold[k + "_act"])
        x = torch.from_numpy(gold[k + "_x"]).cuda()
        shape = gold[k + "_adj"].shape
        adj = (sp.coo_matrix((gold[k + "_vals"], (gold[k + "_rows"], gold[k + "_cols"])), shape) if sparse
               else gold[k + "_adj"])
        layer = GCN(units, residual=bool(res), use_bias=bool(bias), activation=None if act == "linear" else act)
        layer(x, adj)
        with torch.no_grad():
            layer.kernel.copy_(torch.from_numpy(gold[k + "_w"]))
            if bias:
                layer.bias.copy_(torch.from_numpy(gold[k + "_b"]))
        np.testing.assert_allclose(layer(x, adj).detach().cpu().numpy(), gold[k + "_out"], rtol=1e-5, atol=1e-5, err_msg=tag)


_ADJ = np.asarray([[0, 1, 0], [1, 0, 0], [0, 1, 1]], np.float32)
_EMB = np.asarray([[0.1, 0.2, 0.3, 0.0], [0.4, 0.5, 0.6, 0.0], [0.7, 0.8, 0.9, 0.0]], np.float32)


@pytest.mark.parametrize("sparse", [True, False])
def test_reference_gcn_adj_sparse_and_full_matrix(sparse):
    """tests/keras/test_gcn.py:19-69: GCN(2, kernel_initializer="ones") == relu(adj @ emb @ ones)."""
    import scipy.sparse as sp
    from deep_recommenders.keras.models.retrieval import GCN
    expect = np.maximum(_ADJ @ _EMB @ np.ones((4, 2)), 0)
    coo = sp.coo_matrix(_ADJ)
    adj = torch.sparse_coo_tensor(np.stack([coo.row, coo.col]), coo.data, coo.shape) if sparse else _ADJ
    out = GCN(2, kernel_initializer="ones")(torch.from_numpy(_EMB).cuda(), adj)
    np.testing.assert_allclose(out.detach().cpu().numpy(), expect, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("num_nodes,dim", [(8, 4), (16, 8), (32, 16)])
def test_reference_gcn_train_save_load(num_nodes, dim):
    """tests/keras/test_gcn.py:71-111: GCN(16) -> GCN(16) -> GCN(2, softmax), one fit, then save / load with equal
    configs and equal predictions."""
    import scipy.sparse as sp
    from deep_recommenders.keras.layers import Model
    from deep_recommenders.keras.models.retrieval import GCN
    from deep_recommenders_b200.keras.engine import Adam

    class Net(Model):
        def __init__(self):
            super().__init__()
            self.g1, self.g2, self.g3 = GCN(16), GCN(16), GCN(2, activation="softmax")
            self.built = True

        def call(self, inputs, **kwargs):
            adj, emb = inputs
            return self.g3(self.g2(self.g1(emb, adj), adj), adj)

        def get_config(self):
            return {**super().get_config(), "layers": [l.get_config() for l in (self.g1, self.g2, self.g3)]}

    np.random.seed(42)
    torch.manual_seed(42)
    adj = sp.random(num_nodes, num_nodes).tocsr()
    adj.sort_indices()
    emb = torch.from_numpy(np.random.normal(size=(num_nodes, dim)).astype(np.float32)).cuda()
    t = np.random.randint(2, size=num_nodes).astype(np.float32)
    targets = np.stack([t, 1 - t], axis=1)
    model = Net()
    model.compile(optimizer=Adam(0.01), loss="categorical_crossentropy")
    hist = model.fit([adj, emb], targets, batch_size=num_nodes, shuffle=False)
    assert np.isfinite(hist["loss"][0])
    pred = model.predict([adj, emb])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "gcn.pt")
        model.save(path)
        blob = torch.load(path, weights_only=False)
        loaded = Net()
        loaded.predict([adj, emb])
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == model.get_config() == blob["config"]
        assert torch.equal(loaded.predict([adj, emb]), pred)


def test_training_on_synthetic_cora_beats_chance():
    import importlib.util
    import sys
    from deep_recommenders.datasets import write_synthetic_cora
    spec = importlib.util.spec_from_file_location(
        "train_gcn_example", os.path.join(os.path.dirname(HERE), "examples", "train_gcn_on_cora_keras.py"))
    ex = importlib.util.module_from_spec(spec)
    sys.modules["train_gcn_example"] = ex
    spec.loader.exec_module(ex)
    with tempfile.TemporaryDirectory() as d:
        hist, test = ex.train_model(write_synthetic_cora(d, seed=1), epochs=200, seed=1, verbose=0)
    assert hist["val_acc"][-1] > 0.6 and test["acc"] > 0.6, (hist["val_acc"][-1], test)
