"""CPU checks of the GCN feature (run with -m "not gpu"): the float64 oracle against the golden outputs of the
reference's own gcn.py and against torch float64 autograd, the Cora port bit for bit against the reference's
cora.py, the synthetic Cora writer, the host-side validation of the adjacency and of the layer, and the engine's
weighted loss and weighted accuracy."""
import os

import numpy as np
import pytest
import torch

from gcn_oracle import ACTS, gcn_backward, gcn_forward

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "gcn_golden.npz"))
FIXTURE = os.path.join(HERE, "golden", "cora_small")
LAYER_TAGS = sorted({k[len("f64_layer_"):-len("_out")] for k in GOLD.files
                     if k.startswith("f64_layer_") and k.endswith("_out")})


def _case(pre, tag):
    k = f"{pre}layer_{tag}"
    units, bias, res, sparse = GOLD[k + "_args"].tolist()
    act = str(GOLD[k + "_act"])
    return k, act, bool(bias), bool(res)


@pytest.mark.parametrize("tag", LAYER_TAGS)
@pytest.mark.parametrize("pre,tol", [("f64_", 1e-12), ("f32_", 1e-5)])
def test_oracle_matches_reference_golden(tag, pre, tol):
    k, act, bias, res = _case(pre, tag)
    out, _ = gcn_forward(GOLD[k + "_adj"], GOLD[k + "_x"], GOLD[k + "_w"], GOLD[k + "_b"] if bias else None, act, res)
    np.testing.assert_allclose(out, GOLD[k + "_out"], rtol=tol, atol=tol)


def test_golden_covers_the_cases():
    acts = {str(GOLD[f"f64_layer_{t}_act"]) for t in LAYER_TAGS}
    assert acts == set(ACTS)
    args = np.stack([GOLD[f"f64_layer_{t}_args"] for t in LAYER_TAGS])
    assert set(args[:, 1]) == {0, 1} and set(args[:, 2]) == {0, 1} and set(args[:, 3]) == {0, 1}
    widths = [(GOLD[f"f64_layer_{t}_x"].shape[1], GOLD[f"f64_layer_{t}_args"][0]) for t in LAYER_TAGS]
    assert any(f > u for f, u in widths) and any(f < u for f, u in widths) and any(f == u for f, u in widths)
    assert any((GOLD[f"f64_layer_{t}_adj"] == 0).all(axis=1).any() for t in LAYER_TAGS)           # empty rows
    assert any(len(GOLD[f"f64_layer_{t}_rows"]) > len(set(zip(GOLD[f"f64_layer_{t}_rows"], GOLD[f"f64_layer_{t}_cols"])))
               for t in LAYER_TAGS)                                                              # duplicates


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("residual", [False, True])
def test_oracle_backward_matches_torch_autograd(act, residual):
    rng = np.random.default_rng(3)
    n, F = 12, 5
    units = F if residual else 7
    adj = (rng.random((n, n)) < 0.3) * rng.random((n, n))
    x, w, b = rng.standard_normal((n, F)), rng.standard_normal((F, units)), rng.standard_normal(units)
    g = rng.standard_normal((n, units))
    out, saved = gcn_forward(adj, x, w, b, act, residual)
    gx, gw, gb = gcn_backward(adj, x, w, act, residual, saved, g)
    tx, tw, tb = (torch.tensor(t, requires_grad=True) for t in (x, w, b))
    z = torch.tensor(adj) @ tx @ tw + tb
    y = {"linear": z, "relu": torch.relu(z), "sigmoid": torch.sigmoid(z), "tanh": torch.tanh(z),
         "softmax": torch.softmax(z, -1)}[act]
    if residual:
        y = y + tx
    (y * torch.tensor(g)).sum().backward()
    np.testing.assert_allclose(out, y.detach().numpy(), rtol=1e-12, atol=1e-12)
    for got, ref in ((gx, tx.grad), (gw, tw.grad), (gb, tb.grad)):
        np.testing.assert_allclose(got, ref.numpy(), rtol=1e-10, atol=1e-12)


def _cora_replay():
    from deep_recommenders.datasets import Cora
    np.random.seed(int(GOLD["cora_seed"]))
    cora = Cora(FIXTURE)
    ids, features, labels = cora.load_content()
    _, raw, _ = cora.load_content(normalize=False)
    graph = cora.build_graph(ids)
    sg = cora.spectral_graph(graph)
    train_nodes = cora.sample_train_nodes(labels)
    split = cora.split_labels(labels, num_valid_nodes=50)
    return cora, ids, features, raw, labels, graph, sg, train_nodes, split


def test_cora_port_bit_identical_to_reference():
    cora, ids, features, raw, labels, graph, sg, train_nodes, split = _cora_replay()
    assert cora.num_classes == int(GOLD["cora_num_classes"]) == 7
    assert (ids == GOLD["cora_ids"]).all() and (labels == GOLD["cora_labels"]).all()
    for got, ref in ((features.toarray(), GOLD["cora_features"]), (raw.toarray(), GOLD["cora_features_raw"]),
                     (graph.toarray(), GOLD["cora_graph"]), (sg.indptr, GOLD["cora_spectral_indptr"]),
                     (sg.indices, GOLD["cora_spectral_indices"]), (sg.data, GOLD["cora_spectral_data"]),
                     (np.asarray(train_nodes), GOLD["cora_train_nodes"]), (cora.encode_labels(labels), GOLD["cora_encoded"])):
        assert got.dtype == ref.dtype and got.shape == ref.shape
        assert np.array_equal(got, ref)
    names = ("train_labels", "train_mask", "valid_labels", "valid_mask", "test_labels", "test_mask")
    for got, name in zip([a for pair in split for a in pair], names):
        ref = GOLD["cora_" + name]
        assert got.dtype == ref.dtype and np.array_equal(got, ref), name
    assert graph.toarray().max() == 2.0                     # a citation in both directions keeps the value 2
    assert split[0][1].dtype == bool and split[0][0].dtype == np.int32


def test_cora_split_order_matches_reference_set_difference():
    from deep_recommenders.datasets import Cora
    cora = Cora(FIXTURE)
    _, _, labels = cora.load_content()
    np.random.seed(int(GOLD["cora_split_rest_seed"]))
    train = cora.sample_train_nodes(labels)
    rest = list(set(np.arange(labels.shape[0])) - set(train))
    assert np.array_equal(np.asarray(rest), GOLD["cora_split_rest_order"])


def test_cora_missing_files_raise(tmp_path):
    from deep_recommenders.datasets import Cora
    with pytest.raises(RuntimeError):
        Cora(str(tmp_path))


def test_synthetic_cora_round_trip(tmp_path):
    from deep_recommenders.datasets import Cora, write_synthetic_cora
    write_synthetic_cora(str(tmp_path / "a"), seed=3)
    write_synthetic_cora(str(tmp_path / "b"), seed=3)
    for f in ("cora.content", "cora.cites"):
        assert (tmp_path / "a" / "cora" / f).read_bytes() == (tmp_path / "b" / "cora" / f).read_bytes()
    cora = Cora(str(tmp_path / "a"))
    ids, features, labels = cora.load_content()
    assert features.shape == (2708, 1433) and len(set(ids)) == 2708
    assert np.allclose(np.asarray(features.sum(axis=1)).ravel(), 1.0)
    assert sorted(set(labels)) == sorted(cora._cora_classes)
    graph = cora.build_graph(ids)
    assert (graph != graph.T).nnz == 0 and graph.diagonal().sum() == 0
    assert len(open(tmp_path / "a" / "cora" / "cora.cites").readlines()) == 5429
    cls = {c: i for i, c in enumerate(cora._cora_classes)}
    lab = np.array([cls[s] for s in labels])
    g = graph.tocoo()
    assert (lab[g.row] == lab[g.col]).mean() > 0.8            # planted: citations mostly stay within a class
    train, valid, test = cora.split_labels(labels)
    assert train[1].sum() == 140 and valid[1].sum() == 500 and test[1].sum() == 2708 - 640


def test_adjacency_validation():
    from deep_recommenders_b200.ops import CSRAdjacency
    good = (np.array([0, 1, 3]), np.array([1, 0, 2]), np.array([1.0, 2.0, 3.0]))
    a = CSRAdjacency(*good, (2, 3), device="cpu")
    assert a.nnz == 3 and a.values.dtype == torch.float32
    bad = [
        ((np.array([0, 2, 1]), good[1], good[2]), (2, 3)),            # indptr decreases
        ((np.array([1, 1, 3]), good[1], good[2]), (2, 3)),            # indptr[0] != 0
        ((np.array([0, 1, 2]), good[1], good[2]), (2, 3)),            # indptr[-1] != nnz
        ((good[0], np.array([1, 0, 3]), good[2]), (2, 3)),            # column index out of range
        ((good[0], np.array([1, -1, 2]), good[2]), (2, 3)),
        ((good[0], good[1], np.array([1, 2, 3])), (2, 3)),            # integer values
        ((good[0], good[1], np.array(["a", "b", "c"])), (2, 3)),      # non-numeric values
        ((np.array([0, 3]), good[1], good[2]), (2, 3)),               # indptr of the wrong length
    ]
    for args, shape in bad:
        with pytest.raises(ValueError):
            CSRAdjacency(*args, shape, device="cpu")


def test_adjacency_from_scipy_and_torch_and_transpose():
    import scipy.sparse as sp
    from deep_recommenders_b200.ops import CSRAdjacency
    m = sp.random(9, 13, density=0.3, random_state=7, format="csr", dtype=np.float64)
    a = CSRAdjacency.from_any(m, device="cpu")
    at = m.T.tocsr()                                          # rows of A^T in ascending original row
    assert np.array_equal(a.t_indptr.numpy(), at.indptr) and np.array_equal(a.t_indices.numpy(), at.indices)
    assert np.array_equal(a.t_values.numpy(), at.data.astype(np.float32))
    dense = torch.from_numpy(m.toarray())
    for t in (dense.to_sparse_coo(), dense.to_sparse_csr()):
        b = CSRAdjacency.from_any(t, device="cpu")
        assert np.array_equal(b.indptr.numpy(), m.indptr) and np.array_equal(b.indices.numpy(), m.indices)
    with pytest.raises(ValueError):
        CSRAdjacency.from_any(dense, device="cpu")


def test_gcn_layer_validation_and_config():
    from deep_recommenders.keras.models.retrieval import GCN
    with pytest.raises(ValueError):
        GCN(4, activation="elu")
    layer = GCN(4, residual=True)
    with pytest.raises(ValueError):
        layer.build((10, 5))                                  # units != F with a residual
    g = GCN(7, residual=True, use_bias=True, activation="softmax", kernel_regularizer="l2", name="g")
    cfg = g.get_config()
    assert set(cfg) >= {"units", "use_bias", "activation", "kernel_initializer", "kernel_regularizer",
                        "bias_initializer", "bias_regularizer", "residual"}
    assert cfg["kernel_initializer"]["class_name"] == "TruncatedNormal" and cfg["residual"] is True
    assert GCN.from_config(cfg).get_config() == cfg


def _fixed_model(pred):
    from deep_recommenders.keras.layers import Model

    class M(Model):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(()))
            self.built = True

        def call(self, x, **kwargs):
            return torch.as_tensor(pred) + 0 * self.p

    return M()


def test_engine_weighted_loss_and_accuracy():
    from deep_recommenders_b200.keras.engine import categorical_crossentropy
    rng = np.random.default_rng(9)
    n, k = 11, 4
    pred = torch.softmax(torch.from_numpy(rng.standard_normal((n, k)).astype(np.float32)), -1)
    y = np.eye(k, dtype=np.float32)[rng.integers(0, k, n)]
    w = (rng.random(n) < 0.5).astype(np.float32)
    w[0] = 1.0
    m = _fixed_model(pred)
    m.compile(loss="categorical_crossentropy", weighted_metrics=["acc"])
    logs = m.evaluate(None, y, sample_weight=w, batch_size=n)
    per = categorical_crossentropy(torch.from_numpy(y), pred).double().numpy()
    assert logs["loss"] == pytest.approx(float((per * w).sum() / n), rel=1e-6)         # SUM_OVER_BATCH_SIZE
    correct = pred.numpy().argmax(1) == y.argmax(1)
    assert logs["acc"] == pytest.approx(float((w * correct).sum()) / float(w.sum()), rel=1e-12)
    assert m.evaluate(None, y)["acc"] == pytest.approx(float(correct.mean()), rel=1e-12)
    with pytest.raises(NotImplementedError):
        m.evaluate(None, y, batch_size=n - 1)
    with pytest.raises(NotImplementedError):
        m.fit(None, y, batch_size=5)
    hist = m.fit(None, y, sample_weight=w, validation_data=(None, y, w), epochs=2, batch_size=n, shuffle=False)
    assert hist["val_acc"][0] == pytest.approx(logs["acc"]) and hist["val_loss"][0] == pytest.approx(logs["loss"])
    assert hist["loss"][0] == pytest.approx(logs["loss"], rel=1e-6)
    # the batch forms keep their meaning: evaluate(data, steps) and fit over an iterable with validation batches
    assert m.evaluate([(None, y)] * 3, 2)["loss"] == pytest.approx(float(per.mean()), rel=1e-6)
    h2 = m.fit([(None, y)] * 4, epochs=2, steps_per_epoch=2, validation_data=[(None, y)], validation_steps=1)
    assert len(h2["loss"]) == 2 and "val_loss" in h2 and "val_acc" in h2
    with pytest.raises(ValueError):
        m.compile(weighted_metrics=["auc"])
