"""FNN without a GPU: the float64 oracle against the reference's own fnn.py (tests/golden/fnn_golden.npz), the
FM.export file format, and every construction error of ranking.FNN, raised before anything touches CUDA."""
import os

import numpy as np
import pytest
import torch

import fnn_oracle as O
from deep_recommenders_b200 import _lib
from deep_recommenders_b200 import feature_column as fc
from deep_recommenders_b200.estimator.models.feature_interaction.fm import FM
from deep_recommenders_b200.estimator.models.ranking import fnn as fnn_mod
from deep_recommenders_b200.estimator.models.ranking import FNN

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fnn_golden.npz")


def golden_cases():
    z = np.load(GOLDEN)
    out = []
    for k in range(int(z["n_cases"])):
        p = f"c{k}_"
        S = int(z[p + "S"])
        case = {"B": int(z[p + "B"]), "S": S, "D": int(z[p + "D"]),
                "rows": [int(z[f"{p}rows{s}"]) for s in range(S)],
                "ids": [z[f"{p}ids{s}"] for s in range(S)],
                "tables": [z[f"{p}table{s}"] for s in range(S)],
                "lins": [z[f"{p}lin{s}"] for s in range(S)],
                "bias": z[p + "bias"],
                "ws": [z[f"{p}k{i}"] for i in range(int(z[p + "nlayers"]))],
                "bs": [z[f"{p}b{i}"] for i in range(int(z[p + "nlayers"]))],
                "x": z[p + "x"], "out": z[p + "out"]}
        out.append(case)
    return out


@pytest.mark.parametrize("k", [0, 1])
def test_oracle_matches_reference_golden(k):
    c = golden_cases()[k]
    per_slot = [[[i] for i in ids] for ids in c["ids"]]
    state = {kk: c[kk] for kk in ("tables", "lins", "bias", "ws", "bs")}
    x, hs, p = O.forward(state, per_slot)
    np.testing.assert_allclose(x, c["x"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(p, c["out"].reshape(-1), rtol=1e-12, atol=1e-12)
    # the padded layout carries the same function: zero columns against zero kernel rows
    S, D = c["S"], c["D"]
    xp = O.pad_row(x, S, D)
    P, ld = O.layout(S, D)
    assert ld % 4 == 0 and P % 4 == 0 and ld == P + S * D
    assert np.all(xp[:, 1 + S:P] == 0)
    np.testing.assert_array_equal(O.unpad_row(xp, S, D), x)
    np.testing.assert_allclose(xp @ O.pad_kernel(c["ws"][0], S, D), x @ c["ws"][0], rtol=1e-12, atol=1e-12)


def test_oracle_gradients_match_finite_differences():
    c = golden_cases()[1]
    rng = np.random.default_rng(0)
    per_slot = [[[i] for i in ids] for ids in c["ids"]]
    per_slot[0][0] = [0, 2, -1, 2]       # a bag with a pruned id and a duplicate
    per_slot[1][1] = []                  # an empty bag
    state = {kk: [np.array(v, dtype=np.float64) for v in c[kk]] for kk in ("tables", "lins", "ws", "bs")}
    state["bias"] = c["bias"]
    y = rng.integers(0, 2, c["B"]).astype(np.float64)
    _, _, gt, gl, gws, gbs = O.grads(state, per_slot, y)
    h = 1e-6
    for name, idx, g in (("tables", (0, 2, 3), gt[0][2, 3]), ("lins", (0, 2), gl[0][2]), ("lins", (1, 0), gl[1][0]),
                         ("ws", (0, 1 + c["S"] + 5, 2), gws[0][1 + c["S"] + 5, 2]), ("bs", (1, 0), gbs[1][0])):
        arr = state[name][idx[0]]
        old = arr[idx[1:]]
        arr[idx[1:]] = old + h
        lp = O.log_loss(O.forward(state, per_slot)[2], y)
        arr[idx[1:]] = old - h
        lm = O.log_loss(O.forward(state, per_slot)[2], y)
        arr[idx[1:]] = old
        assert abs((lp - lm) / (2 * h) - g) < 1e-6 * max(1.0, abs(g)), (name, idx)


def _fm(rows=(5, 3, 7), D=8, device="cpu"):
    cols = [fc.categorical_column_with_identity(f"f{s}", n) for s, n in enumerate(rows)]
    return cols, FM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols], seed=3,
                    device=device)


def test_fm_export_round_trip(tmp_path):
    cols, fm = _fm()
    coll = fm.collection
    with torch.no_grad():
        coll.lin_view().copy_(torch.randn(coll.total_rows))
        coll.bias.fill_(0.25)
    path = tmp_path / "fm.pt"
    fm.export(path)
    state = torch.load(path, weights_only=True)
    assert state["format"] == 1
    assert state["bias"].shape == (1,) and float(state["bias"][0]) == 0.25
    assert sorted(state["linear"]) == sorted(state["factorized"]) == ["f0", "f1", "f2"]
    for s, c in enumerate(cols):
        lin, emb = state["linear"][c.key], state["factorized"][c.key]
        assert lin.shape == (c.num_buckets, 1) and emb.shape == (c.num_buckets, 8)
        assert lin.device.type == "cpu" and emb.is_contiguous()
        assert torch.equal(lin[:, 0], coll.linear_of(s).detach())
        assert torch.equal(emb, coll.table(s).detach())
    # a copy: changing the model afterwards leaves the file's tensors alone
    with torch.no_grad():
        coll.weight.add_(1.0)
    assert not torch.equal(state["factorized"]["f0"], coll.table(0).detach())


@pytest.fixture
def no_cuda(monkeypatch):
    """Fail loudly if FNN's constructor reaches the library or builds its tables."""
    def boom(*a, **k):
        raise AssertionError("FNN touched CUDA before validating its arguments")
    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(fnn_mod, "EmbeddingCollection", boom)


@pytest.fixture
def export(tmp_path):
    _, fm = _fm()
    path = tmp_path / "fm.pt"
    fm.export(path)
    return path


def _cols(rows=(5, 3, 7), D=8, combiner="mean"):
    cols = [fc.categorical_column_with_identity(f"f{s}", n) for s, n in enumerate(rows)]
    return [fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D, combiner=combiner) for c in cols]


@pytest.mark.parametrize("kw", [{"dnn_batch_normalization": True}, {"dnn_dropout": 0.5}])
def test_tower_options_not_served(no_cuda, export, kw):
    ind, emb = _cols()
    with pytest.raises(NotImplementedError):
        FNN(ind, emb, export, [8], device="cuda", **kw)


def test_column_lists_must_match(no_cuda, export):
    ind, emb = _cols()
    with pytest.raises(NotImplementedError, match="same order"):
        FNN(ind[::-1], emb, export, [8], device="cuda")
    with pytest.raises(NotImplementedError, match="same order"):
        FNN(ind[:2], emb, export, [8], device="cuda")


def test_combiner_mean_only(no_cuda, export):
    ind, emb = _cols(combiner="sqrtn")
    with pytest.raises(NotImplementedError, match="combiner"):
        FNN(ind, emb, export, [8], device="cuda")


def test_bad_export_files(no_cuda, export, tmp_path):
    ind, emb = _cols()
    state = torch.load(export, weights_only=True)

    def write(st):
        p = tmp_path / "bad.pt"
        torch.save(st, p)
        return p

    missing = {**state, "linear": {k: v for k, v in state["linear"].items() if k != "f1"}}
    with pytest.raises(ValueError, match="f1"):
        FNN(ind, emb, write(missing), [8], device="cuda")
    ind2, emb2 = _cols(rows=(5, 4, 7))
    with pytest.raises(ValueError, match="buckets|needs"):
        FNN(ind2, emb2, export, [8], device="cuda")
    ind3, emb3 = _cols(D=16)
    with pytest.raises(ValueError, match="dimension"):
        FNN(ind3, emb3, export, [8], device="cuda")
    with pytest.raises(ValueError, match="format"):
        FNN(ind, emb, write({**state, "format": 2}), [8], device="cuda")
    with pytest.raises(ValueError, match="format"):
        FNN(ind, emb, write([1, 2]), [8], device="cuda")
