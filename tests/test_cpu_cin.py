"""CPU checks of the CIN port (no GPU): the float64 oracle against the golden vectors made by executing the reference's
xdeepfm.py, the reference's known answers, the oracle's gradient against torch-CPU float64 autograd, the reference's
ValueError messages (raised before any CUDA call) and the C-ABI's host-side validation."""
import os

import numpy as np
import pytest
import torch

from cin_oracle import cin, cin_grad

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cin_golden.npz")


def _cases(g, pre):
    return sorted({k[len(pre):-len("_x0")] for k in g.files if k.startswith(pre) and k.endswith("_x0")})


@pytest.mark.parametrize("pre,dtype,tol", [("f64_", np.float64, 1e-12), ("f32_", np.float32, 1e-6)])
def test_oracle_reproduces_golden(pre, dtype, tol):
    g = np.load(GOLDEN)
    cases = _cases(g, pre)
    assert len(cases) == 7
    for c in cases:
        b = g[f"{pre}{c}_bias"] if f"{pre}{c}_bias" in g.files else None
        y = cin(g[f"{pre}{c}_x0"], g[f"{pre}{c}_x"], g[f"{pre}{c}_kernel"], b, str(g[f"{pre}{c}_act"]), dtype)
        assert y.dtype == dtype
        np.testing.assert_allclose(y, g[f"{pre}{c}_y"], rtol=0, atol=tol, err_msg=c)


def test_reference_known_answers():
    x = np.asarray([[[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]]])
    w = np.ones((1, 4, 2))
    np.testing.assert_allclose(cin(x, x, w, None, "relu"), [[[0.25, 0.49, 0.81]] * 2], rtol=1e-12)
    np.testing.assert_allclose(cin(x, x, w, np.ones(2), "relu"), [[[1.25, 1.49, 1.81]] * 2], rtol=1e-12)


@pytest.mark.parametrize("act", ["linear", "relu", "sigmoid", "tanh"])
@pytest.mark.parametrize("same", [False, True])
def test_cin_grad_matches_torch_autograd(act, same):
    rng = np.random.default_rng(4)
    B, m, h, D, H = 5, 4, 3 if not same else 4, 3, 6
    x0 = rng.standard_normal((B, m, D))
    x = x0 if same else rng.standard_normal((B, h, D))
    w, b = rng.standard_normal((1, m * h, H)), rng.standard_normal(H)
    gy, gp = rng.standard_normal((B, H, D)), rng.standard_normal((B, H))
    tx0 = torch.tensor(x0, requires_grad=True)
    tx = tx0 if same else torch.tensor(x, requires_grad=True)
    tw, tb = torch.tensor(w, requires_grad=True), torch.tensor(b, requires_grad=True)
    z = torch.einsum("bid,bjd,ijk->bkd", tx0, tx, tw.view(m, h, H)) + tb[None, :, None]
    y = {"linear": lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}[act](z)
    ((y * torch.tensor(gy)).sum() + (y.sum(2) * torch.tensor(gp)).sum()).backward()
    gx0, gx, gw, gb, _ = cin_grad(x0, x, w, y.detach().numpy(), gy, gp, act)
    np.testing.assert_allclose(cin(x0, x, w, b, act), y.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gx0 + gx if same else gx0, tx0.grad.numpy(), rtol=1e-10, atol=1e-12)
    if not same:
        np.testing.assert_allclose(gx, tx.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gw, tw.grad.numpy(), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gb, tb.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_value_errors_before_any_cuda_call(monkeypatch):
    from deep_recommenders_b200 import _lib
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    monkeypatch.setattr(_lib, "load", lambda: pytest.fail("C-ABI reached"))
    errs = [str(e) for e in np.load(GOLDEN)["f64_errors"]]
    with pytest.raises(ValueError, match=r"`CIN` layer's inputs type should be `tuple`.") as e:
        CIN(feature_map=3)(np.random.normal(size=(2, 3, 5)).astype(np.float32))
    assert str(e.value).split("`<")[0] == errs[0].split("`<")[0]
    with pytest.raises(ValueError) as e:
        CIN(feature_map=3).build(((2, 3, 5),) * 3)
    assert str(e.value) == errs[1]
    inputs = np.random.normal(size=(2, 15)).astype(np.float32)
    with pytest.raises(ValueError) as e:
        CIN(feature_map=3)((inputs, inputs))
    assert str(e.value) == errs[2]


def test_config_keys_and_round_trip():
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    keys = {str(k) for k in np.load(GOLDEN)["f64_config_keys"]}
    layer = CIN(feature_map=5, use_bias=True, activation="relu", kernel_regu="l2")
    cfg = layer.get_config()
    assert keys <= set(cfg)
    assert CIN.from_config(cfg).get_config() == cfg
    assert CIN(activation=None).get_config()["activation"] == "linear"
    with pytest.raises(ValueError):
        CIN(activation="softmax")


def test_kernel_shape_and_regularizer():
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    layer = CIN(feature_map=4, use_bias=True, kernel_regu="l2", bias_regu="l1")
    layer.build(((None, 3, 2), (None, 5, 2)), device="cpu")
    assert tuple(layer.kernel.shape) == (1, 15, 4) and tuple(layer.bias.shape) == (4,)
    assert len(layer.losses) == 2


def test_c_abi_host_validation(lib):
    p = 256
    assert lib.dr_cin_fwd(None, p, p, None, 4, 2, 2, 3, 2, 0, p, None, None) == -1
    assert b"null pointer" in lib.dr_last_error()
    assert lib.dr_cin_fwd(p, p, p, None, -1, 2, 2, 3, 2, 0, p, None, None) == -1
    assert lib.dr_cin_fwd(p, p, p, None, 4, 0, 2, 3, 2, 0, p, None, None) == -1
    assert lib.dr_cin_fwd(p, p, p, None, 4, 2, 2, 3, 2, 9, p, None, None) == -1
    assert b"activation" in lib.dr_last_error()
    assert lib.dr_cin_fwd(p, p, p, None, 4, 2, 2, 200, 2, 0, p, None, None) == -3
    assert lib.dr_cin_bwd(p, p, p, p, None, None, 4, 2, 2, 3, 2, 0, 0, p, p, p, p, None, None) == -1
    assert b"both NULL" in lib.dr_last_error()
    assert lib.dr_cin_bwd(p, p, p, p, p, None, 4, 2, 2, 3, 2, 0, 0, p, p, None, p, None, None) == -1
    assert lib.dr_cin_bwd(p, 512, p, p, p, None, 4, 2, 2, 3, 2, 0, 1, p, p, None, p, None, None) == -1
    assert b"x_is_x0" in lib.dr_last_error()


def test_no_fm_flag_refused_by_sharded_entries(lib):
    """DR_EMBED_NO_FM (2) is served by dr_embed_fm_fwd / _bwd only: the row-sharded entries return DR_ENOTSUP."""
    assert lib.dr_embed_fm_fwd_sharded(None, 1, None, None, None, 8, None, 4, 2, 16, 16, 2, 0, None, None, None,
                                       None) == -3
    assert b"DR_EMBED_NO_FM" in lib.dr_last_error()
    assert lib.dr_embed_fm_bwd_sharded(None, 1, None, None, None, 8, None, None, None, None, 4, 2, 16, 16, 2, 0, None,
                                       1.0, None) == -3


def test_xdeepfm_oracle_linear_unit_and_oov():
    """The oracle's linear unit is bias + the first-order weights of in-range ids; an OOV id contributes nothing."""
    from cin_oracle import xdeepfm_forward
    rng = np.random.default_rng(0)
    tables = [rng.standard_normal((5, 4)) for _ in range(3)]
    lins = [rng.standard_normal(5) for _ in range(3)]
    ids = np.array([[0, 1, 2], [-1, 5, 4]])
    zero_head = np.zeros((3 + 2 + 6, 1))
    _, logit = xdeepfm_forward(tables, lins, 0.5, ids, [rng.standard_normal((1, 9, 3)), rng.standard_normal((1, 9, 2))],
                               "sigmoid", [rng.standard_normal((12, 6))], [np.zeros(6)], "relu", zero_head, [0.0])
    np.testing.assert_allclose(logit, [0.5 + lins[0][0] + lins[1][1] + lins[2][2], 0.5 + lins[2][4]])
