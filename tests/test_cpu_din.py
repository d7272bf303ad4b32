"""CPU checks of the DIN port (no GPU): the float64 oracle against the golden vectors made by executing the reference's
din.py, the reference's known answers, the oracle's gradients against torch-CPU float64 autograd, the layers' errors
(raised before any CUDA call) and config round trips, and the C-ABI's host-side validation."""
import os

import numpy as np
import pytest
import torch

from din_oracle import activation_unit, dice, dice_grad, din_attention, din_attention_grad

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "din_golden.npz")


def _cases(g, pre, kind):
    return sorted({k[len(pre):-len("_x")] for k in g.files if k.startswith(pre + kind) and k.endswith("_x")})


@pytest.mark.parametrize("pre,dtype,tol", [("f64_", np.float64, 1e-12), ("f32_", np.float32, 2e-6)])
def test_oracle_reproduces_golden(pre, dtype, tol):
    g = np.load(GOLDEN)
    au = _cases(g, pre, "au_")
    assert len(au) == 9
    for c in au:
        k = pre + c
        bias = bool(g[k + "_bias"])
        act = str(g[k + "_act"])
        inter = str(g[k + "_inter"])
        layer_act = (lambda z, a=g[k + "_alpha"]: dice(z, a, 1e-8, dtype)) if act == "dice" else None
        out = activation_unit(g[k + "_x"], g[k + "_y"], g[k + "_w1"], g[k + "_b1"] if bias else None, g[k + "_w2"],
                              g[k + "_b2"] if bias else None, act, None if inter == "none" else inter, dtype,
                              layer_act)
        assert out.dtype == dtype
        ref = g[k + "_out"]
        np.testing.assert_allclose(out, ref, rtol=0, atol=tol * (1 + np.abs(ref).max()), err_msg=c)
    dc = _cases(g, pre, "dice_")
    assert len(dc) == 7
    for c in dc:
        k = pre + c
        y = dice(g[k + "_x"], g[k + "_alpha"], float(g[k + "_eps"]), dtype)
        np.testing.assert_allclose(y, g[k + "_y"], rtol=0, atol=tol * (1 + np.abs(g[k + "_y"]).max()), err_msg=c)


def test_reference_known_answers():
    """test_din.py:17-64 against the oracle."""
    rng = np.random.default_rng(0)
    x, y = rng.normal(size=(3, 5)), rng.normal(size=(3, 5))
    relu = lambda z: np.maximum(z, 0)
    out = activation_unit(x, y, np.ones((10, 10)), np.zeros(10), np.ones((10, 1)), np.zeros(1), "relu")
    np.testing.assert_allclose(out, relu(np.concatenate([x, y], 1) @ np.ones((10, 10))).sum(1, keepdims=True))
    out = activation_unit(x, y, np.ones((15, 10)), np.zeros(10), np.ones((10, 1)), np.zeros(1), "relu", "subtract")
    np.testing.assert_allclose(out, relu(np.concatenate([x, y, x - y], 1) @ np.ones((15, 10))).sum(1, keepdims=True))
    inputs = np.asarray([[-0.2, -0.1, 0.1, 0.2]])
    for eps in (1e-7, 1e-8, 1e-9, 1e-10):
        p = 1 / (1 + np.exp(-((inputs - inputs.mean()) / np.sqrt(inputs.std() + eps))))
        xx = np.where(inputs > 0, inputs, 0)
        np.testing.assert_allclose(dice(inputs, np.zeros(4), eps), np.where(xx > 0, p * xx, (1 - p) * xx))


def test_dice_branch_tests_the_prelu_output():
    """With a negative alpha a negative x has a positive PReLU output and takes the p*a branch."""
    x = np.asarray([[-1.0, 0.5, 2.0]])
    alpha = np.asarray([-0.5, 0.0, 0.0])
    mu, sd = x.mean(), x.std()
    p = 1 / (1 + np.exp(-((x - mu) / np.sqrt(sd + 1e-8))))
    a = np.where(x > 0, x, alpha * x)
    np.testing.assert_allclose(dice(x, alpha), p * a)


_TACT = {"linear": lambda v: v, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


@pytest.mark.parametrize("act", list(_TACT))
@pytest.mark.parametrize("inter", [None, "subtract", "multiply"])
def test_attention_grad_matches_torch_autograd(act, inter):
    rng = np.random.default_rng(3)
    B, T, D, U = 4, 6, 5, 7
    keys, q = rng.standard_normal((B, T, D)), rng.standard_normal((B, D))
    w1 = rng.standard_normal(((3 if inter else 2) * D, U)) * 0.5
    b1, w2, b2 = rng.standard_normal(U), rng.standard_normal((U, 1)), rng.standard_normal(1)
    gp, gs = rng.standard_normal((B, D)), rng.standard_normal((B, T))
    t = {k: torch.tensor(v, requires_grad=True) for k, v in dict(k=keys, q=q, w1=w1, b1=b1, w2=w2, b2=b2).items()}
    qb = t["q"][:, None, :].expand(B, T, D)
    parts = [t["k"], qb] + ([] if inter is None else [t["k"] - qb if inter == "subtract" else t["k"] * qb])
    score = _TACT[act](torch.cat(parts, -1) @ t["w1"] + t["b1"]) @ t["w2"][:, 0] + t["b2"]
    pooled = (score[..., None] * t["k"]).sum(1)
    ((pooled * torch.tensor(gp)).sum() + (score * torch.tensor(gs)).sum()).backward()
    p, s, _ = din_attention(keys, q, w1, b1, w2, b2, act, inter)
    np.testing.assert_allclose(p, pooled.detach().numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(s, score.detach().numpy(), rtol=1e-12, atol=1e-12)
    got = din_attention_grad(keys, q, w1, b1, w2, b2, gp, gs, act, inter)
    for g, n in zip(got, ("k", "q", "w1", "b1", "w2", "b2")):
        np.testing.assert_allclose(g, t[n].grad.numpy(), rtol=1e-10, atol=1e-11, err_msg=n)


def test_dice_grad_matches_torch_autograd():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((6, 9))
    x[1, :4] = 0.0
    alpha = rng.standard_normal(9) * 0.5
    gy = rng.standard_normal((6, 9))
    tx, ta = torch.tensor(x, requires_grad=True), torch.tensor(alpha, requires_grad=True)
    mu = tx.mean(1, keepdim=True)
    sd = ((tx - mu) ** 2).mean(1, keepdim=True).sqrt()
    p = torch.sigmoid((tx - mu) / torch.sqrt(sd + 1e-8))
    a = torch.relu(tx) - ta * torch.relu(-tx)                # TensorFlow's PReLU
    y = torch.where(a > 0, p * a, (1 - p) * a)
    (y * torch.tensor(gy)).sum().backward()
    np.testing.assert_allclose(dice(x, alpha), y.detach().numpy(), rtol=1e-12)
    gx, ga = dice_grad(x, alpha, gy)
    np.testing.assert_allclose(gx, tx.grad.numpy(), rtol=1e-9, atol=1e-11)
    np.testing.assert_allclose(ga, ta.grad.numpy(), rtol=1e-9, atol=1e-11)
    # a constant row: no gradient through the std (autodiff of sqrt at 0 is NaN), the rest is finite
    c = np.full((2, 5), 0.3)
    gxc, _ = dice_grad(c, np.full(5, -0.2), np.ones((2, 5)))
    assert np.all(np.isfinite(gxc))


def test_layer_errors_before_any_cuda_call(monkeypatch):
    from deep_recommenders_b200 import _lib
    from deep_recommenders.keras.models.ranking import din
    from deep_recommenders.keras.layers import DIN
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    monkeypatch.setattr(_lib, "load", lambda: pytest.fail("C-ABI reached"))
    with pytest.raises(ValueError, match="rank-2"):
        din.Dice()(np.zeros((2, 3, 4), np.float32))
    with pytest.raises(ValueError, match="call_pooled"):
        din.ActivationUnit(4, activation=din.Dice()).call_pooled(torch.zeros((2, 3, 4)), torch.zeros((2, 4)))
    with pytest.raises(ValueError, match="unsupported activation"):
        din.ActivationUnit(4, activation="softmax")
    with pytest.raises(ValueError, match="multiple of 4"):
        DIN(item_rows=10, dim=5, device="cpu")
    with pytest.raises(ValueError, match="interacter"):
        DIN(item_rows=10, dim=8, interacter="concat", device="cpu")


def test_config_keys_and_round_trip():
    from deep_recommenders.keras.models.ranking import din
    from deep_recommenders.keras.layers import Multiply, Subtract
    g = np.load(GOLDEN)
    au_keys = {str(k) for k in g["f64_au_config_keys"]}
    dice_keys = {str(k) for k in g["f64_dice_config_keys"]}
    for unit in (din.ActivationUnit(8, interacter=Subtract(), kernel_regu="l2"),
                 din.ActivationUnit(8, interacter=Multiply(), use_bias=False, activation="sigmoid"),
                 din.ActivationUnit(8, activation=din.Dice(epsilon=1e-6)),
                 din.ActivationUnit(8, activation=None)):
        cfg = unit.get_config()
        assert au_keys <= set(cfg)
        again = din.ActivationUnit.from_config(cfg)
        assert again.get_config() == cfg
        assert again._fused == unit._fused and again._interact == unit._interact
    assert din.ActivationUnit(8, activation=None).get_config()["activation"] == "linear"
    d = din.Dice(epsilon=1e-6, alpha_regularizer="l2")
    cfg = d.get_config()
    assert dice_keys <= set(cfg)
    assert din.Dice.from_config(cfg).get_config() == cfg


def test_dice_alpha_is_created_in_build():
    from deep_recommenders.keras.models.ranking import din
    d = din.Dice(alpha_initializer="ones", alpha_regularizer="l1")
    assert d.alpha is None and d.losses == []
    d.build((None, 6), device="cpu")
    assert tuple(d.alpha.shape) == (6,) and float(d.alpha.detach().sum()) == 6.0
    assert len(d.losses) == 1


def test_mse_loss_registered():
    from deep_recommenders_b200.keras import engine
    yt, yp = torch.tensor([[1.0], [2.0]]), torch.tensor([[1.5], [1.0]])
    np.testing.assert_allclose(engine._LOSSES["mse"](yt, yp).numpy(), [0.25, 1.0])


def test_reference_import_paths():
    from deep_recommenders.keras.models.ranking import din
    from deep_recommenders.keras.layers import ActivationUnit, DIN, Dice, Multiply, Subtract
    assert din.ActivationUnit is ActivationUnit and din.Dice is Dice and din.DIN is DIN
    assert Subtract()([torch.ones(2), torch.ones(2)]).sum() == 0 and Multiply()([torch.ones(2), 2 * torch.ones(2)]).sum() == 4


def test_c_abi_host_validation(lib):
    p = 256
    #            keys query w1 b1 w2 b2  B  T  D  U inter act score pooled stream
    assert lib.dr_din_attn_fwd(None, p, p, None, p, None, 4, 3, 8, 6, 1, 1, p, None, None) == -1
    assert b"null pointer" in lib.dr_last_error()
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 8, 6, 1, 1, None, None, None) == -1   # no output
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, -1, 3, 8, 6, 1, 1, p, None, None) == -1
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 0, 8, 6, 1, 1, p, None, None) == -1
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 0, 6, 1, 1, p, None, None) == -1
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 8, 6, 3, 1, p, None, None) == -1
    assert b"interaction" in lib.dr_last_error()
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 8, 6, 1, 9, p, None, None) == -1
    assert b"activation" in lib.dr_last_error()
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 129, 6, 1, 1, p, None, None) == -3
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 4, 3, 8, 257, 1, 1, p, None, None) == -3
    assert lib.dr_din_attn_fwd(p, p, p, None, p, None, 1 << 21, 1 << 10, 8, 6, 1, 1, p, None, None) == -3
    assert lib.dr_din_attn_fwd(None, None, p, None, p, None, 0, 3, 8, 6, 1, 1, None, None, None) == 0   # B = 0
    # backward: keys query w1 b1 w2 b2 g_pooled g_score B T D U inter act g_keys g_query gw1 gb1 gw2 gb2 stream
    assert lib.dr_din_attn_bwd(p, p, p, None, p, None, None, None, 4, 3, 8, 6, 1, 1, p, p, p, None, p, None,
                               None) == -1
    assert b"both NULL" in lib.dr_last_error()
    assert lib.dr_din_attn_bwd(p, p, p, p, p, None, p, None, 4, 3, 8, 6, 1, 1, p, p, p, None, p, None, None) == -1
    assert b"bias gradient" in lib.dr_last_error()
    assert lib.dr_din_attn_bwd(p, p, p, None, p, None, p, None, 4, 3, 8, 6, 1, 1, None, p, p, None, p, None,
                               None) == -1
    assert lib.dr_din_attn_bwd(p, p, p, None, p, None, p, None, 4, 3, 128, 300, 1, 1, p, p, p, None, p, None,
                               None) == -3
    assert lib.dr_din_attn_bwd(p, p, p, None, p, None, p, None, 4, 3, 200, 6, 2, 0, p, p, p, None, p, None,
                               None) == -3
    # Dice
    assert lib.dr_dice_fwd(p, None, 4, 3, 1e-8, p, None) == -1
    assert lib.dr_dice_fwd(p, p, -1, 3, 1e-8, p, None) == -1
    assert lib.dr_dice_fwd(p, p, 4, 0, 1e-8, p, None) == -1
    assert lib.dr_dice_fwd(None, p, 0, 3, 1e-8, None, None) == 0
    assert lib.dr_dice_bwd(p, p, None, 4, 3, 1e-8, p, p, None) == -1
    assert lib.dr_dice_bwd(p, p, p, 4, 9000, 1e-8, p, p, None) == -3
