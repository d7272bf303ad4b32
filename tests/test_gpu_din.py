"""GPU tests of DIN's kernels (dr_din_attn_fwd / _bwd, dr_dice_fwd / _bwd), its layers and the DIN model.

Every fp32 result must sit within 1e-5 x (sum of |terms|) of a float64 reference; outputs are written between sentinel
guards so a store outside the output is caught."""
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

from din_oracle import activation_unit, dice, dice_grad, din_forward

pytestmark = pytest.mark.gpu
ACTS = {"linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3}
INTER = {"none": 0, "subtract": 1, "multiply": 2}
SENT = 1234.5
PAD = 4099


def _lib():
    from deep_recommenders_b200 import _lib
    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n):
    full = torch.full((n + 2 * PAD,), SENT, device="cuda", dtype=torch.float32)
    return full, full[PAD:PAD + n]


def _check_guards(full, n):
    f = full.cpu().numpy()
    assert np.all(f[:PAD] == SENT) and np.all(f[PAD + n:] == SENT), "store outside the output"


def _t64(a):
    return None if a is None else torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(
        "cuda", torch.float64)


def _close(got, ref, scale, rel=1e-5, what=""):
    got, ref, scale = _t64(got), _t64(ref), _t64(scale)
    err = (got - ref).abs()
    bound = rel * scale + 4.8e-7 * ref.abs() + 1e-30
    bad = err > bound
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} elements out of bound; worst err {err.max().item():.3g} "
                                 f"vs bound {bound[bad].min().item():.3g}")


_ACT64 = {"linear": lambda z: z, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


def _actp(h, act):
    return {"relu": lambda v: (v > 0).double(), "sigmoid": lambda v: v * (1 - v), "tanh": lambda v: 1 - v * v,
            "linear": torch.ones_like}[act](h)


def ref64(keys, q, w1, b1, w2, b2, act, inter, gp=None, gs=None):
    """float64 forward and backward on the GPU with the sums of |terms| each fp32 result is measured against."""
    k, q, w1, w2 = _t64(keys), _t64(q), _t64(w1), _t64(w2).reshape(-1)
    b1, b2 = _t64(b1), _t64(b2)
    B, T, D = k.shape
    qb = q[:, None, :].expand_as(k)
    f = {"none": None, "subtract": k - qb, "multiply": k * qb}[inter]
    u = torch.cat([k, qb] + ([] if f is None else [f]), -1)
    ua = u.abs()
    z = u @ w1 + (0 if b1 is None else b1)
    za = ua @ w1.abs() + (0 if b1 is None else b1.abs())
    h = _ACT64[act](z)
    score = h @ w2 + (0 if b2 is None else b2.reshape(()))
    pooled = (score[..., None] * k).sum(1)
    sa = za @ w2.abs() + h.abs() @ w2.abs() + (0 if b2 is None else b2.abs().reshape(()))
    pa = ((sa + score.abs())[..., None] * k.abs()).sum(1)
    out = dict(score=score, pooled=pooled, score_abs=sa, pooled_abs=pa)
    if gp is None and gs is None:
        return out
    gp, gs = _t64(gp), _t64(gs)
    ds = torch.zeros_like(score)
    dsa = torch.zeros_like(score)
    gk = torch.zeros_like(k)
    gka = torch.zeros_like(k)
    if gs is not None:
        ds, dsa = ds + gs, dsa + gs.abs()
    if gp is not None:
        ds = ds + torch.einsum("btd,bd->bt", k, gp)
        dsa = dsa + torch.einsum("btd,bd->bt", k.abs(), gp.abs())
        gk = gk + score[..., None] * gp[:, None, :]
        gka = gka + (sa + score.abs())[..., None] * gp.abs()[:, None, :]
    ap = _actp(h, act)
    apa = ap.abs()
    if act == "relu":
        apa = apa + (z.abs() <= 1e-5 * za).double()          # a sign the fp32 recompute may flip
    elif act in ("sigmoid", "tanh"):
        apa = apa + 0.05 * za
    gz = ds[..., None] * w2 * ap
    gza = dsa[..., None] * w2.abs() * apa
    gu, gua = gz @ w1.T, gza @ w1.abs().T
    gk, gka = gk + gu[..., :D], gka + gua[..., :D]
    gq, gqa = gu[..., D:2 * D].sum(1), gua[..., D:2 * D].sum(1)
    if inter == "subtract":
        gk, gka = gk + gu[..., 2 * D:], gka + gua[..., 2 * D:]
        gq, gqa = gq - gu[..., 2 * D:].sum(1), gqa + gua[..., 2 * D:].sum(1)
    elif inter == "multiply":
        gk, gka = gk + gu[..., 2 * D:] * qb, gka + gua[..., 2 * D:] * qb.abs()
        gq, gqa = gq + (gu[..., 2 * D:] * k).sum(1), gqa + (gua[..., 2 * D:] * k.abs()).sum(1)
    out.update(g_keys=gk, g_keys_abs=gka, g_query=gq, g_query_abs=gqa,
               gw1=torch.einsum("btk,btu->ku", u, gz), gw1_abs=torch.einsum("btk,btu->ku", ua, gza),
               gb1=gz.sum((0, 1)), gb1_abs=gza.sum((0, 1)),
               gw2=torch.einsum("btu,bt->u", h, ds), gw2_abs=torch.einsum("btu,bt->u", h.abs() + za, dsa),
               gb2=ds.sum().reshape(1), gb2_abs=dsa.sum().reshape(1))
    return out


def _ptr(t):
    return None if t is None else t.data_ptr()


def _rand(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _inputs(rng, B, T, D, U, inter, bias):
    keys = _rand(rng, B, T, D)
    keys[rng.random((B, T)) < 0.1] = 0.0                      # padded positions gather zero rows
    q = _rand(rng, B, D)
    w1 = _rand(rng, (3 if inter != "none" else 2) * D, U, scale=1.0 / np.sqrt(D))
    w2 = _rand(rng, U, 1, scale=1.0 / np.sqrt(U))
    b1 = _rand(rng, U) if bias else None
    b2 = _rand(rng, 1) if bias else None
    return keys, q, w1, b1, w2, b2


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def attn_fwd(keys, q, w1, b1, w2, b2, act, inter, want_score=True, want_pooled=True):
    B, T, D = keys.shape
    U = w1.shape[1]
    sfull, s = _guarded(B * T) if want_score else (None, None)
    pfull, p = _guarded(B * D) if want_pooled else (None, None)
    rc = _lib().dr_din_attn_fwd(keys.data_ptr(), q.data_ptr(), w1.data_ptr(), _ptr(b1), w2.data_ptr(), _ptr(b2),
                                B, T, D, U, INTER[inter], ACTS[act], _ptr(s), _ptr(p), _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    if want_score:
        _check_guards(sfull, B * T)
    if want_pooled:
        _check_guards(pfull, B * D)
    return (None if s is None else s.view(B, T)), (None if p is None else p.view(B, D))


def attn_bwd(keys, q, w1, b1, w2, b2, gp, gs, act, inter):
    B, T, D = keys.shape
    U = w1.shape[1]
    bufs = {n: _guarded(sz) for n, sz in (("g_keys", B * T * D), ("g_query", B * D), ("gw1", w1.numel()),
                                          ("gw2", U), ("gb1", U), ("gb2", 1))}
    if b1 is None:
        bufs["gb1"] = (None, None)
    if b2 is None:
        bufs["gb2"] = (None, None)
    v = {n: b[1] for n, b in bufs.items()}
    rc = _lib().dr_din_attn_bwd(keys.data_ptr(), q.data_ptr(), w1.data_ptr(), _ptr(b1), w2.data_ptr(), _ptr(b2),
                                _ptr(gp), _ptr(gs), B, T, D, U, INTER[inter], ACTS[act], v["g_keys"].data_ptr(),
                                v["g_query"].data_ptr(), v["gw1"].data_ptr(), _ptr(v["gb1"]), v["gw2"].data_ptr(),
                                _ptr(v["gb2"]), _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    for n, (full, t) in bufs.items():
        if full is not None:
            _check_guards(full, t.numel())
    return {"g_keys": v["g_keys"].view(B, T, D), "g_query": v["g_query"].view(B, D), "gw1": v["gw1"].view(w1.shape),
            "gw2": v["gw2"], "gb1": v["gb1"], "gb2": v["gb2"]}


# (B, T, D, U): tails on the 64-row chunk, the examples-per-CTA split (ceil(512 / T), at most 64), the 16-column
# groups of U (1, 36 -> 48, 256), D in {1, 5, 16, 32, 128} (D = 5: padded to 8), T = 1 (the layer's call), B = 0
FWD_CASES = [
    (1, 1, 1, 1), (5, 1, 5, 36), (3, 64, 16, 36), (7, 65, 32, 256), (300, 7, 5, 1), (37, 200, 128, 36),
    (129, 63, 32, 16), (2, 513, 16, 256), (0, 5, 4, 4), (1000, 1, 32, 36), (65, 9, 128, 256), (33, 50, 1, 17),
    (70, 8, 16, 100),
]


@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: "B{}T{}D{}U{}".format(*c))
@pytest.mark.parametrize("inter", list(INTER))
@pytest.mark.parametrize("act", list(ACTS))
def test_attn_fwd_matches_oracle(case, inter, act):
    B, T, D, U = case
    rng = np.random.default_rng(zlib.crc32(repr((case, inter, act)).encode()))
    bias = (B + U + len(act)) % 2 == 0
    keys, q, w1, b1, w2, b2 = _inputs(rng, B, T, D, U, inter, bias)
    s, p = attn_fwd(_dev(keys), _dev(q), _dev(w1), _dev(b1), _dev(w2), _dev(b2), act, inter)
    if B == 0:
        return
    r = ref64(keys, q, w1, b1, w2, b2, act, inter)
    _close(s, r["score"], r["score_abs"], what="score")
    _close(p, r["pooled"], r["pooled_abs"], what="pooled")
    # the score-only and pooled-only forms write the same bits
    s1, _ = attn_fwd(_dev(keys), _dev(q), _dev(w1), _dev(b1), _dev(w2), _dev(b2), act, inter, want_pooled=False)
    _, p1 = attn_fwd(_dev(keys), _dev(q), _dev(w1), _dev(b1), _dev(w2), _dev(b2), act, inter, want_score=False)
    assert torch.equal(s1, s) and torch.equal(p1, p)


BWD_CASES = [(1, 1, 1, 1), (5, 1, 5, 36), (7, 65, 32, 256), (300, 7, 5, 1), (37, 200, 128, 36), (129, 63, 32, 16),
             (65, 9, 128, 256), (1000, 1, 16, 36), (0, 3, 4, 4)]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "B{}T{}D{}U{}".format(*c))
@pytest.mark.parametrize("inter", list(INTER))
@pytest.mark.parametrize("grads", ["pooled", "score", "both"])
def test_attn_bwd_matches_oracle(case, inter, grads):
    B, T, D, U = case
    act = list(ACTS)[zlib.crc32(repr((case, inter, grads)).encode()) % 4]
    rng = np.random.default_rng(zlib.crc32(repr((case, inter, grads, "b")).encode()))
    bias = (B + T + len(grads)) % 2 == 1
    keys, q, w1, b1, w2, b2 = _inputs(rng, B, T, D, U, inter, bias)
    gp = _rand(rng, B, D) if grads in ("pooled", "both") else None
    gs = _rand(rng, B, T) if grads in ("score", "both") else None
    got = attn_bwd(_dev(keys), _dev(q), _dev(w1), _dev(b1), _dev(w2), _dev(b2), _dev(gp), _dev(gs), act, inter)
    if B == 0:
        assert not bool(got["gw1"].any()) and not bool(got["gw2"].any())
        return
    r = ref64(keys, q, w1, b1, w2, b2, act, inter, gp, gs)
    for n in ("g_keys", "g_query", "gw1", "gw2") + (("gb1", "gb2") if bias else ()):
        _close(got[n].reshape(r[n].shape), r[n], r[n + "_abs"], what=f"{n} ({act})")


@pytest.mark.parametrize("act", list(ACTS))
def test_attn_bwd_each_activation(act):
    """Every activation through the backward, on a multi-chunk case with bias and both gradients."""
    rng = np.random.default_rng(ACTS[act] + 100)
    keys, q, w1, b1, w2, b2 = _inputs(rng, 41, 77, 16, 36, "multiply", True)
    gp, gs = _rand(rng, 41, 16), _rand(rng, 41, 77)
    got = attn_bwd(_dev(keys), _dev(q), _dev(w1), _dev(b1), _dev(w2), _dev(b2), _dev(gp), _dev(gs), act, "multiply")
    r = ref64(keys, q, w1, b1, w2, b2, act, "multiply", gp, gs)
    for n in ("g_keys", "g_query", "gw1", "gw2", "gb1", "gb2"):
        _close(got[n].reshape(r[n].shape), r[n], r[n + "_abs"], what=n)


def test_attn_bit_identical_across_runs():
    rng = np.random.default_rng(9)
    keys, q, w1, b1, w2, b2 = _inputs(rng, 2000, 50, 32, 36, "subtract", True)
    gp, gs = _rand(rng, 2000, 32), _rand(rng, 2000, 50)
    a = [_dev(v) for v in (keys, q, w1, b1, w2, b2)]
    s1, p1 = attn_fwd(*a, "relu", "subtract")
    s2, p2 = attn_fwd(*a, "relu", "subtract")
    assert torch.equal(s1, s2) and torch.equal(p1, p2)
    g1 = attn_bwd(*a, _dev(gp), _dev(gs), "relu", "subtract")
    g2 = attn_bwd(*a, _dev(gp), _dev(gs), "relu", "subtract")
    assert torch.equal(g1["g_keys"], g2["g_keys"]) and torch.equal(g1["g_query"], g2["g_query"])


def test_zero_keys_get_no_gradient_through_score():
    """A padded position (zero key row) adds nothing to pooled; its g_keys is what the score path alone gives."""
    rng = np.random.default_rng(4)
    keys, q, w1, b1, w2, b2 = _inputs(rng, 16, 12, 8, 20, "subtract", True)
    keys[:, 6:] = 0.0
    a = [_dev(v) for v in (keys, q, w1, b1, w2, b2)]
    _, p_full = attn_fwd(*a, "relu", "subtract")
    a_short = [_dev(np.ascontiguousarray(keys[:, :6]))] + a[1:]
    _, p_short = attn_fwd(*a_short, "relu", "subtract")
    r = ref64(keys, q, w1, b1, w2, b2, "relu", "subtract")
    _close(p_full, p_short.double(), r["pooled_abs"], what="pooled with padding")


# ---- Dice ------------------------------------------------------------------------------------------------------------
def _dice_gpu(x, alpha, eps, gy=None):
    N, U = x.shape
    lib = _lib()
    xd, ad = _dev(x), _dev(alpha)
    yfull, y = _guarded(N * U)
    assert lib.dr_dice_fwd(xd.data_ptr(), ad.data_ptr(), N, U, eps, y.data_ptr(), _stream()) == 0, lib.dr_last_error()
    torch.cuda.synchronize()
    _check_guards(yfull, N * U)
    if gy is None:
        return y.view(N, U)
    gxfull, gx = _guarded(N * U)
    gafull, ga = _guarded(U)
    assert lib.dr_dice_bwd(xd.data_ptr(), ad.data_ptr(), _dev(gy).data_ptr(), N, U, eps, gx.data_ptr(), ga.data_ptr(),
                           _stream()) == 0, lib.dr_last_error()
    torch.cuda.synchronize()
    _check_guards(gxfull, N * U)
    _check_guards(gafull, U)
    return y.view(N, U), gx.view(N, U), ga


@pytest.mark.parametrize("N,U", [(1, 1), (7, 4), (300, 36), (1000, 200), (33, 1000)])
@pytest.mark.parametrize("eps", [1e-8, 1e-3])
def test_dice_matches_oracle(N, U, eps):
    rng = np.random.default_rng(N * 7 + U)
    x = _rand(rng, N, U)
    x[0] = 0.5                                               # a constant row
    if N > 2:
        x[1, : U // 2] = 0.0
    alpha = _rand(rng, U) * 0.7                              # negative entries too
    gy = _rand(rng, N, U)
    y, gx, ga = _dice_gpu(x, alpha, eps, gy)
    ref = dice(x, alpha, eps)
    x64, a64 = x.astype(np.float64), alpha.astype(np.float64)
    np.testing.assert_allclose(y.cpu().numpy(), ref, rtol=2e-5, atol=2e-6 * (np.abs(x64).max() + 1))
    rgx, rga = dice_grad(x, alpha, gy, eps)
    # the gradient's terms scale with |gy| |x| / den^3 through the std: measure against the oracle's |terms|
    scale = np.abs(rgx) + np.abs(gy) * (1 + np.abs(a64)) * (1 + np.abs(x64)) / np.sqrt(eps + 1e-3)
    assert np.all(np.isfinite(gx.cpu().numpy()))
    assert np.all(np.abs(gx.cpu().numpy() - rgx) <= 2e-5 * scale + 1e-6), np.abs(gx.cpu().numpy() - rgx).max()
    np.testing.assert_allclose(ga.cpu().numpy(), rga, rtol=1e-4, atol=1e-4 * (np.abs(gy).sum(0).max() + 1))


def test_dice_constant_row_has_finite_gradient():
    x = np.full((3, 8), 0.25, np.float32)
    alpha = np.full(8, -0.5, np.float32)
    y, gx, ga = _dice_gpu(x, alpha, 1e-8, np.ones((3, 8), np.float32))
    np.testing.assert_allclose(y.cpu().numpy(), dice(x, alpha), rtol=1e-6)
    assert np.all(np.isfinite(gx.cpu().numpy()))
    np.testing.assert_allclose(gx.cpu().numpy(), dice_grad(x, alpha, np.ones((3, 8)))[0], rtol=1e-5, atol=1e-6)


# ---- the layers -----------------------------------------------------------------------------------------------------
def test_reference_known_answers():
    """test_din.py:17-64 through the layers on the GPU."""
    from deep_recommenders.keras.models.ranking import din
    from deep_recommenders.keras.layers import Subtract
    rng = np.random.default_rng(0)
    x, y = rng.normal(size=(3, 5)), rng.normal(size=(3, 5))
    relu = lambda z: np.maximum(z, 0)
    out = din.ActivationUnit(10, kernel_init="ones")(x, y).detach().cpu().numpy()
    np.testing.assert_allclose(out, relu(np.concatenate([x, y], 1) @ np.ones((10, 10))).sum(1, keepdims=True),
                               rtol=1e-5, atol=1e-5)
    out = din.ActivationUnit(10, interacter=Subtract(), kernel_init="ones")(x, y).detach().cpu().numpy()
    np.testing.assert_allclose(out, relu(np.concatenate([x, y, x - y], 1) @ np.ones((15, 10))).sum(1, keepdims=True),
                               rtol=1e-5, atol=1e-5)
    inputs = np.asarray([[-0.2, -0.1, 0.1, 0.2]]).astype(np.float32)
    for eps in (1e-7, 1e-8, 1e-9, 1e-10):
        out = din.Dice(epsilon=eps)(inputs).detach().cpu().numpy()
        p = 1 / (1 + np.exp(-((inputs - inputs.mean()) / np.sqrt(inputs.std() + eps))))
        xx = np.where(inputs > 0, inputs, 0)
        np.testing.assert_allclose(out, np.where(xx > 0, p * xx, (1 - p) * xx), rtol=1e-6, atol=1e-7)


def _golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "din_golden.npz"))


def test_activation_unit_matches_golden():
    """The reference's own ActivationUnit outputs (din_golden.npz) through the layer, fused and composed paths."""
    from deep_recommenders.keras.models.ranking import din
    from deep_recommenders.keras.layers import Multiply, Subtract
    g = _golden()
    cases = sorted({k[4:-len("_x")] for k in g.files if k.startswith("f64_au_") and k.endswith("_x")})
    assert len(cases) >= 6
    for c in cases:
        pre = "f64_" + c
        inter = str(g[pre + "_inter"])
        act = str(g[pre + "_act"])
        bias = bool(g[pre + "_bias"])
        layer_act = din.Dice() if act == "dice" else act
        unit = din.ActivationUnit(int(g[pre + "_w1"].shape[1]), use_bias=bias, activation=layer_act,
                                  interacter={"none": None, "subtract": Subtract(), "multiply": Multiply()}[inter])
        x, y = g[pre + "_x"].astype(np.float32), g[pre + "_y"].astype(np.float32)
        unit.build(x.shape, device="cuda")
        with torch.no_grad():
            w1 = torch.from_numpy(g[pre + "_w1"].astype(np.float32)).cuda()
            if unit.dense_kernel.kernel is None:
                unit.dense_kernel.build((None, w1.shape[0]), device="cuda")
                unit.dense_output.build((None, w1.shape[1]), device="cuda")
            unit.dense_kernel.kernel.copy_(w1)
            unit.dense_output.kernel.copy_(torch.from_numpy(g[pre + "_w2"].astype(np.float32)))
            if bias:
                unit.dense_kernel.bias.copy_(torch.from_numpy(g[pre + "_b1"].astype(np.float32)))
                unit.dense_output.bias.copy_(torch.from_numpy(g[pre + "_b2"].astype(np.float32)))
            if act == "dice":
                layer_act(torch.zeros((1, w1.shape[1]), device="cuda"))
                layer_act.alpha.copy_(torch.from_numpy(g[pre + "_alpha"].astype(np.float32)))
        out = unit(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()).detach().cpu().numpy()
        ref = g[pre + "_out"]
        np.testing.assert_allclose(out, ref, rtol=2e-5, atol=2e-5 * (np.abs(ref).max() + 1), err_msg=c)


def _ref_model():
    from deep_recommenders.keras.layers import Model, Subtract
    from deep_recommenders.keras.models.ranking import din

    class Net(Model):
        def __init__(self):
            super().__init__()
            self.unit = din.ActivationUnit(10, interacter=Subtract(), seed=5)
            self.built = True

        def call(self, inputs, **kwargs):
            return self.unit(inputs[0], inputs[1])

        def get_config(self):
            return {**super().get_config(), "unit": self.unit.get_config()}

    return Net()


def test_reference_train_and_save():
    """test_din.py:66-94: ActivationUnit(10, Subtract()) as a model, compile("mse"), fit, save / load, predictions
    equal."""
    rng = np.random.default_rng(0)
    xe = torch.from_numpy(rng.normal(size=(10, 5)).astype(np.float32)).cuda()
    ye = torch.from_numpy(rng.normal(size=(10, 5)).astype(np.float32)).cuda()
    labels = rng.normal(size=(10,)).astype(np.float32)
    model = _ref_model()
    model.compile(loss="mse")
    hist = model.fit([xe, ye], labels, epochs=5, steps_per_epoch=1)
    assert np.all(np.isfinite(hist["loss"])) and hist["loss"][-1] < hist["loss"][0], hist["loss"]
    pred = model.predict([xe, ye])
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "din_model.pt")
        model.save(path)
        blob = torch.load(path, weights_only=False)
        loaded = _ref_model()
        loaded([xe, ye])
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == model.get_config() == blob["config"]
        assert torch.equal(loaded.predict([xe, ye]), pred)


@pytest.mark.parametrize("inter", ["none", "subtract", "multiply"])
def test_activation_unit_autograd_fused_and_composed(inter):
    """The fused unit and the composition (the same weights, a Layer-free activation forced through the composed
    path) give the same output and the same gradients."""
    from deep_recommenders.keras.layers import Multiply, Subtract
    from deep_recommenders.keras.models.ranking import din
    rng = np.random.default_rng(len(inter))
    mk = {"none": lambda: None, "subtract": Subtract, "multiply": Multiply}[inter]
    fused = din.ActivationUnit(24, interacter=mk(), activation="tanh", seed=1)
    xn, yn = _rand(rng, 200, 12), _rand(rng, 200, 12)
    x = torch.from_numpy(xn).cuda().requires_grad_()
    y = torch.from_numpy(yn).cuda().requires_grad_()
    out = fused(x, y)
    g = torch.from_numpy(_rand(rng, 200, 1)).cuda()
    (out * g).sum().backward()
    w1 = fused.dense_kernel.kernel.detach().cpu().numpy()
    b1 = fused.dense_kernel.bias.detach().cpu().numpy()
    w2 = fused.dense_output.kernel.detach().cpu().numpy()
    b2 = fused.dense_output.bias.detach().cpu().numpy()
    ref = activation_unit(xn, yn, w1, b1, w2, b2, "tanh", None if inter == "none" else inter)
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref, rtol=1e-5, atol=1e-5)
    # float64 autograd of the same composition
    t = {k: torch.tensor(v.astype(np.float64), requires_grad=True) for k, v in
         dict(x=xn, y=yn, w1=w1, b1=b1, w2=w2, b2=b2).items()}
    parts = [t["x"], t["y"]] + ([] if inter == "none" else [t["x"] - t["y"] if inter == "subtract" else t["x"] * t["y"]])
    o = torch.tanh(torch.cat(parts, 1) @ t["w1"] + t["b1"]) @ t["w2"] + t["b2"]
    (o * g.double().cpu()).sum().backward()
    for got, name in ((x.grad, "x"), (y.grad, "y"), (fused.dense_kernel.kernel.grad, "w1"),
                      (fused.dense_kernel.bias.grad, "b1"), (fused.dense_output.kernel.grad, "w2"),
                      (fused.dense_output.bias.grad, "b2")):
        r = t[name].grad.numpy()
        np.testing.assert_allclose(got.detach().cpu().numpy().reshape(r.shape), r, rtol=1e-4,
                                   atol=1e-4 * max(np.abs(r).max(), 1e-6), err_msg=name)


def test_activation_unit_with_dice_composes():
    from deep_recommenders.keras.layers import Subtract
    from deep_recommenders.keras.models.ranking import din
    rng = np.random.default_rng(3)
    act = din.Dice(epsilon=1e-6)
    unit = din.ActivationUnit(16, interacter=Subtract(), activation=act, seed=2)
    xn, yn = _rand(rng, 50, 8), _rand(rng, 50, 8)
    out = unit(torch.from_numpy(xn).cuda(), torch.from_numpy(yn).cuda())
    with torch.no_grad():
        act.alpha.copy_(torch.linspace(-0.5, 0.5, 16))
    out = unit(torch.from_numpy(xn).cuda(), torch.from_numpy(yn).cuda())
    alpha = act.alpha.detach().cpu().numpy()
    ref = activation_unit(xn, yn, unit.dense_kernel.kernel.detach().cpu().numpy(),
                          unit.dense_kernel.bias.detach().cpu().numpy(),
                          unit.dense_output.kernel.detach().cpu().numpy(),
                          unit.dense_output.bias.detach().cpu().numpy(), interact="subtract",
                          layer_act=lambda z: dice(z, alpha, 1e-6))
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref, rtol=1e-4, atol=1e-5)
    out.sum().backward()
    assert act.alpha.grad is not None and bool(torch.isfinite(act.alpha.grad).all())
    with pytest.raises(ValueError, match="call_pooled"):
        unit.call_pooled(torch.zeros((2, 3, 8), device="cuda"), torch.zeros((2, 8), device="cuda"))


# ---- the DIN model --------------------------------------------------------------------------------------------------
def _din(**kw):
    from deep_recommenders.keras.layers import DIN
    return DIN(seed=3, device="cuda", **kw)


def _batch(rng, B, T, item_rows, ctx_rows, id_dtype):
    """Ids with -1 padding, OOV ids, a history that contains the target item and one heavily repeated id."""
    item = rng.integers(0, item_rows, size=B)
    hist = rng.integers(0, item_rows, size=(B, T))
    lens = rng.integers(1, T + 1, size=B)
    hist[np.arange(T)[None, :] >= lens[:, None]] = -1
    hist[rng.random((B, T)) < 0.03] = item_rows               # OOV
    item[rng.random(B) < 0.03] = item_rows + 5
    hist[:, 0] = np.where(rng.random(B) < 0.3, item, hist[:, 0])   # the target inside its own history
    hist[rng.random((B, T)) < 0.3] = 1                        # a hot id
    ctx = np.stack([rng.integers(-1, r + 1, size=B) for r in ctx_rows], 1) if ctx_rows else None
    t = lambda a: None if a is None else torch.from_numpy(a.astype(np.int64)).to("cuda", id_dtype)
    return t(ctx), t(item), t(hist)


def _din_params64(m):
    P = {"item": m.item_table.detach().double().cpu().clone().requires_grad_()}
    if m.context is not None:
        P["ctx"] = m.context.emb_view().detach().double().cpu().clone().requires_grad_()
    a = m.attention
    P["w1"] = a.dense_kernel.kernel.detach().double().cpu().clone().requires_grad_()
    P["b1"] = a.dense_kernel.bias.detach().double().cpu().clone().requires_grad_()
    P["w2"] = a.dense_output.kernel.detach().double().cpu().clone().requires_grad_()
    P["b2"] = a.dense_output.bias.detach().double().cpu().clone().requires_grad_()
    for i, l in enumerate(m.mlp):
        for n in ("kernel", "bias", "alpha"):
            if getattr(l, n, None) is not None:
                P[f"mlp{i}.{n}"] = getattr(l, n).detach().double().cpu().clone().requires_grad_()
    P["hw"] = m.head.kernel.detach().double().cpu().clone().requires_grad_()
    P["hb"] = m.head.bias.detach().double().cpu().clone().requires_grad_()
    return P


def _dice_t(z, alpha, eps=1e-8):
    mu = z.mean(1, keepdim=True)
    sd = ((z - mu) ** 2).mean(1, keepdim=True).sqrt()
    p = torch.sigmoid((z - mu) / torch.sqrt(sd + eps))
    a = torch.where(z > 0, z, alpha * z)
    return torch.where(a > 0, p * a, (1 - p) * a)


def _din_logit64(m, P, ctx, item, hist):
    """The DIN composition in float64 torch-CPU autograd (the gradients' oracle)."""
    rows = P["item"].shape[0]

    def gather(t, ids):
        ids = ids.long().cpu()
        ok = (ids >= 0) & (ids < t.shape[0])
        return t[torch.where(ok, ids, torch.zeros_like(ids))] * ok[..., None]

    e = gather(P["item"], item)
    k = gather(P["item"], hist)
    qb = e[:, None, :].expand_as(k)
    u = torch.cat([k, qb, k - qb], -1)
    score = torch.relu(u @ P["w1"] + P["b1"]) @ P["w2"][:, 0] + P["b2"]
    parts = [e, (score[..., None] * k).sum(1)]
    if ctx is not None:
        c = m.context
        ids = ctx.long().cpu()
        okr = (ids >= 0) & (ids < torch.tensor(c.rows_list))
        flat = torch.where(okr, ids + c._offsets.cpu(), torch.zeros_like(ids))
        parts.insert(0, (P["ctx"][flat] * okr[..., None]).reshape(ids.shape[0], -1))
    x = torch.cat(parts, 1)
    for i, l in enumerate(m.mlp):
        if f"mlp{i}.kernel" in P:
            x = x @ P[f"mlp{i}.kernel"] + P[f"mlp{i}.bias"]
        else:
            x = _dice_t(x, P[f"mlp{i}.alpha"])
    del rows
    return (x @ P["hw"]).view(-1) + P["hb"]


@pytest.mark.parametrize("id_dtype", [torch.int64, torch.int32], ids=["i64", "i32"])
def test_din_step_matches_oracle(id_dtype):
    rng = np.random.default_rng(11)
    item_rows, ctx_rows, B, T, dim = 500, [30, 7], 300, 20, 16
    m = _din(item_rows=item_rows, dim=dim, context_rows=ctx_rows, att_units=36, dnn_units=(32, 16))
    with torch.no_grad():
        for l in m.mlp:
            if getattr(l, "alpha", None) is not None:
                l.alpha.uniform_(-0.5, 0.5)
    ctx, item, hist = _batch(rng, B, T, item_rows, ctx_rows, id_dtype)
    y = torch.from_numpy((rng.random(B) < 0.3).astype(np.float32)).cuda()
    prob = m((ctx, item, hist)).view(-1)
    loss = torch.nn.functional.binary_cross_entropy(prob, y)
    loss.backward()
    # forward against the numpy oracle
    a = m.attention
    mlp, layers = [], list(m.mlp)
    for i in range(0, len(layers), 2):
        mlp.append((layers[i].kernel.detach().cpu().numpy(), layers[i].bias.detach().cpu().numpy(),
                    layers[i + 1].alpha.detach().cpu().numpy()))
    c = m.context
    ref_prob, _ = din_forward(m.item_table.detach().cpu().numpy(), [c.table(s).detach().cpu().numpy()
                                                                   for s in range(len(ctx_rows))],
                              ctx.long().cpu().numpy(), item.long().cpu().numpy(), hist.long().cpu().numpy(),
                              (a.dense_kernel.kernel.detach().cpu().numpy(), a.dense_kernel.bias.detach().cpu().numpy(),
                               a.dense_output.kernel.detach().cpu().numpy(),
                               a.dense_output.bias.detach().cpu().numpy(), "relu", "subtract"),
                              mlp, m.head.kernel.detach().cpu().numpy(), m.head.bias.detach().cpu().numpy())
    np.testing.assert_allclose(prob.detach().double().cpu().numpy(), ref_prob, rtol=1e-5, atol=1e-6)
    P = _din_params64(m)
    z = _din_logit64(m, P, ctx, item, hist)
    ref_loss = torch.nn.functional.binary_cross_entropy_with_logits(z, y.double().cpu())
    ref_loss.backward()
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    got = {"item": m.item_table.grad, "ctx": c.weight.grad[:, :dim], "w1": a.dense_kernel.kernel.grad,
           "b1": a.dense_kernel.bias.grad, "w2": a.dense_output.kernel.grad, "b2": a.dense_output.bias.grad,
           "hw": m.head.kernel.grad, "hb": m.head.bias.grad}
    for i, l in enumerate(m.mlp):
        for n in ("kernel", "bias", "alpha"):
            if getattr(l, n, None) is not None:
                got[f"mlp{i}.{n}"] = getattr(l, n).grad
    for k, g in got.items():
        ref = P[k].grad.numpy()
        tol = 1e-4 * max(np.abs(ref).max(), 1e-6)
        np.testing.assert_allclose(g.detach().double().cpu().numpy().reshape(ref.shape), ref, rtol=1e-4, atol=tol,
                                   err_msg=k)


def test_din_save_load_and_config():
    m = _din(item_rows=200, dim=8, context_rows=[10], att_units=12, dnn_units=(16, 8), interacter="multiply")
    ctx, item, hist = _batch(np.random.default_rng(1), 64, 9, 200, [10], torch.int64)
    pred = m.predict((ctx, item, hist))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "din.pt")
        m.save(path)
        blob = torch.load(path, weights_only=False)
        from deep_recommenders.keras.layers import DIN
        cfg = {k: v for k, v in blob["config"].items() if k not in ("name", "trainable", "dtype")}
        loaded = DIN(**cfg, device="cuda")
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == m.get_config()
        assert torch.equal(loaded.predict((ctx, item, hist)), pred)


@pytest.mark.parametrize("sparse_lr", [None, 0.05])
def test_din_fit_through_keras_engine(sparse_lr):
    m = _din(item_rows=300, dim=16, att_units=16, dnn_units=(32, 8), sparse_lr=sparse_lr, dnn_activation="relu"
             if sparse_lr else "dice")
    rng = np.random.default_rng(2)
    _, item, hist = _batch(rng, 512, 10, 300, [], torch.int64)
    y = torch.from_numpy((item.cpu().numpy() % 2).astype(np.float32)).cuda()
    m.compile(loss="binary_crossentropy", optimizer="adam")
    hist_ = m.fit((None, item, hist), y, epochs=8, steps_per_epoch=1)
    losses = hist_["loss"]
    assert np.all(np.isfinite(losses)) and losses[-1] < losses[0], losses
