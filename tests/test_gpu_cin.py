"""GPU tests of the CIN kernels (dr_cin_fwd / dr_cin_bwd) and the CIN layer.

Every fp32 result must sit within 1e-5 x (sum of |terms|) of the float64 oracle (tests/cin_oracle.py); outputs are
written between sentinel guards so a store outside [B, H, D] / [B, H] is caught."""
import os
import tempfile
import zlib

import numpy as np
import pytest
import torch

from cin_oracle import cin_grad

pytestmark = pytest.mark.gpu
ACTS = {"linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3}
SENT = 1234.5
PAD = 4099


def _lib():
    from deep_recommenders_b200 import _lib
    return _lib.load()


def _guarded(n):
    """A device buffer of n floats between PAD sentinels on each side: (full buffer, the n-float view)."""
    full = torch.full((n + 2 * PAD,), SENT, device="cuda", dtype=torch.float32)
    return full, full[PAD:PAD + n]


def _check_guards(full, n):
    f = full.cpu().numpy()
    assert np.all(f[:PAD] == SENT) and np.all(f[PAD + n:] == SENT), "store outside the output"


def _close(got, ref, scale, rel=1e-5):
    """|got - ref| <= rel * sum|terms| + 4 ulp of the result (the rounding of an activation's own fp32 output)."""
    got, ref, scale = (torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to("cuda", torch.float64)
                       for a in (got, ref, scale))
    err = (got - ref).abs()
    bound = rel * scale + 4.8e-7 * ref.abs() + 1e-30
    bad = err > bound
    assert not bool(bad.any()), (f"{int(bad.sum())} elements out of bound; worst err {err.max().item():.3g} "
                                 f"vs bound {bound[bad].min().item():.3g}")


# float64 references computed on the GPU with torch (the numpy oracle in cin_oracle.py is pinned to the reference's own
# code by the golden vectors; this is the same formula, fast enough for the full-size cases)
_ACT64 = {"linear": lambda z: z, "relu": torch.relu, "sigmoid": torch.sigmoid, "tanh": torch.tanh}


def _t64(a):
    return None if a is None else torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a).to(
        "cuda", torch.float64)


def _pre64(x0, x, w, b):
    x0, x, w = _t64(x0), _t64(x), _t64(w)
    m, h = x0.shape[1], x.shape[1]
    z = torch.einsum("bijd,ijk->bkd", x0[:, :, None, :] * x[:, None, :, :], w.view(m, h, -1))
    return z if b is None else z + _t64(b)[None, :, None]


def cin(x0, x, w, b, act):
    return _ACT64[act](_pre64(x0, x, w, b))


def cin_abs(x0, x, w, b):
    return _pre64(_t64(x0).abs(), _t64(x).abs(), _t64(w).abs(), None if b is None else _t64(b).abs())


def cin_grad64(x0, x, w, G):
    """(gx0, gx, gw, gb) for the upstream gradient G of the pre-activation, float64 on the GPU."""
    x0, x, w, G = _t64(x0), _t64(x), _t64(w), _t64(G)
    m, h = x0.shape[1], x.shape[1]
    wk = w.view(m, h, -1)
    t = torch.einsum("ijk,bkd->bijd", wk, G)
    gx0 = (t * x[:, None, :, :]).sum(2)
    gx = (t * x0[:, :, None, :]).sum(1)
    gw = torch.einsum("bijd,bkd->ijk", x0[:, :, None, :] * x[:, None, :, :], G).reshape(1, m * h, -1)
    return gx0, gx, gw, G.sum((0, 2))


def _G64(y, gy, gp, act):
    y = _t64(y)
    g = torch.zeros_like(y)
    if gy is not None:
        g = g + _t64(gy)
    if gp is not None:
        g = g + _t64(gp)[:, :, None]
    d = {"relu": lambda v: (v > 0).double(), "sigmoid": lambda v: v * (1 - v), "tanh": lambda v: 1 - v * v,
         "linear": torch.ones_like}[act](y)
    return g * d


def _ptr(t):
    return None if t is None else t.data_ptr()


def _rand(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32)


def _fwd(x0, x, w, b, act, pooled):
    B, m, D = x0.shape
    h, H = x.shape[1], w.shape[-1]
    yfull, y = _guarded(B * H * D)
    pfull, p = _guarded(B * H) if pooled else (None, None)
    rc = _lib().dr_cin_fwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), _ptr(b), B, m, h, D, H, ACTS[act],
                           y.data_ptr(), _ptr(p), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    _check_guards(yfull, B * H * D)
    if pooled:
        _check_guards(pfull, B * H)
    return y.view(B, H, D), (p.view(B, H) if pooled else None)


# (m, h, H, D, B): every listed value of each dimension, tails on the 64 / 128 row tiles, the 16-step contraction and
# the 128-column tile (D = 3 and 20 leave dead columns, D = 128 one example per tile)
FWD_CASES = [
    (1, 1, 1, 1, 1), (2, 2, 3, 3, 5), (7, 2, 64, 4, 5), (2, 7, 65, 16, 4099), (26, 26, 128, 16, 4099),
    (33, 26, 200, 20, 1), (26, 33, 129, 3, 4099), (1, 33, 64, 128, 5), (33, 1, 3, 16, 4099), (7, 7, 128, 128, 37),
    (26, 7, 1, 20, 4099), (2, 26, 200, 4, 4099), (33, 33, 63, 1, 4099), (7, 26, 127, 3, 1), (26, 2, 3, 128, 5),
    (1, 2, 128, 20, 0), (33, 7, 200, 16, 0), (5, 13, 17, 43, 300),
]


@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: "m{}h{}H{}D{}B{}".format(*c))
@pytest.mark.parametrize("act", list(ACTS))
def test_cin_fwd_matches_oracle(case, act):
    m, h, H, D, B = case
    rng = np.random.default_rng(zlib.crc32(repr((case, act)).encode()))
    x0, x = _rand(rng, B, m, D), _rand(rng, B, h, D)
    w, b = _rand(rng, 1, m * h, H, scale=0.2), _rand(rng, H)
    use_bias = (m + H) % 2 == 0
    dev = lambda a: torch.from_numpy(a).cuda()
    y, p = _fwd(dev(x0), dev(x), dev(w), dev(b) if use_bias else None, act, pooled=True)
    bb = b if use_bias else None
    ref = cin(x0, x, w, bb, act)
    scale = cin_abs(x0, x, w, bb)
    _close(y, ref, scale)
    _close(p, ref.sum(2), scale.sum(2) + ref.abs().sum(2))


def test_cin_fwd_without_pooled_is_bit_identical():
    rng = np.random.default_rng(3)
    x0 = torch.from_numpy(_rand(rng, 777, 26, 16)).cuda()
    x = torch.from_numpy(_rand(rng, 777, 40, 16)).cuda()
    w = torch.from_numpy(_rand(rng, 1, 26 * 40, 96, scale=0.1)).cuda()
    y1, _ = _fwd(x0, x, w, None, "sigmoid", pooled=False)
    y2, _ = _fwd(x0, x, w, None, "sigmoid", pooled=True)
    assert torch.equal(y1, y2)


def _bwd(x0, x, w, y, gy, gpool, act, same):
    B, m, D = x0.shape
    h, H = x.shape[1], w.shape[-1]
    g_ws = torch.empty((B, H, D), device="cuda")
    gx0full, gx0 = _guarded(B * m * D)
    gxfull, gx = (None, None) if same else _guarded(B * h * D)
    gwfull, gw = _guarded(m * h * H)
    gbfull, gb = _guarded(H)
    rc = _lib().dr_cin_bwd(x0.data_ptr(), x.data_ptr(), w.data_ptr(), y.data_ptr(), _ptr(gy), _ptr(gpool), B, m, h,
                           D, H, ACTS[act], int(same), g_ws.data_ptr(), gx0.data_ptr(), _ptr(gx), gw.data_ptr(),
                           gb.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    for full, n in ((gx0full, B * m * D), (gxfull, B * h * D), (gwfull, m * h * H), (gbfull, H)):
        if full is not None:
            _check_guards(full, n)
    return gx0.view(B, m, D), (None if same else gx.view(B, h, D)), gw.view(1, m * h, H), gb


BWD_CASES = [(2, 3, 3, 3, 5), (26, 26, 128, 16, 4099), (7, 33, 200, 20, 300), (33, 2, 64, 1, 4099),
             (1, 7, 65, 128, 37), (26, 13, 1, 4, 1000), (5, 5, 17, 43, 257)]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "m{}h{}H{}D{}B{}".format(*c))
@pytest.mark.parametrize("grads", ["gy", "gpool", "both"])
@pytest.mark.parametrize("act", ["linear", "relu", "sigmoid", "tanh"])
def test_cin_bwd_matches_oracle(case, grads, act):
    m, h, H, D, B = case
    rng = np.random.default_rng(zlib.crc32(repr((case, grads, act)).encode()))
    x0, x = _rand(rng, B, m, D), _rand(rng, B, h, D)
    w, b = _rand(rng, 1, m * h, H, scale=0.2), _rand(rng, H)
    dev = lambda a: torch.from_numpy(a).cuda()
    y, _ = _fwd(dev(x0), dev(x), dev(w), dev(b), act, pooled=False)
    gy = _rand(rng, B, H, D) if grads in ("gy", "both") else None
    gp = _rand(rng, B, H) if grads in ("gpool", "both") else None
    gx0, gx, gw, gb = _bwd(dev(x0), dev(x), dev(w), y, None if gy is None else dev(gy),
                           None if gp is None else dev(gp), act, same=False)
    G = _G64(y, gy, gp, act)
    rx0, rx, rw, rb = cin_grad64(x0, x, w, G)
    # |G| bound: the kernel forms G in fp32 from the same y
    aG = G.abs() + 1e-6 * (_t64(np.abs(gy)) if gy is not None else 0) + \
        1e-6 * (_t64(np.abs(gp))[:, :, None] if gp is not None else 0)
    sx0, sx, sw, sb = cin_grad64(np.abs(x0), np.abs(x), np.abs(w), aG)
    _close(gx0, rx0, sx0)
    _close(gx, rx, sx)
    _close(gw, rw, sw)
    _close(gb, rb, sb)


@pytest.mark.parametrize("case", [(26, 128, 16, 4099), (7, 3, 3, 5), (33, 200, 20, 300), (1, 1, 1, 7)],
                         ids=lambda c: "m{}H{}D{}B{}".format(*c))
def test_cin_bwd_x_is_x0(case):
    """The first layer (x is x0): one gradient buffer holding both contributions."""
    m, H, D, B = case
    rng = np.random.default_rng(11)
    x0 = torch.from_numpy(_rand(rng, B, m, D)).cuda()
    w = torch.from_numpy(_rand(rng, 1, m * m, H, scale=0.2)).cuda()
    y, _ = _fwd(x0, x0, w, None, "sigmoid", pooled=False)
    gy = torch.from_numpy(_rand(rng, B, H, D)).cuda()
    g_same, _, gw_same, gb_same = _bwd(x0, x0, w, y, gy, None, "sigmoid", same=True)
    a, bx, gw_sep, _ = _bwd(x0, x0.clone(), w, y, gy, None, "sigmoid", same=False)
    ref = a.double() + bx.double()
    scale = (a.abs() + bx.abs()).double()
    assert torch.all((g_same.double() - ref).abs() <= 1e-6 * scale + 1e-12)
    G = _G64(y, gy, None, "sigmoid")
    rx0, rx, rw, _ = cin_grad64(x0, x0, w, G)
    sx0, sx, sw, _ = cin_grad64(x0.abs(), x0.abs(), w.abs(), G.abs())
    _close(g_same, rx0 + rx, sx0 + sx)
    _close(gw_same, rw, sw)


def test_cin_bwd_deterministic_input_grads():
    rng = np.random.default_rng(5)
    x0 = torch.from_numpy(_rand(rng, 2000, 26, 16)).cuda()
    x = torch.from_numpy(_rand(rng, 2000, 64, 16)).cuda()
    w = torch.from_numpy(_rand(rng, 1, 26 * 64, 128, scale=0.1)).cuda()
    y, _ = _fwd(x0, x, w, None, "relu", pooled=False)
    gp = torch.from_numpy(_rand(rng, 2000, 128)).cuda()
    r1 = _bwd(x0, x, w, y, None, gp, "relu", same=False)
    r2 = _bwd(x0, x, w, y, None, gp, "relu", same=False)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1])


def test_cin_enotsup_above_caps_and_einval():
    lib = _lib()
    buf = torch.zeros(1 << 16, device="cuda")
    p = buf.data_ptr()
    for (m, h, D, H) in [(1025, 1, 1, 1), (1, 1025, 1, 1), (1, 1, 129, 1), (1, 1, 1, 1025)]:
        assert lib.dr_cin_fwd(p, p, p, None, 1, m, h, D, H, 0, p, None, None) == -3
        assert lib.dr_cin_bwd(p, p, p, p, p, None, 1, m, h, D, H, 0, 0, p, p, p, p, None, None) == -3
    assert lib.dr_cin_fwd(p, p, p, None, 1 << 25, 1, 1, 128, 1, 0, p, None, None) == -3
    assert lib.dr_cin_fwd(p, p, p, None, 1, 1, 1, 1, 1, 7, p, None, None) == -1
    assert lib.dr_cin_bwd(p, p, p, p, p, None, 1, 2, 2, 1, 1, 0, 1, p, p, p, p, None, None) == -1   # x_is_x0 with gx
    torch.cuda.synchronize()


# ---- the reference's own tests (tests/keras/test_xdeepfm.py) through the layer on the GPU ------------------------
def test_reference_known_answers():
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    x0 = np.asarray([[[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]]]).astype(np.float32)
    x = np.asarray([[[0.1, 0.2, 0.3], [0.4, 0.5, 0.6]]]).astype(np.float32)
    out = CIN(feature_map=2, activation="relu", kernel_init="ones")((x0, x))
    np.testing.assert_allclose(out.detach().cpu().numpy(), [[[0.25, 0.49, 0.81], [0.25, 0.49, 0.81]]], rtol=1e-6)
    out = CIN(feature_map=2, use_bias=True, activation="relu", kernel_init="ones", bias_init="ones")((x0, x))
    np.testing.assert_allclose(out.detach().cpu().numpy(), [[[1.25, 1.49, 1.81], [1.25, 1.49, 1.81]]], rtol=1e-6)


def _golden():
    path = os.path.join(os.path.dirname(__file__), "golden", "cin_golden.npz")
    return np.load(path)


def test_layer_matches_golden():
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    g = _golden()
    cases = sorted({k[:-len("_x0")] for k in g.files if k.startswith("f32_") and k.endswith("_x0")})
    assert len(cases) >= 6
    for c in cases:
        act = str(g[f"{c}_act"])
        use_bias = f"{c}_bias" in g.files
        x0, x, w = g[f"{c}_x0"], g[f"{c}_x"], g[f"{c}_kernel"]
        layer = CIN(feature_map=w.shape[-1], use_bias=use_bias, activation=act)
        layer.build(((None,) + x0.shape[1:], (None,) + x.shape[1:]), device="cuda")
        with torch.no_grad():
            layer.kernel.copy_(torch.from_numpy(w))
            if use_bias:
                layer.bias.copy_(torch.from_numpy(g[f"{c}_bias"]))
        out = layer((torch.from_numpy(x0).cuda(), torch.from_numpy(x).cuda())).detach().cpu().numpy()
        scale = cin_abs(x0, x, w, g[f"{c}_bias"] if use_bias else None)
        _close(out, g[f"{c}_y"].astype(np.float64), scale, rel=2e-5)
        _close(out, g["f64_" + c[4:] + "_y"], scale)


def _ref_model():
    from deep_recommenders.keras.layers import Dense, Model
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN

    class Net(Model):
        def __init__(self):
            super().__init__()
            self.c1 = CIN(feature_map=3, seed=1)
            self.c2 = CIN(feature_map=3, seed=2)
            self.out = Dense(1, seed=3)
            self.built = True

        def call(self, x0, **kwargs):
            x = self.c1((x0, x0))
            x = self.c2((x0, x))
            return self.out(x.reshape(x.shape[0], -1))

        def get_config(self):
            return {**super().get_config(), "cin": [self.c1.get_config(), self.c2.get_config()]}

    return Net()


def test_reference_train_model():
    """test_xdeepfm.py:62-80: CIN -> CIN -> Flatten -> Dense(1), mse, fit: the loss is finite and decreases."""
    rng = np.random.default_rng(0)
    x0 = torch.from_numpy(rng.uniform(size=(10, 12, 10)).astype(np.float32)).cuda()
    y = rng.uniform(size=(10,)).astype(np.float32)
    model = _ref_model()
    model.compile(loss=lambda yt, yp: (yt - yp) ** 2, optimizer="adam")     # "mse"
    hist = model.fit(x0, y, epochs=5, steps_per_epoch=1)
    losses = hist["loss"]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


def test_reference_save_model():
    """test_xdeepfm.py:82-109: configs equal and predictions bit-equal after save / load."""
    rng = np.random.default_rng(1)
    x0 = torch.from_numpy(rng.uniform(size=(10, 12, 10)).astype(np.float32)).cuda()
    model = _ref_model()
    pred = model.predict(x0)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m.pt")
        model.save(path)
        blob = torch.load(path, weights_only=False)
        loaded = _ref_model()
        loaded(x0)
        loaded.load_state_dict(blob["state"])
        assert loaded.get_config() == model.get_config() == blob["config"]
        assert torch.equal(loaded.predict(x0), pred)


def test_layer_autograd_and_pooled():
    """CINFn through autograd: y and pooled gradients reach x0, x, kernel and bias."""
    from deep_recommenders.keras.models.ranking.xdeepfm import CIN
    rng = np.random.default_rng(2)
    x0n, xn = _rand(rng, 64, 5, 8), _rand(rng, 64, 6, 8)
    x0 = torch.from_numpy(x0n).cuda().requires_grad_()
    x = torch.from_numpy(xn).cuda().requires_grad_()
    layer = CIN(feature_map=7, use_bias=True, activation="tanh", seed=0)
    y, pooled = layer.call_pooled((x0, x))
    gy, gp = _rand(rng, 64, 7, 8), _rand(rng, 64, 7)
    (y * torch.from_numpy(gy).cuda()).sum().add((pooled * torch.from_numpy(gp).cuda()).sum()).backward()
    w = layer.kernel.detach().cpu().numpy()
    yv = y.detach().cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(pooled.detach().cpu().numpy(), y.detach().cpu().numpy().sum(2), rtol=1e-5, atol=1e-5)
    rx0, rx, rw, rb, _ = cin_grad(x0n, xn, w, yv, gy, gp, "tanh")
    for got, ref in ((x0.grad, rx0), (x.grad, rx), (layer.kernel.grad, rw), (layer.bias.grad, rb)):
        np.testing.assert_allclose(got.cpu().numpy(), ref, rtol=1e-4, atol=1e-4)
