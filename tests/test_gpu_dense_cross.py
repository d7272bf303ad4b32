"""Rows F (standalone), D and X on the GPU through the C-ABI against the numpy oracle, plus the
reference's own known-answer tests ported verbatim:
  tests/keras/test_fm.py:17-26      FM layer vs the numpy formula on (10,5,5)
  tests/estimator/test_fm.py:18-26  fm() output shape (10,1) on (10,2,3)
  tests/keras/test_dcn.py:16-23     Cross, ones kernel -> [[0.55, 0.8, 1.05]]
"""
import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["ffma", "tc", "tc2", "tc2pair"])
def gemm_variant(request):
    """Every test in this file runs under all GEMM cores: FFMA, wgmma 3xTF32 on pre-split planes (tc) and
    wgmma 3xTF32 with the hi/lo split inside the kernel (tc2 = library defaults; tc2pair sets the `tc_pair` knob, which
    selects nothing on H100 -- there is one wgmma kernel -- and must leave every result unchanged)."""
    from deep_recommenders_b200 import _lib
    pair_default = _lib.tune_get("tc_pair")
    if request.param == "tc":
        _lib.enable_tensor_core_gemm(variant=1)
    elif request.param.startswith("tc2"):
        _lib.enable_tensor_core_gemm(variant=2)
        if request.param != "tc2":
            _lib.tune("tc_pair", 2 if request.param == "tc2pair" else 0)
    else:
        _lib.disable_tensor_core_gemm()
    yield request.param
    _lib.tune("tc_pair", pair_default)
    _lib.enable_tensor_core_gemm()


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def close(a, b, scale=None, rtol=1e-5):
    a = a.detach().cpu().numpy().astype(np.float64) if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    sc = np.abs(b).max() if scale is None else scale
    return np.abs(a - b).max() <= rtol * sc + 1e-7


# ---- Row F standalone ------------------------------------------------------------------
def test_ref_kat_fm_layer():
    """tests/keras/test_fm.py:17-26 (zero-init linear term contributes 0)."""
    from deep_recommenders.keras.models.ranking import FM
    rng = np.random.default_rng(0)
    sparse_inputs = rng.integers(0, 2, size=(10, 10)).astype(np.float32)
    embedding_inputs = rng.normal(size=(10, 5, 5)).astype(np.float32)
    x_sum = np.sum(embedding_inputs, axis=1)
    x_square_sum = np.sum(np.power(embedding_inputs, 2), axis=1)
    expected = 0.5 * np.sum(np.power(x_sum, 2) - x_square_sum, axis=1, keepdims=True)
    out = FM()(cu(sparse_inputs), cu(embedding_inputs))
    assert out.shape == (10, 1)
    assert np.allclose(out.detach().cpu().numpy(), expected, rtol=1e-6, atol=1e-6 * np.abs(embedding_inputs).max() ** 2 * 25)
    # linear-only form (fm.py:25-26)
    assert FM()(cu(sparse_inputs)).shape == (10, 1)


def test_ref_estimator_fm_shape_and_rank_check():
    from deep_recommenders.estimator.models.feature_interaction import fm
    x = torch.randn(10, 2, 3, device="cuda")
    assert fm(x).shape == (10, 1)
    with pytest.raises(ValueError, match="rank"):
        fm(torch.randn(10, 6, device="cuda"))


@pytest.mark.parametrize("B,S,D", [(1, 1, 1), (10, 5, 5), (10, 2, 3), (257, 26, 16), (64, 7, 33), (19, 3, 130)])
def test_fm_dense_fwd_bwd(B, S, D):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(B * S + D)
    x = rng.standard_normal((B, S, D)).astype(np.float32)
    g = rng.standard_normal((B, 1)).astype(np.float32)
    xt = cu(x).requires_grad_(True)
    y = ops.FMInteraction.apply(xt)
    y.backward(cu(g))
    x64 = x.astype(np.float64)
    scale = 0.5 * ((x64.sum(1) ** 2).sum(1) + (x64 ** 2).sum((1, 2)))
    ref = R.fm_second_order(x, np.float64).reshape(-1)
    assert (np.abs(y.detach().cpu().numpy().reshape(-1) - ref) <= 1e-5 * scale + 1e-7).all()
    refg = R.fm_second_order_grad(x, g, np.float64)
    gsc = np.abs(g).reshape(-1, 1, 1) * (np.abs(x64).sum(1, keepdims=True) + np.abs(x64))
    assert (np.abs(xt.grad.cpu().numpy() - refg) <= 1e-5 * gsc + 1e-7).all()


# ---- Row D: Dense ----------------------------------------------------------------------
DENSE_CASES = [
    # M, K, N
    (1, 1, 1), (10, 10, 1), (7, 3, 5), (130, 33, 17), (300, 416, 256), (257, 256, 32), (1000, 32, 1),
    (129, 70, 130), (64, 832, 832), (513, 100, 300),
]


@pytest.mark.parametrize("M,K,N", DENSE_CASES)
@pytest.mark.parametrize("act", [None, "relu", "sigmoid", "tanh"])
def test_dense_fwd_bwd(M, K, N, act):
    from deep_recommenders_b200 import ops
    if act in ("sigmoid", "tanh") and M > 300:
        pytest.skip("activation variants covered on the small shapes")
    rng = np.random.default_rng(M + K + N)
    x = rng.standard_normal((M, K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) * 0.1
    gy = rng.standard_normal((M, N)).astype(np.float32)
    xt, wt, bt = cu(x).requires_grad_(True), cu(w).requires_grad_(True), cu(b).requires_grad_(True)
    y = ops.DenseFn.apply(xt, wt, bt, ops.act_code(act))
    y.backward(cu(gy))
    ref = R.dense(x, w, b, act, np.float64)
    pre_scale = (np.abs(x).astype(np.float64) @ np.abs(w).astype(np.float64)) + np.abs(b)
    assert (np.abs(y.detach().cpu().numpy() - ref) <= 1e-5 * pre_scale + 1e-7).all()
    gx, gw, gb = R.dense_grad(x, w, ref, gy, act, np.float64)
    # relu mask computed from the fp32 output; compare where the oracle's pre-activation is not ~0
    if act == "relu":
        gx, gw, gb = R.dense_grad(x, w, y.detach().cpu().numpy(), gy, act, np.float64)
    agz = np.abs(gy).astype(np.float64)
    assert (np.abs(xt.grad.cpu().numpy() - gx) <= 2e-5 * (agz @ np.abs(w).T.astype(np.float64)) + 1e-6).all()
    assert (np.abs(wt.grad.cpu().numpy() - gw) <= 2e-5 * (np.abs(x).T.astype(np.float64) @ agz) + 1e-6).all()
    assert (np.abs(bt.grad.cpu().numpy() - gb) <= 2e-5 * agz.sum(0) + 1e-6).all()


def test_dense_no_bias_and_leading_dims():
    from deep_recommenders_b200 import ops
    x = torch.randn(4, 6, 10, device="cuda")
    w = torch.randn(10, 3, device="cuda")
    y = ops.DenseFn.apply(x, w, None, 0)
    assert y.shape == (4, 6, 3)
    assert torch.allclose(y, x @ w, rtol=1e-5, atol=1e-5)


# ---- Row X: Cross ----------------------------------------------------------------------
def test_ref_kat_cross_full_matrix():
    """tests/keras/test_dcn.py:16-23."""
    from deep_recommenders.keras.models.ranking.dcn import Cross
    x0 = np.asarray([[0.1, 0.2, 0.3]]).astype(np.float32)
    x = np.asarray([[0.4, 0.5, 0.6]]).astype(np.float32)
    cross = Cross(projection_dim=None, kernel_init="ones")
    output = cross(cu(x0), cu(x))
    assert np.allclose(np.asarray([[0.55, 0.8, 1.05]]), output.detach().cpu().numpy(), rtol=1e-6, atol=1e-6)


def test_cross_argument_checks():
    from deep_recommenders.keras.models.ranking.dcn import Cross
    with pytest.raises(AssertionError):
        Cross(diag_scale=-1.0)                                     # dcn.py:32-33
    with pytest.raises(ValueError, match="projection_dim"):
        Cross(projection_dim=7)(torch.randn(2, 13, device="cuda"))  # > last_dim/2, dcn.py:48-53
    with pytest.raises(ValueError, match="dim mismatch"):
        Cross()(torch.randn(2, 13, device="cuda"), torch.randn(2, 12, device="cuda"))   # dcn.py:75-78


@pytest.mark.parametrize("B,d,r,alpha,bias", [
    (1, 3, 0, 0.0, True), (10, 13, 0, 0.0, True), (130, 64, 0, 0.5, True), (257, 832, 0, 0.0, True),
    (33, 40, 0, 0.25, False), (10, 13, 4, 0.0, True), (130, 64, 16, 0.5, True), (65, 100, 50, 0.0, False),
])
@pytest.mark.parametrize("same", [False, True])
def test_cross_fwd_bwd(B, d, r, alpha, bias, same):
    from deep_recommenders_b200 import ops
    rng = np.random.default_rng(B + d + r)
    x0 = rng.standard_normal((B, d)).astype(np.float32)
    x = x0 if same else rng.standard_normal((B, d)).astype(np.float32)
    b = (rng.standard_normal(d) * 0.1).astype(np.float32) if bias else None
    g = rng.standard_normal((B, d)).astype(np.float32)
    if r == 0:
        w = (rng.standard_normal((d, d)) / np.sqrt(d)).astype(np.float32)
        u = v = None
    else:
        w = None
        u = (rng.standard_normal((d, r)) / np.sqrt(d)).astype(np.float32)
        v = (rng.standard_normal((r, d)) / np.sqrt(r)).astype(np.float32)
    t = lambda a: None if a is None else cu(a).requires_grad_(True)
    x0t, wt, ut, vt, bt = t(x0), t(w), t(u), t(v), t(b)
    xt = x0t if same else t(x)
    y = ops.CrossFn.apply(x0t, xt, wt, ut, vt, bt, alpha, same)
    y.backward(cu(g))
    ref, prod = R.cross(x0, x, w, b, u, v, alpha, np.float64)
    ax, ax0 = np.abs(x).astype(np.float64), np.abs(x0).astype(np.float64)
    if r == 0:
        pscale = ax @ np.abs(w) + alpha * ax
    else:
        pscale = (ax @ np.abs(u)) @ np.abs(v) + alpha * ax
    if b is not None:
        pscale = pscale + np.abs(b)
    assert (np.abs(y.detach().cpu().numpy() - ref) <= 1e-5 * (ax0 * pscale + ax) + 1e-7).all()
    gr = R.cross_grad(x0, x, g, w, u, v, b, alpha, np.float64)
    ag = np.abs(g).astype(np.float64)
    ah = ag * ax0
    if same:
        want_x0 = gr["gx0"] + gr["gx"]
    else:
        want_x0 = gr["gx0"]
        if r == 0:
            sx = ah @ np.abs(w).T + alpha * ah + ag
        else:
            sx = (ah @ np.abs(v).T) @ np.abs(u).T + alpha * ah + ag
        assert (np.abs(xt.grad.cpu().numpy() - gr["gx"]) <= 2e-5 * sx + 1e-6).all()
    tol0 = 2e-5 * (ag * pscale + (ah @ (np.abs(w).T if r == 0 else np.abs(v).T @ np.abs(u).T)) + alpha * ah + ag) + 1e-6
    assert (np.abs(x0t.grad.cpu().numpy() - want_x0) <= tol0).all()
    if r == 0:
        assert (np.abs(wt.grad.cpu().numpy() - gr["gw"]) <= 2e-5 * (ax.T @ ah) + 1e-6).all()
    else:
        assert (np.abs(ut.grad.cpu().numpy() - gr["gu"]) <= 2e-5 * (ax.T @ (ah @ np.abs(v).T)) + 1e-6).all()
        assert (np.abs(vt.grad.cpu().numpy() - gr["gv"]) <= 2e-5 * ((ax @ np.abs(u)).T @ ah) + 1e-6).all()
    if b is not None:
        assert (np.abs(bt.grad.cpu().numpy() - gr["gb"]) <= 2e-5 * ah.sum(0) + 1e-6).all()


def test_cross_stack_like_reference_test():
    """tests/keras/test_dcn.py:27-32 stacking: x1 = Cross()(x0, x0); x2 = Cross()(x0, x1); Dense(1)."""
    from deep_recommenders.keras.models.ranking.dcn import Cross
    from deep_recommenders.keras.layers import Dense
    x0 = torch.rand(10, 13, device="cuda")
    c1, c2, head = Cross(projection_dim=None, seed=1), Cross(projection_dim=None, seed=2), Dense(1, seed=3)
    logits = head(c2(x0, c1(x0, x0)))
    assert logits.shape == (10, 1)
    x1, _ = R.cross(x0.cpu().numpy(), None, c1.kernel.detach().cpu().numpy(), c1.bias.detach().cpu().numpy(), dtype=np.float64)
    x2, _ = R.cross(x0.cpu().numpy(), x1, c2.kernel.detach().cpu().numpy(), c2.bias.detach().cpu().numpy(), dtype=np.float64)
    ref = R.dense(x2, head.kernel.detach().cpu().numpy(), head.bias.detach().cpu().numpy(), None, np.float64)
    assert np.allclose(logits.detach().cpu().numpy(), ref, rtol=1e-5, atol=1e-5)
    cfg = c1.get_config()
    assert set(["projection_dim", "diag_scale", "use_bias", "kernel_init", "kernel_regu", "bias_init", "bias_regu"]) <= set(cfg)


@pytest.mark.parametrize("M,K,N", [(300, 256, 32), (257, 416, 256), (1000, 32, 1), (130, 33, 17)])
@pytest.mark.parametrize("prev_act", ["relu", "tanh", None])
def test_dense_bwd_chain_fuses_previous_activation_gradient(M, K, N, prev_act):
    """dr_dense_bwd_chain: gx = (gz @ W^T) * act_prev'(prev_y) -- the activation-gradient pass of the layer below,
    folded into this layer's input-gradient GEMM (deepfm.py:30-34 stack of Dense layers)."""
    from deep_recommenders_b200 import _lib, ops
    lib = _lib.load()
    rng = np.random.default_rng(M + K + N)
    z_prev = rng.standard_normal((M, K)).astype(np.float32)
    x = R.act(z_prev, prev_act).astype(np.float32)                     # output of the layer below = this layer's input
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    gy = rng.standard_normal((M, N)).astype(np.float32)
    xt, wt, gyt = cu(x), cu(w), cu(gy)
    gx = torch.empty((M, K), device="cuda")
    gw = torch.empty((K, N), device="cuda")
    gb = torch.empty((N,), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dr_dense_bwd_chain(xt.data_ptr(), wt.data_ptr(), None, gyt.data_ptr(), M, K, N, 0, None, gx.data_ptr(),
                                      gw.data_ptr(), gb.data_ptr(), xt.data_ptr(), ops.act_code(prev_act), st),
               "dr_dense_bwd_chain")
    gy64 = gy.astype(np.float64)
    gx_lin, gw_ref, gb_ref = gy64 @ w.astype(np.float64).T, x.astype(np.float64).T @ gy64, gy64.sum(0)
    x64 = x.astype(np.float64)
    dact = {"relu": (x64 > 0).astype(np.float64), "tanh": 1 - x64 * x64, None: np.ones_like(x64)}[prev_act]
    agy = np.abs(gy).astype(np.float64)
    sx = (agy @ np.abs(w).T.astype(np.float64)) * np.abs(dact)
    assert (np.abs(gx.cpu().numpy() - gx_lin * dact) <= 2e-5 * sx + 1e-6).all()
    assert (np.abs(gw.cpu().numpy() - gw_ref) <= 2e-5 * (np.abs(x64).T @ agy) + 1e-6).all()
    assert (np.abs(gb.cpu().numpy() - gb_ref) <= 2e-5 * agy.sum(0) + 1e-6).all()


@pytest.mark.parametrize("B,K", [(1, 1), (257, 32), (1000, 8), (300, 100), (129, 256)])
@pytest.mark.parametrize("prev_act", ["relu", None, "sigmoid"])
def test_dense_head_bce_fused_matches_oracle(B, K, prev_act):
    """dr_dense_head_bce_fwd_bwd == Dense(1) forward + (fm + dnn) + mean BCE + backward, composed from the oracle
    (deepfm.py:30-34,46-47; examples/train_deepfm_on_movielens_keras.py:43)."""
    from deep_recommenders_b200 import _lib, ops
    lib = _lib.load()
    rng = np.random.default_rng(B + K)
    a = R.act(rng.standard_normal((B, K)), prev_act).astype(np.float32)
    w = (rng.standard_normal((K, 1)) / np.sqrt(K)).astype(np.float32)
    b = np.asarray([0.3], np.float32)
    zadd = rng.standard_normal(B).astype(np.float32)
    y = rng.integers(0, 2, B).astype(np.float32)
    f = lambda *shape: torch.full(shape, float("nan"), device="cuda")
    logit, prob, loss, gl, gp, gw, gb, gbp = f(B), f(B), f(1), f(B), f(B, K), f(K), f(1), f(K)
    at, wt, bt, zt, yt = cu(a), cu(w), cu(b), cu(zadd), cu(y)
    _lib.check(lib.dr_dense_head_bce_fwd_bwd(at.data_ptr(), wt.data_ptr(), bt.data_ptr(), zt.data_ptr(), yt.data_ptr(), B, K,
                                             ops.act_code(prev_act), logit.data_ptr(), prob.data_ptr(), loss.data_ptr(),
                                             gl.data_ptr(), gp.data_ptr(), gw.data_ptr(), gb.data_ptr(), gbp.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "head")
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    z = (a64 @ w64).reshape(-1) + 0.3
    zi = z + zadd
    p = 1 / (1 + np.exp(-zi))
    ref_loss = np.mean(np.maximum(zi, 0) - zi * y + np.log1p(np.exp(-np.abs(zi))))
    g = (p - y) / B
    dact = {"relu": (a64 > 0).astype(np.float64), "sigmoid": a64 * (1 - a64), None: np.ones_like(a64)}[prev_act]
    ref_gp = g[:, None] * w64.reshape(1, -1) * dact
    zs = np.abs(a64) @ np.abs(w64).reshape(-1) + 0.3
    assert (np.abs(logit.cpu().numpy() - z) <= 1e-5 * zs + 1e-7).all()
    assert np.allclose(prob.cpu().numpy(), p, rtol=1e-5, atol=1e-6)
    assert abs(float(loss) - ref_loss) <= 1e-5 * abs(ref_loss) + 1e-7
    assert np.allclose(gl.cpu().numpy(), g, rtol=1e-4, atol=1e-6 / B)      # sigmoid of an fp32 logit
    assert (np.abs(gp.cpu().numpy() - ref_gp) <= 1e-4 * np.abs(ref_gp) + 1e-6 / B).all()
    ag = np.abs(g)
    assert (np.abs(gw.cpu().numpy() - a64.T @ g) <= 1e-4 * (np.abs(a64).T @ ag) + 1e-9).all()
    assert abs(float(gb) - g.sum()) <= 1e-4 * ag.sum() + 1e-9
    assert (np.abs(gbp.cpu().numpy() - ref_gp.sum(0)) <= 1e-4 * np.abs(ref_gp).sum(0) + 1e-9).all()
