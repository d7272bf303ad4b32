"""Rows D and X at BASELINE.json's FULL sizes (C2: M = 65536, C3: M = 131072) through the C-ABI against the float64
oracle.  These are the shapes the small cases of test_gpu_dense_cross.py never reach: the persistent multi-tile
schedule of the wgmma core, the mbarrier phase wrap of its two rings (hundreds of tiles per CTA) and split-K weight
gradients with K = M = 65536 / 131072.

The check is mask-consistent: the ReLU mask the backward uses is the one of the GPU's own forward output `y`
(a pre-activation within fp32 rounding of 0 may legitimately land on either side; round 1's 0.04-0.09 "errors" at
these sizes were exactly that: the float64 mask applied to a float32 forward), and every bound is
1e-5 / 2e-5 x the sum of |terms| of the dot product it checks (DESIGN.md section 3), never max|ref|.

Rows of the output / of dX are independent, so the float64 oracle is evaluated on a seeded sample of rows
(plus the first and last tiles); dW and db need every row and are checked in full.
"""
import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sample_rows(M, n, rng):
    """first / last 256 rows (first and last tile of the persistent schedule) + n random rows"""
    edge = np.concatenate([np.arange(0, min(256, M)), np.arange(max(0, M - 256), M)])
    return np.unique(np.concatenate([edge, rng.integers(0, M, size=n)]))


@pytest.fixture(params=["tc2", "tc", "ffma", "tc2share", "tc2single", "tc2pair"])
def gemm_core(request):
    """tc2 = the shipped core under the library defaults; tc2single / tc2pair set the `tc_pair` knob (it selects nothing
    on H100, results must not change); tc2share = the weight-gradient GEMM with the shorter raw operand ring (knob
    tc_dw_share)."""
    from deep_recommenders_b200 import _lib
    pair_default = _lib.tune_get("tc_pair")
    if request.param == "tc":
        _lib.enable_tensor_core_gemm(variant=1)
    elif request.param.startswith("tc2"):
        _lib.enable_tensor_core_gemm(variant=2)
        _lib.tune("tc_dw_share", 1 if request.param == "tc2share" else 0)
        if request.param in ("tc2single", "tc2pair", "tc2share"):
            _lib.tune("tc_pair", 2 if request.param == "tc2pair" else 0)
    else:
        _lib.disable_tensor_core_gemm()
    yield request.param
    _lib.tune("tc_dw_share", 0)
    _lib.tune("tc_pair", pair_default)
    _lib.enable_tensor_core_gemm()


FULL_DENSE = [
    # M, K, N, act            the C2 tower (examples/train_deepfm_on_movielens_keras.py:42 -> [256, 32] + [1])
    (65536, 416, 256, "relu"),
    (65536, 416, 256, None),
    (65536, 256, 32, "relu"),
    (65536, 32, 1, None),
    # C3's DNN [512, 256, 128] on d = 832
    (131072, 832, 512, "relu"),
    (131072, 512, 256, "relu"),
    (131072, 256, 128, None),
]


@pytest.mark.parametrize("M,K,N,act", FULL_DENSE)
def test_dense_full_size(M, K, N, act, gemm_core):
    from deep_recommenders_b200 import ops
    if gemm_core not in ("tc2", "tc2pair") and M > 65536:
        pytest.skip("C3 shapes: shipped core only")
    rng = np.random.default_rng(M + K + N)
    x = rng.standard_normal((M, K), dtype=np.float32)
    w = (rng.standard_normal((K, N), dtype=np.float32) / np.float32(np.sqrt(K)))
    b = rng.standard_normal(N, dtype=np.float32) * np.float32(0.1)
    gy = rng.standard_normal((M, N), dtype=np.float32)
    xt, wt, bt = cu(x).requires_grad_(True), cu(w).requires_grad_(True), cu(b).requires_grad_(True)
    y = ops.DenseFn.apply(xt, wt, bt, ops.act_code(act))
    y.backward(cu(gy))
    torch.cuda.synchronize()
    yg = y.detach().cpu().numpy()
    rows = _sample_rows(M, 4096, rng)
    w64, aw = w.astype(np.float64), np.abs(w).astype(np.float64)

    # forward on the sampled rows
    xs = x[rows].astype(np.float64)
    ref = R.dense(x[rows], w, b, act, np.float64)
    pre_scale = np.abs(xs) @ aw + np.abs(b)
    err = np.abs(yg[rows] - ref)
    assert (err <= 1e-5 * pre_scale + 1e-7).all(), f"forward: worst {np.max(err / (pre_scale + 1e-30)):.3e} of sum|terms|"

    # backward with the GPU's own activation mask (mask-consistent)
    if act == "relu":
        gz = gy.astype(np.float64) * (yg > 0)
        # how many pre-activations are within rounding of 0 on the sample (documents why the fp64 mask cannot be used)
        z64 = xs @ w64 + b
        flips = int(((z64 > 0) != (yg[rows] > 0)).sum())
        print(f"relu mask flips fp64 vs gpu on {rows.size}x{N} sampled outputs: {flips}")
    else:
        gz = gy.astype(np.float64)
    agz = np.abs(gz)
    gx_ref = gz[rows] @ w64.T
    gx_err = np.abs(xt.grad[torch.from_numpy(rows).cuda()].cpu().numpy() - gx_ref)
    gx_scale = agz[rows] @ aw.T
    assert (gx_err <= 2e-5 * gx_scale + 1e-6).all(), f"dX: worst {np.max(gx_err / (gx_scale + 1e-30)):.3e}"
    # dW = X^T gZ over ALL M rows (split-K), db = column sums
    x64 = x.astype(np.float64)
    gw_ref = x64.T @ gz
    gw_scale = np.abs(x64).T @ agz
    gw_err = np.abs(wt.grad.cpu().numpy() - gw_ref)
    assert (gw_err <= 2e-5 * gw_scale + 1e-6).all(), f"dW: worst {np.max(gw_err / (gw_scale + 1e-30)):.3e}"
    gb_err = np.abs(bt.grad.cpu().numpy() - gz.sum(0))
    assert (gb_err <= 2e-5 * agz.sum(0) + 1e-6).all(), f"db: worst {np.max(gb_err / (agz.sum(0) + 1e-30)):.3e}"


@pytest.mark.parametrize("B,d,same", [(131072, 832, False), (131072, 832, True), (65536, 416, False)])
def test_cross_full_size(B, d, same, gemm_core):
    """Cross (dcn.py:70-88) at C3: x [131072, 832], full-matrix kernel; forward, dx0, dx, dW, db."""
    from deep_recommenders_b200 import ops
    if gemm_core != "tc2" and B > 65536:
        pytest.skip("C3 shapes: shipped core only")
    rng = np.random.default_rng(B + d + int(same))
    x0 = rng.standard_normal((B, d), dtype=np.float32)
    x = x0 if same else rng.standard_normal((B, d), dtype=np.float32)
    w = rng.standard_normal((d, d), dtype=np.float32) / np.float32(np.sqrt(d))
    b = rng.standard_normal(d, dtype=np.float32) * np.float32(0.1)
    g = rng.standard_normal((B, d), dtype=np.float32)
    alpha = 0.25
    t = lambda a: cu(a).requires_grad_(True)
    x0t, wt, bt = t(x0), t(w), t(b)
    xt = x0t if same else t(x)
    y = ops.CrossFn.apply(x0t, xt, wt, None, None, bt, alpha, same)
    y.backward(cu(g))
    torch.cuda.synchronize()
    rows = _sample_rows(B, 2048, rng)
    ridx = torch.from_numpy(rows).cuda()
    aw = np.abs(w).astype(np.float64)
    ref, prod = R.cross(x0[rows], x[rows], w, b, None, None, alpha, np.float64)
    ax, ax0 = np.abs(x[rows]).astype(np.float64), np.abs(x0[rows]).astype(np.float64)
    pscale = ax @ aw + alpha * ax + np.abs(b)
    err = np.abs(y.detach()[ridx].cpu().numpy() - ref)
    assert (err <= 1e-5 * (ax0 * pscale + ax) + 1e-7).all(), f"forward: worst {np.max(err / (ax0 * pscale + ax)):.3e}"
    gr = R.cross_grad(x0[rows], x[rows], g[rows], w, None, None, b, alpha, np.float64)
    ag = np.abs(g[rows]).astype(np.float64)
    ah = ag * ax0
    sx = ah @ aw.T + alpha * ah + ag
    if same:
        want_x0 = gr["gx0"] + gr["gx"]
        tol0 = 2e-5 * (ag * pscale + sx) + 1e-6
    else:
        want_x0 = gr["gx0"]
        tol0 = 2e-5 * (ag * pscale) + 1e-6
        ex = np.abs(xt.grad[ridx].cpu().numpy() - gr["gx"])
        assert (ex <= 2e-5 * sx + 1e-6).all(), f"dx: worst {np.max(ex / sx):.3e}"
    e0 = np.abs(x0t.grad[ridx].cpu().numpy() - want_x0)
    assert (e0 <= tol0).all(), f"dx0: worst {np.max(e0 / tol0):.3e} of the bound"
    # dW = X^T (g * x0) over all B rows; db = column sums of g * x0
    h = g.astype(np.float64) * x0.astype(np.float64)
    x64 = x.astype(np.float64)
    gw_ref = x64.T @ h
    gw_scale = np.abs(x64).T @ np.abs(h)
    ew = np.abs(wt.grad.cpu().numpy() - gw_ref)
    assert (ew <= 2e-5 * gw_scale + 1e-6).all(), f"dW: worst {np.max(ew / gw_scale):.3e}"
    eb = np.abs(bt.grad.cpu().numpy() - h.sum(0))
    assert (eb <= 2e-5 * np.abs(h).sum(0) + 1e-6).all()
