"""GPU tests of the multi-task kernels (dr_moe_mix_fwd / _bwd, dr_dense_grouped_fwd / _bwd) and of MMoE and ESMM.

Kernel results must sit within 1e-5 x (sum of |terms|) of a float64 reference; outputs are written between sentinel
guards so a store outside them is caught, and reruns must be bit-identical where the header promises it."""
import os

import numpy as np
import pytest
import torch

import mtl_oracle as O

pytestmark = pytest.mark.gpu
SENT = 1234.5
PAD = 4099
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mtl_golden.npz")


def _lib():
    from deep_recommenders_b200 import _lib
    return _lib.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Out:
    """An output of n floats between sentinel guards; .ptr stays a real address when n = 0."""

    def __init__(self, full, n):
        self.full, self.view = full, full[PAD:PAD + n]
        self.ptr = full.data_ptr() + 4 * PAD


def _guarded(n):
    full = torch.full((n + 2 * PAD,), SENT, device="cuda", dtype=torch.float32)
    return full, _Out(full, n)


def _check_guards(full, n):
    f = full.cpu().numpy()
    assert np.all(f[:PAD] == SENT) and np.all(f[PAD + n:] == SENT), "store outside the output"


def _dev(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.size == 0:           # B = 0: the entries still reject null pointers, so pass a real (unread) allocation
        return torch.zeros(1, device="cuda")
    return torch.from_numpy(a).cuda()


def _close(got, ref, scale, what, rel=1e-5):
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    bound = rel * scale + 4.8e-7 * np.abs(ref) + 1e-30
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.size} out of bound; worst err {err.max():.3g}")


# ---- dr_moe_mix ------------------------------------------------------------------------------------------------------
def mix_fwd(experts, logits, B, E, T, H):
    gfull, gates = _guarded(B * T * E)
    ofull, out = _guarded(B * T * H)
    rc = _lib().dr_moe_mix_fwd(experts.data_ptr(), logits.data_ptr(), B, E, T, H, gates.ptr, out.ptr, _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    _check_guards(gfull, B * T * E)
    _check_guards(ofull, B * T * H)
    return gates.view, out.view


def mix_bwd(experts, gates, g_out, B, E, T, H):
    efull, gex = _guarded(B * E * H)
    lfull, glog = _guarded(B * T * E)
    gptr = gates.data_ptr() if gates.numel() else experts.data_ptr()
    rc = _lib().dr_moe_mix_bwd(experts.data_ptr(), gptr, g_out.data_ptr(), B, E, T, H, gex.ptr, glog.ptr, _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    _check_guards(efull, B * E * H)
    _check_guards(lfull, B * T * E)
    return gex.view, glog.view


MIX_CASES = [  # E, T, H, B
    (1, 1, 1, 1), (2, 2, 32, 67), (3, 3, 5, 33), (8, 2, 128, 100), (32, 16, 33, 9), (32, 16, 1024, 3),
    (8, 16, 10, 41), (3, 1, 1024, 17), (2, 3, 33, 0), (1, 2, 128, 5), (32, 1, 10, 13), (2, 16, 1, 70),
]


@pytest.mark.parametrize("E,T,H,B", MIX_CASES)
def test_moe_mix_against_float64(E, T, H, B):
    rng = np.random.default_rng(E * 1000 + T * 10 + H)
    ex = rng.standard_normal((B, E, H)).astype(np.float32)
    lg = (rng.standard_normal((B, T, E)) * 2).astype(np.float32)
    go = rng.standard_normal((B, T, H)).astype(np.float32)
    d_ex, d_lg, d_go = _dev(ex.reshape(B, E * H)), _dev(lg.reshape(B, T * E)), _dev(go.reshape(B, T * H))
    gates, out = mix_fwd(d_ex, d_lg, B, E, T, H)
    gex, glog = mix_bwd(d_ex, gates, d_go, B, E, T, H)
    ex64, go64 = ex.astype(np.float64), go.astype(np.float64)
    rg, rout = O.mix_fwd(ex64, lg.astype(np.float64))
    g_got = gates.cpu().numpy().reshape(B, T, E)
    _close(g_got, rg, np.ones_like(rg), "gates")
    _close(out.cpu().numpy().reshape(B, T, H), rout, np.einsum("bte,beh->bth", rg, np.abs(ex64)), "out")
    # the backward uses the saved fp32 gates: the float64 reference does too
    g64 = g_got.astype(np.float64)
    rgex, rglog = O.mix_bwd(ex64, g64, go64)
    _close(gex.cpu().numpy().reshape(B, E, H), rgex, np.einsum("bte,bth->beh", g64, np.abs(go64)), "g_experts")
    dg_abs = np.einsum("bth,beh->bte", np.abs(go64), np.abs(ex64))
    _close(glog.cpu().numpy().reshape(B, T, E), rglog, g64 * (dg_abs + (g64 * dg_abs).sum(-1, keepdims=True)),
           "g_logits")
    # bit-identical reruns
    gates2, out2 = mix_fwd(d_ex, d_lg, B, E, T, H)
    gex2, glog2 = mix_bwd(d_ex, gates, d_go, B, E, T, H)
    for a, b in ((gates, gates2), (out, out2), (gex, gex2), (glog, glog2)):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


@pytest.mark.parametrize("E,T,H", [(3, 2, 10), (32, 16, 33)])
def test_moe_mix_softmax_extremes(E, T, H):
    B = 4
    rng = np.random.default_rng(1)
    ex = rng.standard_normal((B, E, H)).astype(np.float32)
    lg = np.zeros((B, T, E), np.float32)
    lg[0] = 7.25                                               # equal logits: uniform gates
    lg[1] = np.where(np.arange(E) % 2, 1e4, -1e4)              # +-1e4: no overflow, mass on the +1e4 experts
    lg[2] = -1e4
    lg[3, :, 0] = 1e4
    gates, out = mix_fwd(_dev(ex.reshape(B, -1)), _dev(lg.reshape(B, -1)), B, E, T, H)
    g = gates.cpu().numpy().reshape(B, T, E)
    o = out.cpu().numpy().reshape(B, T, H)
    assert np.isfinite(g).all() and np.isfinite(o).all()
    np.testing.assert_allclose(g[0], 1.0 / E, rtol=2e-7)
    np.testing.assert_allclose(g[2], 1.0 / E, rtol=2e-7)
    n_hi = E // 2
    if n_hi:
        np.testing.assert_allclose(g[1], np.broadcast_to(np.where(np.arange(E) % 2, 1.0 / n_hi, 0.0), (T, E)),
                                   rtol=2e-7)
    np.testing.assert_array_equal(g[3, :, 0], 1.0)
    np.testing.assert_array_equal(o[3], np.broadcast_to(ex[3, 0], (T, H)))


@pytest.mark.parametrize("T,H", [(1, 1), (3, 33), (16, 128)])
def test_moe_mix_single_expert_is_exact(T, H):
    B = 37
    rng = np.random.default_rng(2)
    ex = rng.standard_normal((B, H)).astype(np.float32)
    ex[::3, ::2] = -0.0                                        # signed zeros come through unchanged
    lg = (rng.standard_normal((B, T)) * 50).astype(np.float32)
    gates, out = mix_fwd(_dev(ex), _dev(lg), B, 1, T, H)
    np.testing.assert_array_equal(gates.cpu().numpy(), 1.0)
    o = out.cpu().numpy().reshape(B, T, H)
    for t in range(T):
        assert o[:, t].tobytes() == ex.tobytes()


def test_moe_mix_not_served_just_outside():
    x = torch.zeros(4096, device="cuda")
    lib = _lib()
    assert lib.dr_moe_mix_fwd(x.data_ptr(), x.data_ptr(), 2, 33, 1, 4, x.data_ptr(), x.data_ptr(), _stream()) == -3
    assert lib.dr_moe_mix_fwd(x.data_ptr(), x.data_ptr(), 2, 2, 17, 4, x.data_ptr(), x.data_ptr(), _stream()) == -3
    assert lib.dr_moe_mix_bwd(x.data_ptr(), x.data_ptr(), x.data_ptr(), 2, 33, 1, 4, x.data_ptr(), x.data_ptr(),
                              _stream()) == -3
    assert lib.dr_moe_mix_fwd(x.data_ptr(), x.data_ptr(), 2, 32, 16, 4, x.data_ptr(), x.data_ptr(), _stream()) == 0


# ---- dr_dense_grouped --------------------------------------------------------------------------------------------------
_ACTS = {0: None, 1: "relu", 2: "sigmoid", 3: "tanh"}


def grouped_fwd(x, w, b, M, G, K, N, act):
    yfull, y = _guarded(M * G * N)
    rc = _lib().dr_dense_grouped_fwd(x.data_ptr(), w.data_ptr(), None if b is None else b.data_ptr(), M, G, K, N, act,
                                     y.ptr, _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    _check_guards(yfull, M * G * N)
    return y.view


def grouped_bwd(x, w, y, gy, M, G, K, N, act, want_gx=True, want_gb=True):
    gz = torch.empty(M * G * N, device="cuda") if act else None
    xfull, gx = _guarded(M * G * K)
    wfull, gw = _guarded(G * K * N)
    bfull, gb = _guarded(G * N)
    rc = _lib().dr_dense_grouped_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), gy.data_ptr(), M, G, K, N, act,
                                     None if gz is None else gz.data_ptr(), gx.ptr if want_gx else None,
                                     gw.ptr, gb.ptr if want_gb else None, _stream())
    assert rc == 0, _lib().dr_last_error()
    torch.cuda.synchronize()
    for full, n in ((xfull, M * G * K), (wfull, G * K * N), (bfull, G * N)):
        _check_guards(full, n)
    return gx.view, gw.view, gb.view


@pytest.mark.parametrize("M,K,N", [(300, 64, 32), (257, 10, 1), (1000, 128, 256), (70, 33, 5)])
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_grouped_g1_equals_dense(M, K, N, act):
    from deep_recommenders_b200 import _lib as L
    L.ensure_gemm_workspace(M, K, N)
    rng = np.random.default_rng(M + K + N + act)
    x, w, b = _dev(rng.standard_normal((M, K))), _dev(rng.standard_normal((K, N)) * 0.2), _dev(rng.standard_normal(N))
    gy = _dev(rng.standard_normal((M, N)))
    lib = _lib()
    y1 = torch.empty(M * N, device="cuda")
    assert lib.dr_dense_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, act, y1.data_ptr(), _stream()) == 0
    y2 = grouped_fwd(x, w, b, M, 1, K, N, act)
    assert y1.cpu().numpy().tobytes() == y2.cpu().numpy().tobytes()
    gz = torch.empty(M * N, device="cuda")
    gx1, gw1, gb1 = torch.empty(M * K, device="cuda"), torch.empty(K * N, device="cuda"), torch.empty(N, device="cuda")
    assert lib.dr_dense_bwd(x.data_ptr(), w.data_ptr(), y1.data_ptr(), gy.data_ptr(), M, K, N, act, gz.data_ptr(),
                            gx1.data_ptr(), gw1.data_ptr(), gb1.data_ptr(), _stream()) == 0
    gx2, gw2, gb2 = grouped_bwd(x, w, y1, gy, M, 1, K, N, act)
    assert gx1.cpu().numpy().tobytes() == gx2.cpu().numpy().tobytes()
    # gw / gb: split-K and column atomics, equal up to the summation order
    gz64 = gy.cpu().double().numpy().reshape(M, N)
    if act:
        from mtl_oracle import _act_grad
        gz64 = gz64 * _act_grad(y1.cpu().double().numpy().reshape(M, N), _ACTS[act])
    x64 = x.cpu().double().numpy()
    _close(gw2.cpu().numpy(), gw1.cpu().double().numpy(), (np.abs(x64).T @ np.abs(gz64)).reshape(-1), "gw vs dense")
    _close(gb2.cpu().numpy(), gb1.cpu().double().numpy(), np.abs(gz64).sum(0), "gb vs dense")


GROUPED_CASES = [  # G, K, N, M
    (2, 1, 10, 257), (3, 10, 1, 130), (8, 32, 64, 1000), (2, 64, 32, 513), (3, 64, 64, 300), (8, 10, 10, 77),
    (2, 32, 1, 64), (8, 1, 1, 33), (3, 64, 10, 2048),
]


@pytest.mark.parametrize("G,K,N,M", GROUPED_CASES)
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_grouped_against_float64(G, K, N, M, act):
    from deep_recommenders_b200 import _lib as L
    L.ensure_gemm_workspace(M, G * K, G * N)
    rng = np.random.default_rng(G * 100 + K + N + act)
    x = rng.standard_normal((M, G * K)).astype(np.float32)
    w = (rng.standard_normal((G, K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal((G, N)).astype(np.float32)
    gy = rng.standard_normal((M, G * N)).astype(np.float32)
    y = grouped_fwd(_dev(x), _dev(w), _dev(b), M, G, K, N, act)
    gx, gw, gb = grouped_bwd(_dev(x), _dev(w), y, _dev(gy), M, G, K, N, act)
    yg = y.cpu().numpy().reshape(M, G, N).astype(np.float64)
    x64, w64, gy64 = x.astype(np.float64), w.astype(np.float64), gy.astype(np.float64)
    gxg = gx.cpu().numpy().reshape(M, G, K)
    gwg = gw.cpu().numpy().reshape(G, K, N)
    gbg = gb.cpu().numpy().reshape(G, N)
    for g in range(G):
        xg = x64[:, g * K:(g + 1) * K]
        ref = O._act(xg @ w64[g] + b[g], _ACTS[act])
        scale = np.abs(xg) @ np.abs(w64[g]) + np.abs(b[g])
        if act == 2:
            scale = scale * 0.25
        _close(yg[:, g], ref, scale, f"y group {g}")
        gz = gy64[:, g * N:(g + 1) * N] * O._act_grad(yg[:, g], _ACTS[act])     # from the kernel's own y
        _close(gxg[:, g], gz @ w64[g].T, np.abs(gz) @ np.abs(w64[g]).T, f"gx group {g}")
        _close(gwg[g], xg.T @ gz, np.abs(xg).T @ np.abs(gz), f"gw group {g}")
        _close(gbg[g], gz.sum(0), np.abs(gz).sum(0), f"gb group {g}")


@pytest.fixture(params=["ffma", "tc", "tc2"])
def gemm_core(request):
    """Runs a test under each GEMM core: FFMA (variant 0), wgmma on pre-split planes (1), wgmma with the split in the
    kernel (2, the default); the default is restored afterwards."""
    from deep_recommenders_b200 import _lib as L
    if request.param == "ffma":
        L.disable_tensor_core_gemm()
    else:
        L.enable_tensor_core_gemm(variant=1 if request.param == "tc" else 2)
    yield request.param
    L.enable_tensor_core_gemm()


def _launched(fn):
    """Names of the kernels fn() launched, from torch.profiler (an empty list where the profiler records none)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


@pytest.mark.parametrize("G,K,N,M", [(2, 64, 32, 513), (3, 64, 64, 300), (2, 32, 32, 512), (8, 32, 64, 1000)])
def test_grouped_under_every_gemm_core(gemm_core, G, K, N, M):
    """Shapes the wgmma path takes at G = 1, run under each core against float64.  Under the pre-split core a column
    block (pitch G*K or G*N wider than K) must not go through its flat split, which would read past the block's last
    row: those GEMMs go to FFMA, and only the weight gradient's transposing splits may run."""
    from deep_recommenders_b200 import _lib as L
    L.ensure_gemm_workspace(M, G * K, G * N)
    rng = np.random.default_rng(G + K + N + M)
    x = rng.standard_normal((M, G * K)).astype(np.float32)
    w = (rng.standard_normal((G, K, N)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal((G, N)).astype(np.float32)
    gy = rng.standard_normal((M, G * N)).astype(np.float32)
    dx, dw, db, dgy = _dev(x), _dev(w), _dev(b), _dev(gy)
    res = {}

    def run():
        res["y"] = grouped_fwd(dx, dw, db, M, G, K, N, 1)
        res["g"] = grouped_bwd(dx, dw, res["y"], dgy, M, G, K, N, 1)

    names = _launched(run) if gemm_core == "tc" else (run() or [])
    if gemm_core == "tc" and names:
        flat = [n for n in names if "split_tf32" in n and "transpose" not in n]
        assert not flat, f"flat split of a column block launched: {flat}"
    yg = res["y"].cpu().numpy().reshape(M, G, N).astype(np.float64)
    gx, gw, gb = (t.cpu().numpy() for t in res["g"])
    gxg, gwg, gbg = gx.reshape(M, G, K), gw.reshape(G, K, N), gb.reshape(G, N)
    for g in range(G):
        xg = x[:, g * K:(g + 1) * K].astype(np.float64)
        _close(yg[:, g], np.maximum(xg @ w[g] + b[g], 0), np.abs(xg) @ np.abs(w[g]) + np.abs(b[g]), f"{gemm_core} y {g}")
        gz = gy[:, g * N:(g + 1) * N].astype(np.float64) * (yg[:, g] > 0)
        _close(gxg[:, g], gz @ w[g].T, np.abs(gz) @ np.abs(w[g]).T, f"{gemm_core} gx {g}")
        _close(gwg[g], xg.T @ gz, np.abs(xg).T @ np.abs(gz), f"{gemm_core} gw {g}")
        _close(gbg[g], gz.sum(0), np.abs(gz).sum(0), f"{gemm_core} gb {g}")


def test_moe_mix_fn_rejects_bad_shapes():
    from deep_recommenders_b200 import ops
    ex = torch.zeros((4, 6), device="cuda")
    for logits, T in ((torch.zeros((4, 0), device="cuda"), 1), (torch.zeros((4, 3), device="cuda"), 2),
                      (torch.zeros((4, 4), device="cuda"), 1), (torch.zeros((5, 2), device="cuda"), 1),
                      (torch.zeros((4, 2), device="cuda"), 0)):
        with pytest.raises(ValueError, match="mixture of experts"):
            ops.MoEMixFn.apply(ex, logits, T)
    with pytest.raises(ValueError, match="mixture of experts"):
        ops.MoEMixFn.apply(torch.zeros((4, 0), device="cuda"), torch.zeros((4, 2), device="cuda"), 1)


def test_grouped_null_gx_and_bias():
    M, G, K, N = 200, 3, 32, 16
    rng = np.random.default_rng(9)
    x = rng.standard_normal((M, G * K)).astype(np.float32)
    w = rng.standard_normal((G, K, N)).astype(np.float32) * 0.1
    gy = rng.standard_normal((M, G * N)).astype(np.float32)
    y = grouped_fwd(_dev(x), _dev(w), None, M, G, K, N, 1)
    yg = y.cpu().numpy().reshape(M, G, N)
    for g in range(G):
        ref = np.maximum(x[:, g * K:(g + 1) * K].astype(np.float64) @ w[g], 0)
        _close(yg[:, g], ref, np.abs(x[:, g * K:(g + 1) * K]) @ np.abs(w[g]), "y without bias")
    gx, gw, _ = grouped_bwd(_dev(x), _dev(w), y, _dev(gy), M, G, K, N, 1, want_gx=False, want_gb=False)
    gwg = gw.cpu().numpy().reshape(G, K, N)
    for g in range(G):
        gz = gy[:, g * N:(g + 1) * N].astype(np.float64) * (yg[:, g] > 0)
        xg = x[:, g * K:(g + 1) * K].astype(np.float64)
        _close(gwg[g], xg.T @ gz, np.abs(xg).T @ np.abs(gz), "gw without gx")
    assert np.all(gx.cpu().numpy() == SENT)                     # gx = NULL: nothing written


# ---- MMoE / ESMM ------------------------------------------------------------------------------------------------------
def _columns(n):
    from deep_recommenders_b200 import feature_column as fc
    return [fc.numeric_column("C{}".format(i)) for i in range(n)]


@pytest.mark.parametrize("batch_size", [32, 64, 128, 512])
def test_reference_mmoe_and_esmm_tests(batch_size):
    from deep_recommenders.datasets import SyntheticForMultiTask
    from deep_recommenders.estimator.models.multi_task_learning import ESMM, MMoE
    columns = _columns(100)
    mmoe = MMoE(columns, num_tasks=2, num_experts=2, task_hidden_units=[32, 10], expert_hidden_units=[64, 32])
    esmm = ESMM(columns, hidden_units=[32, 10])
    dataset = SyntheticForMultiTask(5000)
    x, y = next(iter(dataset.input_fn(batch_size=batch_size)))
    y_pred = mmoe(x)
    assert len(y_pred) == 2
    assert tuple(y_pred[0].shape) == (batch_size, 1) and tuple(y_pred[1].shape) == (batch_size, 1)
    p_cvr, p_ctr, p_ctcvr = esmm(x)
    for p in (p_cvr, p_ctr, p_ctcvr):
        assert tuple(p.shape) == (batch_size, 1) and torch.isfinite(p).all()
    assert torch.equal(p_ctcvr, p_ctr * p_cvr)


def _load_mmoe(z, k, device="cuda"):
    from deep_recommenders.estimator.models.multi_task_learning import MMoE
    T, E = (int(v) for v in z[k + "_args"])
    eu, tu = [int(u) for u in z[k + "_expert_units"]], [int(u) for u in z[k + "_task_units"]]
    eact, tact = (str(a) for a in z[k + "_acts"])
    x = z[k + "_x"]
    m = MMoE(_columns(x.shape[1]), num_tasks=T, num_experts=E, expert_hidden_units=eu, task_hidden_units=tu,
             expert_hidden_activation=eact, task_hidden_activation=tact, device=device)
    ws, bs = O.golden_weights(z, k)
    ex_idx, gate_idx, task_idx = O.mmoe_layout(E, T, len(eu), len(tu) + 1)
    used = [i for ix in ex_idx for i in ix] + gate_idx[:T] + [i for ix in task_idx for i in ix]
    views = m.dense_views()
    assert len(views) == len(used)
    with torch.no_grad():
        for (kv, bv), i in zip(views, used):
            kv.copy_(torch.from_numpy(ws[i].astype(np.float32)))
            if bv is not None:
                bv.copy_(torch.from_numpy(bs[i].astype(np.float32)))
    feats = {"C{}".format(i): x[:, i:i + 1] for i in range(x.shape[1])}
    return m, feats, (E, T, eu, tu, eact, tact), used


def _load_esmm(z, k):
    from deep_recommenders.estimator.models.multi_task_learning import ESMM
    x = z[k + "_x"]
    m = ESMM(_columns(x.shape[1]), hidden_units=[int(u) for u in z[k + "_hidden_units"]], activation=str(z[k + "_act"]))
    ws, bs = O.golden_weights(z, k)
    with torch.no_grad():
        for (kv, bv), w, b in zip(m.dense_views(), ws, bs):
            kv.copy_(torch.from_numpy(w.astype(np.float32)))
            bv.copy_(torch.from_numpy(b.astype(np.float32)))
    return m, {"C{}".format(i): x[:, i:i + 1] for i in range(x.shape[1])}


def _grad_views(model):
    """dense_views() of the parameters' gradients (parameters swapped for their .grad while reading)."""
    params = list(model.parameters())
    saved = [p.data for p in params]
    for p in params:
        p.data = p.grad if p.grad is not None else torch.zeros_like(p)
    try:
        return [(k.clone(), None if b is None else b.clone()) for k, b in model.dense_views()]
    finally:
        for p, d in zip(params, saved):
            p.data = d


@pytest.mark.parametrize("case", ["ref", "e3t2", "e1t1", "e4t1", "e5t3"])
def test_mmoe_golden_outputs_and_gradients(case):
    z = np.load(GOLDEN)
    m, feats, (E, T, eu, tu, eact, tact), used = _load_mmoe(z, f"f32_mmoe_{case}")
    outs = m(feats)
    assert len(outs) == T
    for t in range(T):
        np.testing.assert_allclose(outs[t].detach().cpu().numpy(), z[f"f32_mmoe_{case}_out{t}"], rtol=1e-5, atol=1e-5)
    # gradients against the float64 oracle on the same (fp32-rounded) weights
    x = z[f"f32_mmoe_{case}_x"].astype(np.float64)
    ws, bs = O.golden_weights(z, f"f32_mmoe_{case}")
    ws = [w.astype(np.float64) for w in ws]
    bs = [None if b is None else b.astype(np.float64) for b in bs]
    inputs = x[:, O.input_order(x.shape[1])]
    routs, cache = O.mmoe_forward(inputs, ws, bs, E, T, eu, tu, eact, tact)
    rng = np.random.default_rng(3)
    g = [rng.standard_normal((x.shape[0], 1)) for _ in range(T)]
    for t in range(T):
        np.testing.assert_allclose(outs[t].detach().cpu().numpy(), routs[t], rtol=1e-5, atol=1e-5)
    _, gws, gbs = O.mmoe_backward(cache, g)
    sum((o * _dev(gg)).sum() for o, gg in zip(outs, g)).backward()
    for (gk, gbv), i in zip(_grad_views(m), used):
        ref = gws[i]
        tol = 1e-4 * (np.abs(ref).max() + 1e-3)
        np.testing.assert_allclose(gk.cpu().numpy(), ref, rtol=1e-4, atol=tol, err_msg=f"kernel {i}")
        if gbv is not None:
            np.testing.assert_allclose(gbv.cpu().numpy(), gbs[i], rtol=1e-4, atol=1e-4 * (np.abs(gbs[i]).max() + 1e-3),
                                       err_msg=f"bias {i}")


@pytest.mark.parametrize("case", ["ref", "small", "linear"])
def test_esmm_golden_outputs_and_gradients(case):
    z = np.load(GOLDEN)
    k = f"f32_esmm_{case}"
    m, feats = _load_esmm(z, k)
    p_cvr, p_ctr, p_ctcvr = m(feats)
    assert torch.equal(p_ctcvr, p_ctr * p_cvr)
    for name, p in (("p_cvr", p_cvr), ("p_ctr", p_ctr), ("p_ctcvr", p_ctcvr)):
        np.testing.assert_allclose(p.detach().cpu().numpy(), z[f"{k}_{name}"], rtol=1e-5, atol=1e-6)
    x = z[k + "_x"].astype(np.float64)
    ws, bs = O.golden_weights(z, k)
    hu = [int(u) for u in z[k + "_hidden_units"]]
    _, cache = O.esmm_forward(x[:, O.input_order(x.shape[1])], [w.astype(np.float64) for w in ws],
                              [b.astype(np.float64) for b in bs], hu, str(z[k + "_act"]))
    rng = np.random.default_rng(4)
    g = [rng.standard_normal((x.shape[0], 1)) for _ in range(3)]
    _, gws, gbs = O.esmm_backward(cache, *g)
    sum((p * _dev(gg)).sum() for p, gg in zip((p_cvr, p_ctr, p_ctcvr), g)).backward()
    for i, (gk, gbv) in enumerate(_grad_views(m)):
        np.testing.assert_allclose(gk.cpu().numpy(), gws[i], rtol=1e-4, atol=1e-4 * (np.abs(gws[i]).max() + 1e-3))
        np.testing.assert_allclose(gbv.cpu().numpy(), gbs[i], rtol=1e-4, atol=1e-4 * (np.abs(gbs[i]).max() + 1e-3))


def test_towers_are_independent():
    from deep_recommenders.estimator.models.multi_task_learning import ESMM, MMoE
    cols = _columns(16)
    rng = np.random.default_rng(0)
    feats = {"C{}".format(i): rng.standard_normal((64, 1)).astype(np.float32) for i in range(16)}
    m = MMoE(cols, num_tasks=2, num_experts=3, expert_hidden_units=[8, 8], task_hidden_units=[4], seed=0)
    outs = m(feats)
    outs[0].sum().backward()                                    # only task 0 receives a gradient
    gv = _grad_views(m)
    n_ex = 3 * 2
    assert all(float(k.abs().sum()) > 0 for k, _ in gv[:n_ex])             # every expert trains
    assert float(gv[n_ex][0].abs().sum()) > 0 and float(gv[n_ex + 1][0].abs().sum()) == 0   # gate 0 only
    assert all(float(k.abs().sum()) == 0 for k, _ in gv[n_ex + 2 + 2:])    # task tower 1 untouched
    ex = m._experts(torch.from_numpy(np.concatenate([feats[f"C{i}"] for i in sorted(range(16), key=str)], 1)).cuda())
    blocks = ex.detach().cpu().numpy().reshape(64, 3, 8)
    assert not np.array_equal(blocks[:, 0], blocks[:, 1]) and not np.array_equal(blocks[:, 1], blocks[:, 2])
    e = ESMM(cols, [8], seed=1)
    p_cvr, p_ctr, _ = e(feats)
    assert not torch.equal(p_cvr, p_ctr)
    p_cvr.sum().backward()
    gv = _grad_views(e)
    assert float(gv[0][0].abs().sum()) > 0 and all(float(k.abs().sum()) == 0 for k, _ in gv[2:])


def test_short_training_run_loss_falls():
    from deep_recommenders.datasets import SyntheticForMultiTask
    from deep_recommenders.estimator.models.multi_task_learning import MMoE
    np.random.seed(7)
    m = MMoE(_columns(100), num_tasks=2, num_experts=2, task_hidden_units=[32, 10], expert_hidden_units=[64, 32],
             seed=7)
    opt = torch.optim.Adam(list(m.parameters()), lr=0.01, eps=1e-8)
    hist = []
    for x, y in SyntheticForMultiTask(256 * 80).input_fn(batch_size=256):
        outs = m(x)
        l0 = ((outs[0] - _dev(y["labels0"]).unsqueeze(1)) ** 2).mean()
        l1 = ((outs[1] - _dev(y["labels1"]).unsqueeze(1)) ** 2).mean()
        opt.zero_grad(set_to_none=True)
        (l0 + l1).backward()
        opt.step()
        hist.append((float(l0.detach()), float(l1.detach())))
    h = np.asarray(hist)
    assert len(h) == 80
    assert h[-10:, 0].mean() < 0.8 * h[:10, 0].mean() and h[-10:, 1].mean() < 0.8 * h[:10, 1].mean(), h[::10]
