"""Tail tiles and the weight-plane kernel of the wgmma GEMM (gemm_tc.cu), through the C-ABI.

* N tail: the weight-plane kernel runs a tile whose valid width is at most 32 (64) columns with m64n32k8 (m64n64k8)
  MMAs.  Its output must be bit-identical to the same GEMM with B zero-padded to a multiple of 128 columns, where no
  tile has a tail.
* M tail: a consumer warpgroup whose 64 rows all lie past M skips the tile.  Output must be bit-identical to the same
  GEMM with A zero-padded to a multiple of 128 rows.
* Weight planes: with the plane cache on (as inside a train step), the forward and dX GEMMs of a Dense layer over a
  batch (128-wide tiles, more than one k-block) take B's hi / lo planes from the workspace (gemm_tc_wplanes_kernel)
  instead of splitting B on every tile.  The split is the same, so the output is bit-identical to the in-kernel split
  with the cache off.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

RELU = 1
WS_BYTES = 256 << 20
M_BIG = 16384 + 57      # N * 16 <= M for every padded N below: the weight-plane kernel, with a 57-row M tail
M_SMALL = 416           # the layer-0 dW's M: one warpgroup of the last m-tile has no row in range


@pytest.fixture
def lib():
    from deep_recommenders_b200 import _lib
    L = _lib.load()
    saved = {k: _lib.tune_get(k) for k in ("gemm_variant", "gemm_bn", "tc_min_n")}
    if _lib._workspace is None or _lib._workspace.numel() < WS_BYTES:
        _lib.set_workspace(WS_BYTES)
    _lib.enable_tensor_core_gemm(variant=2)
    yield L
    _lib.check(L.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
    _lib.tune("gemm_splitk", 0)
    for k, v in saved.items():
        _lib.tune(k, v)
    _lib.enable_tensor_core_gemm()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _launched(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


def _with_cache(L, on, fn):
    """fn() with the plane cache on (fresh, as at the start of a train step) or off."""
    from deep_recommenders_b200._lib import check
    check(L.dr_gemm_plane_cache(1 if on else 0), "dr_gemm_plane_cache")
    try:
        return fn()
    finally:
        check(L.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bits(got, want, what):
    diff = (_bits(got) != _bits(want))
    assert not bool(diff.any()), f"{what}: {int(diff.sum())} elements differ, max |d| " \
                                 f"{float((got - want).abs().max())}"


def _pad_cols(t, n):
    out = torch.zeros(t.shape[0], n, device=t.device, dtype=t.dtype)
    out[:, :t.shape[1]] = t
    return out


def _pad_rows(t, m):
    out = torch.zeros(m, *t.shape[1:], device=t.device, dtype=t.dtype)
    out[:t.shape[0]] = t
    return out


def _up(v, q=128):
    return (v + q - 1) // q * q


def _dense(L, epi, x, w, b, gz, prev_y):
    """One GEMM of a Dense layer with input x [M, Kd], kernel w [Kd, Nd]:
       fwd:   y  = relu(x @ w + b)                        GEMM M x Nd x Kd, B = w stored [K, N]
       dx:    gx = gz @ w^T                               GEMM M x Kd x Nd, B = w stored [N, K]
       chain: gx = (gz @ w^T) * relu'(prev_y)             the same with the activation-gradient epilogue"""
    from deep_recommenders_b200._lib import check
    M, Kd = x.shape
    Nd = w.shape[1]
    if epi == "fwd":
        y = torch.empty(M, Nd, device="cuda")
        check(L.dr_dense_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), M, Kd, Nd, RELU, y.data_ptr(), _st()), "fwd")
        return y
    gx = torch.empty(M, Kd, device="cuda")
    if epi == "dx":
        check(L.dr_dense_bwd(x.data_ptr(), w.data_ptr(), None, gz.data_ptr(), M, Kd, Nd, 0, None, gx.data_ptr(), None,
                             None, _st()), "dx")
    else:
        check(L.dr_dense_bwd_chain(x.data_ptr(), w.data_ptr(), None, gz.data_ptr(), M, Kd, Nd, 0, None, gx.data_ptr(),
                                   None, None, prev_y.data_ptr(), RELU, _st()), "chain")
    return gx


def _operands(M, Kd, Nd, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, Kd, device="cuda", generator=g)
    w = torch.randn(Kd, Nd, device="cuda", generator=g) / Kd ** 0.5
    b = torch.randn(Nd, device="cuda", generator=g)
    gz = torch.randn(M, Nd, device="cuda", generator=g)
    prev_y = torch.randn(M, Kd, device="cuda", generator=g).relu_()
    return x, w, b, gz, prev_y


def _wplanes_expected(epi, M, Kd, Nd):
    """The Python mirror of the weight-plane selection: 64 < GEMM N <= GEMM M / 16 and GEMM K > 32 (every GEMM here has
    a K-major A, a pitch-K B and the plane cache on)."""
    n, k = (Nd, Kd) if epi == "fwd" else (Kd, Nd)
    return 64 < n and n * 16 <= M and k > 32


@pytest.mark.parametrize("K", [36, 252])
@pytest.mark.parametrize("N", [32, 96, 160, 416, 832])
@pytest.mark.parametrize("M", [M_SMALL, M_BIG])
@pytest.mark.parametrize("epi", ["fwd", "dx", "chain"])
def test_n_tail_matches_zero_padded_b(lib, epi, M, N, K):
    """The GEMM's output width is N and its contraction K: a forward has Dense units N over inputs K, a dX has inputs N
    and units K.  Padding the GEMM's N to 128 with zero weights removes the tail tile."""
    Kd, Nd = (K, N) if epi == "fwd" else (N, K)
    x, w, b, gz, prev_y = _operands(M, Kd, Nd, seed=M + N + K)
    Np = _up(N)
    if epi == "fwd":
        xp, wp, bp, gzp, pyp = x, _pad_cols(w, Np), _pad_cols(b[None], Np)[0], gz, prev_y
    else:
        xp, wp, bp, gzp, pyp = _pad_cols(x, Np), _pad_rows(w, Np), b, gz, _pad_cols(prev_y, Np)
    names = _launched(lambda: _with_cache(lib, True, lambda: _dense(lib, epi, x, w, b, gz, prev_y)))
    assert any("gemm_tc_wplanes_kernel" in n for n in names) == _wplanes_expected(epi, M, Kd, Nd), names
    got = _with_cache(lib, True, lambda: _dense(lib, epi, x, w, b, gz, prev_y))
    want = _with_cache(lib, True, lambda: _dense(lib, epi, xp, wp, bp, gzp, pyp))[:, :N]
    _assert_bits(got, want, f"{epi} M={M} N={N} K={K}")
    # and the in-kernel split (cache off) computes the same bits
    _assert_bits(_with_cache(lib, False, lambda: _dense(lib, epi, x, w, b, gz, prev_y)), got, "cache off")


@pytest.mark.parametrize("cache", [False, True])
@pytest.mark.parametrize("M", [M_SMALL, 4096 + 57, M_BIG])
@pytest.mark.parametrize("epi", ["fwd", "dx", "chain"])
def test_m_tail_matches_zero_padded_a(lib, epi, M, cache):
    """From M = 4096 + 57 on, the cached forward and dX run the weight-plane kernel, with a tile of one live warpgroup."""
    Kd, Nd = 256, 96
    x, w, b, gz, prev_y = _operands(M, Kd, Nd, seed=M)
    Mp = _up(M)
    got = _with_cache(lib, cache, lambda: _dense(lib, epi, x, w, b, gz, prev_y))
    want = _with_cache(lib, cache, lambda: _dense(lib, epi, _pad_rows(x, Mp), w, b, _pad_rows(gz, Mp),
                                                  _pad_rows(prev_y, Mp)))[:M]
    _assert_bits(got, want, f"{epi} M={M} cache={cache}")


@pytest.mark.parametrize("Kd", [416, 4 * 128 + 36])
def test_m_tail_weight_gradient(lib, Kd):
    """The dW gW[Kd, N] = x^T gz has GEMM M = Kd (A transposed): with Kd = 416 the last m-tile's second warpgroup has
    no row in range.  One k-split, so its single reduction per element is deterministic."""
    from deep_recommenders_b200 import _lib
    from deep_recommenders_b200._lib import check
    _lib.tune("gemm_splitk", 1)
    M, N = 2048, 256
    x, w, b, gz, _ = _operands(M, Kd, N, seed=Kd)
    Kp = _up(Kd)

    def dw(xx):
        gw = torch.empty(xx.shape[1], N, device="cuda")
        check(lib.dr_dense_bwd(xx.data_ptr(), w.data_ptr(), None, gz.data_ptr(), M, xx.shape[1], N, 0, None, None,
                               gw.data_ptr(), None, _st()), "dw")
        return gw

    got = dw(x)
    _assert_bits(got, dw(_pad_cols(x, Kp))[:Kd], f"dw Kd={Kd}")
    ref = x.double().T @ gz.double()
    bound = x.double().abs().T @ gz.double().abs()
    assert bool(((got.double() - ref).abs() <= 1e-5 * bound + 1e-30).all()), "dw against float64"


# the GEMMs of the C2 tower (416 -> 256 -> 32) and of the 3328 -> 512 layer: the layer-1 forward (N = 32) and dX (K = 32)
# of C2 stay on the splitter kernel
_STEP_GEMMS = [("fwd", 416, 256), ("dx", 416, 256), ("chain", 416, 256), ("fwd", 256, 32), ("chain", 256, 32),
               ("fwd", 3328, 512), ("dx", 3328, 512)]


@pytest.mark.parametrize("epi,Kd,Nd", _STEP_GEMMS)
def test_weight_planes_bit_identical_to_in_kernel_split(lib, epi, Kd, Nd):
    M = 8192 if Kd < 1000 else 65536
    x, w, b, gz, prev_y = _operands(M, Kd, Nd, seed=Kd + Nd)
    on = _launched(lambda: _with_cache(lib, True, lambda: _dense(lib, epi, x, w, b, gz, prev_y)))
    off = _launched(lambda: _with_cache(lib, False, lambda: _dense(lib, epi, x, w, b, gz, prev_y)))
    assert any("gemm_tc_wplanes_kernel" in n for n in on) == _wplanes_expected(epi, M, Kd, Nd), on
    assert not any("gemm_tc_wplanes_kernel" in n for n in off), off
    _assert_bits(_with_cache(lib, True, lambda: _dense(lib, epi, x, w, b, gz, prev_y)),
                 _with_cache(lib, False, lambda: _dense(lib, epi, x, w, b, gz, prev_y)), f"{epi} {Kd}x{Nd}")


def test_deepfm_step_runs_weight_planes_for_forward_and_dx(lib):
    """One eager step of the C2 model shape: the layer-0 forward and dX GEMMs take the weight-plane kernel; the layer-1
    forward and dX and both weight gradients keep the splitter kernel."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    S, D, rows, B = 26, 16, 1000, 8192
    cols = [fc.categorical_column_with_identity(f"c{i}", rows) for i in range(S)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=[256, 32], seed=0, device="cuda")
    tr = DeepFMTrainStep(model, batch_size=B, lr=0.01, use_graph=False)
    rng = np.random.default_rng(0)
    ids = torch.from_numpy(rng.integers(0, rows, (B, S))).cuda()
    labels = torch.from_numpy(rng.integers(0, 2, B).astype(np.float32)).cuda()
    tr.step(ids, labels)
    names = _launched(lambda: tr.step(ids, labels))
    assert sum("gemm_tc_wplanes_kernel" in n for n in names) == 2, names
    assert sum("gemm_tc_kernel" in n for n in names) == 4, names
    assert np.isfinite(float(tr.loss))
