"""The staged epilogue of the wgmma GEMM (gemm_tc.cu), through dr_debug_gemm_epi.

A GEMM whose only output is C (EPI_STORE, EPI_BIAS_ACT, EPI_ACTGRAD, EPI_ATOMIC) writes each finished tile into shared
memory and stores it with TMA (a TMA reduce-add for split-K) when C is 16-B aligned with ldc % 4 == 0.  With ldc = N + 2
(even, so the register epilogue still uses float2 accesses, but not a multiple of 4) the same GEMM keeps the register
epilogue.  Both do the same arithmetic per element, so their outputs must be bit-identical, across the tile widths
(N = 32, 64, 416: a 32-column tail at BN = 128), the four operand layouts, M = 416 (a last m-tile with one live
warpgroup), an M that is not a multiple of 128, and the weight-plane kernel (plane cache on, N <= M / 16).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WS_BYTES = 256 << 20
EPI_STORE, EPI_BIAS_ACT, EPI_ATOMIC, EPI_ACTGRAD = 0, 1, 2, 3
ACTS = [0, 1, 2, 3]   # none, relu, sigmoid, tanh


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
    for k, v in saved.items():
        _lib.tune(k, v)
    _lib.enable_tensor_core_gemm()


def _gemm(L, A, B, M, N, K, ta, tb, ldc, epi, act=0, bias=None, aux=None, splitk=1, cache=False, C=None):
    from deep_recommenders_b200._lib import check
    if C is None:
        C = torch.full((M, ldc), float("nan"), device="cuda")
    check(L.dr_gemm_plane_cache(1 if cache else 0), "dr_gemm_plane_cache")
    try:
        check(L.dr_debug_gemm_epi(A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, int(ta), int(tb), ldc, epi, act,
                                  None if bias is None else bias.data_ptr(), None if aux is None else aux.data_ptr(),
                                  splitk, torch.cuda.current_stream().cuda_stream), "dr_debug_gemm_epi")
        torch.cuda.synchronize()
    finally:
        check(L.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
    return C


def _operands(M, N, K, ta, tb, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(K, M, device="cuda", generator=g) if ta else torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g) if tb else torch.randn(K, N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    y = torch.rand(M, N + 2, device="cuda", generator=g) * 2 - 0.5   # an activation output, some of it below zero
    return A, B, bias, y


def _assert_bits(got, want, what):
    diff = got.view(torch.int32) != want.view(torch.int32)
    assert not bool(diff.any()), f"{what}: {int(diff.sum())} elements differ"


def _cases():
    for M in (416, 1000):
        for N in (32, 64, 416):
            for ta in (0, 1):
                for tb in (0, 1):
                    yield pytest.param(M, N, ta, tb, False, id=f"M{M}-N{N}-ta{ta}tb{tb}")
    # weight-plane kernel: K-major A, N <= M / 16, more than one k-block
    for tb in (0, 1):
        yield pytest.param(8192 + 57, 416, 0, tb, True, id=f"wplanes-M8249-N416-tb{tb}")


@pytest.mark.parametrize("M, N, ta, tb, cache", list(_cases()))
def test_staged_matches_register_epilogue_bit_for_bit(lib, M, N, ta, tb, cache):
    K = 100   # four k-blocks, the last one partial
    A, B, bias, y = _operands(M, N, K, ta, tb, seed=M + N + 2 * ta + tb)
    modes = [(EPI_STORE, 0)] + [(EPI_BIAS_ACT, a) for a in ACTS] + [(EPI_ACTGRAD, a) for a in ACTS]
    for epi, act in modes:
        aux_reg = y if epi == EPI_ACTGRAD else None                       # pitch N + 2, as C
        aux_stg = y[:, :N].contiguous() if epi == EPI_ACTGRAD else None   # pitch N
        b = bias if epi == EPI_BIAS_ACT else None
        staged = _gemm(lib, A, B, M, N, K, ta, tb, N, epi, act, b, aux_stg, cache=cache)
        reg = _gemm(lib, A, B, M, N, K, ta, tb, N + 2, epi, act, b, aux_reg, cache=cache)[:, :N]
        assert not bool(torch.isnan(staged).any()), f"epi={epi} act={act}: staged output left unwritten"
        _assert_bits(staged, reg, f"epi={epi} act={act} M={M} N={N} ta={ta} tb={tb} cache={cache}")


@pytest.mark.parametrize("M, N", [(416, 256), (256, 32), (1000, 64)])
@pytest.mark.parametrize("splitk", [1, 5])
def test_staged_split_k_reduce_add_matches_float64(lib, M, N, splitk):
    """The weight-gradient form: A = X^T (stored [K, M]), a long K split over several CTAs, each tile's partial sum
    added into C by a TMA reduce-add.  Against float64 under the suite's norm-wise bound 1e-5 x (|A| @ |B|); the
    register form (ldc = N + 2, scalar red.global.add) is held to the same bound."""
    K = 4096
    g = torch.Generator(device="cuda").manual_seed(M + N + splitk)
    X = torch.randn(K, M, device="cuda", generator=g)
    G = torch.randn(K, N, device="cuda", generator=g)
    a64, b64 = X.double().cpu().numpy().T, G.double().cpu().numpy()
    ref, scale = a64 @ b64, np.abs(a64) @ np.abs(b64)
    for ldc in (N, N + 2):
        C = torch.zeros(M, ldc, device="cuda")
        _gemm(lib, X, G, M, N, K, 1, 0, ldc, EPI_ATOMIC, splitk=splitk, C=C)
        err = np.abs(C[:, :N].double().cpu().numpy() - ref)
        ok = err <= 1e-5 * scale
        assert ok.all(), f"ldc={ldc} splitk={splitk}: {int((~ok).sum())} entries off, worst {np.max(err / scale):.3e}"
