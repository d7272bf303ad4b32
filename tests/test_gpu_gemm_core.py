"""Conformance suite of the fp32 GEMM core (gemm.cu FFMA, gemm_tc.cu wgmma 3xTF32) through the C-ABI.

Every case checks three things:
  * the numbers: against a float64 oracle, either under the norm-wise bound 1e-5 x (|A| @ |B|) elementwise (random
    normals with full 24-bit mantissas, which single-pass TF32 cannot meet) or bit for bit (operands whose products and
    sums are exact in fp32, so any indexing, swizzle, tail or lo-plane error shows however small it is);
  * the memory: operands sit between NaN guards (a read outside an operand poisons the result) and C between
    sentinels (a store outside [M, N] is caught);
  * the dispatch: the kernels torch.profiler saw launch are the ones a Python mirror of gemm_tc_eligible and of the
    tile-width choice of gemm_tc_launch predicts (gemm_tc_kernel<BN, A_MN, B_MN, PRESPLIT> or sgemm_kernel).
The knobs gemm_variant, gemm_bn, tc_min_n, tc_stages, tc_l2_promo and gemm_splitk are set per case and restored.
"""
import re
import time
import warnings

import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu

WS_BYTES = 256 << 20            # variant 1 workspace: holds the planes of every shape below with the cache off
PAD = 64                        # NaN floats before and after every operand (256 B: keeps the operand 16-B aligned)
SENTINEL = np.int32(0x7FC0DEAD)  # a quiet NaN with a payload no kernel writes
LAYOUTS = [(0, 0), (0, 1), (1, 0), (1, 1)]
BNS = [0, 32, 64, 128]
MS = [64, 65, 127, 128, 129, 1000]
NS = [32, 36, 64, 68, 100, 128, 132, 260]
KS = [32, 36, 100, 4100]
KS_ODD = [33, 1001]             # a k-tail the TMA zero-fills where K is the row count of an operand
_SEEN = set()                   # gemm_tc_kernel instantiations seen launching in this module


# ---- knobs ----------------------------------------------------------------------------------------------------------
_READABLE = ("gemm_variant", "gemm_bn", "tc_min_n")
_SOURCE_DEFAULTS = {"tc_stages": 0, "gemm_splitk": 0, "tc_l2_promo": 256, "tc_dw_share": 0}


@pytest.fixture
def knobs():
    """knobs(name=value, ...) sets GEMM knobs for the test; the readable ones go back to the value read before, the
    write-only ones to their source defaults.  (l2_fetch_granularity is never touched: it sets a device limit.)"""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    saved = {k: _lib.tune_get(k) for k in _READABLE}

    def set_knobs(**kv):
        variant = kv.pop("gemm_variant", None)
        if variant == 0:
            _lib.disable_tensor_core_gemm()
        elif variant is not None:
            if variant == 1 and (_lib._workspace is None or _lib._workspace.numel() < WS_BYTES):
                _lib.set_workspace(WS_BYTES)
            _lib.enable_tensor_core_gemm(variant=variant)
        for k, v in kv.items():
            _lib.tune(k, v)

    yield set_knobs
    _lib.check(lib.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
    for k, v in _SOURCE_DEFAULTS.items():
        _lib.tune(k, v)
    for k, v in saved.items():
        _lib.tune(k, v)
    _lib.enable_tensor_core_gemm()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- dispatch -------------------------------------------------------------------------------------------------------
_B = r"(true|false|\(bool\)[01]|[01])"
_TC_RE = re.compile(r"gemm_tc_kernel<(\d+), " + _B + ", " + _B + ", " + _B + ">")
_TC_MANGLED_RE = re.compile(r"gemm_tc_kernelILi(\d+)ELb([01])ELb([01])ELb([01])E")
_cupti = {}


def _truth(s):
    return s in ("true", "(bool)1", "1")


def _gemm_kernels(names):
    """{("tc", BN, A_MN, B_MN, PRESPLIT) | ("sgemm",)} of a list of launched kernel names"""
    out = set()
    for n in names:
        m = _TC_RE.search(n)
        if m:
            out.add(("tc", int(m.group(1)), _truth(m.group(2)), _truth(m.group(3)), _truth(m.group(4))))
            continue
        m = _TC_MANGLED_RE.search(n)
        if m:
            out.add(("tc", int(m.group(1)), m.group(2) == "1", m.group(3) == "1", m.group(4) == "1"))
        elif "sgemm_kernel" in n:
            out.add(("sgemm",))
    _SEEN.update(k for k in out if k[0] == "tc")
    return out


def launched(fn, attempts=3):
    """Run fn() under torch.profiler (CUDA activity) and return the names of what it launched.  The profiler keeps only
    kernel records whose device timestamps fall inside its host-clock window and now and then drops those of a short
    window, so the window is padded by a few milliseconds on both sides, and fn (idempotent for every caller that
    passes attempts > 1) runs again until a GEMM kernel shows up."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.002)
            fn()
            torch.cuda.synchronize()
            time.sleep(0.002)
        names = [e.name for e in prof.events()]
        if _gemm_kernels(names):
            break
    return names


def cupti_works():
    """Whether the profiler reports kernel launches here at all (probed once with a torch kernel)."""
    if "ok" not in _cupti:
        x = torch.ones(1024, device="cuda")
        names = launched(lambda: x.mul_(2), attempts=1)
        _cupti["ok"] = any("elementwise" in n.lower() or "kernel" in n.lower() for n in names)
        if not _cupti["ok"]:
            warnings.warn("torch.profiler returned no CUDA kernel records: dispatch assertions are skipped, the numeric "
                          "checks still run")
    return _cupti["ok"]


def check_dispatch(names, expected, what=""):
    """The GEMM kernels in `names` are exactly `expected`.  Skipped, with a warning, where the profiler recorded no GEMM
    kernel at all: C was checked by then, so some GEMM kernel did run and only its record is missing."""
    if not cupti_works():
        return
    got = _gemm_kernels(names)
    if not got:
        warnings.warn(f"{what}: the profiler recorded no GEMM kernel for this call; its dispatch is not checked")
        return
    assert got == set(expected), f"{what}: launched {sorted(got)}, expected {sorted(set(expected))}"


def _round4(v):
    return (v + 3) // 4 * 4


def expected_kernel(M, N, K, ta, tb, lda, ldb, a_ptr=0, b_ptr=0):
    """Python mirror of gemm_tc_eligible + the tile-width choice of gemm_tc_launch (cache off)."""
    from deep_recommenders_b200 import _lib
    variant, bn_knob, min_n = (_lib.tune_get(k) for k in _READABLE)
    ffma = ("sgemm",)
    if variant not in (1, 2):
        return ffma
    if N < min_n or N % 4 or M < 64 or K < 32:
        return ffma
    if variant == 2:
        if lda % 4 or a_ptr % 16 or ldb % 4 or b_ptr % 16:
            return ffma
    else:
        if not ta and (lda % 4 or a_ptr % 16):
            return ffma
        if tb and (ldb % 4 or b_ptr % 16):
            return ffma
        ws = 0 if _lib._workspace is None else _lib._workspace.numel()
        ae = M * (lda if not ta else _round4(K))
        be = N * (ldb if tb else _round4(K))
        if 4 * 2 * (ae + be) > ws:
            return ffma
    bn = 32 if N <= 32 else (64 if N <= 64 else 128)
    if bn_knob in (32, 64):
        bn = bn_knob
    if variant == 2:
        return ("tc", bn, bool(ta), not tb, False)
    return ("tc", bn, False, False, True)


# ---- harness --------------------------------------------------------------------------------------------------------
def _guarded(x, offset_bytes=0):
    """x (numpy float32) copied into a NaN-filled device buffer; returns (buffer, pointer to x's first element)"""
    off = PAD + offset_bytes // 4
    buf = torch.full((off + x.size + PAD,), float("nan"), device="cuda")
    buf[off:off + x.size] = torch.from_numpy(np.ascontiguousarray(x, np.float32).reshape(-1)).cuda()
    return buf, buf.data_ptr() + 4 * off


def run_gemm(A, B, M, N, K, ta, tb, c_offset=0, a_offset=0, b_offset=0):
    """C = op(A) @ op(B) through dr_debug_gemm.  A is stored [K, M] if ta else [M, K]; B is stored [N, K] if tb else
    [K, N].  Operands sit between NaN guards, C between sentinels that must survive the call.  Offsets are in bytes
    (c_offset = 4 puts C off 8-B alignment: the scalar-store epilogue).  Returns (C, launched kernel names, expected
    dispatch)."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    assert A.shape == ((K, M) if ta else (M, K)) and B.shape == ((N, K) if tb else (K, N))
    abuf, ap = _guarded(A, a_offset)
    bbuf, bp = _guarded(B, b_offset)
    c0 = PAD + c_offset // 4
    cbuf = torch.full((c0 + M * N + PAD,), int(SENTINEL), dtype=torch.int32, device="cuda")
    cp = cbuf.data_ptr() + 4 * c0
    expect = expected_kernel(M, N, K, ta, tb, M if ta else K, K if tb else N, ap, bp)
    names = launched(lambda: _lib.check(lib.dr_debug_gemm(ap, bp, cp, M, N, K, int(ta), int(tb), _stream()),
                                        "dr_debug_gemm"))
    bits = cbuf.cpu().numpy()
    outside = np.concatenate([bits[:c0], bits[c0 + M * N:]])
    assert (outside == SENTINEL).all(), f"store outside C: {int((outside != SENTINEL).sum())} sentinels overwritten"
    return bits[c0:c0 + M * N].view(np.float32).reshape(M, N), names, expect


def logical(A, B, ta, tb):
    a = A.astype(np.float64)
    b = B.astype(np.float64)
    return (a.T if ta else a), (b.T if tb else b)


def assert_bound(C, a64, b64, what=""):
    ref = a64 @ b64
    scale = np.abs(a64) @ np.abs(b64)
    err = np.abs(C.astype(np.float64) - ref)
    ok = err <= 1e-5 * scale
    assert ok.all(), f"{what}: {int((~ok).sum())} entries off, worst {np.nanmax(err / scale):.3e} of sum|terms|"


def assert_exact(C, ref, what=""):
    ref32 = ref.astype(np.float32)
    assert np.array_equal(ref32.astype(np.float64), ref), "oracle not exact in fp32: bad probe"
    bad = C != ref32
    assert not bad.any(), f"{what}: {int(bad.sum())} entries differ, first at {np.argwhere(bad)[0].tolist()}"


def normal(rng, *shape):
    return rng.standard_normal(shape).astype(np.float32)       # float64 draws rounded: full 24-bit mantissas


def ints(rng, *shape):
    return rng.integers(-4, 5, size=shape).astype(np.float32)


def operands(gen, rng, M, N, K, ta, tb):
    return gen(rng, *((K, M) if ta else (M, K))), gen(rng, *((N, K) if tb else (K, N)))


def gemm_case(rng, M, N, K, ta, tb, what):
    """One shape: random normals under the norm-wise bound, then integers bit for bit; both with the canaries and
    the dispatch check."""
    A, B = operands(normal, rng, M, N, K, ta, tb)
    C, names, expect = run_gemm(A, B, M, N, K, ta, tb)
    assert_bound(C, *logical(A, B, ta, tb), what=what)
    check_dispatch(names, [expect], what)
    A, B = operands(ints, rng, M, N, K, ta, tb)
    C, names, _ = run_gemm(A, B, M, N, K, ta, tb)
    a64, b64 = logical(A, B, ta, tb)
    assert_exact(C, a64 @ b64, what + " (integers)")
    check_dispatch(names, [expect], what + " (integers)")


def covering_shapes(layout, rot):
    """8 (M, N, K): every N once, every M and every K (odd K where K is a row count of an operand) at least once;
    `rot` shifts which M and K each N meets."""
    ta, tb = layout
    ks = KS + (KS_ODD if (ta or not tb) else [])
    return [(MS[(i + rot) % len(MS)], n, ks[(i + 2 * rot) % len(ks)]) for i, n in enumerate(NS)]


VARIANTS = {"tc2": 2, "tc": 1, "ffma": 0}


# ---- A. layout x tile x tail matrix ---------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: f"ta{l[0]}tb{l[1]}")
@pytest.mark.parametrize("core,bn", [(c, b) for c in ("tc2", "tc") for b in BNS] + [("ffma", 0)])
def test_layout_tile_tail_matrix(core, bn, layout, knobs):
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    rng = np.random.default_rng(1000 * VARIANTS[core] + 10 * bn + 2 * layout[0] + layout[1])
    for M, N, K in covering_shapes(layout, BNS.index(bn)):
        gemm_case(rng, M, N, K, *layout, f"{core} bn={bn} ta,tb={layout} M={M} N={N} K={K}")


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: f"ta{l[0]}tb{l[1]}")
@pytest.mark.parametrize("knob,value", [("tc_stages", 2), ("tc_l2_promo", 128)])
def test_ring_depth_and_l2_promotion_knobs(knob, value, layout, knobs):
    knobs(gemm_variant=2, **{knob: value})
    rng = np.random.default_rng(7)
    for M, N, K in covering_shapes(layout, 1)[::2]:
        gemm_case(rng, M, N, K, *layout, f"{knob}={value} ta,tb={layout} M={M} N={N} K={K}")


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: f"ta{l[0]}tb{l[1]}")
@pytest.mark.parametrize("core", ["tc2", "tc"])
def test_narrow_outputs_under_tc_min_n(core, layout, knobs):
    """tc_min_n = 4: N = 4 ... 28 on the tensor cores, inside a 32-wide tile (a stored [K, 4] B has a 16-B row pitch)."""
    knobs(gemm_variant=VARIANTS[core], tc_min_n=4)
    rng = np.random.default_rng(11)
    for i, N in enumerate([4, 8, 12, 20, 28]):
        M, K = [65, 128, 1000][i % 3], [36, 100, 32][i % 3]
        gemm_case(rng, M, N, K, *layout, f"{core} tc_min_n=4 ta,tb={layout} M={M} N={N} K={K}")


# ---- B. bit-exact probes --------------------------------------------------------------------------------------------
def _low_bits_cleared(rng, *shape):
    """full-mantissa values whose two lowest mantissa bits are 0: the lo part v - hi (13 low bits) fits TF32 exactly"""
    v = normal(rng, *shape)
    return (v.view(np.uint32) & np.uint32(0xFFFFFFFC)).view(np.float32)


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: f"ta{l[0]}tb{l[1]}")
@pytest.mark.parametrize("core,bn", [(c, b) for c in ("tc2", "tc") for b in BNS])
def test_selection_operands_exercise_the_lo_planes(core, bn, layout, knobs):
    """A one-hot selector times full-mantissa values: 3xTF32 gives hi + lo = the value exactly, so C must equal the
    selected rows (columns) bit for bit.  A selects rows of B (checks Ah@Bl); B selects columns of A (checks Al@Bh)."""
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    ta, tb = layout
    rng = np.random.default_rng(13)
    for M, N, K in [(128, 100, 100), (1000, 260, 36), (64, 36, 1000), (256, 68, 4100)]:
        what = f"{core} bn={bn} ta,tb={layout} M={M} N={N} K={K}"
        sel = np.zeros((M, K), np.float32)
        sel[np.arange(M), rng.integers(0, K, M)] = 1
        vals = _low_bits_cleared(rng, K, N)
        A, B = (sel.T if ta else sel), (vals.T if tb else vals)
        C, names, expect = run_gemm(np.ascontiguousarray(A), np.ascontiguousarray(B), M, N, K, ta, tb)
        assert_exact(C, sel.astype(np.float64) @ vals.astype(np.float64), what + " (A selects)")
        check_dispatch(names, [expect], what)
        vals = _low_bits_cleared(rng, M, K)
        sel = np.zeros((K, N), np.float32)
        sel[rng.integers(0, K, N), np.arange(N)] = 1
        A, B = (vals.T if ta else vals), (sel.T if tb else sel)
        C, names, _ = run_gemm(np.ascontiguousarray(A), np.ascontiguousarray(B), M, N, K, ta, tb)
        assert_exact(C, vals.astype(np.float64) @ sel.astype(np.float64), what + " (B selects)")


@pytest.mark.parametrize("stages", [0, 2])
def test_many_tiles_per_cta_bit_exact(stages, knobs):
    """314 work items of 128 k-blocks each on a persistent grid of one CTA per SM: every CTA runs two or three items,
    so the accumulators must restart per item and both mbarrier rings wrap their phase hundreds of times."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=2, gemm_bn=32, tc_stages=stages)
    M, N, K = 20000, 64, 4096
    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randint(-4, 5, (M, K), generator=g, device="cuda").float()
    B = torch.randint(-4, 5, (K, N), generator=g, device="cuda").float()
    C = torch.full((M, N), float("nan"), device="cuda")
    names = launched(lambda: _lib.check(lib.dr_debug_gemm(A.data_ptr(), B.data_ptr(), C.data_ptr(), M, N, K, 0, 0,
                                                          _stream()), "dr_debug_gemm"))
    ref = A.double() @ B.double()          # integers: exact on the GPU too
    assert torch.equal(C.double(), ref), f"{int((C.double() != ref).sum())} entries differ"
    check_dispatch(names, [("tc", 32, False, True, False)], "many tiles")


# ---- C. split-K -----------------------------------------------------------------------------------------------------
def _dense_bwd_gw(lib, x, w, gy, M, K, N):
    from deep_recommenders_b200 import _lib
    gw = torch.full((K, N), float("nan"), device="cuda")
    names = launched(lambda: _lib.check(lib.dr_dense_bwd(x.data_ptr(), w.data_ptr(), None, gy.data_ptr(), M, K, N, 0,
                                                         None, None, gw.data_ptr(), None, _stream()), "dr_dense_bwd"))
    return gw.cpu().numpy(), names


@pytest.mark.parametrize("core", ["tc2", "tc", "ffma"])
@pytest.mark.parametrize("splitk", [1, 2, 3, 7, 64, 10 ** 6])
@pytest.mark.parametrize("M", [1000, 4100])
def test_splitk_weight_gradient_bit_exact(M, splitk, core, knobs):
    """gW = X^T gY with only gw requested (the TN atomic epilogue); splits that leave a short last split, and 10**6
    (clamped to the number of k-blocks).  Integer data: the atomic summation order cannot change a bit."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=VARIANTS[core], gemm_splitk=splitk)
    rng = np.random.default_rng(M + splitk)
    for K, N in [(100, 36), (68, 132)]:
        x, gy = ints(rng, M, K), ints(rng, M, N)
        xt, gyt, wt = (torch.from_numpy(a).cuda() for a in (x, gy, np.zeros((K, N), np.float32)))
        gw, names = _dense_bwd_gw(lib, xt, wt, gyt, M, K, N)
        assert_exact(gw, x.astype(np.float64).T @ gy.astype(np.float64), f"{core} splitk={splitk} M={M} K={K} N={N}")
        check_dispatch(names, [expected_kernel(K, N, M, True, False, K, N)], f"splitk={splitk}")


def test_splitk_weight_gradient_random_normals(knobs):
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=2, gemm_splitk=7)
    rng = np.random.default_rng(3)
    M, K, N = 4100, 100, 132
    x, gy = normal(rng, M, K), normal(rng, M, N)
    xt, gyt, wt = (torch.from_numpy(a).cuda() for a in (x, gy, np.zeros((K, N), np.float32)))
    gw, names = _dense_bwd_gw(lib, xt, wt, gyt, M, K, N)
    assert_bound(gw, x.astype(np.float64).T, gy.astype(np.float64), "split-K 7, random normals")
    check_dispatch(names, [expected_kernel(K, N, M, True, False, K, N)], "split-K normals")


# ---- D. fused epilogues through the public entry points --------------------------------------------------------------
def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


ACTS = {None: 0, "relu": 1, "sigmoid": 2, "tanh": 3}
EPI_CORES = [(c, b) for c in ("tc2", "tc") for b in (0, 32, 64)]


@pytest.mark.parametrize("core,bn", EPI_CORES)
def test_dense_fwd_bias_activation_epilogue(core, bn, knobs):
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    rng = np.random.default_rng(17)
    for M, K, N in [(65, 68, 36), (129, 100, 260), (65, 36, 100), (129, 260, 68)]:
        x, w, b = normal(rng, M, K), normal(rng, K, N), normal(rng, N)
        xt, wt, bt = cu(x), cu(w), cu(b)
        scale = np.abs(x).astype(np.float64) @ np.abs(w).astype(np.float64) + np.abs(b)
        for act, code in ACTS.items():
            y = torch.full((M, N), float("nan"), device="cuda")
            names = launched(lambda: _lib.check(lib.dr_dense_fwd(xt.data_ptr(), wt.data_ptr(), bt.data_ptr(), M, K, N,
                                                                 code, y.data_ptr(), _stream()), "dr_dense_fwd"))
            ref = R.dense(x, w, b, act, np.float64)
            err = np.abs(y.cpu().numpy() - ref)
            assert (err <= 1e-5 * scale + 1e-7).all(), f"{core} bn={bn} {act} M={M} K={K} N={N}"
            check_dispatch(names, [expected_kernel(M, N, K, False, False, K, N)], f"dense_fwd {act}")


@pytest.mark.parametrize("core,bn", EPI_CORES)
def test_dense_bwd_chain_activation_gradient_epilogue(core, bn, knobs):
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    rng = np.random.default_rng(19)
    for M, K, N in [(65, 36, 68), (129, 260, 100), (129, 68, 36)]:
        w, gy = normal(rng, K, N), normal(rng, M, N)
        wt, gyt = cu(w), cu(gy)
        for prev_act, code in ACTS.items():
            x = R.act(normal(rng, M, K).astype(np.float64), prev_act).astype(np.float32)
            xt = cu(x)
            gx = torch.full((M, K), float("nan"), device="cuda")
            names = launched(lambda: _lib.check(lib.dr_dense_bwd_chain(
                xt.data_ptr(), wt.data_ptr(), None, gyt.data_ptr(), M, K, N, 0, None, gx.data_ptr(), None, None,
                xt.data_ptr(), code, _stream()), "dr_dense_bwd_chain"))
            x64 = x.astype(np.float64)
            dact = {None: np.ones_like(x64), "relu": (x64 > 0) * 1.0, "sigmoid": x64 * (1 - x64),
                    "tanh": 1 - x64 * x64}[prev_act]
            ref = (gy.astype(np.float64) @ w.astype(np.float64).T) * dact
            scale = (np.abs(gy).astype(np.float64) @ np.abs(w).astype(np.float64).T) * np.abs(dact)
            err = np.abs(gx.cpu().numpy() - ref)
            assert (err <= 1e-5 * scale + 1e-7).all(), f"{core} bn={bn} prev_act={prev_act} M={M} K={K} N={N}"
            check_dispatch(names, [expected_kernel(M, K, N, False, True, N, N)], f"dense_bwd_chain {prev_act}")


@pytest.mark.parametrize("core,bn", EPI_CORES)
def test_cross_full_rank_epilogues(core, bn, knobs):
    """dr_cross_fwd with u_out and alpha != 0 (EPI_CROSS with out2); dr_cross_bwd (EPI_CROSS_DX and the split-K gW)."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    rng = np.random.default_rng(23)
    alpha = 0.375
    for i, d in enumerate([36, 68, 100, 260]):
        B = [65, 129][i % 2]
        x0, x, w, b, g = normal(rng, B, d), normal(rng, B, d), normal(rng, d, d), normal(rng, d), normal(rng, B, d)
        x0t, xt, wt, bt, gt = cu(x0), cu(x), cu(w), cu(b), cu(g)
        nan = lambda *s: torch.full(s, float("nan"), device="cuda")
        y, u = nan(B, d), nan(B, d)
        names = launched(lambda: _lib.check(lib.dr_cross_fwd(
            x0t.data_ptr(), xt.data_ptr(), wt.data_ptr(), None, None, bt.data_ptr(), alpha, B, d, 0, None, u.data_ptr(),
            y.data_ptr(), _stream()), "dr_cross_fwd"))
        what = f"{core} bn={bn} B={B} d={d}"
        ref, uref = R.cross(x0, x, w, b, None, None, alpha, np.float64)
        ax, ax0 = np.abs(x).astype(np.float64), np.abs(x0).astype(np.float64)
        uscale = ax @ np.abs(w).astype(np.float64) + np.abs(b) + alpha * ax
        assert (np.abs(u.cpu().numpy() - uref) <= 1e-5 * uscale + 1e-7).all(), what + " u"
        assert (np.abs(y.cpu().numpy() - ref) <= 1e-5 * (ax0 * uscale + ax) + 1e-7).all(), what + " y"
        check_dispatch(names, [expected_kernel(B, d, d, False, False, d, d)], what + " fwd")

        h, gx0, gx, gw, gb = nan(B, d), nan(B, d), nan(B, d), nan(d, d), nan(d)
        names = launched(lambda: _lib.check(lib.dr_cross_bwd(
            x0t.data_ptr(), xt.data_ptr(), wt.data_ptr(), None, None, alpha, u.data_ptr(), None, gt.data_ptr(), B, d, 0,
            h.data_ptr(), None, gx0.data_ptr(), gx.data_ptr(), gw.data_ptr(), None, None, gb.data_ptr(), _stream()),
            "dr_cross_bwd"))
        h64 = g.astype(np.float64) * x0.astype(np.float64)          # the prologue's product is one fp32 rounding off
        ah = np.abs(h64)
        w64 = w.astype(np.float64)
        gx_ref = h64 @ w64.T + alpha * h64 + g
        gx_scale = ah @ np.abs(w64).T + alpha * ah + np.abs(g)
        assert (np.abs(gx.cpu().numpy() - gx_ref) <= 2e-5 * gx_scale + 1e-6).all(), what + " gx"
        gw_ref = x.astype(np.float64).T @ h64
        assert (np.abs(gw.cpu().numpy() - gw_ref) <= 2e-5 * (ax.T @ ah) + 1e-6).all(), what + " gW"
        check_dispatch(names, [expected_kernel(B, d, d, False, True, d, d), expected_kernel(d, d, B, True, False, d, d)],
                       what + " bwd")


@pytest.mark.parametrize("core,bn", EPI_CORES)
def test_scores_epilogue_with_correction_and_duplicates(core, bn, knobs):
    """dr_scores_fwd with p and duplicate candidate ids: S = Q C^T - log p, duplicates of row m's positive (candidate
    m) pushed to MIN_FLOAT.  Rows past the last candidate have no positive, so only the correction applies there."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=VARIANTS[core], gemm_bn=bn)
    rng = np.random.default_rng(29)
    for nq, nc, D in [(129, 100, 36), (65, 260, 68), (129, 36, 100)]:
        q, c = normal(rng, nq, D), normal(rng, nc, D)
        p = rng.uniform(0.05, 1, nc).astype(np.float32)
        ids = rng.integers(0, 10, nc).astype(np.int64)
        qt, ct, pt, it = cu(q), cu(c), cu(p), cu(ids)
        s = torch.full((nq, nc), float("nan"), device="cuda")
        names = launched(lambda: _lib.check(lib.dr_scores_fwd(qt.data_ptr(), ct.data_ptr(), pt.data_ptr(), it.data_ptr(),
                                                               nq, nc, D, s.data_ptr(), _stream()), "dr_scores_fwd"))
        s = s.cpu().numpy()
        q64, c64 = q.astype(np.float64), c.astype(np.float64)
        ref = R.sampling_probability_correction(q64 @ c64.T, p.astype(np.float64))
        r = min(nq, nc)
        ref[:r] = R.remove_accidental_negative(ref[:r], np.eye(r, nc), ids)
        masked = np.abs(ref) > 1e30
        what = f"{core} bn={bn} nq={nq} nc={nc} D={D}"
        assert masked.any() and np.array_equal(masked, np.abs(s) > 1e30), what + ": masked set"
        scale = np.abs(q64) @ np.abs(c64).T + np.abs(np.log(p.astype(np.float64)))
        assert (np.abs(s - ref)[~masked] <= (1e-5 * scale + 1e-7)[~masked]).all(), what
        check_dispatch(names, [expected_kernel(nq, nc, D, False, True, D, D)], what)


# ---- E. boundaries and non-finite isolation -------------------------------------------------------------------------
@pytest.mark.parametrize("core", ["tc2", "tc"])
def test_misaligned_operands(core, knobs):
    """An operand 4 B off 16-B alignment, or a row pitch that is not a multiple of 4 floats, cannot be a TMA source: the
    dispatcher must take the FFMA kernel (variant 1 only needs that of operands it splits flat).  C alone misaligned
    stays on the tensor cores and takes the scalar-store epilogue."""
    knobs(gemm_variant=VARIANTS[core])
    rng = np.random.default_rng(31)
    M, N, K = 132, 100, 68
    for ta, tb, offs in [(0, 0, dict(a_offset=4)), (0, 1, dict(b_offset=4)), (1, 0, dict(b_offset=4)),
                         (0, 0, dict(c_offset=4)), (1, 1, dict(c_offset=4)), (0, 1, dict(c_offset=4))]:
        what = f"{core} ta,tb={(ta, tb)} {offs}"
        A, B = operands(normal, rng, M, N, K, ta, tb)
        C, names, expect = run_gemm(A, B, M, N, K, ta, tb, **offs)
        assert_bound(C, *logical(A, B, ta, tb), what=what)
        split_flat = ("a_offset" in offs and not ta) or ("b_offset" in offs and tb)
        if "c_offset" in offs:
            assert expect[0] == "tc", what
        elif core == "tc2" or split_flat:
            assert expect == ("sgemm",), what
        check_dispatch(names, [expect], what)
    for M, N, K in [(128, 36, 33), (64, 100, 1001)]:                # lda = K not a multiple of 4
        A, B = operands(normal, rng, M, N, K, 0, 0)
        C, names, expect = run_gemm(A, B, M, N, K, 0, 0)
        assert expect == ("sgemm",)
        assert_bound(C, *logical(A, B, 0, 0), what=f"{core} lda={K}")
        check_dispatch(names, [expect], f"lda={K}")


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: f"ta{l[0]}tb{l[1]}")
@pytest.mark.parametrize("core", ["tc2", "tc", "ffma"])
def test_poisoned_row_and_column_stay_isolated(core, layout, knobs):
    knobs(gemm_variant=VARIANTS[core])
    ta, tb = layout
    rng = np.random.default_rng(37)
    M, N, K = 1000, 132, 100
    a, b = normal(rng, M, K), normal(rng, K, N)
    r, c = 517, 77
    a[r, 5] = np.nan
    b[40, c] = np.nan
    A, B = np.ascontiguousarray(a.T if ta else a), np.ascontiguousarray(b.T if tb else b)
    C, _, _ = run_gemm(A, B, M, N, K, ta, tb)
    want = np.zeros((M, N), bool)
    want[r, :] = True
    want[:, c] = True
    assert np.array_equal(~np.isfinite(C), want), f"non-finite set: {np.argwhere(~np.isfinite(C) != want)[:4].tolist()}"
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    keep_r, keep_c = np.arange(M) != r, np.arange(N) != c
    assert_bound(C[keep_r][:, keep_c], a64[keep_r], b64[:, keep_c], "finite part")
    A, B = operands(normal, rng, M, N, K, ta, tb)                  # the next call sees nothing of the poison
    C, _, _ = run_gemm(A, B, M, N, K, ta, tb)
    assert np.isfinite(C).all()
    assert_bound(C, *logical(A, B, ta, tb), "clean call after the poisoned one")


@pytest.mark.parametrize("core", ["tc2", "tc", "ffma"])
def test_infinite_inputs_give_the_oracles_non_finite_mask(core, knobs):
    """Only the mask is compared, not Inf against NaN: the tensor-core path splits Inf into hi = Inf and
    lo = Inf - Inf = NaN, so an Inf operand yields NaN where float64 yields +-Inf."""
    knobs(gemm_variant=VARIANTS[core])
    rng = np.random.default_rng(41)
    for ta, tb in LAYOUTS:
        M, N, K = 129, 68, 100
        a, b = normal(rng, M, K), normal(rng, K, N)
        a[3, 10], a[100, 99], b[0, 60], b[50, 7] = np.inf, -np.inf, -np.inf, np.inf
        A, B = np.ascontiguousarray(a.T if ta else a), np.ascontiguousarray(b.T if tb else b)
        C, _, _ = run_gemm(A, B, M, N, K, ta, tb)
        with np.errstate(invalid="ignore"):
            ref = a.astype(np.float64) @ b.astype(np.float64)
        assert np.array_equal(~np.isfinite(C), ~np.isfinite(ref)), f"{core} ta,tb={(ta, tb)}"
        fin = np.isfinite(ref)
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        a64[~np.isfinite(a64)], b64[~np.isfinite(b64)] = 0, 0
        assert (np.abs(C[fin] - ref[fin]) <= (1e-5 * (np.abs(a64) @ np.abs(b64)))[fin]).all()


# ---- F. variant 1 and its plane cache -------------------------------------------------------------------------------
def _dense_fwd_dx_dw(lib, x, w, gy, M, K, N):
    """forward, dX and dW on the same tensors: x is split flat (forward) and transposed (dW), W transposed (forward)
    and flat (dX), gY flat (dX) and transposed (dW)"""
    from deep_recommenders_b200 import _lib
    y = torch.full((M, N), float("nan"), device="cuda")
    gx = torch.full((M, K), float("nan"), device="cuda")
    gw = torch.full((K, N), float("nan"), device="cuda")
    _lib.check(lib.dr_dense_fwd(x.data_ptr(), w.data_ptr(), None, M, K, N, 0, y.data_ptr(), _stream()), "fwd")
    _lib.check(lib.dr_dense_bwd(x.data_ptr(), w.data_ptr(), None, gy.data_ptr(), M, K, N, 0, None, gx.data_ptr(),
                                gw.data_ptr(), None, _stream()), "bwd")
    return y.cpu().numpy(), gx.cpu().numpy(), gw.cpu().numpy()


def test_plane_cache_shares_planes_across_forward_dx_dw(knobs):
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=1)
    rng = np.random.default_rng(43)
    M, K, N = 1000, 132, 100
    x, w, gy = ints(rng, M, K), ints(rng, K, N), ints(rng, M, N)
    xt, wt, gyt = cu(x), cu(w), cu(gy)
    x64, w64, gy64 = x.astype(np.float64), w.astype(np.float64), gy.astype(np.float64)
    refs = (x64 @ w64, gy64 @ w64.T, x64.T @ gy64)
    off = _dense_fwd_dx_dw(lib, xt, wt, gyt, M, K, N)
    _lib.check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")
    names = launched(lambda: _dense_fwd_dx_dw(lib, xt, wt, gyt, M, K, N))
    on = _dense_fwd_dx_dw(lib, xt, wt, gyt, M, K, N)               # every plane from the cache now
    _lib.check(lib.dr_gemm_plane_cache(0), "dr_gemm_plane_cache")
    for name, a, b, ref in zip(("y", "gx", "gw"), off, on, refs):
        assert_exact(a, ref, name + " cache off")
        assert_exact(b, ref, name + " cache on")
    check_dispatch(names, [("tc", 128, False, False, True)], "plane cache")


@pytest.mark.parametrize("first,second", [((128, 64, 64), (64, 64, 128)), ((64, 64, 128), (128, 64, 64))])
def test_plane_cache_tells_apart_shapes_of_one_pointer(first, second, knobs):
    """With the cache on, one pointer read as [128, 64] and then as [64, 128] (same element count, other pitch) must
    not be served the other shape's planes."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=1)
    rng = np.random.default_rng(47)
    a = ints(rng, 128 * 64)
    at = cu(a)
    _lib.check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")
    for M, N, K in (first, second):
        b = ints(rng, K, N)
        bt = cu(b)
        c = torch.full((M, N), float("nan"), device="cuda")
        _lib.check(lib.dr_debug_gemm(at.data_ptr(), bt.data_ptr(), c.data_ptr(), M, N, K, 0, 0, _stream()), "gemm")
        assert_exact(c.cpu().numpy(), a.reshape(M, K).astype(np.float64) @ b.astype(np.float64), f"A as [{M}, {K}]")


def test_plane_cache_tells_apart_k_tails_of_one_pointer(knobs):
    """A stored [K, M] read with K = 33 and then K = 36: both round to a plane pitch of 36, but the first split wrote
    only 33 columns of it."""
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=1)
    rng = np.random.default_rng(53)
    M, N = 128, 64
    a = ints(rng, 36, M)
    at = cu(a)
    _lib.check(lib.dr_gemm_plane_cache(1), "dr_gemm_plane_cache")
    for K in (33, 36):
        b = ints(rng, K, N)
        bt = cu(b)
        c = torch.full((M, N), float("nan"), device="cuda")
        _lib.check(lib.dr_debug_gemm(at.data_ptr(), bt.data_ptr(), c.data_ptr(), M, N, K, 1, 0, _stream()), "gemm")
        assert_exact(c.cpu().numpy(), a[:K].astype(np.float64).T @ b.astype(np.float64), f"K={K}")


def test_variant1_falls_back_to_ffma_when_the_workspace_is_too_small(knobs):
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    knobs(gemm_variant=1)
    ws = _lib._workspace
    _lib.check(lib.dr_set_workspace(ws.data_ptr(), 64 << 10), "dr_set_workspace")
    try:
        rng = np.random.default_rng(59)
        M, N, K = 1000, 132, 100                                      # planes: 2 x (1000 + 132) x 100 floats > 64 KB
        for ta, tb in LAYOUTS:
            A, B = operands(normal, rng, M, N, K, ta, tb)
            C, names, _ = run_gemm(A, B, M, N, K, ta, tb)
            assert_bound(C, *logical(A, B, ta, tb), f"ta,tb={(ta, tb)}")
            check_dispatch(names, [("sgemm",)], "64 KB workspace")
    finally:
        _lib.check(lib.dr_set_workspace(ws.data_ptr(), ws.numel()), "dr_set_workspace")


def _small_deepfm_trainer(B=1000, use_graph=True, rows=(500, 7, 300, 41), dnn=(64, 32), **kw):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, D = list(rows), 16
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=list(dnn), seed=7, device="cuda", sparse_lr=0.05)
    with torch.no_grad():
        model.embeddings.lin_view().normal_(0, 0.1, generator=torch.Generator(device="cuda").manual_seed(3))
    tr = DeepFMTrainStep(model, batch_size=B, lr=0.05, use_graph=use_graph, **kw)
    return rows, model, (tr.capture() if use_graph else tr)


@pytest.mark.parametrize("use_graph", [False, True])
def test_train_step_agrees_across_gemm_cores(use_graph, knobs):
    """Three DeepFM train steps under FFMA (0), pre-split planes with the per-step plane cache (1) and the in-kernel
    split (2) from the same parameters and batches."""
    runs = {}
    for variant in (0, 1, 2):
        knobs(gemm_variant=variant)
        rows, model, tr = _small_deepfm_trainer(use_graph=use_graph)
        rng = np.random.default_rng(5)
        losses, names = [], []
        for k in range(3):
            ids = torch.from_numpy(np.stack([rng.integers(-1, r, size=tr.B) for r in rows], axis=1)).cuda()
            lab = torch.from_numpy(rng.integers(0, 2, size=tr.B).astype(np.float32)).cuda()
            names += launched(lambda: losses.append(float(tr.step(ids, lab).item())), attempts=1)
        torch.cuda.synchronize()
        runs[variant] = (losses, model, tr)
        if cupti_works():
            tc = {k for k in _gemm_kernels(names) if k[0] == "tc"}
            assert (not tc) if variant == 0 else (tc and all(k[4] == (variant == 1) for k in tc)), (variant, tc)
    l0, m0, t0 = runs[0]
    for variant in (1, 2):
        l, m, t = runs[variant]
        for a, b in zip(l0, l):
            assert abs(a - b) <= 5e-6 * abs(a), (variant, l0, l)
        assert float((t0.gw[0] - t.gw[0]).abs().max()) <= 1e-5 * float(t0.gw[0].abs().max())
        assert torch.allclose(m0.embeddings.weight, m.embeddings.weight, rtol=1e-5, atol=1e-7), variant
        for a, b in zip(t0.w + t0.b, t.w + t.b):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), variant


# ---- every instantiation --------------------------------------------------------------------------------------------
def test_every_gemm_tc_kernel_instantiation_runs(knobs):
    """BN in {32, 64, 128} x the four (A_MN, B_MN) of the in-kernel split, and BN in {32, 64, 128} pre-split: each one
    launched once more here on integers (bit for bit), and the set seen over the whole module printed."""
    if not cupti_works():
        pytest.skip("torch.profiler returned no CUDA kernel records: the launched instantiations cannot be observed")
    rng = np.random.default_rng(61)
    want = {("tc", bn, amn, bmn, False) for bn in (32, 64, 128) for amn in (False, True) for bmn in (False, True)}
    want |= {("tc", bn, False, False, True) for bn in (32, 64, 128)}
    got = set()
    for variant in (2, 1):
        knobs(gemm_variant=variant)
        for N in (32, 64, 128):
            for ta, tb in LAYOUTS:
                M, K = 128, 68
                A, B = operands(ints, rng, M, N, K, ta, tb)
                for _ in range(3):                # (each run_gemm already profiles up to three times)
                    C, names, expect = run_gemm(A, B, M, N, K, ta, tb)
                    assert_exact(C, np.matmul(*logical(A, B, ta, tb)), f"variant {variant} N={N} ta,tb={(ta, tb)}")
                    check_dispatch(names, [expect])
                    if _gemm_kernels(names):
                        break
                got |= _gemm_kernels(names)
    print("gemm_tc_kernel instantiations launched in this module:", sorted(_SEEN))
    assert want <= got, f"not launched: {sorted(want - got)}"
