"""ctypes binding of libdeeprec_b200.so (include/deeprec_b200.h).

There is NO fallback: if the library is missing, or a call returns non-zero, this module
raises.  `load()` only dlopens and declares signatures, so it also works on a box without a
GPU (used by the `-m "not gpu"` symbol test); every compute entry needs `cuda:0`.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "lib" / "libdeeprec_b200.so"
HEADER_PATH = _PKG.parent / "include" / "deeprec_b200.h"

_lib = None
_GEMM_ENV = os.environ.get("DR_GEMM", "tc2")

_p = C.c_void_p
_i64 = C.c_int64
_i = C.c_int
_f = C.c_float

# name -> argtypes (restype is int unless listed in _RESTYPES)
_SIGS = {
    "dr_version": [],
    "dr_last_error": [],
    "dr_launch_count": [],
    "dr_tune_set": [C.c_char_p, _i],
    "dr_tune_get": [C.c_char_p, _p],
    "dr_set_workspace": [_p, C.c_uint64],
    "dr_gemm_plane_cache": [_i],
    "dr_debug_gemm": [_p, _p, _p, _i64, _i64, _i64, _i, _i, _p],
    "dr_debug_gemm_epi": [_p, _p, _p, _i64, _i64, _i64, _i, _i, _i64, _i, _i, _p, _p, _i, _p],
    "dr_embed_fm_fwd": [_p, _p, _p, _p, _i, _p, _i64, _i, _i, _i64, _i64, _i, _p, _p, _p, _p],
    "dr_embed_fm_fwd_tma": [_p, _i64, _p, _p, _p, _i, _p, _i64, _i, _i, _i64, _p, _p, _p, _p],
    "dr_embed_fm_bwd": [_p, _i, _p, _p, _p, _p, _p, _i64, _i, _i, _i64, _i64, _i, _p, _p, _p, _f, _p],
    "dr_embed_fm_fwd_sharded": [_p, _i, _p, _p, _p, _i, _p, _i64, _i, _i, _i64, _i, _i64, _p, _p, _p, _p],
    "dr_embed_fm_bwd_sharded": [_p, _i, _p, _p, _p, _i, _p, _p, _p, _p, _i64, _i, _i, _i64, _i, _i64, _p, _f, _p],
    "dr_gather_fwd": [_p, _i64, _p, _i, _i64, _i, _p, _p],
    "dr_scatter_add": [_p, _i64, _p, _i, _i64, _i, _p, _f, _p],
    "dr_fm_fwd": [_p, _i64, _i, _i, _p, _p],
    "dr_fm_bwd": [_p, _p, _i64, _i, _i, _p, _p],
    "dr_dense_fwd": [_p, _p, _p, _i64, _i, _i, _i, _p, _p],
    "dr_dense_bwd": [_p, _p, _p, _p, _i64, _i, _i, _i, _p, _p, _p, _p, _p],
    "dr_dense_bwd_chain": [_p, _p, _p, _p, _i64, _i, _i, _i, _p, _p, _p, _p, _p, _i, _p],
    "dr_dense_grouped_fwd": [_p, _p, _p, _i64, _i, _i, _i, _i, _p, _p],
    "dr_dense_grouped_bwd": [_p, _p, _p, _p, _i64, _i, _i, _i, _i, _p, _p, _p, _p, _p],
    "dr_cross_fwd": [_p, _p, _p, _p, _p, _p, _f, _i64, _i, _i, _p, _p, _p, _p],
    "dr_cross_bwd": [_p, _p, _p, _p, _p, _f, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "dr_cross_bwd_acc": [_p, _p, _p, _p, _p, _f, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _i, _p],
    "dr_cin_fwd": [_p, _p, _p, _p, _i64, _i, _i, _i, _i, _i, _p, _p, _p],
    "dr_cin_bwd": [_p, _p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p],
    "dr_din_attn_fwd": [_p, _p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _i, _p, _p, _p],
    "dr_din_attn_bwd": [_p, _p, _p, _p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p],
    "dr_dice_fwd": [_p, _p, _i64, _i, _f, _p, _p],
    "dr_dice_bwd": [_p, _p, _p, _i64, _i, _f, _p, _p, _p],
    "dr_mha_attn_fwd": [_p, _p, _p, _p, _i64, _i, _i, _i, _i, _i64, _i, _f, C.c_uint64, _p, _p, _p],
    "dr_mha_attn_bwd": [_p, _p, _p, _p, _p, _p, _p, _i64, _i, _i, _i, _i, _i64, _i, _f, C.c_uint64, _p, _p, _p,
                        _p],
    "dr_add_layernorm_fwd": [_p, _p, _p, _p, _i64, _i, _f, _p, _p],
    "dr_add_layernorm_bwd": [_p, _p, _p, _p, _i64, _i, _f, _p, _p, _p, _p],
    "dr_softmax_rows_fwd": [_p, _i64, _i, _p, _p],
    "dr_softmax_rows_bwd": [_p, _p, _i64, _i, _p, _p],
    "dr_spmm_csr_fwd": [_p, _p, _p, _i64, _i64, _i64, _p, _i, _p, _p, _i, _p, _p, _p],
    "dr_act_bwd_colsum": [_p, _p, _i64, _i, _i, _p, _p, _p],
    "dr_moe_mix_fwd": [_p, _p, _i64, _i, _i, _i, _p, _p, _p],
    "dr_moe_mix_bwd": [_p, _p, _p, _i64, _i, _i, _i, _p, _p, _p],
    "dr_inbatch_softmax_fwd": [_p, _p, _p, _p, _p, _f, _i64, _i64, _i, _p, _p, _p],
    "dr_inbatch_softmax_bwd": [_p, _p, _p, _p, _p, _f, _i64, _i64, _i, _p, _p, _p, _p, _p],
    "dr_inbatch_softmax_fwd_ws": [_p, _p, _p, _p, _p, _f, _i64, _i64, _i, _p, _i64, _p, _p, _p],
    "dr_inbatch_softmax_bwd_ws": [_p, _p, _p, _p, _p, _f, _i64, _i64, _i, _p, _p, _p, _i64, _i, _p, _p, _p],
    "dr_scores_fwd": [_p, _p, _p, _p, _i64, _i64, _i, _p, _p],
    "dr_hard_negative_topk": [_p, _i64, _i64, _i, _p, _p, _p, _p],
    "dr_shard_bucket_ids": [_p, _i, _i64, _i, _p, _p, _i, _i64, _p, _p, _p, _p, _p],
    "dr_permute_rows": [_p, _p, _i64, _i, _p, _p],
    "dr_unpermute_rows": [_p, _p, _i64, _i, _p, _p],
    "dr_sgd_step": [_p, _p, _i64, _f, _p],
    "dr_bce_logits_fwd_bwd": [_p, _p, _p, _i64, _p, _p, _p, _p],
    "dr_dense_head_bce_fwd_bwd": [_p, _p, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "dr_dcn_head_bce_fwd_bwd": [_p, _p, _p, _p, _p, _i64, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    # SURVEY 8(f) "next" rows
    "dr_adam_step": [_p, _p, _p, _p, _i64, _f, _f, _f, _f, _i, _p, _p],
    "dr_adam_advance": [_p, _f, _f, _f, _p, _p],
    "dr_adam_step_multi": [_i, _p, _p, _p, _p, _p, _f, _f, _f, _f, _p, _p],
    "dr_lazy_adam_rows": [_p, _i, _i64, _i, _i, _p, _p, _p, _p, _p, _p, _i64, _i, _p, _p, _p, _p, _p, _p, _p,
                          _f, _f, _f, _p],
    "dr_embed_adam_state_stride": [_i],
    "dr_embed_adam_count": [_p, _i, _i64, _i, _i, _p, _p, _p, _p],
    "dr_embed_fm_bwd_adam": [_p, _i, _p, _p, _p, _p, _p, _p, _i64, _i, _i, _i64, _i64, _i, _p, _p, _p, _p, _p,
                             _f, _f, _f, _p],
    "dr_adam_advance_hist": [_p, _f, _f, _f, _p, _p, _i, _p],
    "dr_embed_fm_bwd_adam_tf": [_p, _i, _p, _p, _p, _p, _p, _p, _i64, _i, _i, _i64, _i64, _i, _p, _p, _p, _p, _p, _p, _p,
                                _i, _f, _f, _f, _f, _p],
    "dr_embed_adam_prepare": [_p, _i, _i64, _i, _i, _p, _p, _i64, _i64, _i, _p, _p, _p, _p, _p, _i, _f, _f, _f, _f, _p],
    "dr_embed_adam_flush": [_p, _p, _i, _i, _i64, _i64, _i64, _i, _p, _p, _p, _p, _p, _i, _f, _f, _f, _f, _p],
    "dr_embed_adam_catch_up": [_p, _i, _i64, _i, _i, _p, _p, _i64, _i64, _i, _p, _p, _p, _p, _p, _i, _f, _f, _f, _f, _p],
    "dr_embed_adam_rows_tf": [_p, _i, _i64, _i64, _i, _p, _p, _p, _p, _i64, _i64, _p, _i64, _i64, _i, _i64, _i64, _i,
                              _p, _p, _p, _p, _p, _p, _i, _f, _f, _f, _f, _p],
    "dr_shard_adam_mark": [_p, _i, _i64, _i, _p, _p, _i, _p, _p, _p],
    "dr_shard_adam_prepare": [_p, _i64, _p, _p, _i, _i64, _i64, _i, _p, _p, _p, _p, _i, _f, _f, _f, _f, _p],
    "dr_shard_adam_apply": [_p, _p, _i64, _i, _i64, _i64, _i, _p, _p, _p, _p, _p, _f, _f, _f, _p],
    "dr_hash_bucket_i64": [_p, _i64, _i64, _p, _p],
    "dr_hash_bucket_bytes": [_p, _p, _i64, _i64, _p, _p],
    "dr_hash_bucket_i64_host": [_p, _i64, _i64, _p],
    "dr_hash_bucket_bytes_host": [_p, _p, _i64, _i64, _p],
    "dr_fingerprint64_host": [_p, _i64],
    "dr_vocab_lookup_i64": [_p, _i64, _p, _p, _i64, _i64, _p, _p],
    "dr_cross_hash": [_i, _p, _p, _p, _i64, C.c_uint64, _i64, _p, _p, _p],
    "dr_cross_hash_host": [_i, _p, _p, _p, _i64, C.c_uint64, _i64, _p, _p],
    "dr_wide_fwd": [_p, _i64, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _p, _p],
    "dr_wide_bwd": [_p, _i64, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _p, _p],
    "dr_wide_ftrl": [_p, _i64, _p, _p, _p, _i64, _i, _i, _p, _p, _p, _f, _f, _f, _p],
    "dr_embed_bag_fwd": [_p, _i64, _i64, _p, _i, _p, _i64, _i, _i, _p, _i64, _p],
    "dr_embed_bag_bwd": [_p, _i, _p, _i64, _i, _i, _p, _i64, _i64, _i64, _p, _f, _p],
    "dr_fnn_input_fwd": [_p, _p, _p, _p, _i, _i64, _i64, _i, _p, _i64, _i, _i, _i64, _p, _p],
    "dr_fnn_input_bwd": [_p, _i, _p, _p, _i64, _i, _i, _i64, _i64, _i64, _i, _p, _p, _f, _p],
    "dr_crc32c_host": [_p, _i64],
    "dr_masked_crc32c_host": [_p, _i64],
    "dr_tfrecord_index": [_p, _i64, _i, _p, _p, _i64],
    "dr_example_parse_feature": [_p, _p, _p, _i64, C.c_char_p, _i, _p, _p, _p, _p, _p, _p],
    "dr_example_parse_batch": [_p, _p, _p, _i64, _i, _p, _p, _p, _p, _p, _p, _p, _p],
    "dr_set_host_threads": [_i],
    "dr_vocab_lookup_bytes_host": [_p, _p, _i64, _p, _p, _i64, _i64, _p],
    "dr_topk_rows": [_p, _i64, _i64, _i64, _i, _p, _p, _p],
    "dr_take_long_axis": [_p, _i, _i64, _i64, _i64, _p, _i, _p, _p],
    "dr_exclude_adjust": [_p, _p, _p, _i64, _i64, _i64, _f, _p, _p],
    "dr_rowwise_dot": [_p, _p, _i64, _i, _p, _p],
    "dr_column_rank": [_p, _p, _i64, _i64, _i64, _p, _p],
}
_RESTYPES = {"dr_last_error": C.c_char_p, "dr_launch_count": C.c_uint64, "dr_fingerprint64_host": C.c_uint64,
             "dr_crc32c_host": C.c_uint32, "dr_masked_crc32c_host": C.c_uint32, "dr_tfrecord_index": C.c_int64}


class DeepRecError(RuntimeError):
    """A C-ABI call returned non-zero (mirrors the Python exceptions the reference raises)."""


def header_symbols() -> list[str]:
    """Every function name include/deeprec_b200.h declares."""
    text = HEADER_PATH.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dr_[a-z0-9_]+)\s*\(", text)))


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise DeepRecError(
            f"{LIB_PATH} is missing: build it with `python -m deep_recommenders_b200.build` "
            "(there is no CPU fallback for the hot path)"
        )
    lib = C.CDLL(str(LIB_PATH), mode=os.RTLD_LOCAL | os.RTLD_NOW)
    for name, argtypes in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, C.c_int)
    _lib = lib
    # DR_GEMM names the GEMM core for THIS process (the library's own default is tc2); variant 1 (pre-split planes) is
    # switched on lazily by ensure_gemm_workspace because it needs the registered scratch
    if _GEMM_ENV == "ffma":
        lib.dr_tune_set(b"gemm_variant", 0)
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().dr_last_error().decode(errors="replace")
        if rc < 0:
            raise ValueError(f"{what}: {msg} (rc={rc})")
        raise DeepRecError(f"{what}: CUDA error {rc}: {msg}")


def launch_count() -> int:
    return int(load().dr_launch_count())


def tune(key: str, value: int) -> None:
    check(load().dr_tune_set(key.encode(), int(value)), "dr_tune_set")


def tune_get(key: str) -> int:
    v = C.c_int(0)
    check(load().dr_tune_get(key.encode(), C.byref(v)), "dr_tune_get")
    return int(v.value)


_workspace = None
_retired = []


def set_workspace(nbytes: int, device=None):
    """Allocate (through torch) and register the tensor-core GEMM scratch; 0 unregisters."""
    global _workspace
    import torch
    if nbytes <= 0:
        check(load().dr_set_workspace(None, 0), "dr_set_workspace")
        _workspace = None
        return None
    if _workspace is None or _workspace.numel() < nbytes:
        if _workspace is not None:
            _retired.append(_workspace)      # a captured CUDA graph may still point at it
        _workspace = torch.empty(int(nbytes), dtype=torch.uint8, device=device or "cuda")
    check(load().dr_set_workspace(_workspace.data_ptr(), _workspace.numel()), "dr_set_workspace")
    return _workspace


def enable_tensor_core_gemm(workspace_bytes: int = 0, device=None, variant: int = None) -> None:
    """Route eligible GEMMs (Dense / Cross / scores) to the wgmma 3xTF32 kernel: variant 1 = pre-split hi/lo planes
    (needs the registered workspace), variant 2 = split in shared memory inside the GEMM (no workspace).
    Default: the variant selected by DR_GEMM (tc -> 1, tc2 -> 2)."""
    global _tc_enabled, _tc_applied
    if workspace_bytes:
        set_workspace(workspace_bytes, device)
    tune("gemm_variant", int(variant) if variant is not None else _tc_variant)
    _tc_enabled = True
    _tc_applied = True          # an explicit choice is not overridden by the lazy default


def disable_tensor_core_gemm() -> None:
    global _tc_enabled
    tune("gemm_variant", 0)
    _tc_enabled = False


# DR_GEMM selects the default GEMM core: tc2 (default) = wgmma 3xTF32 with the hi/lo split inside the kernel,
# tc = wgmma 3xTF32 on pre-split planes, ffma = FFMA.
_tc_enabled = _GEMM_ENV != "ffma"
_tc_variant = 1 if _GEMM_ENV == "tc" else 2
_tc_applied = False


def ensure_gemm_workspace(M: int, K: int, N: int, device=None) -> None:
    """Make sure the hi/lo operand planes of a [M,K]x[K,N] GEMM and of its two backward GEMMs fit
    in the registered scratch (grows it if needed); applies the default GEMM variant on first use."""
    global _tc_applied
    if not _tc_enabled:
        return
    if not _tc_applied:
        tune("gemm_variant", _tc_variant)
        _tc_applied = True
    k4, n4, m4 = (K + 3) // 4 * 4, (N + 3) // 4 * 4, (M + 3) // 4 * 4
    need = 8 * max(M * k4 + N * k4, M * n4 + K * n4, K * m4 + N * m4) + (1 << 16)
    if _workspace is None or _workspace.numel() < need:
        set_workspace(int(need * 1.25), device)
