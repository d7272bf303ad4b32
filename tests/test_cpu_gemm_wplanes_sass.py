"""Static check of the built .so (no GPU): the weight-plane wgmma GEMM (gemm_tc_wplanes_kernel<BN>).

It splits A in registers, so every HGMMA takes A from a register (`HGMMA... Rd, Ra, gdesc[..]`).  A tile whose valid
width is at most 32 (64) columns runs 64x32x8 (64x64x8) MMAs, so the BN = 128 kernel holds all three widths and the
BN = 64 one two.  With 288 threads it may use up to 168 registers and uses no local memory."""
import os
import re
import shutil
import subprocess

import pytest

_NAME_RE = re.compile(r"_ZN2dr22gemm_tc_wplanes_kernelILi(\d+)EE\S*")
_HGMMA_RE = re.compile(r"HGMMA\.64x(\d+)x8\.F32\.TF32 R\d+, (\S+)")


def _cuobjdump(*args):
    from deep_recommenders_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not installed")
    _lib.load()
    return subprocess.run([tool, *args, str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout


def test_weight_plane_kernels_take_a_from_registers_at_tail_widths():
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", _cuobjdump("-sass"))[1:]:
        name = chunk.split(None, 1)[0]
        m = _NAME_RE.fullmatch(name)
        if m:
            funcs[int(m.group(1))] = chunk
    assert sorted(funcs) == [32, 64, 128], sorted(funcs)
    for bn, body in funcs.items():
        ops = _HGMMA_RE.findall(body)
        assert {int(n) for n, _ in ops} == {w for w in (32, 64, 128) if w <= bn}, (bn, sorted({n for n, _ in ops}))
        a_srcs = {a.rstrip(",") for _, a in ops}
        assert all(re.fullmatch(r"R\d+", a) for a in a_srcs), f"BN={bn}: A operand not from registers: {a_srcs}"


def test_weight_plane_kernels_use_no_local_memory():
    res = _cuobjdump("-res-usage").splitlines()
    found = {}
    for i, line in enumerate(res):
        m = re.match(r"\s*Function (\S+):", line)
        if m and _NAME_RE.fullmatch(m.group(1)) and i + 1 < len(res):
            r = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res[i + 1])
            found[m.group(1)] = tuple(map(int, r.groups()))
    assert len(found) == 3, found
    for name, (reg, stack, _, local) in found.items():
        # 9 warps are allocated as 12: 65536 / 384 = 170, rounded down to the allocation granule of 8
        assert reg <= 168 and stack == 0 and local == 0, (name, reg, stack, local)
