"""Static check of the built .so (no GPU): the in-kernel-split wgmma GEMM feeds its A operand from registers.

In the default variant (PRESPLIT = 0) each consumer thread reads its own A-fragment elements from the raw TMA stage,
splits them into TF32 hi / lo in registers and passes them to wgmma as a register fragment, so no A planes are written to
or read from shared memory.  In SASS that is `HGMMA... Rd, Ra, gdesc[..]`; an A operand read from shared memory is
`HGMMA... Rd, gdesc[..]`.  The pre-split variant (PRESPLIT = 1) loads both planes of both operands by TMA and keeps
reading A from shared memory."""
import os
import re
import shutil
import subprocess

import pytest

_NAME_RE = re.compile(r"_ZN2dr(?:14gemm_tc_kernelILi(\d+)ELb[01]ELb[01]ELb([01])E|18gemm_tc_acc_kernelILi(\d+)ELb([01])E)\S*")
_HGMMA_RE = re.compile(r"HGMMA\.64x(\d+)x8\.F32\.TF32 R\d+, (\S+)")


def _gemm_tc_sass():
    from deep_recommenders_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    _lib.load()
    sass = subprocess.run([cuobjdump, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name = chunk.split(None, 1)[0]
        if _NAME_RE.fullmatch(name):
            funcs[name] = chunk
    return funcs


def test_in_kernel_split_gemm_takes_a_from_registers():
    funcs = _gemm_tc_sass()
    assert sum("14gemm_tc_kernel" in n for n in funcs) == 15, sorted(funcs)
    assert sum("18gemm_tc_acc_kernel" in n for n in funcs) == 4, sorted(funcs)
    for name, body in funcs.items():
        g = _NAME_RE.fullmatch(name).groups()
        bn, presplit = (g[0], g[1]) if g[0] else (g[2], g[3])
        ops = _HGMMA_RE.findall(body)
        assert ops, f"no TF32 HGMMA in {name}"
        assert {n for n, _ in ops} == {bn}, (name, ops)
        a_srcs = {a.rstrip(",") for _, a in ops}
        if presplit == "0":
            assert all(re.fullmatch(r"R\d+", a) for a in a_srcs), f"{name}: A operand not from registers: {a_srcs}"
        else:
            assert all(a.startswith("gdesc[") for a in a_srcs), f"{name}: A operand not from shared memory: {a_srcs}"
