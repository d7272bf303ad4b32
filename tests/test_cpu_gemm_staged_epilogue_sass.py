"""Static check of the built .so (no GPU): the staged epilogue of the wgmma GEMM.

Every splitter (gemm_tc_kernel) and weight-plane (gemm_tc_wplanes_kernel) instantiation hands its output tile to TMA:
a tensor store (UTMASTG) for the plain modes and a tensor reduce-add (UTMAREDG ... ADD) for split-K.  The staging tile
costs no local memory, and the static shared memory stays within the 2 KB that the shared-memory budget in gemm_tc.cu
allows for."""
import os
import re
import shutil
import subprocess

import pytest

_NAME_RE = re.compile(r"_ZN2dr(?:14gemm_tc_kernelILi\d+ELb[01]ELb[01]ELb[01]E|22gemm_tc_wplanes_kernelILi\d+E)E\S*")


def _cuobjdump(*args):
    from deep_recommenders_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not installed")
    _lib.load()
    return subprocess.run([tool, *args, str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout


def test_gemm_kernels_store_and_reduce_tiles_with_tma():
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", _cuobjdump("-sass"))[1:]:
        name = chunk.split(None, 1)[0]
        if _NAME_RE.fullmatch(name):
            funcs[name] = chunk
    assert len(funcs) == 18, sorted(funcs)   # 15 splitter / pre-split + 3 weight-plane instantiations
    for name, body in funcs.items():
        assert re.search(r"\bUTMASTG\.2D\b", body), f"{name}: no TMA tile store"
        assert re.search(r"\bUTMAREDG\.2D\.ADD\b", body), f"{name}: no TMA tile reduce-add"


def test_gemm_kernels_use_no_local_memory():
    res = _cuobjdump("-res-usage").splitlines()
    found = {}
    for i, line in enumerate(res):
        m = re.match(r"\s*Function (\S+):", line)
        if m and _NAME_RE.fullmatch(m.group(1)) and i + 1 < len(res):
            r = re.search(r"STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", res[i + 1])
            found[m.group(1)] = tuple(map(int, r.groups()))
    assert len(found) == 18, sorted(found)
    for name, (stack, shared, local) in found.items():
        assert stack == 0 and local == 0 and shared <= 2048, (name, stack, shared, local)
