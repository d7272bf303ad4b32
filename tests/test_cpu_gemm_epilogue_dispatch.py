"""Static check of the built .so (no GPU): the wgmma GEMM kernels choose their epilogue mode once per tile.

The epilogue mode (`GemmArgs::epi`) and the activation (`GemmArgs::act`) are run-time values.  Switching on them once per
accumulator element compiles to indirect branches (BRX) in proportion to the tile width and puts a data-dependent branch
behind every bias / auxiliary load; switched on once per tile, each mode is straight-line code and the number of BRX
does not depend on the tile width."""
import os
import re
import shutil
import subprocess
from collections import defaultdict

import pytest

_NAME_RE = re.compile(r"_ZN2dr14gemm_tc_kernelILi(\d+)ELb([01])ELb([01])ELb([01])E\S*")
MAX_BRX = 8


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


def test_gemm_tc_epilogue_dispatch_is_per_tile():
    funcs = _gemm_tc_sass()
    assert len(funcs) == 15, sorted(funcs)   # 3 tile widths x (4 operand layouts split in kernel + pre-split planes)
    by_layout = defaultdict(dict)
    for name, body in funcs.items():
        bn, a_mn, b_mn, presplit = _NAME_RE.fullmatch(name).groups()
        brx = len(re.findall(r"\bBRX\b", body))
        by_layout[(a_mn, b_mn, presplit)][int(bn)] = brx
    for layout, counts in by_layout.items():
        assert sorted(counts) == [32, 64, 128], (layout, counts)
        assert len(set(counts.values())) == 1, f"BRX count grows with the tile width at layout {layout}: {counts}"
        assert max(counts.values()) <= MAX_BRX, f"more than {MAX_BRX} BRX at layout {layout}: {counts}"
