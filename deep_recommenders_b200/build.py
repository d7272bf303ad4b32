"""Builds libdeeprec_b200.so (the C-ABI library of include/deeprec_b200.h) in-tree with nvcc.

sm_90a only: `-gencode arch=compute_90a,code=sm_90a`.  nvcc cross-compiles without a GPU,
so the library can be built on a machine that has none.
Object files are cached per source under deep_recommenders_b200/lib/obj and rebuilt when the
source, a header, or the flags change.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
ROOT = PKG.parent
CSRC = PKG / "csrc"
LIBDIR = PKG / "lib"
LIB = LIBDIR / "libdeeprec_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", str(ROOT / "include"),
    "-I", str(CSRC),
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found: cannot build libdeeprec_b200.so")
    return cand


def _digest(src: Path, headers: list[Path]) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for f in [src, *headers]:
        h.update(f.read_bytes())
    return h.hexdigest()[:16]


def build(verbose: bool = False, force: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link the shared library. Returns its path."""
    nvcc = _nvcc()
    objdir = LIBDIR / "obj"
    objdir.mkdir(parents=True, exist_ok=True)
    headers = sorted(CSRC.glob("*.cuh")) + sorted((ROOT / "include").glob("*.h"))
    sources = sorted(CSRC.glob("*.cu"))
    jobs = []
    objs = []
    for src in sources:
        tag = _digest(src, headers)
        obj = objdir / f"{src.stem}.{tag}.o"
        objs.append(obj)
        if force or not obj.exists():
            for old in objdir.glob(f"{src.stem}.*.o"):
                old.unlink()
            jobs.append((src, obj))

    def _compile(job):
        src, obj = job
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src.name}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(_compile, jobs))
    if jobs or not LIB.exists():
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
