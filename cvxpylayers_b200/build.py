"""Builds libbcone.so (the C-ABI CUDA library) in-tree for the H100 (sm_90a) with nvcc.

Run as ``python -m cvxpylayers_b200.build``; ``__graft_entry__.build()`` calls :func:`build`.
nvcc cross-compiles without a GPU.  The translation units share no device symbols, so each is
compiled on its own (in parallel, into a temporary directory) and the objects are linked into one
shared library.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
SOURCES = ["api.cu", "fwd.cu", "fwd_fast.cu", "bwd.cu", "bwd_fast.cu", "bwd_block.cu", "bwd_lsmr.cu", "bwd_fast_lsmr.cu", "bwd_block_lsmr.cu",
           "pack.cu", "shared.cu", "polish.cu", "polish_large.cu", "refine.cu"]
HEADERS = [CSRC / "common.cuh", PKG.parent / "include" / "bcone.h"]
LIB = PKG / "libbcone.so"
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH_FLAGS, "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found; libbcone.so cannot be built")
    return cand


def stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    return any(p.stat().st_mtime > t for p in [*(CSRC / s for s in SOURCES), *HEADERS])


def build(force: bool = False, verbose: bool = False, defines: tuple = (), out: "Path | None" = None) -> Path:
    """``defines`` / ``out``: development variants (e.g. ``-DBC_SUBPROF`` into another file, loaded with BCONE_LIB=...)."""
    target = Path(out) if out else LIB
    if not force and not defines and not out and not stale():
        return LIB
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory(prefix="bcone_build_") as td:
        objs = [os.path.join(td, Path(s).stem + ".o") for s in SOURCES]

        def compile_one(src_obj):
            src, obj = src_obj
            cmd = [nvcc, *NVCC_FLAGS, *(["-Xptxas=-v"] if verbose else []), *defines, "-c", "-o", obj, str(CSRC / src)]
            return subprocess.run(cmd, capture_output=True, text=True)

        with ThreadPoolExecutor(max_workers=max(1, min(len(SOURCES), os.cpu_count() or 1))) as ex:
            results = list(ex.map(compile_one, zip(SOURCES, objs)))
        link = subprocess.run([nvcc, *ARCH_FLAGS, "-shared", "-o", str(target), *objs], capture_output=True, text=True) \
            if all(r.returncode == 0 for r in results) else None
        for r in [*results, *([link] if link else [])]:
            if r.returncode != 0:
                raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
            if verbose:
                print(r.stderr)
    return target


if __name__ == "__main__":
    _out = sys.argv[sys.argv.index("-o") + 1] if "-o" in sys.argv else None
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, defines=tuple(a for a in sys.argv[1:] if a.startswith("-D")), out=_out))
