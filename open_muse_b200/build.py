"""Builds libmuse_b200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

No torch headers are involved: the library's ABI is plain C (include/muse_b200.h) and the Python
host side binds it with ctypes.  Objects are compiled in parallel and cached by source mtime.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD_DIR = PKG_DIR / "csrc" / "build"
LIB_PATH = PKG_DIR / "libmuse_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: libmuse_b200.so cannot be built (there is no CPU fallback)")


def _newer(src: Path, dst: Path, deps) -> bool:
    if not dst.exists():
        return True
    t = dst.stat().st_mtime
    return any(p.stat().st_mtime > t for p in [src, *deps])


def build(verbose: bool = False, force: bool = False) -> Path:
    nvcc = _nvcc()
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + [PKG_DIR.parent / "include" / "muse_b200.h"]
    objs = []
    jobs = []
    for src in sources:
        obj = BUILD_DIR / (src.stem + ".o")
        objs.append(obj)
        if force or _newer(src, obj, headers):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or force or not LIB_PATH.exists():
        run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB_PATH), *map(str, objs)])
    return LIB_PATH


XCHECK_DIR = PKG_DIR.parent / "tests" / "xcheck"
XCHECK_LIB = XCHECK_DIR / "libmuse_b200_xcheck.so"


def build_xcheck(verbose: bool = False, force: bool = False) -> Path:
    """TEST-ONLY cross-check library (tests/xcheck): the first-generation mma.sync GEMM / attention kernels the GPU tests
    compare the wgmma product kernels against.  Never linked into libmuse_b200.so."""
    nvcc = _nvcc()
    src_dir = XCHECK_DIR / "csrc"
    out_dir = src_dir / "build"
    out_dir.mkdir(parents=True, exist_ok=True)
    sources = sorted(src_dir.glob("*.cu"))
    headers = [CSRC / "common.cuh", PKG_DIR.parent / "include" / "muse_b200.h"]
    objs, jobs = [], []
    for src in sources:
        obj = out_dir / (src.stem + ".o")
        objs.append(obj)
        if force or _newer(src, obj, headers):
            jobs.append([nvcc, *NVCC_FLAGS, "-I", str(CSRC), "-c", str(src), "-o", str(obj)])
    for cmd in jobs:
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    if jobs or force or not XCHECK_LIB.exists():
        r = subprocess.run([nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(XCHECK_LIB), *map(str, objs)],
                           capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc link failed:\n{r.stdout}\n{r.stderr}")
    return XCHECK_LIB


if __name__ == "__main__":
    p = build(verbose=True, force="--force" in sys.argv)
    print(p)
    print(build_xcheck(verbose=True, force="--force" in sys.argv))
