"""Build libmkb200.so (hand-written CUDA for the H100, sm_90a) in-tree with nvcc.

The shared object lands in moleculekit_b200/lib/ (git-ignored).
nvcc cross-compiles without a GPU.  `python -m moleculekit_b200.build [--force]`.
"""
from __future__ import annotations

import glob
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libmkb200.so")
INCLUDE = os.path.join(ROOT, "include")

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stale() -> bool:
    if not os.path.isfile(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(INCLUDE, "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isfile(cand) or cand == "nvcc"):
            return cand
    return "nvcc"


def build(force: bool = False, verbose: bool = True, extra: list[str] | None = None, out: str | None = None) -> str:
    """``out``: alternative output name inside lib/ (tuning experiments, selected at run time with MKB200_LIB)."""
    if out is not None:
        os.makedirs(LIBDIR, exist_ok=True)
        target = os.path.join(LIBDIR, out)
        env_extra = os.environ.get("MKB_NVCC_EXTRA", "").split()
        cmd = [nvcc_path()] + NVCC_FLAGS + (extra or []) + env_extra + [f"-I{INCLUDE}", f"-I{CSRC}", "-o", target] + sources()
        if verbose:
            print("[mkb200 build]", " ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
        return target
    if not force and not _stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    env_extra = os.environ.get("MKB_NVCC_EXTRA", "").split()  # e.g. -DMKB_W_MIN_CTAS=12 for tuning experiments
    cmd = [nvcc_path()] + NVCC_FLAGS + (extra or []) + env_extra + [f"-I{INCLUDE}", f"-I{CSRC}", "-o", LIB] + sources()
    if verbose:
        print("[mkb200 build]", " ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print(LIB)
