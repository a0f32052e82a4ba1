"""ctypes front-end of tests/tmscore_oracle.c, the CPU restatement of the TM-score superposition search (K19 parity
tests, smoke() and bench_tmscore.py).  TEST INFRASTRUCTURE ONLY: the package never imports it.

The shared object is compiled with gcc -O3 -ffp-contract=off into the system's temporary directory, keyed by the
source's hash, so a read-only tree works."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "tmscore_oracle.c")

_lib = None


def build() -> str:
    src = open(SRC, "rb").read()
    tag = hashlib.sha256(src).hexdigest()[:16]
    lib = os.path.join(tempfile.gettempdir(), f"mkb_tmscore_oracle_{os.getuid()}_{tag}.so")
    if not os.path.isfile(lib):
        tmp = f"{lib}.{os.getpid()}"
        subprocess.run(["gcc", "-O3", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-shared", "-fPIC",
                        SRC, "-o", tmp, "-lm"], check=True)
        os.replace(tmp, lib)
    return lib


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.oracle_tmscore_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_double, C.c_double,
                                              C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.oracle_tmscore_frame.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def frame(x, y, lnorm=None):
    """One frame: ``x`` (L, 3) model and ``y`` (L, 3) reference float32, pair k = (x[k], y[k]); ``lnorm`` defaults to L.
    Returns (tm, rmsd, (seeds, fits, pair evaluations))."""
    from moleculekit_b200.tmscore import tm_parameters

    x = np.ascontiguousarray(x, np.float32)
    y = np.ascontiguousarray(y, np.float32)
    L = x.shape[0]
    assert x.shape == (L, 3) and y.shape == (L, 3) and L >= 1
    lnorm = L if lnorm is None else int(lnorm)
    d0, d0s, frag = tm_parameters(L, lnorm)
    frag = np.asarray(frag, np.int32)
    tm, rmsd = np.zeros(1), np.zeros(1)
    counts = np.zeros(3, np.int64)
    rc = lib().oracle_tmscore_frame(_p(x), _p(y), L, lnorm, d0, d0s, _p(frag), frag.size, _p(tm), _p(rmsd),
                                    _p(counts))
    assert rc == 0
    return float(tm[0]), float(rmsd[0]), tuple(int(c) for c in counts)


def tmscore(X, Y, frames=None):
    """Over the listed frames of ``X`` (n, 3, F) float32 against ``Y`` (m, 3) float32: pairs k < min(n, m), Lnorm = m.
    Returns (tm (len,) float64, rmsd (len,) float64)."""
    X = np.asarray(X, np.float32)
    Y = np.asarray(Y, np.float32)
    L = min(X.shape[0], Y.shape[0])
    frames = range(X.shape[2]) if frames is None else list(frames)
    tm = np.zeros(len(frames))
    rmsd = np.zeros(len(frames))
    for k, f in enumerate(frames):
        tm[k], rmsd[k], _ = frame(X[:L, :, f], Y[:L], Y.shape[0])
    return tm, rmsd
