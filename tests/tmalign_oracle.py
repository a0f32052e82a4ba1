"""ctypes front-end of tests/tmalign_oracle.c, the CPU restatement of TM-align (K27 parity tests, smoke() and
bench_tmalign.py).  TEST INFRASTRUCTURE ONLY: the package never imports it.

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
SRC = os.path.join(HERE, "tmalign_oracle.c")

_lib = None


def build() -> str:
    src = open(SRC, "rb").read()
    tag = hashlib.sha256(src).hexdigest()[:16]
    lib = os.path.join(tempfile.gettempdir(), f"mkb_tmalign_oracle_{os.getuid()}_{tag}.so")
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
        vp = C.c_void_p
        _lib.oracle_tmalign_frame.argtypes = [vp, C.c_int32, vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp]
        _lib.oracle_tmalign_frame.restype = C.c_int
        _lib.oracle_tmalign_sec.argtypes = [vp, C.c_int32, vp]
        _lib.oracle_tmalign_sec.restype = None
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def secondary(x) -> str:
    """The secondary-structure codes of one CA trace ``x`` (L, 3)."""
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(x.shape[0], np.uint8)
    lib().oracle_tmalign_sec(_p(x), x.shape[0], _p(out))
    return out.tobytes().decode()


def frame(x, y):
    """One item: ``x`` (xlen, 3) mol trace onto ``y`` (ylen, 3) reference trace, float32.  Returns a dict with tm (2,)
    [TM_ref, TM_mol], rmsd, nali, invmap (ylen,) int32, record (16,) and counts (DP cells, fits, pair evaluations)."""
    from moleculekit_b200.tmalign import tmalign_parameters

    x = np.ascontiguousarray(x, np.float32)
    y = np.ascontiguousarray(y, np.float32)
    params = tmalign_parameters(x.shape[0], y.shape[0])
    tm, rmsd, nali = np.zeros(2), np.zeros(1), np.zeros(1, np.int32)
    invmap = np.zeros(y.shape[0], np.int32)
    rec = np.zeros(16)
    counts = np.zeros(3, np.int64)
    rc = lib().oracle_tmalign_frame(_p(x), x.shape[0], _p(y), y.shape[0], _p(params), _p(tm), _p(rmsd), _p(nali),
                                    _p(invmap), _p(rec), _p(counts))
    assert rc == 0
    return dict(tm=tm, rmsd=float(rmsd[0]), nali=int(nali[0]), invmap=invmap, record=rec, counts=tuple(counts))


def tmalign(X, Y, frames=None, matching=False):
    """Over the listed frames of ``X`` (xlen, 3, F) onto ``Y`` (ylen, 3) (or (ylen, 3, F) with ``matching``: item k
    onto reference frame frames[k]).  Returns (tm (n, 2), rmsd (n,), nali (n,) int32, invmap (n, ylen), records
    (n, 16))."""
    X = np.asarray(X, np.float32)
    Y = np.asarray(Y, np.float32)
    frames = range(X.shape[2]) if frames is None else list(frames)
    n = len(frames)
    tm, rmsd, nali = np.zeros((n, 2)), np.zeros(n), np.zeros(n, np.int32)
    invmap, rec = np.zeros((n, Y.shape[0]), np.int32), np.zeros((n, 16))
    for k, f in enumerate(frames):
        r = frame(X[:, :, f], Y[:, :, f] if matching else Y)
        tm[k], rmsd[k], nali[k], invmap[k], rec[k] = r["tm"], r["rmsd"], r["nali"], r["invmap"], r["record"]
    return tm, rmsd, nali, invmap, rec
