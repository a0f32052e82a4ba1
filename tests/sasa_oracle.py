"""ctypes front-end of tests/sasa_oracle.c, the CPU restatement of mdtraj's Shrake-Rupley loop (K17 parity tests,
smoke() and bench_sasa.py).  TEST INFRASTRUCTURE ONLY: the package never imports it.

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
SRC = os.path.join(HERE, "sasa_oracle.c")

_lib = None


class CoincidentAtoms(ValueError):
    def __init__(self, frame, pair):
        self.frame, self.pair = int(frame), (int(pair[0]), int(pair[1]))
        super().__init__(f"atoms {self.pair} coincide in frame {self.frame}")


def build() -> str:
    src = open(SRC, "rb").read()
    tag = hashlib.sha256(src).hexdigest()[:16]
    lib = os.path.join(tempfile.gettempdir(), f"mkb_sasa_oracle_{os.getuid()}_{tag}.so")
    if not os.path.isfile(lib):
        tmp = f"{lib}.{os.getpid()}"
        subprocess.run(["gcc", "-O3", "-ffp-contract=off", "-fno-fast-math", "-fvisibility=hidden", "-shared", "-fPIC",
                        SRC, "-o", tmp], check=True)
        os.replace(tmp, lib)
    return lib


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.oracle_sasa_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_int32, C.c_void_p, C.c_void_p]
        _lib.oracle_sasa_frame.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def areas_nm(xyz_nm, radii, atoms, sphere):
    """float32 areas in nm^2 of the ``atoms`` of one frame, (n, 3) float32 nm coordinates; CoincidentAtoms (frame -1)
    where the reference would exit."""
    xyz = np.ascontiguousarray(xyz_nm, np.float32)
    radii = np.ascontiguousarray(radii, np.float32)
    atoms = np.ascontiguousarray(atoms, np.int64)
    sphere = np.ascontiguousarray(sphere, np.float32)
    out = np.zeros(atoms.size, np.float32)
    bad = np.zeros(2, np.int64)
    rc = lib().oracle_sasa_frame(_p(xyz), _p(radii), xyz.shape[0], _p(atoms), atoms.size, _p(sphere),
                                 sphere.shape[0], _p(out), _p(bad))
    if rc == 1:
        raise CoincidentAtoms(-1, bad)
    assert rc == 0
    return out


def sasa(coords, radii, query, sphere, groups=None, frames=None):
    """(n, m) float32 Angstrom^2 over the listed frames of ``coords`` (N, 3, F) in Angstrom, every atom of ``coords``
    being an environment atom: per query atom fl(a 100), or with ``groups`` (offsets into ``query``) fl(s 100) of the
    areas of each group added in order into a float32 zero."""
    coords = np.asarray(coords, np.float32)
    query = np.asarray(query, np.int64)
    frames = range(coords.shape[2]) if frames is None else frames
    cols = query.size if groups is None else len(groups) - 1
    out = np.zeros((len(frames), cols), np.float32)
    hundred = np.float32(100)
    for r, f in enumerate(frames):
        x = coords[:, :, f] / np.float32(10)
        try:
            a = areas_nm(x, radii, query, sphere)
        except CoincidentAtoms as e:
            raise CoincidentAtoms(f, e.pair) from None
        if groups is None:
            out[r] = a * hundred
        else:
            for g in range(cols):
                s = np.float32(0)
                for v in a[groups[g]:groups[g + 1]]:
                    s = np.float32(s + v)
                out[r, g] = s * hundred
    return out
