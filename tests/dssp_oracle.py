"""ctypes front-end of tests/dssp_oracle.c, the CPU restatement of the DSSP 2.2.0 assignment that mdtraj's compute_dssp
ports (K18 parity tests, smoke() and bench_dssp.py).  TEST INFRASTRUCTURE ONLY: the package never imports it.

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
SRC = os.path.join(HERE, "dssp_oracle.c")

_lib = None


def build() -> str:
    src = open(SRC, "rb").read()
    tag = hashlib.sha256(src).hexdigest()[:16]
    lib = os.path.join(tempfile.gettempdir(), f"mkb_dssp_oracle_{os.getuid()}_{tag}.so")
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
        _lib.oracle_dssp_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]
        _lib.oracle_dssp_frame.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def frame(bb, flags):
    """One frame: ``bb`` (n, 4, 3) float32 N, CA, C, O per residue, ``flags`` (n,) uint8 (bit 0 PRO, bit 1 chain start).
    Returns (codes (n,) uint8, partner (n, 2) int32, energy (n, 2) float64, (CA pairs screened, energies evaluated))."""
    bb = np.ascontiguousarray(bb, np.float32)
    flags = np.ascontiguousarray(flags, np.uint8)
    n = bb.shape[0]
    assert bb.shape == (n, 4, 3) and flags.shape == (n,)
    codes = np.zeros(n, np.uint8)
    partner = np.zeros((n, 2), np.int32)
    energy = np.zeros((n, 2), np.float64)
    counts = np.zeros(2, np.int64)
    rc = lib().oracle_dssp_frame(_p(bb), _p(flags), n, _p(codes), _p(partner), _p(energy), _p(counts))
    assert rc == 0
    return codes, partner, energy, (int(counts[0]), int(counts[1]))


def _place(a, b, c, bond, angle, torsion):
    """the point d with |cd| = bond, angle bcd = angle and dihedral abcd = torsion (degrees)"""
    bc = c - b
    bc /= np.linalg.norm(bc)
    nrm = np.cross(b - a, bc)
    nrm /= np.linalg.norm(nrm)
    m = np.stack([bc, np.cross(nrm, bc), nrm], 1)
    ang, t = np.radians(angle), np.radians(torsion)
    return c + m @ np.array([-bond * np.cos(ang), bond * np.sin(ang) * np.cos(t), bond * np.sin(ang) * np.sin(t)])


def chain(phi, psi, omega=180.0):
    """(n, 4, 3) float64 N, CA, C, O of a chain with standard bond lengths and angles and the given torsions (degrees);
    O lies in the peptide plane (dihedral N CA C O = psi + 180)."""
    n = len(phi)
    N, CA = [np.zeros(3)], [np.array([1.458, 0.0, 0.0])]
    C = [CA[0] + 1.525 * np.array([-np.cos(np.radians(111.2)), np.sin(np.radians(111.2)), 0.0])]
    O = []
    for i in range(n):
        O.append(_place(N[i], CA[i], C[i], 1.231, 120.5, psi[i] + 180))
        if i + 1 < n:
            N.append(_place(N[i], CA[i], C[i], 1.329, 116.2, psi[i]))
            CA.append(_place(CA[i], C[i], N[i + 1], 1.458, 121.7, omega))
            C.append(_place(C[i], N[i + 1], CA[i + 1], 1.525, 111.2, phi[i + 1]))
    return np.stack([np.stack(N), np.stack(CA), np.stack(C), np.stack(O)], 1)


def strand_pair(n, antiparallel, dist=4.5, shift=None):
    """Two n-residue strands as separate chains: strand B is strand A turned 180 degrees about the axis normal to the
    strand and to its C=O direction (antiparallel) or A itself (parallel), moved ``dist`` A along the C=O direction and
    ``shift`` A along the strand.  Returns ((2n, 4, 3) float32, flags)."""
    phi, psi = (-139, 135) if antiparallel else (-119, 113)
    shift = (-3.5 if antiparallel else -1.5) if shift is None else shift
    A = chain([phi] * n, [psi] * n)
    X = A - A[:, 1].mean(0)
    u = A[-1, 1] - A[0, 1]
    u /= np.linalg.norm(u)
    v = A[n // 2, 3] - A[n // 2, 2]
    v -= (v @ u) * u
    v /= np.linalg.norm(v)
    B = X.copy()
    if antiparallel:
        w = np.cross(u, v)
        B = B @ (2 * np.outer(w, w) - np.eye(3)).T
    B = B + dist * v + shift * u
    flags = np.zeros(2 * n, np.uint8)
    flags[n] = 2
    return np.concatenate([X, B]).astype(np.float32), flags


def dssp(coords, backbone, flags, frames=None):
    """Over the listed frames of ``coords`` (N, 3, F) float32: ``backbone`` (n, 4) atom rows of N, CA, C, O.  Returns
    (codes (m, n) uint8, partner (m, n, 2) int32, energy (m, n, 2) float64)."""
    coords = np.asarray(coords, np.float32)
    backbone = np.asarray(backbone, np.int64).reshape(-1, 4)
    frames = range(coords.shape[2]) if frames is None else list(frames)
    n = backbone.shape[0]
    codes = np.zeros((len(frames), n), np.uint8)
    partner = np.zeros((len(frames), n, 2), np.int32)
    energy = np.zeros((len(frames), n, 2), np.float64)
    for k, f in enumerate(frames):
        codes[k], partner[k], energy[k], _ = frame(coords[backbone, :, f], flags)
    return codes, partner, energy
