"""DSSP secondary structure on the GPU (K18), the assignment of DSSP 2.2.0 that mdtraj's ``compute_dssp`` ports.

  CODES / LETTERS      device codes (uint8) and their DSSP letters: 0 loop ' ', 1 H, 2 B, 3 E, 4 G, 5 I, 6 T, 7 S
  FULL_INT / SIMPLE_INT  the integer tables of MetricSecondaryStructure (full and simplified), indexed by device code
  SIMPLE_LETTERS       the simplified letter of every device code (H G I -> H, E B -> E, T S loop -> C)
  bend_threshold       the smallest double c with acos(c) 180 / pi <= 70, bisected against libm
  dssp_device          (n, n_res) uint8 codes per listed frame, optionally both hydrogen-bond slots of every donor

CUDA tensors in, stream-ordered, like :func:`moleculekit_b200.sasa.sasa_device`.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import functools
import struct

import numpy as np
import torch

from . import _lib
from .coords import _rows

LOOP, HELIX, BRIDGE, STRAND, HELIX3, HELIX5, TURN, BEND = range(8)
LETTERS = np.array([" ", "H", "B", "E", "G", "I", "T", "S"])
SIMPLE_LETTERS = np.array(["C", "H", "E", "E", "H", "H", "C", "C"])
# MetricSecondaryStructure's integer tables, indexed by device code
FULL_INT = np.array([7, 0, 1, 2, 3, 4, 5, 6], np.int64)       # H 0, B 1, E 2, G 3, I 4, T 5, S 6, ' ' 7
SIMPLE_INT = np.array([2, 0, 1, 1, 0, 0, 2, 2], np.int64)     # H 0, E 1, C 2

FLAG_PRO = 1
FLAG_CHAIN_START = 2


def _bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _float(b: int) -> float:
    return struct.unpack("<d", struct.pack("<q", b))[0]


@functools.lru_cache(maxsize=None)
def bend_threshold() -> float:
    """The smallest double c with (acos(c) * 180) / pi <= 70 under the C library's ``acos``: a kappa angle above 70
    degrees (a bend) is exactly c < bend_threshold().  Bisection over the ordered positive doubles."""
    libm = C.CDLL(ctypes.util.find_library("m"))
    libm.acos.argtypes = [C.c_double]
    libm.acos.restype = C.c_double

    def le70(c):
        return (libm.acos(c) * 180) / 3.14159265358979323846 <= 70

    lo, hi = _bits(0.3), _bits(0.4)  # cos(70 deg) = 0.342; acos(0.3) is above 70 degrees, acos(0.4) below
    assert not le70(_float(lo)) and le70(_float(hi))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if le70(_float(mid)):
            hi = mid
        else:
            lo = mid
    return _float(hi)


def chunk_frames(n_res: int) -> int:
    """Listed frames per chunk of one :func:`dssp_device` call (its scratch stays bounded whatever the frame count)."""
    return int(_lib.load().mkb_dssp_chunk_frames(int(n_res)))


def dssp_device(coords, backbone, flags, frames=None, out=None, hbonds=None):
    """DSSP codes (see mkb_dssp in include/mkb200.h for the contract).

    ``coords`` (N, 3, F) float32 frame-minor in Angstrom; ``backbone`` (n, 4) int32 atom rows of the N, CA, C, O of
    every residue of the DSSP sequence; ``flags`` (n,) uint8 (bit 0 proline, bit 1 starts a new chain or segid).
    ``frames`` int32 (None = every frame).  ``out`` (optional) receives the (m, n) uint8 rows (unit column stride, any
    row stride).  ``hbonds`` (optional) = (partner (m, n, 2) int32, energy (m, n, 2) float64) contiguous tensors that
    receive both slots of every donor.  Returns ``out``."""
    dev = _lib.tensor_device(coords, "dssp_device")
    _lib.index_arg(backbone, dev, cols=4)
    nres = int(backbone.shape[0])
    assert flags.dtype == torch.uint8 and flags.device == dev and flags.is_contiguous() and flags.shape == (nres,)
    if nres == 0:
        raise ValueError("dssp_device needs at least one residue")
    _lib.index_arg(frames, dev)
    n = coords.shape[2] if frames is None else int(frames.numel())
    out = _rows(out, n, nres, torch.uint8, dev)
    hp = he = None
    if hbonds is not None:
        hp, he = hbonds
        assert hp.dtype == torch.int32 and he.dtype == torch.float64 and hp.device == dev and he.device == dev
        assert tuple(hp.shape) == (n, nres, 2) and tuple(he.shape) == (n, nres, 2)
        assert hp.is_contiguous() and he.is_contiguous()
    if n == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return out
    ld = max(out.stride(0) if n > 1 else nres, nres)
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_dssp", C.byref(t), _lib.ptr(backbone), _lib.ptr(flags), nres, bend_threshold(),
              _lib.ptr(frames), n, _lib.ptr(out), ld, _lib.ptr(hp), _lib.ptr(he))
    return out
