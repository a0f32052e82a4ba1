"""Torsion angles on the GPU (K16).

  dihedrals_device    (n, m) float32 angles in radians, or (n, 2m) float32 sin, cos pairs, of m atom quadruples
  dihedralAngle       host mirror of ``moleculekit.dihedral.dihedralAngle`` for one (4, 3) position

CUDA tensors in, stream-ordered, like :func:`moleculekit_b200.coords.coordinates_device`: ``coords`` is the (N, 3, F)
float32 frame-minor trajectory (or a frame slice of one), ``quads`` an (m, 4) int32 CUDA tensor of atom rows and
``frames`` an int32 CUDA tensor (None = every frame; row k belongs to frame ``frames[k]``).  The coordinates are used
as given: no minimum image, no superposition (a dihedral does not change under a rigid motion).  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .coords import _rows


def dihedralAngle(pos) -> float:
    """The dihedral angle in radians of the four points ``pos`` (4, 3), in float64: b0 = p0 - p1, b1 = p2 - p1,
    b2 = p3 - p2, u = b1 / |b1|, v and w = b0 and b2 with their components along u removed, angle = atan2((u x v).w,
    v.w).  The sign is IUPAC's: positive when p1-p0 turns clockwise onto p2-p3 seen along p1 -> p2.  The kernel
    evaluates the same expression.  A degenerate quadruple (b0 x b1 or b1 x b2 exactly zero: three collinear points,
    in any orientation, or p1 == p2) gives 0, a non-finite coordinate NaN."""
    p = np.asarray(pos, dtype=np.float64)
    if p.shape != (4, 3):
        raise RuntimeError("dihedralAngles requires a 4x3 sized coordinate matrix as input.")
    if not np.isfinite(p).all():
        return float("nan")
    b0, b1, b2 = p[0] - p[1], p[2] - p[1], p[3] - p[2]
    if not np.cross(b0, b1).any() or not np.cross(b1, b2).any():  # degenerate; numpy does not fuse the products
        return 0.0
    u = b1 / np.sqrt(b1 @ b1)
    v = b0 - (b0 @ u) * u
    w = b2 - (b2 @ u) * u
    x, y = v @ w, np.cross(u, v) @ w
    return 0.0 if x == 0 and y == 0 else float(np.arctan2(y, x))


def dihedrals_device(coords, quads, sincos, frames=None, out=None):
    """Per listed frame and quadruple, the dihedral angle evaluated in float64 and rounded once to float32.

    ``sincos`` False: (n, m) angles in radians, in [-pi, pi].  ``sincos`` True: (n, 2m), columns sin, cos interleaved
    per quadruple, computed from the projected components as (y, x) / hypot(x, y) rather than through the angle.  A
    degenerate quadruple (b0 x b1 or b1 x b2 exactly zero in float64: three collinear points, or coincident middle
    atoms) gives angle 0 and (sin, cos) = (0, 1); a non-finite coordinate gives NaN.  ``frames`` must be an int32
    tensor on the trajectory's device.  ``out`` (optional) receives the rows, e.g. a frame shard's rows of a whole
    trajectory's matrix (unit column stride, any row stride)."""
    dev = _lib.tensor_device(coords, "dihedrals_device")
    _lib.index_arg(quads, dev, cols=4)
    _lib.index_arg(frames, dev)
    m = int(quads.shape[0])
    nv = 2 if sincos else 1
    n = coords.shape[2] if frames is None else int(frames.numel())
    out = _rows(out, n, nv * m, torch.float32, dev)
    if n == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return out
    ld = max(out.stride(0) if n > 1 else nv * m, nv * m)
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_dihedrals", C.byref(t), _lib.ptr(quads), m, _lib.ptr(frames), n, 1 if sincos else 0,
              _lib.ptr(out), ld)
    return out
