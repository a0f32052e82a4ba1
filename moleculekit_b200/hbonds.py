"""Hydrogen-bond detection on the GPU (K12) -- mirror of the reference's ``moleculekit.interactions.hbonds`` extension.

  calculate(donors, acceptors, coords, box, sel1, sel2, dist_threshold=2.5, angle_threshold=120, intra=False,
            ignore_hs=False)                         moleculekit/interactions/hbonds/hbonds.pyx:25-134

Same arguments, same return value (a list over frames of flat int lists ``[heavy, hydrogen | -1, acceptor, ...]`` in
donor-major / acceptor-minor order).  The pair tests run in ``mkb_hbonds_count`` + ``mkb_hbonds_fill`` (csrc/hbonds.cu)
and give the reference's booleans bit for bit; only the atoms the call touches cross PCIe.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .distance_utils import _check, upload_selected


def calculate_device(coords, box, donors, acceptors, sel1, sel2, dist_threshold: float = 2.5,
                     angle_threshold: float = 120, intra: bool = False, ignore_hs: bool = False):
    """K12 on CUDA tensors.  coords (N, 3, F) float32 frame-minor, box (3, F) float32, donors (nd, 2) / acceptors (na,) /
    sel1 / sel2 (N,) int32 (uint32-valued).  Returns (frame_offsets (F+1,) int64 cuda, triples (total, 3) int32 cuda)."""
    dev = coords.device
    F = coords.shape[2]
    nd, na = int(donors.shape[0]), int(acceptors.shape[0])
    tr = _lib.traj(coords, box)
    row_off = torch.empty(F * nd + 1, dtype=torch.int64, device=dev)
    args = (C.byref(tr), _lib.ptr(donors), nd, _lib.ptr(acceptors), na, _lib.ptr(sel1), _lib.ptr(sel2),
            float(np.float32(dist_threshold)), float(np.float32(angle_threshold)),
            int(bool(intra)), int(bool(ignore_hs)))
    (triples,) = _lib.count_fill(dev, "mkb_hbonds_count", "mkb_hbonds_fill", args, row_off,
                                 lambda total: (torch.empty((total, 3), dtype=torch.int32, device=dev),))
    frame_off = row_off[::nd] if nd > 0 else torch.zeros(F + 1, dtype=torch.int64, device=dev)
    return frame_off.contiguous(), triples


def calculate_arrays(donors, acceptors, coords, box, sel1, sel2, dist_threshold=2.5, angle_threshold=120, intra=False,
                     ignore_hs=False, device=None):
    """(frame_offsets (F+1,) int64, triples (total, 3) int32 with ORIGINAL atom indices): the array form of calculate."""
    _check("donors", donors, np.uint32, 2); _check("acceptors", acceptors, np.uint32, 1)
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    _check("sel1", sel1, np.uint32, 1); _check("sel2", sel2, np.uint32, 1)
    F = coords.shape[2]
    if donors.shape[1] == 1:  # hbonds_calculate passes (n, 1) heavy atoms with ignore_hs (interactions.py:445-447)
        if not ignore_hs:
            raise IndexError("donors needs a hydrogen column unless ignore_hs is set")
        donors = np.hstack([donors, donors])
    if F == 0 or donors.shape[0] == 0 or acceptors.shape[0] == 0:
        return np.zeros(F + 1, np.int64), np.zeros((0, 3), np.int32)
    d_coords, d_box, remap, _, _ = upload_selected(coords, box, [donors.reshape(-1), acceptors], device=device)
    dev = d_coords.device
    used = np.flatnonzero(remap >= 0)
    to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).astype(np.int32)).to(dev)
    off, tri = calculate_device(d_coords, d_box, to_dev(remap[donors.astype(np.int64)]),
                                to_dev(remap[acceptors.astype(np.int64)]),
                                torch.from_numpy(np.ascontiguousarray(sel1[used]).view(np.int32)).to(dev),
                                torch.from_numpy(np.ascontiguousarray(sel2[used]).view(np.int32)).to(dev),
                                dist_threshold, angle_threshold, intra, ignore_hs)
    tri = tri.cpu().numpy()
    if tri.size:
        out = used.astype(np.int32)[np.maximum(tri, 0)]
        out[tri < 0] = -1
        tri = out
    return off.cpu().numpy(), tri


def calculate(donors, acceptors, coords, box, sel1, sel2, dist_threshold=2.5, angle_threshold=120, intra=False,
              ignore_hs=False, device=None):
    """Drop-in for hbonds.pyx:25-36: list (per frame) of flat lists [heavy, hydrogen | -1, acceptor, ...]."""
    off, tri = calculate_arrays(donors, acceptors, coords, box, sel1, sel2, dist_threshold, angle_threshold, intra,
                                ignore_hs, device=device)
    return [tri[off[f]:off[f + 1]].reshape(-1).tolist() for f in range(len(off) - 1)]
