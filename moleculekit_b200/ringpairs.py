"""Ring-based interaction kernels on the GPU (K13) -- mirrors of the reference's ``moleculekit.interactions.pipi``,
``.cationpi`` and ``.sigmahole`` extensions.

  pipi_calculate(rings_atoms, rings1_start_indexes, rings2_start_indexes, coords, box, dist_threshold1=4.4,
                 angle_threshold1_max=30, dist_threshold2=5.5, angle_threshold2_min=60)        pipi/pipi.pyx:86-185
  cationpi_calculate(rings_atoms, rings_start_indexes, cations, coords, box, dist_threshold=5,
                     angle_threshold_min=60)                                                   cationpi/cationpi.pyx:91-173
  sigmahole_calculate(rings_atoms, rings_start_indexes, halogen_bond, coords, box, dist_threshold=4.5,
                      angle_threshold_min=60)                                                  sigmahole/sigmahole.pyx:91-174

Same arguments, same return value as the Cython ``calculate`` functions: ``(results, distangles)``, per frame a flat int list
``[ring, partner, ...]`` and a flat float list ``[distance, angle, ...]``.  The pair tests run in ``mkb_ring_pairs_count`` +
``mkb_ring_pairs_fill`` (csrc/rings.cu): pairs and distances are the reference's, angles agree to a few float ulp.  Only the
atoms the call touches cross PCIe.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .distance_utils import _check, upload_selected

PIPI, CATIONPI, SIGMAHOLE = 0, 1, 2


def calculate_device(mode: int, coords, box, rings_atoms, starts1, second, p0, p1=0.0, p2=0.0, p3=0.0):
    """K13 on CUDA tensors.  coords (N, 3, F) float32 frame-minor, box (3, F); rings_atoms / starts1 / second int32
    (uint32-valued).  Returns (frame_offsets (F+1,) int64, pairs (total, 2) int32, distangles (total, 2) float32), all cuda."""
    dev = coords.device
    F = coords.shape[2]
    n1 = int(starts1.shape[0]) - 1
    n2 = int(second.shape[0]) - 1 if mode == PIPI else int(second.shape[0])
    tr = _lib.traj(coords, box)
    row_off = torch.empty(F * max(n1, 0) + 1, dtype=torch.int64, device=dev)
    args = (int(mode), C.byref(tr), _lib.ptr(rings_atoms), _lib.ptr(starts1), n1, _lib.ptr(second), n2,
            float(np.float32(p0)), float(np.float32(p1)), float(np.float32(p2)), float(np.float32(p3)))
    pairs, da = _lib.count_fill(dev, "mkb_ring_pairs_count", "mkb_ring_pairs_fill", args, row_off,
                                lambda total: (torch.empty((total, 2), dtype=torch.int32, device=dev),
                                               torch.empty((total, 2), dtype=torch.float32, device=dev)))
    frame_off = row_off[::n1] if n1 > 0 else torch.zeros(F + 1, dtype=torch.int64, device=dev)
    return frame_off.contiguous(), pairs, da


def check_ring_sizes(name, starts):
    """Every ring needs at least 3 atoms: its normal comes from the first three.  The reference reads atoms of the next ring
    (or past the end of the atom list) for a shorter one, so such a ring has no defined answer and is rejected."""
    sizes = np.diff(np.asarray(starts, dtype=np.int64))
    bad = np.flatnonzero(sizes < 3)
    if bad.size:
        i = int(bad[0])
        raise ValueError(f"ring {i} of {name} has {int(sizes[i])} atoms; rings need at least 3")


def calculate_arrays(mode, rings_atoms, starts1, second, coords, box, p0, p1=0.0, p2=0.0, p3=0.0, device=None):
    """(frame_offsets (F+1,), pairs (total, 2) int32 -- partner atoms as ORIGINAL indexes --, distangles (total, 2) float32).
    Raises ValueError for a ring of fewer than 3 atoms."""
    _check("rings_atoms", rings_atoms, np.uint32, 1); _check("rings_start_indexes", starts1, np.uint32, 1)
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    second = np.ascontiguousarray(second)
    if second.dtype != np.uint32:
        raise ValueError("Buffer dtype mismatch, expected 'uint32'")
    check_ring_sizes("rings_start_indexes" if mode != PIPI else "rings1_start_indexes", starts1)
    if mode == PIPI:
        check_ring_sizes("rings2_start_indexes", second)
    F = coords.shape[2]
    n1 = len(starts1) - 1
    n2 = len(second) - 1 if mode == PIPI else len(second)
    if F == 0 or n1 <= 0 or n2 <= 0:
        return np.zeros(F + 1, np.int64), np.zeros((0, 2), np.int32), np.zeros((0, 2), np.float32)
    sets = [rings_atoms] + ([] if mode == PIPI else [second.reshape(-1)])
    d_coords, d_box, remap, _, _ = upload_selected(coords, box, sets, device=device)
    dev = d_coords.device
    used = np.flatnonzero(remap >= 0)
    to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).astype(np.int32)).to(dev)
    sec_dev = to_dev(second) if mode == PIPI else to_dev(remap[second.astype(np.int64)])
    off, pairs, da = calculate_device(mode, d_coords, d_box, to_dev(remap[rings_atoms.astype(np.int64)]), to_dev(starts1),
                                      sec_dev, p0, p1, p2, p3)
    pairs = pairs.cpu().numpy()
    if mode != PIPI and pairs.size:
        pairs[:, 1] = used.astype(np.int32)[pairs[:, 1]]  # compact ids -> original atom indexes
    return off.cpu().numpy(), pairs, da.cpu().numpy()


def _lists(off, pairs, da):
    F = len(off) - 1
    return ([pairs[off[f]:off[f + 1]].reshape(-1).tolist() for f in range(F)],
            [da[off[f]:off[f + 1]].reshape(-1).tolist() for f in range(F)])


def pipi_calculate(rings_atoms, rings1_start_indexes, rings2_start_indexes, coords, box, dist_threshold1=4.4,
                   angle_threshold1_max=30, dist_threshold2=5.5, angle_threshold2_min=60, device=None):
    """Drop-in for pipi.calculate (pipi.pyx:86-97)."""
    return _lists(*calculate_arrays(PIPI, rings_atoms, rings1_start_indexes, rings2_start_indexes, coords, box,
                                    dist_threshold1, angle_threshold1_max, dist_threshold2, angle_threshold2_min, device=device))


def cationpi_calculate(rings_atoms, rings_start_indexes, cations, coords, box, dist_threshold=5, angle_threshold_min=60,
                       device=None):
    """Drop-in for cationpi.calculate (cationpi.pyx:91-99)."""
    return _lists(*calculate_arrays(CATIONPI, rings_atoms, rings_start_indexes, cations, coords, box, dist_threshold,
                                    angle_threshold_min, device=device))


def sigmahole_calculate(rings_atoms, rings_start_indexes, halogen_bond, coords, box, dist_threshold=4.5,
                        angle_threshold_min=60, device=None):
    """Drop-in for sigmahole.calculate (sigmahole.pyx:91-99)."""
    return _lists(*calculate_arrays(SIGMAHOLE, rings_atoms, rings_start_indexes, halogen_bond, coords, box, dist_threshold,
                                    angle_threshold_min, device=device))
