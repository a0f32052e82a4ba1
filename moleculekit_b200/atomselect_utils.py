"""`within` / `exwithin` atom selections on the GPU (K10, SURVEY 8f row 3).

Mirrors the one hot function of the reference's selection engine:

  within_distance(coords, cutoff, sel1, sel2, sel2_min_coords, sel2_max_coords, results)
        moleculekit/atomselect_utils/atomselect_utils.pyx:612-653   (results updated in place)
  within(mol, cutoff, source, exclude_source)     the node evaluation of moleculekit/atomselect/atomselect.py:231-254

The reference loops over all (query, source) pairs; `mkb_within_distance` bins the source atoms into cutoff-sized cells
(csrc/bonds.cu, the K7 grid) and gives the same mask.  The selection *language* stays with moleculekit (SURVEY 2b).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from .distance_utils import _check


def as_mask(sel, n: int) -> np.ndarray:
    """(n,) bool mask of ``sel``, a boolean mask or an index array (either of what ``atomselect`` returns)."""
    mask = np.asarray(sel)
    if mask.dtype != bool:
        m = np.zeros(n, dtype=bool)
        m[mask] = True
        mask = m
    return mask


def within_distance_device(coords: torch.Tensor, cutoff: float, sel2: torch.Tensor, sel1: torch.Tensor | None = None,
                           results: torch.Tensor | None = None) -> torch.Tensor:
    """K10 on CUDA tensors: coords (N,3) f32 contiguous, sel2 (source) / sel1 (queries; None = all atoms) int32 index
    tensors.  Returns the bool mask over the queries (entries already True in ``results`` stay True)."""
    dev = coords.device
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.is_contiguous() and coords.ndim == 2
    assert coords.shape[1] == 3
    n1 = int(coords.shape[0]) if sel1 is None else int(sel1.numel())
    if results is None:
        results = torch.zeros(n1, dtype=torch.bool, device=dev)
    assert results.dtype == torch.bool and results.is_contiguous() and results.numel() == n1
    _lib.call(dev, "mkb_within_distance", _lib.ptr(coords), int(coords.shape[0]), _lib.ptr(sel1), n1, _lib.ptr(sel2),
              int(sel2.numel()), float(np.float32(cutoff)), _lib.ptr(results))
    return results


def within_distance(coords, cutoff, sel1, sel2, sel2_min_coords, sel2_max_coords, results, device=None):
    """Drop-in for atomselect_utils.pyx:612-620: ``results`` (bool, one per sel1 entry) is updated in place.  The min / max
    arguments exist for signature compatibility (they feed a pre-check that never rejects anything in the reference)."""
    if not isinstance(coords, np.ndarray) or coords.dtype != np.float32:
        raise ValueError("Buffer dtype mismatch, expected 'float32' for coords")
    if coords.ndim != 2:
        raise ValueError(f"Buffer has wrong number of dimensions (expected 2, got {coords.ndim})")
    _check("sel1", sel1, np.uint32, 1); _check("sel2", sel2, np.uint32, 1)
    _check("results", results, np.bool_, 1)
    if len(sel1) == 0 or len(sel2) == 0:
        return
    n = coords.shape[0]
    if int(sel1.max()) >= n or int(sel2.max()) >= n:
        raise IndexError("atom index out of range")
    dev = _lib.device(device)
    d_coords = torch.from_numpy(np.ascontiguousarray(coords[:, :3])).to(dev)
    d1 = torch.from_numpy(np.ascontiguousarray(sel1).view(np.int32)).to(dev)
    d2 = torch.from_numpy(np.ascontiguousarray(sel2).view(np.int32)).to(dev)
    d_res = torch.from_numpy(np.ascontiguousarray(results)).to(dev)
    within_distance_device(d_coords, cutoff, d2, d1, d_res)
    results[...] = d_res.cpu().numpy()


def within(mol, cutoff: float, source, exclude_source: bool = False, device=None) -> np.ndarray:
    """`within <cutoff> of <source>` (exclude_source: `exwithin`) on frame ``mol.frame``: atomselect.py:231-254.
    ``source`` is a boolean mask or an index array; returns the boolean mask over all atoms."""
    n = int(mol.numAtoms)
    src = as_mask(source, n)
    mask = np.zeros(n, dtype=bool)
    if not np.any(src):
        return mask
    frame = getattr(mol, "frame", 0)
    coords = np.ascontiguousarray(mol.coords[:, :, frame])
    source_coor = coords[src]
    within_distance(coords, cutoff, np.arange(0, n).astype(np.uint32), np.where(src)[0].astype(np.uint32),
                    source_coor.min(axis=0), source_coor.max(axis=0), mask, device=device)
    if exclude_source:
        mask[src] = False
    return mask
