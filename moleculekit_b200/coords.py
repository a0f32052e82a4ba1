"""Aligned coordinate features, frame sums and per-atom fluctuations (K15), and per-frame group moments (K20) on the GPU.

  coordinates_device    (n, 3k) float32 rows: the aligned coordinates of the selection, X block | Y block | Z block
  coord_sums_device     (k, 3) float64 sums over the listed frames (the mean is the sum over the frame count)
  fluctuation_device    (n, k) or (n, G) float32 squared deviations from a centre, per atom or averaged per group
  frame_moments_device  (n, G, 6) float64 weighted means and per-axis variances of groups of the selection, per frame

CUDA tensors in, stream-ordered, like :func:`moleculekit_b200.align.rmsd_device`: ``coords`` is the (N, 3, F) float32
frame-minor trajectory (or a frame slice of one), ``sel`` / ``frames`` int32 CUDA tensors (``frames`` None = every
frame; row k belongs to frame ``frames[k]``) and ``records`` the (n, 16) float64 fit records of
:func:`~moleculekit_b200.align.superpose_device` (None = no transform).  An aligned coordinate has the bits
:func:`~moleculekit_b200.align.apply_device` would write; the trajectory is never modified and the aligned trajectory
never materialised.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from .align import RECORD


def _check_records(records, n):
    if records is not None:
        assert records.dtype == torch.float64 and tuple(records.shape) == (n, RECORD) and records.is_contiguous()


def _rows(out, n, width, dtype, dev):
    """``out`` or a new (n, width) tensor; a given ``out`` may be a row / column slice of a larger matrix (unit column
    stride, any row stride)."""
    if out is None:
        return torch.empty((n, width), dtype=dtype, device=dev)
    assert out.dtype == dtype and out.device == dev and out.ndim == 2 and tuple(out.shape) == (n, width)
    assert n <= 1 or width == 0 or out.stride(1) == 1, "out needs unit column stride"
    return out


def coordinates_device(coords, sel, records=None, frames=None, out=None):
    """(n, 3k) float32: row r = the aligned coordinates of the ``sel`` atoms in listed frame r, all X of the selection in
    selection order, then all Y, then all Z.  ``out`` (optional) receives them, e.g. a frame shard's rows of a whole
    trajectory's matrix."""
    dev = _lib.tensor_device(coords, "coordinates_device")
    _lib.index_arg(sel, dev)
    _lib.index_arg(frames, dev)
    k = int(sel.numel())
    n = coords.shape[2] if frames is None else int(frames.numel())
    _check_records(records, n)
    out = _rows(out, n, 3 * k, torch.float32, dev)
    if n == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return out
    ld = max(out.stride(0) if n > 1 else 3 * k, 3 * k)
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_coordinates", C.byref(t), _lib.ptr(sel), k, _lib.ptr(frames), n, _lib.ptr(records),
              _lib.ptr(out), ld)
    return out


def coord_sums_device(coords, sel, records=None, frames=None):
    """(k, 3) float64: per selected atom and axis, the sum over the listed frames of the aligned float32 coordinate.  The
    summation order depends only on the selection and the ordered frame list (fixed chunks of 64 frames, added in
    order), so repeated calls, a frame slice and the equivalent explicit list give the same bits."""
    dev = _lib.tensor_device(coords, "coord_sums_device")
    _lib.index_arg(sel, dev)
    _lib.index_arg(frames, dev)
    k = int(sel.numel())
    n = coords.shape[2] if frames is None else int(frames.numel())
    _check_records(records, n)
    sums = torch.empty((k, 3), dtype=torch.float64, device=dev)
    if n == 0:
        return sums.zero_()
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_coord_sums", C.byref(t), _lib.ptr(sel), k, _lib.ptr(frames), n, _lib.ptr(records),
              _lib.ptr(sums))
    return sums


def fluctuation_device(coords, sel, centre, records=None, frames=None, groups=None, out=None):
    """Per listed frame and selected atom, fl32(sum_d (c_d - centre_d)^2) evaluated in float64, c the aligned float32
    coordinate and ``centre`` a (k, 3) float64 CUDA tensor (the mean or a reference structure): (n, k) float32.  With
    ``groups`` (G + 1,) int64 offsets over selection positions (0 first, k last, nondecreasing, no empty group) the
    result is (n, G): the float64 mean of each group's per-atom values, rounded once."""
    dev = _lib.tensor_device(coords, "fluctuation_device")
    _lib.index_arg(sel, dev)
    _lib.index_arg(frames, dev)
    _lib.index_arg(groups, dev, torch.int64)
    k = int(sel.numel())
    n = coords.shape[2] if frames is None else int(frames.numel())
    _check_records(records, n)
    assert centre.dtype == torch.float64 and tuple(centre.shape) == (k, 3) and centre.is_contiguous()
    G = k if groups is None else int(groups.numel()) - 1
    out = _rows(out, n, G, torch.float32, dev)
    if n == 0:
        return out
    ld = max(out.stride(0) if n > 1 else G, G)
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_fluctuation", C.byref(t), _lib.ptr(sel), k, _lib.ptr(frames), n, _lib.ptr(records),
              _lib.ptr(centre), _lib.ptr(groups), G, _lib.ptr(out), ld)
    return out


def frame_moments_device(coords, sel, records=None, frames=None, weights=None, groups=None):
    """(n, G, 6) float64 CUDA (K20): per listed frame and group of selection positions, the weighted mean of the aligned
    float32 coordinate (columns 0-2) and the weighted variance around it per axis (columns 3-5), both over the group's
    weight total.  ``weights`` (k,) float64 (None = all 1) and ``groups`` (G + 1,) int64 offsets over the selection
    positions (None = one group of all k) are small host-side arrays -- a CPU tensor, a numpy array or a list; CUDA
    tensors are copied back.  The library rejects offsets that do not increase strictly from 0 to k and groups whose
    weights do not sum to a finite value > 0.  The bits of a frame's row depend only on the selection, groups and weights,
    so repeated calls, a frame slice and the equivalent explicit frame list agree bit for bit."""
    dev = _lib.tensor_device(coords, "frame_moments_device")
    _lib.index_arg(sel, dev)
    _lib.index_arg(frames, dev)
    k = int(sel.numel())
    n = coords.shape[2] if frames is None else int(frames.numel())
    _check_records(records, n)
    if weights is not None:
        weights = torch.as_tensor(weights, dtype=torch.float64, device="cpu").contiguous()
        assert tuple(weights.shape) == (k,), f"weights must be ({k},), got {tuple(weights.shape)}"
    groups = torch.tensor([0, k]) if groups is None else groups
    groups = torch.as_tensor(groups, dtype=torch.int64, device="cpu").contiguous()
    assert groups.ndim == 1, "groups must be 1-D offsets"
    G = int(groups.numel()) - 1
    out = torch.empty((n, max(G, 0), 6), dtype=torch.float64, device=dev)
    if n == 0:
        return out
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_frame_moments", C.byref(t), _lib.ptr(sel), k, _lib.ptr(frames), n, _lib.ptr(records),
              _lib.ptr(weights), _lib.ptr(groups), G, _lib.ptr(out))
    return out
