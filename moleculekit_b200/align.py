"""Trajectory superposition on the GPU (K14): Molecule.align and molRMSD.

Mirrors the reference's alignment (moleculekit/align.py, called by Molecule.align) and molRMSD
(moleculekit/projections/metricrmsd.py):

  superpose_device / apply_device / rmsd_device    CUDA tensors, stream-ordered (mkb_align_fit / _apply / mkb_rmsd)
  align(mol, sel, refmol, refsel, frames, matchingframes, mode)    Molecule.align, ``mol.coords`` updated in place
  molRMSD(mol, refmol, rmsdsel1, rmsdsel2)                          per-frame RMSD without fitting

The reference fits every frame with a float32 SVD in a Python loop; here every frame is fitted in float64 on the device
(Kabsch through Horn's quaternion form, csrc/align.cu) and the coordinates are rounded to float32 once: within 1 float32
ulp of the float64 superposition, where the reference's own float32 path is several ulp away from it.  Deliberate
differences: the reference frame is read before any frame moves (the reference, with ``refmol is mol``, first aligns the
reference frame onto itself); a non-finite selected coordinate raises ``numpy.linalg.LinAlgError`` before anything is
written (the reference raises from its SVD with the earlier frames already moved); empty selections and repeated frame
indices raise ``ValueError``.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

RECORD = 16  # doubles per frame record: R (row-major, x' = R (x - p) + q), p_bar, q_bar, pad


# ---------------------------------------------------------------------------------------------- device level
def superpose_device(coords, sel, refcoords, refsel, frames=None):
    """Fit the ``sel`` atoms of every listed frame of ``coords`` (N, 3, F) onto the ``refsel`` atoms of ``refcoords``
    (M, 3, 1): one reference frame, or (M, 3, F): frame f onto reference frame f.  ``sel`` / ``refsel`` / ``frames``
    are int32 CUDA tensors (``frames`` None = all frames).  Returns (records (n, 16) float64, status (n,) int32); row k
    belongs to frame ``frames[k]``; status 1 = non-finite coordinates in the selection."""
    dev = _lib.tensor_device(coords, "superpose_device")
    for x in (sel, refsel, frames):
        _lib.index_arg(x, dev)
    if int(sel.numel()) != int(refsel.numel()):
        raise ValueError(f"selections differ in size: {int(sel.numel())} and {int(refsel.numel())}")
    n = coords.shape[2] if frames is None else int(frames.numel())
    records = torch.empty((n, RECORD), dtype=torch.float64, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    t, r = _lib.traj(coords), _lib.traj(refcoords)
    _lib.call(dev, "mkb_align_fit", C.byref(t), _lib.ptr(sel), C.byref(r), _lib.ptr(refsel), int(sel.numel()),
              _lib.ptr(frames), n, _lib.ptr(records), _lib.ptr(status))
    return records, status


def apply_device(coords, records, frames=None, status=None):
    """Superpose the listed frames of ``coords`` IN PLACE with the records of :func:`superpose_device` (frames whose
    ``status`` is not 0 are left as they are) and return ``coords``."""
    dev = _lib.tensor_device(coords, "apply_device")
    _lib.index_arg(frames, dev)
    n = coords.shape[2] if frames is None else int(frames.numel())
    assert records.dtype == torch.float64 and tuple(records.shape) == (n, RECORD) and records.is_contiguous()
    t = _lib.traj(coords, writable=True)
    _lib.call(dev, "mkb_align_apply", C.byref(t), _lib.ptr(frames), n, _lib.ptr(records), _lib.ptr(status))
    return coords


def rmsd_device(coords, sel, refcoords, refsel, records=None, frames=None):
    """Per listed frame, sqrt(mean |T(x) - q|^2) over the selections as float32 (n,); T = the frame's fit record, or
    no transform when ``records`` is None.  The trajectory is not modified."""
    dev = _lib.tensor_device(coords, "rmsd_device")
    for x in (sel, refsel, frames):
        _lib.index_arg(x, dev)
    if int(sel.numel()) != int(refsel.numel()):
        raise ValueError(f"selections differ in size: {int(sel.numel())} and {int(refsel.numel())}")
    n = coords.shape[2] if frames is None else int(frames.numel())
    if records is not None:
        assert records.dtype == torch.float64 and tuple(records.shape) == (n, RECORD) and records.is_contiguous()
    out = torch.empty(n, dtype=torch.float32, device=dev)
    t, r = _lib.traj(coords), _lib.traj(refcoords)
    _lib.call(dev, "mkb_rmsd", C.byref(t), _lib.ptr(sel), C.byref(r), _lib.ptr(refsel), int(sel.numel()),
              _lib.ptr(frames), n, _lib.ptr(records), _lib.ptr(out))
    return out


def raise_if_nonfinite(status, frames) -> None:
    """The reference's SVD raises LinAlgError on a non-finite covariance; ``status`` is the fit's (synchronises)."""
    bad = status.cpu().numpy() != 0
    if bad.any():
        raise np.linalg.LinAlgError(
            f"SVD did not converge: non-finite coordinates in the alignment selection of frame(s) "
            f"{np.asarray(frames)[bad][:8].tolist()}")


# ------------------------------------------------------------------------------------------------ host mirrors
def _indices(mol, sel) -> np.ndarray:
    mask = np.asarray(mol.atomselect(sel))
    idx = np.where(mask)[0] if mask.dtype == bool else mask.astype(np.int64)
    return idx.astype(np.int32)


def _frame_list(frames, F: int) -> np.ndarray:
    fl = np.asarray(frames).ravel()
    if fl.size == 0:
        return fl.astype(np.int64)
    if not np.issubdtype(fl.dtype, np.integer):
        raise ValueError("frames must be integer frame indices")
    fl = fl.astype(np.int64)
    if fl.min() < -F or fl.max() >= F:
        raise IndexError(f"frame index out of range for {F} frames")
    fl = np.where(fl < 0, fl + F, fl)
    if np.unique(fl).size != fl.size:
        raise ValueError("frames lists a frame more than once")
    return fl


def align(mol, sel, refmol=None, refsel=None, frames=None, matchingframes=False, mode="index", device=None):
    """Mirror of Molecule.align: superpose the ``sel`` atoms of every listed frame of ``mol`` onto the ``refsel`` atoms of
    ``refmol`` (default ``mol``, ``refsel`` default ``sel``) at ``refmol.frame``, or frame by frame with
    ``matchingframes``; ``mol.coords`` is updated in place, frames not listed stay byte-identical."""
    if mode == "structure":
        raise NotImplementedError("mode='structure' (TM-align residue matching) is not supported; use mode='index'")
    if mode != "index":
        raise ValueError(f"Invalid alignment mode {mode!r}: 'index' or 'structure'")
    if refmol is None:
        refmol = mol
    if refsel is None:
        refsel = sel
    F = mol.coords.shape[2]
    if matchingframes and F != refmol.coords.shape[2]:
        raise RuntimeError("This is only supported when both molecules have equal number of frames.")
    idx, ridx = _indices(mol, sel), _indices(refmol, refsel)
    if idx.size != ridx.size:
        raise RuntimeError(
            f"Cannot align molecules. The two selections produced different number of atoms ({idx.size} and "
            f"{ridx.size}). Either fix the selections or use mode='structure'")
    if idx.size == 0:
        raise ValueError("the alignment selection is empty")
    fl = None if frames is None else _frame_list(frames, F)
    if F == 0 or (fl is not None and fl.size == 0):
        return
    dev = _lib.device(device)
    d = torch.from_numpy(np.ascontiguousarray(mol.coords, dtype=np.float32)).to(dev)
    if refmol is mol:
        ref = d if matchingframes else d[:, :, int(mol.frame):int(mol.frame) + 1]
    else:
        rc = refmol.coords if matchingframes else refmol.coords[:, :, int(refmol.frame):int(refmol.frame) + 1]
        ref = torch.from_numpy(np.ascontiguousarray(rc, dtype=np.float32)).to(dev)
    d_sel = torch.from_numpy(idx).to(dev)
    d_ref = torch.from_numpy(ridx).to(dev)
    d_frames = None if fl is None else torch.from_numpy(fl.astype(np.int32)).to(dev)
    records, status = superpose_device(d, d_sel, ref, d_ref, d_frames)
    raise_if_nonfinite(status, np.arange(F) if fl is None else fl)
    apply_device(d, records, d_frames)
    mol.coords[...] = d.cpu().numpy()


def molRMSD(mol, refmol, rmsdsel1, rmsdsel2, device=None):
    """Mirror of molRMSD: per frame sqrt(mean |x - q|^2) between the ``rmsdsel1`` atoms of ``mol`` and the ``rmsdsel2``
    atoms of ``refmol`` (1 frame, or as many frames as ``mol``), float32, squeezed like numpy.  Only the selected rows
    travel to the device."""
    i1 = np.where(np.asarray(rmsdsel1))[0] if np.asarray(rmsdsel1).dtype == bool else np.asarray(rmsdsel1).ravel()
    i2 = np.where(np.asarray(rmsdsel2))[0] if np.asarray(rmsdsel2).dtype == bool else np.asarray(rmsdsel2).ravel()
    if i1.size != i2.size:
        raise ValueError(f"RMSD selections differ in size: {i1.size} and {i2.size}")
    if i1.size == 0:
        raise ValueError("the RMSD selection is empty")
    F, Fr = mol.coords.shape[2], refmol.coords.shape[2]
    if Fr not in (1, F):
        raise ValueError(f"the reference has {Fr} frames: 1 or the molecule's {F}")
    if F == 0:
        return np.zeros(0, np.float32)
    dev = _lib.device(device)
    x = torch.from_numpy(np.ascontiguousarray(mol.coords[i1], dtype=np.float32)).to(dev)
    q = torch.from_numpy(np.ascontiguousarray(refmol.coords[i2], dtype=np.float32)).to(dev)
    ar = torch.arange(i1.size, dtype=torch.int32, device=dev)
    return np.squeeze(rmsd_device(x, ar, q, ar).cpu().numpy())
