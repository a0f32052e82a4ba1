"""TM-align on the GPU (K27): the sequence-independent structural alignment of Zhang & Skolnick (Nucleic Acids Res.
2005) of every listed frame against a reference, as moleculekit's ``molTMalign`` runs it one frame at a time.

  tmalign_parameters(xlen, ylen)   the search and final-score parameters, on the host with C ``pow``
  max_residues()                   the largest trace either side of one call may have
  tmalign_device                   (tm, rmsd, nali, invmap, records) per listed frame, CUDA tensors, stream-ordered
  molTMalign(mol, ref, ...)        host mirror of molTMalign: numpy (tmscore, rmsd, nali) per listed frame

x is the mol CA trace (xlen residues), y the reference's (ylen).  ``invmap[j]`` is the x residue aligned to y residue
j, or -1.  The contract is ``mkb_tmalign`` in include/mkb200.h.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .align import RECORD
from .tmscore import ca_atoms

N_PARAMS = 10


def _d0(L: float) -> float:
    return 1.24 * math.pow(L - 15, 1.0 / 3.0) - 1.8


def tmalign_parameters(xlen: int, ylen: int) -> np.ndarray:
    """float64 [10]: the search's d0, d0_search, score_d8, D0_MIN, ddcc and dcu0, then d0 and d0_search of the final
    score normalised by ylen, then by xlen."""
    xlen, ylen = int(xlen), int(ylen)
    if min(xlen, ylen) < 5:
        raise ValueError(f"TM-align needs at least 5 residues on each side, got {xlen} and {ylen} (too short)")
    lnorm = min(xlen, ylen)
    d0 = 0.168 if lnorm <= 19 else _d0(lnorm)
    d0_min = d0 + 0.8
    d0 = d0_min
    d0_search = min(8.0, max(4.5, d0))
    score_d8 = 1.5 * math.pow(lnorm, 0.3) + 3.5
    ddcc = 0.1 if lnorm <= 40 else 0.4
    out = [d0, d0_search, score_d8, d0_min, ddcc, 4.25]
    for L in (ylen, xlen):
        f = 0.5 if L <= 21 else max(0.5, _d0(L))
        out += [f, min(8.0, max(4.5, f))]
    return np.asarray(out, np.float64)


def max_residues() -> int:
    """The largest xlen or ylen :func:`tmalign_device` accepts."""
    return int(_lib.load().mkb_tmalign_max_residues())


def chunk_frames(xlen: int, ylen: int) -> int:
    """How many items the library processes per launch for these lengths (its scratch grows with this)."""
    return int(_lib.load().mkb_tmalign_chunk_frames(int(xlen), int(ylen)))


def tmalign_device(coords, sel, refcoords, refsel, frames=None):
    """TM-align of the ``sel`` rows of every listed frame of ``coords`` (N, 3, F) float32 onto the ``refsel`` rows of
    ``refcoords``: (M, 3, 1) one reference, or (M, 3, F) frame k onto reference frame k (``matchingframes``; item k
    uses reference frame frames[k]).  ``sel`` (xlen,) / ``refsel`` (ylen,) / ``frames`` int32 CUDA tensors.

    Returns ``(tm (n, 2) float64, rmsd (n,) float64, nali (n,) int32, invmap (n, ylen) int32, records (n, 16)
    float64)``: tm[:, 0] is normalised by ylen (TM_ref), tm[:, 1] by xlen; records are K14's (x' = R (x - p) + q),
    ready for :func:`moleculekit_b200.align.apply_device`.  A frame with a non-finite selected coordinate gets NaN
    scores and rmsd, nali 0, an all -1 map and the identity record.  ``ValueError`` for fewer than 5 residues either
    side, more than :func:`max_residues`, or a non-finite reference coordinate."""
    dev = _lib.tensor_device(coords, "tmalign_device")
    xlen, ylen = int(sel.numel()), int(refsel.numel())
    params = tmalign_parameters(xlen, ylen)
    cap = max_residues()
    if max(xlen, ylen) > cap:
        raise ValueError(f"TM-align of {xlen} onto {ylen} residues: at most {cap} residues fit one call")
    for x in (sel, refsel, frames):
        _lib.index_arg(x, dev)
    per_frame = refcoords.shape[2] != 1
    rf = refcoords[refsel.long()]
    if per_frame and frames is not None:
        rf = rf[:, :, frames.long()]
    if not bool(torch.isfinite(rf).all()):
        raise ValueError("the reference has non-finite coordinates among the selected residues")
    n = coords.shape[2] if frames is None else int(frames.numel())
    if per_frame and refcoords.shape[2] < coords.shape[2]:
        raise ValueError("matching frames need a reference frame for every frame")
    tm = torch.empty((n, 2), dtype=torch.float64, device=dev)
    rmsd = torch.empty(n, dtype=torch.float64, device=dev)
    nali = torch.empty(n, dtype=torch.int32, device=dev)
    invmap = torch.empty((n, ylen), dtype=torch.int32, device=dev)
    records = torch.empty((n, RECORD), dtype=torch.float64, device=dev)
    if n == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return tm, rmsd, nali, invmap, records
    t, r = _lib.traj(coords), _lib.traj(refcoords)
    _lib.call(dev, "mkb_tmalign", C.byref(t), _lib.ptr(sel), xlen, C.byref(r), _lib.ptr(refsel), ylen, int(per_frame),
              params.ctypes.data_as(C.c_void_p), _lib.ptr(frames), n, _lib.ptr(tm), _lib.ptr(rmsd), _lib.ptr(nali),
              _lib.ptr(invmap), _lib.ptr(records))
    return tm, rmsd, nali, invmap, records


def molTMalign(mol, ref, molsel="protein", refsel="protein", return_alignments=False, frames=None,
               matchingframes=False, device=None):
    """Mirror of moleculekit's ``molTMalign``: TM-align every listed frame of ``mol`` (``frames``: None for all, an
    int, a list, an array or a slice) onto ``ref`` at ``ref.frame`` (or, with ``matchingframes``, onto the same frame
    of ``ref``).  Both selections are reduced to their CA atoms, in atom order.

    Returns numpy ``(tmscore (F,) float64, rmsd (F,) float64, nali (F,) int64)``; ``tmscore`` is normalised by the
    reference's CA count.  With ``return_alignments`` also ``alignments``, per frame an (nali, 2) int64 array of
    (mol CA index, ref CA index) atom pairs of the final map, and ``(rotation (F, 3, 3), translation (F, 3))``, the
    superposition x' = rotation x + translation of the mol onto the reference.  Only the selected CA rows travel to
    the device.

    Not confirmed against moleculekit (its source is not available here): the function's keyword names and defaults,
    the return shape, that ``tmscore`` is the reference-normalised score, the alignment format (atom indices, pairs
    with d <= score_d8 only), and that ``frames`` lists mol frames with ``ref.frame`` fixed unless ``matchingframes``.
    """
    idx = ca_atoms(mol, molsel, "Molecule TM-align")
    ridx = ca_atoms(ref, refsel, "Reference TM-align")
    tmalign_parameters(idx.size, ridx.size)  # argument errors before any device work
    cap = max_residues()
    if max(idx.size, ridx.size) > cap:
        raise ValueError(f"TM-align of {idx.size} onto {ridx.size} CA atoms: at most {cap} residues fit one call")
    F = mol.coords.shape[2]
    if frames is None:
        flist = np.arange(F)
    elif isinstance(frames, slice):
        flist = np.arange(F)[frames]
    else:
        flist = np.atleast_1d(np.asarray(frames, np.int64))
        if flist.size and (flist.min() < -F or flist.max() >= F):
            raise IndexError(f"frame index out of range for {F} frames")
        flist = np.where(flist < 0, flist + F, flist)
    n = flist.size
    dev = _lib.device(device)
    x = torch.from_numpy(np.ascontiguousarray(mol.coords[idx], dtype=np.float32)).to(dev)
    if matchingframes:
        if ref.coords.shape[2] != F:
            raise ValueError(f"matchingframes needs as many reference frames ({ref.coords.shape[2]}) as frames ({F})")
        y = torch.from_numpy(np.ascontiguousarray(ref.coords[ridx], dtype=np.float32)).to(dev)
    else:
        fr = int(getattr(ref, "frame", 0))
        y = torch.from_numpy(np.ascontiguousarray(ref.coords[ridx][:, :, fr:fr + 1], dtype=np.float32)).to(dev)
    fl = None if frames is None else torch.from_numpy(flist.astype(np.int32)).to(dev)
    if n == 0:
        tm = np.zeros((0, 2)); rmsd = np.zeros(0); nali = np.zeros(0, np.int32)
        invmap = np.zeros((0, ridx.size), np.int32); rec = np.zeros((0, RECORD))
    else:
        out = tmalign_device(x, torch.arange(idx.size, dtype=torch.int32, device=dev), y,
                             torch.arange(ridx.size, dtype=torch.int32, device=dev), fl)
        tm, rmsd, nali, invmap, rec = (o.cpu().numpy() for o in out)
    if not return_alignments:
        return tm[:, 0].copy(), rmsd, nali.astype(np.int64)
    alignments = []
    for k in range(n):
        j = np.where(invmap[k] >= 0)[0]
        alignments.append(np.stack([idx[invmap[k][j]], ridx[j]], axis=1).astype(np.int64))
    R = rec[:, :9].reshape(n, 3, 3).copy()
    trans = rec[:, 12:15] - np.einsum("fij,fj->fi", R, rec[:, 9:12])
    return tm[:, 0].copy(), rmsd, nali.astype(np.int64), alignments, (R, trans)
