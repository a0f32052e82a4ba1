"""TM-score on the GPU (K19): the superposition search of the TMscore program (Zhang & Skolnick, Proteins 2004) that
moleculekit's ``molTMscore`` runs once per frame.

  tm_parameters(L, Lnorm)      d0, d0_search and the seed fragment lengths, on the host with C ``pow``
  ca_atoms(mol, sel, what)     the atoms named CA of a selection, in atom order
  tmscore_device               (tm, rmsd) float64 per listed frame, CUDA tensors in and out, stream-ordered
  molTMscore(mol, ref, ...)    host mirror of molTMscore: numpy (tmscore, rmsd, nali) per frame

Pair k joins the k-th CA of the trajectory selection and the k-th CA of the reference selection, for k < L = min(n, m);
the score is normalised by m, the reference's CA count.  The contract is ``mkb_tmscore`` in include/mkb200.h.  No CPU
fallback.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .atomselect_utils import as_mask


def tm_parameters(L: int, lnorm: int):
    """(d0, d0_search, fragment lengths) of the search over L pairs normalised by ``lnorm``."""
    if L < 1 or lnorm < 1:
        raise ValueError(f"TM-score needs at least one pair and a normaliser >= 1, got L={L}, Lnorm={lnorm}")
    d0 = 0.5 if lnorm <= 15 else max(0.5, 1.24 * math.pow(lnorm - 15, 1.0 / 3.0) - 1.8)
    d0_search = min(8.0, max(4.5, d0))
    lmin = min(4, L)
    frag = []
    for i in range(5):
        v = L // 2 ** i
        if v <= lmin:
            frag.append(lmin)
            break
        frag.append(v)
    else:
        frag.append(lmin)
    return d0, d0_search, tuple(frag)


def max_pairs() -> int:
    """The largest L one :func:`tmscore_device` call accepts (the pairs live in shared memory)."""
    return int(_lib.load().mkb_tmscore_max_pairs())


def ca_atoms(mol, sel, what: str) -> np.ndarray:
    """int64 indices of the atoms of ``sel`` named CA, ascending; RuntimeError when there are none."""
    mask = as_mask(mol.atomselect(sel), mol.numAtoms)
    idx = np.where(mask & (np.asarray(mol.name).astype(str) == "CA"))[0]
    if idx.size == 0:
        raise RuntimeError(f"{what} selection resulted in 0 CA atoms.")
    return idx


def tmscore_device(coords, sel, refcoords, refsel, frames=None):
    """TM-score and RMSD of every listed frame of ``coords`` (N, 3, F) float32 against frame 0 of ``refcoords``
    (M, 3, 1).  ``sel`` (n,) and ``refsel`` (m,) int32 CUDA tensors are the paired atoms in pairing order: L = min(n, m)
    pairs, normalised by m.  ``frames`` int32 (None = every frame).  Returns (tm (len,) float64, rmsd (len,) float64);
    a frame with a non-finite paired coordinate gets NaN for both."""
    dev = _lib.tensor_device(coords, "tmscore_device")
    n, m = int(sel.numel()), int(refsel.numel())
    if n == 0 or m == 0:
        raise RuntimeError(f"TM-score selections resulted in {n} and {m} atoms.")
    L = min(n, m)
    cap = max_pairs()
    if L > cap:
        raise ValueError(f"TM-score over {L} pairs: at most {cap} pairs fit one call")
    for x in (sel, refsel, frames):
        _lib.index_arg(x, dev)
    if not bool(torch.isfinite(refcoords[refsel[:L].long(), :, 0]).all()):
        raise ValueError("the reference has non-finite coordinates among the paired atoms")
    d0, d0s, frag = tm_parameters(L, m)
    frag = np.asarray(frag, np.int32)
    cnt = coords.shape[2] if frames is None else int(frames.numel())
    tm = torch.empty(cnt, dtype=torch.float64, device=dev)
    rmsd = torch.empty(cnt, dtype=torch.float64, device=dev)
    if cnt == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return tm, rmsd
    t, r = _lib.traj(coords), _lib.traj(refcoords)
    _lib.call(dev, "mkb_tmscore", C.byref(t), _lib.ptr(sel), C.byref(r), _lib.ptr(refsel), L, m, d0, d0s,
              frag.ctypes.data_as(C.c_void_p), int(frag.size), _lib.ptr(frames), cnt, _lib.ptr(tm), _lib.ptr(rmsd))
    return tm, rmsd


def molTMscore(mol, ref, selCAmol, selCAref, device=None):
    """Mirror of molTMscore: per frame of ``mol`` the TM-score against ``ref`` at ``ref.frame``, the RMSD under the
    all-pairs fit and the number of aligned pairs.  Both selections are reduced to their CA atoms.  Returns numpy
    (tmscore (F,) float64, rmsd (F,) float64, nali (F,) int64).  Only the paired rows travel to the device."""
    idx = ca_atoms(mol, selCAmol, "Trajectory TM-score")
    ridx = ca_atoms(ref, selCAref, "Reference TM-score")
    L = min(idx.size, ridx.size)
    F = mol.coords.shape[2]
    if F == 0:
        return np.zeros(0), np.zeros(0), np.zeros(0, np.int64)
    dev = _lib.device(device)
    x = torch.from_numpy(np.ascontiguousarray(mol.coords[idx[:L]], dtype=np.float32)).to(dev)
    fr = int(getattr(ref, "frame", 0))
    y = torch.from_numpy(np.ascontiguousarray(ref.coords[ridx][:, :, fr:fr + 1], dtype=np.float32)).to(dev)
    tm, rmsd = tmscore_device(x, torch.arange(L, dtype=torch.int32, device=dev), y,
                              torch.arange(ridx.size, dtype=torch.int32, device=dev))
    return tm.cpu().numpy(), rmsd.cpu().numpy(), np.full(F, L, np.int64)
