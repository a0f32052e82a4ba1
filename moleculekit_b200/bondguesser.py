"""Drop-in for ``moleculekit.bondguesser.guess_bonds`` / ``bond_grid_search`` (SURVEY row a13, K7).

The reference finds bonds with a uniform non-periodic cell grid built in Python (one dict insertion per atom, one
Cython call per occupied box: moleculekit/bondguesser.py:259-392, bondguesser_utils.pyx:30-163).  Here the whole
search runs on the GPU (csrc/bonds.cu).  The returned SET of bonds is identical to the reference's: the pairs that pass
its float32 ``_is_close`` test AND that its float32 box grid compares -- boxes floor((x - xyzmin) / pairdist) at most one
apart on every axis, which two atoms pairdist apart can fail by rounding.  Rows come back
canonical -- (min, max) pairs sorted lexicographically, the order ``calculateUniqueBonds`` produces and the
reference's own test compares in -- rather than in the reference's box-traversal order.
"""
from __future__ import annotations

import logging

import numpy as np
import torch

from . import _lib

logger = logging.getLogger(__name__)

# Bond-perception radii per element (Bondi 1964; H lowered to 1.0; unavailable -> 2.0; ions from CHARMM27), the
# values the reference tabulates at moleculekit/bondguesser.py:16-129.
vdw_radii = {
    "H": 1.0, "He": 1.4, "Li": 1.82, "Be": 2.0, "B": 2.0, "C": 1.7,
    "N": 1.55, "O": 1.52, "F": 1.47, "Ne": 1.54, "Na": 1.36, "Mg": 1.18,
    "Al": 2.0, "Si": 2.1, "P": 1.8, "S": 1.8, "Cl": 2.27, "Ar": 1.88,
    "K": 1.76, "Ca": 1.37, "Sc": 2.0, "Ti": 2.0, "V": 2.0, "Cr": 2.0,
    "Mn": 2.0, "Fe": 2.0, "Co": 2.0, "Ni": 1.63, "Cu": 1.4, "Zn": 1.39,
    "Ga": 1.07, "Ge": 2.0, "As": 1.85, "Se": 1.9, "Br": 1.85, "Kr": 2.02,
    "Rb": 2.0, "Sr": 2.0, "Y": 2.0, "Zr": 2.0, "Nb": 2.0, "Mo": 2.0,
    "Tc": 2.0, "Ru": 2.0, "Rh": 2.0, "Pd": 1.63, "Ag": 1.72, "Cd": 1.58,
    "In": 1.93, "Sn": 2.17, "Sb": 2.0, "Te": 2.06, "I": 1.98, "Xe": 2.16,
    "Cs": 2.1, "Ba": 2.0, "La": 2.0, "Ce": 2.0, "Pr": 2.0, "Nd": 2.0,
    "Pm": 2.0, "Sm": 2.0, "Eu": 2.0, "Gd": 2.0, "Tb": 2.0, "Dy": 2.0,
    "Ho": 2.0, "Er": 2.0, "Tm": 2.0, "Yb": 2.0, "Lu": 2.0, "Hf": 2.0,
    "Ta": 2.0, "W": 2.0, "Re": 2.0, "Os": 2.0, "Ir": 2.0, "Pt": 1.72,
    "Au": 1.66, "Hg": 1.55, "Tl": 1.96, "Pb": 2.02, "Bi": 2.0, "Po": 2.0,
    "At": 2.0, "Rn": 2.0, "Fr": 2.0, "Ra": 2.0, "Ac": 2.0, "Th": 2.0,
    "Pa": 2.0, "U": 1.86, "Np": 2.0, "Pu": 2.0, "Am": 2.0, "Cm": 2.0,
    "Bk": 2.0, "Cf": 2.0, "Es": 2.0, "Fm": 2.0, "Md": 2.0, "No": 2.0,
    "Lr": 2.0, "Rf": 2.0, "Db": 2.0, "Sg": 2.0, "Bh": 2.0, "Hs": 2.0,
    "Mt": 2.0, "Ds": 2.0, "Rg": 2.0,
}

_NAME_DEFAULTS = {"H": 1.0, "C": 1.5, "N": 1.4, "O": 1.3, "F": 1.2, "S": 1.9}


def bond_radii(element, name) -> np.ndarray:
    """float32 radius per atom: element table, else first letter of the atom name, else 1.5 (bondguesser.py:161-172)."""
    out = np.empty(len(element), dtype=np.float32)
    for i, el in enumerate(element):
        r = 1.5
        if el in vdw_radii:
            r = vdw_radii[el]
        else:
            nn = str(name[i])[:1].upper()
            if nn in _NAME_DEFAULTS:
                r = _NAME_DEFAULTS[nn]
        out[i] = r
    return out


def guess_bonds(mol) -> np.ndarray:
    """(nbonds, 2) uint32 bonds guessed from the coordinates of ``mol.frame`` (bondguesser.py:131-187)."""
    if mol.numAtoms <= 1:
        return np.zeros((0, 2), dtype=np.uint32)
    frame = getattr(mol, "frame", 0)
    if frame >= mol.numFrames:
        raise RuntimeError(
            f"Frame {frame} (defined in mol.frame) is out of range. "
            f"Must be less than the number of coordinate frames ({mol.numFrames}) in this molecule."
        )
    coords = mol.coords[:, :, frame].copy()
    radii = bond_radii(mol.element, mol.name)
    is_hydrogen = (np.asarray(mol.element) == "H").astype(np.uint32)
    grid_cutoff = np.max(radii) * 1.2  # grid box edge: 1.2 x the largest radius
    return bond_grid_search(coords, grid_cutoff, is_hydrogen, radii)


def bond_grid_search(coords: np.ndarray, grid_cutoff: float, is_hydrogen: np.ndarray, radii: np.ndarray,
                     max_boxes: float = 4e6, cutoff_incr: float = 1.26, device=None) -> np.ndarray:
    """Bonded atom pairs by uniform-grid neighbour search; same arguments, validation and box-size enlargement rule
    as the reference (bondguesser.py:259-392)."""
    coords = np.asarray(coords)
    if not np.isfinite(coords).all():
        raise ValueError("bond_grid_search received non-finite coordinates (NaN or inf). Coordinates must be finite.")
    if not (grid_cutoff > 0 and np.isfinite(grid_cutoff)):
        raise ValueError(f"bond_grid_search requires a positive, finite grid_cutoff; got {grid_cutoff!r}.")
    n = coords.shape[0]
    if n == 0:
        return np.zeros((0, 2), dtype=np.uint32)
    coords = np.ascontiguousarray(coords, dtype=np.float32)
    xyzrange = coords.max(axis=0) - coords.min(axis=0)

    def n_boxes(pd):
        ax = (np.floor(xyzrange / pd).astype(np.int64) + 1).tolist()
        return ax[0] * ax[1] * ax[2]

    pairdist = float(grid_cutoff)
    while n_boxes(pairdist) > max_boxes:  # unwrapped systems: widen the boxes until the grid is affordable
        pairdist *= cutoff_incr
    if n_boxes(pairdist) > 1e6:
        logger.warning(
            "It seems like you might be guessing bonds on an unwrapped simulation. "
            "This can consume large amounts of memory and possibly crash. If you already have "
            "all the bonds in Molecule pass `guessBonds=False` to the function or perform "
            "the bond guessing on a wrapped frame."
        )
    dev = _lib.device(device)
    d_c = torch.from_numpy(coords).to(dev)
    d_r = torch.from_numpy(np.ascontiguousarray(radii, dtype=np.float32)).to(dev)
    d_h = torch.from_numpy(np.ascontiguousarray(is_hydrogen, dtype=np.uint32).view(np.int32)).to(dev)
    off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    args = (_lib.ptr(d_c), _lib.ptr(d_r), _lib.ptr(d_h), n, float(np.float32(pairdist)))
    (pairs,) = _lib.count_fill(dev, "mkb_bonds_count", "mkb_bonds_fill", args, off,
                               lambda total: (torch.empty((total, 2), dtype=torch.int32, device=dev),))
    if pairs.shape[0] == 0:
        return np.zeros((0, 2), dtype=np.uint32)
    out = pairs.cpu().numpy().view(np.uint32)
    return out[np.lexsort((out[:, 1], out[:, 0]))]  # rows are (i < j); canonical order
