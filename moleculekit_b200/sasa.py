"""Solvent-accessible surface area on the GPU (K17), the Shrake-Rupley algorithm of mdtraj's ``shrake_rupley``.

  sphere_points     (n, 3) float32 golden-section spiral of mdtraj's ``generate_sphere_points``
  ATOMIC_RADII      element radii in nm of mdtraj's SASA (``mdtraj.geometry.sasa._ATOMIC_RADII``)
  sasa_radii        float32 radius plus probe in nm per element, as the reference passes them
  sasa_device       (n, m) float32 areas in Angstrom^2 per listed frame, per query atom or per group of query atoms

CUDA tensors in, stream-ordered, like :func:`moleculekit_b200.dihedral.dihedrals_device`.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .coords import _rows

MAX_SPHERE_POINTS = 65536

# mdtraj/geometry/sasa.py _ATOMIC_RADII (nm).  H 0.120, C 0.170, N 0.155, O 0.152, F 0.147, P 0.180 and S 0.180 are
# Bondi's van der Waals radii; the other entries restate mdtraj's table and are not confirmed against a checkout.
ATOMIC_RADII = {
    "H": 0.120, "He": 0.140, "Li": 0.076, "Be": 0.059, "B": 0.192, "C": 0.170, "N": 0.155, "O": 0.152, "F": 0.147,
    "Ne": 0.154, "Na": 0.102, "Mg": 0.086, "Al": 0.184, "Si": 0.210, "P": 0.180, "S": 0.180, "Cl": 0.181, "Ar": 0.188,
    "K": 0.138, "Ca": 0.114, "Sc": 0.211, "Ti": 0.200, "V": 0.200, "Cr": 0.200, "Mn": 0.200, "Fe": 0.200, "Co": 0.200,
    "Ni": 0.163, "Cu": 0.140, "Zn": 0.139, "Ga": 0.187, "Ge": 0.211, "As": 0.185, "Se": 0.190, "Br": 0.185,
    "Kr": 0.202, "Rb": 0.303, "Sr": 0.249, "Y": 0.200, "Zr": 0.200, "Nb": 0.200, "Mo": 0.200, "Tc": 0.200,
    "Ru": 0.200, "Rh": 0.200, "Pd": 0.163, "Ag": 0.172, "Cd": 0.158, "In": 0.193, "Sn": 0.217, "Sb": 0.206,
    "Te": 0.206, "I": 0.198, "Xe": 0.216, "Cs": 0.167, "Ba": 0.149, "La": 0.200, "Ce": 0.200, "Pr": 0.200,
    "Nd": 0.200, "Pm": 0.200, "Sm": 0.200, "Eu": 0.200, "Gd": 0.200, "Tb": 0.200, "Dy": 0.200, "Ho": 0.200,
    "Er": 0.200, "Tm": 0.200, "Yb": 0.200, "Lu": 0.200, "Hf": 0.200, "Ta": 0.200, "W": 0.200, "Re": 0.200,
    "Os": 0.200, "Ir": 0.200, "Pt": 0.175, "Au": 0.166, "Hg": 0.155, "Tl": 0.196, "Pb": 0.202, "Bi": 0.207,
    "Po": 0.197, "At": 0.202, "Rn": 0.220, "Fr": 0.348, "Ra": 0.283, "Ac": 0.200, "Th": 0.200, "Pa": 0.200,
    "U": 0.186, "Np": 0.200, "Pu": 0.200, "Am": 0.200, "Cm": 0.200, "Bk": 0.200, "Cf": 0.200, "Es": 0.200,
    "Fm": 0.200, "Md": 0.200, "No": 0.200, "Lr": 0.200,
}


class CoincidentAtomsError(ValueError):
    """Two atoms closer than 1e-5 nm in some frame (the reference stops the process there).  ``frame`` is the frame
    index of the trajectory; ``atoms`` the two atom rows of the trajectory, the first one a query atom."""

    def __init__(self, frame, atoms):
        self.frame, self.atoms = int(frame), (int(atoms[0]), int(atoms[1]))
        super().__init__(f"atoms {self.atoms[0]} and {self.atoms[1]} coincide in frame {self.frame} (distance below "
                         "1e-5 nm): the Shrake-Rupley area is undefined there")


def sphere_points(n: int) -> np.ndarray:
    """(n, 3) float32 points of mdtraj's generate_sphere_points with its C promotions: inc = fl(pi (3 - sqrt 5)) and
    offset = fl(2 / n) are float32; y = fl((double)fl(j offset) - 1.0 + offset / 2.0); r = fl(sqrt(1.0 - fl(y y)));
    phi = fl(j inc); the point is (fl(cos(phi) r), y, fl(sin(phi) r)) with cos / sin / sqrt in float64."""
    n = int(n)
    if n < 1 or n > MAX_SPHERE_POINTS:
        raise ValueError(f"numSpherePoints must be in [1, {MAX_SPHERE_POINTS}], got {n}")
    f32 = np.float32
    inc = f32(np.pi * (3.0 - np.sqrt(5.0)))
    offset = f32(2) / f32(n)
    j = np.arange(n, dtype=np.float32)
    y = ((j * offset).astype(np.float64) - 1.0 + np.float64(offset) / 2.0).astype(np.float32)
    r = np.sqrt(1.0 - (y * y).astype(np.float64)).astype(np.float32)
    phi = (j * inc).astype(np.float64)
    out = np.empty((n, 3), np.float32)
    out[:, 0] = (np.cos(phi) * r.astype(np.float64)).astype(np.float32)
    out[:, 1] = y
    out[:, 2] = (np.sin(phi) * r.astype(np.float64)).astype(np.float32)
    return out


def _symbol(e) -> str:
    s = str(e).strip()
    return s[:1].upper() + s[1:].lower()


def sasa_radii(elements, probe: float) -> np.ndarray:
    """float32 R = fl(rad_nm[element] + fl(probe / 10)) per atom, ``probe`` in Angstrom.  Raises ValueError listing
    the elements missing from :data:`ATOMIC_RADII`."""
    sym = [_symbol(e) for e in elements]
    missing = sorted({s for s in sym if s not in ATOMIC_RADII})
    if missing:
        raise ValueError(f"no SASA radius for element(s) {missing}")
    rad = np.array([ATOMIC_RADII[s] for s in sym], dtype=np.float32)
    return rad + np.float32(float(probe) / 10.0)


def chunk_frames(n_env: int, n_query: int, n_groups: int = 0) -> int:
    """Listed frames per chunk of one :func:`sasa_device` call (its scratch stays bounded whatever the frame count)."""
    return int(_lib.load().mkb_sasa_chunk_frames(int(n_env), int(n_query), int(n_groups)))


def sasa_device(coords, env, radii, query, sphere, groups=None, frames=None, out=None):
    """Shrake-Rupley areas in Angstrom^2 (see mkb_sasa in include/mkb200.h for the arithmetic).

    ``coords`` (N, 3, F) float32 frame-minor in Angstrom; ``env`` int32 atom rows of ``coords`` that can bury a point;
    ``radii`` float32 radius plus probe in nm per ``env`` atom; ``query`` int32 positions in ``env`` of the atoms whose
    area is computed; ``sphere`` (n, 3) float32 unit points (:func:`sphere_points`).  ``groups`` (optional) int64
    offsets into ``query``: column g is then the float32 sum, in order, of the areas of query[groups[g]:groups[g+1]].
    ``frames`` int32 (None = every frame).  ``out`` (optional) receives the rows (unit column stride, any row stride).
    Raises :class:`CoincidentAtomsError` when a query atom coincides with another ``env`` atom."""
    dev = _lib.tensor_device(coords, "sasa_device")
    _lib.index_arg(env, dev)
    _lib.index_arg(query, dev)
    _lib.index_arg(groups, dev, torch.int64)
    _lib.index_arg(frames, dev)
    for t in (radii, sphere):
        assert t.dtype == torch.float32 and t.device == dev and t.is_contiguous()
    assert radii.shape == env.shape and sphere.ndim == 2 and sphere.shape[1] == 3
    cols = int(query.numel()) if groups is None else int(groups.numel()) - 1
    n = coords.shape[2] if frames is None else int(frames.numel())
    out = _rows(out, n, cols, torch.float32, dev)
    if n == 0:  # an empty frame list has a NULL data pointer, which the library reads as "every frame"
        return out
    ld = max(out.stride(0) if n > 1 else cols, cols)
    status = torch.empty(1, dtype=torch.int64, device=dev)
    t = _lib.traj(coords)
    _lib.call(dev, "mkb_sasa", C.byref(t), _lib.ptr(env), int(env.numel()), _lib.ptr(radii), _lib.ptr(query),
              int(query.numel()), _lib.ptr(groups), max(cols, 0) if groups is not None else 0, _lib.ptr(sphere),
              int(sphere.shape[0]), _lib.ptr(frames), n, _lib.ptr(out), ld, _lib.ptr(status))
    key = int(status.item())
    if key != -1:
        _raise_coincident(coords, env, query, frames, key)
    return out


def _raise_coincident(coords, env, query, frames, key):
    """The partner of the reported (item, query) pair: the first env atom within 1e-10 nm^2, found on the host with the
    kernel's float32 arithmetic."""
    k, q = key >> 32, key & 0xFFFFFFFF
    f = int(frames[k].item()) if frames is not None else k
    rows = env.long()
    x = (coords[rows, :, f].cpu().numpy() / np.float32(10)).astype(np.float32)
    i = int(query[q].item())
    d = x[i] - x
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    d2[i] = np.inf
    j = int(np.argmax(d2 < np.float32(1e-10)))
    raise CoincidentAtomsError(f, (int(rows[i]), int(rows[j])))
