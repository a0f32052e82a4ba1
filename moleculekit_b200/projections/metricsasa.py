"""Drop-in for ``moleculekit.projections.metricsasa.MetricSasa``: Shrake-Rupley solvent-accessible surface area per
atom or per residue, one row per frame.

``project`` uploads only the ``filtersel`` atoms (compact rows) and computes every (frame, atom) with K17.  ``mol`` is
duck-typed (a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from ..atomselect_utils import as_mask
from .common import column, nonempty, residues
from .projection import Projection


class MetricSasa(Projection):
    """Solvent-accessible surface area in Angstrom^2: ``project`` returns (numFrames, ncols) float32.

    Rules (mdtraj's ``shrake_rupley`` as moleculekit calls it, restated in :func:`moleculekit_b200.sasa.sasa_device`):

    - Only the ``filtersel`` atoms exist for the calculation: they are the atoms that can bury a point.  Coordinates go
      to nm as fl(x / 10); radii are mdtraj's element radii in nm (:data:`moleculekit_b200.sasa.ATOMIC_RADII`) plus
      fl(probeRadius / 10); ``numSpherePoints`` points of the golden-section spiral per atom.
    - ``mode="atom"``: one column per ``sel`` atom, in atom order.  ``mode="residue"``: one column per residue of the
      ``filtersel`` atoms that contains a ``sel`` atom; the column is the float32 sum, in atom order, of the areas of
      every ``filtersel`` atom of the residue.  Residues are runs of consecutive atoms with the same resid, insertion
      code, chain and segid (:func:`moleculekit_b200.projections.common.residues`).
    - Every value is bit-identical to the reference's float32 arithmetic: the area is a count of accessible points.
    - No wrapping and no minimum image.  An atom with a non-finite coordinate takes part in no neighbour relation: its
      own area is that of the full sphere, and it buries no point of another atom.
    - ``getMapping``: one row per column, ``type`` "SASA", ``atomIndexes`` the atom (atom mode) or the residue's
      ``filtersel`` atoms, ``description`` "SASA of {resname} {resid} {name}" or "SASA of residue {resname} {resid}".

    Divergences from the reference: where mdtraj ends the process on two atoms closer than 1e-5 nm, ``project`` raises
    ``ValueError`` naming the first frame and atom pair (the check covers the pairs that contain an atom whose area is
    computed); an element missing from the radius table raises ``ValueError`` listing the elements; a ``sel`` atom
    outside ``filtersel`` raises ``ValueError``; an empty ``sel`` raises ``RuntimeError``.

    Not confirmed against a moleculekit or mdtraj checkout: the nm round trip and the final multiplication by 100, the
    summation order of the squared distance (SSE ``dpps``), the float32 / float64 promotions of the sphere-point
    generator, the radius table beyond Bondi's H, C, N, O, F, P and S, the residue rule and the mapping text.
    """

    def __init__(self, sel="protein", probeRadius=1.4, numSpherePoints=960, mode="atom", filtersel="all"):
        super().__init__()
        if mode not in ("atom", "residue"):
            raise ValueError(f"mode must be 'atom' or 'residue', got {mode!r}")
        from ..sasa import sphere_points

        self._sel, self._filtersel, self._mode = sel, filtersel, mode
        self._probe = float(probeRadius)
        self._sphere = sphere_points(numSpherePoints)
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        """``sasa``: (env atom indices, radii, query positions in env, group offsets or None, column atom lists)."""
        from ..sasa import sasa_radii

        props = ("sasa",) if props == "all" else props
        res = {}
        if "sasa" not in props:
            return res
        sel = nonempty(mol, self._sel, "Atom")
        filt = as_mask(mol.atomselect(self._filtersel), mol.numAtoms)
        if (sel & ~filt).any():
            raise ValueError(f"{int((sel & ~filt).sum())} sel atom(s) lie outside filtersel; their area is undefined")
        env = np.where(filt)[0]
        radii = sasa_radii(column(mol, "element", "")[env], self._probe)
        pos = np.full(mol.numAtoms, -1, np.int64)
        pos[env] = np.arange(env.size)
        if self._mode == "atom":
            cols = [np.array([a]) for a in np.where(sel)[0]]
            query, groups = pos[np.where(sel)[0]], None
        else:
            cols = [r for r in residues(mol, filt) if sel[r].any()]
            query = pos[np.concatenate(cols)]
            groups = np.concatenate([[0], np.cumsum([len(r) for r in cols])]).astype(np.int64)
        res["sasa"] = (env, radii, query, groups, cols)
        return res

    def project(self, mol) -> np.ndarray:
        """(numFrames, ncols) float32 areas in Angstrom^2."""
        import torch

        from .. import _lib
        from ..sasa import CoincidentAtomsError, sasa_device

        env, radii, query, groups, cols = self._getMolProp(mol, "sasa")
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros((0, len(cols)), np.float32)
        dev = _lib.device(self.device)

        def up(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)

        d = up(mol.coords[env], np.float32)
        try:
            out = sasa_device(d, up(np.arange(env.size), np.int32), up(radii, np.float32), up(query, np.int32),
                              up(self._sphere, np.float32), None if groups is None else up(groups, np.int64))
        except CoincidentAtomsError as e:
            raise CoincidentAtomsError(e.frame, (env[e.atoms[0]], env[e.atoms[1]])) from None
        return out.cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        _, _, _, _, cols = self._getMolProp(mol, "sasa")
        resname, resid, name = column(mol, "resname", ""), column(mol, "resid", 0), column(mol, "name", "")
        if self._mode == "atom":
            desc = [f"SASA of {resname[c[0]]} {resid[c[0]]} {name[c[0]]}" for c in cols]
        else:
            desc = [f"SASA of residue {resname[c[0]]} {resid[c[0]]}" for c in cols]
        return DataFrame({"type": ["SASA"] * len(cols), "atomIndexes": [c.copy() for c in cols], "description": desc})
