"""Drop-in for ``moleculekit.projections.metricfluctuation.MetricFluctuation``: per-atom (or per-residue) squared
deviation of every frame from the mean structure or from a reference -- what an RMSF is computed from.

``project`` runs the shared pipeline of ``common`` (one upload, wrap, fit) and then, without a reference, the frame
sums of the selection (K15, a fixed-order float64 reduction) for the mean, and the squared deviations straight from the
trajectory (K15): the (numFrames, 3n) coordinate matrix is never materialised, and only the result comes back.
Frames are not independent without a reference (the mean spans all of them): shard such a projection with
:func:`moleculekit_b200.sharding.fluctuation_sharded`, not ``project_sharded``.
"""
from __future__ import annotations

import numpy as np

from .common import check_sizes, fit, nonempty, reference, selections, upload_wrapped
from .projection import Projection


def residue_groups(resid):
    """(order, offsets, residues) for the resids of a selection in selection order: ``order`` stably sorts the
    selection by resid, group g is ``order[offsets[g]:offsets[g + 1]]`` and holds the atoms of ``residues[g]`` (the
    distinct resids, ascending)."""
    resid = np.asarray(resid)
    order = np.argsort(resid, kind="stable")
    residues, starts = np.unique(resid[order], return_index=True)
    return order, np.append(starts, resid.size).astype(np.int64), residues


class MetricFluctuation(Projection):
    """Squared deviation of the ``atomsel`` atoms from the mean over the projected frames (no ``refmol``) or from the
    same selection of ``refmol`` at ``refmol.frame``.

    Rules (the reference's documented API):

    - Without ``refmol`` nothing is superposed and the centre is the mean over the projected frames of the (wrapped)
      coordinates.  With ``refmol`` every frame is first superposed onto it: the ``trajalnstr`` atoms onto the
      ``refalnstr`` atoms (default ``trajalnstr``), and the centre is ``atomsel`` applied to ``refmol`` at
      ``refmol.frame``; the two ``atomsel`` selections must have the same size, else ``RuntimeError``.
    - With ``pbc`` the trajectory is first wrapped around ``centerstr`` exactly as Molecule.wrap (and MetricRmsd) does.
    - ``mode="atom"``: (numFrames, n) float32, ``sum_d (c_d - m_d)^2`` per selected atom in atom order (c the aligned
      float32 coordinate, the sum in float64, rounded once).  ``mode="residue"``: (numFrames, R) float32, the float64
      mean of that over each residue's selected atoms; residues are the distinct ``resid`` values of the selection in
      ascending order.  Any other mode raises ``ValueError``.
    - ``getMapping``: one row per atom (``atomIndexes`` the atom, "Fluctuation of {resname} {resid} {name}") or per
      residue (``atomIndexes`` the residue's selected atoms, "Fluctuation of residue {resname} {resid}"), ``type``
      "fluctuation".
    - A non-finite coordinate in the alignment selection raises ``numpy.linalg.LinAlgError``; empty selections raise
      ``RuntimeError`` ("... selection resulted in 0 atoms.").  ``mol`` is not modified.
    """

    def __init__(self, atomsel, refmol=None, trajalnstr="protein and name CA", refalnstr=None, centerstr="protein",
                 pbc=True, mode="atom"):
        super().__init__()
        if mode not in ("atom", "residue"):
            raise ValueError(f"mode must be 'atom' or 'residue', not {mode!r}")
        if refalnstr is None:
            refalnstr = trajalnstr
        self._refmol = self._refcoords = self._refalnsel = self._refatomsel = None
        if refmol is not None:
            self._refmol, self._refcoords = reference(refmol)
            self._refalnsel = nonempty(self._refmol, refalnstr, "Reference alignment")
            self._refatomsel = nonempty(self._refmol, atomsel, "Reference atom")
        self._atomsel, self._trajalnsel, self._centersel = atomsel, trajalnstr, centerstr
        self._pbc = pbc
        self._mode = mode
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        return selections(mol, props, (("atomsel", self._atomsel, "Atom", True),
                                       ("trajalnsel", self._trajalnsel, "Alignment", self._refmol is not None),
                                       ("centersel", self._centersel, "Centering", self._pbc)))

    def _layout(self, mol):
        """(selected atoms in output order (int64), group offsets or None): residue mode orders the selection by resid."""
        idx = np.where(self._getMolProp(mol, "atomsel"))[0]
        if self._mode == "atom":
            return idx, None
        order, offsets, _ = residue_groups(np.asarray(mol.resid)[idx])
        return idx[order], offsets

    def reference_centre(self, mol):
        """(n, 3) float64: the reference's ``atomsel`` atoms in the output order of :meth:`_layout` (None without one)."""
        if self._refmol is None:
            return None
        atomsel = self._getMolProp(mol, "atomsel")
        check_sizes("atom", atomsel, self._refatomsel)
        idx = np.where(atomsel)[0]
        rc = self._refcoords[np.where(self._refatomsel)[0], :, 0].astype(np.float64)
        if self._mode == "residue":
            rc = rc[residue_groups(np.asarray(mol.resid)[idx])[0]]
        return np.ascontiguousarray(rc)

    def _device(self, mol):
        """(the wrapped trajectory on the device, fit records or None, selection, group offsets) -- all checks first"""
        import torch

        props = self._getMolProp(mol, "all")
        if self._refmol is not None:
            check_sizes("alignment", props["trajalnsel"], self._refalnsel)
            self.reference_centre(mol)
        sel, offsets = self._layout(mol)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        records = None if self._refmol is None else fit(d, props["trajalnsel"], self._refcoords, self._refalnsel)
        d_sel = torch.from_numpy(sel.astype(np.int32)).to(d.device)
        d_off = None if offsets is None else torch.from_numpy(offsets).to(d.device)
        return d, records, d_sel, d_off

    def _n_out(self, mol):
        sel, offsets = self._layout(mol)
        return sel.size if offsets is None else offsets.size - 1

    def frame_sums(self, mol) -> np.ndarray:
        """(n, 3) float64 sums over the frames of ``mol`` of the wrapped (and, with a reference, aligned) float32
        coordinates, in the output order of the selection; the mean is this over numFrames."""
        from ..coords import coord_sums_device

        if mol.coords.shape[2] == 0:
            return np.zeros((self._layout(mol)[0].size, 3))
        d, records, d_sel, _ = self._device(mol)
        return coord_sums_device(d, d_sel, records).cpu().numpy()

    def deviations(self, mol, centre) -> np.ndarray:
        """:meth:`project` with the centre given: ``centre`` (n, 3) float64 in the output order of the selection."""
        import torch

        from ..coords import fluctuation_device

        if mol.coords.shape[2] == 0:
            return np.zeros((0, self._n_out(mol)), np.float32)
        d, records, d_sel, d_off = self._device(mol)
        c = torch.from_numpy(np.ascontiguousarray(centre, dtype=np.float64)).to(d.device)
        return fluctuation_device(d, d_sel, c, records, groups=d_off).cpu().numpy()

    def project(self, mol) -> np.ndarray:
        """(numFrames, n atoms or R residues) float32 squared deviations."""
        import torch

        from ..coords import coord_sums_device, fluctuation_device

        F = mol.coords.shape[2]
        if F == 0:
            self._getMolProp(mol, "all")  # the selections are still checked
            return np.zeros((0, self._n_out(mol)), np.float32)
        d, records, d_sel, d_off = self._device(mol)
        if self._refmol is None:
            centre = coord_sums_device(d, d_sel, records) / F
        else:
            centre = torch.from_numpy(self.reference_centre(mol)).to(d.device)
        return fluctuation_device(d, d_sel, centre, records, groups=d_off).cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        atomsel = self._getMolProp(mol, "atomsel")
        idx = np.where(atomsel)[0]
        types, indexes, desc = [], [], []
        if self._mode == "atom":
            for i in idx:
                types.append("fluctuation")
                indexes.append(int(i))
                desc.append(f"Fluctuation of {mol.resname[i]} {mol.resid[i]} {mol.name[i]}")
        else:
            resid = np.asarray(mol.resid)[idx]
            order, offsets, residues = residue_groups(resid)
            for g, r in enumerate(residues):
                atoms = idx[order[offsets[g]:offsets[g + 1]]]
                types.append("fluctuation")
                indexes.append(atoms)
                desc.append(f"Fluctuation of residue {mol.resname[atoms[0]]} {r}")
        return DataFrame({"type": types, "atomIndexes": indexes, "description": desc})
