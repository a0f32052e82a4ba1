"""Drop-in for ``moleculekit.projections.metriccoordinate.MetricCoordinate``: the aligned Cartesian coordinates of a
selection, one row per frame (a standard TICA / MSM featurisation).

``project`` uploads the trajectory once, wraps it on the device (K9 / K9b, the decisions of Molecule.wrap, as
MetricRmsd does), fits every frame onto the reference (K14) and writes the (numFrames, 3n) feature matrix straight from
the trajectory (K15): the aligned trajectory is never written and nothing is gathered on the host.  ``mol`` is
duck-typed (a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from .metricrmsd import _nonempty
from .projection import Projection


def _reference(refmol, alnsel):
    """(refmol copy, its coordinates at refmol.frame as (N, 3, 1) float32, the alignment mask on it)"""
    ref = refmol.copy()
    frame = int(getattr(refmol, "frame", 0))
    coords = np.ascontiguousarray(refmol.coords[:, :, frame:frame + 1], dtype=np.float32)
    return ref, coords, _nonempty(ref, alnsel, "Reference alignment")


def _check_sizes(what, a, b):
    if int(a.sum()) != int(b.sum()):
        raise RuntimeError(f"The {what} selections of the trajectory and the reference differ in size: "
                           f"{int(a.sum())} and {int(b.sum())} atoms.")


def _upload_wrap_fit(mol, centersel, pbc, refcoords, trajalnsel, refalnsel, device):
    """The device pipeline shared by MetricCoordinate and MetricFluctuation: upload ``mol.coords`` once, wrap it around
    ``centersel`` when ``pbc`` (``wrap_plan(...).run_device``), and with a reference fit every frame's ``trajalnsel``
    atoms onto its ``refalnsel`` atoms (``LinAlgError`` on a non-finite fit, before anything else is computed).
    Returns (the (N, 3, F) CUDA tensor, the fit records or None)."""
    import torch

    from ..align import raise_if_nonfinite, superpose_device
    from .. import _lib
    from ..wrapping import wrap_plan

    dev = _lib.device(device)
    d = torch.from_numpy(np.ascontiguousarray(mol.coords, dtype=np.float32)).to(dev)
    if pbc:
        plan = wrap_plan(mol, centersel)
        if plan is not None:
            plan.run_device(d, torch.from_numpy(np.ascontiguousarray(mol.box, dtype=np.float32)).to(dev))
    if refcoords is None:
        return d, None

    def idx(mask):
        return torch.from_numpy(np.where(mask)[0].astype(np.int32)).to(dev)

    records, status = superpose_device(d, idx(trajalnsel), torch.from_numpy(refcoords).to(dev), idx(refalnsel))
    raise_if_nonfinite(status, np.arange(d.shape[2]))
    return d, records


class MetricCoordinate(Projection):
    """Aligned coordinates of the ``atomsel`` atoms: ``project`` returns (numFrames, 3n) float32, columns all X of the
    selection (atom order), then all Y, then all Z.

    Rules (the reference's documented API):

    - With ``refmol``, every frame is first superposed onto ``refmol`` at ``refmol.frame``: the ``trajalnsel`` atoms of the
      trajectory onto the ``refalnsel`` atoms of the reference.  ``trajalnsel`` defaults to ``"protein and name CA"``
      and ``refalnsel`` to ``trajalnsel``.  Without ``refmol`` nothing is superposed.
    - With ``pbc`` the trajectory is first wrapped around ``centersel`` exactly as Molecule.wrap (and MetricRmsd) does.
    - A non-finite coordinate in the alignment selection raises ``numpy.linalg.LinAlgError`` before anything is computed.
    - ``getMapping``: 3n rows in column order, ``type`` "coordinate", ``atomIndexes`` the atom, ``description``
      "{X|Y|Z} coordinate of {resname} {resid} {name}".
    - Empty selections raise ``RuntimeError`` ("... selection resulted in 0 atoms.").
    - ``mol`` is not modified.
    """

    def __init__(self, atomsel, refmol=None, trajalnsel=None, refalnsel=None, centersel="protein", pbc=True):
        super().__init__()
        self._refmol = self._refcoords = self._refalnsel = None
        if refmol is not None:
            if trajalnsel is None:
                trajalnsel = "protein and name CA"
            if refalnsel is None:
                refalnsel = trajalnsel
            self._refmol, self._refcoords, self._refalnsel = _reference(refmol, refalnsel)
        self._atomsel, self._trajalnsel, self._centersel = atomsel, trajalnsel, centersel
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        props = ("atomsel", "trajalnsel", "centersel") if props == "all" else props
        res = {}
        if "atomsel" in props:
            res["atomsel"] = _nonempty(mol, self._atomsel, "Atom")
        if "trajalnsel" in props and self._refmol is not None:
            res["trajalnsel"] = _nonempty(mol, self._trajalnsel, "Alignment")
        if "centersel" in props and self._pbc:
            res["centersel"] = _nonempty(mol, self._centersel, "Centering")
        return res

    def project(self, mol) -> np.ndarray:
        """(numFrames, 3n) float32 aligned coordinates."""
        import torch

        from ..coords import coordinates_device

        props = self._getMolProp(mol, "all")
        sel = np.where(props["atomsel"])[0]
        if self._refmol is not None:
            _check_sizes("alignment", props["trajalnsel"], self._refalnsel)
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros((0, 3 * sel.size), np.float32)
        d, records = _upload_wrap_fit(mol, props.get("centersel"), self._pbc, self._refcoords, props.get("trajalnsel"),
                                      self._refalnsel, self.device)
        d_sel = torch.from_numpy(sel.astype(np.int32)).to(d.device)
        return coordinates_device(d, d_sel, records).cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        idx = np.where(self._getMolProp(mol, "atomsel"))[0]
        types, indexes, desc = [], [], []
        for xyz in ("X", "Y", "Z"):
            for i in idx:
                types.append("coordinate")
                indexes.append(int(i))
                desc.append(f"{xyz} coordinate of {mol.resname[i]} {mol.resid[i]} {mol.name[i]}")
        return DataFrame({"type": types, "atomIndexes": indexes, "description": desc})
