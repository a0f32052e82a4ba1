"""Drop-in for ``moleculekit.projections.metriccoordinate.MetricCoordinate``: the aligned Cartesian coordinates of a
selection, one row per frame (a standard TICA / MSM featurisation).

``project`` uploads the trajectory once, wraps it on the device (K9 / K9b, the decisions of Molecule.wrap, as
MetricRmsd does), fits every frame onto the reference (K14) and writes the (numFrames, 3n) feature matrix straight from
the trajectory (K15): the aligned trajectory is never written and nothing is gathered on the host.  ``mol`` is
duck-typed (a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from .common import check_sizes, fit, nonempty, reference, selections, upload_wrapped
from .projection import Projection


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
            self._refmol, self._refcoords = reference(refmol)
            self._refalnsel = nonempty(self._refmol, refalnsel, "Reference alignment")
        self._atomsel, self._trajalnsel, self._centersel = atomsel, trajalnsel, centersel
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        return selections(mol, props, (("atomsel", self._atomsel, "Atom", True),
                                       ("trajalnsel", self._trajalnsel, "Alignment", self._refmol is not None),
                                       ("centersel", self._centersel, "Centering", self._pbc)))

    def project(self, mol) -> np.ndarray:
        """(numFrames, 3n) float32 aligned coordinates."""
        import torch

        from ..coords import coordinates_device

        props = self._getMolProp(mol, "all")
        sel = np.where(props["atomsel"])[0]
        if self._refmol is not None:
            check_sizes("alignment", props["trajalnsel"], self._refalnsel)
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros((0, 3 * sel.size), np.float32)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        records = None if self._refmol is None else fit(d, props["trajalnsel"], self._refcoords, self._refalnsel)
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
