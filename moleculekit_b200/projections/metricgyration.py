"""Drop-in for ``moleculekit.projections.metricgyration.MetricGyration``: the mass-weighted radius of gyration of a
selection per frame, with its per-axis components.

``project`` runs the shared pipeline of ``common`` (one upload, wrap, optional fit) and then one K20 call, the
mass-weighted centre and per-axis spread of the selection in every frame: the aligned trajectory is never written and
only six float64 values per frame come back.  ``mol`` is duck-typed (a moleculekit ``Molecule`` or
:class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from .common import check_sizes, fit, nonempty, reference, selections, upload_wrapped
from .projection import Projection


def selection_masses(mol, idx) -> np.ndarray:
    """(k,) float64 weights of the atoms ``idx``: ``mol.masses`` when the container has them and they sum to more than
    0 over the selection, else the element masses of ``mol.element`` (KeyError on an unknown symbol)."""
    from ..elements import masses_of

    masses = getattr(mol, "masses", None)
    if masses is not None:
        m = np.asarray(masses, dtype=np.float64)[idx]
        if m.sum() > 0:
            return m
    return masses_of(np.asarray(mol.element)[idx]).astype(np.float64)


def gyration_features(moments) -> np.ndarray:
    """(F, 4) float32 ``[rg, rg_x, rg_y, rg_z]`` from (F, 6) moments (mean, then per-axis variance): rg_d = sqrt(v_d)
    and rg = sqrt(v_x + v_y + v_z), in float64 and rounded once."""
    v = np.asarray(moments, dtype=np.float64)[:, 3:6]
    rg = np.sqrt((v[:, 0] + v[:, 1]) + v[:, 2])
    return np.column_stack([rg, np.sqrt(v)]).astype(np.float32)


class MetricGyration(Projection):
    """Radius of gyration of the ``atomsel`` atoms, weighted by mass, with its x, y and z components.

    Rules (the reference's documented API):

    - ``project`` returns (numFrames, 4) float32 ``[rg, rg_x, rg_y, rg_z]``.  With mu = sum m c / M the mass-weighted
      centre of the selection in a frame (c the float32 coordinate, M the selection's total mass) and
      v_d = sum m (c_d - mu_d)^2 / M per axis: rg_d = sqrt(v_d) and rg = sqrt(v_x + v_y + v_z).  Everything is float64,
      rounded to float32 once.
    - Masses: ``mol.masses`` of the selection when the container has that attribute and they sum to more than 0, else
      the element masses of ``mol.element`` (``KeyError`` on an unknown symbol).
    - With ``refmol`` every frame is first superposed onto ``refmol`` at ``refmol.frame``: the ``trajalnstr`` atoms onto
      the ``refalnstr`` atoms (default ``trajalnstr``).  rg does not change, but the components are then measured along
      the reference's axes.  Without ``refmol`` nothing is superposed.
    - With ``pbc`` the trajectory is first wrapped around ``centerstr`` exactly as Molecule.wrap (and MetricRmsd) does.
    - ``getMapping``: 4 rows, ``type`` "gyration", ``atomIndexes`` the selection, descriptions "Radius of gyration",
      "x component", "y component", "z component".
    - A non-finite coordinate in the alignment selection raises ``numpy.linalg.LinAlgError`` before anything is
      computed; a non-finite coordinate in the selection gives NaN in that frame.  Empty selections raise
      ``RuntimeError`` ("... selection resulted in 0 atoms.").  Zero frames give (0, 4).  ``mol`` is not modified.
    """

    def __init__(self, atomsel, refmol=None, trajalnstr="protein and name CA", refalnstr=None, centerstr="protein",
                 pbc=True):
        super().__init__()
        if refalnstr is None:
            refalnstr = trajalnstr
        self._refmol = self._refcoords = self._refalnsel = None
        if refmol is not None:
            self._refmol, self._refcoords = reference(refmol)
            self._refalnsel = nonempty(self._refmol, refalnstr, "Reference alignment")
        self._atomsel, self._trajalnsel, self._centersel = atomsel, trajalnstr, centerstr
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        return selections(mol, props, (("atomsel", self._atomsel, "Atom", True),
                                       ("trajalnsel", self._trajalnsel, "Alignment", self._refmol is not None),
                                       ("centersel", self._centersel, "Centering", self._pbc)))

    def project(self, mol) -> np.ndarray:
        """(numFrames, 4) float32 ``[rg, rg_x, rg_y, rg_z]``."""
        import torch

        from ..coords import frame_moments_device

        props = self._getMolProp(mol, "all")
        if self._refmol is not None:
            check_sizes("alignment", props["trajalnsel"], self._refalnsel)
        sel = np.where(props["atomsel"])[0]
        masses = selection_masses(mol, sel)
        if mol.coords.shape[2] == 0:
            return np.zeros((0, 4), np.float32)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        records = None if self._refmol is None else fit(d, props["trajalnsel"], self._refcoords, self._refalnsel)
        d_sel = torch.from_numpy(sel.astype(np.int32)).to(d.device)
        moments = frame_moments_device(d, d_sel, records, weights=masses)
        return gyration_features(moments[:, 0].cpu().numpy())

    def getMapping(self, mol):
        from pandas import DataFrame

        idx = np.where(self._getMolProp(mol, "atomsel"))[0]
        return DataFrame({"type": ["gyration"] * 4, "atomIndexes": [idx] * 4,
                          "description": ["Radius of gyration", "x component", "y component", "z component"]})
