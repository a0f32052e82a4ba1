"""Drop-in for ``moleculekit.projections.metricrmsd.MetricRmsd``: RMSD of every frame to a reference structure after
wrapping and superposition.

Constructor defaults follow the reference's documented API: the alignment selection defaults to the RMSD selection, the
reference selections to the trajectory ones, and a multi-frame reference is used at ``refmol.frame`` with a warning.
``project`` uploads the trajectory once, wraps it on the device (K9 / K9b, the decisions of Molecule.wrap), fits every
frame (K14) and computes the RMSD over the RMSD selection from the fit records: the aligned trajectory is never
written and only one float per frame comes back.  ``mol`` is duck-typed (a moleculekit ``Molecule`` or
:class:`moleculekit_b200.molecule_lite.MolLite`).
"""
from __future__ import annotations

import logging

import numpy as np

from .projection import Projection

logger = logging.getLogger(__name__)


def _nonempty(mol, sel, what):
    mask = np.asarray(mol.atomselect(sel))
    if mask.dtype != bool:
        m = np.zeros(mol.numAtoms, dtype=bool)
        m[mask] = True
        mask = m
    if not mask.any():
        raise RuntimeError(f"{what} selection resulted in 0 atoms.")
    return mask


class MetricRmsd(Projection):
    """RMSD of ``trajrmsdstr`` atoms to the ``refrmsdstr`` atoms of ``refmol`` after aligning ``trajalnstr`` onto
    ``refalnstr``; with ``pbc`` the trajectory is first wrapped around ``centerstr``."""

    def __init__(self, refmol, trajrmsdstr, trajalnstr=None, refrmsdstr=None, refalnstr=None, centerstr="protein",
                 pbc=True):
        super().__init__()
        if trajalnstr is None:
            trajalnstr = trajrmsdstr
        if refalnstr is None:
            refalnstr = trajalnstr
        if refrmsdstr is None:
            refrmsdstr = trajrmsdstr
        self._refmol = refmol.copy()
        frame = int(getattr(refmol, "frame", 0))
        if self._refmol.coords.shape[2] > 1:
            logger.warning(f"Reference molecule contains multiple frames. MetricRmsd will use frame {frame} as reference.")
        self._refcoords = np.ascontiguousarray(refmol.coords[:, :, frame:frame + 1], dtype=np.float32)
        self._refalnsel = _nonempty(self._refmol, refalnstr, "Reference alignment")
        self._refrmsdsel = _nonempty(self._refmol, refrmsdstr, "Reference RMSD")
        self._trajalnsel, self._trajrmsdsel = trajalnstr, trajrmsdstr
        self._centersel = centerstr
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        props = ("trajalnsel", "trajrmsdsel", "centersel") if props == "all" else props
        res = {}
        if "trajalnsel" in props:
            res["trajalnsel"] = _nonempty(mol, self._trajalnsel, "Alignment")
        if "trajrmsdsel" in props:
            res["trajrmsdsel"] = _nonempty(mol, self._trajrmsdsel, "RMSD atom")
        if "centersel" in props and self._pbc:
            res["centersel"] = _nonempty(mol, self._centersel, "Centering")
        return res

    def project(self, mol) -> np.ndarray:
        """(numFrames,) float32 RMSDs."""
        import torch

        from ..align import raise_if_nonfinite, rmsd_device, superpose_device
        from .. import _lib
        from ..wrapping import wrap_plan

        props = self._getMolProp(mol, "all")
        aln, rms = props["trajalnsel"], props["trajrmsdsel"]
        for what, a, b in (("alignment", aln, self._refalnsel), ("RMSD", rms, self._refrmsdsel)):
            if a.sum() != b.sum():
                raise RuntimeError(f"The {what} selections of the trajectory and the reference differ in size: "
                                   f"{int(a.sum())} and {int(b.sum())} atoms.")
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros(0, np.float32)
        dev = _lib.device(self.device)
        d = torch.from_numpy(np.ascontiguousarray(mol.coords, dtype=np.float32)).to(dev)
        if self._pbc:
            plan = wrap_plan(mol, props["centersel"])
            if plan is not None:
                plan.run_device(d, torch.from_numpy(np.ascontiguousarray(mol.box, dtype=np.float32)).to(dev))
        ref = torch.from_numpy(self._refcoords).to(dev)

        def idx(mask):
            return torch.from_numpy(np.where(mask)[0].astype(np.int32)).to(dev)

        records, status = superpose_device(d, idx(aln), ref, idx(self._refalnsel))
        raise_if_nonfinite(status, np.arange(F))
        return rmsd_device(d, idx(rms), ref, idx(self._refrmsdsel), records).cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        rms = self._getMolProp(mol, "trajrmsdsel")
        return DataFrame({"type": ["rmsd"], "atomIndexes": [np.where(rms)[0]],
                          "description": ["RMSD to reference structure."]})
