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

from .common import check_sizes, device_indices, fit, nonempty, reference, selections, upload_wrapped
from .projection import Projection

logger = logging.getLogger(__name__)


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
        self._refmol, self._refcoords = reference(refmol, logger, "MetricRmsd")
        self._refalnsel = nonempty(self._refmol, refalnstr, "Reference alignment")
        self._refrmsdsel = nonempty(self._refmol, refrmsdstr, "Reference RMSD")
        self._trajalnsel, self._trajrmsdsel = trajalnstr, trajrmsdstr
        self._centersel = centerstr
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        return selections(mol, props, (("trajalnsel", self._trajalnsel, "Alignment", True),
                                       ("trajrmsdsel", self._trajrmsdsel, "RMSD atom", True),
                                       ("centersel", self._centersel, "Centering", self._pbc)))

    def project(self, mol) -> np.ndarray:
        """(numFrames,) float32 RMSDs."""
        import torch

        from ..align import rmsd_device

        props = self._getMolProp(mol, "all")
        aln, rms = props["trajalnsel"], props["trajrmsdsel"]
        check_sizes("alignment", aln, self._refalnsel)
        check_sizes("RMSD", rms, self._refrmsdsel)
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros(0, np.float32)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        ref = torch.from_numpy(self._refcoords).to(d.device)
        records = fit(d, aln, ref, self._refalnsel)
        return rmsd_device(d, device_indices(rms, d.device), ref, device_indices(self._refrmsdsel, d.device),
                           records).cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        rms = self._getMolProp(mol, "trajrmsdsel")
        return DataFrame({"type": ["rmsd"], "atomIndexes": [np.where(rms)[0]],
                          "description": ["RMSD to reference structure."]})
