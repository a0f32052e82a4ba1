"""Drop-in for ``moleculekit.projections.metrictmscore.MetricTMscore``: the TM-score of every frame against a reference
structure.

``project`` uploads the trajectory once, wraps it on the device around ``centerstr`` (K9 / K9b, as
``MetricRmsd.project`` does) and runs the TM-score search of every frame (K19); one float per frame comes back.  ``mol``
is duck-typed (a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import logging

import numpy as np

from .common import nonempty, reference, upload_wrapped
from .projection import Projection

logger = logging.getLogger(__name__)


class MetricTMscore(Projection):
    """TM-score of the ``trajtmstr`` CA atoms against the ``reftmstr`` CA atoms of ``refmol`` at ``refmol.frame``:
    ``project`` returns (numFrames,) float32.

    Rules (the superposition search of the TMscore program, restated in ``mkb_tmscore`` of include/mkb200.h):

    - Both selections are reduced to the atoms named CA, in atom order.  Pair k joins the k-th CA of each, for
      k < L = min(n, m); the score is normalised by m, the reference's CA count.
    - d0 = 1.24 (m - 15)^(1/3) - 1.8 (at least 0.5; 0.5 for m <= 15), d0_search = d0 clamped to [4.5, 8].  Seeds are
      every window of the fragment lengths L, L / 2, ... L / 16 (floored, down to 4) and 4; each seed is fitted, then
      refitted on its cut set (d0_search - 1 for the seed, d0_search + 1 after it, widened by 0.5 below 3 pairs) up to
      20 times or until the set repeats.  The TM-score is the best score of any fit.
    - Everything is float64 from the float32 coordinates, every operation rounded on its own.
    - With ``pbc`` the trajectory is first wrapped around ``centerstr`` on the device, as Molecule.wrap does.
    - A frame with a non-finite paired coordinate gives NaN (the reference keeps its initial -1 there).  A non-finite
      reference coordinate raises ``ValueError``, selections without CA atoms ``RuntimeError``, more pairs than
      :func:`moleculekit_b200.tmscore.max_pairs` ``ValueError``.
    - ``getMapping``: one row, ``type`` "tmscore", ``atomIndexes`` the trajectory's CA atoms, ``description``
      "TM-score to reference structure."

    Not confirmed against moleculekit (its compiled routine's sources were not available):

    - The exact parameter names and defaults.
    - The dtype and shape of ``project`` (float32 (F,) here, not float64 or (F, 1)).
    - The d0 rule for Lnorm <= 15, where the reference's C ``pow`` sees a negative base.
    - The ``pbc`` switch and what is wrapped.
    - Whether the extension loop runs 19 or 20 times.
    - Whether ``dcut`` persists across calls of the score function in the reference (here every cut starts afresh).
    - The NaN behaviour for non-finite coordinates.
    - The mapping text.
    """

    def __init__(self, refmol, trajtmstr, reftmstr=None, centerstr="protein", pbc=True):
        from ..tmscore import ca_atoms

        super().__init__()
        if reftmstr is None:
            reftmstr = trajtmstr
        self._refmol, refcoords = reference(refmol, logger, "MetricTMscore")
        self._refca = ca_atoms(self._refmol, reftmstr, "Reference TM-score")
        self._refcoords = refcoords[self._refca]
        self._trajtmsel = trajtmstr
        self._centersel = centerstr
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        from ..tmscore import ca_atoms

        props = ("trajca", "centersel") if props == "all" else props
        res = {}
        if "trajca" in props:
            res["trajca"] = ca_atoms(mol, self._trajtmsel, "TM-score")
        if "centersel" in props and self._pbc:
            res["centersel"] = nonempty(mol, self._centersel, "Centering")
        return res

    def project(self, mol) -> np.ndarray:
        """(numFrames,) float32 TM-scores."""
        import torch

        from ..tmscore import tmscore_device

        props = self._getMolProp(mol, "all")
        ca = props["trajca"]
        F = mol.coords.shape[2]
        if F == 0:
            return np.zeros(0, np.float32)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        dev = d.device
        ref = torch.from_numpy(self._refcoords).to(dev)
        sel = torch.from_numpy(ca.astype(np.int32)).to(dev)
        refsel = torch.arange(self._refca.size, dtype=torch.int32, device=dev)
        tm, _ = tmscore_device(d, sel, ref, refsel)
        return tm.float().cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        ca = self._getMolProp(mol, "trajca")
        return DataFrame({"type": ["tmscore"], "atomIndexes": [ca.copy()],
                          "description": ["TM-score to reference structure."]})
