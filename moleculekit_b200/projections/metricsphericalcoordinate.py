"""Drop-in for ``moleculekit.projections.metricsphericalcoordinate.MetricSphericalCoordinate``: the spherical
coordinates of one selection's centre relative to another's, per frame, after superposition onto a reference.

``project`` runs the shared pipeline of ``common`` (one upload, wrap, fit) and then one K20 call with two unweighted
groups, the reference atoms and the target atoms: only their two centres per frame come back.  ``mol`` is duck-typed
(a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from .common import check_sizes, fit, nonempty, reference, selections, upload_wrapped
from .projection import Projection


def spherical_features(moments) -> np.ndarray:
    """(F, 3) float32 ``[r, theta, phi]`` from (F, 2, 6) moments (group 0 the reference atoms, group 1 the target
    atoms; columns 0-2 the centre): x = mu_target - mu_ref, r = |x|, theta = arccos(x_z / r), phi = arctan2(x_y, x_x),
    in float64 and rounded once.  r = 0 gives theta NaN and phi 0."""
    m = np.asarray(moments, dtype=np.float64)
    x = m[:, 1, :3] - m[:, 0, :3]
    r = np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        theta = np.arccos(x[:, 2] / r)
    phi = np.arctan2(x[:, 1], x[:, 0])
    return np.column_stack([r, theta, phi]).astype(np.float32)


class MetricSphericalCoordinate(Projection):
    """Spherical coordinates ``[r, theta, phi]`` of the centre of the ``targetcom`` atoms relative to the centre of the
    ``refcom`` atoms.

    Rules (the reference's documented API):

    - Every frame is first superposed onto ``refmol`` at ``refmol.frame`` (required): the ``trajalnstr`` atoms onto the
      ``refalnstr`` atoms (default ``trajalnstr``), so the angles are measured in the reference's frame.
    - With ``pbc`` the trajectory is first wrapped around ``centerstr`` exactly as Molecule.wrap (and MetricRmsd) does.
    - The centres are plain (unweighted) means of the float32 aligned coordinates.  With x = mu_target - mu_ref:
      r = |x|, theta = arccos(x_z / r) in [0, pi], phi = arctan2(x_y, x_x) in [-pi, pi], all in float64 and rounded
      to float32 once; r = 0 gives theta NaN and phi 0, as numpy does.  The two selections may overlap.
    - ``project`` returns (numFrames, 3) float32.  ``getMapping``: 3 rows, ``type`` "sphericalcoordinate",
      ``atomIndexes`` the ``refcom`` atoms followed by the ``targetcom`` atoms, descriptions "r", "theta", "phi".
    - A non-finite coordinate in the alignment selection raises ``numpy.linalg.LinAlgError`` before anything is
      computed; one in either centre's selection gives NaN in that frame.  Empty selections raise ``RuntimeError``
      ("... selection resulted in 0 atoms.").  Zero frames give (0, 3).  ``mol`` is not modified.
    """

    def __init__(self, refmol, targetcom, refcom, trajalnstr="protein and name CA", refalnstr=None,
                 centerstr="protein", pbc=True):
        super().__init__()
        if refmol is None:
            raise ValueError("MetricSphericalCoordinate needs refmol: every frame is superposed onto it")
        if refalnstr is None:
            refalnstr = trajalnstr
        self._refmol, self._refcoords = reference(refmol)
        self._refalnsel = nonempty(self._refmol, refalnstr, "Reference alignment")
        self._targetcom, self._refcom = targetcom, refcom
        self._trajalnsel, self._centersel = trajalnstr, centerstr
        self._pbc = pbc
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        return selections(mol, props, (("targetcom", self._targetcom, "Target COM", True),
                                       ("refcom", self._refcom, "Reference COM", True),
                                       ("trajalnsel", self._trajalnsel, "Alignment", True),
                                       ("centersel", self._centersel, "Centering", self._pbc)))

    def _layout(self, props):
        """(selection: the refcom atoms then the targetcom atoms, group offsets [0, n_ref, n_ref + n_target])"""
        ref, tgt = np.where(props["refcom"])[0], np.where(props["targetcom"])[0]
        return np.concatenate([ref, tgt]), np.array([0, ref.size, ref.size + tgt.size], np.int64)

    def project(self, mol) -> np.ndarray:
        """(numFrames, 3) float32 ``[r, theta, phi]``."""
        import torch

        from ..coords import frame_moments_device

        props = self._getMolProp(mol, "all")
        check_sizes("alignment", props["trajalnsel"], self._refalnsel)
        sel, offsets = self._layout(props)
        if mol.coords.shape[2] == 0:
            return np.zeros((0, 3), np.float32)
        d = upload_wrapped(mol, props.get("centersel"), self.device)
        records = fit(d, props["trajalnsel"], self._refcoords, self._refalnsel)
        d_sel = torch.from_numpy(sel.astype(np.int32)).to(d.device)
        moments = frame_moments_device(d, d_sel, records, groups=offsets)
        return spherical_features(moments.cpu().numpy())

    def getMapping(self, mol):
        from pandas import DataFrame

        sel, _ = self._layout({p: self._getMolProp(mol, p) for p in ("targetcom", "refcom")})
        return DataFrame({"type": ["sphericalcoordinate"] * 3, "atomIndexes": [sel] * 3,
                          "description": ["r", "theta", "phi"]})
