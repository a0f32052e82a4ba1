"""Drop-in for ``moleculekit.projections.metricdistance`` (MetricDistance / MetricSelfDistance).

Constructor arguments, defaults, output shapes / dtypes, error messages and ``getMapping`` follow
moleculekit/projections/metricdistance.py:19-364; ``project`` runs on the GPU through libmkb200 (K3 dense
distances / K5 group reductions, post-ops fused).  ``mol`` is duck-typed: a moleculekit ``Molecule`` or
:class:`moleculekit_b200.molecule_lite.MolLite` (needs coords, box, chain, resid, resname, name, element,
numAtoms, numFrames, atomselect).
"""
from __future__ import annotations

import logging

import numpy as np

from .projection import Projection

logger = logging.getLogger(__name__)


def _is_index_or_mask(x) -> bool:
    return isinstance(x, np.ndarray) and (np.issubdtype(x.dtype, np.integer) or x.dtype == bool)


class MetricDistance(Projection):
    """Distances / contacts between two atom selections over a trajectory.

    Parameters mirror the reference (metricdistance.py:81-94): ``sel1``/``sel2`` (selection string, boolean mask,
    integer index array, or a list / 2-D array of those for explicit groups), ``periodic`` (None | "chains" |
    "selections"), ``groupsel1/2`` (None | "all" | "residue"), ``metric`` ("distances" | "contacts"), ``threshold``,
    ``truncate``, ``groupreduce1/2`` ("closest" | "com"), ``pairs``.
    """

    def __init__(self, sel1, sel2, periodic, groupsel1=None, groupsel2=None, metric: str = "distances",
                 threshold: float = 8, truncate: float | None = None, groupreduce1: str = "closest",
                 groupreduce2: str = "closest", pairs: bool = False):
        super().__init__()
        if periodic is not None and periodic not in ["chains", "selections"]:
            raise RuntimeError("Option `periodic` can only be None, 'chains' or 'selections'.")
        self.sel1, self.sel2, self.periodic = sel1, sel2, periodic
        self.groupsel1, self.groupsel2 = groupsel1, groupsel2
        self.metric, self.threshold, self.truncate = metric, threshold, truncate
        self.groupreduce1, self.groupreduce2, self.pairs = groupreduce1, groupreduce2, pairs
        self.device = None  # CUDA device for project(); None = current device
        # True: float32 distances bit-identical to the reference.  False: atom-atom distances within 4 ulp of them
        # (MKB_DIST_DISTANCES_FAST, about twice the kernel throughput); contacts and group reductions are unaffected
        self.exact = True

    # ------------------------------------------------------------------ selections
    def _calculateMolProp(self, mol, props="all"):
        props = ("sel1", "sel2") if props == "all" else props
        res = {}
        if "sel1" in props:
            res["sel1"] = self._processSelection(mol, self.sel1, self.groupsel1)
        if "sel2" in props:
            res["sel2"] = self._processSelection(mol, self.sel2, self.groupsel2)
        return res

    def _processSelection(self, mol, sel, groupsel):
        simple = isinstance(sel, str) or (_is_index_or_mask(sel) and sel.ndim == 1)
        if simple:
            if groupsel is None:
                out = mol.atomselect(sel)
            elif groupsel == "all":
                out = self._processMultiSelections(mol, [sel])
            elif groupsel == "residue":
                out = self._groupByResidue(mol, sel)
            else:
                raise RuntimeError("Invalid groupsel argument")
        elif isinstance(sel, (np.ndarray, list)):  # user-defined groups
            out = self._processMultiSelections(mol, sel)
        else:
            raise RuntimeError(
                "Invalid atom selection. Either provide a string, a list of string, a 1D numpy array (int/bool) or a 2D numpy array for groups."
            )
        if np.sum(out) == 0:
            raise RuntimeError("Selection returned 0 atoms")
        return out

    def _processMultiSelections(self, mol, sel):
        groups = np.zeros((len(sel), mol.numAtoms), dtype=bool)
        for g, s in enumerate(sel):
            if isinstance(s, str):
                groups[g, :] = mol.atomselect(s)
            elif _is_index_or_mask(s):
                groups[g, s] = True
            else:
                raise RuntimeError("Invalid selection provided for groups")
        return groups

    def _groupByResidue(self, mol, sel):
        idx = mol.atomselect(sel, indexes=True)
        resids = np.asarray(mol.resid)[idx]
        uq = np.unique(resids)  # sorted; same grouping as the reference's pandas groupby on resid
        groups = np.zeros((len(uq), mol.numAtoms), dtype=bool)
        for g, r in enumerate(uq):
            groups[g, idx[resids == r]] = True
        return groups

    def _checkChains(self, mol, sel1, sel2):
        if np.array_equal(sel1, sel2):
            return
        a = np.any(np.atleast_2d(sel1), axis=0)
        b = np.any(np.atleast_2d(sel2), axis=0)
        if len(np.intersect1d(np.asarray(mol.chain)[a], np.asarray(mol.chain)[b])):
            logger.warning(
                "Atomselections sel1 and sel2 of MetricDistance contain atoms belonging to a common chain. "
                "Atoms within the same chain will not have periodic distances computed. "
                "Ensure that chains are properly defined in your topology file."
            )

    # ------------------------------------------------------------------ projection
    def project(self, mol):
        """(numFrames, ndims) float32 distances or bool contacts."""
        from .util import get_reduced_distances, pp_calcDistances

        sel1 = self._getMolProp(mol, "sel1")
        sel2 = self._getMolProp(mol, "sel2")
        if self.periodic == "chains":
            self._checkChains(mol, sel1, sel2)
        if np.ndim(sel1) == 1 and np.ndim(sel2) == 1:
            if self.pairs:
                raise RuntimeError("Pairs calculation not implemented without groups")
            return pp_calcDistances(mol, sel1, sel2, self.periodic, self.metric, self.threshold,
                                    truncate=self.truncate, device=self.device, exact=self.exact)
        return get_reduced_distances(mol, sel1, sel2, self.periodic, self.metric, self.threshold,
                                     truncate=self.truncate, reduction1=self.groupreduce1,
                                     reduction2=self.groupreduce2, pairs=self.pairs, device=self.device)

    def getMapping(self, mol):
        """DataFrame (type, atomIndexes, description), one row per projected dimension (metricdistance.py:244-318)."""
        from pandas import DataFrame

        sel1 = self._getMolProp(mol, "sel1")
        sel2 = self._getMolProp(mol, "sel2")

        def members(sel):
            if np.ndim(sel) == 2:
                return [np.where(row)[0] for row in sel]
            return np.where(sel)[0]

        atoms1, atoms2 = members(sel1), members(sel2)
        kind = self.metric[:-1]

        def label(i):
            return f"{mol.resname[i]} {mol.resid[i]} {mol.name[i]}"

        lab1 = [label(i) for i in atoms1]
        rows = []
        if np.array_equal(sel1, sel2):
            for i in range(len(atoms1)):
                for j in range(i + 1, len(atoms1)):
                    rows.append((kind, [atoms1[i], atoms1[j]], f"{kind} between {lab1[i]} and {lab1[j]}"))
        else:
            lab2 = [label(i) for i in atoms2]
            if not self.pairs:
                for i in range(len(atoms1)):
                    for j in range(len(atoms2)):
                        rows.append((kind, [atoms1[i], atoms2[j]], f"{kind} between {lab1[i]} and {lab2[j]}"))
            else:
                for i in range(len(atoms1)):
                    rows.append((kind, [atoms1[i], atoms2[i]], f"{kind} between {lab1[i]} and {lab2[i]}"))
        return DataFrame({"type": [r[0] for r in rows], "atomIndexes": [r[1] for r in rows],
                          "description": [r[2] for r in rows]})


class MetricSelfDistance(MetricDistance):
    """All pairs inside one selection (metricdistance.py:321-364)."""

    def __init__(self, sel, groupsel=None, metric: str = "distances", threshold: float = 8, periodic=None,
                 truncate: float | None = None):
        super().__init__(sel1=sel, sel2=sel, periodic=periodic, groupsel1=groupsel, groupsel2=groupsel,
                         metric=metric, threshold=threshold, truncate=truncate)
