"""Drop-in for ``moleculekit.projections.metricsecondarystructure.MetricSecondaryStructure``: the DSSP secondary
structure of every residue, one row per frame.

``project`` uploads only the N, CA, C and O atoms of the residues in the DSSP sequence (compact rows) and assigns every
frame with K18.  ``mol`` is duck-typed (a moleculekit ``Molecule`` or :class:`moleculekit_b200.molecule_lite.MolLite`)
and is not modified.
"""
from __future__ import annotations

import numpy as np

from .common import column, nonempty, residues
from .projection import Projection

BACKBONE_NAMES = ("N", "CA", "C", "O")


def dssp_residues(mol, sel):
    """(backbone (n, 4) int64 atom indices of N, CA, C, O, flags (n,) uint8, position (ncols,) int64 of every ``sel``
    residue in the DSSP sequence or -1, residue atom lists) of the ``sel`` residues
    (:func:`moleculekit_b200.projections.common.residues`).  A residue enters the sequence when it has atoms
    named N, CA, C and O (the first atom of a repeated name); flag bit 0 marks resname PRO, bit 1 a residue whose chain
    or segid differs from the previous residue of the sequence."""
    from ..dssp import FLAG_CHAIN_START, FLAG_PRO

    res = residues(mol, sel)
    name, resname = column(mol, "name", ""), column(mol, "resname", "")
    chain, segid = column(mol, "chain", ""), column(mol, "segid", "")
    backbone, flags, pos = [], [], np.full(len(res), -1, np.int64)
    prev = None
    for r, atoms in enumerate(res):
        names = {}
        for a in atoms:
            names.setdefault(str(name[a]), int(a))
        if not all(n in names for n in BACKBONE_NAMES):
            continue
        a0 = atoms[0]
        f = FLAG_PRO if str(resname[a0]) == "PRO" else 0
        if prev is not None and (chain[a0] != chain[prev] or segid[a0] != segid[prev]):
            f |= FLAG_CHAIN_START
        pos[r] = len(backbone)
        backbone.append([names[n] for n in BACKBONE_NAMES])
        flags.append(f)
        prev = a0
    return (np.array(backbone, np.int64).reshape(-1, 4), np.array(flags, np.uint8), pos, res)


class MetricSecondaryStructure(Projection):
    """DSSP secondary structure per residue: ``project`` returns (numFrames, ncols), one column per residue of ``sel``.

    - ``integer=True``: int64 codes, simplified ``H 0, E 1, C 2`` or full ``H 0, B 1, E 2, G 3, I 4, T 5, S 6, ' ' 7``;
      a residue without all four backbone atoms gives -1.
    - ``integer=False``: a ``'<U2'`` string array, as mdtraj returns: the full letters (``' '`` for loop) or, with
      ``simplified``, ``H G I -> H``, ``E B -> E`` and ``T S ' ' -> C``; ``'NA'`` for a residue without all four
      backbone atoms.

    Rules (DSSP 2.2.0 as mdtraj ports it, restated in ``mkb_dssp`` of include/mkb200.h):

    - Residues are runs of consecutive ``sel`` atoms with the same resid, insertion code, chain and segid.  A residue
      with atoms named N, CA, C and O (the first atom of a repeated name) enters the DSSP sequence; the sequence
      concatenates all chains in atom order.  Only resname PRO is a proline.
    - A chain break lies between sequence neighbours that differ in chain or segid or whose C-N distance exceeds 2.5 A.
    - Everything is float64 from the float32 Angstrom coordinates with every operation rounded on its own: the amide H
      (N plus the unit C=O vector of the previous residue, or N after a break or on a proline), the Kabsch-Sander energy
      with DSSP's 0.001 rounding, its -9.9 floor and its 0.5 A minimum distance, the 9 A CA screen, the two best
      acceptors per donor, and the kappa bend (> 70 degrees, decided against libm's ``acos``).
    - Helices, bridges, ladders (with DSSP's bulge rule and its uint32 differences) and the codes H, B, E, G, I, T, S
      follow DSSP 2.2.0; G and I need two consecutive helix starts, as H does; there is no pi-helix priority.
    - ``getMapping``: one row per column, ``type`` "secondary structure", ``atomIndexes`` the residue's atoms,
      ``description`` "Secondary structure of residue {resname} {resid}".
    - An empty ``sel`` raises ``RuntimeError``.  ``project_sharded`` works on frame blocks; in string mode the rows
      cannot be all-gathered, so it raises ``ValueError`` there with ``gather=True`` on more than one rank.

    Not confirmed against mdtraj or moleculekit:

    - mdtraj's own arithmetic: it works in float32 nm with SSE, where this uses float64 Angstrom.  A bond within rounding
      of -0.5, or a bend within rounding of 70 degrees, can flip.
    - Whether mdtraj keeps DSSP's 0.001 energy rounding and the 0.5 A minimum distance.
    - Whether it breaks chains on the 2.5 A C-N distance as well as on topology chains.
    - The H placement after a break.
    - The tie order of DSSP's ``std::sort`` of the bridges (creation order is kept here).
    - moleculekit's parameter names and defaults, its integer tables, the ``NA`` handling in integer mode, and the
      mapping text.
    """

    def __init__(self, sel="protein", simplified=True, integer=True):
        super().__init__()
        self._sel = sel
        self._simplified = bool(simplified)
        self._integer = bool(integer)
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        """``dssp``: (backbone (n, 4) atom indices, flags (n,) uint8, sequence position per column or -1, column atom
        lists)."""
        props = ("dssp",) if props == "all" else props
        res = {}
        if "dssp" in props:
            res["dssp"] = dssp_residues(mol, nonempty(mol, self._sel, "Atom"))
        return res

    def _encode(self, codes, pos):
        """(F, ncols) output of the device codes (F, n) for the columns' sequence positions ``pos``."""
        from ..dssp import FULL_INT, LETTERS, SIMPLE_INT, SIMPLE_LETTERS

        have = pos >= 0
        F = codes.shape[0]
        if self._integer:
            out = np.full((F, pos.size), -1, np.int64)
            table = SIMPLE_INT if self._simplified else FULL_INT
        else:
            out = np.full((F, pos.size), "NA", "<U2")
            table = SIMPLE_LETTERS if self._simplified else LETTERS
        out[:, have] = table[codes[:, pos[have]]]
        return out

    def project(self, mol) -> np.ndarray:
        """(numFrames, ncols) int64 codes or '<U2' letters."""
        import torch

        from ..dssp import dssp_device
        from .. import _lib

        backbone, flags, pos, _ = self._getMolProp(mol, "dssp")
        F, n = mol.coords.shape[2], backbone.shape[0]
        if F == 0 or n == 0:
            return self._encode(np.zeros((F, 0), np.uint8), pos)
        dev = _lib.device(self.device)
        atoms, rows = np.unique(backbone, return_inverse=True)
        d = torch.from_numpy(np.ascontiguousarray(mol.coords[atoms], dtype=np.float32)).to(dev)
        d_bb = torch.from_numpy(rows.reshape(n, 4).astype(np.int32)).to(dev)
        d_flags = torch.from_numpy(flags).to(dev)
        codes = dssp_device(d, d_bb, d_flags).cpu().numpy()
        return self._encode(codes, pos)

    def getMapping(self, mol):
        from pandas import DataFrame

        _, _, _, cols = self._getMolProp(mol, "dssp")
        resname, resid = column(mol, "resname", ""), column(mol, "resid", 0)
        desc = [f"Secondary structure of residue {resname[c[0]]} {resid[c[0]]}" for c in cols]
        return DataFrame({"type": ["secondary structure"] * len(cols), "atomIndexes": [c.copy() for c in cols],
                          "description": desc})
