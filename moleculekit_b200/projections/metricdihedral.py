"""Drop-in for ``moleculekit.projections.metricdihedral.MetricDihedral``: backbone and side-chain torsion angles, one
row per frame (by default sin / cos of psi and phi, the usual Markov state model featurisation).

The quadruples are chosen on the host from the residue bookkeeping of ``mol``; ``project`` uploads only the atoms some
quadruple references (compact rows, so the device never sees the rest of the system) and evaluates every (frame,
dihedral) with K16.  ``mol`` is duck-typed (a moleculekit ``Molecule`` or
:class:`moleculekit_b200.molecule_lite.MolLite`) and is not modified.
"""
from __future__ import annotations

import numpy as np

from .common import column, nonempty, residues
from .projection import Projection

# (residue offset, atom name) of the four atoms; offset -1 = the previous residue, +1 = the next one
BACKBONE = {
    "phi": ((-1, "C"), (0, "N"), (0, "CA"), (0, "C")),
    "psi": ((0, "N"), (0, "CA"), (0, "C"), (1, "N")),
    "omega": ((-1, "CA"), (-1, "C"), (0, "N"), (0, "CA")),
}

# the standard (IUPAC-IUB 1970) side-chain torsions, per residue
CHI = {
    "chi1": {"ARG": "N CA CB CG", "ASN": "N CA CB CG", "ASP": "N CA CB CG", "CYS": "N CA CB SG",
             "GLN": "N CA CB CG", "GLU": "N CA CB CG", "HIS": "N CA CB CG", "ILE": "N CA CB CG1",
             "LEU": "N CA CB CG", "LYS": "N CA CB CG", "MET": "N CA CB CG", "PHE": "N CA CB CG",
             "PRO": "N CA CB CG", "SER": "N CA CB OG", "THR": "N CA CB OG1", "TRP": "N CA CB CG",
             "TYR": "N CA CB CG", "VAL": "N CA CB CG1"},
    "chi2": {"ARG": "CA CB CG CD", "ASN": "CA CB CG OD1", "ASP": "CA CB CG OD1", "GLN": "CA CB CG CD",
             "GLU": "CA CB CG CD", "HIS": "CA CB CG ND1", "ILE": "CA CB CG1 CD1", "LEU": "CA CB CG CD1",
             "LYS": "CA CB CG CD", "MET": "CA CB CG SD", "PHE": "CA CB CG CD1", "PRO": "CA CB CG CD",
             "TRP": "CA CB CG CD1", "TYR": "CA CB CG CD1"},
    "chi3": {"ARG": "CB CG CD NE", "GLN": "CB CG CD OE1", "GLU": "CB CG CD OE1", "LYS": "CB CG CD CE",
             "MET": "CB CG SD CE"},
    "chi4": {"ARG": "CG CD NE CZ", "LYS": "CG CD CE NZ"},
    "chi5": {"ARG": "CD NE CZ NH1"},
}

# force-field names of protonation / disulfide variants, looked up as the standard residue
ALIASES = {"HID": "HIS", "HIE": "HIS", "HIP": "HIS", "HSD": "HIS", "HSE": "HIS", "HSP": "HIS",
           "CYX": "CYS", "CYM": "CYS", "ASH": "ASP", "GLH": "GLU", "LYN": "LYS"}

# atom names some force fields use instead of the IUPAC ones (CHARMM calls the isoleucine delta carbon CD)
ALT_NAMES = {("ILE", "CD1"): "CD"}

TYPES = tuple(BACKBONE) + tuple(CHI)


def _check_types(dih):
    bad = [d for d in dih if d not in TYPES]
    if bad:
        raise ValueError(f"Unknown dihedral type(s) {bad}; supported: {', '.join(TYPES)}")


def select_dihedrals(mol, sel, dih):
    """(quads (m, 4) int64 atom indices, labels [(type, residue's first atom)]) of the ``dih`` torsions of the ``sel``
    residues, residue by residue and, within a residue, in the order of ``dih``.  A torsion is skipped when one of its
    atoms is missing or when it needs a neighbour residue that is not the adjacent residue of the same chain and
    segid."""
    _check_types(dih)
    res = residues(mol, sel)
    name, resname = column(mol, "name", ""), column(mol, "resname", "")
    chain, segid = column(mol, "chain", ""), column(mol, "segid", "")
    lookup = []
    for atoms in res:
        names = {}
        for a in atoms:
            names.setdefault(str(name[a]), int(a))  # the first atom of a repeated name (alternative locations)
        lookup.append(names)

    def neighbour(r, off):
        s = r + off
        if s < 0 or s >= len(res):
            return None
        a, b = res[r][0], res[s][0]
        return s if chain[a] == chain[b] and segid[a] == segid[b] else None

    quads, labels = [], []
    for r, atoms in enumerate(res):
        rn = str(resname[atoms[0]])
        rn = ALIASES.get(rn, rn)
        for d in dih:
            if d in BACKBONE:
                spec = BACKBONE[d]
            elif rn in CHI[d]:
                spec = tuple((0, n) for n in CHI[d][rn].split())
            else:
                continue
            q = []
            for off, n in spec:
                s = r if off == 0 else neighbour(r, off)
                if s is None:
                    break
                a = lookup[s].get(n)
                if a is None and (rn, n) in ALT_NAMES:
                    a = lookup[s].get(ALT_NAMES[(rn, n)])
                if a is None:
                    break
                q.append(a)
            if len(q) == 4:
                quads.append(q)
                labels.append((d, int(atoms[0])))
    return np.array(quads, dtype=np.int64).reshape(-1, 4), labels


class MetricDihedral(Projection):
    """Dihedral angles of the ``protsel`` residues: ``project`` returns (numFrames, 2m) float32 with ``sincos`` (columns
    sin, cos interleaved per dihedral: sin d0, cos d0, sin d1, ...) or (numFrames, m) float32 angles in radians.

    Rules:

    - ``dih`` names the torsion types: ``phi`` (C(i-1) N CA C), ``psi`` (N CA C N(i+1)), ``omega`` (CA(i-1) C(i-1) N CA)
      and ``chi1`` - ``chi5`` from the standard per-residue side-chain table in this module (``CHI``): ILE uses CG1 and
      CD1 (chi1 N CA CB CG1, chi2 CA CB CG1 CD1; CHARMM's CD is accepted for CD1), LEU chi2 uses CD1, HIS chi2 uses ND1,
      VAL chi1 CG1, THR chi1 OG1.  HID, HIE, HIP, HSD, HSE and HSP use the HIS entries; CYX and CYM use CYS; ASH, GLH and
      LYN use ASP, GLU and LYS.  GLY and ALA have no chi.
    - Residues are runs of consecutive ``protsel`` atoms with the same resid, insertion code, chain and segid, in atom
      order.  phi and omega need the previous residue, psi the next one: the neighbour is the adjacent residue in that
      order, and the dihedral is skipped when the neighbour does not exist (first / last residue) or lies in another
      chain or segid.  A gap in the residue numbering is not a break.
    - A dihedral whose four atoms are not all present is skipped; a repeated atom name uses the first such atom.
    - Columns go residue by residue, and within a residue in the order of ``dih``.
    - Angles are computed on the coordinates as given: no wrapping and no minimum image, so a dihedral across a periodic
      boundary is the one of the unwrapped coordinates.  Sign: IUPAC (see :func:`moleculekit_b200.dihedral.dihedralAngle`).
    - A degenerate dihedral (three collinear atoms in any orientation, or coincident middle atoms: b0 x b1 or b1 x b2
      exactly zero) gives angle 0, (sin, cos) = (0, 1); a non-finite coordinate NaN.
    - ``getMapping``: one row per column, ``type`` "dihedral", ``atomIndexes`` the four atoms, ``description``
      "Sine of {type} angle of {resname} {resid}", "Cosine of ..." or, without ``sincos``, "Angle of ...".
    - An empty ``protsel`` raises ``RuntimeError`` ("Protein selection resulted in 0 atoms."); an unknown type
      ``ValueError``.

    Not confirmed against a moleculekit checkout: the interleaved column order, the residue-major order of the
    columns, the mapping text, the variant residue names and CHARMM's ILE CD, treating a residue-numbering gap as
    connected, and skipping (rather than raising on) a missing atom.  The reference documents no minimum image for this
    projection, and none is applied here.  Custom quadruples (the reference's ``Dihedral`` objects) are not accepted.
    """

    def __init__(self, dih=("psi", "phi"), sincos=True, protsel="protein"):
        super().__init__()
        self._dih = tuple(dih)
        _check_types(self._dih)
        self._sincos = bool(sincos)
        self._protsel = protsel
        self.device = None  # CUDA device for project(); None = current device

    def _calculateMolProp(self, mol, props="all"):
        props = ("dihedrals",) if props == "all" else props
        res = {}
        if "dihedrals" in props:
            res["dihedrals"] = select_dihedrals(mol, nonempty(mol, self._protsel, "Protein"), self._dih)
        return res

    def project(self, mol) -> np.ndarray:
        """(numFrames, 2m) float32 sin / cos pairs, or (numFrames, m) float32 angles in radians."""
        import torch

        from ..dihedral import dihedrals_device
        from .. import _lib

        quads, _ = self._getMolProp(mol, "dihedrals")
        F, m = mol.coords.shape[2], quads.shape[0]
        nv = 2 if self._sincos else 1
        if F == 0 or m == 0:
            return np.zeros((F, nv * m), np.float32)
        atoms, rows = np.unique(quads, return_inverse=True)
        dev = _lib.device(self.device)
        d = torch.from_numpy(np.ascontiguousarray(mol.coords[atoms], dtype=np.float32)).to(dev)
        d_quads = torch.from_numpy(rows.reshape(m, 4).astype(np.int32)).to(dev)
        return dihedrals_device(d, d_quads, self._sincos).cpu().numpy()

    def getMapping(self, mol):
        from pandas import DataFrame

        quads, labels = self._getMolProp(mol, "dihedrals")
        resname, resid = column(mol, "resname", ""), column(mol, "resid", 0)
        kinds = ("Sine", "Cosine") if self._sincos else ("Angle",)
        types, indexes, desc = [], [], []
        for q, (d, a) in zip(quads, labels):
            for kind in kinds:
                types.append("dihedral")
                indexes.append(q.copy())
                desc.append(f"{kind} of {d} angle of {resname[a]} {resid[a]}")
        return DataFrame({"type": types, "atomIndexes": indexes, "description": desc})
