"""Float64 restatement of the reference's dihedral projection -- TEST INFRASTRUCTURE ONLY.

  moleculekit/dihedral.py                       dihedralAngle: the torsion of four points
  moleculekit/projections/metricdihedral.py     the protein's phi / psi / omega / chi quadruples and the sin / cos columns

Written apart from the package (which never imports this module): the angle is the textbook normal-vector form
(atan2 of |b1| b0 . (b1 x b2) over (b0 x b1) . (b1 x b2)), not the projected-vector form the kernel evaluates, and the
quadruple selection walks the atoms once with its own copy of the side-chain table.
"""
from __future__ import annotations

import numpy as np

SIDECHAIN = {  # IUPAC-IUB 1970 chi1 .. chi5 atoms per residue
    "ARG": ["N CA CB CG", "CA CB CG CD", "CB CG CD NE", "CG CD NE CZ", "CD NE CZ NH1"],
    "ASN": ["N CA CB CG", "CA CB CG OD1"],
    "ASP": ["N CA CB CG", "CA CB CG OD1"],
    "CYS": ["N CA CB SG"],
    "GLN": ["N CA CB CG", "CA CB CG CD", "CB CG CD OE1"],
    "GLU": ["N CA CB CG", "CA CB CG CD", "CB CG CD OE1"],
    "HIS": ["N CA CB CG", "CA CB CG ND1"],
    "ILE": ["N CA CB CG1", "CA CB CG1 CD1"],
    "LEU": ["N CA CB CG", "CA CB CG CD1"],
    "LYS": ["N CA CB CG", "CA CB CG CD", "CB CG CD CE", "CG CD CE NZ"],
    "MET": ["N CA CB CG", "CA CB CG SD", "CB CG SD CE"],
    "PHE": ["N CA CB CG", "CA CB CG CD1"],
    "PRO": ["N CA CB CG", "CA CB CG CD"],
    "SER": ["N CA CB OG"],
    "THR": ["N CA CB OG1"],
    "TRP": ["N CA CB CG", "CA CB CG CD1"],
    "TYR": ["N CA CB CG", "CA CB CG CD1"],
    "VAL": ["N CA CB CG1"],
}
VARIANT = {"HID": "HIS", "HIE": "HIS", "HIP": "HIS", "HSD": "HIS", "HSE": "HIS", "HSP": "HIS", "CYX": "CYS",
           "CYM": "CYS", "ASH": "ASP", "GLH": "GLU", "LYN": "LYS"}


def _xy(P):
    """(x, y) with angle = atan2(y, x): b0 = p1 - p0, b1 = p2 - p1, b2 = p3 - p2, y = |b1| b0.(b1 x b2),
    x = (b0 x b1).(b1 x b2); both exactly 0 where a normal vector b0 x b1 or b1 x b2 is the zero vector (three
    collinear points: y alone would be rounding noise there)"""
    b0, b1, b2 = P[1] - P[0], P[2] - P[1], P[3] - P[2]
    with np.errstate(invalid="ignore"):
        n1 = np.cross(b0, b1, axis=0)
        n2 = np.cross(b1, b2, axis=0)
        x, y = (n1 * n2).sum(0), np.sqrt((b1 * b1).sum(0)) * (b0 * n2).sum(0)
    degenerate = ~n1.any(axis=0) | ~n2.any(axis=0)
    return np.where(degenerate, 0.0, x), np.where(degenerate, 0.0, y)


def angles(P):
    """P (4, 3, F) -> (F,) float64 dihedral angles in radians (IUPAC sign); 0 where the quadruple is degenerate (a
    normal vector b0 x b1 or b1 x b2 is exactly zero, so x = y = 0), NaN where a coordinate is not finite."""
    P = np.asarray(P, dtype=np.float64)
    x, y = _xy(P)
    a = np.where((x == 0) & (y == 0), 0.0, np.arctan2(y, x))
    a[~np.isfinite(P).all(axis=(0, 1))] = np.nan
    return a


def sincos(P):
    """(F, 2) float64 (sin, cos) of :func:`angles` from the unnormalised components: (0, 1) when degenerate."""
    P = np.asarray(P, dtype=np.float64)
    x, y = _xy(P)
    r = np.hypot(x, y)
    with np.errstate(invalid="ignore", divide="ignore"):
        out = np.stack([np.where(r > 0, y / r, 0.0), np.where(r > 0, x / r, 1.0)], axis=1)
    out[~np.isfinite(P).all(axis=(0, 1))] = np.nan
    return out


def project(coords, quads, use_sincos):
    """(F, m) angles or (F, 2m) interleaved sin, cos of the quadruples over coords (N, 3, F)"""
    X = np.asarray(coords, dtype=np.float64)
    if use_sincos:
        cols = [sincos(X[q]) for q in quads]
        return np.concatenate(cols, axis=1) if cols else np.zeros((X.shape[2], 0))
    return np.stack([angles(X[q]) for q in quads], axis=1) if len(quads) else np.zeros((X.shape[2], 0))


def quadruples(name, resname, resid, chain, segid, sel, dih, insertion=None):
    """(m, 4) int64 atom indices and the type of each, residue by residue in atom order and types in ``dih`` order.
    A residue is a run of selected atoms sharing (resid, insertion, chain, segid); phi / omega use the previous run and
    psi the next, only within one (chain, segid); missing atoms skip the torsion."""
    n = len(name)
    ins = [""] * n if insertion is None else insertion
    runs, prev = [], None
    for i in range(n):
        if not sel[i]:
            continue
        key = (resid[i], ins[i], chain[i], segid[i])
        if key != prev:
            runs.append({"key": key, "resname": resname[i], "atoms": {}})
            prev = key
        runs[-1]["atoms"].setdefault(str(name[i]), i)

    def atom(r, nm):
        if r < 0 or r >= len(runs):
            return None
        a = runs[r]["atoms"].get(nm)
        if a is None and nm == "CD1" and VARIANT.get(runs[r]["resname"], runs[r]["resname"]) == "ILE":
            a = runs[r]["atoms"].get("CD")
        return a

    def linked(r, s):
        return 0 <= s < len(runs) and runs[r]["key"][2:] == runs[s]["key"][2:]

    out, kinds = [], []
    for r, run in enumerate(runs):
        rn = VARIANT.get(run["resname"], run["resname"])
        for d in dih:
            if d == "phi":
                q = [atom(r - 1, "C") if linked(r, r - 1) else None, atom(r, "N"), atom(r, "CA"), atom(r, "C")]
            elif d == "psi":
                q = [atom(r, "N"), atom(r, "CA"), atom(r, "C"), atom(r + 1, "N") if linked(r, r + 1) else None]
            elif d == "omega":
                ok = linked(r, r - 1)
                q = [atom(r - 1, "CA") if ok else None, atom(r - 1, "C") if ok else None, atom(r, "N"), atom(r, "CA")]
            else:
                k = int(d[3:]) - 1
                chis = SIDECHAIN.get(rn, [])
                if k >= len(chis):
                    continue
                q = [atom(r, nm) for nm in chis[k].split()]
            if all(a is not None for a in q):
                out.append(q)
                kinds.append(d)
    return np.array(out, dtype=np.int64).reshape(-1, 4), kinds


def collinear_quads(n, seed):
    """(4, 3, n) float64 of float32 quadruples, three points collinear in each, none axis-aligned: half with
    p0, p1, p2 collinear, half with p1, p2, p3; half as power-of-two multiples of a random point (4d, 2d, d), half as an
    arithmetic progression a, a + d, a + 2d of multiples of 1/64, both exact in float32"""
    rng = np.random.default_rng(seed)
    out = np.empty((4, 3, n))
    for k in range(n):
        if k % 4 < 2:
            d = rng.normal(0, 10, 3).astype(np.float32)
            line = [4 * d, 2 * d, d]
        else:
            a = rng.integers(-4000, 4000, 3) / 64.0
            d = rng.integers(-300, 300, 3) / 64.0
            while np.count_nonzero(d) < 3:
                d = rng.integers(-300, 300, 3) / 64.0
            line = [a, a + d, a + 2 * d]
        other = rng.normal(0, 10, 3)
        pts = line + [other] if k % 2 == 0 else [other] + line[::-1]
        out[:, :, k] = np.array(pts, dtype=np.float32)
    return out
