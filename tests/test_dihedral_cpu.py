"""Dihedral projection without a GPU: the float64 oracle (oracle/dihedral_oracle.py) and the host mirror
dihedralAngle on constructed geometries of known angle under rigid motions, the IUPAC sign, degenerate and non-finite
quadruples, the quadruple selection of MetricDihedral on the committed structures (3PTB and the traj20 system; the
pdb_5vl5 golden file carries no atom names, so it cannot be used), chain breaks, mapping text and column order, and the
loud failure without a device."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import dihedral_oracle as do

ALL = ("phi", "psi", "omega", "chi1", "chi2", "chi3", "chi4", "chi5")


def _quad(theta_deg):
    """four points whose dihedral is theta: p1 at the origin, p2 on +z, p0 along +x, p3 at angle theta about z"""
    t = np.deg2rad(theta_deg)
    return np.array([[1.2, 0.0, -0.4], [0.0, 0.0, 0.0], [0.0, 0.0, 1.5], [0.9 * np.cos(t), 0.9 * np.sin(t), 2.1]])


def _wrapped(a, b):
    return np.abs((np.asarray(a) - np.asarray(b) + np.pi) % (2 * np.pi) - np.pi)


@pytest.mark.parametrize("theta", [0.0, 60.0, -60.0, 90.0, -90.0, 179.999, -179.999, 180.0])
def test_known_angles_under_rigid_motion(theta):
    from moleculekit_b200.dihedral import dihedralAngle

    P0 = _quad(theta)
    rng = np.random.default_rng(int(abs(theta) * 1000) % 2**31)
    frames = [P0 @ Rotation.random(random_state=s).as_matrix().T + rng.normal(0, 30, 3) for s in range(16)]
    P = np.stack(frames, axis=2)  # (4, 3, F)
    want = np.deg2rad(theta)
    a = do.angles(P)
    assert _wrapped(a, want).max() < 1e-12
    sc = do.sincos(P)
    assert np.abs(sc - [np.sin(want), np.cos(want)]).max() < 1e-12
    for f in range(P.shape[2]):
        assert _wrapped(dihedralAngle(P[:, :, f]), want) < 1e-12
    if theta in (0.0, 60.0, -60.0, 90.0, -90.0):
        assert np.abs(a - want).max() < 1e-12  # away from +-pi the value itself, not only modulo 2 pi


def test_sign_convention():
    """Looking along p1 -> p2 (+z), p1-p0 points along +x and p2-p3 along +y: p0 turns clockwise by 90 degrees onto
    p3, so the angle is +90 (right-handed); the mirror image is -90."""
    from moleculekit_b200.dihedral import dihedralAngle

    right = np.array([[1.0, 0, 0], [0, 0, 0], [0, 0, 1], [0, 1, 1]])
    left = right * [1, -1, 1]
    assert dihedralAngle(right) == pytest.approx(np.pi / 2, abs=1e-15)
    assert dihedralAngle(left) == pytest.approx(-np.pi / 2, abs=1e-15)
    assert do.angles(right[:, :, None])[0] == pytest.approx(np.pi / 2, abs=1e-15)
    assert do.angles(left[:, :, None])[0] == pytest.approx(-np.pi / 2, abs=1e-15)
    cis = np.array([[1.0, 0, 0], [0, 0, 0], [0, 0, 1], [1, 0, 1]])
    trans = cis * [[1, 1, 1], [1, 1, 1], [1, 1, 1], [-1, 1, 1]]
    assert dihedralAngle(cis) == 0.0 and abs(dihedralAngle(trans)) == pytest.approx(np.pi, abs=1e-15)


def test_protein_backbone_sign(g_3ptb):
    """the IUPAC sign on a real structure: nearly every phi of trypsin (beta sheet and helix) is negative"""
    from moleculekit_b200.projections.metricdihedral import select_dihedrals

    mol = _lite(g_3ptb)
    quads, labels = select_dihedrals(mol, g_3ptb["sel_protein"], ("phi",))
    phi = do.project(g_3ptb["coords"], quads, False)[0]
    assert (phi < 0).mean() > 0.85


def test_degenerate_and_nonfinite():
    from moleculekit_b200.dihedral import dihedralAngle

    line = np.array([[0.0, 0, 0], [1, 0, 0], [2, 0, 0], [2, 1, 0]])          # p0, p1, p2 collinear
    tail = np.array([[0.0, 1, 0], [0, 0, 0], [1, 0, 0], [3, 0, 0]])          # p1, p2, p3 collinear
    same = np.array([[0.0, 1, 0], [1, 0, 0], [1, 0, 0], [2, 0, 1]])          # p1 == p2
    for P in (line, tail, same):
        assert dihedralAngle(P) == 0.0
        assert do.angles(P[:, :, None])[0] == 0.0
        assert do.sincos(P[:, :, None])[0].tolist() == [0.0, 1.0]
    for bad in (np.nan, np.inf, -np.inf):
        for atom in range(4):
            P = _quad(40.0)[:, :, None].copy()
            P[atom, 1, 0] = bad
            assert np.isnan(do.angles(P)[0]) and np.isnan(do.sincos(P)[0]).all()
    P = _quad(40.0)
    P[2, 0] = np.nan
    assert np.isnan(dihedralAngle(P))
    with pytest.raises(RuntimeError, match="4x3"):
        dihedralAngle(np.zeros((3, 3)))


def _lite(g, **over):
    from moleculekit_b200.molecule_lite import MolLite

    prot = g["sel_protein"] if "sel_protein" in g else g["sel_masks"][5]
    kw = dict(name=g["name"], resname=g["resname"], resid=g["resid"], chain=g["chain"], segid=g["segid"],
              named_selections={"protein": prot})
    kw.update(over)
    return MolLite(g["coords"], **kw)


def _per_type(mol, quads, labels):
    counts = {}
    for q, (d, a) in zip(quads, labels):
        key = (str(mol.resname[a]), d)
        counts[key] = counts.get(key, 0) + 1
    return counts


@pytest.mark.parametrize("which", ["3ptb", "traj20"])
def test_selection_counts(which, g_3ptb, g_traj):
    from moleculekit_b200.projections.common import residues
    from moleculekit_b200.projections.metricdihedral import ALIASES, CHI, select_dihedrals

    g = g_3ptb if which == "3ptb" else g_traj
    mol = _lite(g)
    prot = mol.atomselect("protein")
    quads, labels = select_dihedrals(mol, prot, ALL)
    q2, kinds = do.quadruples(mol.name, mol.resname, mol.resid, mol.chain, mol.segid, prot, ALL)
    assert np.array_equal(quads, q2) and [d for d, _ in labels] == kinds
    totals = {d: kinds.count(d) for d in ALL}
    if which == "3ptb":
        assert totals == dict(phi=219, psi=219, omega=219, chi1=181, chi2=108, chi3=30, chi4=15, chi5=2)
    else:
        assert totals == dict(phi=276, psi=276, omega=276, chi1=244, chi2=195, chi3=76, chi4=41, chi5=20)
    # every residue of a type with a chi_k entry has that chi exactly once; backbone torsions at most once per residue
    n_of = {}
    for r in residues(mol, prot):
        rn = str(mol.resname[r[0]])
        n_of[rn] = n_of.get(rn, 0) + 1
    counts = _per_type(mol, quads, labels)
    for (rn, d), c in counts.items():
        assert c <= n_of[rn]
        if d.startswith("chi"):
            assert ALIASES.get(rn, rn) in CHI[d]
            assert c == n_of[rn], (rn, d)  # the committed structures have complete side chains
    for rn in ("GLY", "ALA"):
        assert not any(d.startswith("chi") for (r, d) in counts if r == rn)
    # the four atoms of every torsion are distinct and, for side chains, in one residue
    assert all(len(set(q.tolist())) == 4 for q in quads)
    for q, (d, a) in zip(quads, labels):
        if d.startswith("chi"):
            assert len(set(mol.resid[q].tolist())) == 1


def test_ends_and_chain_breaks(g_3ptb):
    from moleculekit_b200.projections.common import residues
    from moleculekit_b200.projections.metricdihedral import select_dihedrals

    mol = _lite(g_3ptb)
    prot = mol.atomselect("protein")
    res = residues(mol, prot)
    quads, labels = select_dihedrals(mol, prot, ("phi", "psi", "omega"))
    first, last = int(res[0][0]), int(res[-1][0])
    assert [d for d, a in labels if a == first] == ["psi"]
    assert [d for d, a in labels if a == last] == ["phi", "omega"]
    base = {d: sum(1 for x, _ in labels if x == d) for d in ("phi", "psi", "omega")}
    cut = int(res[100][0])  # the first atom of the 101st residue
    for field in ("chain", "segid"):
        col = getattr(mol, field).copy()
        col[cut:] = "Z"
        broken = _lite(g_3ptb, **{field: col})
        q, lab = select_dihedrals(broken, prot, ("phi", "psi", "omega"))
        assert {d: sum(1 for x, _ in lab if x == d) for d in base} == {d: c - 1 for d, c in base.items()}
        side = np.asarray(getattr(broken, field))[q]
        assert (side == side[:, :1]).all(), f"a dihedral spans the {field} break"
        assert [d for d, a in lab if a == cut] == ["psi"] and [d for d, a in lab if a == int(res[99][0])] == ["phi",
                                                                                                            "omega"]


def test_mapping_and_column_order(g_3ptb):
    from moleculekit_b200.projections.metricdihedral import MetricDihedral

    mol = _lite(g_3ptb)
    m = MetricDihedral()
    assert m._dih == ("psi", "phi") and m._sincos and m._protsel == "protein"
    mp = m.getMapping(mol)
    quads, labels = m._getMolProp(mol, "dihedrals")
    assert len(mp) == 2 * len(quads) == 2 * 438
    assert set(mp["type"]) == {"dihedral"}
    assert mp["description"].tolist()[:6] == [
        "Sine of psi angle of ILE 16", "Cosine of psi angle of ILE 16",
        "Sine of psi angle of VAL 17", "Cosine of psi angle of VAL 17",
        "Sine of phi angle of VAL 17", "Cosine of phi angle of VAL 17"]
    assert [a.tolist() for a in mp["atomIndexes"][:2]] == [quads[0].tolist()] * 2
    assert [d for d, _ in labels[:4]] == ["psi", "psi", "phi", "psi"]  # residue-major, types in the order asked
    a = MetricDihedral(dih=("chi1", "phi"), sincos=False).getMapping(mol)
    assert a["description"].tolist()[:3] == ["Angle of chi1 angle of ILE 16", "Angle of chi1 angle of VAL 17",
                                             "Angle of phi angle of VAL 17"]
    with pytest.raises(ValueError, match="Unknown dihedral"):
        MetricDihedral(dih=("phi", "chi6"))
    with pytest.raises(RuntimeError, match="Protein selection resulted in 0 atoms"):
        MetricDihedral(protsel=np.zeros(mol.numAtoms, bool)).getMapping(mol)
    empty = _lite(dict(g_3ptb, coords=g_3ptb["coords"][:, :, :0]))
    assert MetricDihedral().project(empty).shape == (0, 876)


def test_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from moleculekit_b200 import _lib
    from moleculekit_b200.dihedral import dihedrals_device
    from moleculekit_b200.projections.metricdihedral import MetricDihedral

    X = torch.zeros((4, 3, 2))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        dihedrals_device(X, torch.arange(4, dtype=torch.int32).reshape(1, 4), True)
    from moleculekit_b200.molecule_lite import MolLite

    mol = MolLite(np.zeros((4, 3, 2), np.float32), name=["C", "N", "CA", "C"], resid=[1, 2, 2, 2])
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        MetricDihedral(dih=("phi",), protsel="all").project(mol)
