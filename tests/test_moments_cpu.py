"""Group moments without a GPU: the float64 oracle (tests/moments_oracle.py) on analytic geometry, the feature functions
that turn K20 moments into MetricGyration / MetricSphericalCoordinate rows, the mass rule, and the constructor defaults,
mappings and selection errors of both projections (all checked before any device work)."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import moments_oracle as mo


def _rows(P):
    """(F, k, 3) points -> (F, 3k) rows, X block | Y block | Z block"""
    P = np.asarray(P, dtype=np.float64)
    return np.ascontiguousarray(np.transpose(P, (0, 2, 1)).reshape(P.shape[0], -1))


def _ring(R, n=12, centre=(0.0, 0.0, 0.0)):
    a = 2 * np.pi * np.arange(n) / n
    return np.stack([R * np.cos(a), R * np.sin(a), np.zeros(n)], axis=1) + np.asarray(centre)


def test_oracle_ring_gives_radius_and_components():
    R = 3.5
    rows = _rows(_ring(R)[None])
    g = mo.gyration(rows, np.ones(12))
    assert np.allclose(g, [[R, R / np.sqrt(2), R / np.sqrt(2), 0.0]], rtol=1e-14, atol=1e-14)
    # a rigid translation leaves every component unchanged; a rotation keeps rg
    moved = _rows(np.stack([_ring(R), _ring(R, centre=(40.0, -7.0, 3.0))]))
    assert np.allclose(mo.gyration(moved, np.full(12, 2.0)), g[[0, 0]], rtol=1e-12, atol=1e-12)
    rot = _ring(R) @ Rotation.random(random_state=4).as_matrix().T
    assert np.isclose(mo.gyration(_rows(rot[None]), np.ones(12))[0, 0], R, rtol=1e-13)


def test_oracle_moments_weights_and_groups():
    P = np.array([[[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 0.0, 6.0], [5.0, 5.0, 5.0]]])
    m = mo.moments(_rows(P), [1.0, 3.0, 2.0, 1.0], [0, 2, 4])
    assert m.shape == (1, 2, 6)
    assert np.allclose(m[0, 0], [1.5, 0, 0, 0.75, 0, 0])  # weights 1 and 3 at x = 0 and 2
    assert np.allclose(m[0, 1], [5 / 3, 5 / 3, 17 / 3, 50 / 9, 50 / 9, 2 / 9])
    sph = mo.spherical(_rows(P), [0, 1], [3])
    x = np.array([4.0, 5.0, 5.0])
    assert np.allclose(sph, [[np.linalg.norm(x), np.arccos(5 / np.linalg.norm(x)), np.arctan2(5, 4)]])


def test_gyration_features_match_oracle():
    from moleculekit_b200.projections.metricgyration import gyration_features

    rng = np.random.default_rng(2)
    P = rng.normal(0, 4, size=(5, 30, 3))
    w = rng.uniform(1, 16, size=30)
    rows = _rows(P)
    got = gyration_features(mo.moments(rows, w)[:, 0])
    assert got.dtype == np.float32 and got.shape == (5, 4)
    assert np.array_equal(got, mo.gyration(rows, w).astype(np.float32))


def _sph_moments(x):
    """(F, 2, 6) moments with the reference centre at the origin and the target centre at x"""
    m = np.zeros((len(x), 2, 6))
    m[:, 0, :3] = [1.0, -2.0, 0.5]
    m[:, 1, :3] = np.asarray(x, dtype=np.float64) + m[:, 0, :3]
    return m


def test_spherical_features_quadrants_poles_and_origin():
    from moleculekit_b200.projections.metricsphericalcoordinate import spherical_features

    x = [[1, 1, 0], [-1, 1, 0], [-1, -1, 0], [1, -1, 0], [0, 0, 2], [0, 0, -3], [0, 0, 0]]
    got = spherical_features(_sph_moments(x))
    assert got.dtype == np.float32 and got.shape == (7, 3)
    q = np.pi / 4
    assert np.allclose(got[:4, 2], np.float32([q, 3 * q, -3 * q, -q]))  # phi in all four quadrants
    assert np.allclose(got[:4, 1], np.float32(np.pi / 2)) and np.allclose(got[:4, 0], np.float32(np.sqrt(2)))
    assert got[4].tolist() == [2.0, 0.0, 0.0]  # north pole
    assert got[5, 0] == 3.0 and got[5, 1] == np.float32(np.pi) and got[5, 2] == 0.0  # south pole
    assert got[6, 0] == 0.0 and np.isnan(got[6, 1]) and got[6, 2] == 0.0  # r = 0: theta NaN, phi 0 (numpy)
    rng = np.random.default_rng(5)
    X = rng.normal(0, 10, size=(40, 3))
    rows = _rows(np.stack([np.zeros((40, 3)), X], axis=1))
    assert np.allclose(spherical_features(_sph_moments(X)), mo.spherical(rows, [0], [1]), rtol=1e-6, atol=1e-6)


def _mol(F=3, n=12, seed=0, masses=None, element=None):
    from moleculekit_b200.molecule_lite import MolLite

    rng = np.random.default_rng(seed)
    names = {"protein": np.arange(n) < n - 2, "protein and name CA": np.arange(n) % 3 == 0,
             "sel": np.isin(np.arange(n), [1, 2, 5, 9]), "lig": np.arange(n) >= n - 2}
    mol = MolLite(rng.normal(0, 5, size=(n, 3, F)).astype(np.float32), named_selections=names,
                  element=element if element is not None else ["C", "N", "O", "S"] * (n // 4),
                  resname=[f"R{i % 4}" for i in range(n)], name=[f"A{i}" for i in range(n)], resid=np.arange(n) // 3)
    if masses is not None:
        mol.masses = np.asarray(masses, dtype=np.float32)
    return mol


def test_mass_rule():
    from moleculekit_b200.elements import ELEMENT_DATA
    from moleculekit_b200.projections.metricgyration import selection_masses

    idx = np.array([1, 2, 5, 9])
    element_masses = [ELEMENT_DATA[e][0] for e in ("N", "O", "N", "N")]
    got = selection_masses(_mol(), idx)
    assert got.dtype == np.float64 and np.array_equal(got, np.float32(element_masses).astype(np.float64))
    own = np.arange(12, dtype=np.float32) + 0.5
    assert np.array_equal(selection_masses(_mol(masses=own), idx), own[idx].astype(np.float64))
    zero = np.zeros(12, np.float32)
    zero[0] = 7.0  # masses outside the selection do not count
    assert np.array_equal(selection_masses(_mol(masses=zero), idx), np.float32(element_masses).astype(np.float64))
    with pytest.raises(KeyError):
        selection_masses(_mol(element=["C", "Xx", "O", "S"] * 3), idx)


def test_metricgyration_defaults_mapping_and_errors():
    from moleculekit_b200.projections.metricgyration import MetricGyration

    ref = _mol(seed=1)
    ref.frame = 2
    m = MetricGyration("sel", refmol=ref)
    assert m._trajalnsel == "protein and name CA" and m._centersel == "protein" and m._pbc
    assert np.array_equal(m._refalnsel, ref.atomselect("protein and name CA"))  # refalnstr defaults to trajalnstr
    assert np.array_equal(m._refcoords[:, :, 0], ref.coords[:, :, 2])
    assert MetricGyration("sel")._refmol is None
    mol = _mol()
    mp = m.getMapping(mol)
    assert mp["type"].tolist() == ["gyration"] * 4
    assert [a.tolist() for a in mp["atomIndexes"]] == [[1, 2, 5, 9]] * 4
    assert mp["description"].tolist() == ["Radius of gyration", "x component", "y component", "z component"]
    assert MetricGyration("sel", pbc=False).project(_mol(F=0)).shape == (0, 4)
    assert MetricGyration("sel", refmol=ref).project(_mol(F=0)).shape == (0, 4)

    with pytest.raises(RuntimeError, match="Atom selection resulted in 0 atoms"):
        MetricGyration(np.zeros(12, bool), pbc=False).project(mol)
    with pytest.raises(RuntimeError, match="Atom selection resulted in 0 atoms"):
        MetricGyration(np.zeros(12, bool), pbc=False).project(_mol(F=0))  # checked with zero frames too
    with pytest.raises(RuntimeError, match="Reference alignment selection resulted in 0 atoms"):
        MetricGyration("sel", refmol=ref, trajalnstr=np.zeros(12, bool))
    with pytest.raises(RuntimeError, match="Alignment selection resulted in 0 atoms"):
        MetricGyration("sel", refmol=ref, trajalnstr=np.zeros(12, bool), refalnstr="protein").project(mol)
    with pytest.raises(RuntimeError, match="Centering selection resulted in 0 atoms"):
        MetricGyration("sel", centerstr=np.zeros(12, bool)).project(mol)
    with pytest.raises(RuntimeError, match=r"alignment selections .* differ in size: 4 and 10"):
        MetricGyration("sel", refmol=ref, refalnstr="protein", pbc=False).project(mol)
    with pytest.raises(KeyError):
        MetricGyration("sel", pbc=False).project(_mol(element=["C", "Xx", "O", "S"] * 3))


def test_metricsphericalcoordinate_defaults_mapping_and_errors():
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate

    ref = _mol(seed=1)
    ref.frame = 1
    m = MetricSphericalCoordinate(ref, "lig", "sel")
    assert m._trajalnsel == "protein and name CA" and m._centersel == "protein" and m._pbc
    assert np.array_equal(m._refalnsel, ref.atomselect("protein and name CA"))
    assert np.array_equal(m._refcoords[:, :, 0], ref.coords[:, :, 1])
    mol = _mol()
    mp = m.getMapping(mol)
    assert mp["type"].tolist() == ["sphericalcoordinate"] * 3 and mp["description"].tolist() == ["r", "theta", "phi"]
    assert [a.tolist() for a in mp["atomIndexes"]] == [[1, 2, 5, 9, 10, 11]] * 3  # refcom atoms, then targetcom
    sel, off = m._layout({"refcom": mol.atomselect("sel"), "targetcom": mol.atomselect("protein")})
    assert sel.tolist() == [1, 2, 5, 9] + list(range(10)) and off.tolist() == [0, 4, 14]  # overlap is fine
    assert MetricSphericalCoordinate(ref, "lig", "sel").project(_mol(F=0)).shape == (0, 3)

    with pytest.raises(ValueError, match="refmol"):
        MetricSphericalCoordinate(None, "lig", "sel")
    with pytest.raises(RuntimeError, match="Target COM selection resulted in 0 atoms"):
        MetricSphericalCoordinate(ref, np.zeros(12, bool), "sel", pbc=False).project(mol)
    with pytest.raises(RuntimeError, match="Reference COM selection resulted in 0 atoms"):
        MetricSphericalCoordinate(ref, "lig", np.zeros(12, bool), pbc=False).project(_mol(F=0))
    with pytest.raises(RuntimeError, match="Reference alignment selection resulted in 0 atoms"):
        MetricSphericalCoordinate(ref, "lig", "sel", trajalnstr=np.zeros(12, bool))
    with pytest.raises(RuntimeError, match="Alignment selection resulted in 0 atoms"):
        MetricSphericalCoordinate(ref, "lig", "sel", trajalnstr=np.zeros(12, bool), refalnstr="protein").project(mol)
    with pytest.raises(RuntimeError, match="Centering selection resulted in 0 atoms"):
        MetricSphericalCoordinate(ref, "lig", "sel", centerstr=np.zeros(12, bool)).project(mol)
    with pytest.raises(RuntimeError, match=r"alignment selections .* differ in size: 4 and 10"):
        MetricSphericalCoordinate(ref, "lig", "sel", refalnstr="protein", pbc=False).project(mol)


def test_project_sharded_accepts_both_metrics(monkeypatch):
    """frames are independent: project_sharded passes both metrics through to project (world size 1 here)"""
    from moleculekit_b200.projections.metricgyration import MetricGyration
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate
    from moleculekit_b200.sharding import project_sharded

    mol = _mol(F=5)
    for m in (MetricGyration("sel", pbc=False), MetricSphericalCoordinate(_mol(seed=1), "lig", "sel", pbc=False)):
        monkeypatch.setattr(m, "project", lambda view: np.full((view.numFrames, 2), 7.0, np.float32))
        assert project_sharded(m, mol).shape == (5, 2)
