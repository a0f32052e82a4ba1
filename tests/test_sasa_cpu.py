"""SASA projection without a GPU: the sphere table, the C oracle (tests/sasa_oracle.c) against an independent numpy
float32 restatement and against analytic areas, MetricSasa's column selection, mapping and errors, and the loud
failure without a device."""
import numpy as np
import pytest

import sasa_oracle as so


def _numpy_areas(X_nm, radii, sphere):
    """float32 restatement without the neighbour cycling: a point is accessible when no neighbour buries it"""
    f32 = np.float32
    n, N = X_nm.shape[0], sphere.shape[0]
    c = f32(4.0 * np.pi / N)
    out = np.zeros(n, np.float32)
    for i in range(n):
        d = X_nm[i] - X_nm
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        rc = radii[i] + radii
        nb = np.where((d2 < rc * rc) & (np.arange(n) != i))[0]
        P = X_nm[i] + radii[i] * sphere  # (N, 3) float32, each product and sum rounded on its own
        e = P[:, None, :] - X_nm[nb][None, :, :]
        e2 = (e[..., 0] * e[..., 0] + e[..., 1] * e[..., 1]) + e[..., 2] * e[..., 2]
        buried = (e2 < (radii[nb] * radii[nb])[None, :]).any(axis=1)
        out[i] = c * radii[i] * radii[i] * f32(N - int(buried.sum()))
    return out


def test_sphere_table():
    from moleculekit_b200.sasa import sphere_points

    for n in (1, 2, 31, 33, 960, 4000):
        S = sphere_points(n)
        assert S.shape == (n, 3) and S.dtype == np.float32
        assert np.abs(np.linalg.norm(S.astype(np.float64), axis=1) - 1).max() < 4e-7
        assert (np.diff(S[:, 1]) > 0).all()
    assert np.array_equal(sphere_points(960), sphere_points(960))
    for bad in (0, -3, 65537):
        with pytest.raises(ValueError):
            sphere_points(bad)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_against_numpy(seed):
    from moleculekit_b200.sasa import sphere_points

    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 200))
    X = rng.uniform(0, 1.2 + n ** (1 / 3) * 0.25, size=(n, 3)).astype(np.float32)
    radii = rng.uniform(0.1, 0.35, size=n).astype(np.float32)
    S = sphere_points(int(rng.choice([1, 31, 100, 960])))
    got = so.areas_nm(X, radii, np.arange(n), S)
    want = _numpy_areas(X, radii, S)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert (got > 0).any() and (got < want.max()).any()


def test_oracle_analytic():
    from moleculekit_b200.sasa import sphere_points

    f32 = np.float32
    S = sphere_points(960)
    c = f32(4 * np.pi / 960)
    R = f32(0.31)
    iso = so.areas_nm(np.zeros((1, 3), np.float32), np.array([R]), [0], S)[0]
    assert iso == f32(f32(f32(c * R) * R) * f32(960))
    # an atom enclosed by a shell of large atoms has no accessible point
    shell = sphere_points(60).astype(np.float64) * 0.3
    X = np.concatenate([np.zeros((1, 3)), shell]).astype(np.float32)
    radii = np.concatenate([[0.15], np.full(60, 0.25)]).astype(np.float32)
    assert so.areas_nm(X, radii, [0], S)[0] == 0
    # two overlapping spheres: each loses a cap of area 2 pi R h, h = R - (d^2 + R^2 - r^2) / 2d
    R1, R2, d = 0.3, 0.25, 0.4
    X = np.array([[0, 0, 0], [d, 0, 0]], np.float32)
    a = so.areas_nm(X, np.array([R1, R2], np.float32), [0, 1], sphere_points(4000))
    for got, Ra, Rb in ((a[0], R1, R2), (a[1], R2, R1)):
        h = Ra - (d * d + Ra * Ra - Rb * Rb) / (2 * d)
        want = 4 * np.pi * Ra * Ra - 2 * np.pi * Ra * h
        assert abs(got - want) / want < 5e-3


def _lite(g, **kw):
    from moleculekit_b200.molecule_lite import MolLite

    return MolLite(g["coords"], element=g["element"], name=g["name"], resname=g["resname"], resid=g["resid"],
                   chain=g["chain"], segid=g["segid"], named_selections={"protein": g["sel_protein"]}, **kw)


def test_columns_and_mapping(g_3ptb):
    from moleculekit_b200.projections.common import residues
    from moleculekit_b200.projections.metricsasa import MetricSasa

    mol = _lite(g_3ptb)
    prot = g_3ptb["sel_protein"]
    m = MetricSasa(sel="protein", mode="atom")
    env, radii, query, groups, cols = m._getMolProp(mol, "sasa")
    assert np.array_equal(env, np.arange(mol.numAtoms)) and groups is None
    assert np.array_equal(query, np.where(prot)[0]) and len(cols) == prot.sum()
    assert radii.dtype == np.float32 and radii[0] == np.float32(np.float32(0.155) + np.float32(0.14))
    mp = m.getMapping(mol)
    assert len(mp) == prot.sum() and mp["type"][0] == "SASA" and mp["description"][0] == "SASA of ILE 16 N"
    # residue mode over filtersel = protein: every protein residue, its atoms in order
    m = MetricSasa(sel="protein", mode="residue", filtersel="protein")
    env, radii, query, groups, cols = m._getMolProp(mol, "sasa")
    res = residues(mol, prot)
    assert np.array_equal(env, np.where(prot)[0]) and len(cols) == len(res)
    assert np.array_equal(env[query], np.concatenate(res))
    assert np.array_equal(np.diff(groups), [len(r) for r in res])
    mp = m.getMapping(mol)
    assert mp["description"][0] == "SASA of residue ILE 16" and np.array_equal(mp["atomIndexes"][0], res[0])
    # a residue counts when one of its atoms is in sel; its column adds every filtersel atom of it
    sel = np.zeros(mol.numAtoms, bool)
    sel[[5, 6, 40]] = True
    m = MetricSasa(sel=sel, mode="residue")
    _, _, query, groups, cols = m._getMolProp(mol, "sasa")
    assert len(cols) == 2 and 5 in cols[0] and 40 in cols[1] and groups[-1] == len(query)


def test_residue_sums_in_oracle():
    f32 = np.float32
    X = np.array([[[0], [0], [0]], [[30], [0], [0]], [[60], [0], [0]]], np.float32)
    radii = np.array([0.2, 0.3, 0.25], np.float32)
    S = np.array([[1, 0, 0], [0, 1, 0]], np.float32)
    a = so.areas_nm(X[:, :, 0] / f32(10), radii, [0, 1, 2], S)
    got = so.sasa(X, radii, [0, 1, 2], S, groups=[0, 2, 3])
    assert got[0, 0] == f32(f32(a[0] + a[1]) * f32(100)) and got[0, 1] == f32(a[2] * f32(100))


def test_errors(g_3ptb):
    from moleculekit_b200.projections.metricsasa import MetricSasa
    from moleculekit_b200.sasa import sasa_radii

    mol = _lite(g_3ptb)
    with pytest.raises(ValueError, match="no SASA radius"):
        sasa_radii(["C", "Xx", "Qq"], 1.4)
    bad = _lite(dict(g_3ptb, element=np.where(np.arange(1701) == 3, "Xx", g_3ptb["element"])))
    with pytest.raises(ValueError, match="Xx"):
        MetricSasa().project(bad)
    with pytest.raises(ValueError, match="outside filtersel"):
        MetricSasa(sel="all", filtersel="protein").getMapping(mol)
    with pytest.raises(RuntimeError, match="0 atoms"):
        MetricSasa(sel=np.zeros(1701, bool)).getMapping(mol)
    with pytest.raises(ValueError, match="mode"):
        MetricSasa(mode="chain")
    with pytest.raises(ValueError, match="numSpherePoints"):
        MetricSasa(numSpherePoints=0)
    assert sasa_radii(["CL", "cl", " Cl"], 0.0).tolist() == [np.float32(0.181)] * 3
    empty = _lite(dict(g_3ptb, coords=g_3ptb["coords"][:, :, :0]))
    assert MetricSasa().project(empty).shape == (0, 1629)


def test_no_cpu_fallback(g_3ptb):
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from moleculekit_b200 import _lib
    from moleculekit_b200.projections.metricsasa import MetricSasa
    from moleculekit_b200.sasa import sasa_device, sphere_points

    z = torch.zeros
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        sasa_device(z((4, 3, 2)), z(4, dtype=torch.int32), z(4), z(1, dtype=torch.int32),
                    torch.from_numpy(sphere_points(10)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        MetricSasa().project(_lite(g_3ptb))
