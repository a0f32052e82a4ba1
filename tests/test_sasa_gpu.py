"""GPU parity of K17 (Shrake-Rupley SASA) against the C restatement of mdtraj's loop (tests/sasa_oracle.c): every area
is compared bit for bit (int32 views), since the result is a count of float32 decisions."""
import numpy as np
import pytest

import sasa_oracle as so

pytestmark = pytest.mark.gpu


def _t(a, dtype):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to("cuda:0")


def _same(got, want):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    diff = got.view(np.int32) != want.view(np.int32)
    assert not diff.any(), f"{int(diff.sum())} areas differ, e.g. {got[diff][:4]} vs {want[diff][:4]}"


def _device(X, radii, query, sphere, groups=None, frames=None):
    from moleculekit_b200.sasa import sasa_device

    out = sasa_device(_t(X, np.float32), _t(np.arange(X.shape[0]), np.int32), _t(radii, np.float32),
                      _t(query, np.int32), _t(sphere, np.float32), None if groups is None else _t(groups, np.int64),
                      None if frames is None else _t(frames, np.int32))
    return out.cpu().numpy()


def _mol(g, coords=None):
    from moleculekit_b200.molecule_lite import MolLite

    prot = g["sel_protein"] if "sel_protein" in g else g["sel_masks"][5]
    return MolLite(g["coords"] if coords is None else coords, element=g["element"], name=g["name"],
                   resname=g["resname"], resid=g["resid"], chain=g["chain"], segid=g["segid"],
                   named_selections={"protein": prot})


def _oracle_project(m, mol):
    """the oracle on the filtersel atoms, columns chosen as MetricSasa chooses them"""
    env, radii, query, groups, _ = m._getMolProp(mol, "sasa")
    return so.sasa(mol.coords[env], radii, query, m._sphere, groups)


@pytest.mark.parametrize("filtersel", ["all", "protein"])
@pytest.mark.parametrize("mode", ["atom", "residue"])
def test_3ptb(g_3ptb, filtersel, mode):
    from moleculekit_b200.projections.metricsasa import MetricSasa

    mol = _mol(g_3ptb)
    m = MetricSasa(sel="protein", mode=mode, filtersel=filtersel)
    got = m.project(mol)
    _same(got, _oracle_project(m, mol))
    assert got.shape[1] == (1629 if mode == "atom" else len(m.getMapping(mol)))
    assert (got > 0).any() and (got == 0).any()


@pytest.mark.parametrize("mode", ["atom", "residue"])
def test_traj20_all_frames(g_traj, mode):
    from moleculekit_b200.projections.metricsasa import MetricSasa
    from moleculekit_b200.sharding import _frame_view, project_sharded

    mol = _mol(g_traj)
    m = MetricSasa(sel="protein", mode=mode)
    got = m.project(mol)
    assert got.shape[0] == 20
    _same(got, _oracle_project(m, mol))
    parts = [m.project(_frame_view(mol, a, b)) for a, b in ((0, 7), (7, 8), (8, 20))]
    _same(np.concatenate(parts), got)
    _same(project_sharded(m, mol), got)
    assert np.array_equal(mol.coords, g_traj["coords"])


@pytest.mark.parametrize("npts", [1, 31, 33, 960, 4000])
@pytest.mark.parametrize("probe", [0.0, 1.4])
def test_sphere_sizes_and_probe(g_3ptb, npts, probe):
    from moleculekit_b200.sasa import sasa_radii, sphere_points

    X = g_3ptb["coords"]
    radii = sasa_radii(g_3ptb["element"], probe)
    S = sphere_points(npts)
    q = np.arange(0, X.shape[0], 3)
    _same(_device(X, radii, q, S), so.sasa(X, radii, q, S))


def test_dense_clouds_overflow_the_buffer():
    """4 000 atoms in a 3 nm box with radii up to 0.5 nm: every atom has several hundred neighbours, far more than the
    per-warp buffer holds, so the lists are walked in pieces and gathered again for each pass"""
    from moleculekit_b200.sasa import sphere_points

    rng = np.random.default_rng(17)
    n, F = 4000, 2
    X = rng.uniform(0, 30, size=(n, 3, F)).astype(np.float32)
    radii = rng.uniform(0.2, 0.5, size=n).astype(np.float32)
    S = sphere_points(600)
    q = rng.choice(n, 300, replace=False)
    got = _device(X, radii, q, S)
    _same(got, so.sasa(X, radii, q, S))
    assert (got > 0).any()


def test_near_tangent_points():
    """neighbours placed so that sphere points sit within a few float32 ulp of the neighbour's surface, on both sides:
    the decision d2 < R^2 must be taken with the reference's roundings"""
    from moleculekit_b200.sasa import sphere_points

    rng = np.random.default_rng(3)
    S = sphere_points(97)
    Ri, Rk = np.float32(0.31), np.float32(0.27)
    rows, radii = [], []
    for c in range(40):
        centre = rng.uniform(-5, 5, 3)
        rows.append(centre)
        radii.append(Ri)
        for j in rng.choice(97, 6, replace=False):
            p = centre + float(Ri) * S[j].astype(np.float64)
            u = rng.normal(size=3)
            u /= np.linalg.norm(u)
            if u @ S[j] < 0:
                u = -u
            rows.append(p + float(Rk) * u)
            radii.append(Rk)
    X = (np.array(rows) * 10).astype(np.float32)
    steps = rng.integers(-4, 5, size=X.shape)
    for _ in range(4):  # walk each coordinate a few ulp either way
        X = np.where(steps > 0, np.nextafter(X, np.float32(np.inf)), np.where(steps < 0, np.nextafter(X, -np.inf), X))
        steps = steps - np.sign(steps)
    X = np.ascontiguousarray(X[:, :, None].repeat(3, axis=2))
    X[:, :, 1] = np.nextafter(X[:, :, 0], np.float32(np.inf))
    X[:, :, 2] = np.nextafter(X[:, :, 0], -np.float32(np.inf))
    radii = np.array(radii, np.float32)
    q = np.arange(0, X.shape[0], 7)
    _same(_device(X, radii, q, S), so.sasa(X, radii, q, S))


def test_nan_coordinates(g_3ptb):
    from moleculekit_b200.sasa import sasa_radii, sphere_points

    X = np.repeat(g_3ptb["coords"], 3, axis=2)
    X[10, 0, 0] = np.nan
    X[11:14, 1, 1] = np.nan
    X[500, 2, 2] = np.inf
    radii = sasa_radii(g_3ptb["element"], 1.4)
    S = sphere_points(960)
    q = np.arange(X.shape[0])
    got = _device(X, radii, q, S)
    _same(got, so.sasa(X, radii, q, S))
    full = np.float32(np.float32(np.float32(np.float32(4 * np.pi / 960) * radii[10]) * radii[10]) * np.float32(960))
    assert got[0, 10] == np.float32(full * np.float32(100))


def test_more_than_65535_query_atoms():
    """one frame of a 70 000-atom lattice solute, every atom queried; the oracle checks a sample including the last
    atoms"""
    from moleculekit_b200 import workloads
    from moleculekit_b200.sasa import sphere_points

    rng = np.random.default_rng(5)
    n = 70000
    X = workloads._sphere_lattice(rng, n, 60.0, np.zeros(3), spacing=1.5)[:, :, None]
    radii = np.where(rng.random(n) < 0.5, 0.26, 0.31).astype(np.float32)
    S = sphere_points(960)
    got = _device(X, radii, np.arange(n), S)
    sample = np.concatenate([rng.choice(n, 300, replace=False), np.arange(n - 50, n)])
    _same(got[:, sample], so.sasa(X, radii, sample, S))


def test_chunk_boundary(g_traj):
    """enough frames that the call crosses a frame-chunk boundary: the frames either side match the oracle and every
    frame equals a single-frame call"""
    from moleculekit_b200.sasa import chunk_frames, sasa_radii, sphere_points

    X0 = g_traj["coords"]
    prot = np.where(g_traj["sel_masks"][5])[0]
    fc = chunk_frames(X0.shape[0], prot.size, 0)
    F = fc + 5
    X = np.ascontiguousarray(np.tile(X0, (1, 1, F // 20 + 1))[:, :, :F])
    radii = sasa_radii(g_traj["element"], 1.4)
    S = sphere_points(960)
    whole = _device(X, radii, prot, S)
    _same(whole[fc - 1:fc + 1], so.sasa(X, radii, prot, S, frames=[fc - 1, fc]))
    from moleculekit_b200.sasa import sasa_device

    d, env, r, q, s = (_t(X, np.float32), _t(np.arange(X.shape[0]), np.int32), _t(radii, np.float32),
                       _t(prot, np.int32), _t(S, np.float32))
    for k in range(F):
        one = sasa_device(d, env, r, q, s, frames=_t([k], np.int32)).cpu().numpy()
        assert np.array_equal(one.view(np.int32), whole[k:k + 1].view(np.int32)), f"frame {k}"


def test_frames_slices_and_shards(g_traj):
    import torch
    from moleculekit_b200.sasa import sasa_device, sasa_radii, sphere_points

    X = g_traj["coords"]
    prot = np.where(g_traj["sel_masks"][5])[0]
    radii = sasa_radii(g_traj["element"], 1.4)
    S = sphere_points(240)
    d, env, r, q, s = (_t(X, np.float32), _t(np.arange(X.shape[0]), np.int32), _t(radii, np.float32),
                       _t(prot, np.int32), _t(S, np.float32))
    groups = _t([0, 100, 100, 2000, prot.size], np.int64)
    for g in (None, groups):
        whole = sasa_device(d, env, r, q, s, g)
        cols = whole.shape[1]
        wide = torch.full((20, cols + 11), -1.0, device="cuda:0")
        for f0, f1 in ((0, 6), (6, 7), (7, 20)):
            sasa_device(d[:, :, f0:f1], env, r, q, s, g, out=wide[f0:f1, 5:5 + cols])
        assert torch.equal(wide[:, 5:5 + cols].contiguous().view(torch.int32), whole.view(torch.int32))
        assert bool((wide[:, :5] == -1).all()) and bool((wide[:, 5 + cols:] == -1).all())
        fl = _t([19, 3, 3, 0, 11], np.int32)
        got = sasa_device(d, env, r, q, s, g, frames=fl)
        assert torch.equal(got.view(torch.int32), whole[fl.long()].view(torch.int32))
        assert sasa_device(d, env, r, q, s, g, frames=_t([], np.int32)).shape == (0, cols)
    want = so.sasa(X, radii, prot, S, groups=[0, 100, 100, 2000, prot.size])
    _same(sasa_device(d, env, r, q, s, groups).cpu().numpy(), want)
    assert want[:, 1].tolist() == [0.0] * 20  # an empty group is a float32 zero


def test_coincident_atoms_raise(g_3ptb):
    from moleculekit_b200.projections.metricsasa import MetricSasa
    from moleculekit_b200.sasa import CoincidentAtomsError

    X = np.repeat(g_3ptb["coords"], 4, axis=2)
    X[700, :, 2] = X[40, :, 2]
    X[900, :, 3] = X[41, :, 3] + np.float32(1e-6)
    mol = _mol(g_3ptb, X)
    with pytest.raises(ValueError, match="frame 2") as e:
        MetricSasa(sel="protein").project(mol)
    assert isinstance(e.value, CoincidentAtomsError) and e.value.atoms == (40, 700)
    with pytest.raises(so.CoincidentAtoms):
        so.sasa(X[:, :, 2:3], np.full(X.shape[0], 0.3, np.float32), [40], np.eye(3, dtype=np.float32))
    # pairs outside the computed atoms are not checked
    sel = np.zeros(X.shape[0], bool)
    sel[100:200] = True
    got = MetricSasa(sel=sel).project(mol)
    assert got.shape == (4, 100)
