"""GPU parity of K20 (weighted per-frame group moments) and the MetricGyration / MetricSphericalCoordinate drop-ins:
moments within 1e-12 relative of the two-pass float64 oracle (tests/moments_oracle.py) on the device's own aligned
coordinates, bits that depend only on the selection, groups and weights, groups of many segments (and more segments
than a grid dimension holds), NaN confined to its (frame, group), the argument checks, and the projections within 1e-6
relative of the float64 oracle on the float64 superposition rounded to float32."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import moments_oracle as mo
from oracle import coords_oracle as co

pytestmark = pytest.mark.gpu


def _t(a, dev, dtype=None):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).to(dev)


def _bits(t):
    import torch

    return t.contiguous().view(torch.int64)


def _f32(rows64):
    return rows64.astype(np.float32).astype(np.float64)


def _rotated(frame, seed):
    G = Rotation.random(random_state=seed).as_matrix()
    return (frame.astype(np.float64) @ G + [12.5, -30.0, 7.25]).astype(np.float32)


def _close_moments(got, want, scale):
    """means within 1e-12 relative (or 1e-12 of the coordinate scale); variances within 1e-12 relative (or the square of
    that absolute bound: the oracle's mean of a one-atom group can differ from the atom in the last bit)"""
    got = np.asarray(got)
    assert got.shape == want.shape
    assert np.allclose(got[..., :3], want[..., :3], rtol=1e-12, atol=1e-12 * scale)
    assert np.allclose(got[..., 3:], want[..., 3:], rtol=1e-12, atol=(1e-12 * scale) ** 2)


def _setup(g_traj):
    import torch
    from moleculekit_b200.align import superpose_device

    dev = torch.device("cuda:0")
    X = g_traj["coords"]
    ca = g_traj["sel_masks"][0]
    d = _t(X, dev)
    ref = _rotated(X[:, :, 7], 2)[:, :, None]
    d_ca = _t(np.where(ca)[0], dev, np.int32)
    rec, st = superpose_device(d, d_ca, _t(ref, dev), d_ca)
    assert int(st.sum()) == 0
    return dev, X, d, ref, rec


def _groups(g_traj):
    """unequal, overlapping groups: heavy protein atoms (5 segments), the ligand, one atom, the CA atoms (again)"""
    ca, lig, noh = g_traj["sel_masks"][0], g_traj["resname"] == "MOL", g_traj["sel_masks"][2]
    parts = [np.where(noh)[0], np.where(lig)[0], np.array([1234]), np.where(ca)[0]]
    return np.concatenate(parts), np.concatenate([[0], np.cumsum([p.size for p in parts])]).astype(np.int64)


@pytest.mark.parametrize("with_ref", [False, True])
def test_moments_match_oracle_on_device_coordinates(g_traj, with_ref):
    import torch
    from moleculekit_b200.coords import coordinates_device, frame_moments_device

    dev, X, d, ref, rec = _setup(g_traj)
    records = rec if with_ref else None
    idx, off = _groups(g_traj)
    sel = _t(idx, dev, np.int32)
    w = np.random.default_rng(1).uniform(1.0, 16.0, idx.size)
    got = frame_moments_device(d, sel, records, weights=w, groups=off)
    assert got.shape == (20, 4, 6) and got.dtype == torch.float64 and got.device == dev
    rows = coordinates_device(d, sel, records).cpu().numpy().astype(np.float64)
    _close_moments(got.cpu().numpy(), mo.moments(rows, w, off), np.abs(rows).max())
    assert bool((got[:, 2, 3:] == 0).all())  # a one-atom group has no spread
    assert torch.equal(got[:, 2, :3], torch.from_numpy(co.as_points(rows)[:, off[2]]).to(dev))
    # unit weights given explicitly give the bits of weights=None
    plain = frame_moments_device(d, sel, records, groups=off)
    assert torch.equal(_bits(plain), _bits(frame_moments_device(d, sel, records, weights=np.ones(idx.size), groups=off)))
    _close_moments(plain.cpu().numpy(), mo.moments(rows, None, off), np.abs(rows).max())
    # the whole trajectory as one group: 9 segments of at most 512 positions
    all_sel = _t(np.arange(X.shape[0]), dev, np.int32)
    one = frame_moments_device(d, all_sel, records)
    rows_all = coordinates_device(d, all_sel, records).cpu().numpy().astype(np.float64)
    _close_moments(one.cpu().numpy(), mo.moments(rows_all), np.abs(rows_all).max())
    assert np.array_equal(d.cpu().numpy(), X)  # the trajectory is not modified


def test_moments_bits_depend_only_on_selection_groups_and_weights(g_traj):
    import torch
    from moleculekit_b200.coords import frame_moments_device

    dev, X, d, ref, rec = _setup(g_traj)
    idx, off = _groups(g_traj)
    sel = _t(idx, dev, np.int32)
    w = np.random.default_rng(2).uniform(1.0, 16.0, idx.size)
    whole = frame_moments_device(d, sel, rec, weights=w, groups=off)
    assert torch.equal(_bits(whole), _bits(frame_moments_device(d, sel, rec, weights=w, groups=off)))
    f0, f1 = 3, 17
    view = frame_moments_device(d[:, :, f0:f1], sel, rec[f0:f1], weights=w, groups=off)
    fl = _t(np.arange(f0, f1), dev, np.int32)
    listed = frame_moments_device(d, sel, rec[f0:f1], fl, weights=w, groups=off)
    assert torch.equal(_bits(view), _bits(listed)) and torch.equal(_bits(view), _bits(whole[f0:f1]))
    perm = np.array([19, 4, 11, 0, 7])
    picked = frame_moments_device(d, sel, rec[perm], _t(perm, dev, np.int32), weights=w, groups=off)
    assert torch.equal(_bits(picked), _bits(whole[perm]))
    # weights and offsets may arrive as CUDA tensors too (copied back to the host)
    dw = frame_moments_device(d, sel, rec, weights=_t(w, dev), groups=_t(off, dev))
    assert torch.equal(_bits(dw), _bits(whole))
    empty = frame_moments_device(d, sel, rec[:0], _t(np.zeros(0), dev, np.int32), weights=w, groups=off)
    assert empty.shape == (0, 4, 6)


def test_moments_many_segments_and_grid_limit():
    """more than 60 000 positions in one group (137 segments), and more than 65 535 segments in one call"""
    import torch
    from moleculekit_b200.align import superpose_device
    from moleculekit_b200.coords import coordinates_device, frame_moments_device

    dev = torch.device("cuda:0")
    N, F = 70000, 33
    g = torch.Generator(device=dev).manual_seed(11)
    base = torch.randn((N, 3, 1), generator=g, device=dev) * 25 + 60
    X = (base + torch.randn((N, 3, F), generator=g, device=dev) * 0.8).contiguous()
    aln = _t(np.arange(0, N, 50), dev, np.int32)
    rec, st = superpose_device(X, aln, X[:, :, 5:6], aln)
    assert int(st.sum()) == 0
    sel = _t(np.random.default_rng(3).permutation(N), dev, np.int32)
    w = np.random.default_rng(4).uniform(1.0, 16.0, N)
    got = frame_moments_device(X, sel, rec, weights=w)
    rows = coordinates_device(X, sel, rec).cpu().numpy().astype(np.float64)
    _close_moments(got.cpu().numpy(), mo.moments(rows, w), np.abs(rows).max())
    # 66 000 one-atom groups and one group of the other 4 000: 66 008 segments, so the grid strides over segments
    off = np.concatenate([np.arange(66001), [N]]).astype(np.int64)
    few = frame_moments_device(X[:, :, :3], sel, rec[:3], weights=w, groups=off)
    assert few.shape == (3, 66001, 6)
    pts = co.as_points(rows[:3])
    assert torch.equal(few[:, :66000, :3], torch.from_numpy(pts[:, :66000]).to(dev))
    assert bool((few[:, :66000, 3:] == 0).all())
    _close_moments(few[:, 66000].cpu().numpy(), mo.moments(rows[:3, :], w, off[[0, -2, -1]])[:, 1],
                   np.abs(rows).max())


def test_moments_nan_stays_in_its_frame_and_group(g_traj):
    import torch
    from moleculekit_b200.coords import frame_moments_device

    dev, X, d, ref, rec = _setup(g_traj)
    idx, off = _groups(g_traj)
    sel = _t(idx, dev, np.int32)
    clean = frame_moments_device(d, sel, rec, groups=off)
    atom = int(np.where(g_traj["sel_masks"][2] & ~g_traj["sel_masks"][0])[0][2])  # heavy, not CA: group 0, not the fit
    assert np.count_nonzero(idx == atom) == 1
    Xn = X.copy()
    Xn[atom, 1, 9] = np.nan
    got = frame_moments_device(_t(Xn, dev), sel, rec, groups=off)
    nan = torch.isnan(got)
    assert bool(nan[9, 0].all()) and int(nan.sum()) == 6
    keep = ~nan
    assert torch.equal(got[keep], clean[keep])


def test_moments_argument_checks(g_traj):
    from moleculekit_b200 import _lib
    from moleculekit_b200.coords import frame_moments_device

    dev, X, d, ref, rec = _setup(g_traj)
    sel = _t(np.arange(10), dev, np.int32)
    cases = [([0, 6, 4, 10], None, "decrease"), ([0, 4, 4, 10], None, "empty"), ([0, 4, 9], None, "0 to n_sel"),
             ([1, 4, 10], None, "0 to n_sel"), ([0, 4, 10], [1.0] * 4 + [0.0] * 6, "weights of group 1"),
             ([0, 4, 10], [1.0] * 4 + [-1.0, 1.0] * 3, "weights of group 1"), ([0], None, "n_groups")]
    for off, w, msg in cases:
        with pytest.raises(_lib.MkbError, match=msg):
            frame_moments_device(d, sel, rec, weights=w, groups=np.array(off))


def _names(g_traj):
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    return {"protein and name CA": ca, "protein and noh": noh, "protein": g_traj["sel_masks"][5],
            "resname MOL": g_traj["resname"] == "MOL"}


def _lite(coords, g=None, **kw):
    from moleculekit_b200.molecule_lite import MolLite

    if g is not None:
        kw.update(resid=g["resid"], resname=g["resname"], name=g["name"], element=g["element"],
                  named_selections=_names(g))
    return MolLite(coords, **kw)


def test_projections_traj20(g_traj):
    from moleculekit_b200.elements import masses_of
    from moleculekit_b200.projections.metricgyration import MetricGyration
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate

    X = g_traj["coords"]
    ca, noh, lig = g_traj["sel_masks"][0], g_traj["sel_masks"][2], g_traj["resname"] == "MOL"
    idx = np.where(noh)[0]
    masses = masses_of(g_traj["element"][idx]).astype(np.float64)
    ref = _lite(np.stack([X[:, :, 0], _rotated(X[:, :, 7], 2)], axis=2), g_traj, frame=1)
    R = ref.coords[:, :, 1:2]
    mol = _lite(X.copy(), g_traj)
    aligned = MetricGyration("protein and noh", refmol=ref, pbc=False).project(mol)
    plain = MetricGyration("protein and noh", pbc=False).project(mol)
    assert aligned.dtype == np.float32 and aligned.shape == (20, 4)
    want = mo.gyration(_f32(co.coordinates(X, idx, R, ca, ca)), masses)
    assert np.allclose(aligned, want, rtol=1e-6, atol=0)
    assert np.allclose(plain, mo.gyration(co.coordinates(X, idx), masses), rtol=1e-6, atol=0)
    assert np.allclose(aligned[:, 0], plain[:, 0], rtol=1e-6, atol=0)  # rg does not depend on the orientation
    assert not np.allclose(aligned[:, 1:], plain[:, 1:], rtol=1e-3)  # its components do

    ci, li = np.where(ca)[0], np.where(lig)[0]
    sph = MetricSphericalCoordinate(ref, "resname MOL", "protein and name CA", pbc=False).project(mol)
    assert sph.dtype == np.float32 and sph.shape == (20, 3)
    rows = _f32(co.coordinates(X, np.concatenate([ci, li]), R, ca, ca))
    want = mo.spherical(rows, np.arange(ci.size), np.arange(ci.size, ci.size + li.size))
    assert np.allclose(sph, want, rtol=1e-6, atol=1e-6)
    assert np.array_equal(mol.coords, X)  # project does not modify the molecule


def test_projections_pbc_wrap(g_wrap):
    """pbc=True wraps on the device exactly as Molecule.wrap around `centerstr`: the expected values are the oracle on
    the reference's own wrapped coordinates; the selections hold solvent atoms the wrap moves"""
    from moleculekit_b200.projections.metricgyration import MetricGyration
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate

    g = g_wrap
    X, W = g["coords"], g["ref_wrapped"]
    N = X.shape[0]
    protein = np.zeros(N, bool)
    protein[g["centersel"]] = True
    aln = protein & (np.arange(N) % 4 == 0)
    moved = np.where(np.any(X != W, axis=(1, 2)) & ~protein)[0][:400]
    sel = protein & (np.arange(N) % 3 == 0)
    sel[moved] = True
    solvent = np.zeros(N, bool)
    solvent[moved[:40]] = True
    idx = np.where(sel)[0]
    names = {"protein": protein, "aln": aln, "sel": sel, "solvent": solvent}
    masses = 1.0 + (np.arange(N) % 7).astype(np.float32)
    ref = _lite(X[:, :, 0], named_selections=names)
    mol = _lite(X.copy(), box=g["box"], bonds=g["bonds"], named_selections=names)
    mol.masses = masses
    m64 = masses[idx].astype(np.float64)
    got = MetricGyration("sel", refmol=ref, trajalnstr="aln").project(mol)
    assert np.allclose(got, mo.gyration(_f32(co.coordinates(W, idx, ref.coords, aln, aln)), m64), rtol=1e-6, atol=0)
    got = MetricGyration("sel").project(mol)
    assert np.allclose(got, mo.gyration(co.coordinates(W, idx), m64), rtol=1e-6, atol=0)
    assert not np.allclose(got, mo.gyration(co.coordinates(X, idx), m64), rtol=1e-3)  # the wrap matters
    pi, si = np.where(protein)[0], np.where(solvent)[0]
    sph = MetricSphericalCoordinate(ref, "solvent", "protein", trajalnstr="aln").project(mol)
    rows = _f32(co.coordinates(W, np.concatenate([pi, si]), ref.coords, aln, aln))
    want = mo.spherical(rows, np.arange(pi.size), np.arange(pi.size, pi.size + si.size))
    assert np.allclose(sph, want, rtol=1e-6, atol=1e-6)
    assert np.array_equal(mol.coords, X)


def test_projections_nonfinite_and_shards(g_traj):
    from moleculekit_b200.projections.metricgyration import MetricGyration
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate
    from moleculekit_b200.sharding import _frame_view, project_sharded

    X = g_traj["coords"]
    ca = g_traj["sel_masks"][0]
    ref = _lite(_rotated(X[:, :, 3], 5), g_traj)
    mol = _lite(X.copy(), g_traj)
    metrics = [MetricGyration("protein and noh", refmol=ref, pbc=False), MetricGyration("protein", pbc=False),
               MetricSphericalCoordinate(ref, "resname MOL", "protein and name CA", pbc=False)]
    for m in metrics:
        whole = m.project(mol)
        parts = np.concatenate([m.project(_frame_view(mol, 0, 7)), m.project(_frame_view(mol, 7, 20))])
        assert np.array_equal(whole.view(np.uint32), parts.view(np.uint32))
        assert np.array_equal(project_sharded(m, mol).view(np.uint32), whole.view(np.uint32))
    Xn = X.copy()
    Xn[int(np.where(ca)[0][3]), 1, 5] = np.nan
    for m in (metrics[0], metrics[2]):
        with pytest.raises(np.linalg.LinAlgError):
            m.project(_lite(Xn.copy(), g_traj))
    lig_atom = int(np.where(g_traj["resname"] == "MOL")[0][2])
    Xn = X.copy()
    Xn[lig_atom, 0, 12] = np.nan
    got = metrics[2].project(_lite(Xn, g_traj))
    assert np.isnan(got[12]).all() and np.isnan(got).sum() == 3
    assert np.array_equal(np.delete(got, 12, 0), np.delete(metrics[2].project(mol), 12, 0))
