"""GPU parity of K16 (dihedral angles) against the float64 oracle (oracle/dihedral_oracle.py).

Bounds: a sine or cosine is within one float32 ulp of the float64 value rounded to float32 (never below 1e-12: the
kernel's float64 expression and the oracle's differ by a few float64 ulps, which only matters next to zero).  An angle
with |angle| < pi - 1e-6 is within one float32 ulp the same way; closer to +-pi the sign of a nearly-zero y decides
between +pi and -pi, so those angles are compared as the difference wrapped into [-pi, pi), bounded by one float32 ulp
of pi (2.4e-7 rad)."""
import numpy as np
import pytest

from oracle import dihedral_oracle as do

pytestmark = pytest.mark.gpu
ALL = ("phi", "psi", "omega", "chi1", "chi2", "chi3", "chi4", "chi5")
PI_ULP = float(np.spacing(np.float32(np.pi)))


def _t(a, dev, dtype=None):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).to(dev)


def _bits(t):
    import torch

    return t.contiguous().view(torch.int32)


def _check_sincos(got, want64):
    w32 = want64.astype(np.float32)
    assert got.dtype == np.float32 and got.shape == w32.shape
    nan = np.isnan(w32)
    assert np.array_equal(np.isnan(got), nan)
    err = np.abs(got.astype(np.float64) - w32.astype(np.float64))[~nan]
    ok = err <= np.maximum(np.spacing(np.abs(w32[~nan])).astype(np.float64), 1e-12)
    assert ok.all(), f"{np.count_nonzero(~ok)} values off by up to {err[~ok].max():.3e}"


def _check_angles(got, want64):
    w32 = want64.astype(np.float32)
    assert got.dtype == np.float32 and got.shape == w32.shape
    nan = np.isnan(w32)
    assert np.array_equal(np.isnan(got), nan)
    g, w, w3 = got[~nan].astype(np.float64), want64[~nan], w32[~nan].astype(np.float64)
    inner = np.abs(w) < np.pi - 1e-6
    err = np.abs(g - w3)[inner]
    ok = err <= np.maximum(np.spacing(np.abs(w3[inner]).astype(np.float32)).astype(np.float64), 1e-12)
    assert ok.all(), f"{np.count_nonzero(~ok)} angles off by up to {err[~ok].max():.3e}"
    wrapped = np.abs((g - w + np.pi) % (2 * np.pi) - np.pi)[~inner]
    assert (wrapped <= PI_ULP).all(), f"angles near +-pi off by {wrapped.max():.3e} rad (wrapped)"
    assert (np.abs(g) <= np.float32(np.pi)).all()


def _traj20_quads(g_traj):
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricdihedral import select_dihedrals

    prot = g_traj["sel_masks"][5]
    mol = MolLite(g_traj["coords"], name=g_traj["name"], resname=g_traj["resname"], resid=g_traj["resid"],
                  chain=g_traj["chain"], segid=g_traj["segid"], named_selections={"protein": prot})
    return mol, select_dihedrals(mol, prot, ALL)[0]


def test_traj20_against_oracle(g_traj):
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda:0")
    mol, quads = _traj20_quads(g_traj)
    X = g_traj["coords"]
    d = _t(X, dev)
    q = _t(quads, dev, np.int32)
    sc = dihedrals_device(d, q, True).cpu().numpy()
    ang = dihedrals_device(d, q, False).cpu().numpy()
    assert sc.shape == (20, 2 * len(quads)) and ang.shape == (20, len(quads))
    _check_sincos(sc, do.project(X, quads, True))
    _check_angles(ang, do.project(X, quads, False))
    assert np.abs(np.abs(ang) - np.pi).min() < 0.05  # omega of trans peptides: the +-pi comparison is exercised


def test_large_seeded_system_and_shards():
    """60 000 atoms x 3 000 frames, 20 000 random quadruples: frame lists, slices and shards written through the row
    stride give the bits of the whole call, and sampled frames match the oracle"""
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda:0")
    N, F, m = 60000, 3000, 20000
    g = torch.Generator(device=dev).manual_seed(16)
    X = (torch.randn((N, 3, 1), generator=g, device=dev) * 20
         + torch.randn((N, 3, F), generator=g, device=dev) * 1.5).contiguous()
    rng = np.random.default_rng(16)
    quads = np.stack([rng.choice(N, 4, replace=False) for _ in range(m)]).astype(np.int32)
    q = _t(quads, dev)
    for sincos in (True, False):
        nv = 2 if sincos else 1
        whole = dihedrals_device(X, q, sincos)
        assert whole.shape == (F, nv * m)
        wide = torch.full((F, nv * m + 19), -1.0, device=dev)
        for f0, f1 in ((0, 1000), (1000, 1001), (1001, 2333), (2333, 3000)):
            dihedrals_device(X[:, :, f0:f1], q, sincos, out=wide[f0:f1, 7:7 + nv * m])
        assert torch.equal(_bits(wide[:, 7:7 + nv * m]), _bits(whole))
        assert bool((wide[:, :7] == -1).all()) and bool((wide[:, 7 + nv * m:] == -1).all())
        fl = _t(np.array([2999, 5, 1234, 5, 0, 77]), dev, np.int32)
        assert torch.equal(_bits(dihedrals_device(X, q, sincos, frames=fl)), _bits(whole[fl.long()]))
        sub = X[:, :, 100:400]
        assert torch.equal(_bits(dihedrals_device(sub, q, sincos)), _bits(whole[100:400]))
        sample = np.random.default_rng(1).choice(F, 8, replace=False)
        Xs = X[:, :, sample].cpu().numpy()
        want = do.project(Xs, quads, sincos)
        (_check_sincos if sincos else _check_angles)(whole[sample].cpu().numpy(), want)
    empty = dihedrals_device(X, q, True, frames=_t(np.zeros(0), dev, np.int32))
    assert empty.shape == (0, 2 * m)


def test_degenerate_and_nonfinite():
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda:0")
    P = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [2, 1, 0],       # 0-3: p0, p1, p2 collinear
                  [0, 1, 0], [0, 0, 0], [1, 0, 0], [3, 0, 0],       # 4-7: p1, p2, p3 collinear
                  [0, 1, 0], [1, 0, 0], [1, 0, 0], [2, 0, 1],       # 8-11: p1 == p2
                  [1, 0, 0], [0, 0, 0], [0, 0, 1], [0, 1, 1]],      # 12-15: +90 degrees
                 dtype=np.float32)
    F = 5
    X = np.repeat(P[:, :, None], F, axis=2).copy()
    X[13, 0, 1] = np.nan      # frame 1: the +90 quadruple has a NaN
    X[15, 2, 2] = np.inf      # frame 2: an infinity
    X[12, 1, 3] = -np.inf     # frame 3: a negative infinity
    X[0, 0, 4] = np.nan       # frame 4: NaN in a degenerate quadruple
    quads = np.arange(16, dtype=np.int32).reshape(4, 4)
    d, q = _t(X, dev), _t(quads, dev)
    sc = dihedrals_device(d, q, True).cpu().numpy()
    ang = dihedrals_device(d, q, False).cpu().numpy()
    for f in range(F):
        for j in range(3):
            if f == 4 and j == 0:
                assert np.isnan(sc[f, 0:2]).all() and np.isnan(ang[f, 0])
            else:
                assert sc[f, 2 * j:2 * j + 2].tolist() == [0.0, 1.0] and ang[f, j] == 0.0
        if f in (1, 2, 3):
            assert np.isnan(sc[f, 6:8]).all() and np.isnan(ang[f, 3])
        else:
            assert sc[f, 6:8].tolist() == [1.0, 0.0] and ang[f, 3] == np.float32(np.pi / 2)
    _check_sincos(sc, do.project(X, quads, True))
    _check_angles(ang, do.project(X, quads, False))


def test_metricdihedral_project(g_traj):
    from moleculekit_b200.projections.metricdihedral import MetricDihedral
    from moleculekit_b200.sharding import _frame_view, project_sharded

    mol, _ = _traj20_quads(g_traj)
    X = mol.coords.copy()
    for dih, sincos in ((("psi", "phi"), True), (ALL, False), (("omega", "chi2"), True)):
        m = MetricDihedral(dih=dih, sincos=sincos)
        got = m.project(mol)
        quads, _ = m._getMolProp(mol, "dihedrals")
        want = do.project(X, quads, sincos)
        assert got.shape == want.shape == (20, (2 if sincos else 1) * len(quads))
        (_check_sincos if sincos else _check_angles)(got, want)
        assert len(m.getMapping(mol)) == got.shape[1]
        # frames are independent: frame blocks projected apart give the same bits
        parts = [m.project(_frame_view(mol, a, b)) for a, b in ((0, 7), (7, 8), (8, 20))]
        assert np.array_equal(np.concatenate(parts).view(np.uint32), got.view(np.uint32))
        assert np.array_equal(project_sharded(m, mol).view(np.uint32), got.view(np.uint32))
    assert np.array_equal(mol.coords, X)  # project does not modify the molecule
