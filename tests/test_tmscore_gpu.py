"""GPU parity of K19 (TM-score) against the C restatement of the search (tests/tmscore_oracle.c): TM-scores and RMSDs
are bit-identical as float64, so a fit that differs in its last bit is caught even when it does not change the maximum."""
import numpy as np
import pytest

import tmscore_oracle as to

pytestmark = pytest.mark.gpu


def _t(a, dtype):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to("cuda:0")


def _device(X, Y, frames=None):
    """(tm, rmsd) of tmscore_device for model rows X (n, 3, F) against reference rows Y (m, 3), pairs in row order"""
    from moleculekit_b200.tmscore import tmscore_device

    tm, rmsd = tmscore_device(_t(X, np.float32), _t(np.arange(X.shape[0]), np.int32), _t(Y[:, :, None], np.float32),
                              _t(np.arange(Y.shape[0]), np.int32), None if frames is None else _t(frames, np.int32))
    return tm.cpu().numpy(), rmsd.cpu().numpy()


def _same(got, want):
    for g, w, what in zip(got, want, ("TM-scores", "RMSDs")):
        assert g.shape == w.shape and np.array_equal(np.isnan(g), np.isnan(w)), what
        ok = np.isnan(w) | (g.view(np.int64) == w.view(np.int64))
        assert ok.all(), f"{what} differ at {np.where(~ok)[0][:5].tolist()}: {g[~ok][:3]} vs {w[~ok][:3]}"


def _check(X, Y, frames=None):
    got = _device(X, Y, frames)
    _same(got, to.tmscore(X, Y, frames))
    return got


def _ca(g):
    return np.ascontiguousarray(g["coords"][g["name"] == "CA"])


def test_traj20_all_frames(g_traj):
    X = _ca(g_traj)
    tm, rmsd = _check(X, X[:, :, 0])
    assert tm[0] == 1.0 and (tm[1:] < 1).all() and (tm > 0.3).all()


def test_traj20_noisy_frames(g_traj):
    """100 frames with 0.1-3 A of Gaussian noise: cut sets widen, converge and cycle differently in every frame"""
    X = _ca(g_traj)
    rng = np.random.default_rng(11)
    Xn = np.ascontiguousarray(np.tile(X, (1, 1, 5)))
    sigma = rng.uniform(0.1, 3.0, size=Xn.shape[2]).astype(np.float32)
    Xn += (rng.normal(size=Xn.shape) * sigma).astype(np.float32)
    tm, _ = _check(Xn, X[:, :, 0])
    assert len(set(tm.tolist())) == 100 and tm.min() < 0.7 and tm.max() > 0.95


@pytest.mark.parametrize("direction", ["traj20_on_3ptb", "3ptb_on_traj20"])
def test_traj20_against_3ptb(g_traj, g_3ptb, direction):
    """unequal selections (277 and 224 CA atoms) of unrelated proteins: L = 224, normalised by the reference's count"""
    A, B = _ca(g_traj)[:, :, :4], _ca(g_3ptb)[:, :, 0]
    X, Y = (A, B) if direction == "traj20_on_3ptb" else (B[:, :, None], A[:, :, 0])
    tm, _ = _check(X, Y)
    assert (tm < 0.4).all()


@pytest.mark.parametrize("L", [1, 2, 3, 4, 5, 31, 32, 33])
def test_small_selections(g_traj, L):
    X = _ca(g_traj)[:L]
    rng = np.random.default_rng(L)
    Xn = X + (rng.normal(size=X.shape) * 1.5).astype(np.float32)
    _check(np.ascontiguousarray(Xn), X[:, :, 0])


def test_multichain_2216_pairs(g_traj):
    """8 copies of the protein 100 A apart as one selection: 2 216 pairs, 9 004 seeds per frame"""
    X = _ca(g_traj)
    big = np.concatenate([X[:, :, [0, 13]] + np.float32(100 * c) for c in range(8)])
    rng = np.random.default_rng(2)
    model = big + (rng.normal(size=big.shape) * 1.0).astype(np.float32)
    tm, _ = _check(np.ascontiguousarray(model), big[:, :, 0])
    assert big.shape[0] >= 2000


def test_nonfinite_frames(g_traj):
    X = np.ascontiguousarray(_ca(g_traj)[:, :, :6]).copy()
    X[17, 0, 2] = np.nan
    X[200, 2, 4] = np.inf
    tm, rmsd = _check(X, _ca(g_traj)[:, :, 0])
    assert np.isnan(tm[[2, 4]]).all() and np.isnan(rmsd[[2, 4]]).all()
    assert np.isfinite(tm[[0, 1, 3, 5]]).all() and np.isfinite(rmsd[[0, 1, 3, 5]]).all()


def test_nonfinite_reference_raises(g_traj):
    X = _ca(g_traj)
    Y = X[:, :, 0].copy()
    Y[5, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        _device(X[:, :, :2], Y)


def test_frames_slices_and_shards(g_traj):
    import torch
    from moleculekit_b200.tmscore import tmscore_device

    X = _ca(g_traj)
    d, ref = _t(X, np.float32), _t(X[:, :, :1], np.float32)
    sel = _t(np.arange(277), np.int32)
    whole = [a.cpu().numpy() for a in tmscore_device(d, sel, ref, sel)]
    _same(whole, to.tmscore(X, X[:, :, 0]))
    fr = [19, 3, 0, 11]
    _same([a.cpu().numpy() for a in tmscore_device(d, sel, ref, sel, _t(fr, np.int32))], [w[fr] for w in whole])
    _same([a.cpu().numpy() for a in tmscore_device(d[:, :, 5:12], sel, ref, sel)], [w[5:12] for w in whole])
    strided = list(range(1, 20, 3))
    _same([a.cpu().numpy() for a in tmscore_device(d, sel, ref, sel, _t(strided, np.int32))],
          [w[strided] for w in whole])
    empty = tmscore_device(d, sel, ref, sel, _t([], np.int32))
    assert empty[0].shape == (0,) and empty[0].dtype == torch.float64


def test_pair_cap(g_traj):
    """a selection at the cap runs; one pair more raises ValueError before any launch"""
    from moleculekit_b200.tmscore import max_pairs, tmscore_device

    cap = max_pairs()
    assert cap >= 5000
    X = _ca(g_traj)[:, :, 0]
    copies = -(-cap // 277) + 1
    big = np.concatenate([X + np.float32(100 * c) for c in range(copies)])
    d = _t(big[:, :, None], np.float32)
    tm, rmsd = tmscore_device(d, _t(np.arange(cap), np.int32), d, _t(np.arange(cap), np.int32))
    assert tm.cpu().item() == 1.0 and rmsd.cpu().item() < 1e-9
    with pytest.raises(ValueError, match="at most"):
        tmscore_device(d, _t(np.arange(cap + 1), np.int32), d, _t(np.arange(cap + 1), np.int32))


@pytest.mark.parametrize("n, m", [(277, 277), (200, 277), (277, 200)])
def test_moltmscore_pairing(g_traj, n, m):
    """CA filtering in atom order, pairs k < min(n, m), normalised by m, nali = min(n, m)"""
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tmscore import molTMscore

    g = g_traj
    ca = np.where(g["name"] == "CA")[0]
    sel_mol = np.zeros(g["coords"].shape[0], bool)
    sel_mol[ca[:n]] = True
    sel_mol[ca[0] + 1] = True  # a non-CA atom in the selection is dropped
    sel_ref = np.zeros_like(sel_mol)
    sel_ref[ca[:m]] = True
    mol = MolLite(g["coords"][:, :, :5], name=g["name"])
    ref = MolLite(g["coords"], name=g["name"], frame=3)
    tm, rmsd, nali = molTMscore(mol, ref, sel_mol, sel_ref)
    L = min(n, m)
    want = to.tmscore(g["coords"][ca[:L], :, :5], g["coords"][ca[:m], :, 3])
    _same((tm, rmsd), want)
    assert nali.tolist() == [L] * 5
    assert tm[3] == L / m


@pytest.mark.parametrize("cell", ["orthorhombic", "triclinic"])
def test_metric_pbc_wrap(cell, request):
    """pbc=True wraps on the device around `centerstr`: project equals the oracle on the fixture's own wrapped
    coordinates.  Some solvent atoms that the wrap moves are named CA, so a missing wrap changes the result."""
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metrictmscore import MetricTMscore

    if cell == "orthorhombic":
        g = request.getfixturevalue("g_wrap")
        W, bonds, angles = g["ref_wrapped"], g["bonds"], None
    else:
        g = request.getfixturevalue("g_tric")
        W, angles = g["ref_rectangular"], g["boxangles"]
        gr = g["groups"].astype(np.int64)
        bonds = np.concatenate([np.stack([np.arange(a, b - 1), np.arange(a + 1, b)], 1)
                                for a, b in zip(gr[:-1], gr[1:]) if b - a > 1]).astype(np.uint32)
    X = g["coords"]
    N = X.shape[0]
    protein = np.zeros(N, bool)
    protein[g["centersel"]] = True
    moved = np.where(np.any(X != W, axis=(1, 2)) & ~protein)[0][:60]
    assert moved.size == 60
    names = np.array(["X"] * N, object)
    names[np.where(protein)[0][::5]] = "CA"
    names[moved] = "CA"
    tmsel = protein.copy()
    tmsel[moved] = True
    sels = {"protein": protein, "tm": tmsel}
    ref = MolLite(X[:, :, 0], name=names, named_selections=sels)
    mol = MolLite(X.copy(), box=g["box"], bonds=bonds, boxangles=angles, name=names, named_selections=sels)
    m = MetricTMscore(ref, "tm", centerstr="protein")
    got = m.project(mol)
    ca = np.where(tmsel & (names == "CA"))[0]
    want = to.tmscore(W[ca], X[ca, :, 0])[0].astype(np.float32)
    assert got.dtype == np.float32 and got.shape == (X.shape[2],)
    assert np.array_equal(got, want)
    unwrapped = MetricTMscore(ref, "tm", pbc=False).project(mol)
    assert np.array_equal(unwrapped, to.tmscore(X[ca], X[ca, :, 0])[0].astype(np.float32))
    assert not np.array_equal(got[1:], unwrapped[1:])  # the wrap changes the result
    assert np.array_equal(mol.coords, X)  # project does not modify the molecule


def test_metric_mapping_shards_and_errors(g_traj):
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metrictmscore import MetricTMscore
    from moleculekit_b200.sharding import _frame_view, project_sharded

    g = g_traj
    prot = g["sel_masks"][5]
    mol = MolLite(g["coords"], name=g["name"], named_selections={"protein": prot})
    ref = MolLite(g["coords"], name=g["name"], frame=6, named_selections={"protein": prot})
    m = MetricTMscore(ref, "protein", pbc=False)
    got = m.project(mol)
    ca = np.where(prot & (g["name"] == "CA"))[0]
    assert np.array_equal(got, to.tmscore(g["coords"][ca], g["coords"][ca, :, 6])[0].astype(np.float32))
    assert got[6] == 1.0
    mp = m.getMapping(mol)
    assert mp.shape == (1, 3) and mp["type"][0] == "tmscore" and np.array_equal(mp["atomIndexes"][0], ca)
    parts = [m.project(_frame_view(mol, a, b)) for a, b in ((0, 7), (7, 8), (8, 20))]
    assert np.array_equal(np.concatenate(parts), got)
    assert np.array_equal(project_sharded(m, mol), got)
    assert np.array_equal(mol.coords, g["coords"])
    with pytest.raises(RuntimeError):
        MetricTMscore(ref, np.zeros(mol.numAtoms, bool))
    with pytest.raises(RuntimeError):
        MetricTMscore(ref, "protein", reftmstr=np.where(g["name"] != "CA")[0][:5])
    with pytest.raises(RuntimeError):
        MetricTMscore(ref, np.where(g["name"] != "CA")[0][:5], reftmstr="protein").project(mol)
