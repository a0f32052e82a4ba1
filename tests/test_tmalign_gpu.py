"""GPU parity of K27 (TM-align) against the C restatement (tests/tmalign_oracle.c): scores, RMSDs, aligned counts,
maps and superposition records are bit-identical, on frames of one protein, across two proteins, across a deleted loop,
at the short-length rule boundaries and at the residue cap."""
import numpy as np
import pytest

import tmalign_oracle as to

pytestmark = pytest.mark.gpu


def _t(a, dtype):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to("cuda:0")


def _device(X, Y, frames=None):
    """tmalign_device of x rows X (xlen, 3, F) onto y rows Y (ylen, 3) or (ylen, 3, F), all outputs as numpy"""
    from moleculekit_b200.tmalign import tmalign_device

    Yd = Y[:, :, None] if Y.ndim == 2 else Y
    out = tmalign_device(_t(X, np.float32), _t(np.arange(X.shape[0]), np.int32), _t(Yd, np.float32),
                         _t(np.arange(Y.shape[0]), np.int32), None if frames is None else _t(frames, np.int32))
    return tuple(o.cpu().numpy() for o in out)


def _same(got, want):
    for g, w, what in zip(got, want, ("tm", "rmsd", "nali", "invmap", "records")):
        assert g.shape == w.shape, what
        if g.dtype == np.float64:
            assert np.array_equal(np.isnan(g), np.isnan(w)), what
            ok = np.isnan(w) | (g.view(np.int64) == w.view(np.int64))
        else:
            ok = g == w
        assert ok.all(), f"{what} differs at {np.argwhere(~ok)[:5].tolist()}"


def _check(X, Y, frames=None):
    got = _device(X, Y, frames)
    _same(got, to.tmalign(X, Y, frames, matching=Y.ndim == 3))
    return got


def _ca(g):
    return np.ascontiguousarray(g["coords"][g["name"] == "CA"])


def _ca3(g):
    return np.ascontiguousarray(g["coords"][(g["name"] == "CA") & g["sel_protein"], :, 0])


def test_traj20_onto_frame0(g_traj):
    X = _ca(g_traj)
    tm = _check(X, X[:, :, 0])[0]
    assert tm[0, 0] == 1.0 and (tm[1:, 0] > 0.8).all()


@pytest.mark.parametrize("direction", ["traj_onto_3ptb", "3ptb_onto_traj"])
def test_different_proteins(g_traj, g_3ptb, direction):
    X, P = _ca(g_traj), _ca3(g_3ptb)
    if direction == "traj_onto_3ptb":
        _check(X[:, :, :4], P)
    else:
        _check(np.ascontiguousarray(P[:, :, None].repeat(2, axis=2)), X[:, :, 7])


def test_deleted_loop(g_3ptb):
    P = _ca3(g_3ptb)
    keep = np.r_[0:60, 66:P.shape[0]]
    _check(P[keep][:, :, None], P)


@pytest.mark.parametrize("L", [5, 6, 19, 20, 21, 22])
def test_short_lengths(g_traj, L):
    X = _ca(g_traj)
    _check(np.ascontiguousarray(X[40:40 + L, :, :3]), X[40:40 + L + 3, :, 0])
    _check(np.ascontiguousarray(X[100:100 + L + 7, :, :2]), X[100:100 + L, :, 5])


def test_at_the_cap():
    from moleculekit_b200.tmalign import max_residues

    cap = max_residues()
    rng = np.random.default_rng(5)
    X = np.cumsum(rng.normal(0, 2.2, size=(cap, 3, 1)), axis=0).astype(np.float32)
    _check(X, X[300:330, :, 0] + np.float32(0.3))


def test_nonfinite_frames(g_traj):
    X = _ca(g_traj)[:, :, :4].copy()
    X[17, 1, 1] = np.nan
    X[200, 2, 3] = np.inf
    tm, rmsd, nali, invmap, rec = _check(X, X[:, :, 0])
    for f in (1, 3):
        assert np.isnan(tm[f]).all() and np.isnan(rmsd[f]) and nali[f] == 0 and (invmap[f] == -1).all()
        assert np.array_equal(rec[f], [1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0])


def test_frame_lists(g_traj):
    X = _ca(g_traj)
    full = _device(X[:, :, :8], X[:, :, 0])
    for frames in ([5, 2, 2, 7], list(range(1, 8, 3)), [0]):
        got = _check(X[:, :, :8], X[:, :, 0], np.asarray(frames))
        _same(got, tuple(a[frames] for a in full))


def test_mol_tmalign_frames_and_matching(g_traj):
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tmalign import molTMalign

    g = g_traj
    X = _ca(g)
    mol = MolLite(g["coords"], name=g["name"])
    ref = MolLite(g["coords"], name=g["name"], frame=4)
    for frames, flist in ((None, range(20)), (slice(2, 12, 3), range(2, 12, 3)), ([9, 0, 9], [9, 0, 9]), (6, [6])):
        tm, rmsd, nali = molTMalign(mol, ref, "all", "all", frames=frames)
        w = to.tmalign(X, X[:, :, 4], list(flist))
        assert np.array_equal(tm.view(np.int64), w[0][:, 0].view(np.int64))
        assert np.array_equal(rmsd.view(np.int64), w[1].view(np.int64)) and np.array_equal(nali, w[2])
    shifted = MolLite(np.ascontiguousarray(g["coords"][:, :, ::-1]), name=g["name"])
    tm, rmsd, nali, aln, (R, T) = molTMalign(mol, shifted, "all", "all", frames=[1, 3], matchingframes=True,
                                             return_alignments=True)
    Y = np.ascontiguousarray(X[:, :, ::-1])
    w = to.tmalign(X, Y, [1, 3], matching=True)
    assert np.array_equal(tm.view(np.int64), w[0][:, 0].view(np.int64)) and np.array_equal(nali, w[2])
    ca = np.where(g["name"] == "CA")[0]
    for k in range(2):
        j = np.where(w[3][k] >= 0)[0]
        assert np.array_equal(aln[k], np.stack([ca[w[3][k][j]], ca[j]], axis=1))
        Rk = w[4][k][:9].reshape(3, 3)
        assert np.array_equal(R[k], Rk) and np.allclose(T[k], w[4][k][12:15] - Rk @ w[4][k][9:12], rtol=0, atol=1e-12)


def test_apply_device_with_records(g_traj):
    """the records move every atom within 1 float32 ulp of the oracle's float64 transform; unlisted frames untouched"""
    import torch
    from moleculekit_b200.align import apply_device
    from moleculekit_b200.tmalign import tmalign_device

    g = g_traj
    ca = np.where(g["name"] == "CA")[0]
    frames = np.array([3, 11, 19, 0])
    dev = torch.device("cuda:0")
    d = torch.from_numpy(g["coords"]).to(dev)
    out = tmalign_device(d, _t(ca, np.int32), d[:, :, 5:6], _t(ca, np.int32), _t(frames, np.int32))
    rec = out[4]
    moved = apply_device(d.clone(), rec, frames=_t(frames, np.int32)).cpu().numpy()
    want_rec = to.tmalign(g["coords"][ca], g["coords"][ca, :, 5], list(frames))[4]
    assert np.array_equal(rec.cpu().numpy().view(np.int64), want_rec.view(np.int64))
    X = g["coords"]
    for k, f in enumerate(frames):
        R, p, q = want_rec[k][:9].reshape(3, 3), want_rec[k][9:12], want_rec[k][12:15]
        want = ((X[:, :, f].astype(np.float64) - p) @ R.T + q).astype(np.float32)
        diff = np.abs(moved[:, :, f].view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert diff.max() <= 1, f
    rest = np.setdiff1d(np.arange(X.shape[2]), frames)
    assert np.array_equal(moved[:, :, rest].view(np.uint32), X[:, :, rest].view(np.uint32))


def test_rejects(g_traj):
    import torch
    from moleculekit_b200.tmalign import max_residues, tmalign_device

    X = _ca(g_traj)
    d = _t(X, np.float32)
    with pytest.raises(ValueError):
        tmalign_device(d, _t(np.arange(4), np.int32), d[:, :, :1], _t(np.arange(50), np.int32))
    big = torch.zeros((max_residues() + 1, 3, 1), device="cuda:0")
    with pytest.raises(ValueError):
        tmalign_device(big, _t(np.arange(max_residues() + 1), np.int32), d[:, :, :1], _t(np.arange(50), np.int32))
    bad = d[:, :, :1].clone()
    bad[3, 0, 0] = float("nan")
    with pytest.raises(ValueError):
        tmalign_device(d, _t(np.arange(50), np.int32), bad, _t(np.arange(50), np.int32))


def test_cap_by_cap():
    """one item at the residue cap on both sides: a random walk onto a noisy copy of itself"""
    from moleculekit_b200.tmalign import max_residues

    cap = max_residues()
    rng = np.random.default_rng(9)
    steps = rng.normal(size=(cap, 3))
    Y = np.cumsum(3.8 * steps / np.linalg.norm(steps, axis=1, keepdims=True), axis=0).astype(np.float32)
    X = (Y + rng.normal(0, 0.5, size=Y.shape)).astype(np.float32)[:, :, None]
    tm = _check(X, Y)[0]
    assert tm[0, 0] > 0.5
