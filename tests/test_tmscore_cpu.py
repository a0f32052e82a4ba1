"""CPU checks of K19 (TM-score): the host parameters, the CA pairing, and the C restatement of the search
(tests/tmscore_oracle.c) against an independent float64 numpy restatement that fits by SVD."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import tmscore_oracle as to

SIZES = [1, 2, 3, 4, 5, 15, 16, 21, 22, 31, 277, 5000]


@pytest.mark.parametrize("L", SIZES)
def test_fragment_lengths(L):
    from moleculekit_b200.tmscore import tm_parameters

    frag = tm_parameters(L, L)[2]
    lmin = min(4, L)
    assert frag[0] == (L if L > lmin else lmin) and frag[-1] == lmin and len(frag) <= 6
    assert all(f == L // 2 ** i for i, f in enumerate(frag[:-1]))
    assert all(a > b for a, b in zip(frag, frag[1:]))
    known = {1: (1,), 2: (2,), 3: (3,), 4: (4,), 5: (5, 4), 15: (15, 7, 4), 16: (16, 8, 4), 21: (21, 10, 5, 4),
             22: (22, 11, 5, 4), 31: (31, 15, 7, 4), 277: (277, 138, 69, 34, 17, 4),
             5000: (5000, 2500, 1250, 625, 312, 4)}
    assert frag == known[L]


@pytest.mark.parametrize("lnorm", SIZES)
def test_d0(lnorm):
    from moleculekit_b200.tmscore import tm_parameters

    d0, d0s, _ = tm_parameters(1, lnorm)
    if lnorm <= 21:  # 1.24 * 6^(1/3) - 1.8 = 0.453 is still below the 0.5 floor; 7^(1/3) gives 0.572
        assert d0 == 0.5
    else:
        assert d0 == 1.24 * math.pow(lnorm - 15, 1.0 / 3.0) - 1.8 and d0 > 0.5
    if lnorm > 21:
        assert abs(d0 - (1.24 * np.cbrt(lnorm - 15.0) - 1.8)) < 1e-12
    spot = {22: 0.5720, 31: 1.3246, 277: 6.1345}
    if lnorm in spot:
        assert abs(d0 - spot[lnorm]) < 1e-4
    assert d0s == (8.0 if lnorm == 5000 else d0 if lnorm == 277 else 4.5)


def test_parameters_reject_empty():
    from moleculekit_b200.tmscore import tm_parameters

    with pytest.raises(ValueError):
        tm_parameters(0, 5)


def test_ca_atoms():
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tmscore import ca_atoms

    names = ["N", "CA", "C", "O", "CB", "CA", "N", "CA"]
    mol = MolLite(np.zeros((8, 3), np.float32), name=names, named_selections={"s": np.arange(8) < 6})
    assert ca_atoms(mol, "all", "x").tolist() == [1, 5, 7]
    assert ca_atoms(mol, "s", "x").tolist() == [1, 5]
    assert ca_atoms(mol, np.array([0, 5, 6]), "x").tolist() == [5]
    with pytest.raises(RuntimeError, match="0 CA atoms"):
        ca_atoms(mol, np.array([0, 2]), "x")


# ------------------------------------------------------------------------------ independent numpy restatement
def _kabsch(x, y):
    p, q = x.mean(0), y.mean(0)
    U, _, Vt = np.linalg.svd((x - p).T @ (y - q))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    return Vt.T @ D @ U.T, p, q


def _numpy_tmscore(x, y, lnorm):
    """the search of the contract with numpy's SVD Kabsch (float64 throughout, numpy's own summation order)"""
    from moleculekit_b200.tmscore import tm_parameters

    x, y = x.astype(np.float64), y.astype(np.float64)
    L = len(x)
    d0, d0s, frag = tm_parameters(L, lnorm)

    def cut(dis, d):
        while True:
            c = np.where(dis < d)[0]
            if len(c) < 3 and L > 3:
                d += 0.5
            else:
                return c

    best, rmsd = -1.0, None
    for Li in frag:
        for iL in range(L - Li + 1):
            fitset = np.arange(iL, iL + Li)
            d = d0s - 1
            for it in range(21):
                R, p, q = _kabsch(x[fitset], y[fitset])
                dis = np.sqrt((((x - p) @ R.T + q - y) ** 2).sum(1))
                if rmsd is None:
                    rmsd = math.sqrt((dis ** 2).sum() / L)
                best = max(best, (1.0 / (1.0 + (dis / d0) ** 2)).sum() / lnorm)
                c = cut(dis, d)
                if len(c) == 0 or (it > 0 and np.array_equal(c, fitset)):
                    break
                fitset, d = c, d0s + 1
    return best, rmsd


def _ca(g):
    return g["coords"][g["name"] == "CA"]


@pytest.mark.parametrize("f", [3, 11, 19])
def test_oracle_matches_numpy_traj20(g_traj, f):
    X = _ca(g_traj)
    tm, rmsd, counts = to.frame(X[:, :, f], X[:, :, 0])
    want_tm, want_rmsd = _numpy_tmscore(X[:, :, f], X[:, :, 0], 277)
    assert abs(tm - want_tm) < 1e-9 and abs(rmsd - want_rmsd) < 1e-9
    assert counts[0] == 1129 and counts[0] <= counts[1] <= 21 * counts[0] and counts[2] == 277 * counts[1]


@pytest.mark.parametrize("sigma", [0.5, 2.0, 3.0])
def test_oracle_matches_numpy_noisy(g_traj, sigma):
    X = _ca(g_traj)
    rng = np.random.default_rng(int(sigma * 10))
    x = (X[:, :, 7] + rng.normal(0, sigma, size=(277, 3))).astype(np.float32)
    tm, rmsd, _ = to.frame(x, X[:, :, 0])
    want_tm, want_rmsd = _numpy_tmscore(x, X[:, :, 0], 277)
    assert abs(tm - want_tm) < 1e-9 and abs(rmsd - want_rmsd) < 1e-9


def test_identical_frame_scores_one(g_traj):
    X = _ca(g_traj)
    tm, rmsd, _ = to.frame(X[:, :, 4], X[:, :, 4])
    assert tm == 1.0 and rmsd < 1e-12


def test_rigid_copy_scores_one(g_traj):
    X = _ca(g_traj)[:, :, 9].astype(np.float64)
    G = Rotation.random(random_state=5).as_matrix()
    x = (X @ G.T + [30.0, -12.5, 4.0]).astype(np.float32)
    tm, rmsd, _ = to.frame(x, X.astype(np.float32))
    assert abs(tm - 1.0) < 1e-12 or tm == 1.0
    assert rmsd < 1e-4  # the float32 rounding of the moved copy


@pytest.mark.parametrize("n, m", [(277, 277), (200, 277), (277, 200)])
def test_pairing_and_normalisation(g_traj, n, m):
    """pairs k < min(n, m), normalised by m: a model that equals the reference's first pairs scores min(n, m) / m"""
    X = _ca(g_traj)[:, :, 2]
    Y = X[:m]
    Xm = np.concatenate([X[:min(n, m)], X[:n - min(n, m)] + 50.0]) if n > m else X[:n]
    tm, rmsd = to.tmscore(Xm[:, :, None], Y)
    assert tm[0] == min(n, m) / m and rmsd[0] < 1e-12


@pytest.mark.parametrize("f", [1, 8, 15])
def test_search_beats_all_pairs_fit(g_traj, f):
    X = _ca(g_traj)
    x, y = X[:, :, f].astype(np.float64), X[:, :, 0].astype(np.float64)
    rng = np.random.default_rng(f)
    x[:100] += rng.normal(0, 4.0, size=(100, 3))  # a badly fitting third pulls the all-pairs fit away
    x = x.astype(np.float32)
    R, p, q = _kabsch(x.astype(np.float64), y)
    dis = np.sqrt((((x - p) @ R.T + q - y) ** 2).sum(1))
    d0 = 1.24 * (277 - 15) ** (1 / 3) - 1.8
    all_pairs = (1.0 / (1.0 + (dis / d0) ** 2)).sum() / 277
    tm, rmsd, _ = to.frame(x, y.astype(np.float32))
    assert 0 < all_pairs <= tm <= 1 and tm > all_pairs + 1e-3
    assert abs(rmsd - math.sqrt((dis ** 2).sum() / 277)) < 1e-9


@pytest.mark.parametrize("L", [1, 2, 3, 4, 5])
def test_small_L(g_traj, L):
    X = _ca(g_traj)
    tm, rmsd, counts = to.frame(X[:L, :, 6], X[:L, :, 0])
    assert 0 < tm <= 1 and np.isfinite(rmsd) and counts[0] == (3 if L == 5 else 1)  # L = 5: 1 seed of 5, 2 of 4
    assert to.frame(X[:L, :, 6], X[:L, :, 6])[0] == 1.0


def test_nonfinite_frame_is_nan(g_traj):
    X = _ca(g_traj)[:, :, 1].copy()
    X[40, 1] = np.inf
    tm, rmsd, counts = to.frame(X, _ca(g_traj)[:, :, 0])
    assert np.isnan(tm) and np.isnan(rmsd) and counts == (0, 0, 0)
