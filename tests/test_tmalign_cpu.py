"""CPU checks of K27 (TM-align): the host parameters at their rule boundaries, and the C restatement
(tests/tmalign_oracle.c) on structures whose alignment is known: identical, rigidly moved, loop-deleted."""
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import tmalign_oracle as to


def _ca3(g):
    return np.ascontiguousarray(g["coords"][(g["name"] == "CA") & g["sel_protein"], :, 0])


def _d0(L):
    return 1.24 * math.pow(L - 15, 1.0 / 3.0) - 1.8


@pytest.mark.parametrize("lnorm", [19, 20])
def test_search_parameters(lnorm):
    from moleculekit_b200.tmalign import tmalign_parameters

    p = tmalign_parameters(lnorm, lnorm + 30)
    d0 = (0.168 if lnorm <= 19 else _d0(lnorm)) + 0.8
    assert p[0] == d0 and p[3] == d0 and p[1] == min(8.0, max(4.5, d0))
    assert p[2] == 1.5 * math.pow(lnorm, 0.3) + 3.5 and p[4] == 0.1 and p[5] == 4.25
    assert tmalign_parameters(41, 41)[4] == 0.4 and tmalign_parameters(40, 41)[4] == 0.1


@pytest.mark.parametrize("L", [21, 22])
def test_final_parameters(L):
    from moleculekit_b200.tmalign import tmalign_parameters

    p = tmalign_parameters(L + 9, L)  # ylen = L, xlen = L + 9
    want = 0.5 if L <= 21 else max(0.5, _d0(L))
    assert p[6] == want and p[7] == 4.5
    assert (L == 21 and want == 0.5) or (L == 22 and abs(want - 0.5720) < 1e-4)
    assert p[8] == max(0.5, _d0(L + 9)) and tmalign_parameters(L, 100)[8] == want


def test_secondary_structure_3ptb(g_3ptb):
    s = to.secondary(_ca3(g_3ptb))
    assert len(s) == 223 and set(s) <= set("HETC")
    assert s[:2] == "CC" and s[-2:] == "CC"
    # trypsin is mostly beta: two six-stranded barrels, and its C-terminal helix (residues 235-245)
    assert s.count("E") > 50 and "HHHHHHHH" in s[-20:]
    # a straight line is strand-free and helix-free; an ideal helix is all H inside
    line = np.zeros((12, 3), np.float32)
    line[:, 0] = 3.8 * np.arange(12)
    assert to.secondary(line) == "C" * 12
    t = np.arange(15) * np.deg2rad(100.0)
    helix = np.stack([2.3 * np.cos(t), 2.3 * np.sin(t), 1.5 * np.arange(15)], axis=1).astype(np.float32)
    assert to.secondary(helix) == "CC" + "H" * 11 + "CC"


def test_identical(g_3ptb):
    P = _ca3(g_3ptb)
    r = to.frame(P, P)
    assert np.array_equal(r["invmap"], np.arange(P.shape[0]))
    assert abs(r["tm"][0] - 1) < 1e-12 and abs(r["tm"][1] - 1) < 1e-12 and r["rmsd"] < 1e-6
    assert r["nali"] == P.shape[0]


def test_rigid_motion(g_3ptb):
    P = _ca3(g_3ptb)
    R = Rotation.random(random_state=11).as_matrix()
    Q = (P.astype(np.float64) @ R.T + np.array([13.0, -40.0, 7.5])).astype(np.float32)
    r = to.frame(Q, P)
    assert np.array_equal(r["invmap"], np.arange(P.shape[0]))
    assert abs(r["tm"][0] - 1) < 1e-9 and abs(r["tm"][1] - 1) < 1e-9
    rec = r["record"]
    moved = (Q.astype(np.float64) - rec[9:12]) @ rec[:9].reshape(3, 3).T + rec[12:15]
    assert np.abs(moved - P).max() < 1e-3


def test_deleted_loop(g_3ptb):
    P = _ca3(g_3ptb)
    keep = np.r_[0:60, 66:P.shape[0]]
    r = to.frame(P[keep], P)
    m = r["invmap"]
    assert all(keep[m[j]] == j for j in keep), "a kept residue maps elsewhere"
    assert (m[60:66] == -1).all() and r["nali"] == keep.size and abs(r["tm"][1] - 1) < 1e-9


def test_equal_lengths_same_bits(g_traj):
    X = np.ascontiguousarray(g_traj["coords"][g_traj["name"] == "CA"])
    r = to.frame(X[:, :, 3], X[:, :, 0])
    assert r["tm"][0].tobytes() == r["tm"][1].tobytes()


def test_rmsd_matches_svd_fit(g_traj, g_3ptb):
    X = np.ascontiguousarray(g_traj["coords"][g_traj["name"] == "CA"])
    P = _ca3(g_3ptb)
    for x, y in ((X[:, :, 9], P), (P, X[:, :, 2]), (X[:, :, 12], X[:, :, 0])):
        r = to.frame(x, y)
        j = np.where(r["invmap"] >= 0)[0]
        assert j.size == r["nali"] > 0
        a = x[r["invmap"][j]].astype(np.float64)
        b = y[j].astype(np.float64)
        a0, b0 = a - a.mean(0), b - b.mean(0)
        U, _, Vt = np.linalg.svd(a0.T @ b0)
        D = np.diag([1, 1, np.sign(np.linalg.det(U @ Vt))])
        Rm = (U @ D @ Vt).T
        want = math.sqrt(((a0 @ Rm.T - b0) ** 2).sum() / j.size)
        assert abs(r["rmsd"] - want) < 1e-9


def test_argument_errors(g_3ptb):
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tmalign import molTMalign, tmalign_parameters

    with pytest.raises(ValueError):
        tmalign_parameters(4, 100)
    with pytest.raises(ValueError):
        tmalign_parameters(100, 4)
    with pytest.raises(ValueError):
        to.frame(np.zeros((4, 3)), np.zeros((30, 3)))
    P = _ca3(g_3ptb)
    short = MolLite(P[:4, :, None], name=["CA"] * 4)
    full = MolLite(P[:, :, None], name=["CA"] * P.shape[0])
    with pytest.raises(ValueError):
        molTMalign(short, full, "all", "all")
    with pytest.raises(RuntimeError, match="0 CA atoms"):
        molTMalign(MolLite(P[:, :, None], name=["CB"] * P.shape[0]), full, "all", "all")


def test_over_the_cap_before_device_work():
    """more CA atoms than the cap on either side raise ValueError before anything is uploaded"""
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tmalign import max_residues, molTMalign

    n = max_residues() + 1
    big = MolLite(np.zeros((n, 3, 1), np.float32), name=["CA"] * n)
    small = MolLite(np.zeros((30, 3, 1), np.float32), name=["CA"] * 30)
    with pytest.raises(ValueError, match="at most"):
        molTMalign(big, small, "all", "all")
    with pytest.raises(ValueError, match="at most"):
        molTMalign(small, big, "all", "all")
