"""The exact superposition reference (oracle/exact_superposition.py) on the CPU: it agrees with the float64 SVD oracle
where that is accurate, reproduces exact answers on integer data, reports the degenerate cases as degenerate, and its
rounding, frame-sum and moment helpers are exact."""
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import align_oracle
from oracle import exact_superposition as ex

def _f(x):
    return np.array([[float(v) for v in row] for row in x]) if isinstance(x[0], list) else np.array([float(v) for v in x])


def _cloud(seed, k=40, scale=10.0):
    return np.random.default_rng(seed).normal(0, scale, (k, 3)).astype(np.float32)


@pytest.mark.parametrize("seed", range(4))
def test_agrees_with_svd_oracle_on_well_conditioned_data(seed):
    P = _cloud(seed)
    noise = np.random.default_rng(seed + 10).normal(0, 0.5, P.shape)
    Q = (P.astype(np.float64) @ Rotation.random(random_state=seed).as_matrix() + [3.0, -7.5, 1.25] + noise).astype(np.float32)
    f = ex.ExactFit(P, Q)
    rot, pc, qc = align_oracle.measure_fit(P, Q)
    assert f.gap / f.lam1 > 1e-2
    assert np.abs(_f(f.R) - rot.T).max() <= 1e-13
    assert np.abs(_f(f.p_bar) - pc).max() <= 1e-13 * np.abs(P).max()
    assert np.abs(_f(f.q_bar) - qc).max() <= 1e-13 * np.abs(Q).max()
    assert abs(float(f.min_rmsd()) - float(f.rmsd(rot.T, pc, qc))) <= 1e-13 * float(f.min_rmsd())
    assert abs(float(f.rmsd()) - float(align_oracle.mol_rmsd(P[:, :, None], Q[:, :, None], slice(None), slice(None)))) \
        <= 1e-13 * float(f.rmsd())
    # the residual of a record is an exact rational, and about the exact centroids it is the objective
    assert isinstance(f.residual(rot.T, pc, qc), Fraction)
    p64, q64 = _f(f.p_bar), _f(f.q_bar)
    if all(Fraction(float(x)) == x for x in f.p_bar + f.q_bar):
        assert f.residual(rot.T, p64, q64) == f.objective(rot.T)


SIGNED_PERMUTATIONS = [np.diag([1, -1, -1]), np.diag([-1, 1, -1]), np.diag([-1, -1, 1]),
                       np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]]), np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]]),
                       np.array([[0, 0, 1], [0, 1, 0], [-1, 0, 0]]), np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]])]


@pytest.mark.parametrize("j", range(len(SIGNED_PERMUTATIONS)))
def test_integer_rotations_are_exact(j):
    """integer points under 90 and 180 degree rotations: R* is the signed permutation, the residual is exactly 0, and
    the transform gives back the integers"""
    M = SIGNED_PERMUTATIONS[j]
    P = np.random.default_rng(j).integers(-50, 50, (25, 3)).astype(np.float32)
    Q = (P @ M.T + [7, -3, 11]).astype(np.float32)
    f = ex.ExactFit(P, Q)
    assert np.abs(_f(f.R) - M).max() <= 1e-50
    assert f.E < mp.mpf(10) ** -40 * f.lam1
    assert f.objective(M) == 0 and f.rmsd() > 0
    assert np.array_equal(ex.transform_f32(M, [0, 0, 0], [7, -3, 11], P), Q)


@pytest.mark.parametrize("axis", range(3))
def test_axis_mirror(axis):
    """the mirror image of a cloud flat in another axis is a 180 degree turn of it: R* is exact and E* = 0; a solid
    cloud's mirror image is no rotation of it: E* > 0, and R* is still proper"""
    flat = (axis + 1) % 3
    P = np.random.default_rng(axis).integers(-20, 20, (30, 3)).astype(np.float32)
    P[:, flat] = 0
    s = np.ones(3)
    s[axis] = -1
    f = ex.ExactFit(P, (P * s).astype(np.float32))
    turn = np.ones(3)
    turn[[axis, flat]] = -1
    assert f.E < mp.mpf(10) ** -40 * f.lam1
    assert np.abs(_f(f.R) - np.diag(turn)).max() <= 1e-50
    P3 = np.random.default_rng(9).integers(-20, 20, (30, 3)).astype(np.float32)
    f3 = ex.ExactFit(P3, (P3 * s).astype(np.float32))
    assert f3.E > 1 and f3.gap > 0 and abs(np.linalg.det(_f(f3.R)) - 1) < 1e-15


def test_degenerate_cases_report_gap_zero():
    rng = np.random.default_rng(3)
    P = rng.normal(0, 5, (2, 3)).astype(np.float32)
    assert ex.ExactFit(P, (P + 1).astype(np.float32)).gap == 0
    assert ex.ExactFit(P, rng.normal(0, 5, (2, 3)).astype(np.float32)).gap == 0
    t = np.arange(-6, 7, dtype=np.float32)[:, None]
    line = (t * np.float32([1, 2, -2])).astype(np.float32)
    f = ex.ExactFit(line, (line @ np.float32([[0, 1, 0], [1, 0, 0], [0, 0, 1]]) + 4).astype(np.float32))
    assert f.gap == 0 and f.R is None
    z = np.zeros((5, 3), np.float32) + np.float32(3.5)
    f0 = ex.ExactFit(z, z)
    assert f0.gap == 0 and f0.lam1 == 0 and f0.G == 0
    f1 = ex.ExactFit(P[:1], P[:1] + 1)
    assert f1.gap == 0 and f1.E == 0


def test_transform_rounds_exactly():
    """fl32 of the exact value, including values that lie exactly on a float32 midpoint and values one float64 step
    beside one (where rounding through float64 first would err)"""
    one = np.float32(1.0)
    half_ulp = float(np.spacing(one)) / 2
    X = np.zeros((4, 3), np.float32)
    q = np.array([1.0 + half_ulp, 1.0 + 3 * half_ulp, 1.0])
    got = np.array([ex.transform_f32(np.eye(3), [0, 0, 0], [v, 0, 0], X[:1])[0, 0] for v in q])
    assert got[0] == one and got[1] == np.float32(1.0 + 4 * half_ulp) and got[2] == one
    # 1 + half_ulp + 2^-60 is not a float64; the record x' = 2^-60 x + (1 + half_ulp) reaches it exactly
    y = ex.transform_f32(np.diag([2.0 ** -60, 1, 1]), [0, 0, 0], [1.0 + half_ulp, 0, 0], np.float32([[1, 0, 0]]))
    assert y[0, 0] == np.nextafter(one, np.float32(2))
    y = ex.transform_f32(np.diag([2.0 ** -60, 1, 1]), [0, 0, 0], [1.0 + half_ulp, 0, 0], np.float32([[-1, 0, 0]]))
    assert y[0, 0] == one


def test_frame_sums_and_moments_are_exact():
    rng = np.random.default_rng(5)
    rows = rng.normal(0, 1, (65, 7, 3)).astype(np.float32)
    rows[::2] += np.float32(1e4)
    rows[1::2] -= np.float32(1e4)
    s = ex.frame_sums(rows)
    for i in range(7):
        for d in range(3):
            assert s[i, d] == sum(Fraction(float(v)) for v in rows[:, i, d])
    pts = (rng.normal(0, 1e-3, (2, 6, 3)) + 1e4).astype(np.float32)
    w = np.array([1e-3, 2.5, 1e3, 7.0, 0.125, 3.0])
    m = ex.moments(pts, w, [0, 1, 6])
    for f in range(2):
        for g, (a, b) in enumerate(((0, 1), (1, 6))):
            W = sum(Fraction(float(x)) for x in w[a:b])
            for d in range(3):
                mu = sum(Fraction(float(x)) * Fraction(float(c)) for x, c in zip(w[a:b], pts[f, a:b, d])) / W
                v = sum(Fraction(float(x)) * (Fraction(float(c)) - mu) ** 2 for x, c in zip(w[a:b], pts[f, a:b, d])) / W
                assert m[f, g, d] == mu and m[f, g, 3 + d] == v
    assert all(m[f, 0, 3 + d] == 0 for f in range(2) for d in range(3))


def test_large_selection_is_exact_and_fast():
    """2^20 points through the integer path: the sums are exact (a rigid integer shift gives E = 0 and the exact
    centroid shift) in a few seconds"""
    rng = np.random.default_rng(6)
    P = rng.integers(-2 ** 20, 2 ** 20, (1 << 20, 3)).astype(np.float32) / np.float32(64)
    Q = (P + np.float32(1e4)).astype(np.float32)
    f = ex.ExactFit(P, Q)
    assert all(qb - pb == 10000 for pb, qb in zip(f.p_bar, f.q_bar))
    assert f.E < mp.mpf(10) ** -40 * f.lam1
    assert np.abs(_f(f.R) - np.eye(3)).max() < 1e-50
