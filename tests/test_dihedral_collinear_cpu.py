"""Degenerate dihedrals in any orientation, without a GPU: three collinear float32 points that are not axis-aligned
give angle 0 and (sin, cos) = (0, 1) in the host mirror dihedralAngle and in the float64 oracle, although the
projected form on its own returns rounding noise for them."""
import numpy as np

from oracle import dihedral_oracle as do


def _projected_only(P):
    """the projected form without the degeneracy test: what the angle would be from rounding noise"""
    b0, b1, b2 = P[0] - P[1], P[2] - P[1], P[3] - P[2]
    u = b1 / np.sqrt(b1 @ b1)
    v, w = b0 - (b0 @ u) * u, b2 - (b2 @ u) * u
    return np.arctan2(np.cross(u, v) @ w, v @ w)


def test_collinear_in_any_orientation():
    from moleculekit_b200.dihedral import dihedralAngle

    P = do.collinear_quads(1000, 5)
    assert not np.any(P[:, :, :, None] == 0)  # no coordinate is zero: nothing lies on an axis
    assert np.array_equal(do.angles(P), np.zeros(1000))
    assert np.array_equal(do.sincos(P), np.tile([0.0, 1.0], (1000, 1)))
    assert all(dihedralAngle(P[:, :, k]) == 0.0 for k in range(1000))
    noisy = sum(_projected_only(P[:, :, k]) != 0 for k in range(1000))
    assert noisy > 100  # the cases are ones the projected form alone gets wrong
    # the example of three points (0.1, 0.2, 0.3) x 1, 2, 4
    Q = np.array([[0.1, 0.2, 0.3], [0.2, 0.4, 0.6], [0.4, 0.8, 1.2], [1, 0, 0]], np.float32).astype(np.float64)
    assert dihedralAngle(Q) == 0.0 and do.sincos(Q[:, :, None])[0].tolist() == [0.0, 1.0]


def test_coincident_middle_atoms_and_bent_neighbours():
    from moleculekit_b200.dihedral import dihedralAngle

    rng = np.random.default_rng(6)
    for _ in range(200):
        p = rng.normal(0, 10, (4, 3)).astype(np.float32).astype(np.float64)
        assert abs(dihedralAngle(p) - do.angles(p[:, :, None])[0]) < 1e-9  # a generic quadruple is not degenerate
        p[2] = p[1]
        assert dihedralAngle(p) == 0.0 and do.sincos(p[:, :, None])[0].tolist() == [0.0, 1.0]
