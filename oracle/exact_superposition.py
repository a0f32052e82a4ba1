"""Exact superposition, frame-sum and group-moment references -- TEST INFRASTRUCTURE ONLY.

Every float32 coordinate, float64 weight and float64 fit-record entry is an exact dyadic rational, and everything
here but one step is computed exactly from those rationals: the values are scaled by a common power of two to Python
integers (numpy object arrays, about a second per million atoms and sum), summed as integers and combined as
``fractions.Fraction``.  So centroids, the covariance H, Horn's 4x4 matrix, G = sum |p - p_bar|^2 + sum |q - q_bar|^2,
the residual of a given float64 record, frame sums and weighted moments carry no rounding error at any selection size,
offset or spread.  The one approximate step is the eigen-decomposition of Horn's matrix: ``mpmath.eigsy`` at ``DPS``
decimal digits, some 45 digits beyond float64.

Conventions are the device's (csrc/align.cu): H[a][b] = sum (p_a - p_bar_a)(q_b - q_bar_b), R row-major with q ~ R p,
so a record maps x to R (x - p_bar) + q_bar.  ``align_oracle.measure_fit`` returns R transposed (row vectors).
"""
from __future__ import annotations

from fractions import Fraction

import mpmath as mp
import numpy as np

DPS = 60
# an eigenvalue gap below this fraction of the spectrum's scale is not resolved at DPS digits and is reported as 0
GAP_ZERO = mp.mpf(10) ** (15 - DPS)


def _p2(s: int) -> Fraction:
    """2**-s as a Fraction"""
    return Fraction(1, 1 << s) if s >= 0 else Fraction(1 << -s)


def scaled_ints(a):
    """(X, s): an object array of Python ints of ``a``'s shape and an int s with a == X * 2**-s exactly (``a`` float32
    or float64, finite)"""
    a = np.asarray(a)
    if a.dtype not in (np.float32, np.float64):
        raise TypeError(f"float32 or float64 expected, got {a.dtype}")
    a = a.astype(np.float64)
    if not np.isfinite(a).all():
        raise ValueError("non-finite value")
    m, e = np.frexp(a)
    M = (m * 2.0 ** 53).astype(np.int64)  # exact: a = M 2**(e - 53), |M| < 2**53
    sh = e.astype(np.int64) - 53
    nz = M != 0
    s = -int(sh[nz].min()) if nz.any() else 0
    shift = np.where(nz, sh + s, 0)
    return np.left_shift(M.astype(object), shift.astype(object)), s


def _isum(X) -> int:
    return int(X.sum()) if X.size else 0


def to_mpf(x: Fraction):
    return mp.mpf(x.numerator) / x.denominator


def _horn(H):
    """Horn's symmetric 4x4 matrix of H (nested lists of numbers), the device's layout"""
    (Sxx, Sxy, Sxz), (Syx, Syy, Syz), (Szx, Szy, Szz) = H
    return [[Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx],
            [Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz],
            [Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy],
            [Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz]]


def quat_rotation(q):
    """row-major 3x3 rotation (nested lists) of the quaternion q = (q0, q1, q2, q3), normalised first"""
    n = mp.sqrt(sum(x * x for x in q))
    q0, q1, q2, q3 = (x / n for x in q)
    return [[q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3, 2 * (q1 * q2 - q0 * q3), 2 * (q1 * q3 + q0 * q2)],
            [2 * (q1 * q2 + q0 * q3), q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3, 2 * (q2 * q3 - q0 * q1)],
            [2 * (q1 * q3 - q0 * q2), 2 * (q2 * q3 + q0 * q1), q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3]]


class ExactFit:
    """The exact superposition of the float32 points P onto Q (both (k, 3), pairwise).

    p_bar, q_bar   exact centroids (3 Fractions each)
    H              exact covariance (3x3 Fractions), G exact sum of both centred squared norms (Fraction)
    eigenvalues    of Horn's matrix, descending (mpf); lam1 the largest, gap = lam1 - lam2 (0 when unresolved)
    R              the optimal proper rotation (3x3 mpf, nested lists), None when gap == 0 (not unique)
    E              G - 2 lam1 (>= 0), the least sum of squared deviations over proper rotations (mpf)
    """

    def __init__(self, P, Q):
        mp.mp.dps = DPS
        P = np.asarray(P, dtype=np.float32).reshape(-1, 3)
        Q = np.asarray(Q, dtype=np.float32).reshape(-1, 3)
        if P.shape != Q.shape or P.shape[0] == 0:
            raise ValueError(f"P and Q must be the same non-empty (k, 3): {P.shape}, {Q.shape}")
        k = self.k = P.shape[0]
        X, sp = scaled_ints(P)
        Y, sq = scaled_ints(Q)
        up, uq = _p2(sp), _p2(sq)
        self.P1 = [_isum(X[:, a]) * up for a in range(3)]
        self.Q1 = [_isum(Y[:, a]) * uq for a in range(3)]
        self.P2 = [[None] * 3 for _ in range(3)]
        self.Q2 = [[None] * 3 for _ in range(3)]
        for a in range(3):
            for b in range(a, 3):
                self.P2[a][b] = self.P2[b][a] = _isum(X[:, a] * X[:, b]) * up * up
                self.Q2[a][b] = self.Q2[b][a] = _isum(Y[:, a] * Y[:, b]) * uq * uq
        self.PQ = [[_isum(X[:, a] * Y[:, b]) * up * uq for b in range(3)] for a in range(3)]
        self.p_bar = [s / k for s in self.P1]
        self.q_bar = [s / k for s in self.Q1]
        self.H = [[self.PQ[a][b] - self.P1[a] * self.Q1[b] / k for b in range(3)] for a in range(3)]
        self.G = sum(self.P2[a][a] - self.P1[a] ** 2 / k + self.Q2[a][a] - self.Q1[a] ** 2 / k for a in range(3))
        N = mp.matrix([[to_mpf(x) for x in row] for row in _horn(self.H)])
        ev, V = mp.eigsy(N)
        order = sorted(range(4), key=lambda j: ev[j], reverse=True)
        self.eigenvalues = [ev[j] for j in order]
        self.lam1 = self.eigenvalues[0]
        scale = max(abs(x) for x in self.eigenvalues)
        gap = self.eigenvalues[0] - self.eigenvalues[1]
        self.gap = gap if gap > GAP_ZERO * scale else mp.mpf(0)
        self.R = quat_rotation([V[r, order[0]] for r in range(4)]) if self.gap > 0 else None
        self.E = max(to_mpf(self.G) - 2 * self.lam1, mp.mpf(0))

    def residual(self, R, p_bar, q_bar) -> Fraction:
        """exact sum over the pairs of |R (p - p_bar) + q_bar - q|^2 for a float64 record (R row-major 3x3 or 9,
        p_bar, q_bar 3): the deviations' exact second moments, no rounding and so no cancellation"""
        R = [[Fraction(float(x)) for x in row] for row in np.asarray(R, dtype=np.float64).reshape(3, 3)]
        a = [Fraction(float(x)) for x in np.asarray(p_bar, dtype=np.float64).ravel()]
        b = [Fraction(float(x)) for x in np.asarray(q_bar, dtype=np.float64).ravel()]
        k, P1, Q1 = self.k, self.P1, self.Q1
        # u = p - a, w = q - b: Cuu = sum u u^T, Cwu = sum w u^T, sum |w|^2
        Cuu = [[self.P2[j][l] - a[j] * P1[l] - P1[j] * a[l] + k * a[j] * a[l] for l in range(3)] for j in range(3)]
        Cwu = [[self.PQ[j][i] - b[i] * P1[j] - Q1[i] * a[j] + k * b[i] * a[j] for j in range(3)] for i in range(3)]
        ww = sum(self.Q2[i][i] - 2 * b[i] * Q1[i] + k * b[i] * b[i] for i in range(3))
        RtR = [[sum(R[i][j] * R[i][l] for i in range(3)) for l in range(3)] for j in range(3)]
        uu = sum(RtR[j][l] * Cuu[j][l] for j in range(3) for l in range(3))
        wu = sum(R[i][j] * Cwu[i][j] for i in range(3) for j in range(3))
        return uu - 2 * wu + ww

    def objective(self, R) -> Fraction:
        """exact sum |R (p - p_bar) - (q - q_bar)|^2 about the exact centroids: the fit objective of the float64
        rotation R"""
        R =[[Fraction(float(x)) for x in row] for row in np.asarray(R, dtype=np.float64).reshape(3, 3)]
        k, P1, Q1 = self.k, self.P1, self.Q1
        Cpp = [[self.P2[j][l] - P1[j] * P1[l] / k for l in range(3)] for j in range(3)]
        RtR = [[sum(R[i][j] * R[i][l] for i in range(3)) for l in range(3)] for j in range(3)]
        qq = sum(self.Q2[i][i] - Q1[i] * Q1[i] / k for i in range(3))
        return sum(RtR[j][l] * Cpp[j][l] for j in range(3) for l in range(3)) \
            - 2 * sum(R[i][j] * self.H[j][i] for i in range(3) for j in range(3)) + qq

    def rmsd(self, R=None, p_bar=None, q_bar=None):
        """exact sqrt(mean |T(p) - q|^2) (mpf) under a float64 record, or without a transform when R is None"""
        if R is None:
            e = sum(self.P2[a][a] - 2 * self.PQ[a][a] + self.Q2[a][a] for a in range(3))
        else:
            e = self.residual(R, p_bar, q_bar)
        return mp.sqrt(to_mpf(e) / self.k)

    def min_rmsd(self):
        """sqrt(E / k): the Kabsch RMSD (mpf)"""
        return mp.sqrt(self.E / self.k)


def measure_fit(P, Q):
    """(R, p_bar, q_bar) in float64 from the exact fit (R None when the optimum is not unique)"""
    f = ExactFit(P, Q)
    R = None if f.R is None else np.array([[float(x) for x in row] for row in f.R])
    return R, np.array([float(x) for x in f.p_bar]), np.array([float(x) for x in f.q_bar])


def _round_f32(num, s: int) -> np.ndarray:
    """fl32(num * 2**-s), round to nearest even, for an object array of Python ints"""
    num = np.asarray(num, dtype=object)
    if s >= 0:
        f64 = np.array([n / (1 << s) for n in num.ravel()], dtype=np.float64).reshape(num.shape)  # correctly rounded
    else:
        f64 = np.array([float(n << -s) for n in num.ravel()], dtype=np.float64).reshape(num.shape)
    out = f64.astype(np.float32)
    # float64 first, then float32, rounds twice: it errs only where the float64 value is a float32 midpoint
    other = np.where(out.astype(np.float64) < f64, np.nextafter(out, np.float32(np.inf)),
                     np.nextafter(out, np.float32(-np.inf)))
    tie = (out.astype(np.float64) != f64) & ((out.astype(np.float64) + other.astype(np.float64)) / 2 == f64)
    for i in zip(*np.nonzero(tie)):
        exact = Fraction(int(num[i])) * _p2(s)
        mid = Fraction(float(f64[i]))
        if exact != mid:  # not a true tie: the side of the midpoint decides
            lo, hi = sorted([out[i], other[i]])
            out[i] = hi if exact > mid else lo
    return out


def transform_f32(R, p_bar, q_bar, X):
    """fl32 of the exact R (x - p_bar) + q_bar for every row x of the float32 (n, 3) ``X`` under a float64 record"""
    X = np.asarray(X, dtype=np.float32).reshape(-1, 3)
    R = np.asarray(R, dtype=np.float64).reshape(3, 3)
    xp, s1 = scaled_ints(np.concatenate([X.astype(np.float64), np.asarray(p_bar, np.float64).reshape(1, 3)]))
    Ri, s2 = scaled_ints(R)
    qi, s3 = scaled_ints(np.asarray(q_bar, dtype=np.float64).ravel())
    U = xp[:-1] - xp[-1]
    S = max(s1 + s2, s3)
    out = np.empty(X.shape, dtype=np.float32)
    for d in range(3):
        y = U[:, 0] * Ri[d, 0] + U[:, 1] * Ri[d, 1] + U[:, 2] * Ri[d, 2]
        num = np.left_shift(y, S - s1 - s2) + (int(qi[d]) << (S - s3))
        out[:, d] = _round_f32(num, S)
    return out


def frame_sums(rows):
    """exact per-axis sums over the frames of float32 ``rows`` (F, k, 3): a (k, 3) object array of Fractions"""
    X, s = scaled_ints(np.asarray(rows, dtype=np.float32))
    u = _p2(s)
    S = X.sum(axis=0) if X.shape[0] else np.zeros(X.shape[1:], dtype=object)
    return np.vectorize(lambda n: Fraction(int(n)) * u, otypes=[object])(S)


def moments(points, weights=None, offsets=None):
    """exact two-pass weighted moments of float32 ``points`` (F, m, 3) over groups of positions [offsets[g],
    offsets[g+1]) with float64 ``weights`` (m,) (None = 1): a (F, G, 6) object array of Fractions, the weighted mean
    (0-2) and the weighted per-axis variance around it (3-5), both over the group's weight total"""
    P = np.asarray(points, dtype=np.float32)
    F, m, _ = P.shape
    w = np.ones(m) if weights is None else np.asarray(weights, dtype=np.float64)
    offsets = np.array([0, m]) if offsets is None else np.asarray(offsets)
    X, s = scaled_ints(P)
    Wi, sw = scaled_ints(w)
    ux, uw = _p2(s), _p2(sw)
    out = np.empty((F, offsets.size - 1, 6), dtype=object)
    for g, (a, b) in enumerate(zip(offsets[:-1], offsets[1:])):
        wg = Wi[a:b]
        W = _isum(wg) * uw
        for f in range(F):
            for d in range(3):
                c = X[f, a:b, d]
                s1 = _isum(wg * c) * uw * ux
                s2 = _isum(wg * c * c) * uw * ux * ux
                mu = s1 / W
                out[f, g, d] = mu
                out[f, g, 3 + d] = s2 / W - mu * mu
    return out
