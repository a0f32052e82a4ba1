"""numpy restatement of the K3 contact-map shortcut (csrc/distance.cu, `pair_contact` / `contact_band`) and of the
reference's float32 minimum-image sequence it must agree with (distance_utils.pyx `_dist`).

TEST INFRASTRUCTURE ONLY.  Every float32 operation of both sequences is restated with its own rounding: plain float32
numpy arithmetic for the unfused operations (IEEE, round to nearest even) and `fma32` for the fused ones.  Inputs are
per-axis differences `d` (..., 3) and boxes `b` (..., 3), float32; the threshold enters as `T`, the largest float32
whose correctly rounded square root is <= thr (what the host side of the launch passes to the kernel).
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
MAGIC = f32(12582912.0)  # 1.5 * 2^23: x + MAGIC - MAGIC rounds x to an integer (ties to even) for |x| < 2^22

# the current rule (pair_contact): pairs less than QMAX boxes apart, outside a band of BAND_REL * T + BAND_D * sqrt(T) *
# bmax * (QMAX + 1/2) around T; frames where (b/2)^2 (1 - 1e-4) > T and the band stays below T / 4
QMAX = 8.0
BAND_REL = 4e-6
BAND_D = 2.5e-7


def fma32(a, b, c):
    """float32 fused multiply-add, correctly rounded: the product of two float32 is exact in float64, the float64 sum is
    made round-to-odd (its rounding error from a two-sum), and round-to-odd at 53 bits then nearest at 24 bits is the
    correctly rounded result -- no double-rounding error."""
    a, b, c = (np.asarray(x, dtype=f32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    bits = s.view(np.int64)
    fix = (err != 0) & ((bits & 1) == 0) & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(f32)


def threshold_d2(thr):
    """The largest float32 T with sqrtf(T) <= thr (mkb_dist_trajectory computes the same before the launch)."""
    thr = f32(thr)
    T = f32(thr * thr)
    while np.sqrt(T) > thr:
        T = np.nextafter(T, f32(-np.inf))
    while np.sqrt(np.nextafter(T, f32(np.inf))) <= thr:
        T = np.nextafter(T, f32(np.inf))
    return T


def reference_w(d, b):
    """distance_utils.pyx:41-52: w = d - fl(b * roundf(fl(d / b))), every operation rounded to float32."""
    d, b = np.asarray(d, f32), np.asarray(b, f32)
    with np.errstate(all="ignore"):
        q = (d / b).astype(np.float64)
        n = (np.sign(q) * np.floor(np.abs(q) + 0.5)).astype(f32)  # roundf: half away from zero (exact in float64)
        return (d - (b * n).astype(f32)).astype(f32)


def reference_d2(d, b):
    w = reference_w(d, b)
    with np.errstate(all="ignore"):
        return ((w[..., 0] * w[..., 0] + w[..., 1] * w[..., 1]) + w[..., 2] * w[..., 2]).astype(f32)


def estimate(d, b, contract):
    """pair_contact's fused estimate of d2 and its largest quotient qm.  `contract` selects the form in which the compiler
    may emit `q + MAGIC`: fused with `q = d * (1/b)` into one FFMA, or after q is rounded (both occur in practice)."""
    d, b = np.asarray(d, f32), np.asarray(b, f32)
    with np.errstate(all="ignore"):
        rb = (f32(1.0) / b).astype(f32)
        q = (d * rb).astype(f32)
        t = fma32(d, rb, MAGIC) if contract else (q + MAGIC).astype(f32)
        n = (t - MAGIC).astype(f32)
        w = fma32(-b, n, d)
        d2 = fma32(w[..., 0], w[..., 0], fma32(w[..., 1], w[..., 1], (w[..., 2] * w[..., 2]).astype(f32)))
        qm = np.abs(q).max(axis=-1)
    return d2, qm


def shortcut_ok(b, T):
    """contact_band(...).ok: per frame (box) -- half the smallest box edge positive and above the threshold, the widest band
    below T / 4."""
    b = np.asarray(b, f32)
    T = f32(T)
    with np.errstate(all="ignore"):
        m = (b * f32(0.5)).astype(f32).min(axis=-1)
        return (m > 0) & ((m * m * (f32(1.0) - f32(1e-4))).astype(f32) > T) & (band(b, T) <= f32(0.25) * T)


def band(b, T):
    """contact_band(...).band: the half-width of the band around T, one number per frame."""
    b = np.asarray(b, f32)
    with np.errstate(all="ignore"):
        b1 = (f32(BAND_D) * np.sqrt(f32(T)) * b.max(axis=-1)).astype(f32)
        return fma32(f32(QMAX + 0.5), b1, (f32(BAND_REL) * f32(T)).astype(f32))


def decide(d, b, T, contract):
    """(decided, answer): whether the shortcut decides the pair, and its boolean where it does."""
    d2, qm = estimate(d, b, contract)
    with np.errstate(all="ignore"):
        decided = shortcut_ok(b, T) & (np.abs(d2 - f32(T)) > band(b, T)) & (qm < f32(QMAX))
    return decided, d2 <= f32(T)


def decide_before_fix(d, b, T, contract):
    """The rule the shortcut used before: a fixed 4e-6 band for quotients up to 2^21.  It is wrong far from the origin,
    where the reference's rounding of fl(b n) moves w by up to half an ulp of |d| (tests assert that the case sets
    they build contain such pairs)."""
    d2, qm = estimate(d, b, contract)
    b = np.asarray(b, f32)
    T = f32(T)
    with np.errstate(all="ignore"):
        m = (b * f32(0.5)).astype(f32).min(axis=-1)
        ok = (m * m * f32(1.0 - 1e-4)).astype(f32) > T
        decided = ok & (np.abs(d2 - T) > (f32(4e-6) * T).astype(f32)) & (qm < f32(2097152.0))
    return decided, d2 <= T
