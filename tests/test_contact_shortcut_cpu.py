"""Host-side check of the ARITHMETIC of the K3 contact-map shortcut (csrc/distance.cu `pair_contact`; DESIGN.md, K3).

The dense contact map decides `sqrtf(d2) <= thr` of the reference's float32 minimum-image sequence from a fused estimate
of d2 whenever the estimate lies outside a band around T.  The reference rounds fl(b n), so its w moves by up to half an
ulp of |d| -- an error that grows with the number of boxes between the atoms, not with |w|.  These tests restate both
float32 sequences in numpy (oracle/contact_shortcut.py) and check, on pairs whose wrapped distance lies within 1e-4 of the
threshold, from 0 to 2^21 boxes apart, that wherever the shortcut decides, it gives the reference's boolean.  No GPU."""
import numpy as np
import pytest

from oracle import contact_shortcut as cs

f32 = np.float32

THRESHOLDS = [0.5, 1.0, 2.5, 3.0, 3.65, 5.0, 8.0, 12.0, 17.3, 25.0, 40.0]
# image integers: small, around the shortcut's quotient limit, powers of two (fl(b n) exact), odd, and up to 2^21
N_SET = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 1023, 1024, 1025, 4097,
                  65535, 65536, 2 ** 20 - 1, 2 ** 20, 2 ** 21 - 1, 2 ** 21], np.int64)


def _cases(thr, rng, N):
    """N pairs (d, b): per-axis boxes from just above the shortcut's limit (b/2)^2 (1 - 1e-4) > T up to 1e4, per-axis image
    integers of both signs, and a wrapped vector of length thr (1 +- 1e-4) in a random direction; d = fl(b n + w)."""
    lo = 2.0 * thr / np.sqrt(1.0 - 1e-4) * (1.0 + 1e-6)
    kind = rng.random((N, 3))
    b = np.where(kind < 0.2, lo * (1.0 + rng.uniform(0.0, 1e-3, size=(N, 3))),        # just above the limit
                 np.exp(rng.uniform(np.log(lo), np.log(np.where(kind < 0.6, 30.0 * thr, 1e4)), size=(N, 3))))
    b = b.astype(f32)
    pick = rng.random((N, 3))
    n = np.where(pick < 0.5, rng.choice(N_SET, size=(N, 3)),
                 np.where(pick < 0.8, rng.integers(0, 80, size=(N, 3)),
                          np.round(np.exp(rng.uniform(0.0, np.log(2.0 ** 21), size=(N, 3))))))
    n = n * rng.choice([-1, 1], size=(N, 3))
    v = rng.normal(size=(N, 3))
    v /= np.linalg.norm(v, axis=1)[:, None]
    w = v * (thr * (1.0 + rng.uniform(-1e-4, 1e-4, size=N)))[:, None]
    d = (b.astype(np.float64) * n + w).astype(f32)
    return d, b


def _check(d, b, thr, rule):
    T = cs.threshold_d2(thr)
    with np.errstate(all="ignore"):
        want = np.sqrt(cs.reference_d2(d, b)) <= f32(thr)
    out = []
    for contract in (False, True):
        decided, got = rule(d, b, T, contract)
        out.append((decided, decided & (got != want)))
    return want, out


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_shortcut_gives_the_reference_boolean_far_from_the_origin(thr):
    rng = np.random.default_rng(int(thr * 100))
    d, b = _cases(thr, rng, 150_000)
    want, res = _check(d, b, thr, cs.decide)
    assert want.any() and not want.all()
    for contract, (decided, wrong) in zip((False, True), res):
        bad = np.flatnonzero(wrong)
        assert bad.size == 0, (contract, d[bad[:3]].tolist(), b[bad[:3]].tolist())
        # the shortcut still decides most pairs that are close enough to the origin for it
        _, qm = cs.estimate(d, b, contract)
        near = cs.shortcut_ok(b, cs.threshold_d2(thr)) & (qm < cs.QMAX) & (b.max(axis=1) < 10 * thr)
        assert near.sum() > 100 and decided[near].mean() > 0.75, (near.sum(), decided[near].mean())
    # the case set is meaningful: the former rule (fixed 4e-6 band up to 2^21 boxes) misjudges some of these pairs
    _, old = _check(d, b, thr, cs.decide_before_fix)
    assert old[0][1].any() or old[1][1].any()


def test_named_case_1228_in_a_34_box():
    """Atom 0 at the origin, atom 1 at x = 1228.8972 (36 boxes of 34.0527 away), threshold 3: the reference's
    w = 3.0 exactly, d2 = 9, a contact.  The fused estimate gets d2 = 9.000092, 1.0e-5 above T -- outside a 4e-6 band."""
    d = np.array([[f32(0.0) - f32(1228.8972), 0.0, 0.0]], f32)
    b = np.full((1, 3), f32(34.0527), f32)
    T = cs.threshold_d2(3.0)
    assert cs.reference_w(d, b)[0, 0] == f32(-3.0) and cs.reference_d2(d, b)[0] == f32(9.0)
    for contract in (False, True):
        d2, qm = cs.estimate(d, b, contract)
        assert abs(float(d2[0]) - 9.000092) < 2e-6 and 36 < qm[0] < 37
        decided, got = cs.decide_before_fix(d, b, T, contract)
        assert decided[0] and not got[0]  # the former rule: decided, no contact
        decided, got = cs.decide(d, b, T, contract)
        assert not decided[0] or got[0]


def test_far_image_failures_of_the_former_rule_start_a_few_dozen_thresholds_out():
    """The former rule's failures are not a corner case: at 3 A they appear once the atoms are ~40 thresholds apart,
    within 40 boxes of 17 to 40 A; within 4 boxes there are none (which is why origin-near tests never saw them)."""
    rng = np.random.default_rng(3)
    M = 400_000
    T = cs.threshold_d2(3.0)
    b = np.repeat(rng.uniform(17.0, 40.0, M).astype(f32)[:, None], 3, axis=1)
    for nmax, expect in ((4, False), (40, True)):
        n = rng.integers(1, nmax + 1, M).astype(np.float64)
        d = np.zeros((M, 3), f32)
        d[:, 0] = (b[:, 0].astype(np.float64) * n + rng.uniform(2.997, 3.003, M)).astype(f32)
        want = np.sqrt(cs.reference_d2(d, b)) <= f32(3.0)
        decided, got = cs.decide_before_fix(d, b, T, False)
        wrong = decided & (got != want)
        assert wrong.any() == expect, (nmax, int(wrong.sum()))
        if expect:
            assert np.abs(d[wrong, 0]).min() > 100.0
        decided, got = cs.decide(d, b, T, False)
        assert not (decided & (got != want)).any()


def test_fma32_is_correctly_rounded():
    """The emulated FFMA against exact rational arithmetic on products and sums that straddle float32 midpoints."""
    from fractions import Fraction

    rng = np.random.default_rng(1)
    a = rng.normal(size=4000).astype(f32)
    b = rng.normal(size=4000).astype(f32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.normal(size=4000) * 1e-7)).astype(f32)
    got = cs.fma32(a, b, c)
    for i in range(4000):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = f32(float(exact))
        cands = [np.nextafter(lo, f32(-np.inf)), lo, np.nextafter(lo, f32(np.inf))]
        best = min(cands, key=lambda x: (abs(Fraction(float(x)) - exact), int(np.array(x).view(np.uint32)) & 1))
        assert got[i] == best, i
