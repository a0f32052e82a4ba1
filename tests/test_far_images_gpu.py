"""GPU parity of the periodic pair kernels on atoms 1 to 2^20 boxes apart (unwrapped trajectories, e.g. NAMD without
wrapAll), against the oracle's float32 restatement of the reference.  The wrapped differences are placed a few ulps either
side of each kernel's threshold and of half a box, where a fast route that estimates the minimum image has to hand the
pair to the exact sequence.  The reference rounds fl(b n), so far from the origin its w is off the exact d - b n by up to
half an ulp of |d|: every kernel must reproduce that, not the exact value."""
import numpy as np
import pytest

from oracle import contact_shortcut as cs

pytestmark = pytest.mark.gpu

f32 = np.float32
# image integers per axis: near, a few dozen boxes (where a fixed-band contact shortcut starts to misjudge), powers of
# two (fl(b n) exact for every b), odd counts (fl(b n) mostly inexact), up to 2^20
FAR_N = np.array([0, 1, 2, 3, 5, 7, 36, 37, 63, 64, 65, 255, 1023, 1025, 2 ** 15 + 1, 2 ** 17, 2 ** 20 - 1, 2 ** 20])
BOXES = np.array([[34.0527, 34.0527, 34.0527], [17.3, 23.9, 31.1], [40.1, 18.7, 25.3], [33.3, 33.3, 100.7],
                  [19.9, 37.1, 24.2], [36.84, 36.84, 36.84]], np.float32).T  # (3, F), a different box per frame


def _bits(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


def _ulp_steps(x, k):
    x = f32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf if k > 0 else -np.inf))
    return x


def _far_case(thr, seed, per=240):
    """(coords (3 + per, 3, F), box (3, F), chains): three centres -- the origin, a point inside the box and a point 2^16
    boxes out -- and `per` partners per frame at b n + w from the origin, |w| = thr +- a few ulps in a random direction
    (two thirds of them) or w_k = +-(b_k/2 +- a few ulps) on one axis (the rest).  Partner 0 of frame 0 is the named far
    contact: x = 1228.8972 in a 34.0527 box, w = 3.0."""
    rng = np.random.default_rng(seed)
    F = BOXES.shape[1]
    c = np.zeros((3 + per, 3, F), np.float32)
    for f in range(F):
        b = BOXES[:, f].astype(np.float64)
        c[1, :, f] = rng.uniform(0, 1, 3) * b
        c[2, :, f] = b * 65536 + rng.uniform(-0.5, 0.5, 3) * b
        n = rng.choice(FAR_N, size=(per, 3)) * rng.choice([-1, 1], size=(per, 3))
        v = rng.normal(size=(per, 3))
        v /= np.linalg.norm(v, axis=1)[:, None]
        w = v * np.array([float(_ulp_steps(thr, int(k))) for k in rng.integers(-4, 5, per)])[:, None]
        half = rng.random(per) < 1 / 3
        ax = rng.integers(0, 3, per)
        for p in np.flatnonzero(half):
            w[p] = rng.uniform(-0.2, 0.2, 3) * thr
            w[p, ax[p]] = rng.choice([-1, 1]) * float(_ulp_steps(f32(b[ax[p]] / 2), int(rng.integers(-3, 4))))
        c[3:, :, f] = (b * n + w).astype(np.float32)
    c[3, :, 0] = (f32(1228.8972), 0.0, 0.0)
    ch = np.zeros(3 + per, np.uint32)
    ch[3:] = 1 + np.arange(per) % 2  # partners of two chains: partner-partner pairs are periodic as well
    return c, BOXES.copy(), ch


def _host_checks(c, bx, thr):
    """The case set is meaningful: the former fixed-band contact rule misjudges some origin-partner pairs, and many of the
    reference's fl(b n) are inexact."""
    d = np.moveaxis(f32(0.0) - c[3:], 2, 1).reshape(-1, 3)         # (partners * F, 3) differences origin - partner
    b = np.repeat(bx.T[None], c.shape[0] - 3, axis=0).reshape(-1, 3)
    T = cs.threshold_d2(thr)
    want = np.sqrt(cs.reference_d2(d, b)) <= f32(thr)
    old_wrong = np.zeros(len(d), bool)
    for contract in (False, True):
        dec, got = cs.decide_before_fix(d, b, T, contract)
        old_wrong |= dec & (got != want)
    with np.errstate(all="ignore"):
        n = np.round(d.astype(np.float64) / b)
    inexact = (b.astype(np.float64) * n) != (b * n.astype(f32)).astype(np.float64)
    assert old_wrong.sum() >= 10 and (old_wrong[0] or thr != 3.0), int(old_wrong.sum())
    assert inexact.any(axis=1).mean() > 0.3
    assert want.sum() > 50 and (~want).sum() > 50


@pytest.fixture(scope="module")
def du():
    from moleculekit_b200 import distance_utils

    return distance_utils


@pytest.mark.parametrize("thr", [3.0, 8.0])
def test_k3_far_images_every_mode(du, oracle, thr):
    """dense distances (bits), contact maps with and without truncate (booleans of the reference's distances), fast
    distances within their documented 2e-6; self and non-self"""
    c, bx, ch = _far_case(thr, seed=int(thr * 10))
    _host_checks(c, bx, thr)
    N = c.shape[0]
    s1 = np.arange(0, 3, dtype=np.uint32)
    s2 = np.arange(3, N, dtype=np.uint32)
    sall = np.arange(N, dtype=np.uint32)
    F = c.shape[2]
    for selfd, a, b in ((False, s1, s2), (True, sall, sall)):
        P = du.n_columns(len(a), len(b), selfd)
        want = np.zeros((F, P), np.float32)
        oracle.dist_trajectory(c, bx, a, b, ch, selfd, True, want)
        got = np.zeros((F, P), np.float32)
        du.dist_trajectory(c, bx, a, b, ch, selfd, True, got)
        bad = np.flatnonzero(_bits(got) != _bits(want))
        assert bad.size == 0, ("distances", selfd, bad[:5])
        con = du.dist_trajectory(c, bx, a, b, ch, selfd, True, None, metric="contacts", threshold=thr)
        bad = np.flatnonzero(con != (want <= f32(thr)))
        assert bad.size == 0, ("contacts", selfd, bad[:5], want.reshape(-1)[bad[:5]])
        if not selfd:
            assert con[0, 0], "the named far contact (1228.8972 in a 34.0527 box) is a contact"
            assert (np.abs(want - f32(thr)) < 1e-5 * thr).sum() > 20  # pairs really sit at the threshold
        for tr in (thr * 1.5, thr * 0.75):
            ct = du.dist_trajectory(c, bx, a, b, ch, selfd, True, None, metric="contacts", threshold=thr, truncate=tr)
            wt = want.copy(); wt[wt > f32(tr)] = f32(tr)
            assert np.array_equal(ct, wt <= f32(thr)), ("contacts+truncate", selfd, tr)
        fast = np.zeros((F, P), np.float32)
        du.dist_trajectory(c, bx, a, b, ch, selfd, True, fast, exact=False)
        np.testing.assert_allclose(fast, want, rtol=2e-6, atol=0, err_msg=f"fast selfdist={selfd}")


@pytest.mark.parametrize("thr", [3.0, 8.0])
def test_k4_far_images_count_and_fill(du, oracle, monkeypatch, thr):
    """ordered contact lists: count + fill from the count's ballots, and with the distances evaluated again"""
    c, bx, ch = _far_case(thr, seed=int(thr * 10) + 1)
    N = c.shape[0]
    s1 = np.arange(0, 3, dtype=np.uint32); s2 = np.arange(3, N, dtype=np.uint32); sall = np.arange(N, dtype=np.uint32)
    for selfd, a, b in ((False, s1, s2), (True, sall, sall)):
        want = oracle.contacts_trajectory(c, bx, a, b, ch, selfd, True, thr)
        assert sum(len(x) for x in want) > 40
        assert du.contacts_trajectory(c, bx, a, b, ch, selfd, True, thr) == want, (selfd, "ballots")
        with monkeypatch.context() as m:
            m.setenv("MKB_K4_NO_BALLOTS", "1")
            assert du.contacts_trajectory(c, bx, a, b, ch, selfd, True, thr) == want, (selfd, "recomputed")


def test_k5_far_groups_thread_and_warp_kernels(du, oracle, monkeypatch):
    """group minimum distances and COM distances with groups many boxes apart: the thread-per-pair kernel (>= 4096
    small group pairs per frame) and the warp kernel (MKB_K5_WARP)"""
    c, bx, ch = _far_case(3.0, seed=5, per=400)
    N = c.shape[0]
    F = c.shape[2]
    rng = np.random.default_rng(6)
    perm = 3 + rng.permutation(N - 3)
    groups = [perm[i:i + 5].tolist() for i in range(0, 400, 5)]                 # 80 groups of 5 far partners
    g1 = [[0], [1], [2]] + groups[:67]                                         # 70 x 80 = 5600 group pairs
    gc1 = np.array([0, 0, 0] + [1 + k % 2 for k in range(67)], np.uint32)
    gc2 = np.array([2 - k % 2 for k in range(80)], np.uint32)
    masses = rng.uniform(1, 16, N).astype(np.float32)
    for r1, r2 in ((0, 0), (1, 0), (1, 1)):
        want = np.zeros((F, len(g1) * len(groups)), np.float32)
        oracle.dist_trajectory_reduction(c, bx, g1, groups, gc1, gc2, False, True, masses, r1, r2, want)
        got = np.zeros_like(want)
        du.dist_trajectory_reduction(c, bx, g1, groups, gc1, gc2, False, True, masses, r1, r2, got)
        assert np.array_equal(_bits(got), _bits(want)), (r1, r2, "thread")
        with monkeypatch.context() as m:
            m.setenv("MKB_K5_WARP", "1")
            warp = np.zeros_like(want)
            du.dist_trajectory_reduction(c, bx, g1, groups, gc1, gc2, False, True, masses, r1, r2, warp)
        assert np.array_equal(_bits(warp), _bits(want)), (r1, r2, "warp")
    P = du.n_columns(len(groups), len(groups), True)
    want = np.zeros((F, P), np.float32)
    oracle.dist_trajectory_reduction(c, bx, groups, groups, gc2, gc2, True, True, masses, 0, 0, want)
    got = np.zeros_like(want)
    du.dist_trajectory_reduction(c, bx, groups, groups, gc2, gc2, True, True, masses, 0, 0, got)
    assert np.array_equal(_bits(got), _bits(want))


def test_k8_far_shells(du, oracle):
    """radial shell counts with shell edges at the thresholds the partners sit on"""
    c, bx, ch = _far_case(3.0, seed=7)
    N = c.shape[0]
    F = c.shape[2]
    s1 = np.arange(0, 3, dtype=np.uint32); s2 = np.arange(3, N, dtype=np.uint32)
    edges = np.array([0.0, 1.5, 3.0, 4.5, 6.0, 12.0])
    for tr in (None, 4.5):
        want_d = np.zeros((F, 3 * len(s2)), np.float32)
        oracle.dist_trajectory(c, bx, s1, s2, ch, False, True, want_d)
        if tr is not None:
            want_d[want_d > f32(tr)] = f32(tr)
        dd = want_d.reshape(F, 3, len(s2)).astype(np.float64)
        want = np.stack([((dd > edges[e]) & (dd <= edges[e + 1])).sum(axis=2) for e in range(len(edges) - 1)], axis=2)
        got = du.shell_counts(c, bx, s1, s2, ch, False, True, edges, truncate=tr)
        assert np.array_equal(got, want), tr
        assert want[:, :, 1].sum() > 20


def test_k12_far_hbonds(oracle):
    """hydrogen bonds between waters displaced by up to 2^20 boxes: distance and angle criteria on the minimum image"""
    from moleculekit_b200 import hbonds
    from test_hbonds_gpu import _water_box

    rng = np.random.default_rng(43)
    coords, box, donors, acc = _water_box(rng, 400, 6, 24.6)
    n = rng.choice(FAR_N, size=(400, 3, 1)) * rng.choice([-1, 1], size=(400, 3, 1))
    coords = (coords.astype(np.float64) + np.repeat(n, 3, axis=0) * box[None].astype(np.float64)).astype(np.float32)
    N = coords.shape[0]
    s1 = np.ones(N, np.uint32)
    half = (np.arange(N) // 3 % 2 == 0).astype(np.uint32)
    total = 0
    for sa, sb, intra in ((s1, s1, True), (half, 1 - half, False)):
        for dth, ath in ((2.5, 120.0), (3.2, 100.0)):
            want = oracle.hbonds_calculate(donors, acc, coords, box, sa, sb, dth, ath, intra, False)
            got = hbonds.calculate(donors, acc, coords, box, sa, sb, dist_threshold=dth, angle_threshold=ath, intra=intra)
            assert got == want, (intra, dth, ath)
            total += sum(len(x) for x in got) // 3
    assert total > 200


def test_k13_far_rings(oracle):
    """pi-pi, cation-pi and sigma-hole detectors with partners up to 2^20 boxes from the rings"""
    from moleculekit_b200 import ringpairs
    from test_rings_gpu import _arrays, _check

    rng = np.random.default_rng(22)
    nr, N, F = 30, 180 + 300, 8
    L = (18.0 * (1 + 0.01 * rng.normal(size=(3, F)))).astype(np.float32)
    xyz = rng.uniform(0, 18, size=(N, 3, F))
    for r in range(nr):
        ctr = rng.uniform(0, 18, size=(3, 1)) + np.cumsum(rng.normal(0, .2, size=(3, F)), axis=1)
        u = rng.normal(size=3); u /= np.linalg.norm(u); v = np.cross(u, rng.normal(size=3)); v /= np.linalg.norm(v)
        for j in range(6):
            xyz[6 * r + j] = (ctr + 1.39 * (np.cos(j * np.pi / 3) * u[:, None] + np.sin(j * np.pi / 3) * v[:, None])
                              + rng.normal(0, .05, size=(3, F)))
    shift = np.zeros((N, 3, 1))
    shift[6 * nr:] = rng.choice(FAR_N, size=(N - 6 * nr, 3, 1)) * rng.choice([-1, 1], size=(N - 6 * nr, 3, 1))
    ring_shift = rng.choice(FAR_N[:12], size=(nr, 3, 1)) * rng.choice([-1, 1], size=(nr, 3, 1))
    shift[:6 * nr] = np.repeat(ring_shift, 6, axis=0)
    xyz = (xyz + shift * L[None].astype(np.float64)).astype(np.float32)
    ra = np.arange(6 * nr, dtype=np.uint32); st = np.arange(0, 6 * nr + 1, 6, dtype=np.uint32)
    cations = np.arange(6 * nr, N, dtype=np.uint32)
    hal = np.stack([cations, np.roll(cations, 1)], 1).astype(np.uint32)
    hits = 0
    for mode, fn, args in ((0, ringpairs.pipi_calculate, (ra, st, st, xyz, L, 5.5, 30.0, 7.5, 60.0)),
                           (1, ringpairs.cationpi_calculate, (ra, st, cations, xyz, L, 6.0, 45.0)),
                           (2, ringpairs.sigmahole_calculate, (ra, st, hal, xyz, L, 6.0, 30.0))):
        wc, wp, wd = _arrays(oracle.ring_interactions(mode, *args))
        _check(fn(*args), wp, wd, wc)
        hits += len(wp)
    assert hits > 100


def test_k9_far_groups_wrap(oracle):
    """rectangular wrapping (K9) and the triclinic / compact / rectangular unit cells (K9b) of groups that drifted many
    boxes away"""
    from moleculekit_b200.wrapping import wrap_box
    from test_wrapping_gpu import TRIC_MODES, _dodecahedron, _fbits, _gpu_tric, _oracle_tric, _solvated

    rng = np.random.default_rng(29)
    groups, coords, box = _solvated(rng, 90, 400, 6, box_edge=30.0)
    n = rng.choice(FAR_N, size=(400, 1, 3, 1)) * rng.choice([-1, 1], size=(400, 1, 3, 1))
    far = coords.copy()
    far[90:] = (coords[90:].astype(np.float64) + np.repeat(n, 3, axis=1).reshape(1200, 3, 1) * box[None]).astype(np.float32)
    centersel = np.arange(0, 90, 3, dtype=np.uint32)
    zero = np.zeros(3, np.float32)
    want = far.copy(); oracle.wrap_box(groups, want, box, centersel, zero)
    got = far.copy(); wrap_box(groups, got, box, centersel, zero)
    assert np.array_equal(_fbits(got), _fbits(want))
    # the triclinic cells step one cell vector per iteration (the reference's `while` loops): keep them within 1025 cells
    bv = _dodecahedron(rng, 6, L=31.0)
    nt = rng.choice(FAR_N[:14], size=(400, 1, 3, 1)) * rng.choice([-1, 1], size=(400, 1, 3, 1))
    tric = coords.copy()
    tric[90:] = (coords[90:].astype(np.float64) + np.repeat(nt, 3, axis=1).reshape(1200, 3, 1) * 31.0).astype(np.float32)
    for name, mode in TRIC_MODES:
        want = tric.copy(); _oracle_tric(oracle, mode, groups, want, bv, centersel, zero)
        got = tric.copy(); _gpu_tric(mode, groups, got, bv, centersel, zero)
        assert np.array_equal(_fbits(got), _fbits(want)), name
