"""GPU parity of the hydrogen-bond (K12) and ring (K13) kernels at their cut-offs: every probe of tests/cutoff_probes.py (one
frame each, its cosine, dot product or squared distance on a transition float or 1-3 floats from it) through
`hbonds.calculate` and `ringpairs.*_calculate` against the oracle -- identical pair lists in identical order, equal per-frame
counts, bit-identical distances, angles within one float ulp of acos of the known dot product.  Also the warp edges of
the count / fill kernels, rings of 3 to 8 atoms, and identical ring sets."""
import math

import numpy as np
import pytest

import cutoff_probes as cp

pytestmark = pytest.mark.gpu

ANGLE_TOL = 2e-5  # degrees, as tests/test_rings_gpu.py


@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    s = cp.run_scan(tmp_path_factory.mktemp("acosf_scan"))
    if s is None:
        pytest.skip("no host C compiler")
    return s


def _ring_arrays(res):
    pairs, da = res
    return (np.array([len(x) // 2 for x in pairs]), np.array([v for x in pairs for v in x], np.int32).reshape(-1, 2),
            np.array([v for x in da for v in x], np.float32).reshape(-1, 2))


def _angle_candidates(dot, to_plane):
    """the reported angle for a dot product, with acos rounded to float correctly or one float either side"""
    r = np.float32(math.acos(float(dot)))
    out = []
    for a in (np.nextafter(r, np.float32(-1)), r, np.nextafter(r, np.float32(4))):
        ang = float(a) * cp.ANGLE_SCALE
        if ang > 90.0:
            ang = 180.0 - ang
        if to_plane:
            ang = 90.0 - ang
        out.append(np.float32(ang))
    return out


def _check_parity(ps, want, got):
    if ps.kind == "hb":
        assert got == want, ps.name
        return cp.hits_of(ps, got)
    wc, wp, wd = _ring_arrays(want)
    gc, gp, gd = _ring_arrays(got)
    assert np.array_equal(gc, wc), ps.name
    assert np.array_equal(gp, wp), ps.name
    assert np.array_equal(gd[:, 0].view(np.uint32), wd[:, 0].view(np.uint32)), ps.name
    assert np.allclose(gd[:, 1], wd[:, 1], rtol=0, atol=ANGLE_TOL), ps.name
    hits = cp.hits_of(ps, got)
    if ps.what and ps.what[0] == "dot":  # the dot product is known exactly: the angle against float64 acos
        for row, f in enumerate(np.flatnonzero(hits)):
            assert gd[row, 1] in _angle_candidates(ps.value[f], ps.kind != "pipi"), (ps.name, f, gd[row, 1])
    return hits


def test_cutoff_probes_vs_oracle(oracle, scan):
    """every probe set: device == oracle; every boundary group holds both outcomes and its transition float"""
    total = groups = 0
    for ps in cp.angle_sets(scan) + cp.distance_sets():
        hits = _check_parity(ps, cp.call(ps, oracle), cp.call(ps, None))
        for name, frames in ps.groups().items():
            assert hits[frames].any() and not hits[frames].all(), (ps.name, name)
            assert any(ps.edge[f] for f in frames), (ps.name, name)
            groups += 1
        total += len(ps)
    assert total > 2000 and groups > 150


def test_hbond_clamped_and_degenerate_probes(oracle):
    """collinear D-H-A whose cosine rounds past +-1, H on A or D, NaN / infinite coordinates, ignore_hs with a failing
    angle: the expected decisions, as the oracle"""
    ps, ign = cp.hb_special_sets()
    hits = _check_parity(ps, cp.call(ps, oracle), cp.call(ps, None))
    cl = cp.hb_clamp_pairs()
    n, m = len(cl[1]), len(cl[1]) + len(cl[-1])
    assert not hits[:n].any() and hits[n:m].all()              # c > 1 clamps to angle 0, c < -1 to 180
    assert not hits[m] and not hits[m + 1] and hits[m + 2]     # H on A, H on D, straight D-H-A
    assert not hits[m + 3:].any()                              # NaN / infinite coordinates
    assert list(_check_parity(ign, cp.call(ign, oracle), cp.call(ign, None))) == [True, True, False, True]


def _hit_patterns(n, rng):
    pats = [np.zeros(n, bool), np.ones(n, bool)]
    for lanes in ([31, 63], [n - 1], [0, 31, 32, 63, 64], [40], [30, 31], [n // 2]):
        p = np.zeros(n, bool)
        p[[i for i in lanes if i < n]] = True
        pats.append(p)
    pats.append(rng.random(n) < 0.3)
    p = rng.random(n) < 0.5
    p[min(n - 1, 40):] = False  # the last hit ends mid-chunk
    pats.append(p)
    return pats


@pytest.mark.parametrize("n2", [1, 31, 32, 33, 63, 64, 65, 1000])
def test_warp_edges(oracle, n2):
    """rows of n2 partners with hits on a chunk's last lane, rows whose last hit ends mid-chunk, empty and full rows: the
    fill kernels stop at the row's end and rank hits by ballot; K12 donor rows and K13 cation-pi / pi-pi rows"""
    from moleculekit_b200 import hbonds, ringpairs

    rng = np.random.default_rng(n2)
    pats = _hit_patterns(n2, rng)
    F = len(pats)
    # K12: H 0 at the origin with D 1 behind it; a second donor far away (a row with no bond); acceptors at 2.. on a line
    xyz = np.zeros((4 + n2, 3, F), np.float32)
    xyz[1, 0] = -1
    xyz[2, 0], xyz[3, 0] = 100, 101
    for f, p in enumerate(pats):
        xyz[4:, 0, f] = np.where(p, 2.0, 10.0)
        xyz[4:, 1, f] = np.arange(n2) * 1e-3
    box = np.zeros((3, F), np.float32)
    don = np.array([[1, 0], [3, 2]], np.uint32)
    acc = np.arange(4, 4 + n2, dtype=np.uint32)
    ones = np.ones(4 + n2, np.uint32)
    want = oracle.hbonds_calculate(don, acc, xyz, box, ones, ones, 2.5, 120.0, True, False)
    got = hbonds.calculate(don, acc, xyz, box, ones, ones, dist_threshold=2.5, angle_threshold=120.0, intra=True)
    assert got == want
    assert [len(x) // 3 for x in got] == [int(p.sum()) for p in pats]
    # K13 cation-pi: the hexagon at the origin, cations 3 above it (hit) or 30 away
    xyz = np.zeros((6 + n2, 3, F), np.float32)
    xyz[:6] = cp.HEX[:, :, None]
    for f, p in enumerate(pats):
        xyz[6:, 2, f] = np.where(p, 3.0, 30.0)
        xyz[6:, 0, f] = np.arange(n2) * 1e-3
    ra, st = np.arange(6, dtype=np.uint32), np.array([0, 6], np.uint32)
    cat = np.arange(6, 6 + n2, dtype=np.uint32)
    args = (ra, st, cat, xyz, box, 5.0, 60.0)
    wc, wp, wd = _ring_arrays(oracle.ring_interactions(1, *args))
    gc, gp, gd = _ring_arrays(ringpairs.cationpi_calculate(*args))
    assert np.array_equal(gc, wc) and np.array_equal(gp, wp)
    assert np.array_equal(gd[:, 0], wd[:, 0]) and np.allclose(gd[:, 1], wd[:, 1], rtol=0, atol=ANGLE_TOL)
    assert list(gc) == [int(p.sum()) for p in pats]
    # K13 pi-pi: n2 3-atom rings stacked 3 above the hexagon (hit) or 30 away
    xyz = np.zeros((6 + 3 * n2, 3, F), np.float32)
    xyz[:6] = cp.HEX[:, :, None]
    tri = np.array([[1, 0, 0], [0, 1, 0], [-1, -1, 0]], np.float32)
    for f, p in enumerate(pats):
        for k in range(n2):
            xyz[6 + 3 * k:9 + 3 * k, :, f] = tri + np.float32([k * 1e-3, 0, 3.0 if p[k] else 30.0])
    ra = np.arange(6 + 3 * n2, dtype=np.uint32)
    st2 = np.arange(6, 6 + 3 * n2 + 1, 3, dtype=np.uint32)
    args = (ra, st, st2, xyz, box, 4.4, 30.0, 5.5, 60.0)
    wc, wp, wd = _ring_arrays(oracle.ring_interactions(0, *args))
    gc, gp, gd = _ring_arrays(ringpairs.pipi_calculate(*args))
    assert np.array_equal(gc, wc) and np.array_equal(gp, wp)
    assert np.array_equal(gd[:, 0], wd[:, 0]) and np.allclose(gd[:, 1], wd[:, 1], rtol=0, atol=ANGLE_TOL)
    assert list(gc) == [int(p.sum()) for p in pats]


def test_ring_sizes_vs_oracle(oracle):
    """rings of 3, 4, 5, 7 and 8 atoms (centroids divided by counts that are not powers of two) in a periodic box, the three
    detectors against the oracle"""
    from moleculekit_b200 import ringpairs

    rng = np.random.default_rng(8)
    sizes = [3, 4, 5, 7, 8] * 6
    F, n_part = 40, 200
    na = sum(sizes)
    L = (16.0 * (1 + 0.01 * rng.normal(size=(3, F)))).astype(np.float32)
    xyz = (rng.uniform(0, 16, size=(na + n_part, 3, F)) + rng.integers(-2, 3, size=(na + n_part, 3, 1)) * 16.0)
    pos = 0
    for n in sizes:
        ctr = rng.uniform(0, 16, size=(3, 1)) + np.cumsum(rng.normal(0, .2, size=(3, F)), axis=1)
        u = rng.normal(size=3); u /= np.linalg.norm(u); v = np.cross(u, rng.normal(size=3)); v /= np.linalg.norm(v)
        for j in range(n):
            xyz[pos + j] = ctr + 1.4 * (np.cos(2 * np.pi * j / n) * u[:, None] + np.sin(2 * np.pi * j / n) * v[:, None])
        pos += n
    xyz = xyz.astype(np.float32)
    ra = np.arange(na, dtype=np.uint32)
    st = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    part = np.arange(na, na + n_part, dtype=np.uint32)
    hal = np.stack([part, np.roll(part, 1)], 1).astype(np.uint32)
    hits = 0
    for mode, fn, args in ((0, ringpairs.pipi_calculate, (ra, st, st, xyz, L, 6.5, 40.0, 8.0, 50.0)),
                           (1, ringpairs.cationpi_calculate, (ra, st, part, xyz, L, 6.0, 30.0)),
                           (2, ringpairs.sigmahole_calculate, (ra, st, hal, xyz, L, 6.0, 20.0))):
        wc, wp, wd = _ring_arrays(oracle.ring_interactions(mode, *args))
        gc, gp, gd = _ring_arrays(fn(*args))
        assert np.array_equal(gc, wc) and np.array_equal(gp, wp), mode
        assert np.array_equal(gd[:, 0].view(np.uint32), wd[:, 0].view(np.uint32)), mode
        assert np.allclose(gd[:, 1], wd[:, 1], rtol=0, atol=ANGLE_TOL), mode
        for size in set(sizes):  # every ring size takes part
            assert np.isin(wp[:, 0], np.flatnonzero(np.diff(st) == size)).any(), (mode, size)
        hits += len(wp)
    assert hits > 1000


def test_identical_ring_sets(oracle):
    """the same ring list as both pi-pi sets: ringpairs skips each ring against itself (equal start indexes), as the
    reference's kernel; the interactions mirror offsets the second set's starts, as the reference's interactions.py, so the
    self-pairs come back at distance 0"""
    from moleculekit_b200 import ringpairs
    from moleculekit_b200.interactions import pipi_calculate

    rng = np.random.default_rng(4)
    F, nr = 5, 12
    xyz = np.zeros((6 * nr, 3, F), np.float32)
    for r in range(nr):
        xyz[6 * r:6 * r + 6] = (cp.HEX[:, :, None] * 0.7 + rng.uniform(0, 9, size=(1, 3, F))).astype(np.float32)
    box = np.full((3, F), 12.0, np.float32)
    ra = np.arange(6 * nr, dtype=np.uint32)
    st = np.arange(0, 6 * nr + 1, 6, dtype=np.uint32)
    args = (ra, st, st, xyz, box, 4.4, 30.0, 5.5, 60.0)
    wc, wp, wd = _ring_arrays(oracle.ring_interactions(0, *args))
    gc, gp, gd = _ring_arrays(ringpairs.pipi_calculate(*args))
    assert np.array_equal(gc, wc) and np.array_equal(gp, wp) and np.array_equal(gd[:, 0], wd[:, 0])
    assert len(gp) > 0 and not np.any(gp[:, 0] == gp[:, 1])

    class Mol:
        numAtoms, numFrames = 6 * nr, F

    Mol.coords, Mol.box = xyz, box
    rings = [ra[6 * r:6 * r + 6] for r in range(nr)]
    pp, da = pipi_calculate(Mol, rings, rings)
    ra2 = np.concatenate([ra, ra]).astype(np.uint32)
    want_c, want_p, want_d = _ring_arrays(oracle.ring_interactions(0, ra2, st, st + st[-1], xyz, box, 4.4, 30, 5.5, 60))
    got_p = np.array([p for fr in pp for p in fr], np.int32).reshape(-1, 2)
    got_d = np.array([d for fr in da for d in fr], np.float32).reshape(-1, 2)
    assert np.array_equal(got_p, want_p) and [len(x) for x in pp] == list(want_c)
    assert np.array_equal(got_d[:, 0], want_d[:, 0])
    self_pairs = got_p[:, 0] == got_p[:, 1]
    assert self_pairs.sum() == nr * F and np.all(got_d[self_pairs, 0] == 0)
