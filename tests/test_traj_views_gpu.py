"""GPU tests of the pair kernels on the trajectory layouts their entry points take in place.

Every entry point that takes an `mkb_traj` accepts a frame slice of a resident trajectory without a copy: `coords + f0`
with `frame_stride` = the resident tensor's frame count, and a box with its own `frame_stride_box` (a one-frame box is
normalised to stride 1).  Sharding, the projections and users who walk a long device trajectory in windows rely on it.
With contiguous inputs the three numbers are equal, so a kernel that mixes them up passes every contiguous test.

1. One seeded periodic system (coordinates and box change every frame, atoms outside the box, two chain ids) run through
   K3 (distances, fast mode, contact maps, self distances, truncate), K4 (ordered contacts, with and without cached
   ballots), K5 (group reductions, thread and warp kernels), K8 (radial shells), K12 (hydrogen bonds) and K13 (ring
   interactions) on frame slices with the box in a longer tensor, with the box copied, one frame, and frame counts at the
   32-frame gather tiles: every view gives the bits of the contiguous layout, and the contiguous layout the oracle's.
2. Trajectories longer than the 65 535 frames of one K3 launch (grid z), the ordinary input of MetricDistance for
   Markov-model work: every frame against the oracle, and K5 on both sides of its thread-kernel frame limit.
3. The K4 count -> fill ballot cache across two views that share every pointer and differ only in frame stride.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ANGLE_TOL = 2e-5  # degrees, as tests/test_rings_gpu.py: emitted angles come from the device's acos


def _bits(a):
    """float32 bit patterns with NaNs canonicalised (x86 and the GPU produce different NaN words)"""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


def _same(a, b):
    """bit equality of two device tensors: float32 compared as int32 words"""
    import torch

    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


def _unit(v, axis):
    return v / np.linalg.norm(v, axis=axis, keepdims=True)


def _rings(rng, n, F, lo, hi):
    """n planar hexagons (1.39 A) whose centres (uniform in [lo, hi)) and orientations are drawn anew every frame,
    each displaced by a whole number of 24 A as one piece: (6 n, 3, F)"""
    ctr = rng.uniform(lo, hi, size=(n, 3, F)) + rng.integers(-2, 3, size=(n, 3, 1)) * 24.0
    u = _unit(rng.normal(size=(n, 3, F)), 1)
    v = _unit(np.cross(u, rng.normal(size=(n, 3, F)), axis=1), 1)
    ang = np.arange(6) * np.pi / 3
    atoms = ctr[:, None] + 1.39 * (np.cos(ang)[None, :, None, None] * u[:, None] + np.sin(ang)[None, :, None, None] * v[:, None])
    return atoms.reshape(6 * n, 3, F)


def _rows_ok(off, rows, want, width):
    """Per frame: are the device's rows off[f]:off[f+1] the oracle's flat list want[f]?"""
    cnt_w = np.array([len(x) // width for x in want], dtype=np.int64)
    ok = np.diff(off) == cnt_w
    if ok.all():
        flat = np.array([v for x in want for v in x], dtype=rows.dtype).reshape(-1, width)
        bad_rows = ~np.all(rows == flat, axis=1)
        ok &= np.bincount(np.repeat(np.arange(len(want)), cnt_w)[bad_rows], minlength=len(want)) == 0
    return ok


# ------------------------------------------------------------------------------------------ 1. layouts of one system
N_RING, N_DON, N_FREE = 12, 40, 248
N = 6 * N_RING + 2 * N_DON + N_FREE
FB = 100          # frames of the resident box tensor
THR = 8.0         # K3 contact threshold
TRUNC = 11.5      # K3 truncate
CT_THR = 7.5      # K4 threshold
NS, SW = 5, 2.5   # K8 shells
HB = (3.2, 100.0)  # K12 distance, angle
RING_P = {0: (6.5, 40.0, 7.5, 50.0), 1: (6.5, 30.0), 2: (6.5, 30.0)}

# (name, frames of the resident coords tensor, f0, f1, box): "slice" = box[:, f0:f1] of the 100-frame box tensor
# (frame_stride_box 100, or 1 for one frame), "copy" = that slice made contiguous (frame_stride_box = n_frames)
LAYOUTS = (("slices", 64, 7, 47, "slice"), ("slice_boxcopy", 64, 7, 47, "copy"), ("one_frame", 64, 29, 30, "slice"),
           ("F1", 97, 50, 51, "slice"), ("F31", 97, 3, 34, "slice"), ("F32", 97, 33, 65, "slice"),
           ("F33", 97, 60, 93, "slice"), ("F65", 97, 31, 96, "slice"))


@pytest.fixture(scope="module")
def psys():
    """400 atoms over 100 frames: 12 rings, 40 donor heavy atoms with their hydrogens, 248 free atoms; a box of 18 to 30 A
    per axis and frame; every molecule displaced by up to two 24 A steps, so most atoms lie outside the box."""
    import torch

    assert torch.cuda.is_available()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(20261017)
    box = rng.uniform(18.0, 30.0, size=(3, FB)).astype(np.float32)
    ring = _rings(rng, N_RING, FB, 0.0, 24.0)
    heavy = rng.uniform(0.0, 24.0, size=(N_DON, 3, FB)) + rng.integers(-2, 3, size=(N_DON, 3, 1)) * 24.0
    hyd = heavy + _unit(rng.normal(size=(N_DON, 3, FB)), 1)
    free = rng.uniform(0.0, 24.0, size=(N_FREE, 3, FB)) + rng.integers(-2, 3, size=(N_FREE, 3, 1)) * 24.0
    c = np.concatenate([ring, heavy, hyd, free]).astype(np.float32)
    d0, h0, f0 = 6 * N_RING, 6 * N_RING + N_DON, 6 * N_RING + 2 * N_DON
    p = dict(dev=dev)
    p["ch"] = rng.integers(1, 3, N).astype(np.uint32)   # two chain ids: same-chain pairs are not wrapped
    p["s1"] = np.sort(rng.choice(N, 40, replace=False)).astype(np.uint32)
    p["s2"] = np.sort(rng.choice(N, 300, replace=False)).astype(np.uint32)   # > 256: both column halves of K3's threads
    p["sself"] = np.sort(rng.choice(N, 260, replace=False)).astype(np.uint32)
    p["masses"] = rng.uniform(1.0, 16.0, N).astype(np.float32)
    groups = lambda n: [np.sort(rng.choice(N, k, replace=False)).tolist() for k in rng.integers(1, 4, n)]
    p["g1"], p["g2"] = groups(90), groups(70)
    p["gp1"], p["gp2"] = groups(4100), groups(4100)   # pairs=True: 4100 group pairs per frame
    p["donors"] = np.stack([np.arange(d0, h0), np.arange(h0, f0)], 1).astype(np.uint32)
    p["acceptors"] = np.concatenate([np.arange(d0, h0), np.arange(f0, f0 + 80)]).astype(np.uint32)
    p["hsel1"] = rng.integers(0, 2, N).astype(np.uint32)
    p["ring_atoms"] = np.arange(6 * N_RING, dtype=np.uint32)
    p["ring_starts"] = np.arange(0, 6 * N_RING + 1, 6, dtype=np.uint32)
    p["cations"] = np.arange(f0 + 80, f0 + 140, dtype=np.uint32)
    p["halogens"] = np.stack([np.arange(f0 + 140, f0 + 170), np.arange(f0 + 170, f0 + 200)], 1).astype(np.uint32)
    p["c64"], p["b64"] = np.ascontiguousarray(c[:, :, :64]), np.ascontiguousarray(box[:, :64])
    i32 = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to(dev)
    p["C64"], p["C97"] = torch.from_numpy(p["c64"]).to(dev), torch.from_numpy(np.ascontiguousarray(c[:, :, :97])).to(dev)
    p["B"] = torch.from_numpy(box).to(dev)
    p["B64"] = p["B"][:, :64].contiguous()
    for k in ("ch", "s1", "s2", "sself", "acceptors", "hsel1", "ring_atoms", "ring_starts", "cations", "halogens"):
        p["d_" + k] = i32(p[k])
    p["d_hsel2"] = i32(1 - p["hsel1"])
    p["d_ones"] = i32(np.ones(N, np.uint32))
    p["d_masses"] = torch.from_numpy(p["masses"]).to(dev)
    return p


def _views(p):
    """(name, view, contiguous copy) of every layout, after checking that `_lib.traj` passes the view in place with
    the intended strides (a silent copy would leave nothing to test)"""
    from moleculekit_b200 import _lib

    for name, fc, f0, f1, boxmode in LAYOUTS:
        vc = (p["C64"] if fc == 64 else p["C97"])[:, :, f0:f1]
        vb = p["B"][:, f0:f1]
        if boxmode == "copy":
            vb = vb.contiguous()
        F = f1 - f0
        t = _lib.traj(vc, vb)
        assert t.coords == vc.data_ptr() and t.n_frames == F and t.frame_stride == fc and t.frame_stride > t.n_frames, name
        assert t.frame_stride_box == (1 if F == 1 else F if boxmode == "copy" else FB), name
        if F > 1:
            assert t.box == vb.data_ptr(), name
        yield name, (vc, vb), (vc.contiguous(), vb.contiguous())


def _check_views(p, run):
    """run(coords, box) -> tuple of device tensors: bit-identical on every view and its contiguous copy"""
    for name, view, contig in _views(p):
        want, got = run(*contig), run(*view)
        assert len(got) == len(want) and all(_same(g, w) for g, w in zip(got, want)), name


K3_CASES = [(m, tr, sd, pbc) for m in ("exact", "fast", "contacts") for tr in (None, TRUNC) for sd in (False, True)
            for pbc in (True, False)]


@pytest.mark.parametrize("metric,truncate,selfdist,pbc", K3_CASES)
def test_dist_trajectory_views(psys, oracle, metric, truncate, selfdist, pbc):
    """K3 (contacts without truncate: DIST_CONTACTS_D2) on every layout; the contiguous result against the oracle:
    distances bit for bit, fast mode within the tolerance of test_distance_gpu.py, contact maps exactly"""
    from moleculekit_b200 import distance_utils as du

    p = psys
    k1, k2 = ("sself", "sself") if selfdist else ("s1", "s2")
    kw = dict(metric="contacts" if metric == "contacts" else "distances", truncate=truncate, threshold=THR,
              exact=metric != "fast")
    run = lambda c, b: (du.dist_trajectory_device(c, b, p["d_" + k1], p["d_" + k2], p["d_ch"], selfdist, pbc, **kw),)
    _check_views(p, run)
    got = run(p["C64"], p["B64"])[0].cpu().numpy()
    want = np.zeros(got.shape, np.float32)
    oracle.dist_trajectory(p["c64"], p["b64"], p[k1], p[k2], p["ch"], selfdist, pbc, want)
    if truncate is not None:
        want[want > truncate] = truncate
    if metric == "contacts":
        assert np.array_equal(got, want <= np.float32(THR)) and 0.002 < got.mean() < 0.5
    elif metric == "exact":
        assert np.array_equal(_bits(got), _bits(want))
    else:
        assert np.array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_allclose(got, want, rtol=2e-6, atol=0)
        ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert (ulps <= 4).mean() >= 0.999, ulps.max()
    assert not np.array_equal(want[0], want[1])  # the answer depends on the frame


@pytest.mark.parametrize("selfdist", (False, True))
@pytest.mark.parametrize("ballots", (True, False))
def test_contacts_views(psys, oracle, monkeypatch, ballots, selfdist):
    """K4 count + fill on every layout, with the ballots of the count pass and with MKB_K4_NO_BALLOTS (distances
    evaluated again in the fill); ordered pairs of the contiguous layout against the oracle"""
    from moleculekit_b200 import distance_utils as du

    p = psys
    if not ballots:
        monkeypatch.setenv("MKB_K4_NO_BALLOTS", "1")
    k1, k2 = ("sself", "sself") if selfdist else ("s1", "s2")
    run = lambda c, b: du.contacts_trajectory_device(c, b, p["d_" + k1], p["d_" + k2], p["d_ch"], selfdist, True, CT_THR)
    _check_views(p, run)
    off, pairs = run(p["C64"], p["B64"])
    want = oracle.contacts_trajectory(p["c64"], p["b64"], p[k1], p[k2], p["ch"], selfdist, True, CT_THR)
    ok = _rows_ok(off.cpu().numpy(), pairs.cpu().numpy().view(np.uint32), want, 2)
    assert ok.all(), np.flatnonzero(~ok)
    assert sum(map(len, want)) > 2000 and want[0] != want[1]


@pytest.mark.parametrize("truncate,selfdist", ((None, False), (9.0, False), (None, True), (9.0, True)))
def test_shell_counts_views(psys, oracle, truncate, selfdist):
    """K8 on every layout; the contiguous counts over the shell volumes equal the oracle's MetricShell densities"""
    import torch

    from moleculekit_b200 import distance_utils as du

    p = psys
    k1, k2 = ("sself", "sself") if selfdist else ("s1", "s2")
    edges = np.arange(SW * (NS + 1), step=SW)
    d_edges = torch.from_numpy(edges).to(p["dev"])
    run = lambda c, b: (du.shell_counts_device(c, b, p["d_" + k1], p["d_" + k2], p["d_ch"], selfdist, True, d_edges,
                                               truncate=truncate),)
    _check_views(p, run)
    counts = run(p["C64"], p["B64"])[0].cpu().numpy().astype(np.int64)
    vol = 4 / 3 * np.pi * (edges[1:] ** 3 - edges[:-1] ** 3)
    got = (counts / vol[None, None, :]).reshape(64, -1)
    want = oracle.metric_shell(p["c64"], p["b64"], p[k1], p[k2], p["ch"], selfdist, True, NS, SW, truncate)
    assert np.array_equal(got, want) and counts.sum() > 10000 and not np.array_equal(counts[0], counts[1])


K5_CASES = (("com_com", 1, 1, False, False), ("com_closest", 1, 0, False, False), ("closest_closest", 0, 0, False, False),
            ("self", 0, 0, True, False), ("pairs", 0, 0, False, True), ("pairs_com_closest", 1, 0, False, True))


@pytest.mark.parametrize("kernel", ("thread", "warp"))
@pytest.mark.parametrize("name,red1,red2,selfdist,pairs", K5_CASES)
def test_dist_reduction_views(psys, oracle, monkeypatch, kernel, name, red1, red2, selfdist, pairs):
    """K5 on every layout.  Groups of 1 to 3 atoms with >= 4096 group pairs per frame (90 x 70, 90 x 90 self, 4100 pairs)
    take the thread-per-pair kernel; MKB_K5_WARP=1 forces the warp kernel on the same input.  Contiguous result against
    the oracle, bit for bit."""
    import torch

    from moleculekit_b200 import distance_utils as du

    p = psys
    ga, gb = (p["gp1"], p["gp2"]) if pairs else (p["g1"], p["g1"] if selfdist else p["g2"])
    assert (len(ga) if pairs else len(ga) * len(gb)) >= 4096  # the host's rule for the thread kernel
    if kernel == "warp":
        monkeypatch.setenv("MKB_K5_WARP", "1")
    gca, gcb = (np.array([p["ch"][g[0]] for g in gs], np.uint32) for gs in (ga, gb))
    d_gca, d_gcb = (torch.from_numpy(x.view(np.int32)).to(p["dev"]) for x in (gca, gcb))
    run = lambda c, b: (du.dist_reduction_device(c, b, ga, gb, d_gca, d_gcb, selfdist, True, p["d_masses"], red1, red2,
                                                 pairs=pairs),)
    _check_views(p, run)
    got = run(p["C64"], p["B64"])[0].cpu().numpy()
    want = np.zeros(got.shape, np.float32)
    if pairs:
        oracle.dist_trajectory_reduction_pairs(p["c64"], p["b64"], ga, gb, gca, gcb, True, p["masses"], red1, red2, want)
    else:
        oracle.dist_trajectory_reduction(p["c64"], p["b64"], ga, gb, gca, gcb, selfdist, True, p["masses"], red1, red2, want)
    assert np.array_equal(_bits(got), _bits(want)) and not np.array_equal(want[0], want[1])


@pytest.mark.parametrize("intra", (True, False))
@pytest.mark.parametrize("ignore_hs", (False, True))
def test_hbonds_views(psys, oracle, intra, ignore_hs):
    """K12 on every layout, with hydrogens and with ignore_hs; contiguous triples against the oracle"""
    import torch

    from moleculekit_b200 import hbonds

    p = psys
    dn = p["donors"][:, :1] if ignore_hs else p["donors"]
    d_dn = torch.from_numpy(np.ascontiguousarray(np.hstack([dn, dn]) if ignore_hs else dn).view(np.int32)).to(p["dev"])
    sa, sb = (p["d_ones"], p["d_ones"]) if intra else (p["d_hsel1"], p["d_hsel2"])
    run = lambda c, b: hbonds.calculate_device(c, b, d_dn, p["d_acceptors"], sa, sb, *HB, intra=intra,
                                               ignore_hs=ignore_hs)
    _check_views(p, run)
    off, tri = run(p["C64"], p["B64"])
    h1, h2 = (np.ones(N, np.uint32),) * 2 if intra else (p["hsel1"], 1 - p["hsel1"])
    want = oracle.hbonds_calculate(dn, p["acceptors"], p["c64"], p["b64"], h1, h2, *HB, intra, ignore_hs)
    ok = _rows_ok(off.cpu().numpy(), tri.cpu().numpy(), want, 3)
    assert ok.all(), np.flatnonzero(~ok)
    assert sum(map(len, want)) // 3 > 300 and want[0] != want[1]


@pytest.mark.parametrize("mode", (0, 1, 2))
def test_ring_interactions_views(psys, oracle, mode):
    """K13 (0 pi-pi, 1 cation-pi, 2 sigma hole) on every layout, angles included bit for bit; contiguous pairs and
    distances against the oracle exactly, angles within ANGLE_TOL"""
    from moleculekit_b200 import ringpairs

    p = psys
    key = {0: "ring_starts", 1: "cations", 2: "halogens"}[mode]
    run = lambda c, b: ringpairs.calculate_device(mode, c, b, p["d_ring_atoms"], p["d_ring_starts"], p["d_" + key],
                                                  *RING_P[mode])
    _check_views(p, run)
    off, pairs, da = (x.cpu().numpy() for x in run(p["C64"], p["B64"]))
    res, dist = oracle.ring_interactions(mode, p["ring_atoms"], p["ring_starts"], p[key], p["c64"], p["b64"], *RING_P[mode])
    ok = _rows_ok(off, pairs, res, 2)
    assert ok.all(), np.flatnonzero(~ok)
    wda = np.array([v for x in dist for v in x], np.float32).reshape(-1, 2)
    assert np.array_equal(_bits(da[:, 0]), _bits(wda[:, 0]))
    assert np.allclose(da[:, 1], wda[:, 1], rtol=0, atol=ANGLE_TOL)
    assert len(wda) > 200 and res[0] != res[1]


# ------------------------------------------------------------------------------------------ 2. long trajectories
FL = 2 * 65535 + 7  # three K3 launches along grid z, the last one partial
LS1, LS2 = [0, 6, 12], [3, 9, 13, 14, 15]   # 15 pairs per frame
LSELF = [0, 3, 6, 9, 12, 14]                 # 15 pairs per frame
L_THR, L_TRUNC = 4.5, 5.25


@pytest.fixture(scope="module")
def lsys():
    """16 atoms over FL frames in a box of 10 to 16 A per axis and frame: two hexagonal rings (atoms 0-5, 6-11), a donor
    (12) with its hydrogen (13), two free atoms (14, 15); every position drawn anew each frame, mostly outside the box."""
    import torch

    assert torch.cuda.is_available()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(65536)
    box = rng.uniform(10.0, 16.0, size=(3, FL)).astype(np.float32)
    ring = _rings(rng, 2, FL, -8.0, 24.0)
    heavy = rng.uniform(-8.0, 24.0, size=(1, 3, FL))
    hyd = heavy + _unit(rng.normal(size=(1, 3, FL)), 1)
    free = rng.uniform(-8.0, 24.0, size=(2, 3, FL))
    c = np.concatenate([ring, heavy, hyd, free]).astype(np.float32)
    ch = np.array([1, 1, 1, 2, 2, 2, 1, 2, 1, 2, 1, 2, 1, 1, 2, 2], np.uint32)
    return dict(c=c, box=box, ch=ch, dev=dev, C=torch.from_numpy(c).to(dev), B=torch.from_numpy(box).to(dev),
                d_ch=torch.from_numpy(ch.view(np.int32)).to(dev))


def _frame_report(ok):
    """the failure message of a per-frame comparison: frames that differ, and the frames around the launch edges"""
    bad = np.flatnonzero(~ok)
    edges = {f: bool(ok[f]) for f in (65534, 65535, 65536, len(ok) - 1)}
    return f"{bad.size} of {len(ok)} frames differ (first {bad[:8].tolist()}); frame equal at the launch edges: {edges}"


def _i32(a, dev):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).to(dev)


@pytest.mark.parametrize("selfdist", (False, True))
@pytest.mark.parametrize("mode", ("exact", "fast", "contacts", "contacts_d2"))
def test_long_dist_trajectory(lsys, oracle, mode, selfdist):
    """K3 on 131 077 frames (three launches of up to 65 535 frames) in its four kernel modes, every frame against the
    oracle"""
    from moleculekit_b200 import distance_utils as du

    L = lsys
    a, b = (LSELF, LSELF) if selfdist else (LS1, LS2)
    truncate = L_TRUNC if mode == "contacts" else None
    out = du.dist_trajectory_device(L["C"], L["B"], _i32(a, L["dev"]), _i32(b, L["dev"]), L["d_ch"], selfdist, True,
                                    metric="contacts" if mode.startswith("contacts") else "distances", truncate=truncate,
                                    threshold=L_THR, exact=mode != "fast")
    got = out.cpu().numpy()
    want = np.zeros((FL, 15), np.float32)
    oracle.dist_trajectory(L["c"], L["box"], np.array(a, np.uint32), np.array(b, np.uint32), L["ch"], selfdist, True, want)
    if truncate is not None:
        want[want > truncate] = truncate
    if mode.startswith("contacts"):
        ok = np.all(got == (want <= np.float32(L_THR)), axis=1)
        assert 0.02 < got.mean() < 0.5
    elif mode == "exact":
        ok = np.all(_bits(got) == _bits(want), axis=1)
    else:
        ok = np.all(np.abs(got - want) <= 2e-6 * np.abs(want), axis=1)
        ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert (ulps <= 4).mean() >= 0.999, ulps.max()
    assert ok.all(), _frame_report(ok)


@pytest.mark.parametrize("selfdist", (False, True))
def test_long_contacts(lsys, oracle, selfdist):
    """K4 count + fill on 131 077 frames, ordered pairs of every frame against the oracle"""
    from moleculekit_b200 import distance_utils as du

    L = lsys
    a, b = (LSELF, LSELF) if selfdist else (LS1, LS2)
    off, pairs = du.contacts_trajectory_device(L["C"], L["B"], _i32(a, L["dev"]), _i32(b, L["dev"]), L["d_ch"], selfdist,
                                               True, L_THR)
    want = oracle.contacts_trajectory(L["c"], L["box"], np.array(a, np.uint32), np.array(b, np.uint32), L["ch"], selfdist,
                                      True, L_THR)
    ok = _rows_ok(off.cpu().numpy(), pairs.cpu().numpy().view(np.uint32), want, 2)
    assert ok.all(), _frame_report(ok)
    assert sum(map(len, want)) > 100000


def test_long_shells(lsys, oracle):
    """K8 on 131 077 frames against the oracle's MetricShell densities"""
    import torch

    from moleculekit_b200 import distance_utils as du

    L = lsys
    edges = np.arange(1.5 * 5, step=1.5)
    counts = du.shell_counts_device(L["C"], L["B"], _i32(LS1, L["dev"]), _i32(LS2, L["dev"]), L["d_ch"], False, True,
                                    torch.from_numpy(edges).to(L["dev"])).cpu().numpy().astype(np.int64)
    vol = 4 / 3 * np.pi * (edges[1:] ** 3 - edges[:-1] ** 3)
    got = (counts / vol[None, None, :]).reshape(FL, -1)
    want = oracle.metric_shell(L["c"], L["box"], np.array(LS1, np.uint32), np.array(LS2, np.uint32), L["ch"], False, True,
                               4, 1.5)
    ok = np.all(got == want, axis=1)
    assert ok.all(), _frame_report(ok)
    assert counts.sum() > 100000


@pytest.mark.parametrize("ignore_hs", (False, True))
def test_long_hbonds(lsys, oracle, ignore_hs):
    """K12 on 131 077 frames: donor 12 (hydrogen 13), acceptors 0, 6, 14, 15; triples of every frame against the oracle"""
    from moleculekit_b200 import hbonds

    L = lsys
    dn = np.array([[12, 12]] if ignore_hs else [[12, 13]], np.uint32)
    acc = np.array([0, 6, 14, 15], np.uint32)
    ones = np.ones(16, np.uint32)
    off, tri = hbonds.calculate_device(L["C"], L["B"], _i32(dn, L["dev"]), _i32(acc, L["dev"]), _i32(ones, L["dev"]),
                                       _i32(ones, L["dev"]), 3.2, 100.0, intra=True, ignore_hs=ignore_hs)
    want = oracle.hbonds_calculate(dn[:, :1] if ignore_hs else dn, acc, L["c"], L["box"], ones, ones, 3.2, 100.0, True,
                                   ignore_hs)
    ok = _rows_ok(off.cpu().numpy(), tri.cpu().numpy(), want, 3)
    assert ok.all(), _frame_report(ok)
    assert sum(map(len, want)) // 3 > 5000


@pytest.mark.parametrize("mode", (0, 1, 2))
def test_long_rings(lsys, oracle, mode):
    """K13 on 131 077 frames: the two rings against each other, against the cations 14 and 15, against the halogen bonds
    14-15 and 15-14; pairs and distances of every frame against the oracle, angles within ANGLE_TOL"""
    from moleculekit_b200 import ringpairs

    L = lsys
    ra, st = np.arange(12, dtype=np.uint32), np.array([0, 6, 12], np.uint32)
    second = {0: st, 1: np.array([14, 15], np.uint32), 2: np.array([[14, 15], [15, 14]], np.uint32)}[mode]
    prm = {0: (6.0, 40.0, 7.5, 50.0), 1: (6.0, 30.0), 2: (6.0, 30.0)}[mode]
    off, pairs, da = (x.cpu().numpy() for x in ringpairs.calculate_device(mode, L["C"], L["B"], _i32(ra, L["dev"]),
                                                                          _i32(st, L["dev"]), _i32(second, L["dev"]), *prm))
    res, dist = oracle.ring_interactions(mode, ra, st, second, L["c"], L["box"], *prm)
    ok = _rows_ok(off, pairs, res, 2)
    assert ok.all(), _frame_report(ok)
    wda = np.array([v for x in dist for v in x], np.float32).reshape(-1, 2)
    assert np.array_equal(_bits(da[:, 0]), _bits(wda[:, 0]))
    assert np.allclose(da[:, 1], wda[:, 1], rtol=0, atol=ANGLE_TOL)
    assert len(wda) > 5000


def test_long_reduction_across_thread_kernel_limit(lsys, oracle):
    """K5 with 64 x 64 groups of 1 to 3 atoms (4096 group pairs per frame, the least for the thread kernel) on 65 536
    frames: one frame past the thread kernel's limit, so the warp kernel runs; the halves [0, 32768) and [32768, 65536),
    frame slices of it, each run the thread kernel.  The halves give the whole result's rows bit for bit, and frames 0, 1,
    65 534 and 65 535 equal the oracle."""
    import torch

    from moleculekit_b200 import _lib, distance_utils as du

    L = lsys
    F, half = 65536, 32768
    rng = np.random.default_rng(4096)
    groups = lambda: [np.sort(rng.choice(16, k, replace=False)).tolist() for k in rng.integers(1, 4, 64)]
    g1, g2 = groups(), groups()
    gc1, gc2 = (np.array([L["ch"][g[0]] for g in gs], np.uint32) for gs in (g1, g2))
    masses = rng.uniform(1.0, 16.0, 16).astype(np.float32)
    d_gc1, d_gc2, d_m = _i32(gc1, L["dev"]), _i32(gc2, L["dev"]), torch.from_numpy(masses).to(L["dev"])
    c, b = L["C"][:, :, :F].contiguous(), L["B"][:, :F].contiguous()
    run = lambda cc, bb: du.dist_reduction_device(cc, bb, g1, g2, d_gc1, d_gc2, False, True, d_m, 1, 0)
    whole = run(c, b)
    assert whole.shape == (F, 4096)
    for lo, hi in ((0, half), (half, F)):
        vc, vb = c[:, :, lo:hi], b[:, lo:hi]
        t = _lib.traj(vc, vb)
        assert t.coords == vc.data_ptr() and t.box == vb.data_ptr() and (t.n_frames, t.frame_stride, t.frame_stride_box) == (half, F, F)
        part = run(vc, vb)
        assert torch.equal(part.view(torch.int32), whole[lo:hi].view(torch.int32)), (lo, hi)
        del part
    frames = [0, 1, 65534, 65535]
    want = np.zeros((len(frames), 4096), np.float32)
    oracle.dist_trajectory_reduction(np.ascontiguousarray(L["c"][:, :, frames]), np.ascontiguousarray(L["box"][:, frames]),
                                     g1, g2, gc1, gc2, False, True, masses, 1, 0, want)
    got = whole[frames].cpu().numpy()
    del whole
    torch.cuda.empty_cache()
    assert np.array_equal(_bits(got), _bits(want)) and not np.array_equal(want[2], want[3])


def test_long_metric_distance_project(lsys, oracle):
    """MetricDistance.project on a 70 000-frame MolLite (no host path cuts it into launches): every frame equals the
    oracle's distances"""
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricdistance import MetricDistance

    L = lsys
    F = 70000
    mol = MolLite(L["c"][:, :, :F], L["box"][:, :F])
    got = MetricDistance(np.array(LS1), np.array(LS2), periodic="selections").project(mol)
    chains = np.ones(16, np.uint32)
    chains[LS2] = 2
    want = np.zeros((F, 15), np.float32)
    oracle.dist_trajectory(mol.coords, mol.box, np.array(LS1, np.uint32), np.array(LS2, np.uint32), chains, False, True,
                           want)
    ok = np.all(_bits(got) == _bits(want), axis=1)
    assert got.shape == (F, 15) and ok.all(), _frame_report(ok)


# ------------------------------------------------------------------------------------------ 3. the K4 ballot cache
def test_contacts_fill_cache_across_frame_strides(psys):
    """mkb_contacts_fill reuses the ballots its count call left behind when the call's key matches (K4Key, common.cuh).
    Views A and B share coords, box, n_frames, selections and threshold and differ only in frame stride (64 and 80 over
    one buffer): count A, count B, fill A with A's offsets must give A's own pairs, not pairs from B's ballots."""
    import torch

    from moleculekit_b200 import _lib, distance_utils as du

    p = psys
    dev = p["dev"]
    F, sa, sb = 40, 64, 80
    rng = np.random.default_rng(80)
    buf = torch.from_numpy((rng.uniform(0.0, 24.0, size=N * 3 * sb) +
                            np.repeat(rng.integers(-2, 3, size=N * 3), sb) * 24.0).astype(np.float32)).to(dev)
    A = torch.as_strided(buf, (N, 3, F), (3 * sa, sa, 1))
    B = torch.as_strided(buf, (N, 3, F), (3 * sb, sb, 1))
    box = p["B"][:, :F]
    ta, tb = _lib.traj(A, box), _lib.traj(B, box)
    assert ta.coords == tb.coords == buf.data_ptr() and ta.box == tb.box == box.data_ptr()
    assert (ta.n_frames, ta.frame_stride, ta.frame_stride_box) == (F, sa, FB)
    assert (tb.n_frames, tb.frame_stride, tb.frame_stride_box) == (F, sb, FB)
    s1, s2, ch = p["d_s1"], p["d_s2"], p["d_ch"]
    n1, n2 = len(p["s1"]), len(p["s2"])
    thr = float(np.float32(CT_THR))
    args = lambda t: (C.byref(t), _lib.ptr(s1), n1, _lib.ptr(s2), n2, _lib.ptr(ch), 0, 1, thr)

    def count(t):
        off, total = torch.empty(F * n1 + 1, dtype=torch.int64, device=dev), C.c_int64(0)
        _lib.call(dev, "mkb_contacts_count", *args(t), _lib.ptr(off), C.byref(total))
        return off, total.value

    def fill(t, off, total):
        pairs = torch.empty((total, 2), dtype=torch.int32, device=dev)
        _lib.call(dev, "mkb_contacts_fill", *args(t), _lib.ptr(off), _lib.ptr(pairs))
        return pairs

    want_a = du.contacts_trajectory_device(A.contiguous(), box.contiguous(), s1, s2, ch, False, True, CT_THR)
    want_b = du.contacts_trajectory_device(B.contiguous(), box.contiguous(), s1, s2, ch, False, True, CT_THR)
    assert not torch.equal(want_a[1], want_b[1])  # the two views have different contacts
    off_a, tot_a = count(ta)
    assert _same(fill(ta, off_a, tot_a), want_a[1])  # count -> fill of the same view: the cached ballots
    off_a, tot_a = count(ta)
    off_b, tot_b = count(tb)
    got = fill(ta, off_a, tot_a)
    assert torch.equal(off_a[::n1], want_a[0]) and torch.equal(off_b[::n1], want_b[0])
    assert _same(got, want_a[1])
