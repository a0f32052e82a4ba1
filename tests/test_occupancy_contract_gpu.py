"""The occupancy entry points (K1 / K1b / K2) through the whole C-ABI descriptor contract, not only the descriptors
``getVoxelDescriptors`` and ``VoxelBatch`` build: per-grid voxel sizes, shared / overlapping / empty atom ranges, arbitrary
``out_offset`` layouts, misaligned outputs, accumulate in both layouts, launch chunking beyond 65 535 grids, scratch reuse
on one handle, degenerate shapes, bad descriptors and a sigma sweep.

Every kernel path writes into a buffer poisoned with a NaN bit pattern and framed by guard regions, so a skipped store or a
store past a grid shows.  The reference is the float64 oracle (``oracle.calculate_occupancy``) on each grid's own centres
and atom slice; the rule is the suite's: identical zero pattern, then 1e-5 relative.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-5
SENT = np.uint32(0x7FC0DEAD)  # quiet NaN with a payload no kernel produces
GUARD = 64                    # floats before and after every output

PATHS = {
    "runs": (),
    "runs_notmap": ("MKB_OCC_NO_TMAP",),
    "v6": ("MKB_OCC_V6",),
    "generic": ("MKB_OCC_GENERIC",),
}


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ou():
    import torch

    assert torch.cuda.is_available()
    from moleculekit_b200 import occupancy_utils

    return occupancy_utils


def _dev():
    import torch

    return torch.device("cuda", torch.cuda.current_device())


def _assert_occ_close(got, want, rtol=RTOL, what=""):
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == want.shape
    assert not np.isnan(got).any(), f"{what}: {np.count_nonzero(np.isnan(got))} entries never written"
    bad = (got != 0) != (want != 0)
    assert not bad.any(), f"{what}: zero pattern differs at {np.count_nonzero(bad)} entries"
    nz = want != 0
    if nz.any():
        rel = np.abs(got[nz] - want[nz]) / np.abs(want[nz])
        assert rel.max() <= rtol, f"{what}: max rel err {rel.max():.3e}"


def _atoms(rng, n, center, radius):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.asarray(center) + d * (radius * rng.random((n, 1)) ** (1 / 3))).astype(np.float32)


def _channels(rng, n, Cn, multi=0.15):
    """Boolean channels times one radius per atom (the common case), and a share of atoms with several distinct sigmas."""
    s = rng.choice([1.52, 1.7, 1.8, 2.0], n)[:, None] * (rng.random((n, Cn)) < 0.45)
    k = rng.random(n) < multi
    s[k] = rng.choice([0.0, 1.1, 1.55, 2.3], (int(k.sum()), Cn))
    return s


def _centers(d):
    from moleculekit_b200.tools.voxeldescriptors import _centers_from_spec

    return _centers_from_spec(d["origin"], d["dims"], float(d["voxelsize"]))


def _want(oracle, d, coords, sigmas, prefill=None):
    ctr = _centers(d)
    a0, a1 = int(d["atom_begin"]), int(d["atom_end"])
    Cn = sigmas.shape[1]
    want = np.zeros((len(ctr), Cn)) if prefill is None else np.array(prefill, dtype=np.float64)
    oracle.calculate_occupancy(ctr, coords[a0:a1], sigmas[a0:a1], want)
    return want


def _grid(flat, d, Cn, layout):
    """Grid of descriptor d out of a flat float32 output, as (M, C) voxel-major."""
    M = int(np.prod(d["dims"]))
    g = flat[int(d["out_offset"]) * Cn: (int(d["out_offset"]) + M) * Cn]
    return g.reshape(M, Cn) if layout == "xyzc" else g.reshape(Cn, M).T


def _put(flat, d, Cn, layout, arr):
    M = int(np.prod(d["dims"]))
    o = int(d["out_offset"]) * Cn
    flat[o:o + M * Cn] = (arr if layout == "xyzc" else arr.T).reshape(-1)


def _poison(n):
    return np.full(n, SENT, np.uint32).view(np.float32)


def _run_grid(ou, coords, sigmas, descs, n_floats, layout="xyzc", lead=GUARD, tail=GUARD, init=None, accumulate=False,
              envs=(), monkeypatch=None):
    """One occupancy_grid_batch call into a poisoned, guarded buffer; returns (whole buffer, output view) as numpy."""
    import torch

    dev = _dev()
    host = _poison(lead + n_floats + tail)
    if init is not None:
        host[lead:lead + n_floats] = init
    buf = torch.from_numpy(host).to(dev)
    out = buf[lead:lead + n_floats]
    ct = torch.from_numpy(np.ascontiguousarray(coords)).to(dev)
    st = torch.from_numpy(np.ascontiguousarray(sigmas, dtype=np.float64)).to(dev)
    with monkeypatch.context() as m:
        for e in envs:
            m.setenv(e, "1")
        ou.occupancy_grid_batch(ct, st, descs, out, accumulate=accumulate, layout=layout, n_channels=sigmas.shape[1])
    got = buf.cpu().numpy()
    return got, got[lead:lead + n_floats]


def _assert_guards(buf, lead=GUARD, tail=GUARD):
    u = buf.view(np.uint32)
    assert np.all(u[:lead] == SENT), "store before the output"
    assert np.all(u[len(u) - tail:] == SENT), "store past the output"


def _n_floats(descs, Cn):
    return int((descs["out_offset"] + descs["dims"].astype(np.int64).prod(axis=1)).max()) * Cn


def _pocket_batch(ou, rng, Cn, uniform, n_per=120, vs=1.0):
    """Three grids at 1 A (or vs) with ragged dims; grid 0 has its atoms in one corner (most of its blocks empty)."""
    dims = [(21, 18, 27)] * 3 if uniform else [(21, 18, 27), (13, 30, 9), (17, 17, 17)]
    coords, sigmas, origins = [], [], []
    for b, dm in enumerate(dims):
        org = rng.uniform(-40, 40, 3).round(3)
        ext = (np.asarray(dm, dtype=np.float64) - 1) * vs
        if b == 0:
            xyz = _atoms(rng, n_per, org + 1.0, 3.0)            # corner: the far blocks see no atom
        else:
            xyz = _atoms(rng, n_per, org + ext / 2, ext.max() / 2 + 2)
        coords.append(xyz)
        sigmas.append(_channels(rng, n_per, Cn))
        origins.append(org)
    off = np.cumsum([0] + [len(c) for c in coords])
    descs, _ = ou.make_grid_descs(np.array(origins), vs, np.array(dims), off)
    return np.concatenate(coords), np.concatenate(sigmas), descs


# ---------------------------------------------------------------------------------------------------------------------
# 1. every kernel path, guarded and poisoned output
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cn", [3, 8, 12])
@pytest.mark.parametrize("path", list(PATHS))
def test_guarded_poisoned_output_every_path(ou, oracle, monkeypatch, path, Cn):
    """Every voxel of every grid is written with the oracle's value and nothing outside the batch is touched: uniform and
    ragged batches, both layouts, 3 / 8 / 12 channels, on every kernel selector."""
    rng = np.random.default_rng(1000 + 10 * Cn + list(PATHS).index(path))
    for uniform in (True, False):
        coords, sigmas, descs = _pocket_batch(ou, rng, Cn, uniform)
        wants = [_want(oracle, d, coords, sigmas) for d in descs]
        assert wants[0].any() and not wants[0][-1].any()  # the corner grid: occupied near its origin, empty far away
        for layout in ("xyzc", "cxyz"):
            buf, out = _run_grid(ou, coords, sigmas, descs, _n_floats(descs, Cn), layout, envs=PATHS[path],
                                 monkeypatch=monkeypatch)
            _assert_guards(buf)
            for b, d in enumerate(descs):
                _assert_occ_close(_grid(out, d, Cn, layout), wants[b], what=f"{path} uniform={uniform} {layout} grid {b}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. mixed voxel sizes in one call
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["runs", "v6", "generic"])
def test_mixed_voxel_sizes_one_call(ou, oracle, monkeypatch, path):
    """Grids at 0.3, 0.5, 1.0 and 1.9 A in one batch (the kernel variant and the list table are chosen for the whole batch
    from its finest grid), two of them with identical dims that differ only in voxel size.  With the run kernel every grid
    is also bit-identical to a one-grid call of its descriptor (the per-voxel minimum does not depend on list order)."""
    rng = np.random.default_rng(2)
    Cn = 8
    spec = [(0.3, (37, 33, 40)), (0.5, (24, 24, 24)), (1.0, (24, 24, 24)), (1.9, (11, 9, 14))]
    coords, sigmas, origins = [], [], []
    for vs, dm in spec:
        org = rng.uniform(-30, 30, 3).round(2)
        ext = (np.asarray(dm) - 1) * vs
        coords.append(_atoms(rng, 150, org + ext / 2, ext.max() / 2 + 1.5))
        sigmas.append(_channels(rng, 150, Cn))
        origins.append(org)
    coords, sigmas = np.concatenate(coords), np.concatenate(sigmas)
    off = np.arange(len(spec) + 1) * 150
    descs, _ = ou.make_grid_descs(np.array(origins), np.array([s[0] for s in spec]), np.array([s[1] for s in spec]), off)
    n = _n_floats(descs, Cn)
    buf, out = _run_grid(ou, coords, sigmas, descs, n, envs=PATHS[path], monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        g = _grid(out, d, Cn, "xyzc")
        _assert_occ_close(g, _want(oracle, d, coords, sigmas), what=f"{path} vs={spec[b][0]}")
        if path == "runs":
            one = d.copy()
            one["out_offset"] = 0
            _, single = _run_grid(ou, coords, sigmas, np.array([one]), int(np.prod(d["dims"])) * Cn, monkeypatch=monkeypatch)
            assert np.array_equal(g.reshape(-1).view(np.uint32), single.view(np.uint32)), f"grid {b} differs from its single call"


@pytest.mark.parametrize("path", ["runs", "runs_notmap", "v6"])
def test_same_dims_different_voxel_sizes(ou, oracle, monkeypatch, path):
    """Grids with identical dims and contiguous offsets from 0 that differ only in voxel size: the batch is not uniform
    (the uniform launches take the first grid's geometry for all), and every grid equals the oracle."""
    rng = np.random.default_rng(22)
    vss = [0.5, 1.0, 1.0, 1.9]
    dm = (20, 22, 18)
    coords, sigmas, origins = [], [], []
    for vs in vss:
        org = rng.uniform(-30, 30, 3).round(2)
        ext = (np.asarray(dm) - 1) * vs
        coords.append(_atoms(rng, 150, org + ext / 2, ext.max() / 2 + 1.5))
        sigmas.append(_channels(rng, 150, 8))
        origins.append(org)
    coords, sigmas = np.concatenate(coords), np.concatenate(sigmas)
    descs, _ = ou.make_grid_descs(np.array(origins), np.array(vss), np.array([dm] * 4), np.arange(5) * 150)
    buf, out = _run_grid(ou, coords, sigmas, descs, _n_floats(descs, 8), envs=PATHS[path], monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        _assert_occ_close(_grid(out, d, 8, "xyzc"), _want(oracle, d, coords, sigmas), what=f"{path} vs={vss[b]}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. shared, overlapping and empty atom ranges (pockets cut from one protein)
# ---------------------------------------------------------------------------------------------------------------------
def _pockets_of_one_protein(ou, rng):
    """A ~3000-atom protein; 12 pocket grids with (B, 2) ranges.  Atoms [0, 100) are decoys placed at the pocket centres
    that no grid owns: a grid that saw them would differ from the oracle on its own slice."""
    N0, N = 100, 3100
    prot = _atoms(rng, N - N0, (5.0, -3.0, 8.0), 22.0)
    ctrs = prot[rng.choice(len(prot), 12, replace=False)].astype(np.float64)
    decoys = (ctrs[rng.integers(0, 12, N0)] + rng.normal(size=(N0, 3)) * 2).astype(np.float32)
    coords = np.concatenate([decoys, prot])
    sigmas = _channels(rng, N, 8)
    ranges = np.array([[N0, N], [N0, N], [N0, N], [N0, N],       # several whole-protein grids
                       [N0, 1700], [1200, 2600], [1500, 3100],   # overlapping
                       [900, 900],                               # empty, in the middle
                       [N0, 2000], [2000, 3100], [N0, N],
                       [N, N]])                                  # empty, at the end
    dims = np.array([[20, 20, 20]] * 12)
    descs, _ = ou.make_grid_descs(ctrs - 9.5, 1.0, dims, ranges)
    return coords, sigmas, descs


def test_shared_overlapping_empty_ranges_dense_compact_to_host(ou, oracle, monkeypatch):
    import torch

    rng = np.random.default_rng(3)
    coords, sigmas, descs = _pockets_of_one_protein(ou, rng)
    n = _n_floats(descs, 8)
    buf, dense = _run_grid(ou, coords, sigmas, descs, n, monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        want = _want(oracle, d, coords, sigmas)
        _assert_occ_close(_grid(dense, d, 8, "xyzc"), want, what=f"pocket {b}")
        if d["atom_begin"] == d["atom_end"]:
            assert not _grid(dense, d, 8, "xyzc").any()
    # the same through the other kernel selectors: ranges are numbered per grid in K2 as well
    for path in ("v6", "generic"):
        _, alt = _run_grid(ou, coords, sigmas, descs, n, envs=PATHS[path], monkeypatch=monkeypatch)
        for b, d in enumerate(descs):
            _assert_occ_close(_grid(alt, d, 8, "xyzc"), _grid(dense, d, 8, "xyzc").astype(np.float64), rtol=2e-5,
                              what=f"{path} pocket {b}")
    # compact records + host expansion, and the direct-to-host route: the dense bytes
    dev = _dev()
    ct, st = torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev)
    records, blk_rank = ou.occupancy_grid_batch_compact(ct, st, descs)
    rank = blk_rank.cpu().numpy()
    host = _poison(n).reshape(-1, 8).copy()
    ou.expand_compact_host(descs, 0, len(descs), rank, records[:int(rank[-1])].cpu().numpy(), 0, host)
    assert np.array_equal(host.reshape(-1).view(np.uint32), dense.view(np.uint32))
    pinned = torch.from_numpy(_poison(n).reshape(-1, 8).copy()).pin_memory()
    host_rank, _ = ou.occupancy_grid_batch_to_host(ct, st, descs, pinned)
    ou.wait_index(dev)
    ou.expand_compact_host(descs, 0, len(descs), host_rank.numpy(), None, 0, pinned.numpy())
    torch.cuda.synchronize()
    assert np.array_equal(pinned.numpy().reshape(-1).view(np.uint32), dense.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# 4. out_offset layouts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["xyzc", "cxyz"])
@pytest.mark.parametrize("path", ["runs", "v6", "generic"])
def test_out_offsets_reversed_with_gaps(ou, monkeypatch, path, layout):
    """Grids stored in reverse order, with poisoned gaps between them and a non-zero first offset: the gaps stay
    untouched and every grid's bytes equal the contiguous call (the uniform batch, TMA tensor store by default)."""
    rng = np.random.default_rng(4)
    coords, sigmas, descs = _pocket_batch(ou, rng, 8, uniform=True)
    M = int(np.prod(descs["dims"][0]))
    _, ref = _run_grid(ou, coords, sigmas, descs, _n_floats(descs, 8), layout, monkeypatch=monkeypatch)
    gap, first = 37, 211
    moved = descs.copy()
    B = len(descs)
    moved["out_offset"] = [first + (B - 1 - b) * (M + gap) for b in range(B)]
    n = first + B * (M + gap)
    buf, out = _run_grid(ou, coords, sigmas, moved, n * 8, layout, envs=PATHS[path], monkeypatch=monkeypatch)
    _assert_guards(buf)
    touched = np.zeros(n * 8, bool)
    for b in range(B):
        o = int(moved["out_offset"][b]) * 8
        touched[o:o + M * 8] = True
        a, r = _grid(out, moved[b], 8, layout), _grid(ref, descs[b], 8, layout)
        if path == "runs":
            assert np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(r).view(np.uint32)), f"grid {b}"
        else:
            _assert_occ_close(a, r.astype(np.float64), rtol=2e-5, what=f"{path} grid {b}")
    assert np.all(out.view(np.uint32)[~touched] == SENT), "a gap between grids was written"


# ---------------------------------------------------------------------------------------------------------------------
# 5. fill kernel dispatch
# ---------------------------------------------------------------------------------------------------------------------
# id: (channels, voxel size, accumulate, layout, misaligned output, the fill kernel the input alone selects)
DISPATCH = {
    "runs_c8_1A": (8, 1.0, False, "xyzc", False, "occ_fill_runs_kernel"),
    "runs_c8_03A": (8, 0.3, False, "xyzc", False, "occ_fill_runs_kernel"),        # cutoff 17 voxels: still the run kernel
    "v6_misaligned_xyzc": (8, 1.0, False, "xyzc", True, "occ_fill8v_kernel"),      # 16-byte stores impossible
    "v6_misaligned_cxyz": (8, 1.0, False, "cxyz", True, "occ_fill8v_kernel"),
    "v6_accumulate": (8, 1.0, True, "xyzc", False, "occ_fill8v_kernel"),
    "v6_c5": (5, 1.0, False, "xyzc", False, "occ_fill8v_kernel"),
    "generic_accumulate_03A": (8, 0.3, True, "xyzc", False, "occ_fill_kernel"),   # cutoff 15..40 voxels off the run kernel
    "generic_c5_03A": (5, 0.3, False, "xyzc", False, "occ_fill_kernel"),
    "generic_misaligned_03A": (8, 0.3, False, "xyzc", True, "occ_fill_kernel"),
    "generic_c8_012A": (8, 0.12, False, "xyzc", False, "occ_fill_kernel"),        # cutoff 42 voxels: beyond the run kernel
    "generic_c12_1A": (12, 1.0, False, "xyzc", False, "occ_fill_kernel"),
}


@pytest.mark.parametrize("case", list(DISPATCH))
def test_fill_kernel_dispatch_table(ou, oracle, monkeypatch, case):
    """Without a selector the fill kernel follows from the input alone: the run kernel for 8 channels, no accumulate, a
    16-byte aligned output and a cutoff <= 40 voxels; otherwise the v6 warp kernel for <= 8 channels and a cutoff <= 14
    voxels, and the generic tile kernel for the rest.  Every case equals the oracle with its guards intact (a uniform
    batch; accumulate on a zero prefill, misaligned outputs 4 bytes past a 16-byte boundary with scalar stores)."""
    from moleculekit_b200 import _lib

    Cn, vs, accumulate, layout, misaligned, kernel = DISPATCH[case]
    rng = np.random.default_rng(5)
    coords, sigmas, descs = _pocket_batch(ou, rng, Cn, uniform=True, vs=vs)
    n = _n_floats(descs, Cn)
    lead = GUARD + 1 if misaligned else GUARD
    buf, out = _run_grid(ou, coords, sigmas, descs, n, layout, lead=lead, init=np.zeros(n, np.float32) if accumulate else None,
                         accumulate=accumulate, monkeypatch=monkeypatch)
    assert _lib.last_fill_kernel(_dev().index) == kernel
    _assert_guards(buf, lead=lead)
    for b, d in enumerate(descs):
        _assert_occ_close(_grid(out, d, Cn, layout), _want(oracle, d, coords, sigmas), what=f"{case} grid {b}")


# ---------------------------------------------------------------------------------------------------------------------
# 6. accumulate
# ---------------------------------------------------------------------------------------------------------------------
def _prefill_like(rng, v32):
    """Per entry one of: 0, 0.3, 1, one ulp above / below the computed value, the value itself, NaN, -1, -inf."""
    k = rng.integers(0, 9, v32.shape)
    p = np.select([k == 0, k == 1, k == 2, k == 3, k == 4, k == 5, k == 6, k == 7],
                  [np.float32(0), np.float32(0.3), np.float32(1), np.nextafter(v32, np.float32(np.inf)),
                   np.nextafter(v32, np.float32(-np.inf)), v32, np.float32(np.nan), np.float32(-1)],
                  np.float32(-np.inf)).astype(np.float32)
    return p


def _check_accumulated(got, prefill, want, reached_val, what):
    """want: the oracle on the prefill; reached_val: the oracle on a -inf prefill (-inf = no atom reached the entry).
    Entries the reference leaves untouched keep the prefill's bits, unless the computed value ties the prefill within
    the tolerance (then either side is right); updated entries are within 1e-5."""
    p64 = prefill.astype(np.float64)
    untouched = (want == p64) | (np.isnan(want) & np.isnan(p64))
    with np.errstate(invalid="ignore"):
        tie = np.isfinite(reached_val) & np.isfinite(p64) & (np.abs(reached_val - p64) <= RTOL * np.abs(reached_val))
    exact = untouched & ~tie
    assert np.array_equal(got[exact].view(np.uint32), prefill[exact].view(np.uint32)), (
        f"{what}: {np.count_nonzero(got[exact].view(np.uint32) != prefill[exact].view(np.uint32))} untouched entries changed")
    rest = ~exact
    w, g = want[rest], got[rest].astype(np.float64)
    assert np.all(np.isfinite(g)), f"{what}: non-finite value where the reference updates"
    assert np.all(np.abs(g - w) <= RTOL * np.abs(w)), f"{what}: max abs err {np.abs(g - w).max():.3e}"


@pytest.mark.parametrize("layout", ["xyzc", "cxyz"])
@pytest.mark.parametrize("path", ["default", "generic"])
def test_accumulate_prefills_grid_paths(ou, oracle, monkeypatch, path, layout):
    """MKB_OCC_ACCUMULATE follows the reference's update rule on every grid kernel (accumulate calls never take the run
    kernel: "default" is the v6 kernel): an entry is updated only when an atom with a non-zero sigma lies within 5 A and
    its value is larger; NaN sticks; negative prefills stay where no atom reaches."""
    rng = np.random.default_rng(6)
    coords, sigmas, descs = _pocket_batch(ou, rng, 8, uniform=False)
    envs = () if path == "default" else PATHS[path]
    n = _n_floats(descs, 8)
    _, v = _run_grid(ou, coords, sigmas, descs, n, layout, envs=envs, monkeypatch=monkeypatch)
    init = np.empty(n, np.float32)
    pre = []
    for d in descs:
        p = _prefill_like(rng, _grid(v, d, 8, layout))
        _put(init, d, 8, layout, p)
        pre.append(p)
    buf, out = _run_grid(ou, coords, sigmas, descs, n, layout, init=init, accumulate=True, envs=envs, monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        want = _want(oracle, d, coords, sigmas, pre[b])
        reached = _want(oracle, d, coords, sigmas, np.full(pre[b].shape, -np.inf))
        _check_accumulated(np.ascontiguousarray(_grid(out, d, 8, layout)), pre[b], want, reached, f"{path} {layout} grid {b}")


@pytest.mark.parametrize("Cn", [3, 8, 20])
def test_accumulate_prefills_points(ou, oracle, Cn):
    import torch

    rng = np.random.default_rng(60 + Cn)
    xyz = _atoms(rng, 200, (0.0, 0.0, 0.0), 9.0)
    sg = _channels(rng, 200, Cn)
    ctr = rng.normal(size=(6000, 3)) * 8
    dev = _dev()
    args = [torch.from_numpy(ctr).to(dev), torch.from_numpy(xyz).to(dev), torch.from_numpy(sg).to(dev)]
    v = ou.occupancy_points(*args, torch.empty((6000, Cn), dtype=torch.float32, device=dev)).cpu().numpy()
    p = _prefill_like(rng, v)
    got = ou.occupancy_points(*args, torch.from_numpy(p.copy()).to(dev), accumulate=True).cpu().numpy()
    want = p.astype(np.float64)
    oracle.calculate_occupancy(ctr, xyz, sg, want)
    reached = np.full(p.shape, -np.inf)
    oracle.calculate_occupancy(ctr, xyz, sg, reached)
    _check_accumulated(got, p, want, reached, "points")


# ---------------------------------------------------------------------------------------------------------------------
# 7. launch chunking
# ---------------------------------------------------------------------------------------------------------------------
CHUNK_CASES = {
    "c4_v6": (4, 8, ()),                 # warp kernel: 16 383 grids per launch (8-voxel x extent); block totals at 65 535
    "c8_runs": (8, 8, ()),               # persistent run kernel over the whole batch
    "c8_generic": (8, 8, ("MKB_OCC_GENERIC",)),  # tile kernel, 8 channels: 65 535 grids per launch
    "c12_generic": (12, 4, ()),          # generic kernel: 65 535 grids per launch
}


@pytest.mark.parametrize("case", list(CHUNK_CASES))
def test_launch_chunking_70k_grids(ou, oracle, monkeypatch, case):
    """70 001 grids: grid b is an integer translate of template b % 7 (atoms on a 1/64 A lattice, so every float operation
    of the kernels sees the same numbers).  Every grid must equal its template bit for bit -- 7 is coprime with every chunk
    size, so a chunk written one grid off shows -- and the grids around every chunk boundary equal the oracle."""
    import torch

    Cn, n, envs = CHUNK_CASES[case]
    B, T = 70001, 7
    rng = np.random.default_rng(7)
    cnt = rng.integers(4, 14, T)
    tmpl = [np.round((rng.random((k, 3)) * (n + 6) - 3) * 64) / 64 for k in cnt]
    tsig = [_channels(rng, k, Cn, multi=0.3) for k in cnt]
    tm = np.arange(B) % T
    counts = cnt[tm]
    off = np.zeros(B + 1, np.int64)
    np.cumsum(counts, out=off[1:])
    shifts = (n + 3) * np.stack([np.arange(B) % 41, (np.arange(B) // 41) % 41, np.arange(B) // 1681], 1).astype(np.float64)
    tstart = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    local = np.arange(off[-1]) - np.repeat(off[:-1], counts)
    atom_t = np.repeat(tm, counts)
    coords = (np.concatenate(tmpl)[tstart[atom_t] + local] + np.repeat(shifts, counts, axis=0)).astype(np.float32)
    assert np.array_equal(coords.astype(np.float64) - np.repeat(shifts, counts, axis=0), np.concatenate(tmpl)[tstart[atom_t] + local])
    sigmas = np.concatenate(tsig)[tstart[atom_t] + local]
    descs, _ = ou.make_grid_descs(shifts, 1.0, np.array([[n, n, n]] * B), off)
    dev = _dev()
    out = torch.full((B * n ** 3 * Cn,), float("nan"), dtype=torch.float32, device=dev)
    with monkeypatch.context() as m:
        for e in envs:
            m.setenv(e, "1")
        ou.occupancy_grid_batch(torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev), descs, out)
    g = out.view(B, -1).view(torch.int32)
    idx = torch.arange(B, device=dev) % T
    same = (g == g[idx]).all(dim=1)
    assert bool(same.all()), f"grids differing from their template: {torch.nonzero(~same).flatten()[:10].tolist()}"
    host = out.view(B, -1)
    check = sorted(set(range(T)) | {b + k for b in (16383, 32766, 49149, 65535, 65532) for k in (-1, 0, 1)} | {B - 1})
    for b in check:
        want = _want(oracle, descs[b], coords, sigmas)
        assert want.any()
        _assert_occ_close(host[b].cpu().numpy().reshape(-1, Cn), want, what=f"{case} grid {b}")


# ---------------------------------------------------------------------------------------------------------------------
# 8. scratch reuse on one handle
# ---------------------------------------------------------------------------------------------------------------------
def test_scratch_reuse_large_tiny_medium_large(ou, oracle, monkeypatch):
    """The handle's scratch only grows and its memsets are sized by the current call: a large call, a tiny one, a medium
    one and the large one again -- alternating the run kernel and the v6 kernel -- each give the oracle's result (the
    large grid on a sample of voxels and one full plane) or the first call's bytes."""
    rng = np.random.default_rng(8)
    cases = {}
    for name, vs, dm, na, rad in (("large", 0.5, (128, 128, 128), 2500, 24.0), ("tiny", 1.0, (8, 8, 8), 3, 2.0),
                                  ("medium", 1.0, (40, 36, 44), 500, 14.0)):
        org = rng.uniform(-20, 20, 3).round(2)
        ext = (np.asarray(dm) - 1) * vs
        xyz = _atoms(rng, na, org + ext / 2, rad)
        sg = _channels(rng, na, 8)
        descs, _ = ou.make_grid_descs(org[None], vs, np.array([dm]), [0, na])
        cases[name] = (xyz, sg, descs)
    pick = np.sort(rng.choice(128 ** 3, 20000, replace=False))
    plane = np.arange(64 * 128 * 128, 65 * 128 * 128)
    wants = {}

    def check(name, out, first=None):
        xyz, sg, descs = cases[name]
        g = out.reshape(-1, 8)
        if name != "large":
            if name not in wants:
                wants[name] = _want(oracle, descs[0], xyz, sg)
            _assert_occ_close(g, wants[name], what=name)
            return
        if first is not None and np.array_equal(out.view(np.uint32), first.view(np.uint32)):
            return
        assert not np.isnan(g).any()
        ctr = _centers(descs[0])
        for idx in (pick, plane):
            want = np.zeros((len(idx), 8))
            oracle.calculate_occupancy(np.ascontiguousarray(ctr[idx]), xyz, sg, want)
            _assert_occ_close(g[idx], want, what=name)

    def run(name, path):
        xyz, sg, descs = cases[name]
        buf, out = _run_grid(ou, xyz, sg, descs, _n_floats(descs, 8), envs=PATHS[path], monkeypatch=monkeypatch)
        _assert_guards(buf)
        return out

    first = run("large", "runs")
    check("large", first)
    for name, path in (("tiny", "v6"), ("medium", "runs"), ("large", "runs"), ("tiny", "runs"), ("medium", "v6"),
                       ("large", "v6"), ("tiny", "v6"), ("large", "runs")):
        out = run(name, path)
        check(name, out, first if path == "runs" else None)
        if name == "large" and path == "runs":
            assert np.array_equal(out.view(np.uint32), first.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# 9. degenerate shapes and bad descriptors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["xyzc", "cxyz"])
@pytest.mark.parametrize("path", ["runs", "v6", "generic"])
def test_degenerate_shapes(ou, oracle, monkeypatch, path, layout):
    """1x1x1, 1x1xN and Nx1x1 grids, a grid whose atoms all sit beyond the 5 A halo and a grid without atoms, in one call."""
    rng = np.random.default_rng(9)
    dims = np.array([[1, 1, 1], [1, 1, 37], [29, 1, 1], [1, 23, 1], [9, 10, 11], [12, 12, 12]])
    origins = rng.uniform(-30, 30, (6, 3)).round(2)
    coords, sigmas, off = [], [], [0]
    for b in range(6):
        ext = dims[b] - 1.0
        if b == 4:
            xyz = (origins[b] + ext + 5.5 + rng.random((40, 3)) * 3).astype(np.float32)  # all beyond the halo
        elif b == 5:
            xyz = np.zeros((0, 3), np.float32)
        else:  # along the grid, up to ~4 A off it
            xyz = (origins[b] + rng.random((30, 3)) * ext + rng.normal(size=(30, 3)) * 1.5).astype(np.float32)
        coords.append(xyz)
        sigmas.append(_channels(rng, len(xyz), 8))
        off.append(off[-1] + len(xyz))
    coords, sigmas = np.concatenate(coords), np.concatenate(sigmas)
    descs, _ = ou.make_grid_descs(origins, 1.0, dims, off)
    buf, out = _run_grid(ou, coords, sigmas, descs, _n_floats(descs, 8), layout, envs=PATHS[path], monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        want = _want(oracle, d, coords, sigmas)
        assert want.any() == (b < 4)
        _assert_occ_close(_grid(out, d, 8, layout), want, what=f"{path} grid {b} dims {dims[b].tolist()}")


def test_bad_descriptors_raise(ou, oracle, monkeypatch):
    """Descriptors the kernels cannot serve are refused with MkbError before anything is launched, and the handle keeps
    working afterwards."""
    import torch
    from moleculekit_b200 import _lib

    rng = np.random.default_rng(10)
    coords, sigmas, descs = _pocket_batch(ou, rng, 8, uniform=True)
    n = _n_floats(descs, 8)
    dev = _dev()
    ct, st = torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev)
    out = torch.from_numpy(_poison(n + 2 * GUARD)).to(dev)

    def bad(field, value, b=1):
        d = descs.copy()
        d[field][b] = value
        return d

    cases = [bad("dims", [12, 0, 9]), bad("dims", [-3, 4, 4]), bad("out_offset", -1), bad("atom_end", len(coords) + 1),
             bad("atom_begin", int(descs["atom_end"][1]) + 1),
             bad("voxelsize", 0.0), bad("voxelsize", np.nan), bad("voxelsize", -1.0), bad("voxelsize", np.inf),
             bad("origin", [np.nan, 0.0, 0.0])]
    for path in ("runs", "v6", "generic"):
        with monkeypatch.context() as m:
            for e in PATHS[path]:
                m.setenv(e, "1")
            for d in cases:
                with pytest.raises(_lib.MkbError):
                    ou.occupancy_grid_batch(ct, st, d, out[GUARD:GUARD + n])
            with pytest.raises(_lib.MkbError):
                ou.occupancy_grid_batch_compact(ct, st, bad("out_offset", -1))
    # more than 32 channels: refused by the C entry points themselves, not only by the Python wrapper
    wide = torch.zeros((len(coords), 33), dtype=torch.float64, device=dev)
    lib, h = _lib.load(), _lib.handle(dev.index)
    rc = lib.mkb_occupancy_grid_batch(h, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), C.c_void_p(ct.data_ptr()),
                                      C.c_void_p(wide.data_ptr()), len(coords), 33, descs.ctypes.data_as(C.c_void_p),
                                      len(descs), C.c_void_p(out.data_ptr()), 0)
    assert rc == -1
    with pytest.raises(ValueError):
        ou.occupancy_grid_batch(ct, wide, descs, out[GUARD:GUARD + n])
    torch.cuda.synchronize()
    host = out.cpu().numpy()
    assert np.all(host.view(np.uint32) == SENT), "a refused call wrote to the output"
    # the handle still serves a good call
    buf, got = _run_grid(ou, coords, sigmas, descs, n, monkeypatch=monkeypatch)
    _assert_guards(buf)
    for b, d in enumerate(descs):
        _assert_occ_close(_grid(got, d, 8, "xyzc"), _want(oracle, d, coords, sigmas), what=f"grid {b}")


# ---------------------------------------------------------------------------------------------------------------------
# 10. sigma sweep
# ---------------------------------------------------------------------------------------------------------------------
SIGMAS = [0.05, 0.1, 0.2, 0.3, 0.45, 0.5, 0.55, 0.6, 0.65, 0.69, 0.7, 0.8, 1.0, 3.0, 10.0, 100.0, -0.3, -1.7]


def _sweep_case(ou, s):
    """A 24^3 grid at 0.5 A; half the atoms carry sigma s on a random channel subset, the other half s on some channels
    and 1.7 on others (the per-channel path); atoms at every distance from the voxels, up to and across the 5 A gate."""
    rng = np.random.default_rng(int(abs(s) * 1000) + (s < 0))
    n = 160
    xyz = _atoms(rng, n, (6.0, 6.0, 6.0), 11.0)
    mask = rng.random((n, 8)) < 0.5
    mask[:, 0] = True
    sg = s * mask
    half = np.arange(n) >= n // 2
    sg[half] = np.where(rng.random((int(half.sum()), 8)) < 0.5, s, 1.7)
    descs, _ = ou.make_grid_descs(np.zeros((1, 3)), 0.5, np.array([[24, 24, 24]]), [0, n])
    return xyz, sg, descs


@pytest.mark.parametrize("layout", ["xyzc", "cxyz"])
@pytest.mark.parametrize("accumulate", [False, True])
def test_small_radii_bitmask_channels(ou, oracle, layout, accumulate):
    """Bit-mask channels (one radius per atom): atoms with a radius below SIGMA_EXACT move to the float64 pass as a whole,
    in a ragged batch, in both layouts, with and without accumulate (on a -1 prefill)."""
    import torch

    rng = np.random.default_rng(23)
    coords, sigmas, descs = _pocket_batch(ou, rng, 8, uniform=False)
    n = len(coords)
    radii = rng.choice([0.2, 0.4, 0.6, 1.5, 1.8], n)
    bits = rng.random((n, 8)) < 0.5
    mask = (bits.astype(np.uint64) << np.arange(8, dtype=np.uint64)).sum(axis=1).astype(np.uint32).view(np.int32)
    sg = radii[:, None] * bits
    nf = _n_floats(descs, 8)
    dev = _dev()
    host = _poison(nf + 2 * GUARD)
    host[GUARD:GUARD + nf] = -1.0 if accumulate else np.nan
    buf = torch.from_numpy(host).to(dev)
    ou.occupancy_grid_batch(torch.from_numpy(coords).to(dev), None, descs, buf[GUARD:GUARD + nf], accumulate=accumulate,
                            layout=layout, radii=torch.from_numpy(radii).to(dev), chanmask=torch.from_numpy(mask).to(dev),
                            n_channels=8)
    got = buf.cpu().numpy()
    _assert_guards(got)
    for b, d in enumerate(descs):
        g = _grid(got[GUARD:GUARD + nf], d, 8, layout)
        if accumulate:
            want = _want(oracle, d, coords, sg, np.full((int(np.prod(d["dims"])), 8), -1.0))
            assert (want == -1).any()
            assert np.array_equal(g[want == -1], np.full(int((want == -1).sum()), -1.0, np.float32))
            g, want = np.where(want == -1, 0, g), np.where(want == -1, 0, want)
        else:
            want = _want(oracle, d, coords, sg)
        _assert_occ_close(g, want, what=f"{layout} grid {b}")


@pytest.mark.parametrize("path", ["runs", "v6", "generic", "points"])
@pytest.mark.parametrize("sigma", SIGMAS)
def test_sigma_sweep(ou, oracle, monkeypatch, path, sigma):
    """Channel sigmas from 0.05 to 100 A and a negative one (the reference squares x, so -1.7 acts as 1.7): equal to the
    oracle including the zero pattern.  Sigmas below SIGMA_EXACT = 0.7 A are evaluated with the reference's float64
    operations (the points kernel; for grids after the grid kernels, which see them zeroed), so the sweep crosses that
    threshold from both sides."""
    import torch

    xyz, sg, descs = _sweep_case(ou, sigma)
    want = _want(oracle, descs[0], xyz, sg)
    assert want[:, 0].any()
    if path == "points":
        dev = _dev()
        ctr = torch.from_numpy(_centers(descs[0])).to(dev)
        got = ou.occupancy_points(ctr, torch.from_numpy(xyz).to(dev), torch.from_numpy(sg).to(dev),
                                  torch.from_numpy(_poison(want.size).reshape(want.shape)).to(dev)).cpu().numpy()
    else:
        buf, got = _run_grid(ou, xyz, sg, descs, want.size, envs=PATHS[path], monkeypatch=monkeypatch)
        _assert_guards(buf)
        got = got.reshape(want.shape)
    _assert_occ_close(got, want, what=f"{path} sigma={sigma}")
