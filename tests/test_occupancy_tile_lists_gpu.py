"""The candidate lists of the 8-channel occupancy path (K2') are kept per tile of 2 x 2 x 1 blocks (8 x 8 x 8 voxels) and
every entry carries one bit per block of the tile; the fill kernel, the float64 fix-up and the compact index keep the
entries / read the bit of their own 4 x 4 x 8-voxel block.  Cases that depend on that split: grids whose block counts in
x and y are odd or 1 (tiles with missing blocks), an atom that reaches one block of a tile only, a tile list several
times the fill kernel's round of which a block keeps a handful of entries (or none), the list table on and off on one
handle, the dense / compact / to-host routes with the record count from the reach rule, and a gate-band voxel whose tile
list is mostly other blocks' atoms.

Every dense call writes into a buffer poisoned with a NaN bit pattern and framed by guard regions; the reference is the
float64 oracle on each grid's own centres and atoms: identical zero pattern, then 1e-5 relative.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-5
SENT = np.uint32(0x7FC0DEAD)  # quiet NaN with a payload no kernel produces
GUARD = 64                    # floats before and after every output
R_CAP = 224                   # candidates per round of the fill kernel
LIST_SLACK = 2e-4             # relative slack the list walk adds to the squared reach


@pytest.fixture(scope="module")
def ou():
    import torch

    assert torch.cuda.is_available()
    from moleculekit_b200 import occupancy_utils

    return occupancy_utils


def _dev():
    import torch

    return torch.device("cuda", torch.cuda.current_device())


def _sigmas(rng, n):
    rad = rng.choice([1.37, 1.52, 1.55, 1.7, 1.8], size=n)
    mask = rng.random((n, 8)) < np.array([.62, .08, .34, .05, .57, .39, .02, 1.0])
    return rad[:, None] * mask


def _descs(ou, origins, vs, dims, sizes):
    return ou.make_grid_descs(np.asarray(origins, np.float64), vs, np.asarray(dims), np.concatenate([[0], np.cumsum(sizes)]))[0]


def _n_floats(descs):
    return int((descs["out_offset"] + descs["dims"].astype(np.int64).prod(axis=1)).max()) * 8


def _dense(ou, coords, sigmas, descs):
    """One occupancy_grid_batch call into a poisoned, guarded buffer; the output as numpy."""
    import torch

    dev = _dev()
    n = _n_floats(descs)
    buf = torch.from_numpy(np.full(GUARD + n + GUARD, SENT, np.uint32).view(np.float32)).to(dev)
    ou.occupancy_grid_batch(torch.from_numpy(np.ascontiguousarray(coords, np.float32)).to(dev),
                            torch.from_numpy(np.ascontiguousarray(sigmas, np.float64)).to(dev), descs, buf[GUARD:GUARD + n],
                            n_channels=8)
    got = buf.cpu().numpy()
    u = got.view(np.uint32)
    assert np.all(u[:GUARD] == SENT), "store before the output"
    assert np.all(u[GUARD + n:] == SENT), "store past the output"
    return got[GUARD:GUARD + n]


def _grid(flat, d):
    M = int(np.prod(d["dims"]))
    return flat[int(d["out_offset"]) * 8:(int(d["out_offset"]) + M) * 8].reshape(M, 8)


def _want(oracle, d, coords, sigmas):
    from moleculekit_b200.tools.voxeldescriptors import _centers_from_spec

    a0, a1 = int(d["atom_begin"]), int(d["atom_end"])
    ctr = _centers_from_spec(d["origin"], d["dims"], float(d["voxelsize"]))
    want = np.zeros((len(ctr), 8))
    oracle.calculate_occupancy(ctr, np.asarray(coords[a0:a1], np.float32), np.asarray(sigmas[a0:a1], np.float64), want)
    return want


def _check(ou, oracle, coords, sigmas, descs, what=""):
    """The batch against the oracle; returns (dense output, the oracle's grids)."""
    dense = _dense(ou, coords, sigmas, descs)
    wants = []
    for b, d in enumerate(descs):
        got = _grid(dense, d).astype(np.float64)
        want = _want(oracle, d, coords, sigmas)
        assert not np.isnan(got).any(), f"{what} grid {b}: {np.count_nonzero(np.isnan(got))} entries never written"
        assert np.array_equal(got != 0, want != 0), f"{what} grid {b}: zero pattern differs"
        nz = want != 0
        if nz.any():
            assert (np.abs(got[nz] - want[nz]) / want[nz]).max() <= RTOL, f"{what} grid {b}"
        wants.append(want)
    return dense, wants


def _blocks_in_reach(coords, d):
    """[nbx, nby, nbz] bool: the 4 x 4 x 8-voxel blocks of grid d with one of its atoms within the list walk's reach, and
    the least relative distance of any (atom, block) pair's squared gap from the reach (the float32 walk decides a pair
    that close either way)."""
    vs = float(d["voxelsize"])
    dims = [int(x) for x in d["dims"]]
    nb = [(dims[0] + 3) // 4, (dims[1] + 3) // 4, (dims[2] + 7) // 8]
    thr = (5.0 / vs) ** 2 * (1 + LIST_SLACK)
    hit = np.zeros(nb, bool)
    margin = np.inf
    for p in (np.asarray(coords[int(d["atom_begin"]):int(d["atom_end"])], np.float64) - d["origin"]) / vs:
        gap = []
        for k, e in enumerate((4, 4, 8)):
            lo = np.arange(nb[k]) * e
            gap.append(np.maximum(np.maximum(lo - p[k], p[k] - (lo + e - 1)), 0.0))
        d2 = gap[0][:, None, None] ** 2 + gap[1][None, :, None] ** 2 + gap[2][None, None, :] ** 2
        hit |= d2 <= thr
        margin = min(margin, np.abs(d2 / thr - 1).min())
    return hit, margin


def _block_view(grid, dims, bx, by, bz=None):
    g = grid.reshape(*dims, 8)
    return g[4 * bx:4 * bx + 4, 4 * by:4 * by + 4] if bz is None else g[4 * bx:4 * bx + 4, 4 * by:4 * by + 4, 8 * bz:8 * bz + 8]


# ---------------------------------------------------------------------------------------------------------------------
ODD_DIMS = [(4, 4, 8), (12, 20, 9), (5, 7, 3), (20, 4, 17), (9, 33, 8)]  # blocks in x, y: 1x1, 3x5, 2x2, 5x1, 3x9


def _odd_batch(ou, rng, dims, n_per=90):
    origins = rng.uniform(-40, 40, size=(len(dims), 3)).round(3)
    coords = [(origins[b] + rng.uniform(-4.0, np.asarray(dm) + 3.0, size=(n_per, 3))).astype(np.float32) for b, dm in enumerate(dims)]
    sigmas = [_sigmas(rng, n_per) for _ in dims]
    return np.concatenate(coords), np.concatenate(sigmas), _descs(ou, origins, 1.0, dims, [n_per] * len(dims))


@pytest.mark.parametrize("uniform", [False, True])
def test_tiles_with_missing_blocks(ou, oracle, uniform):
    """Block counts in x and y that are odd or 1: the last tile of a row or column has one or two blocks only.  Ragged batch
    (row copies) and a batch of equal grids (tensor-map stores)."""
    rng = np.random.default_rng(101 + uniform)
    dims = [ODD_DIMS[1]] * 3 if uniform else ODD_DIMS
    _, wants = _check(ou, oracle, *_odd_batch(ou, rng, dims), what=f"uniform={uniform}")
    assert all(w.any() for w in wants)


@pytest.mark.parametrize("sub", range(4))
def test_atom_reaching_one_block_of_a_tile(ou, oracle, sub):
    """One 8 x 8 x 8-voxel grid at 2.5 A (one tile, cutoff = 2 voxels) and one atom in the middle of block (sub >> 1,
    sub & 1): it is 2.5 voxels from the sibling blocks, so the tile's list has one entry with one bit.  The block matches
    the oracle and the three siblings are zeros."""
    bx, by = sub >> 1, sub & 1
    vs, dims = 2.5, (8, 8, 8)
    origin = np.array([3.0, -7.5, 12.25])
    coords = (origin + vs * np.array([[4 * bx + 1.5, 4 * by + 1.5, 3.4]])).astype(np.float32)
    sigmas = np.array([[1.7, 0, 1.7, 0, 0, 1.7, 0, 1.7]])
    descs = _descs(ou, [origin], vs, [dims], [1])
    hit, margin = _blocks_in_reach(coords, descs[0])
    assert hit.sum() == 1 and hit[bx, by, 0] and margin > 1e-3
    dense, wants = _check(ou, oracle, coords, sigmas, descs)
    g = _grid(dense, descs[0])
    assert _block_view(g, dims, bx, by).any()
    for s in set(range(4)) - {sub}:
        assert not _block_view(g, dims, s >> 1, s & 1).any()


def test_long_tile_list_of_which_a_block_keeps_little(ou, oracle):
    """One tile at 2.5 A whose list holds 500 atoms packed into a corner of block (1, 1), out of reach of the other three
    blocks, plus one atom that only block (0, 0) reaches and five that only block (0, 1) reaches: 506 entries, more than
    two rounds of the fill kernel, of which block (0, 0) keeps one (whole stretches of 224 entries hold none of its
    own), block (0, 1) five, block (1, 1) 500 (several rounds), and block (1, 0) none at all -- zeros through the empty
    path although its tile's list is long."""
    rng = np.random.default_rng(113)
    vs, dims = 2.5, (8, 8, 8)
    origin = np.array([-11.0, 4.5, 20.0])
    vox = np.concatenate([np.column_stack([rng.uniform(6.2, 7.4, 500), rng.uniform(6.2, 7.4, 500), rng.uniform(0.5, 6.5, 500)]),
                          [[1.5, 1.4, 3.3]],
                          np.column_stack([rng.uniform(0.8, 1.9, 5), rng.uniform(5.2, 5.9, 5), rng.uniform(1.0, 6.0, 5)])])
    perm = rng.permutation(len(vox))  # the few kept entries land anywhere in the list
    coords = (origin + vs * vox[perm]).astype(np.float32)
    sigmas = _sigmas(rng, len(vox))
    descs = _descs(ou, [origin], vs, [dims], [len(vox)])
    reach = lambda rows: _blocks_in_reach(coords[np.isin(perm, rows)], _descs(ou, [origin], vs, [dims], [len(rows)])[0])  # noqa: E731
    hit, margin = reach(np.arange(500))
    assert hit.sum() == 1 and hit[1, 1, 0] and margin > 1e-3
    hit, margin = reach([500])
    assert hit.sum() == 1 and hit[0, 0, 0] and margin > 1e-3
    hit, margin = reach(np.arange(501, 506))
    assert hit.sum() == 1 and hit[0, 1, 0] and margin > 1e-3
    assert len(vox) > 2 * R_CAP
    dense, _ = _check(ou, oracle, coords, sigmas, descs)
    g = _grid(dense, descs[0])
    assert _block_view(g, dims, 0, 0).any() and _block_view(g, dims, 0, 1).any() and _block_view(g, dims, 1, 1).any()
    assert not _block_view(g, dims, 1, 0).any()


def test_table_on_and_off_on_one_handle(ou, oracle):
    """The list table is used while an atom reaches at most 64 tiles (voxels of 0.5 A and coarser) and is off below
    (0.35 A: up to 5 tiles per axis).  One handle runs: 1 A alone, 1 A with 0.35 A (off), 1 A with 0.5 A (on, 64 tiles),
    a large 1 A batch, a small one after it, and the first again -- bit for bit as at first."""
    rng = np.random.default_rng(127)

    def batch(spec, n_per):
        origins = rng.uniform(-30, 30, size=(len(spec), 3)).round(2)
        coords, sigmas = [], []
        for (vs, dm), org in zip(spec, origins):
            ext = (np.asarray(dm) - 1) * vs
            coords.append((org + rng.uniform(-3.0, ext + 3.0, size=(n_per, 3))).astype(np.float32))
            sigmas.append(_sigmas(rng, n_per))
        return np.concatenate(coords), np.concatenate(sigmas), _descs(ou, origins, np.array([s[0] for s in spec]),
                                                                     [s[1] for s in spec], [n_per] * len(spec))

    first = batch([(1.0, (12, 20, 9))], 120)
    ref, _ = _check(ou, oracle, *first, what="1 A")
    _check(ou, oracle, *batch([(1.0, (20, 12, 17)), (0.35, (44, 36, 41))], 140), what="1 A + 0.35 A")
    _check(ou, oracle, *batch([(1.0, (13, 9, 20)), (0.5, (36, 44, 33))], 140), what="1 A + 0.5 A")
    _check(ou, oracle, *batch([(1.0, (28, 20, 24))] * 6, 400), what="large")
    _check(ou, oracle, *batch([(1.0, (5, 7, 3)), (1.0, (4, 4, 8))], 30), what="small after large")
    assert np.array_equal(_dense(ou, *first).view(np.uint32), ref.view(np.uint32))


def test_routes_agree_and_records_follow_the_reach_rule(ou, oracle):
    """Dense, compact and to-host routes give the same bytes on grids with missing blocks, and the compact index has a
    record for exactly the blocks the reach rule (evaluated here in float64) gives a candidate."""
    import torch

    rng = np.random.default_rng(131)
    coords, sigmas, descs = _odd_batch(ou, rng, ODD_DIMS, n_per=12)
    dense, _ = _check(ou, oracle, coords, sigmas, descs)
    flags = []
    for d in descs:
        hit, margin = _blocks_in_reach(coords, d)
        assert margin > 1e-5, "an (atom, block) pair too close to the reach for float32 to decide"
        flags.append(hit.reshape(-1))  # block order: (x * nby + y) * nbz + z
    flags = np.concatenate(flags)
    assert 0 < flags.sum() < flags.size
    dev = _dev()
    ct, st = torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev)
    records, blk_rank = ou.occupancy_grid_batch_compact(ct, st, descs)
    rank = blk_rank.cpu().numpy()
    assert rank.size == flags.size + 1 and rank[0] == 0
    assert np.array_equal(np.diff(rank.astype(np.int64)), flags.astype(np.int64))
    n = dense.size
    host = np.full((n // 8, 8), np.nan, np.float32)
    ou.expand_compact_host(descs, 0, len(descs), rank, records[:int(rank[-1])].cpu().numpy(), 0, host)
    assert np.array_equal(host.reshape(-1).view(np.uint32), dense.view(np.uint32))
    pinned = torch.full((n // 8, 8), float("nan"), dtype=torch.float32).pin_memory()
    host_rank, _ = ou.occupancy_grid_batch_to_host(ct, st, descs, pinned)
    ou.wait_index(dev)
    assert np.array_equal(host_rank.numpy(), rank)
    ou.expand_compact_host(descs, 0, len(descs), host_rank.numpy(), None, 0, pinned.numpy())
    torch.cuda.synchronize()
    assert np.array_equal(pinned.numpy().reshape(-1).view(np.uint32), dense.view(np.uint32))


@pytest.mark.parametrize("sub", range(4))
def test_gate_band_voxel_in_a_shared_tile_list(ou, oracle, sub):
    """A 16 x 16 x 8-voxel grid at 1 A with integer voxel centres.  Voxel V of block (sub >> 1, sub & 1) has one atom one
    float32 ulp inside 5 A (channel 7 only) and one at exactly 5 A (channel 6 only): both pairs lie in the band that the
    float64 fix-up re-evaluates, which has to pick V's block's entries out of a tile list that 60 other atoms (channels
    0..5, spread over the tile's four blocks) share.  Channel 7 of V is the first atom's value, channel 6 is zero; through
    the dense and the compact route."""
    import torch

    rng = np.random.default_rng(137 + sub)
    dims = (16, 16, 8)
    origin = np.array([10.0, -20.0, 30.0])
    v = np.array([4 * (sub >> 1) + 1, 4 * (sub & 1) + 2, 3])
    inside = (origin + v + [5.0, 0, 0]).astype(np.float32)
    inside[0] = np.nextafter(inside[0], np.float32(-np.inf))
    at_gate = (origin + v + [0, 5.0, 0]).astype(np.float32)
    others = (origin + rng.uniform(-1.0, [8.0, 8.0, 8.0], size=(60, 3))).astype(np.float32)
    coords = np.concatenate([others[:30], inside[None], others[30:], at_gate[None]])
    sigmas = _sigmas(rng, 62)
    sigmas[:, 6:] = 0.0
    sigmas[30] = [0, 0, 0, 0, 0, 0, 0, 1.7]
    sigmas[61] = [0, 0, 0, 0, 0, 0, 1.9, 0]
    descs = _descs(ou, [origin], 1.0, [dims], [62])
    d2 = ((coords[[30, 61]].astype(np.float64) - (origin + v)) ** 2).sum(axis=1)
    assert 0 < 25.0 - d2[0] < 25.0 * 2e-6 and d2[1] == 25.0
    dense, wants = _check(ou, oracle, coords, sigmas, descs)
    vi = (v[0] * dims[1] + v[1]) * dims[2] + v[2]
    assert wants[0][vi, 7] > 0 and wants[0][vi, 6] == 0
    assert _grid(dense, descs[0])[vi, 7] > 0 and _grid(dense, descs[0])[vi, 6] == 0
    dev = _dev()
    records, blk_rank = ou.occupancy_grid_batch_compact(torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev), descs)
    rank = blk_rank.cpu().numpy()
    host = np.full((dense.size // 8, 8), np.nan, np.float32)
    ou.expand_compact_host(descs, 0, 1, rank, records[:int(rank[-1])].cpu().numpy(), 0, host)
    assert np.array_equal(host.reshape(-1).view(np.uint32), dense.view(np.uint32))
