"""The list segments of the 8-channel occupancy path (K2'): the count pass reserves one segment per (CTA, block) in the
block's list and the fill pass writes into it, while insertions that find no table slot are counted and placed one by one
in the same list.  Batches where one block's list holds in-table segments of several CTAs and direct insertions of a CTA
whose table overflowed, CTAs that span grids, a smaller batch after a larger one on the same handle, and the dense,
compact and to-host routes on the same inputs; against the float64 oracle and one call per grid.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-5
CTA_ATOMS = 256
TABLE = 2048


@pytest.fixture(scope="module")
def ou():
    import torch

    assert torch.cuda.is_available()
    from moleculekit_b200 import occupancy_utils

    return occupancy_utils


@pytest.fixture(scope="module")
def oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


def _dev():
    import torch

    return torch.device("cuda", torch.cuda.current_device())


def _sigmas(rng, n):
    rad = rng.choice([1.37, 1.52, 1.55, 1.7, 1.8], size=n)
    mask = rng.random((n, 8)) < np.array([.62, .08, .34, .05, .57, .39, .02, 1.0])
    return rad[:, None] * mask


def _batch(ou, rng, sizes, dim=16, spread=1.5):
    """Grids of dim^3 voxels at 1 A; grid b holds sizes[b] atoms packed around its centre (every atom then reaches
    nearly all of the grid's 4 x 4 x 8-voxel blocks)."""
    B = len(sizes)
    origins = rng.uniform(-40, 40, size=(B, 3)).round(3)
    ctr = origins + (dim - 1) / 2
    coords = np.concatenate([(ctr[b] + rng.normal(0, spread, size=(n, 3))).astype(np.float32) for b, n in enumerate(sizes)])
    sigmas = np.concatenate([_sigmas(rng, n) for n in sizes])
    dims = np.full((B, 3), dim)
    descs, _ = ou.make_grid_descs(origins, 1.0, dims, np.concatenate([[0], np.cumsum(sizes)]))
    return coords, sigmas, descs


def _dense(ou, coords, sigmas, descs):
    import torch

    dev = _dev()
    n = int((descs["out_offset"] + descs["dims"].astype(np.int64).prod(axis=1)).max()) * 8
    out = torch.full((n,), float("nan"), dtype=torch.float32, device=dev)
    ou.occupancy_grid_batch(torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev), descs, out, n_channels=8)
    return out.cpu().numpy()


def _grid(flat, d):
    M = int(np.prod(d["dims"]))
    return flat[int(d["out_offset"]) * 8:(int(d["out_offset"]) + M) * 8].reshape(M, 8)


def _check(ou, oracle, coords, sigmas, descs):
    """The batch against the oracle and against one call per grid (bit for bit); returns the batch's dense output."""
    from moleculekit_b200.tools.voxeldescriptors import _centers_from_spec

    dense = _dense(ou, coords, sigmas, descs)
    assert not np.isnan(dense).any(), "voxels never written"
    for b, d in enumerate(descs):
        a0, a1 = int(d["atom_begin"]), int(d["atom_end"])
        got = _grid(dense, d).astype(np.float64)
        want = np.zeros_like(got)
        oracle.calculate_occupancy(_centers_from_spec(d["origin"], d["dims"], float(d["voxelsize"])), coords[a0:a1],
                                   sigmas[a0:a1], want)
        assert np.array_equal(got != 0, want != 0), f"grid {b}: zero pattern differs"
        nz = want != 0
        assert nz.any()
        assert (np.abs(got[nz] - want[nz]) / want[nz]).max() <= RTOL, f"grid {b}"
        one, _ = ou.make_grid_descs(d["origin"][None], float(d["voxelsize"]), d["dims"][None], [[a0, a1]])
        assert np.array_equal(_dense(ou, coords, sigmas, one).view(np.uint32), _grid(dense, d).reshape(-1).view(np.uint32)), \
            f"grid {b}: batch and single call differ"
    return dense


def _mixed_batch(ou, rng):
    """Grid 0 (32 blocks) has 2 x 256 + 16 atoms: CTAs 0 and 1 hold only its atoms and count every block in their tables.
    CTA 2 holds its last 16 atoms and 240 one-atom grids of 32 blocks each: ~7 700 distinct blocks for 2048 slots, so
    that CTA's table fills up and most of its insertions go to the lists one by one -- with 32 of those blocks, grid 0's
    lists all but surely mix both kinds.  CTA 2 spans 241 grids, CTA 3 the last two."""
    sizes = [2 * CTA_ATOMS + 16] + [1] * 240 + [200, 150]
    coords, sigmas, descs = _batch(ou, rng, sizes)
    assert sum(sizes[1:241]) + 16 == CTA_ATOMS and 32 * 240 > 3 * TABLE
    return coords, sigmas, descs


def test_segments_of_several_ctas_and_direct_insertions(ou, oracle):
    rng = np.random.default_rng(71)
    _check(ou, oracle, *_mixed_batch(ou, rng))


def test_cta_spanning_two_grids(ou, oracle):
    """Two grids of 300 and 212 atoms: CTA 1 holds the last 44 atoms of grid 0 and all of grid 1, both in its table."""
    rng = np.random.default_rng(73)
    _check(ou, oracle, *_batch(ou, rng, [300, 212]))


def test_smaller_batch_after_a_larger_one(ou, oracle):
    """One handle: a batch of 4 CTAs and 243 grids, then one CTA over two grids, then the large batch again -- the second
    call reads no segment or count the first one left, and the third equals the first bit for bit."""
    rng = np.random.default_rng(79)
    big = _mixed_batch(ou, rng)
    first = _check(ou, oracle, *big)
    _check(ou, oracle, *_batch(ou, rng, [130, 90], dim=12))
    assert np.array_equal(_dense(ou, *big).view(np.uint32), first.view(np.uint32))


def test_compact_and_to_host_routes(ou):
    """The compact records (the flag scan reuses the per-block counts) and the direct-to-host route give the dense bytes."""
    import torch

    rng = np.random.default_rng(83)
    coords, sigmas, descs = _mixed_batch(ou, rng)
    dense = _dense(ou, coords, sigmas, descs)
    n = dense.size
    dev = _dev()
    ct, st = torch.from_numpy(coords).to(dev), torch.from_numpy(sigmas).to(dev)
    records, blk_rank = ou.occupancy_grid_batch_compact(ct, st, descs)
    rank = blk_rank.cpu().numpy()
    host = np.full((n // 8, 8), np.nan, np.float32)
    ou.expand_compact_host(descs, 0, len(descs), rank, records[:int(rank[-1])].cpu().numpy(), 0, host)
    assert np.array_equal(host.reshape(-1).view(np.uint32), dense.view(np.uint32))
    pinned = torch.full((n // 8, 8), float("nan"), dtype=torch.float32).pin_memory()
    host_rank, _ = ou.occupancy_grid_batch_to_host(ct, st, descs, pinned)
    ou.wait_index(dev)
    ou.expand_compact_host(descs, 0, len(descs), host_rank.numpy(), None, 0, pinned.numpy())
    torch.cuda.synchronize()
    assert np.array_equal(pinned.numpy().reshape(-1).view(np.uint32), dense.view(np.uint32))
