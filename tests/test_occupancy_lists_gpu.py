"""The per-block candidate lists of the 8-channel occupancy path (K2') on batches whose list passes certainly use the
shared-memory table only, certainly overflow it, and run without it, against the CPU oracle and one call per grid.

The list passes count the insertions of 256 atoms (one CTA) per block in a 2048-slot hash table with linear probing
(at most 8 probes); insertions that find no slot go to global memory one by one.  A CTA whose atoms reach at most 8
distinct blocks never overflows (8 probes always meet the key or a free slot); one whose atoms reach more than 2048
distinct blocks always does.  The fill pass stages the first 4096 in-table entries of a CTA in shared memory and
stores the rest directly.  The table is off when one atom can reach more than 64 blocks (fine voxels).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-5
CTA_ATOMS = 256
TABLE = 2048
PROBES = 8
STAGE = 4096


@pytest.fixture(scope="module")
def vd():
    import torch

    assert torch.cuda.is_available()
    from moleculekit_b200.tools import voxeldescriptors

    return voxeldescriptors


@pytest.fixture(scope="module")
def oracle():
    from oracle import cpu_oracle

    cpu_oracle.build()
    return cpu_oracle


def _sigmas(rng, n):
    rad = rng.choice([1.37, 1.52, 1.55, 1.7, 1.8], size=n)
    mask = rng.random((n, 8)) < np.array([.62, .08, .34, .05, .57, .39, .02, 1.0])
    return rad[:, None] * mask


def _blocks_surely_reached(coords, origin, dims, vs):
    """(x, y, z) block ids (4 x 4 x 8 voxels) whose voxel-centre box lies within 5 A of each atom -- a subset of the
    blocks the list passes insert the atom into (they add a relative slack of 2e-4 to the reach)"""
    cut = 5.0 / vs
    nb = [(dims[0] + 3) // 4, (dims[1] + 3) // 4, (dims[2] + 7) // 8]
    out = set()
    for p in (np.asarray(coords, np.float64) - origin) / vs:
        gap = []
        for d, e in enumerate((4, 4, 8)):
            lo = np.arange(nb[d]) * e
            gap.append(np.maximum(np.maximum(lo - p[d], p[d] - (lo + e - 1)), 0.0))
        d2 = gap[0][:, None, None] ** 2 + gap[1][None, :, None] ** 2 + gap[2][None, None, :] ** 2
        out.update(map(tuple, np.argwhere(d2 <= cut * cut * (1 - 1e-6))))
    return out


def _keys_surely_in_table(keys):
    """True when linear probing places every key whatever the insertion order: the occupant of a slot s has its home slot
    in [s - PROBES + 1, s], so a key with fewer than PROBES other homes within PROBES - 1 slots of its own finds a slot"""
    home = [((k * 2654435761) % 2 ** 32) >> 21 for k in keys]
    near = lambda a, b: min((a - b) % TABLE, (b - a) % TABLE) <= PROBES - 1  # noqa: E731
    return all(sum(1 for j, hj in enumerate(home) if j != i and near(hi, hj)) < PROBES for i, hi in enumerate(home))


def _check(vd, oracle, coords, sigmas, boxsize, centers, vs):
    feats, _ = vd.getVoxelDescriptorsBatch(coords, sigmas, boxsize=boxsize, centers=centers, voxelsize=vs)
    for b in range(len(coords)):
        c, _ = vd.getCenters(boxsize=boxsize, center=centers[b], voxelsize=vs)
        want = np.zeros((c.shape[0], 8))
        oracle.calculate_occupancy(c, coords[b], sigmas[b], want)
        got = np.asarray(feats[b], np.float64)
        assert np.array_equal(got != 0, want != 0), f"grid {b}: zero pattern differs"
        nz = want != 0
        assert nz.any()
        assert (np.abs(got[nz] - want[nz]) / want[nz]).max() <= RTOL
        single, _, _ = vd.getVoxelDescriptors(None, boxsize=boxsize, center=centers[b], voxelsize=vs,
                                              userchannels=sigmas[b], usercoords=coords[b])
        assert np.array_equal(single, feats[b])  # list order differs between batch and single call, the values do not


def test_lists_within_the_table(vd, oracle):
    """Grids of 8^3 voxels (4 blocks each) with 300 atoms packed around the centre: a CTA spans at most two grids, so
    at most 8 distinct blocks -- no insertion leaves the table -- and every list is longer than a fill round."""
    rng = np.random.default_rng(41)
    B, n = 5, 300
    boxsize = [8.0, 8.0, 8.0]
    centers = rng.uniform(-20, 20, size=(B, 3))
    coords = [(centers[b] + rng.normal(0, 1.5, size=(n, 3))).astype(np.float32) for b in range(B)]
    sigmas = [_sigmas(rng, n) for _ in range(B)]
    assert n >= CTA_ATOMS and 2 * 4 <= PROBES
    _check(vd, oracle, coords, sigmas, boxsize, centers, 1.0)


def test_lists_beyond_the_stage(vd, oracle):
    """Two grids of 16^3 voxels at 1 A (32 blocks each, block slots 0..63) with 256 atoms packed around the centre: each
    CTA holds one grid, all its keys sit in the table, and its in-table insertions exceed the 4096 entries the fill pass
    stages in shared memory, so the rest are stored directly."""
    rng = np.random.default_rng(53)
    B, n = 2, CTA_ATOMS
    boxsize = [16.0, 16.0, 16.0]
    centers = rng.uniform(-20, 20, size=(B, 3))
    coords = [(centers[b] + rng.normal(0, 1.5, size=(n, 3))).astype(np.float32) for b in range(B)]
    sigmas = [_sigmas(rng, n) for _ in range(B)]
    assert all(_keys_surely_in_table(range(32 * b, 32 * b + 32)) for b in range(B))
    for b in range(B):
        assert sum(len(_blocks_surely_reached(coords[b][i:i + 1], centers[b] - 8.0, (16, 16, 16), 1.0)) for i in range(n)) > STAGE
    _check(vd, oracle, coords, sigmas, boxsize, centers, 1.0)


def test_lists_overflowing_the_table(vd, oracle):
    """256 grids of 16^3 voxels at 1 A with one atom each: the one CTA reaches far more than 2048 distinct blocks, so
    many insertions overflow the table while the first keys are counted in it."""
    rng = np.random.default_rng(43)
    B = CTA_ATOMS
    boxsize = [16.0, 16.0, 16.0]
    centers = rng.uniform(-30, 30, size=(B, 3))
    coords = [(centers[b] + rng.uniform(-3, 3, size=(1, 3))).astype(np.float32) for b in range(B)]
    sigmas = [_sigmas(rng, 1) for _ in range(B)]
    distinct = sum(len(_blocks_surely_reached(coords[b], centers[b] - 8.0, (16, 16, 16), 1.0)) for b in range(B))
    assert distinct > TABLE
    _check(vd, oracle, coords, sigmas, boxsize, centers, 1.0)


def test_lists_without_the_table(vd, oracle):
    """64 grids of 16 A at 0.5 A with 4 atoms each: an atom can reach more than 64 blocks, so the list passes run
    without the table."""
    rng = np.random.default_rng(47)
    B, n = 64, 4
    boxsize = [16.0, 16.0, 16.0]
    centers = rng.uniform(-30, 30, size=(B, 3))
    coords = [(centers[b] + rng.uniform(-6, 6, size=(n, 3))).astype(np.float32) for b in range(B)]
    sigmas = [_sigmas(rng, n) for _ in range(B)]
    _check(vd, oracle, coords, sigmas, boxsize, centers, 0.5)
