"""GPU parity of the occupancy path (K1/K1b/K2) against the CPU oracle and the reference goldens.

Tolerance (BASELINE.json north_star): 1e-5 relative on float32 values; the zero / non-zero pattern must be identical
(the 5 A gate is decided exactly).  Mirrors tests/test_voxeldescriptors.py of the reference.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def _assert_occ_close(got, want, rtol=RTOL):
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == want.shape
    assert np.array_equal(got != 0, want != 0), (
        f"zero pattern differs at {np.count_nonzero((got != 0) != (want != 0))} entries")
    nz = want != 0
    if nz.any():
        rel = np.abs(got[nz] - want[nz]) / want[nz]
        assert rel.max() <= rtol, f"max rel err {rel.max():.3e}"


def _grid_centers(origin, dims, vs):
    ax = [(np.arange(n) * vs).astype(np.float64) + origin[d] for d, n in enumerate(dims)]
    return np.stack(np.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3)


@pytest.fixture(scope="module")
def vd():
    import torch

    assert torch.cuda.is_available()
    from moleculekit_b200.tools import voxeldescriptors

    return voxeldescriptors


def test_3ptb_grid_vs_oracle_and_golden(vd, oracle, g_voxel3ptb):
    """tests/test_voxeldescriptors.py:71-86 (test_old_voxelization): 3PTB, buffer 8, 1 A -> (214500, 8), [60 55 65]."""
    from moleculekit_b200.molecule_lite import MolLite

    g = g_voxel3ptb
    mol = MolLite(g["coords"])
    feats, centers, nvox = vd.getVoxelDescriptors(mol, userchannels=g["sigmas"], buffer=8, voxelsize=1)
    assert feats.dtype == np.float64 and feats.shape == (214500, 8) and list(nvox) == [60, 55, 65]
    want = np.zeros_like(feats)
    oracle.calculate_occupancy(centers, g["coords"], g["sigmas"], want)
    _assert_occ_close(feats, want)
    gold = np.zeros(feats.size)
    gold[g["gold_nz_idx"]] = g["gold_nz_val"]
    assert np.allclose(feats.reshape(-1), gold, rtol=1e-5, atol=1e-8)  # the reference's own assertion


def test_3ptb_usercenters_points_path(vd, oracle, g_voxel3ptb):
    g = g_voxel3ptb
    centers = _grid_centers(g["bb_min"], g["nvoxels"], 1.0)[::7].copy()
    res = vd.getVoxelDescriptors(None, usercenters=centers, userchannels=g["sigmas"], usercoords=g["coords"])
    assert len(res) == 2  # no nvoxels when user centres are given (voxeldescriptors.py:362-365)
    want = np.zeros((centers.shape[0], 8))
    oracle.calculate_occupancy(centers, g["coords"], g["sigmas"], want)
    _assert_occ_close(res[0], want)


@pytest.mark.parametrize("case", ["a", "b", "c"])
def test_small_goldens_points(vd, g_voxelsmall, case):
    g = g_voxelsmall
    feats, _ = vd.getVoxelDescriptors(None, usercenters=g[f"{case}_centers"], userchannels=g[f"{case}_sigmas"],
                                      usercoords=g[f"{case}_coords"])
    _assert_occ_close(feats, g[f"{case}_out"])


def test_small_goldens_grid_exact_ties(vd, oracle, g_voxelsmall):
    """case b: integer lattice, many d2 == 25 exactly (must be excluded: strict <); case c: |x| ~ 200 A, 0.5 A grid."""
    g = g_voxelsmall
    for case, origin, dims, vs in (("b", np.zeros(3), (9, 9, 9), 1.0),
                                   ("c", g["c_centers"][0], (24, 24, 24), 0.5)):
        bs = np.array(dims) * vs
        feats, centers, nv = vd.getVoxelDescriptors(None, boxsize=list(bs), center=list(origin + bs / 2), voxelsize=vs,
                                                    userchannels=g[f"{case}_sigmas"], usercoords=g[f"{case}_coords"])
        assert tuple(nv) == dims
        want = np.zeros_like(feats)
        oracle.calculate_occupancy(centers, g[f"{case}_coords"], g[f"{case}_sigmas"], want)
        _assert_occ_close(feats, want)
        if case == "b":  # origin 4.5 - 4.5 == 0 exactly: same centres as the stored reference output
            assert np.array_equal(centers, g["b_centers"])
            _assert_occ_close(feats, g["b_out"])
        else:
            assert np.allclose(centers, g["c_centers"], rtol=0, atol=1e-12)
            assert np.allclose(feats, g["c_out"], rtol=1e-5, atol=1e-8)


def test_calculate_occupancy_accumulates(oracle):
    from moleculekit_b200.occupancy_utils import calculate_occupancy

    rng = np.random.default_rng(3)
    xyz = (rng.normal(size=(64, 3)) * 4).astype(np.float32)
    ctr = rng.normal(size=(900, 3)) * 5
    sg = rng.choice([0.0, 1.2, 1.7], size=(64, 5))
    sg[3, 1] = np.nan
    for fill in (0.25, -1.0, -np.inf):  # a negative prefill stays wherever no atom with a non-zero sigma reaches
        want = np.full((900, 5), fill); oracle.calculate_occupancy(ctr, xyz, sg, want)
        got = np.full((900, 5), fill); calculate_occupancy(ctr, xyz, sg, got)
        assert np.allclose(got, want, rtol=RTOL, atol=0)
        assert np.array_equal(got == fill, want == fill)
    with pytest.raises(ValueError):
        calculate_occupancy(ctr.astype(np.float32), xyz, sg, got)


@pytest.mark.parametrize("C", [1, 3, 8, 12, 20, 40])
def test_channel_counts_and_multisigma(vd, oracle, C):
    """Arbitrary float channels: several distinct sigmas per atom, any channel count (chunks of 32)."""
    rng = np.random.default_rng(100 + C)
    N = 300
    xyz = (rng.normal(size=(N, 3)) * 6 + np.array([12.0, -7.0, 3.0])).astype(np.float32)
    sg = rng.choice([0.0, 0.0, 1.1, 1.55, 1.7, 2.3], size=(N, C))
    feats, centers, nv = vd.getVoxelDescriptors(None, boxsize=[21, 19, 26], center=[12.0, -7.0, 3.0], voxelsize=1.0,
                                                userchannels=sg, usercoords=xyz)
    want = np.zeros((centers.shape[0], C)); oracle.calculate_occupancy(centers, xyz, sg, want)
    _assert_occ_close(feats, want)


@pytest.mark.parametrize("vs", [0.3, 0.4, 0.5, 0.7, 1.0, 1.9, 2.6])  # the run kernel at every size (cutoff <= 40 voxels)
def test_voxel_sizes_buffer_mode(vd, oracle, vs):
    from moleculekit_b200.molecule_lite import MolLite

    rng = np.random.default_rng(int(vs * 10))
    xyz = (rng.normal(size=(200, 3)) * 3.5 + 40).astype(np.float32)
    sg = rng.choice([1.52, 1.7, 1.8], size=200)[:, None] * (rng.random((200, 8)) < 0.4)
    feats, centers, nv = vd.getVoxelDescriptors(MolLite(xyz), userchannels=sg, buffer=3, voxelsize=vs)
    want = np.zeros_like(feats); oracle.calculate_occupancy(centers, xyz, sg, want)
    _assert_occ_close(feats, want)


def test_edge_cases(vd, oracle):
    # no atoms
    f, c, nv = vd.getVoxelDescriptors(None, boxsize=[5, 5, 5], center=[0, 0, 0], userchannels=np.zeros((0, 8)),
                                      usercoords=np.zeros((0, 3), np.float32))
    assert f.shape == (125, 8) and not f.any()
    # atoms far outside, one voxel grid, coincident atom/voxel (value 1), NaN coordinate
    xyz = np.array([[100, 100, 100], [0.5, 0.5, 0.5], [np.nan, 0, 0], [0.5, 0.5, 3.0]], np.float32)
    sg = np.full((4, 2), 1.7)
    f, c, nv = vd.getVoxelDescriptors(None, boxsize=[1, 1, 1], center=[1.0, 1.0, 1.0], userchannels=sg, usercoords=xyz)
    assert f.shape == (1, 2) and np.allclose(c, 0.5) and np.all(f == 1.0)
    # 3-D coords with one frame are squeezed, several frames rejected (voxeldescriptors.py:345-352)
    with pytest.raises(RuntimeError, match="Only a single set of coordinates"):
        vd.getVoxelDescriptors(None, boxsize=[2, 2, 2], center=[0, 0, 0], userchannels=sg,
                               usercoords=np.zeros((4, 3, 2), np.float32))
    with pytest.raises(RuntimeError, match="only support C implementation"):
        vd.getVoxelDescriptors(None, boxsize=[2, 2, 2], center=[0, 0, 0], userchannels=sg, usercoords=xyz, method="X")


def test_batch_matches_singles_and_oracle(vd, oracle):
    """Reduced C3 (3 pockets x 600 atoms, 33x33x33) through the batched API; ragged atom counts."""
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=3, n_atoms=600, box=33.0, radius=11.0, seed=5)
    w["coords"][1] = w["coords"][1][:411]
    w["sigmas"][1] = w["sigmas"][1][:411]
    feats, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], boxsize=w["boxsize"], centers=w["centers"],
                                              voxelsize=1.0)
    assert dims.tolist() == [[33, 33, 33]] * 3
    for b in range(3):
        centers, nv = vd.getCenters(boxsize=w["boxsize"], center=w["centers"][b], voxelsize=1.0)
        want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, w["coords"][b], w["sigmas"][b], want)
        _assert_occ_close(feats[b], want)
        single, _, _ = vd.getVoxelDescriptors(None, boxsize=w["boxsize"], center=w["centers"][b], voxelsize=1.0,
                                              userchannels=w["sigmas"][b], usercoords=w["coords"][b])
        assert np.array_equal(single, feats[b])  # batching must not change a single bit


def test_full_size_c3_properties(vd, oracle):
    """BASELINE config 3 at full per-GPU size (256 x 64^3 x 8): size-independent properties + two pockets vs oracle."""
    import torch
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=256)
    out, dims, offs = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], boxsize=w["boxsize"], centers=w["centers"],
                                                  voxelsize=1.0, return_tensor=True)
    assert out.shape == (256 * 64 ** 3, 8) and out.dtype == torch.float32
    assert float(out.min()) >= 0.0 and float(out.max()) <= 1.0 and not bool(torch.isnan(out).any())
    occ = out.view(256, 64, 64, 64, 8)
    # atoms live in a sphere R=20 centred in the box: nothing beyond 25 A of the centre can be non-zero
    ax = torch.arange(64, device=out.device, dtype=torch.float32) - 32.0
    r2 = ax[:, None, None] ** 2 + ax[None, :, None] ** 2 + ax[None, None, :] ** 2
    assert not bool((occ[:, r2 > 26.5 ** 2]).any())
    assert bool((occ[:, r2 < 15.0 ** 2][..., 7] > 0).all())  # the all-atom channel fills the core
    for b in (0, 255):
        centers, _ = vd.getCenters(boxsize=w["boxsize"], center=w["centers"][b], voxelsize=1.0)
        want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, w["coords"][b], w["sigmas"][b], want)
        _assert_occ_close(out[offs[b]:offs[b + 1]].cpu().numpy(), want)


@pytest.mark.parametrize("envs", [("MKB_OCC_GENERIC",), ("MKB_OCC_V6",), ("MKB_OCC_NO_TMAP",)])
def test_alternative_kernel_paths_agree(vd, monkeypatch, envs):
    """MKB_OCC_NO_TMAP: the default run kernel with 16 bulk row copies per block instead of one TMA tensor store (the route of
    non-uniform batches and of the compact / to-host transfers; the grid dims here are not multiples of the 4 x 4 x 8 block, so
    the tensor store is clipped by the TMA unit and the row copies by hand).
    The generic tile kernel and the v6 warp kernel (2x4x8 blocks, two voxels per lane) agree with the default run kernel
    (ragged grid: dims not multiples of the block / tile sizes)."""
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=2, n_atoms=700, box=37.0, radius=12.0, seed=21)
    for vs, bs in ((1.0, [37.0, 29.0, 22.0]), (0.5, [18.5, 14.0, 11.5])):
        kw = dict(boxsize=bs, centers=w["centers"], voxelsize=vs)
        ref, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], **kw)
        with monkeypatch.context() as m:
            for e in envs:
                m.setenv(e, "1")
            alt, _ = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], **kw)
        assert dims.tolist() == [[37, 29, 22 if vs == 1.0 else 23]] * 2 or vs == 0.5
        for a, b in zip(ref, alt):
            # different kernels place atoms in different local frames: each within 1e-5 of the float64 oracle, zero pattern identical
            assert np.array_equal(a != 0, b != 0)
            assert np.allclose(a, b, rtol=1.5e-5, atol=0)
            if envs == ("MKB_OCC_NO_TMAP",):  # the same arithmetic, only the store differs
                assert np.array_equal(a, b)


def test_nonuniform_batch_buffer_mode(vd, oracle):
    """Grids of different shapes in one batch (bounding-box mode): exercises the non-uniform launch path."""
    rng = np.random.default_rng(17)
    coords, sigmas = [], []
    for n, spread in ((150, 3.0), (40, 1.5), (300, 5.0)):
        coords.append((rng.normal(size=(n, 3)) * spread + rng.uniform(-30, 30, 3)).astype(np.float32))
        sigmas.append(rng.choice([1.52, 1.7, 1.8], n)[:, None] * (rng.random((n, 8)) < 0.45))
    feats, dims = vd.getVoxelDescriptorsBatch(coords, sigmas, buffer=4.0, voxelsize=1.0)
    assert len({tuple(d) for d in dims.tolist()}) == 3
    from moleculekit_b200.molecule_lite import MolLite
    for b in range(3):
        centers, nv = vd.getCenters(MolLite(coords[b]), buffer=4.0, voxelsize=1.0)
        assert nv.tolist() == dims[b].tolist()
        want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, coords[b], sigmas[b], want)
        _assert_occ_close(feats[b], want)


def test_compact_transfer_equals_dense(vd):
    """transfer="compact" (block records + index over PCIe, dense array rebuilt by host threads) returns the bytes of the
    dense transfer: uniform and ragged batches, float32 into a caller's array and the reference-typed float64 lists."""
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=5, n_atoms=600, box=33.0, radius=10.0, seed=31)
    for kw in (dict(boxsize=[33.0, 26.0, 41.0], centers=w["centers"], voxelsize=1.0),
               dict(buffer=3.0, voxelsize=0.7)):
        dense, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], transfer="dense", dtype=np.float32, **kw)
        comp, dims2 = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], transfer="compact", dtype=np.float32, **kw)
        assert np.array_equal(dims, dims2)
        for a, b in zip(dense, comp):
            assert a.any() and np.array_equal(a.view(np.uint32), b.view(np.uint32))
        f64, _ = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], transfer="compact", **kw)
        for a, b in zip(dense, f64):
            assert b.dtype == np.float64 and np.array_equal(a.astype(np.float64), b)
        total = int(sum(a.shape[0] for a in dense))
        out = vd.pinned_array((total, 8), np.float32)
        out[:] = 3.0
        vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], out=out, transfer="compact", **kw)
        assert vd.LAST_TRANSFER["mode"] == "compact" and vd.LAST_TRANSFER["d2h_bytes"] < out.nbytes
        assert np.array_equal(out, np.concatenate(dense))
        for fill in (7.0, np.nan):  # "direct": the fill kernel stores non-empty blocks into the pinned result, host zeros the rest
            out[:] = fill
            vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], out=out, transfer="direct", **kw)
            assert vd.LAST_TRANSFER["mode"] == "direct" and vd.LAST_TRANSFER["d2h_bytes"] < out.nbytes
            assert np.array_equal(out.view(np.uint32), np.concatenate(dense).view(np.uint32))
        with pytest.raises(ValueError):
            vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], out=np.empty((total, 8), np.float32), transfer="direct", **kw)
        out[:] = 5.0
        vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], out=out, **kw)  # "auto": a batch this small goes dense
        assert vd.LAST_TRANSFER["mode"] == "dense" and np.array_equal(out, np.concatenate(dense))


def test_full_size_c2_all_poses_vs_oracle(vd, oracle):
    """BASELINE config 2 at full size: 1024 ligand poses x 24^3 x 8, EVERY pose against the float64 oracle."""
    from moleculekit_b200 import workloads

    w = workloads.ligand_poses(B=1024)
    feats, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], boxsize=w["boxsize"], centers=w["centers"],
                                              voxelsize=1.0, dtype=np.float32)
    assert dims.tolist() == [[24, 24, 24]] * 1024
    for b in range(1024):
        centers, _ = vd.getCenters(boxsize=w["boxsize"], center=w["centers"][b], voxelsize=1.0)
        want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, w["coords"][b], w["sigmas"][b], want)
        _assert_occ_close(feats[b], want)


def test_full_size_c5_fine_grid_vs_oracle(vd, oracle):
    """BASELINE config 5 at full grid size: one 200^3 @ 0.5 A grid of 8000 atoms (64 M voxel-channels).  The oracle checks a
    random 1 % of the voxels and one full x-plane through the protein (values to 1e-5, identical zero pattern)."""
    from moleculekit_b200 import workloads

    w = workloads.fine_grids(B=1)
    out, dims, offs = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], boxsize=w["boxsize"], centers=w["centers"],
                                                  voxelsize=0.5, return_tensor=True)
    assert dims.tolist() == [[200, 200, 200]] and out.shape == (200 ** 3, 8)
    got = out.cpu().numpy()
    assert got.min() >= 0.0 and got.max() <= 1.0 and not np.isnan(got).any()
    centers, nv = vd.getCenters(boxsize=w["boxsize"], center=w["centers"][0], voxelsize=0.5)
    rng = np.random.default_rng(9)
    pick = np.sort(rng.choice(200 ** 3, 80000, replace=False))
    plane = np.arange(100 * 200 * 200, 101 * 200 * 200)
    for idx in (pick, plane):
        want = np.zeros((len(idx), 8)); oracle.calculate_occupancy(np.ascontiguousarray(centers[idx]), w["coords"][0], w["sigmas"][0], want)
        assert want.any()
        _assert_occ_close(got[idx], want)


def test_cxyz_layout_at_64cubed(vd, oracle):
    """layout="cxyz" (the (B, C, X, Y, Z) tensor a Conv3d consumer wants) on full 64^3 pocket grids: a bit-exact permutation
    of the voxel-major result, and within 1e-5 of the oracle."""
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=3)
    kw = dict(boxsize=w["boxsize"], centers=w["centers"], voxelsize=1.0, dtype=np.float32)
    ref, _ = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], **kw)
    cx, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], layout="cxyz", **kw)
    for b in range(3):
        assert cx[b].shape == (8, 64, 64, 64)
        assert np.array_equal(cx[b].view(np.uint32), np.ascontiguousarray(ref[b].reshape(64, 64, 64, 8).transpose(3, 0, 1, 2)).view(np.uint32))
    centers, _ = vd.getCenters(boxsize=w["boxsize"], center=w["centers"][1], voxelsize=1.0)
    want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, w["coords"][1], w["sigmas"][1], want)
    _assert_occ_close(cx[1].transpose(1, 2, 3, 0).reshape(-1, 8), want)


def test_two_streams_share_one_handle(vd):
    """The per-device handle owns grow-only scratch; calls issued on different torch streams are ordered by the library
    (event recorded at the end of each entry point), so interleaving two streams gives the single-stream bytes."""
    import torch
    from moleculekit_b200 import workloads

    w = workloads.protein_pockets(B=4, n_atoms=500, box=30.0, radius=10.0, seed=77)
    batches = [vd.VoxelBatch(w["coords"][i:i + 2], w["sigmas"][i:i + 2], boxsize=w["boxsize"], centers=w["centers"][i:i + 2],
                             voxelsize=1.0) for i in (0, 2)]
    dev = torch.device("cuda", torch.cuda.current_device())
    ins = [b.to_device(dev) for b in batches]
    want = [b.run(*i).clone() for b, i in zip(batches, ins)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [torch.zeros_like(x) for x in want]
    for _ in range(5):
        for k in range(2):
            with torch.cuda.stream(streams[k]):
                batches[k].run(*ins[k], outs[k])
    torch.cuda.synchronize()
    for a, b in zip(outs, want):
        assert torch.equal(a, b)


@pytest.mark.parametrize("vs", [1.0, 0.8, 0.5])
def test_gate_decisions_on_many_random_grids(vd, oracle, vs):
    """The run kernel decides the 5 A gate in float32 and repairs the +-2e-6 band in float64 (occ_band / occ_fix kernels):
    16 random grids per voxel size (57 k voxels, 700 atoms each, ~6 M in-gate pairs in total) must reproduce the oracle's
    zero pattern everywhere and its values to 1e-5."""
    from moleculekit_b200 import workloads

    n = int(round(36 * 1.0 / vs)) if vs >= 0.8 else 48
    box = n * vs
    w = workloads.protein_pockets(B=16, n_atoms=700, box=box, radius=0.38 * box, seed=int(1000 * vs) + 3)
    feats, dims = vd.getVoxelDescriptorsBatch(w["coords"], w["sigmas"], boxsize=[box] * 3, centers=w["centers"], voxelsize=vs,
                                              dtype=np.float32)
    assert dims.tolist() == [[n, n, n]] * 16
    for b in range(16):
        centers, _ = vd.getCenters(boxsize=[box] * 3, center=w["centers"][b], voxelsize=vs)
        want = np.zeros((centers.shape[0], 8)); oracle.calculate_occupancy(centers, w["coords"][b], w["sigmas"][b], want)
        _assert_occ_close(feats[b], want)
