"""Host-side logic of the mirrors that needs no GPU: rotation matrices, channel bit masks, grid specs, charged-atom tables."""
import numpy as np
import pytest


def test_rotation_matrices_equal_reference(g_rotate):
    """rotation_matrices reproduces moleculekit.util.rotationMatrix bit for bit (same scalar operations)."""
    from moleculekit_b200.tools.voxeldescriptors import rotation_matrices, rotationMatrix

    g = g_rotate
    for c in range(int(g["ncase"])):
        assert np.array_equal(rotation_matrices(g[f"c{c}_rot"])[0], g[f"c{c}_mats"])
    m = rotationMatrix([0, 0, 1], 1.5708)  # the reference's doctest (util.py:90-94)
    assert np.allclose(m.round(4), [[0, -1, 0], [1, 0, 0], [0, 0, 1]])
    assert np.allclose(np.dot(rotationMatrix([4.0, 4.0, 1.0], 1.2), [3.0, 5.0, 0.0]).round(2), [2.75, 4.77, 1.92])


def test_voxelbatch_channel_masks_and_grid_specs():
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(0)
    coords = [rng.normal(0, 5, (7, 3)).astype(np.float32), rng.normal(9, 3, (4, 3)).astype(np.float32)]
    chans = [rng.random((7, 5)) < 0.5, rng.random((4, 5)) < 0.5]
    els = [np.array(["C", "N", "O", "S", "H", "C", "N"]), np.array(["C", "C", "O", "N"])]
    b = vd.VoxelBatch(coords, chans, boxsize=[6, 8, 10], centers=[c.mean(0) for c in coords], voxelsize=2.0, elements=els)
    assert b.sigmas is None and b.C == 5 and b.chanmask.dtype == np.int32 and b.radii.dtype == np.float64
    cat = np.concatenate(chans)
    for a in range(11):
        assert [(int(b.chanmask[a]) >> h) & 1 for h in range(5)] == cat[a].astype(int).tolist()
    assert np.array_equal(b.radii, np.concatenate([vd.vdw_radii_of(e) for e in els]))
    assert b.dims.tolist() == [[3, 4, 5]] * 2 and b.out_offsets.tolist() == [0, 60, 120] and b.total_voxels == 120
    assert np.allclose(b.origins[1], coords[1].mean(0).astype(np.float64) - np.array([3, 4, 5.0]))
    # float channels keep the sigma-matrix form; bounding-box grids follow getCenters (+1 voxel, float32 bbox)
    sig = [c * 1.7 for c in chans]
    b2 = vd.VoxelBatch(coords, sig, buffer=1.0, voxelsize=1.0)
    assert b2.sigmas is not None and b2.sigmas.dtype == np.float64 and b2.radii is None
    for i in range(2):
        bb_min = coords[i].min(0) - np.float32(1.0)
        bb_max = coords[i].max(0) + np.float32(1.0)
        assert b2.dims[i].tolist() == (np.ceil((bb_max - bb_min) / 1.0).astype(int) + 1).tolist()
        assert np.array_equal(b2.origins[i], bb_min.astype(np.float64))
    assert vd.VoxelBatch(coords, chans, boxsize=[4, 4, 4], centers=np.zeros((2, 3)), radii=[np.ones(7), np.ones(4)]).sigmas is None


def test_charged_atoms_and_metal_tables(g_interactions):
    from moleculekit_b200 import interactions as it
    from moleculekit_b200.molecule_lite import MolLite

    g = g_interactions
    mol = MolLite(g["me6_coords"], resname=g["me6_resname"], name=g["me6_name"], element=g["me6_element"])
    pos, neg = it.get_protein_charged(mol)
    assert np.array_equal(pos, g["me6_pos"]) and np.array_equal(neg, g["me6_neg"])
    assert len(it.METAL_ELEMENTS) == 84 and {"Zn", "Fe", "Ca", "Na"} <= it.METAL_ELEMENTS and "C" not in it.METAL_ELEMENTS
    m = it._mask(mol, np.array([1, 5]))
    assert m.dtype == bool and m.sum() == 2 and m[1] and m[5]


def test_wrap_argument_errors_without_gpu():
    from moleculekit_b200 import wrapping as wr
    from moleculekit_b200.molecule_lite import MolLite

    mol = MolLite(np.zeros((4, 3, 2), np.float32), box=np.ones((3, 2), np.float32))
    with pytest.raises(ValueError, match="Invalid unit cell type"):
        wr.wrap(mol, unitcell="hexagonal")
    mol.box = np.zeros((3, 2), np.float32)
    assert wr.wrap(mol) is None  # zero box: logged no-op, never reaches the GPU
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        wr.wrap_box(np.array([0, 4]), mol.coords, np.ones((3, 2), np.float32), np.zeros(0, np.uint32), np.zeros(3, np.float32))


def test_expand_compact_host_matches_numpy():
    """mkb_occupancy_expand_host (host half of the compact end-to-end transfer): dense grids rebuilt from 4 KB block records
    + the block index, ragged dims, float32 and float64 targets, chunks of grids -- against a plain numpy scatter."""
    from moleculekit_b200 import _lib, occupancy_utils as occ

    rng = np.random.default_rng(5)
    dims = np.array([[9, 6, 17], [4, 4, 8], [13, 10, 23]], dtype=np.int64)
    nvox = dims.prod(axis=1)
    off = np.concatenate([[0], np.cumsum(nvox)])
    descs = np.zeros(3, dtype=_lib.GRID_DESC)
    descs["dims"] = dims
    descs["voxelsize"] = 1.0
    descs["out_offset"] = off[:-1]
    nblk = ((dims[:, 0] + 3) // 4) * ((dims[:, 1] + 3) // 4) * ((dims[:, 2] + 7) // 8)
    bbase = np.concatenate([[0], np.cumsum(nblk)])
    present = rng.random(bbase[-1]) < 0.4
    rank = np.concatenate([[0], np.cumsum(present)]).astype(np.uint32)
    recs = rng.random((int(rank[-1]), 1024)).astype(np.float32)
    want = np.zeros((off[-1], 8), dtype=np.float32)
    for g in range(3):
        nx, ny, nz = dims[g]
        nby, nbz = (ny + 3) // 4, (nz + 7) // 8
        grid = want[off[g]:off[g + 1]].reshape(nx, ny, nz, 8)
        for b in range(nblk[g]):
            if not present[bbase[g] + b]:
                continue
            bz, by, bx = b % nbz, (b // nbz) % nby, b // (nbz * nby)
            blk = recs[rank[bbase[g] + b]].reshape(4, 4, 8, 8)
            x1, y1, z1 = min(4, nx - 4 * bx), min(4, ny - 4 * by), min(8, nz - 8 * bz)
            grid[4 * bx:4 * bx + x1, 4 * by:4 * by + y1, 8 * bz:8 * bz + z1] = blk[:x1, :y1, :z1]
    for dt in (np.float32, np.float64):
        got = np.full((off[-1], 8), 7.0, dtype=dt)
        # two chunks of grids, as the transfer does: [0, 1) then [1, 3)
        occ.expand_compact_host(descs, 0, 1, rank, recs, 0, got, n_threads=3)
        r0 = int(rank[bbase[1]])
        occ.expand_compact_host(descs, 1, 3, rank, recs[r0:], r0, got, n_threads=2)
        assert np.array_equal(got, want.astype(dt))


def test_wrap_box_rejects_unordered_groups():
    """K9 wraps groups in parallel, so overlapping / descending group offsets (which the reference walks sequentially) are
    refused on the host before anything reaches the GPU (ADVICE round 1)."""
    from moleculekit_b200.wrapping import wrap_box

    xyz = np.zeros((10, 3, 2), np.float32)
    box = np.full((3, 2), 10.0, np.float32)
    with pytest.raises(ValueError, match="ascending"):
        wrap_box(np.array([0, 6, 3, 10], np.uint32), xyz, box, np.arange(3, dtype=np.uint32), np.zeros(3, np.float32))


def test_waterbridge_host_logic(g_waterbridge, oracle, monkeypatch):
    """The graph walk of the waterbridge_calculate mirror (interactions.py:470-618) with the hydrogen-bond shells supplied by
    the CPU oracle instead of K12 (test stand-in): the paths written in tests/test_interactions.py:279-326."""
    from moleculekit_b200 import interactions as it

    g = g_waterbridge

    class Mol:
        coords, box = g["coords"], g["box"]
        numAtoms, numFrames = g["coords"].shape[0], g["coords"].shape[2]

    def hb_stand_in(mol, donors, acceptors, sel1="all", sel2=None, dist_threshold=2.5, angle_threshold=120, ignore_hs=False,
                    device=None):
        s1 = np.asarray(sel1, bool).astype(np.uint32)
        s2 = s1.copy() if sel2 is None else np.asarray(sel2, bool).astype(np.uint32)
        sel_idx = np.where(s1.astype(bool) | s2.astype(bool))[0]
        donors = donors[np.all(np.isin(donors, sel_idx), axis=1)]
        acceptors = acceptors[np.isin(acceptors, sel_idx)]
        if ignore_hs:
            donors = np.unique(donors[:, 0])[:, None]
        r = oracle.hbonds_calculate(donors.astype(np.uint32), acceptors.astype(np.uint32), mol.coords, mol.box, s1, s2,
                                    float(dist_threshold), float(angle_threshold), sel2 is None, bool(ignore_hs))
        return [np.asarray(x, dtype=np.int64).reshape(-1, 3) for x in r]

    monkeypatch.setattr(it, "hbonds_calculate", hb_stand_in)
    kw = dict(dist_threshold=3.8, ignore_hs=True, water=g["water"])
    wb = it.waterbridge_calculate(Mol, g["donors"], g["acceptors"], g["gol"], g["asn155"], order=1, **kw)
    assert [list(map(int, p)) for p in wb[0]] == [[3140, 2899, 2024]]
    wb = it.waterbridge_calculate(Mol, g["donors"], g["acceptors"], g["gol"], g["asn155"], order=2, **kw)
    assert [list(map(int, p)) for p in wb[0]] == [[3140, 2899, 2944, 2023], [3140, 2899, 2024]]
    wb = it.waterbridge_calculate(Mol, g["donors"], g["acceptors"], g["gol"], g["protein"], order=1, **kw)
    assert [list(map(int, p)) for p in wb[0]] == [[3140, 2899, 2024], [3142, 2857, 1317], [3142, 2857, 2720],
                                                  [3142, 2857, 2737], [3142, 2857, 2789]]


def test_ring_decision_intervals(tmp_path):
    """rings.cu turns the reference's tests on the double angle into intervals of the float dot product (host code, bisection
    with libm's acosf): tests/cuda/ringsets.cu checks them against the direct evaluation on 6e6 floats."""
    import os
    import shutil
    import subprocess

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "ringsets")
    subprocess.run([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", f"-I{root}/include",
                    f"-I{root}/moleculekit_b200/csrc", os.path.join(root, "tests", "cuda", "ringsets.cu"), "-o", exe],
                   check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "mismatches 0" in r.stdout, r.stdout[-500:]
