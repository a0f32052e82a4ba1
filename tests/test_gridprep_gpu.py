"""GPU tests of SURVEY 8f row 1: channel-major (C,X,Y,Z) output, device-side channel assembly (radius + bit mask),
voxel centres and rotation augmentation on the device."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _pockets(rng, B, n, span, C=8):
    coords, chans, elems = [], [], []
    els = np.array(["C", "N", "O", "S", "H"])
    for _ in range(B):
        coords.append((rng.random((n, 3)) * span + rng.normal(0, 30, 3)).astype(np.float32))
        m = rng.random((n, C)) < 0.3
        m[:, -1] = True
        chans.append(m)
        elems.append(rng.choice(els, n))
    return coords, chans, elems


def _run(vd, coords, chans, *, layout, elements=None, radii=None, boxsize=None, centers=None, buffer=0.0, voxelsize=1.0):
    batch = vd.VoxelBatch(coords, chans, boxsize=boxsize, centers=centers, buffer=buffer, voxelsize=voxelsize,
                          elements=elements, radii=radii)
    d_c, d_ch = batch.to_device()
    return batch, batch.run(d_c, d_ch, layout=layout).cpu().numpy()


@pytest.mark.parametrize("case", ["runs_1A", "runs_05A", "generic_12ch", "v6_c5", "runs_ragged"])
def test_cxyz_layout_is_a_bit_exact_permutation(case):
    """MKB_OCC_LAYOUT_CXYZ in every fill kernel: out[b] as (C,X,Y,Z) equals the voxel-major result transposed."""
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(5)
    C, vs, B, box = 8, 1.0, 3, [24, 24, 24]
    if case == "runs_05A":
        vs, box = 0.5, [14, 14, 14]
    elif case == "generic_12ch":
        C = 12
    elif case == "v6_c5":
        C = 5
    coords, chans, elems = _pockets(rng, B, 300, 20.0, C)
    if case == "runs_ragged":
        kw = dict(buffer=3.0)                       # bounding-box grids of different sizes
        coords = [c[: 100 + 90 * i] for i, c in enumerate(coords)]
        chans = [c[: 100 + 90 * i] for i, c in enumerate(chans)]
        elems = [e[: 100 + 90 * i] for i, e in enumerate(elems)]
    else:
        kw = dict(boxsize=box, centers=[c.mean(axis=0) for c in coords])
    sig = [vd._channels_to_sigmas(ch, el) for ch, el in zip(chans, elems)]
    batch, a = _run(vd, coords, sig, layout="xyzc", voxelsize=vs, **kw)
    _, b = _run(vd, coords, sig, layout="cxyz", voxelsize=vs, **kw)
    assert a.any()
    for i in range(batch.B):
        nx, ny, nz = (int(v) for v in batch.dims[i])
        want = a[batch.out_offsets[i]:batch.out_offsets[i + 1]].reshape(nx, ny, nz, C).transpose(3, 0, 1, 2)
        got = batch.as_cxyz(b, i)
        assert got.shape == (C, nx, ny, nz)
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want).view(np.uint32)), (case, i)


def test_cxyz_accumulate_and_batch_api():
    """accumulate (max into the caller's buffer) in the channel-major layout; the host API returns (C,X,Y,Z) items and a
    (B,C,X,Y,Z) device tensor for uniform batches."""
    import torch
    from moleculekit_b200 import occupancy_utils as occ
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(6)
    coords, chans, elems = _pockets(rng, 2, 200, 16.0)
    ctr = [c.mean(axis=0) for c in coords]
    feats, nvox = vd.getVoxelDescriptorsBatch(coords, chans, elements=elems, boxsize=[20, 20, 20], centers=ctr,
                                              layout="cxyz", dtype=np.float32)
    ref, _ = vd.getVoxelDescriptorsBatch(coords, chans, elements=elems, boxsize=[20, 20, 20], centers=ctr,
                                         dtype=np.float32)
    assert feats[0].shape == (8, 20, 20, 20) and nvox.tolist() == [[20, 20, 20]] * 2
    for f, r in zip(feats, ref):
        assert np.array_equal(f, r.reshape(20, 20, 20, 8).transpose(3, 0, 1, 2))
    t, _, _ = vd.getVoxelDescriptorsBatch(coords, chans, elements=elems, boxsize=[20, 20, 20], centers=ctr,
                                          layout="cxyz", return_tensor=True)
    assert t.is_cuda and tuple(t.shape) == (2, 8, 20, 20, 20)
    assert np.array_equal(t[1].cpu().numpy(), feats[1])
    # accumulate: a buffer pre-filled with 0.5 keeps max(0.5, value)
    batch = vd.VoxelBatch(coords, chans, boxsize=[20, 20, 20], centers=ctr, elements=elems)
    d_c, d_ch = batch.to_device()
    out = torch.full((batch.total_voxels, 8), 0.5, dtype=torch.float32, device=d_c.device)
    occ.occupancy_grid_batch(d_c, None, batch.descs, out, accumulate=True, layout="cxyz", radii=d_ch[0], chanmask=d_ch[1],
                             n_channels=8)
    got = batch.as_cxyz(out.cpu().numpy())
    # accumulate runs the v6 warp kernel (occ_fill8v_kernel), the plain call the run kernel (occ_fill_runs_kernel): each
    # within 1e-5 of the oracle, not bit-identical
    want = np.maximum(np.stack(feats), np.float32(0.5))
    assert np.array_equal(got == 0.5, want == 0.5)
    assert np.allclose(got, want, rtol=1.5e-5, atol=0)


def test_masked_channels_equal_sigma_matrix():
    """device-side channel assembly: (radius, bit mask) input == the reference's radius * mask float64 matrix, bit for bit;
    zero / NaN radii switch an atom off, mask bits above C are ignored."""
    import torch
    from moleculekit_b200 import occupancy_utils as occ
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(7)
    for C, vs in ((8, 1.0), (3, 1.0), (12, 1.0), (8, 0.5)):
        coords, chans, elems = _pockets(rng, 3, 250, 18.0, C)
        ctr = [c.mean(axis=0) for c in coords]
        radii = [vd.vdw_radii_of(e).astype(np.float64) for e in elems]
        radii[0][3] = 0.0
        radii[1][5] = np.nan
        sig = [r[:, None] * ch.astype(float) for r, ch in zip(radii, chans)]
        box = [20, 20, 20] if vs == 1.0 else [12, 12, 12]
        b1, a = _run(vd, coords, sig, layout="xyzc", boxsize=box, centers=ctr, voxelsize=vs)
        b2, m = _run(vd, coords, chans, radii=radii, layout="xyzc", boxsize=box, centers=ctr, voxelsize=vs)
        assert b1.sigmas is not None and b2.sigmas is None and b2.chanmask.dtype == np.int32
        assert a.any() and np.array_equal(a.view(np.uint32), m.view(np.uint32)), (C, vs)
    # stray high bits in the mask
    d_c, (d_r, d_m) = b2.to_device()
    out1 = b2.run(d_c, (d_r, d_m))
    out2 = b2.run(d_c, (d_r, d_m | torch.tensor(-(1 << 20), dtype=torch.int32, device=d_m.device)))
    assert torch.equal(out1, out2)
    # elements -> radii lookup is the default for boolean channels
    b3 = vd.VoxelBatch(coords, chans, boxsize=box, centers=ctr, voxelsize=vs, elements=elems)
    assert b3.sigmas is None and np.array_equal(b3.radii, np.concatenate([vd.vdw_radii_of(e) for e in elems]))
    with pytest.raises(ValueError, match="at most 32 channels"):
        vd.VoxelBatch([coords[0]], [np.ones((250, 33), bool)], boxsize=box, centers=ctr[:1], elements=elems[:1])


def test_centers_on_device_equal_getcenters():
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(8)
    coords, chans, elems = _pockets(rng, 3, 120, 15.0)
    batch = vd.VoxelBatch(coords, chans, buffer=2.5, voxelsize=0.7, elements=elems)
    got = batch.centers_device().cpu().numpy()
    assert got.dtype == np.float64 and got.shape == (batch.total_voxels, 3)
    for b in range(batch.B):
        want, nvox = vd.getCenters(MolLite(coords[b]), buffer=2.5, voxelsize=0.7)
        assert list(nvox) == list(batch.dims[b])
        assert np.array_equal(got[batch.out_offsets[b]:batch.out_offsets[b + 1]], want), b
    batch = vd.VoxelBatch(coords, chans, boxsize=[9.5, 12, 7], centers=[c.mean(axis=0) for c in coords], voxelsize=1.0,
                          elements=elems)
    got = batch.centers_device().cpu().numpy()
    want, _ = vd.getCenters(boxsize=[9.5, 12, 7], center=coords[2].mean(axis=0), voxelsize=1.0)
    assert np.array_equal(got[batch.out_offsets[2]:], want)


def test_rotate_coordinates_vs_reference_golden(g_rotate):
    """rotateCoordinates drop-in against the reference's own outputs (tests/golden/rotate.npz).  numpy evaluates the three
    (N,3)x(3,3) products through BLAS, whose summation order is unspecified: tolerance 1e-12 relative to the coordinate
    scale, float64."""
    from moleculekit_b200.tools import voxeldescriptors as vd

    g = g_rotate
    for c in range(int(g["ncase"])):
        out = vd.rotateCoordinates(g[f"c{c}_coords"], list(g[f"c{c}_rot"]), list(g[f"c{c}_center"]))
        want = g[f"c{c}_out"]
        assert out.dtype == np.float64 and out.shape == want.shape
        scale = np.abs(want).max()
        assert np.abs(out - want).max() <= 1e-12 * scale, c
        assert np.array_equal(vd.rotation_matrices(g[f"c{c}_rot"])[0], g[f"c{c}_mats"])
    with pytest.raises(ValueError):
        vd.rotateCoordinates(np.zeros((4, 2), np.float32), [0, 0, 0], [0, 0, 0])


def test_rotation_augmentation_in_the_batch(oracle):
    """per-item random rotations applied on the device before voxelisation: the device-rotated float32 coordinates match
    numpy's (float64 -> float32) up to one ulp, and the grids equal the oracle evaluated on exactly those coordinates."""
    import torch
    from moleculekit_b200.tools import voxeldescriptors as vd

    rng = np.random.default_rng(9)
    B = 4
    coords, chans, elems = _pockets(rng, B, 150, 14.0)
    ctr = np.stack([c.mean(axis=0) for c in coords]).astype(np.float64)
    rots = rng.uniform(-np.pi, np.pi, size=(B, 3))
    batch = vd.VoxelBatch(coords, chans, boxsize=[18, 18, 18], centers=ctr, elements=elems)
    d_c, d_ch = batch.to_device()
    d_rot = batch.rotate(d_c, rots, ctr)
    assert d_rot.dtype == torch.float32 and d_rot.shape == d_c.shape
    rot_host = d_rot.cpu().numpy()
    mats = vd.rotation_matrices(rots)
    for b in range(B):
        x = coords[b].astype(np.float64)
        for r in range(3):
            x = np.dot(x - ctr[b], mats[b, r].T) + ctr[b]
        got = rot_host[batch.atom_offsets[b]:batch.atom_offsets[b + 1]]
        assert np.abs(got - x).max() <= 4e-6 and not np.allclose(got, coords[b], atol=1e-2)
        # rotation about the centre preserves the distances to it
        assert np.allclose(np.linalg.norm(got - ctr[b], axis=1), np.linalg.norm(coords[b] - ctr[b], axis=1), atol=1e-4)
    feats, _ = vd.getVoxelDescriptorsBatch(coords, chans, elements=elems, boxsize=[18, 18, 18], centers=ctr,
                                           rotations=rots, rotation_centers=ctr, dtype=np.float32)
    for b in range(B):
        sig = vd._channels_to_sigmas(chans[b], elems[b])
        want = np.zeros((18 ** 3, 8))
        oracle.calculate_occupancy(batch.centers(b), rot_host[batch.atom_offsets[b]:batch.atom_offsets[b + 1]], sig, want)
        got = feats[b].astype(np.float64)
        assert np.array_equal(got != 0, want != 0)
        nz = want != 0
        assert (np.abs(got[nz] - want[nz]) / want[nz]).max() <= 1e-5
    with pytest.raises(ValueError, match="rotation_centers"):
        vd.getVoxelDescriptorsBatch(coords, chans, elements=elems, boxsize=[18, 18, 18], centers=ctr, rotations=rots)
