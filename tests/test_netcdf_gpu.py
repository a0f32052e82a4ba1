"""K23 on the device: AMBER NetCDF coordinates decoded into (natoms, 3, F) and encoded back, bit for bit against
scipy.io.netcdf_file, an independent implementation of netCDF-3."""
import ctypes
import os

import numpy as np
import pytest

import netcdf_scipy as ns
from test_netcdf_cpu import VARIANTS, _angles, _box, _coords

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _special(x):
    """x with -0.0, quiet NaNs with a payload, negative signalling NaNs and the smallest subnormal sprinkled in"""
    bits = x.view(np.uint32)
    bits.flat[::5] = 0x80000000
    bits.flat[1::7] = 0x7FC12345
    bits.flat[2::11] = 0xFF800001
    bits.flat[3::13] = 0x00000001
    return x


def _want(raw):
    """scipy's coords (N, 3, F), box and angles (3, F) as float32"""
    v = ns.read(raw)["variables"]
    F = v["coordinates"].shape[0]
    box = v["cell_lengths"].astype(np.float32).T if "cell_lengths" in v else np.zeros((3, F), np.float32)
    ang = v["cell_angles"].astype(np.float32).T if "cell_angles" in v else np.full((3, F), 90, np.float32)
    return v["coordinates"].astype(np.float32).transpose(1, 2, 0), box, ang


def _file(tmp_path, raw, name="t.nc"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


@pytest.mark.parametrize("name,F,N,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_reader_is_bit_identical_to_scipy(tmp_path, name, F, N, kw):
    from moleculekit_b200 import netcdf as pn

    raw = ns.amber_file(_special(_coords(F, N, seed=len(name))), **kw)
    fn = _file(tmp_path, raw)
    coords, box, ang = _want(raw)
    got, gbox, gang, info = pn.read_netcdf(fn)
    assert got.shape == (N, 3, F) and np.array_equal(_bits(got), _bits(coords))
    assert np.array_equal(gbox, box) and np.array_equal(gang, ang)
    assert info["natoms"] == N and info["n_frames"] == F and info["Conventions"] == "AMBER"
    if F == 0:
        return
    # a shuffled frame list with repeats that leaves out frame 0, then one that starts with it
    rng = np.random.default_rng(7)
    for sel in (rng.integers(1, F, size=2 * F + 3) if F > 1 else np.zeros(3, np.int64),
                np.concatenate([[0], rng.permutation(F), [F - 1, 0]])):
        got, gbox, gang, info = pn.read_netcdf_frames(fn, sel)
        assert np.array_equal(_bits(got), _bits(coords[:, :, sel])), sel
        assert np.array_equal(gbox, box[:, sel]) and np.array_equal(gang, ang[:, sel])
        assert np.array_equal(info["time"], ns.read(raw)["variables"]["time"].astype(np.float32)[sel])


@pytest.mark.parametrize("N", [1, 33, 65])
@pytest.mark.parametrize("F", [1, 31, 33, 70])
def test_sizes_off_the_tile_and_special_bit_patterns(tmp_path, F, N):
    from moleculekit_b200 import netcdf as pn

    x = _special(_coords(F, N, seed=F * N))
    for kw in ({}, dict(box=_box(F), angles=_angles(F), extras=True, version=1)):
        raw = ns.amber_file(x, **kw)
        coords, _, _ = _want(raw)
        got = pn.read_netcdf(_file(tmp_path, raw))[0]
        assert np.array_equal(_bits(got), _bits(coords))
        assert np.array_equal(_bits(got), _bits(x.transpose(1, 2, 0)))


def test_large_trajectory_and_many_chunks(tmp_path):
    from moleculekit_b200 import netcdf as pn

    F, N = 2000, 5000
    x = np.random.default_rng(5).normal(0, 30, size=(F, N, 3)).astype(np.float32)
    raw = ns.amber_file(x, box=_box(F))
    fn = _file(tmp_path, raw)
    coords, box, _ = _want(raw)
    one = pn.read_netcdf_device(fn)[0]
    assert np.array_equal(_bits(one.cpu().numpy()), _bits(coords))
    slab = 12 * N
    many = pn.read_netcdf_device(fn, chunk_bytes=37 * slab)[0]  # 55 chunks
    assert np.array_equal(_bits(many.cpu().numpy()), _bits(coords))
    sel = np.random.default_rng(9).integers(0, F, size=3001)
    sel[sel == 0] = 1
    part, pbox, _, _ = pn.read_netcdf_device(fn, frames=sel, chunk_bytes=100 * slab)
    assert np.array_equal(_bits(part.cpu().numpy()), _bits(coords[:, :, sel])) and np.array_equal(pbox, box[:, sel])


@pytest.mark.parametrize("with_box", [False, True])
@pytest.mark.parametrize("F,N", [(1, 1), (5, 33), (67, 100), (300, 2)])
def test_writer_matches_scipy(tmp_path, with_box, F, N):
    import torch
    from moleculekit_b200 import netcdf as pn

    rng = np.random.default_rng(F + N)
    x = _special(_coords(F, N, seed=N))
    box = rng.uniform(10, 80, size=(3, F)).astype(np.float32) if with_box else None
    ang = rng.uniform(60, 120, size=(3, F)).astype(np.float32) if with_box else None
    time = rng.uniform(0, 1e4, size=F).astype(np.float32)
    title = "written in a test"
    want = ns.amber_file(x, box=None if box is None else box.T, angles=None if ang is None else ang.T, time=time,
                         title=title)
    coords = np.ascontiguousarray(x.transpose(1, 2, 0))
    assert pn.netcdf_bytes(coords, box, ang, time, title) == want
    # a device tensor with a frame stride: the middle F frames of a wider trajectory
    wide = torch.zeros((N, 3, F + 7), dtype=torch.float32, device="cuda")
    wide[:, :, 3:3 + F] = torch.from_numpy(coords).cuda()
    assert pn.netcdf_bytes(wide[:, :, 3:3 + F], box, ang, time, title, chunk_bytes=1000) == want
    assert pn.netcdf_bytes(torch.from_numpy(coords).cuda().transpose(0, 1).contiguous().transpose(0, 1), box, ang,
                           time, title) == want  # another layout: copied first
    # scipy reads our file back with equal variables
    s = ns.read(want)["variables"]
    assert np.array_equal(_bits(s["coordinates"].astype(np.float32)), _bits(x))
    # the file comes back with the input bits, and the records on the device are the file's
    fn = str(tmp_path / "w.nc")
    pn.write_netcdf(fn, wide[:, :, 3:3 + F], box, ang, time, title, chunk_bytes=(4 + 12 * N) * 2)
    assert open(fn, "rb").read() == want
    back, bbox, bang, info = pn.read_netcdf_device(fn, chunk_bytes=5000)
    assert torch.equal(back.view(torch.int32), wide[:, :, 3:3 + F].contiguous().view(torch.int32))
    assert info["n_frames"] == F and info["title"] == title and np.array_equal(info["time"], time)
    if with_box:
        assert np.array_equal(bbox, box) and np.array_equal(bang, ang)
    dev = pn.encode_netcdf_device(wide[:, :, 3:3 + F], box, ang, time)
    assert bytes(dev.cpu().numpy()) == want[len(pn.netcdf_header(N, F, with_box, title)):]


def test_default_time_and_angles():
    from moleculekit_b200 import netcdf as pn

    x = _coords(4, 3)
    box = np.full((3, 4), 20.0, np.float32)
    want = ns.amber_file(x, box=box.T)
    assert pn.netcdf_bytes(np.ascontiguousarray(x.transpose(1, 2, 0)), box) == want


def test_xtc_and_dcd_to_netcdf_keep_the_bits(tmp_path):
    import torch
    from moleculekit_b200 import dcd as pd
    from moleculekit_b200 import netcdf as pn
    from moleculekit_b200 import xtc as px

    gold = os.path.join(ROOT, "tests", "golden", "xtc")
    names = sorted(f[:-4] for f in os.listdir(gold) if f.endswith(".xtc"))
    assert len(names) == 9
    for name in names:
        coords, box, time, _ = px.read_xtc_device(os.path.join(gold, name + ".xtc"), scale=10)
        lengths = np.ascontiguousarray(np.diagonal(box, axis1=0, axis2=1).T) * 10
        out = str(tmp_path / (name + ".nc"))
        pn.write_netcdf(out, coords, box=lengths, time=time)
        back, bbox, bang, info = pn.read_netcdf_device(out)
        assert torch.equal(back.view(torch.int32), coords.view(torch.int32)), name
        assert np.array_equal(bbox, lengths.astype(np.float32)) and (bang == 90).all()
        assert np.array_equal(info["time"], np.asarray(time, np.float32))
        # the same trajectory through DCD comes out of both readers with equal bits
        dfn = str(tmp_path / (name + ".dcd"))
        pd.write_dcd(dfn, coords, box=lengths)
        dback, dbox, _, _ = pd.read_dcd_device(dfn)
        assert torch.equal(dback.view(torch.int32), back.view(torch.int32)) and np.array_equal(dbox, bbox)


def _at(t, offset):
    """a pointer ``offset`` bytes into a tensor"""
    return ctypes.c_void_p(t.data_ptr() + offset)


def test_abi_argument_checks():
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import netcdf as pn

    dev = torch.device("cuda", 0)
    coords = torch.zeros((10, 3, 4), device=dev)
    rb = 4 + 120
    out = torch.empty(4 * rb, dtype=torch.uint8, device=dev)
    extra = torch.zeros(4 * 4, dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.MkbCapacity, match=str(4 * rb)):
        _lib.call(dev, "mkb_netcdf_encode", _lib.ptr(coords), 4, 4, 10, rb, 4, _lib.ptr(extra), _lib.ptr(out), 4 * rb - 4)
    for record_bytes, coord_offset in ((rb + 2, 4), (rb, 2), (rb, 8), (120 - 4, 0)):
        with pytest.raises(_lib.MkbError, match="multiples of 4"):
            _lib.call(dev, "mkb_netcdf_encode", _lib.ptr(coords), 4, 4, 10, record_bytes, coord_offset,
                      _lib.ptr(extra), _lib.ptr(out), 8 * rb)
    with pytest.raises(_lib.MkbError, match="4-byte aligned"):
        _lib.call(dev, "mkb_netcdf_encode", _lib.ptr(coords), 4, 4, 10, rb, 4, _lib.ptr(extra),
                  _at(out, 2), 4 * rb - 4)
    buf = torch.zeros(1024, dtype=torch.uint8, device=dev)
    for offsets in ([0, 1000], [2], [-4], [1024 - 120 + 4]):
        with pytest.raises(_lib.MkbError, match="offset"):
            pn.decode_netcdf_device(buf, np.array(offsets), 10)
    with pytest.raises(_lib.MkbError, match="4-byte aligned"):
        _lib.call(dev, "mkb_netcdf_decode", _at(buf, 1), 1000, np.zeros(1, np.int64).ctypes.data_as(ctypes.c_void_p),
                  1, 10, _lib.ptr(coords), 4)
    ok = pn.decode_netcdf_device(buf, np.array([1024 - 120, 0]), 10)
    assert ok.shape == (10, 3, 2) and not ok.any()
