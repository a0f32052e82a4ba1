"""The host side of AMBER NetCDF reading and writing (moleculekit_b200/netcdf.py; K23 moves the coordinates on the
device): index_netcdf against scipy.io.netcdf_file's view of files scipy wrote, the frame-count rules, the rejections,
the header and non-coordinate record bytes the writer produces, the argument checks that run before any device work,
and the C-ABI symbols."""
import logging
import os
import struct

import numpy as np
import pytest

import netcdf_scipy as ns

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _coords(F, N, seed=0):
    return np.random.default_rng(seed).normal(0, 12, size=(F, N, 3)).astype(np.float32)


def _box(F, seed=1):
    return np.random.default_rng(seed).uniform(20, 60, size=(F, 3))


def _angles(F, seed=2):
    return np.random.default_rng(seed).uniform(60, 120, size=(F, 3))


# every layout the reader must accept: (name, F, N, amber_file keywords)
VARIANTS = [
    ("plain", 5, 17, {}),
    ("cdf1", 5, 17, dict(version=1)),
    ("box", 6, 40, dict(box=_box(6))),
    ("box_angles_cdf1", 4, 9, dict(box=_box(4), angles=_angles(4), version=1)),
    ("extras", 5, 11, dict(extras=True)),
    ("extras_box", 3, 8, dict(extras=True, box=_box(3), angles=_angles(3))),
    ("extras_cdf1", 3, 8, dict(extras=True, version=1)),
    ("time", 4, 6, dict(time=[0.5, 1.5, -2.0, 1e9])),
    ("zero_frames", 0, 7, {}),
    ("zero_frames_box", 0, 7, dict(box=np.zeros((0, 3)))),
    ("one_frame", 1, 1, dict(box=_box(1))),
]


def _check_index(idx, raw, F, N, kw):
    s = ns.read(raw)
    v = s["variables"]
    assert idx["natoms"] == N and idx["n_frames"] == F and idx["numrecs"] == s["numrecs"] == F
    assert idx["version"] == kw.get("version", 2)
    if F:
        assert idx["recsize"] == s["recsize"]
        got = np.stack([np.frombuffer(raw, ">f4", 3 * N, idx["begin"] + k * idx["recsize"]) for k in range(F)])
        assert np.array_equal(got.reshape(F, N, 3).view(np.int32), v["coordinates"].astype(np.float32).view(np.int32))
    assert np.array_equal(idx["time"], v["time"].astype(np.float32))
    if "cell_lengths" in v:
        assert np.array_equal(idx["box"], v["cell_lengths"].astype(np.float32).T)
        assert np.array_equal(idx["boxangles"], v["cell_angles"].astype(np.float32).T)
    else:
        assert np.array_equal(idx["box"], np.zeros((3, F), np.float32))
        assert np.array_equal(idx["boxangles"], np.full((3, F), 90, np.float32))
    for key in ("title", "application", "program", "programVersion", "Conventions", "ConventionVersion"):
        assert idx[key] == s["attributes"][key].decode(), key
    assert idx["variables"] == list(v)


@pytest.mark.parametrize("name,F,N,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_index_matches_scipy(name, F, N, kw):
    from moleculekit_b200 import netcdf as pn

    raw = ns.amber_file(_coords(F, N), **kw)
    _check_index(pn.index_netcdf(raw), raw, F, N, kw)


def _with_numrecs(raw, n):
    return raw[:4] + struct.pack(">I", n) + raw[8:]


def test_frame_count_rules(caplog):
    from moleculekit_b200 import netcdf as pn

    F, N = 6, 9
    for kw in ({}, dict(extras=True, box=_box(F)), dict(version=1)):
        raw = ns.amber_file(_coords(F, N), **kw)
        idx = pn.index_netcdf(raw)
        rs, start = idx["recsize"], idx["record_start"]
        assert start + F * rs == len(raw)
        # STREAMING: the count comes from the file size
        with caplog.at_level(logging.WARNING, logger="moleculekit_b200.netcdf"):
            caplog.clear()
            got = pn.index_netcdf(_with_numrecs(raw, pn.STREAMING))
            assert got["n_frames"] == F and got["numrecs"] == -1 and not caplog.records
            got = pn.index_netcdf(_with_numrecs(raw, pn.STREAMING)[:-5])
            assert got["n_frames"] == F - 1 and caplog.records
            # a cut inside the last record drops it with a warning, wherever the cut falls
            for cut in (1, 4, rs // 2, rs - 1):
                caplog.clear()
                got = pn.index_netcdf(raw[:len(raw) - cut])
                assert got["n_frames"] == F - 1 and got["numrecs"] == F and caplog.records
                assert np.array_equal(got["time"], idx["time"][:F - 1]) and np.array_equal(got["box"], idx["box"][:, :F - 1])
            # a numrecs beyond the records present
            caplog.clear()
            assert pn.index_netcdf(_with_numrecs(raw, F + 3))["n_frames"] == F and caplog.records
            # records cut away entirely, down to none
            assert pn.index_netcdf(raw[:start + 2 * rs])["n_frames"] == 2
            assert pn.index_netcdf(raw[:start])["n_frames"] == 0
        # numrecs below the data present: the header's count holds
        for n in (0, 2, F - 1):
            assert pn.index_netcdf(_with_numrecs(raw, n))["n_frames"] == n


def _patched_begin(pn, raw, var, value):
    h = pn._parse(np.frombuffer(raw, np.uint8))
    fmt = ">i" if h["version"] == 1 else ">q"
    old = struct.pack(fmt, h["variables"][var]["begin"])
    at = raw.index(struct.pack(">i", h["variables"][var]["vsize"]) + old)
    return raw[:at + 4] + struct.pack(fmt, value) + raw[at + 4 + len(old):]


def _scipy_raw(build):
    import io

    from scipy.io import netcdf_file

    fh = io.BytesIO()
    f = netcdf_file(fh, "w", version=2)
    build(f)
    f.flush()
    raw = fh.getvalue()
    f.fp = io.BytesIO()
    f.close()
    return raw


def test_rejections():
    from moleculekit_b200 import netcdf as pn

    raw = ns.amber_file(_coords(3, 5), box=_box(3))
    with pytest.raises(ValueError, match="HDF5"):
        pn.index_netcdf(b"\x89HDF\r\n\x1a\n" + raw[8:])
    with pytest.raises(ValueError, match="CDF-5"):
        pn.index_netcdf(b"CDF\x05" + raw[4:])
    for bad in (b"", b"CD", b"CDF\x03" + raw[4:], b"\x00" * 64):
        with pytest.raises(RuntimeError, match="Malformed NetCDF file"):
            pn.index_netcdf(bad)
    header_end = pn._parse(np.frombuffer(raw, np.uint8))["header_end"]
    for cut in range(0, header_end, 7):
        with pytest.raises(RuntimeError, match="Malformed NetCDF file"):
            pn.index_netcdf(raw[:cut])
    for var, value in (("spatial", len(raw)), ("cell_angular", 2**40), ("coordinates", 8), ("spatial", -4)):
        with pytest.raises(RuntimeError, match=f"Malformed NetCDF file: .*{var}"):
            pn.index_netcdf(_patched_begin(pn, raw, var, value))
    cdf1 = ns.amber_file(_coords(3, 5), version=1)
    with pytest.raises(RuntimeError, match="Malformed NetCDF file: .*spatial"):
        pn.index_netcdf(_patched_begin(pn, cdf1, "spatial", len(cdf1) + 100))

    def no_coordinates(f):
        f.createDimension("frame", None)
        f.createDimension("atom", 4)
        f.createVariable("velocities", "f", ("frame", "atom"))[:] = np.ones((2, 4), np.float32)

    with pytest.raises(ValueError, match="no 'coordinates'"):
        pn.index_netcdf(_scipy_raw(no_coordinates))

    def double_coordinates(f):
        f.createDimension("frame", None)
        f.createDimension("atom", 4)
        f.createDimension("spatial", 3)
        f.createVariable("coordinates", "d", ("frame", "atom", "spatial"))[:] = np.ones((2, 4, 3))

    with pytest.raises(ValueError, match="NC_FLOAT"):
        pn.index_netcdf(_scipy_raw(double_coordinates))

    def restart(f):
        f.Conventions = "AMBERRESTART"
        f.ConventionVersion = "1.0"
        f.createDimension("spatial", 3)
        f.createDimension("atom", 4)
        f.createVariable("time", "d", ())
        f.createVariable("coordinates", "d", ("atom", "spatial"))[:] = np.ones((4, 3))

    with pytest.raises(ValueError, match="restart"):
        pn.index_netcdf(_scipy_raw(restart))

    def flat_coordinates(f):
        f.createDimension("frame", None)
        f.createDimension("atom", 4)
        f.createVariable("coordinates", "f", ("frame", "atom"))[:] = np.ones((2, 4), np.float32)

    with pytest.raises(ValueError, match="frame, atom, spatial"):
        pn.index_netcdf(_scipy_raw(flat_coordinates))


@pytest.mark.parametrize("title", [None, "a title of odd length", "x" * 80])
@pytest.mark.parametrize("with_box", [False, True])
def test_header_and_record_bytes_match_scipy(title, with_box):
    from moleculekit_b200 import netcdf as pn

    N = 23
    kw = {} if title is None else dict(title=title)
    for F in (1, 4):
        box = _box(F).astype(np.float32) if with_box else None
        ang = _angles(F).astype(np.float32) if with_box else None
        time = np.float32([0.25, -1.0, 3e5, 7.0])[:F]
        want = ns.amber_file(_coords(F, N), box=box, angles=ang, time=time, **kw)
        hdr = pn.netcdf_header(N, F, with_box, title)
        assert want[:len(hdr)] == hdr
        # every record byte outside the coordinates comes from the host-built array the encoder copies
        record_bytes, coord_offset = pn._record_layout(N, with_box)
        assert len(want) == len(hdr) + F * record_bytes
        recs = np.frombuffer(want, np.uint8, offset=len(hdr)).reshape(F, record_bytes)
        extra = pn._extra(F, None if box is None else box.T, None if ang is None else ang.T, time)
        assert np.array_equal(np.concatenate([recs[:, :coord_offset], recs[:, coord_offset + 12 * N:]], 1), extra)
    # the default time is the frame index
    assert np.array_equal(pn._extra(3, None, None, None).view(">f4").ravel(), np.float32([0, 1, 2]))
    # no frames: the header is the whole file, needs no device, and scipy reads it
    got = pn.netcdf_bytes(np.zeros((N, 3, 0), np.float32), box=np.zeros((3, 0)) if with_box else None, title=title)
    s = ns.read(got)
    assert s["numrecs"] == 0 and s["variables"]["coordinates"].shape == (0, N, 3)
    assert ("cell_lengths" in s["variables"]) == with_box and s["attributes"]["Conventions"] == b"AMBER"
    idx = pn.index_netcdf(got)
    assert idx["n_frames"] == 0 and idx["natoms"] == N


def test_arguments_are_checked_before_the_device_is_touched(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import netcdf as pn

    c = np.zeros((12, 3, 4), np.float32)
    box = np.ones((3, 4), np.float32)
    for args, kw in (((c[:, :2],), {}), ((c[0],), {}), ((c,), dict(box=box[:, :3])), ((c,), dict(box=box[:2])),
                     ((c,), dict(box=box, boxangles=box[:, :2])), ((c,), dict(boxangles=box)),
                     ((c,), dict(time=np.zeros(3))), ((c,), dict(title="café")), ((c,), dict(title=["a"])),
                     ((c,), dict(chunk_bytes=0)), ((np.zeros((0, 3, 4), np.float32),), {}),
                     ((np.broadcast_to(np.float32(0), (pn.MAX_ATOMS + 1, 3, 1)),), {})):
        with pytest.raises(ValueError):
            pn.netcdf_bytes(*args, **kw)
        fn = tmp_path / "untouched.nc"
        with pytest.raises(ValueError):
            pn.write_netcdf(str(fn), *args, **kw)
        assert not fn.exists()
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pn.encode_netcdf_device(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pn.netcdf_bytes(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pn.decode_netcdf_device(torch.zeros(16, dtype=torch.uint8), np.zeros(0, np.int64), 4)
    fn = tmp_path / "t.nc"
    fn.write_bytes(ns.amber_file(_coords(3, 5)))
    for bad in ([3], [-4], [0, 7]):
        with pytest.raises(IndexError):
            pn.read_netcdf_frames(str(fn), bad)
    with pytest.raises(ValueError):
        pn.read_netcdf_device(str(fn), chunk_bytes=0)
    empty = tmp_path / "empty.nc"
    empty.write_bytes(b"")
    with pytest.raises(RuntimeError, match="Malformed NetCDF file"):
        pn.read_netcdf(str(empty))
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pn.netcdf_bytes(c)
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pn.read_netcdf(str(fn))


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_netcdf_decode", 9), ("mkb_netcdf_encode", 11)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
