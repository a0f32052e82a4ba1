"""K22 on the device: DCD frame records decoded into (natoms, 3, F) and encoded back, bit for bit against the
independent restatement of the format in oracle/dcd_format.py."""
import os

import numpy as np
import pytest

from oracle import dcd_format as od
from test_dcd_cpu import VARIANTS, _cells, _coords

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _want(raw):
    """oracle coords (N, 3, F), box and angles (3, F)"""
    o = od.read(raw)
    return o["coords"].transpose(1, 2, 0), o["box"].T, o["angles"].T


def _file(tmp_path, raw, name="t.dcd"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


@pytest.mark.parametrize("name,F,N,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_reader_is_bit_identical_to_the_oracle(tmp_path, name, F, N, kw):
    from moleculekit_b200 import dcd as pd

    raw = od.write(_coords(F, N, seed=len(name)), **kw)
    fn = _file(tmp_path, raw)
    coords, box, ang = _want(raw)
    got, gbox, gang, info = pd.read_dcd(fn)
    assert _bits(got).tolist() == _bits(coords).tolist()
    assert np.array_equal(gbox, box) and np.array_equal(gang, ang)
    assert info["natoms"] == N and info["n_frames"] == F and info["namnf"] == (N - len(kw["free"]) if "free" in kw else 0)
    # a shuffled frame list with repeats that leaves out frame 0, then one that starts with it
    rng = np.random.default_rng(7)
    for sel in (rng.integers(1, F, size=2 * F + 3) if F > 1 else np.zeros(3, np.int64),
                np.concatenate([[0], rng.permutation(F), [F - 1, 0]])):
        got, gbox, gang, _ = pd.read_dcd_frames(fn, sel)
        assert np.array_equal(_bits(got), _bits(coords[:, :, sel])), sel
        assert np.array_equal(gbox, box[:, sel]) and np.array_equal(gang, ang[:, sel])


@pytest.mark.parametrize("endian", ["<", ">"])
@pytest.mark.parametrize("F,N", [(33, 65), (64, 32), (1, 1), (31, 33), (70, 1), (1, 100)])
def test_sizes_off_the_tile_and_special_bit_patterns(tmp_path, endian, F, N):
    from moleculekit_b200 import dcd as pd

    x = _coords(F, N, seed=F * N)
    bits = x.view(np.uint32)
    bits.flat[::5] = 0x80000000  # -0.0
    bits.flat[1::7] = 0x7FC12345  # quiet NaN with a payload
    bits.flat[2::11] = 0xFF800001  # signalling NaN, negative
    bits.flat[3::13] = 0x00000001  # smallest subnormal
    free = np.arange(1, N + 1, 2) if N > 2 else None
    for kw in (dict(endian=endian), dict(endian=endian, free=free, cells=_cells(F))):
        if kw.get("free", 0) is None:
            continue
        raw = od.write(x, **kw)
        coords, _, _ = _want(raw)
        got = pd.read_dcd(_file(tmp_path, raw))[0]
        assert np.array_equal(_bits(got), _bits(coords))


@pytest.mark.parametrize("fixed", [False, True])
def test_large_trajectory_and_many_chunks(tmp_path, fixed):
    from moleculekit_b200 import dcd as pd

    F, N = 2000, 5000
    x = np.random.default_rng(5).normal(0, 30, size=(F, N, 3)).astype(np.float32)
    kw = dict(cells=_cells(F), free=np.arange(1, N + 1, 3) if fixed else None, endian=">" if fixed else "<")
    raw = od.write(x, **kw)
    fn = _file(tmp_path, raw)
    coords, box, _ = _want(raw)
    one = pd.read_dcd_device(fn)[0]
    assert np.array_equal(_bits(one.cpu().numpy()), _bits(coords))
    frame = 3 * 4 * N
    many = pd.read_dcd_device(fn, chunk_bytes=37 * frame)[0]  # 55 chunks
    assert np.array_equal(_bits(many.cpu().numpy()), _bits(coords))
    sel = np.random.default_rng(9).integers(0, F, size=3001)
    sel[sel == 0] = 1
    part, pbox, _, _ = pd.read_dcd_device(fn, frames=sel, chunk_bytes=100 * frame)
    assert np.array_equal(_bits(part.cpu().numpy()), _bits(coords[:, :, sel])) and np.array_equal(pbox, box[:, sel])


@pytest.mark.parametrize("with_box", [False, True])
@pytest.mark.parametrize("F,N", [(1, 1), (5, 33), (67, 100), (300, 2)])
def test_writer_matches_the_oracle_writer(tmp_path, with_box, F, N):
    import torch
    from moleculekit_b200 import dcd as pd

    rng = np.random.default_rng(F + N)
    x = _coords(F, N, seed=N)
    x.view(np.uint32).flat[::9] = 0x7FC0BEEF
    box = rng.uniform(10, 80, size=(3, F)).astype(np.float32) if with_box else None
    ang = rng.uniform(60, 120, size=(3, F)).astype(np.float32) if with_box else None
    title = ["REMARKS written in a test", "y" * 81]
    cells = np.array([od.cosine_cell(*box[:, f], *ang[:, f]) for f in range(F)]) if with_box else None
    want = od.write(x, cells=cells, title=title, istart=10, nsavc=5, delta=0.5)
    coords = np.ascontiguousarray(x.transpose(1, 2, 0))
    got = pd.dcd_bytes(coords, box, ang, istart=10, nsavc=5, delta=0.5, title=title)
    assert got == want
    # a device tensor with a frame stride: the middle F frames of a wider trajectory
    wide = torch.zeros((N, 3, F + 7), dtype=torch.float32, device="cuda")
    wide[:, :, 3:3 + F] = torch.from_numpy(coords).cuda()
    assert pd.dcd_bytes(wide[:, :, 3:3 + F], box, ang, istart=10, nsavc=5, delta=0.5, title=title,
                        chunk_bytes=1000) == want
    assert pd.dcd_bytes(torch.from_numpy(coords).cuda().transpose(0, 1).contiguous().transpose(0, 1), box, ang,
                        istart=10, nsavc=5, delta=0.5, title=title) == want  # another layout: copied first
    # and the file comes back with the input bits
    fn = str(tmp_path / "w.dcd")
    pd.write_dcd(fn, wide[:, :, 3:3 + F], box, ang, title=title, chunk_bytes=3 * (8 + 4 * N) * 2)
    back, bbox, bang, info = pd.read_dcd_device(fn, chunk_bytes=5000)
    assert torch.equal(back.view(torch.int32), wide[:, :, 3:3 + F].contiguous().view(torch.int32))
    assert info["n_frames"] == F and info["has_extra"] == with_box
    if with_box:
        assert np.array_equal(bbox, box)
        assert np.allclose(bang, ang, rtol=0, atol=1e-4)
    dev = pd.encode_dcd_device(wide[:, :, 3:3 + F], box, ang)
    hdr = pd.dcd_header(N, F, istart=10, nsavc=5, delta=0.5, title=title, with_unitcell=with_box)
    assert bytes(dev.cpu().numpy()) == want[len(hdr):]


def test_no_atoms_writes_markers_only():
    from moleculekit_b200 import dcd as pd

    x = np.zeros((0, 3, 4), np.float32)
    box = np.full((3, 4), 20.0, np.float32)
    want = od.write(np.zeros((4, 0, 3)), cells=[od.cosine_cell(20, 20, 20, 90, 90, 90)] * 4, title=["t"])
    assert pd.dcd_bytes(x, box, title=["t"]) == want


def test_xtc_to_dcd_keeps_the_bits(tmp_path):
    import torch
    from moleculekit_b200 import dcd as pd
    from moleculekit_b200 import xtc as px

    gold = os.path.join(ROOT, "tests", "golden", "xtc")
    names = sorted(f[:-4] for f in os.listdir(gold) if f.endswith(".xtc"))
    assert len(names) == 9
    for name in names:
        fn = os.path.join(gold, name + ".xtc")
        coords, box, _, _ = px.read_xtc_device(fn, scale=10)
        out = str(tmp_path / (name + ".dcd"))
        lengths = np.ascontiguousarray(np.diagonal(box, axis1=0, axis2=1).T) * 10
        pd.write_dcd(out, coords, box=lengths)
        back, bbox, bang, _ = pd.read_dcd_device(out)
        assert torch.equal(back.view(torch.int32), coords.view(torch.int32)), name
        assert np.array_equal(bbox, lengths.astype(np.float32)) and (bang == 90).all()


def test_abi_argument_checks():
    import ctypes as C

    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import dcd as pd

    dev = torch.device("cuda", 0)
    coords = torch.zeros((10, 3, 4), device=dev)
    out = torch.empty(4 * 3 * 48, dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.MkbCapacity):
        _lib.call(dev, "mkb_dcd_encode", _lib.ptr(coords), 4, 4, 10, None, _lib.ptr(out), 4 * 3 * 48 - 4)
    with pytest.raises(_lib.MkbError, match="int32 record markers"):
        _lib.call(dev, "mkb_dcd_encode", _lib.ptr(coords), 4, 4, 2**29, None, _lib.ptr(out), 4 * 3 * 48)
    buf = torch.zeros(1024, dtype=torch.uint8, device=dev)
    fr = np.zeros(1, pd.FRAME_DESC)
    fr["count"] = 10
    fr["offset"] = [[4, 48, 1000]]  # Z runs past the end of the buffer
    with pytest.raises(_lib.MkbError, match="frame descriptor 0"):
        pd.decode_dcd_device(buf, fr, 10)
    fr["offset"] = [[4, 48, 98]]  # not on a 4-byte boundary
    with pytest.raises(_lib.MkbError, match="frame descriptor 0"):
        pd.decode_dcd_device(buf, fr, 10)
    fr["offset"] = [[4, 48, 96]]
    fr["count"] = 9  # neither natoms nor a free-atom count
    with pytest.raises(_lib.MkbError, match="frame descriptor 0"):
        pd.decode_dcd_device(buf, fr, 10)
    assert C.sizeof(C.c_int64) * 4 == pd.FRAME_DESC.itemsize
