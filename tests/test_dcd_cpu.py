"""The host side of DCD reading and writing (moleculekit_b200/dcd.py; K22 moves the coordinates on the device): the
independent format restatement in oracle/dcd_format.py, the header and frame walk of index_dcd against it, the unit-cell
conversions, the header write_dcd writes, the argument checks that run before any device work, and the C-ABI symbols."""
import os
import struct

import numpy as np
import pytest

from oracle import dcd_format as od

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _coords(F, N, seed=0):
    return np.random.default_rng(seed).normal(0, 12, size=(F, N, 3)).astype(np.float32)


def _cells(F, seed=1):
    rng = np.random.default_rng(seed)
    return np.array([od.cosine_cell(*rng.uniform(20, 60, 3), *rng.uniform(60, 120, 3)) for _ in range(F)])


# every layout the reader must accept: (name, F, N, writer keywords)
VARIANTS = [
    ("plain", 5, 17, {}),
    ("big_endian", 5, 17, dict(endian=">")),
    ("markers_64", 4, 9, dict(marker=8)),
    ("big_endian_markers_64", 4, 9, dict(endian=">", marker=8)),
    ("xplor", 3, 11, dict(charmm=False, delta=0.002)),
    ("cosine_cell", 6, 40, dict(cells=_cells(6))),
    ("degree_cell", 3, 8, dict(cells=np.tile([[31.0, 70.0, 32.0, 80.0, 95.0, 33.0]], (3, 1)))),
    ("odd_extra_block", 3, 8, dict(cells=np.ones((3, 4)))),
    ("four_d", 4, 12, dict(cells=_cells(4), four_d=True)),
    ("fixed", 5, 33, dict(free=np.arange(1, 34, 3))),
    ("fixed_cell_be64", 4, 20, dict(free=[2, 5, 6, 19], cells=_cells(4), endian=">", marker=8, four_d=True)),
    ("title", 2, 5, dict(title=["REMARKS first", "x" * 95, ""], istart=100, nsavc=50)),
    ("nset_zero", 4, 6, dict(nset=0)),
    ("one_atom_one_frame", 1, 1, {}),
]


def _expected(x, kw):
    """what a reader returns for coords x written with ``kw``: a fixed atom keeps its first-frame position"""
    if "free" not in kw:
        return x
    fixed = np.ones(x.shape[1], bool)
    fixed[np.asarray(kw["free"]) - 1] = False
    e = x.copy()
    e[1:, fixed] = x[0, fixed]
    return e


def _host_decode(raw, idx):
    """coords (N, 3, F) from index_dcd's frame table, with the fixed-atom rule of K22 (a host restatement)"""
    dt = (">" if idx["swap"] else "<") + "f4"
    N, F = idx["natoms"], idx["n_frames"]
    slot = None
    if idx["free"] is not None:
        slot = np.full(N, -1)
        slot[idx["free"]] = np.arange(len(idx["free"]))
    out = np.zeros((N, 3, F), np.float32)
    first = idx["frames"][0] if F else None
    for k, fr in enumerate(idx["frames"]):
        for d in range(3):
            rec = np.frombuffer(raw, dt, count=int(fr["count"]), offset=int(fr["offset"][d]))
            if fr["count"] == N:
                out[:, d, k] = rec
            else:
                base = np.frombuffer(raw, dt, count=N, offset=int(first["offset"][d]))
                out[:, d, k] = np.where(slot >= 0, rec[np.maximum(slot, 0)], base)
    return out


@pytest.mark.parametrize("name,F,N,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_oracle_round_trip(name, F, N, kw):
    x = _coords(F, N)
    got = od.read(od.write(x, **kw))
    assert got["natoms"] == N and got["coords"].shape == (F, N, 3)
    assert np.array_equal(got["coords"].view(np.int32), _expected(x, kw).view(np.int32))
    assert got["endian"] == kw.get("endian", "<") and got["marker"] == kw.get("marker", 4)
    assert got["charmm"] == kw.get("charmm", True) and got["four_d"] == kw.get("four_d", False)
    assert got["nset"] == kw.get("nset", F) and got["trailing"] == 0
    cells = kw.get("cells")
    if cells is not None and cells.shape[1] == 6:
        assert np.array_equal(got["cells"], cells)
    if "free" in kw:
        assert got["namnf"] == N - len(kw["free"]) and np.array_equal(got["free"], kw["free"])
    if "title" in kw:
        assert [t.rstrip() for t in got["title"]] == [t[:80] for t in kw["title"]]


@pytest.mark.parametrize("name,F,N,kw", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_index_matches_the_oracle(name, F, N, kw):
    from moleculekit_b200 import dcd as pd

    x = _coords(F, N)
    raw = od.write(x, **kw)
    want = od.read(raw)
    idx = pd.index_dcd(raw)
    for key, okey in (("natoms", "natoms"), ("nset", "nset"), ("istart", "istart"), ("nsavc", "nsavc"),
                      ("namnf", "namnf"), ("charmm", "charmm"), ("has_extra", "extra"), ("has_4d", "four_d"),
                      ("title", "title"), ("marker_bytes", "marker")):
        assert idx[key] == want[okey], key
    assert idx["swap"] == (want["endian"] == ">") and idx["n_frames"] == F
    assert np.float32(idx["delta"]) == np.float32(want["delta"])
    assert np.array_equal(idx["box"], want["box"].T) and np.array_equal(idx["boxangles"], want["angles"].T)
    assert np.array_equal(_host_decode(raw, idx).view(np.int32), want["coords"].transpose(1, 2, 0).view(np.int32))
    assert idx["start"][0] + idx["size"].sum() == len(raw)


def test_truncated_files_drop_the_partial_frame():
    from moleculekit_b200 import dcd as pd

    for kw in ({}, dict(free=[1, 4, 7], cells=_cells(5), four_d=True), dict(marker=8, endian=">")):
        raw = od.write(_coords(5, 9), **kw)
        header_end = int(pd.index_dcd(raw)["start"][0])
        for cut in range(len(raw) - 1, header_end - 1, -13):
            want = od.read(raw[:cut])
            idx = pd.index_dcd(raw[:cut])
            assert idx["n_frames"] == len(want["coords"]) and (cut > header_end or idx["n_frames"] == 0)
            assert np.array_equal(_host_decode(raw[:cut], idx), want["coords"].transpose(1, 2, 0))
        for cut in range(0, header_end, 3):  # a cut inside the header is an error, not an empty trajectory
            with pytest.raises(RuntimeError, match="Malformed DCD file"):
                pd.index_dcd(raw[:cut])
    with pytest.raises(RuntimeError, match="Malformed DCD file"):
        pd.index_dcd(od.write(_coords(1, 4))[:50])
    with pytest.raises(RuntimeError, match="Malformed DCD file"):
        pd.index_dcd(b"\x00" * 200)


def test_bad_markers_name_the_frame():
    from moleculekit_b200 import dcd as pd

    F, N = 6, 10
    for kw in ({}, dict(cells=_cells(F)), dict(free=[2, 3], marker=8)):
        raw = od.write(_coords(F, N), **kw)
        idx = pd.index_dcd(raw)
        for f in (0, 1, 4, 5):
            for d in range(3):
                mw = idx["marker_bytes"]
                at = int(idx["frames"]["offset"][f, d]) + 4 * int(idx["frames"]["count"][f])  # trailing marker
                bad = bytearray(raw)
                bad[at:at + mw] = struct.pack("<i" if mw == 4 else "<q", 12345)
                with pytest.raises(RuntimeError, match=f"Malformed DCD file: frame {f}"):
                    pd.index_dcd(bytes(bad))


def test_nset_disagreeing_with_the_bytes_is_not_an_error():
    from moleculekit_b200 import dcd as pd

    for nset in (0, 2, 99):
        idx = pd.index_dcd(od.write(_coords(5, 3), nset=nset))
        assert idx["nset"] == nset and idx["n_frames"] == 5


def test_unit_cell_conversions():
    from moleculekit_b200 import dcd as pd

    # a zero cosine comes back as exactly 90 degrees
    box, ang = pd.unitcell_to_box([[10.0, 0.0, 11.0, 0.0, 0.0, 12.0]])
    assert np.array_equal(ang[:, 0], np.float32([90, 90, 90])) and np.array_equal(box[:, 0], np.float32([10, 11, 12]))
    assert np.array_equal(pd.box_to_unitcell(np.float32([[10], [11], [12]]))[0], [10, 0, 11, 0, 0, 12])
    # degrees are taken as they are once any angle slot is outside [-1, 1]
    box, ang = pd.unitcell_to_box([[30.0, 70.5, 31.0, 0.5, 95.25, 32.0]])
    assert np.array_equal(ang[:, 0], np.float32([95.25, 0.5, 70.5]))
    # against the oracle on random cells, and the writer's cosines
    rng = np.random.default_rng(3)
    cells = _cells(300, seed=4)
    cells[::7, 1] = 0.0
    cells[::11, 0] = -0.0
    box, ang = pd.unitcell_to_box(cells)
    for f in range(len(cells)):
        want = od.cell_to_box(cells[f])
        assert np.array_equal(np.concatenate([box[:, f], ang[:, f]]).view(np.int32), np.array(want).view(np.int32))
    b = rng.uniform(10, 90, size=(3, 50)).astype(np.float32)
    a = rng.uniform(50, 130, size=(3, 50)).astype(np.float32)
    got = pd.box_to_unitcell(b, a)
    want = np.array([od.cosine_cell(*b[:, f], *a[:, f]) for f in range(50)])
    assert np.array_equal(got.view(np.int64), want.view(np.int64))
    # round trip of 90 degrees through the writer's cosine and the reader's asin
    box, ang = pd.unitcell_to_box(pd.box_to_unitcell(b, np.full((3, 50), 90, np.float32)))
    assert np.array_equal(ang, np.full((3, 50), 90, np.float32)) and np.array_equal(box, b)


@pytest.mark.parametrize("title", [None, "one line", ["REMARKS a", "b" * 100, ""]])
@pytest.mark.parametrize("with_box", [False, True])
def test_header_bytes_match_the_oracle(title, with_box):
    from moleculekit_b200 import dcd as pd

    N = 23
    lines = list(pd.DEFAULT_TITLE) if title is None else ([title] if isinstance(title, str) else title)
    for F in (0, 3):
        want = od.write(_coords(F, N), cells=_cells(F) if with_box else None, title=lines, istart=7, nsavc=3,
                        delta=0.25)
        hdr = pd.dcd_header(N, F, istart=7, nsavc=3, delta=0.25, title=title, with_unitcell=with_box)
        assert want[:len(hdr)] == hdr
        assert od.read(hdr + want[len(hdr):])["icntrl3"] == 7 + 3 * F
    # no frames: the header is the whole file and needs no device
    box = np.zeros((3, 0), np.float32) if with_box else None
    got = pd.dcd_bytes(np.zeros((N, 3, 0), np.float32), box=box, istart=7, nsavc=3, delta=0.25, title=title)
    assert got == od.write(np.zeros((0, N, 3)), cells=np.zeros((0, 6)) if with_box else None, title=lines, istart=7,
                           nsavc=3, delta=0.25)


def test_arguments_are_checked_before_the_device_is_touched(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import dcd as pd

    c = np.zeros((12, 3, 4), np.float32)
    box = np.ones((3, 4), np.float32)
    for args, kw in (((c[:, :2],), {}), ((c[0],), {}), ((c,), dict(box=box[:, :3])), ((c,), dict(box=box[:2])),
                     ((c,), dict(box=box, boxangles=box[:, :2])), ((c,), dict(boxangles=box)),
                     ((c,), dict(istart=2**31)), ((c,), dict(nsavc=-2**31 - 1)), ((c,), dict(title=[1, 2])),
                     ((c,), dict(chunk_bytes=0)),
                     ((np.broadcast_to(np.float32(0), (pd.MAX_ATOMS + 1, 3, 1)),), {})):
        with pytest.raises(ValueError):
            pd.dcd_bytes(*args, **kw)
        fn = tmp_path / "untouched.dcd"
        with pytest.raises(ValueError):
            pd.write_dcd(str(fn), *args, **kw)
        assert not fn.exists()
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pd.encode_dcd_device(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pd.dcd_bytes(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pd.decode_dcd_device(torch.zeros(16, dtype=torch.uint8), np.zeros(0, pd.FRAME_DESC), 4)
    fn = tmp_path / "t.dcd"
    fn.write_bytes(od.write(_coords(3, 5)))
    for bad in ([3], [-4], [0, 7]):
        with pytest.raises(IndexError):
            pd.read_dcd_frames(str(fn), bad)
    with pytest.raises(ValueError):
        pd.read_dcd_device(str(fn), chunk_bytes=0)
    empty = tmp_path / "empty.dcd"
    empty.write_bytes(b"")
    with pytest.raises(RuntimeError, match="Malformed DCD file"):
        pd.read_dcd(str(empty))
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pd.dcd_bytes(c)
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pd.read_dcd(str(fn))


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    for name, nargs in (("mkb_dcd_decode", 15), ("mkb_dcd_encode", 9)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    assert "} mkb_dcd_frame;" in hdr
    from moleculekit_b200 import dcd as pd

    assert pd.FRAME_DESC.itemsize == 32
