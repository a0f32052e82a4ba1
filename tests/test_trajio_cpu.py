"""The host plumbing the trajectory modules share (moleculekit_b200/_trajio.py): the text files' line lookups, the slab
gather, the whole-frame stager, the readback of host lines, the decode outputs' check, the writable-range search, and
the rule that every writer checks its arguments before it opens, and so creates or truncates, its file."""
import importlib

import numpy as np
import pytest
import torch

C = np.zeros((12, 3, 4), np.float32)
BOX = np.ones((3, 4), np.float32)
NAN = C.copy()
NAN[5, 1, 2] = np.nan
BOX33 = np.repeat(np.eye(3, dtype=np.float32)[:, :, None] * 10, 4, axis=2)  # (3, 3, F) box vectors, orthorhombic

# what each writer is given besides the file name: arguments it accepts, then changes to them it rejects
WRITERS = {
    "dcd": dict(coords=C),
    "netcdf": dict(coords=C),
    "trr": dict(coords=C, box=np.ones((3, 3, 4), np.float32), time=np.zeros(4), step=np.zeros(4, np.int32)),
    "mdcrd": dict(coords=C),
    "xyz": dict(coords=C, element=["C"] * 12),
    "pdb": dict(coords=C, topology={}),
    "gro": dict(coords=C, topology={}, box=BOX33),
    "cif": dict(coords=C, topology={}),
    "bcif": dict(coords=C, topology={}),
    "lammpstrj": dict(coords=C, box=BOX33),
}
REJECTED = {
    "dcd": [dict(coords=C[:, :2]), dict(box=BOX[:, :3]), dict(boxangles=BOX), dict(box=BOX, boxangles=BOX[:2]),
            dict(istart=2**31), dict(nsavc=-2**31 - 1), dict(title=[1, 2]), dict(chunk_bytes=0)],
    "netcdf": [dict(coords=C[:, :2]), dict(coords=np.zeros((0, 3, 4), np.float32)), dict(box=BOX[:2]),
               dict(boxangles=BOX), dict(time=np.zeros(3)), dict(title="café"), dict(chunk_bytes=0)],
    "trr": [dict(coords=C[0]), dict(box=None), dict(time=np.zeros(3)), dict(step=np.zeros(5)),
            dict(lambd=np.zeros(2)), dict(velocities=C[:, :, :3]), dict(forces=C[:5]), dict(scale=float("nan")),
            dict(chunk_bytes=0)],
    "mdcrd": [dict(coords=C[:, :2]), dict(box=np.ones((2, 4), np.float32)), dict(title="x" * 81), dict(coords=NAN),
              dict(box=np.full((3, 4), 1e4, np.float32)), dict(chunk_bytes=0)],
    "xyz": [dict(coords=C[:, :2]), dict(element=["C"] * 11), dict(element=["C"] * 11 + ["C a"]),
            dict(comment="a\nb"), dict(coords=NAN), dict(chunk_bytes=0)],
    "pdb": [dict(coords=C[:, :2]), dict(box=BOX[:, :3]), dict(boxangles=BOX), dict(topology=dict(name=["CA123"] * 12)),
            dict(coords=NAN), dict(box=np.full((3, 4), 1e6, np.float32)), dict(chunk_bytes=0)],
    "gro": [dict(coords=C[:, :2]), dict(box=None), dict(box=BOX), dict(time=np.zeros(3)), dict(title="a\nb"),
            dict(topology=dict(resname=["SOLVNT"] * 12)), dict(coords=NAN), dict(velocities=C[:, :, :3]),
            dict(chunk_bytes=0)],
    "cif": [dict(coords=C[:, :2]), dict(title="a b"), dict(boxangles=BOX), dict(box=np.arange(12.0).reshape(3, 4)),
            dict(topology=dict(resid=[0.5] * 12)), dict(coords=NAN), dict(chunk_bytes=0)],
    "bcif": [dict(coords=C[:, :2]), dict(coords=C[:, :, :0]), dict(title=""), dict(boxangles=BOX),
             dict(box=np.arange(12.0).reshape(3, 4)), dict(topology=dict(resid=[0.5] * 12)), dict(coords=NAN)],
    "lammpstrj": [dict(coords=C[:, :2]), dict(box=None), dict(box=np.ones((3, 3, 4), np.float32)),
                  dict(step=np.zeros(3)), dict(ids=np.arange(11)), dict(units="two words"),
                  dict(velocities=C[:, :, :3]), dict(chunk_bytes=0)],
}


@pytest.mark.parametrize("fmt", list(WRITERS))
def test_rejected_arguments_leave_an_existing_file_alone(tmp_path, fmt):
    write = getattr(importlib.import_module(f"moleculekit_b200.{fmt}"), f"write_{fmt}")
    fn = tmp_path / f"precious.{fmt}"
    for change in REJECTED[fmt]:
        fn.write_bytes(b"precious")
        with pytest.raises(ValueError):
            write(str(fn), **dict(WRITERS[fmt], **change))
        assert fn.read_bytes() == b"precious", change


def test_slab_gather_reads_only_the_slabs(tmp_path):
    from moleculekit_b200 import _trajio

    rng = np.random.default_rng(4)
    raw = rng.integers(0, 256, size=300000, dtype=np.uint8)
    fn = tmp_path / "bytes"
    fn.write_bytes(raw.tobytes())
    slab = 96
    for starts in (np.arange(0, 200000, 100), np.arange(0, 290000, 96), np.array([8, 104, 5000, 5096, 299900 - 96]),
                   np.sort(rng.choice(2000, size=700, replace=False)) * 140 + 4, np.arange(0, 1100 * 200, 200)):
        out = np.zeros((len(starts), slab), np.uint8)
        with open(fn, "rb") as fh:
            _trajio.gather_slabs(fh.fileno(), starts.astype(np.int64), slab, out, "NetCDF")
        assert np.array_equal(out, raw[starts[:, None] + np.arange(slab)[None, :]])
    with open(fn, "rb") as fh, pytest.raises(RuntimeError, match="changed while it was read"):
        _trajio.gather_slabs(fh.fileno(), np.array([299990], np.int64), slab, np.zeros((1, slab), np.uint8), "NetCDF")


@pytest.mark.parametrize("piece", [1 << 30, 1000])
def test_stage_frames_reads_whole_frames_back_to_back(tmp_path, monkeypatch, piece):
    from moleculekit_b200 import _trajio

    monkeypatch.setattr(_trajio, "PREADV_BYTES", piece)  # 1000: every run longer than that takes several reads
    rng = np.random.default_rng(5)
    raw = rng.integers(0, 256, size=300000, dtype=np.uint8)
    fn = tmp_path / "bytes"
    fn.write_bytes(raw.tobytes())
    size = rng.integers(1, 290, size=1000)  # uneven frames back to back from byte 17
    start = 17 + np.concatenate([[0], np.cumsum(size[:-1])])
    for uniq in (np.arange(1000), np.array([0]), np.array([999]), np.array([3, 4, 5, 9, 10, 500, 998, 999]),
                 np.sort(rng.choice(1000, size=300, replace=False))):
        want = np.concatenate([raw[start[j]:start[j] + size[j]] for j in uniq])
        out = np.zeros(len(want) + 5, np.uint8)
        with open(fn, "rb") as fh:
            at = _trajio.stage_frames(fh.fileno(), start, size, uniq, out, "Test")
        assert at.tolist() == [0] + np.cumsum(size[uniq]).tolist()
        assert np.array_equal(out[:len(want)], want) and not out[len(want):].any()
    with open(fn, "rb") as fh, pytest.raises(RuntimeError, match="Malformed Test file: the file changed while it was"):
        _trajio.stage_frames(fh.fileno(), np.array([299000, 299500]), np.array([500, 501]), np.array([0, 1]),
                             np.zeros(1001, np.uint8), "Test")


def test_stage_frames_starts_a_read_at_each_gap(tmp_path, monkeypatch):
    from moleculekit_b200 import _trajio

    reads = []
    read_exact = _trajio.read_exact
    monkeypatch.setattr(_trajio, "read_exact", lambda fd, buf, pos, fmt: (reads.append(pos), read_exact(fd, buf, pos,
                                                                                                         fmt)))
    rng = np.random.default_rng(6)
    raw = rng.integers(0, 256, size=300000, dtype=np.uint8)
    fn = tmp_path / "bytes"
    fn.write_bytes(raw.tobytes())
    size = rng.integers(1, 200, size=1000)
    gap = rng.integers(0, 3, size=1000) * rng.integers(0, 40, size=1000)  # two in three frames after a gap
    start = 17 + np.concatenate([[0], np.cumsum((size + gap)[:-1])])
    for uniq in (np.arange(1000), np.array([0]), np.array([3, 4, 5, 9, 10, 500, 998, 999]),
                 np.sort(rng.choice(1000, size=300, replace=False))):
        reads.clear()
        want = np.concatenate([raw[start[j]:start[j] + size[j]] for j in uniq])
        out = np.zeros(len(want) + 5, np.uint8)
        with open(fn, "rb") as fh:
            at = _trajio.stage_frames(fh.fileno(), start, size, uniq, out, "Test")
        assert at.tolist() == [0] + np.cumsum(size[uniq]).tolist()
        assert np.array_equal(out[:len(want)], want) and not out[len(want):].any()
        # one read per run of frames that touch in the file
        touch = [start[b] == start[a] + size[a] for a, b in zip(uniq[:-1], uniq[1:])]
        assert reads == [int(start[j]) for j, t in zip(uniq, [False] + touch) if not t]


def _line_ref(raw: bytes, pos: int):
    return raw.count(b"\n", 0, pos), pos - raw.rfind(b"\n", 0, pos)


def test_line_col_and_line_at(tmp_path):
    from moleculekit_b200 import _trajio

    rng = np.random.default_rng(7)
    lines = [bytes(rng.integers(33, 127, size=n, dtype=np.uint8)) for n in (0, 3, 5000, 70, 9000, 1)]
    for raw in (b"\r\n".join(lines) + b"\r\n", b"\n".join(lines), b"\r\n".join(lines)):  # CRLF, no final newline
        fn = tmp_path / "lines"
        fn.write_bytes(raw)
        starts = [0] + [i + 1 for i in range(len(raw)) if raw[i] == 10]
        with open(fn, "rb") as fh:
            for pos in sorted(set(starts + [1, 2, 4, 4100, len(raw) - 1, len(raw)])):
                assert _trajio.line_col(fh.fileno(), pos) == _line_ref(raw, pos), pos
                assert _trajio.line_at(fh.fileno(), pos, len(raw)) == raw[pos:].split(b"\n")[0], pos
            s = starts[2]  # the 5000-byte line
            assert _trajio.line_at(fh.fileno(), s, s + 100) == raw[s:s + 100]  # not past end


def test_line_col_past_the_read_step(tmp_path):
    from moleculekit_b200 import _trajio

    raw = bytearray(b"x" * ((64 << 20) + 3000))  # longer than line_col's 64 MiB read step
    for at in (10, (64 << 20) - 1, (64 << 20) + 5, (64 << 20) + 2000):
        raw[at] = 10
    raw = bytes(raw)
    fn = tmp_path / "long"
    fn.write_bytes(raw)
    with open(fn, "rb") as fh:
        for pos in (0, 11, (64 << 20) - 1, 64 << 20, (64 << 20) + 1, (64 << 20) + 6, (64 << 20) + 2500, len(raw)):
            assert _trajio.line_col(fh.fileno(), pos) == _line_ref(raw, pos), pos


def test_content_end(tmp_path):
    from moleculekit_b200 import _trajio

    fn = tmp_path / "text"
    tail = b" \t\n\v\f\r\x1c\x1d\x1e\x1f"
    for raw in (b"", b" \n\t", tail * 10000, b"abc", b"abc\n", b"a b\x1c" + tail * 10000, b"\x1fa" + tail):
        fn.write_bytes(raw)
        with open(fn, "rb") as fh:
            assert _trajio.content_end(fh.fileno(), len(raw)) == len(raw.decode("ascii").rstrip()), raw[:8]


def _first_bad_ref(x, lo, hi, scale):
    """the first out-of-range value of (natoms, 3, F) or (3, F) ``x`` in file order, element by element"""
    rows = x[None] if x.ndim == 2 else x
    for f in range(x.shape[-1]):
        for atom in range(rows.shape[0]):
            for axis in range(3):
                v = float(rows[atom, axis, f])
                if not (np.isfinite(v) and lo <= np.rint(v * scale) <= hi):
                    return f, atom if x.ndim == 3 else None, axis, v
    return None


@pytest.mark.parametrize("kind", ["numpy", "torch"])
def test_first_bad(kind):
    from moleculekit_b200 import _trajio

    lo, hi = -5000, 7000  # with scale 1000: -5.0 to 7.0
    cases = []
    for shape in ((6, 3, 5), (3, 5)):
        base = np.linspace(-4.9, 6.9, int(np.prod(shape)), dtype=np.float32).reshape(shape)
        first, last = (0,) * len(shape), tuple(n - 1 for n in shape)
        cases.append(base)
        for pos, v in ((first, np.nan), (last, np.nan), (first, -5.0), (last, 7.0), (first, -5.001), (last, 7.001),
                       (last, -5.0005), (last, 7.0005), (last, 6.9995), (last, np.inf)):
            x = base.copy()
            x[pos] = v
            cases.append(x)
        x = base.copy()
        x[(1,) * len(shape)] = 8.0
        x[(0, 2, 1)[3 - len(shape):]] = -6.0  # the earlier frame comes first in the file
        cases.append(x)
        x = base.copy()
        x[(4, 0, 3)[3 - len(shape):]] = 9.0
        x[(2, 1, 3)[3 - len(shape):]] = 9.0  # the same frame: the earlier atom (or axis) first
        cases.append(x)
    for x in cases:
        got = _trajio.first_bad(x if kind == "numpy" else torch.from_numpy(x), lo, hi, 1000)
        want = _first_bad_ref(x, lo, hi, 1000)
        assert (got is None) == (want is None) and (got is None or got[:3] == want[:3]), (got, want)
        if got is not None:
            assert got[3] == want[3] or (np.isnan(got[3]) and np.isnan(want[3]))
    assert _trajio.first_bad(np.zeros((0, 3, 2), np.float32), lo, hi, 1000) is None


def test_flagged_lines():
    from moleculekit_b200 import _trajio

    flags = torch.zeros(1 + 2 * 4, dtype=torch.int64)
    flags[0] = 3
    flags[1:7] = torch.tensor([2 * 5 + 1, 40, 0 * 5 + 4, 7, 1 * 5 + 0, 0])
    k, a, rel = _trajio.flagged(flags, 3, 5, 4, 2)
    assert k.tolist() == [2, 0, 1] and a.tolist() == [1, 4, 0] and rel.tolist() == [40, 7, 0]
    k, a, rel = _trajio.flagged(torch.tensor([3, 2 * 5 + 1, 0 * 5 + 4, 1 * 5 + 0, 0]), 3, 5, 4, 1)
    assert k.tolist() == [2, 0, 1] and a.tolist() == [1, 4, 0] and rel is None
    flags[0] = 5  # past the cap: every atom line of the 3 listed frames
    k, a, rel = _trajio.flagged(flags, 3, 5, 4, 2)
    assert k.tolist() == np.repeat(np.arange(3), 5).tolist() and a.tolist() == list(range(5)) * 3 and rel is None
    flags[0] = 0
    assert [len(v) for v in _trajio.flagged(flags, 3, 5, 4, 1)[:2]] == [0, 0]


def test_decode_outputs():
    from moleculekit_b200 import _trajio

    cpu = torch.device("cpu")
    full = torch.empty(7, 3, 10)
    assert _trajio.decode_outputs(cpu, 7, 10, full) == 10
    assert _trajio.decode_outputs(cpu, 7, 4, full[:, :, 3:7], None, torch.empty(7, 3, 10)[:, :, :4]) == 10
    assert _trajio.decode_outputs(cpu, 7, 1, full[:, :, 9:]) == 10
    assert _trajio.decode_outputs(cpu, 7, 1, torch.empty(7, 3, 1)) == 1
    assert _trajio.decode_outputs(cpu, 7, 5) == 5
    assert _trajio.decode_outputs(cpu, 7, 0, full[:, :, :0]) == 10
    for bad in ((full[:, :, :4], torch.empty(7, 3, 4)),  # two strides
                (torch.empty(10, 7, 3).permute(1, 2, 0)[:, :, :4],),  # frame-major
                (torch.empty(7, 3, 10)[:, :, ::2][:, :, :4],),  # frames apart
                (torch.empty(7, 3, 4, dtype=torch.float64),), (torch.empty(6, 3, 4),)):
        with pytest.raises(AssertionError):
            _trajio.decode_outputs(cpu, 7, 4, *bad)
