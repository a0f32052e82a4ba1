"""K25 on the device: AMBER ASCII trajectories parsed into (natoms, 3, F) and formatted back, bit for bit and byte for
byte against oracle/mdcrd_format.py (float() per field, '%8.3f' per value), an exhaustive table of every F8.3 field,
every malformed-input rule, and grids past 65 535 frame tiles."""
import ctypes
import os

import numpy as np
import pytest

from oracle import mdcrd_format as of
from test_mdcrd_cpu import boxes, frames

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT64_MAX = 2**63 - 1


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _file(tmp_path, raw, name="t.mdcrd"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def _special(xs):
    """-0.0, small negatives that print as -0.000, ties (odd multiples of 1/16) and the range ends sprinkled in"""
    pats = np.float32([-0.0, -0.0004, 0.0625, -0.0625, 0.1875, 9999.999, -999.999, 0.0, -0.0005, 0.0005])
    for k, x in enumerate(xs):
        x.reshape(-1)[k % 3::7] = pats[np.arange(len(x.reshape(-1)[k % 3::7])) % len(pats)]
        np.clip(x, -999.999, 9999.999, out=x)
    return xs


def _want(raw, N, with_box):
    o = of.read(raw, N, with_box)
    c = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
    b = np.ascontiguousarray(o["box"].T) if with_box else np.zeros((3, c.shape[2]), np.float32)
    return c, b


@pytest.mark.parametrize("with_box", [False, True])
@pytest.mark.parametrize("N", [1, 2, 3, 4, 31, 33, 97])
@pytest.mark.parametrize("F", [1, 31, 33, 97])
def test_decoding_matches_the_oracle(tmp_path, with_box, N, F):
    from moleculekit_b200 import mdcrd as pm

    xs = _special(frames(N, F, N * 1000 + F, scale=150.0))
    raw = of.write(xs, boxes(F, F) if with_box else None, title=f"N={N} F={F}")
    fn = _file(tmp_path, raw)
    want_c, want_b = _want(raw, N, with_box)
    coords, box = pm.read_mdcrd(fn, N, box=with_box if N == 1 else None)
    assert coords.shape == (N, 3, F) and np.array_equal(_bits(coords), _bits(want_c))
    assert np.array_equal(_bits(box), _bits(want_b))
    dev, dbox, info = pm.read_mdcrd_device(fn, N, box=with_box, chunk_bytes=1)  # one frame per chunk
    assert np.array_equal(_bits(dev.cpu().numpy()), _bits(want_c)) and np.array_equal(_bits(dbox), _bits(want_b))
    assert info["title"] == f"N={N} F={F}" and info["has_box"] == with_box and info["n_frames"] == F


def _fields_text(fields: np.ndarray, per_frame: int) -> bytes:
    """(n, 8) uint8 fields -> the frames of an mdcrd file with ``per_frame`` (a multiple of 10) fields each, no box"""
    F = len(fields) // per_frame
    lines = fields.reshape(F * per_frame // 10, 80)
    return np.concatenate([lines, np.full((len(lines), 1), 10, np.uint8)], axis=1).tobytes()


def test_every_field(tmp_path):
    from moleculekit_b200 import mdcrd as pm

    k = np.arange(10**7, dtype=np.int64)
    pos = np.stack([(k // 10**6) % 10, (k // 10**5) % 10, (k // 10**4) % 10, (k // 1000) % 10, np.full_like(k, -2),
                    (k // 100) % 10, (k // 10) % 10, k % 10], axis=1).astype(np.uint8) + 48  # "dddd.ddd"
    m = np.arange(1, 10**6, dtype=np.int64)
    neg = np.frombuffer("".join("%8.3f" % -(v / 1000) for v in m.tolist()).encode(), np.uint8).reshape(-1, 8)
    odd = np.frombuffer(b"    .500   -.500-000.500  -0.000", np.uint8).reshape(-1, 8)
    want = np.concatenate([np.float32(k / 1000.0), -np.float32(m / 1000.0), np.float32([0.5, -0.5, -0.5, -0.0])])
    fields = np.concatenate([pos, neg, odd])
    pad = -len(fields) % 30
    fields = np.concatenate([fields, np.frombuffer(b"   0.000" * pad, np.uint8).reshape(-1, 8)])
    want = np.concatenate([want, np.zeros(pad, np.float32)])
    fn = _file(tmp_path, b"every F8.3 field\n" + _fields_text(fields, 30))
    coords, _ = pm.read_mdcrd(fn, 10, box=False)
    got = coords.transpose(2, 0, 1).reshape(-1)
    bad = np.flatnonzero(_bits(got) != _bits(want))
    assert not len(bad), [(bytes(fields[i]), got[i], want[i]) for i in bad[:5]]
    sample = np.random.default_rng(0).integers(0, len(fields), size=20000)
    assert all(_bits(np.float32(float(bytes(fields[i]))))[()] == _bits(got[i])[()] for i in sample)


def _line_col(raw: bytes, at: int):
    """1-based line and column of byte ``at`` of a file"""
    start = raw.rfind(b"\n", 0, at) + 1
    return raw.count(b"\n", 0, at) + 1, at - start + 1


@pytest.mark.parametrize("chunk_frames", [1000, 5])
def test_malformed_input_names_frame_line_and_column(tmp_path, chunk_frames):
    from moleculekit_b200 import mdcrd as pm

    N, F = 7, 40  # 21 values: lines of 80, 80 and 8 characters, then the box line; S = 168 + 3 + 25 = 196
    raw = of.write(frames(N, F, 3), boxes(F, 4), title="malformed")
    S, t0 = pm.frame_bytes(N, True), 81
    chunk = chunk_frames * ((S + 15) & ~15)

    def check(frame, b, new, field_start):
        at = t0 + frame * S + b
        bad = raw[:at] + new + raw[at + len(new):]
        fn = _file(tmp_path, bad)
        with pytest.raises(ValueError) as e:
            pm.read_mdcrd_device(fn, N, box=True, chunk_bytes=chunk)  # a broken box line of frame 0 hides the box
        line, col = _line_col(bad, t0 + frame * S + field_start)
        msg = str(e.value)
        assert f"frame {frame} " in msg and f"line {line}, column {col}:" in msg, (msg, line, col)
        return msg

    for frame in (0, 33, 39):
        for b, new in ((8, b"********"), (13, b"x"), (8, b"+"), (10, b"\t"), (85, b"0"), (163, b"\r")):
            check(frame, b, new, b - (b % 81) % 8)
        msg = check(frame, 80, b" ", 80)  # the first line's newline is missing
        assert "expected the newline" in msg
        check(frame, 40, b"\n", 40)  # a newline inside a field
        check(frame, 171 + 9, b"a", 171 + 8)  # the box line's second field
        check(frame, 171 + 24, b"0", 171 + 24)  # the box line's newline
    # the first bad byte in file order wins, across chunks
    bad = bytearray(raw)
    bad[t0 + 20 * S + 100] = ord("?")
    bad[t0 + 12 * S + 171 + 2] = ord("x")
    bad[t0 + 12 * S + 90] = ord("y")
    fn = _file(tmp_path, bytes(bad))
    with pytest.raises(ValueError, match=r"frame 12 .*line %d, column %d:" % _line_col(bytes(bad), t0 + 12 * S + 89)):
        pm.read_mdcrd_device(fn, N, chunk_bytes=chunk)
    # only the listed frames are parsed
    ok = [k for k in range(F) if k not in (12, 20)]
    got = pm.read_mdcrd_device(fn, N, frames=ok, chunk_bytes=chunk)[0].cpu().numpy()
    assert np.array_equal(_bits(got), _bits(_want(raw, N, True)[0][:, :, ok]))
    # the wrong atom count puts newlines where fields should be
    fn = _file(tmp_path, raw)
    for n in (6, 8, 3):
        with pytest.raises(ValueError, match=rf"frame 0 \(natoms={n}, with box line\), line \d+, column \d+: "):
            pm.read_mdcrd_device(fn, n, box=True)


def test_frame_lists_chunks_and_odd_frame_sizes(tmp_path):
    from moleculekit_b200 import mdcrd as pm

    for N, with_box in ((5, True), (6, False), (45, True)):  # S = 147, 146, 1119
        F = 60
        raw = of.write(frames(N, F, N), boxes(F, N) if with_box else None)
        fn = _file(tmp_path, raw)
        want_c, want_b = _want(raw, N, with_box)
        rng = np.random.default_rng(N)
        for sel in (rng.integers(0, F, size=77), np.arange(F)[::-1], [F - 1, 0, F - 1, 0], [-1]):
            for chunk in (1, 3 * pm.frame_bytes(N, with_box), 1 << 20):
                c, b, info = pm.read_mdcrd_device(fn, N, frames=sel, chunk_bytes=chunk)
                sel_ = np.arange(F)[np.asarray(sel)]
                assert np.array_equal(_bits(c.cpu().numpy()), _bits(want_c[:, :, sel_]))
                assert np.array_equal(_bits(b), _bits(want_b[:, sel_])) and np.array_equal(info["frames"], sel_)
        c, b = pm.read_mdcrd_frames(fn, N, [3, 3, 1])
        assert np.array_equal(_bits(c), _bits(want_c[:, :, [3, 3, 1]]))
        for bad in ([F], [-F - 1]):
            with pytest.raises(IndexError):
                pm.read_mdcrd_device(fn, N, frames=bad)
    # a truncated last frame is dropped
    raw = of.write(frames(5, 4, 1), None)
    c, _ = pm.read_mdcrd(_file(tmp_path, raw[:-30]), 5)
    assert c.shape == (5, 3, 3) and np.array_equal(_bits(c), _bits(_want(raw, 5, False)[0][:, :, :3]))


def test_past_65535_frame_tiles(tmp_path):
    import torch
    from moleculekit_b200 import mdcrd as pm

    F = 65536 * 32 + 37  # one-atom frames: 65 538 frame tiles
    k = (np.arange(3 * F, dtype=np.int64) * 7919) % 10**7 - 999999
    x = np.float32(k / 1000.0)
    text = "".join("%8.3f%8.3f%8.3f\n" % tuple(v) for v in x.reshape(F, 3)[:3].tolist())
    assert len(text) == 75
    # every frame's line at once: fields built from the integers, checked against '%8.3f' on the first frames above
    a = np.abs(k)
    ch = np.full((3 * F, 8), 32, np.uint8)
    ch[:, 4] = 46
    for c, p in ((7, 1), (6, 10), (5, 100), (3, 1000), (2, 10**4), (1, 10**5), (0, 10**6)):
        d = (a // p) % 10
        keep = (a >= p) | (c >= 3)
        ch[:, c] = np.where(keep, d + 48, ch[:, c])
    nd = 1 + (a >= 10**4) + (a >= 10**5) + (a >= 10**6)
    neg = np.flatnonzero(k < 0)
    ch[neg, 3 - nd[neg]] = 45
    lines = np.concatenate([ch.reshape(F, 24), np.full((F, 1), 10, np.uint8)], axis=1)
    assert lines[:3].tobytes().decode() == text
    raw = b"long\n" + lines.tobytes()
    fn = _file(tmp_path, raw)
    want = x.reshape(F, 1, 3).transpose(1, 2, 0)
    got, _, _ = pm.read_mdcrd_device(fn, 1, box=False)
    g = got.cpu().numpy()
    bad = np.flatnonzero((_bits(g) != _bits(want)).any(axis=(0, 1)))
    assert not len(bad), (bad[:5], g[:, :, bad[:3]], want[:, :, bad[:3]])
    # and back: one encode launch over all frames, from a device copy kept alive
    src = torch.from_numpy(np.ascontiguousarray(want)).cuda()
    enc = pm.encode_mdcrd_device(src)
    assert enc.numel() == 25 * F and bytes(enc.cpu().numpy()) == raw[5:]


@pytest.mark.parametrize("F,N", [(1, 1), (5, 33), (67, 100), (300, 2)])
def test_writer_matches_the_oracle(tmp_path, F, N):
    import torch
    from moleculekit_b200 import mdcrd as pm

    xs = _special(frames(N, F, F + N, scale=150.0))
    x = np.ascontiguousarray(np.stack(xs, axis=2))
    bx = np.ascontiguousarray(np.stack(boxes(F, N), axis=1))
    for b in (None, bx):
        want = of.write(xs, None if b is None else list(b.T), title="writer")
        assert pm.mdcrd_bytes(x, b, title="writer") == want
        S = pm.frame_bytes(N, b is not None)
        wide = torch.zeros((N, 3, F + 7), dtype=torch.float32, device="cuda")
        wide[:, :, 3:3 + F] = torch.from_numpy(x).cuda()
        wbox = None
        if b is not None:
            wbox = torch.zeros((3, F + 5), dtype=torch.float32, device="cuda")
            wbox[:, 2:2 + F] = torch.from_numpy(b).cuda()
            wbox = wbox[:, 2:2 + F]
        view = wide[:, :, 3:3 + F]
        assert pm.mdcrd_bytes(view, wbox, title="writer", chunk_bytes=2 * S + 1) == want
        fn = str(tmp_path / "w.mdcrd")
        pm.write_mdcrd(fn, view, b, title="writer", chunk_bytes=S)
        assert open(fn, "rb").read() == want
        assert bytes(pm.encode_mdcrd_device(view, wbox).cpu().numpy()) == want[81:]
        back, bbox = pm.read_mdcrd(fn, N, box=b is not None)
        want_c, want_b = _want(want, N, b is not None)
        assert np.array_equal(_bits(back), _bits(want_c)) and np.array_equal(_bits(bbox), _bits(want_b))


def test_writer_rounding_and_range():
    import torch
    from moleculekit_b200 import mdcrd as pm

    # every odd multiple of 1/16 in the writable range, both signs: the ties of '%8.3f'
    m = np.arange(1, 160000, 2)
    v = np.concatenate([np.float32(m / 16), -np.float32(m[m < 16000] / 16)])
    v = np.concatenate([v, np.float32([-0.0, -1e-30, -0.0004, -0.00049, 0.0004, 0.0])])
    v = np.concatenate([v, np.zeros(-len(v) % 3, np.float32)])
    x = v.reshape(-1, 3, 1)
    got = pm.mdcrd_bytes(x)[81:]
    want = "".join("%8.3f" % f for f in v.tolist())
    assert got.replace(b"\n", b"") == want.encode() and "  -0.000" * 4 + "   0.000" * 2 in want
    # the range ends: the largest float32 that rounds to 9999.999 / -999.999 is written, the next one rejected
    hi = np.float32(9999.999)
    while np.rint(np.float64(np.nextafter(hi, np.float32(np.inf))) * 1000) <= 9999999:
        hi = np.nextafter(hi, np.float32(np.inf))
    lo = np.float32(-999.999)
    while np.rint(np.float64(np.nextafter(lo, np.float32(-np.inf))) * 1000) >= -999999:
        lo = np.nextafter(lo, np.float32(-np.inf))
    for dev in (False, True):
        def put(val):
            a = np.zeros((4, 3, 2), np.float32)
            a[2, 1, 1] = val
            return torch.from_numpy(a).cuda() if dev else a

        assert pm.mdcrd_bytes(put(hi))[81 + 98 + 56:][:8] == b"9999.999"  # frame 1, value 7
        assert b"-999.999" in pm.mdcrd_bytes(put(lo))
        for bad in (np.nextafter(hi, np.float32(np.inf)), np.nextafter(lo, np.float32(-np.inf)), np.nan, np.inf,
                    -np.inf):
            with pytest.raises(ValueError, match="frame 1, atom 2, axis y"):
                pm.mdcrd_bytes(put(bad))
        with pytest.raises(ValueError, match="frame 1, atom 2, axis y"):
            pm.encode_mdcrd_device(put(np.nan) if dev else torch.from_numpy(put(np.nan)).cuda())


def test_xtc_goldens_through_mdcrd(tmp_path):
    from moleculekit_b200 import mdcrd as pm
    from moleculekit_b200 import xtc as px

    gold = os.path.join(ROOT, "tests", "golden", "xtc")
    names = sorted(f[:-4] for f in os.listdir(gold) if f.endswith(".xtc"))
    assert len(names) == 9
    for name in names:
        coords, box, _, _ = px.read_xtc_device(os.path.join(gold, name + ".xtc"), scale=10)
        c = coords.cpu().numpy()
        lengths = np.float32(np.diagonal(np.asarray(box), axis1=0, axis2=1).T * np.float32(10))
        out = str(tmp_path / (name + ".mdcrd"))
        k = np.rint(c.astype(np.float64) * 1000)
        if ((k > 9999999) | (k < -999999)).any():  # the wide goldens reach +-90 000 Angstrom: F8.3 cannot hold them
            f, a, d = np.argwhere(((k > 9999999) | (k < -999999)).transpose(2, 0, 1))[0]
            with pytest.raises(ValueError, match=f"frame {f}, atom {a}, axis {'xyz'[d]}"):
                pm.write_mdcrd(out, coords, lengths, title=name)
            assert not os.path.exists(out)
            continue
        pm.write_mdcrd(out, coords, lengths, title=name)
        raw = of.write(list(c.transpose(2, 0, 1)), list(lengths.T), title=name)
        assert open(out, "rb").read() == raw, name
        back, bbox = pm.read_mdcrd(out, c.shape[0], box=True)
        want_c, want_b = _want(raw, c.shape[0], True)
        assert np.array_equal(_bits(back), _bits(want_c)) and np.array_equal(_bits(bbox), _bits(want_b)), name


def _at(t, offset):
    """a pointer ``offset`` bytes into a tensor"""
    return ctypes.c_void_p(t.data_ptr() + offset)


def test_abi_argument_checks():
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import mdcrd as pm

    dev = torch.device("cuda", 0)
    N, F = 10, 4
    S = pm.frame_bytes(N, True)  # 240 + 3 + 25 = 268
    x = torch.zeros((N, 3, F), device=dev)
    box = torch.full((3, F), 30.0, device=dev)
    out = torch.empty(F * S + 16, dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.MkbCapacity, match=str(F * S)):
        _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F, F, N, _lib.ptr(box), F, _lib.ptr(out), F * S - 1)
    with pytest.raises(_lib.MkbCapacity, match=str(F * (S - 25))):
        _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F, F, N, None, 0, _lib.ptr(out), F * (S - 25) - 1)
    with pytest.raises(_lib.MkbError, match="4-byte aligned"):
        _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F, F, N, _lib.ptr(box), F, _at(out, 2), F * S)
    with pytest.raises(_lib.MkbError, match="frame stride"):
        _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F - 1, F, N, _lib.ptr(box), F, _lib.ptr(out), F * S)
    with pytest.raises(_lib.MkbError, match="natoms"):
        _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F, F, 0, _lib.ptr(box), F, _lib.ptr(out), F * S)
    with pytest.raises(_lib.MkbError, match="null"):
        _lib.call(dev, "mkb_mdcrd_encode", None, F, F, N, _lib.ptr(box), F, _lib.ptr(out), F * S)
    _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), F, F, N, _lib.ptr(box), F, _lib.ptr(out), F * S)
    frame = bytes(out[:S].cpu().numpy())
    assert frame == (b"   0.000" * 10 + b"\n") * 3 + b"  30.000" * 3 + b"\n"
    # decode: staged rows of 272 bytes
    row = (S + 15) & ~15
    buf = torch.zeros(F * row, dtype=torch.uint8, device=dev)
    for k in range(F):
        buf[k * row:k * row + S] = out[k * S:(k + 1) * S]
    c = torch.empty((N, 3, F), device=dev)
    b = torch.empty((3, F), device=dev)
    bad = torch.full((1,), INT64_MAX, dtype=torch.int64, device=dev)
    offs = np.arange(F, dtype=np.int64) * row
    pm.decode_mdcrd_device(buf, offs, N, True, out=c, box_out=b, bad=bad)
    assert int(bad.item()) == INT64_MAX and not c.any() and (b == 30).all()

    def dec(offsets, n=N, nbytes=None, bp=None, cp=None, badp=None):
        o = np.asarray(offsets, np.int64)
        _lib.call(dev, "mkb_mdcrd_decode", _lib.ptr(buf) if bp is None else bp,
                  buf.numel() if nbytes is None else nbytes, o.ctypes.data_as(ctypes.c_void_p), len(o), n, 1,
                  _lib.ptr(c) if cp is None else cp, F, _lib.ptr(b), F, _lib.ptr(bad) if badp is None else badp)

    for offsets in ([8], [-16], [F * row - 256], [F * row]):
        with pytest.raises(_lib.MkbError, match="offset"):
            dec(offsets)
    dec([F * row - 272])  # the last row: 268 bytes, 268 in whole words
    with pytest.raises(_lib.MkbError, match="offset"):
        dec([0], nbytes=S - 1)
    with pytest.raises(_lib.MkbError, match="16-byte aligned"):
        dec([0], bp=_at(buf, 4), nbytes=F * row - 16)
    with pytest.raises(_lib.MkbError, match="8-byte aligned"):
        dec([0], badp=_at(bad, 4))
    with pytest.raises(_lib.MkbError, match="4-byte aligned"):
        dec([0], cp=_at(c, 2))
    with pytest.raises(_lib.MkbError, match="natoms"):
        dec([0], n=0)
    with pytest.raises(_lib.MkbError, match="null"):
        dec([0], badp=ctypes.c_void_p(0))
    with pytest.raises(_lib.MkbError, match="null"):
        _lib.call(dev, "mkb_mdcrd_decode", _lib.ptr(buf), buf.numel(), np.zeros(1, np.int64).ctypes.data_as(
            ctypes.c_void_p), 1, N, 1, _lib.ptr(c), F, None, F, _lib.ptr(bad))
    assert int(bad.item()) == INT64_MAX
