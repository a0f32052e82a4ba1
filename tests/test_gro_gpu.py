"""K29 on the GPU: GRO files indexed and parsed on the device bit for bit as the oracle reader (np.float32(float(field))
of the column slices, NaN signs included), field widths 7, 8 and 10 with and without velocities, fields outside the
fast paths, the lines left to the host, 3- and 9-value boxes, titles with and without time and step, line endings,
chunking and frame lists, every error message, the writer byte for byte Python's '%' formatting, and more than 65 535
frame tiles in one index, decode and encode."""
import logging

import numpy as np
import pytest
import torch

from oracle import gro_format as og

pytestmark = pytest.mark.gpu

WATERS = b"""MD of 2 waters, t= 0.0
    6
    1WATER  OW1    1   0.126   1.624   1.679  0.1227 -0.0580  0.0434
    1WATER  HW2    2   0.190   1.661   1.747  0.8085  0.3191 -0.7791
    1WATER  HW3    3   0.177   1.568   1.613 -0.9045 -2.6469  1.3180
    2WATER  OW1    4   1.275   0.053   0.622  0.2519  0.3140 -0.1734
    2WATER  HW2    5   1.337   0.002   0.680 -1.0641 -1.1349  0.0257
    2WATER  HW3    6   1.326   0.120   0.568  1.9427 -0.8216 -0.0244
   1.82060   1.82060   1.82060
"""


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def put(tmp_path, raw, name="t.gro"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def check(tmp_path, raw, host_lines=0, frames=None, **kw):
    """read_gro_device against the oracle reader: positions, velocities, box, time and step bit for bit"""
    from moleculekit_b200 import gro

    want = og.read(raw)
    fields = ("x", "v") if want["velocities"] else ("x",)
    got, box, info = gro.read_gro_device(put(tmp_path, raw), frames=frames, fields=fields, **kw)
    sel = slice(None) if frames is None else np.asarray(frames)
    assert np.array_equal(bits(got["x"].cpu().numpy()), bits(want["coords"].transpose(1, 2, 0)[:, :, sel]))
    if want["velocities"]:
        assert np.array_equal(bits(got["v"].cpu().numpy()), bits(want["vels"].transpose(1, 2, 0)[:, :, sel]))
    assert np.array_equal(bits(box), bits(want["box"].transpose(1, 2, 0)[:, :, sel]))
    assert np.array_equal(bits(info["time"]), bits(want["time"][sel]))
    assert np.array_equal(info["step"], want["step"][sel])
    assert info["width"] == want["width"] and info["velocities"] == want["velocities"]
    if host_lines is not None:
        assert info["host_lines"] == host_lines
    return info


def hand_file(N, F, seed, w=8, d=3, vel=False, nl="\n", nine=False,
              title=lambda f: f"frame {f} t= {f * 0.5} step= {f}"):
    """a file written line by line with '%w.df' positions and '%w.(d+1)f' velocities"""
    rng = np.random.default_rng(seed)
    out = []
    for f in range(F):
        out.append(title(f))
        out.append("%5d" % N)
        for a in range(N):
            line = "%5d%-5s%5s%5d" % (a // 3 + 1, "SOL", "OW", a + 1)
            line += "".join(f"%{w}.{d}f" % v for v in rng.uniform(-9.9, 99.9, 3))
            if vel:
                line += "".join(f"%{w}.{d + 1}f" % v for v in rng.uniform(-9.9, 9.9, 3))
            out.append(line)
        b = rng.uniform(1, 9, 9)
        out.append(" ".join("%.5f" % v for v in (b if nine else b[:3])))
    return (nl.join(out) + nl).encode()


def test_two_waters_in_the_manual_layout(tmp_path):
    from moleculekit_b200 import gro

    got, box, info = gro.read_gro_device(put(tmp_path, WATERS), fields=("x", "v"))
    x = np.float32([[0.126, 1.624, 1.679], [0.190, 1.661, 1.747], [0.177, 1.568, 1.613],
                    [1.275, 0.053, 0.622], [1.337, 0.002, 0.680], [1.326, 0.120, 0.568]])
    v = np.float32([[0.1227, -0.0580, 0.0434], [0.8085, 0.3191, -0.7791], [-0.9045, -2.6469, 1.3180],
                    [0.2519, 0.3140, -0.1734], [-1.0641, -1.1349, 0.0257], [1.9427, -0.8216, -0.0244]])
    assert np.array_equal(bits(got["x"][:, :, 0].cpu().numpy()), bits(x))
    assert np.array_equal(bits(got["v"][:, :, 0].cpu().numpy()), bits(v))
    assert np.array_equal(bits(box[:, :, 0]), bits(np.diag(np.float32([1.82060] * 3))))
    assert info["time"].tolist() == [0.0] and info["step"].tolist() == [-1]
    assert info["natoms"] == 6 and info["n_frames"] == 1 and info["width"] == 8 and info["velocities"]
    t = info["topology"]
    assert t["resid"].tolist() == [1, 1, 1, 2, 2, 2] and list(t["resname"]) == ["WATER"] * 6
    assert list(t["name"]) == ["OW1", "HW2", "HW3"] * 2 and t["serial"].tolist() == [1, 2, 3, 4, 5, 6]
    check(tmp_path, WATERS)
    back, b10, t10, s10 = gro.read_gro(put(tmp_path, WATERS), scale=10.0)  # read_trr's return shape
    assert np.array_equal(bits(back[:, :, 0]), bits(x * np.float32(10)))
    assert t10.dtype == np.float64 and t10.tolist() == [0.0] and s10.dtype == np.int64 and s10.tolist() == [-1]
    assert np.array_equal(bits(b10), bits(box))  # scale touches positions only


@pytest.mark.parametrize("w, d, vel", [(8, 3, False), (8, 3, True), (10, 5, True), (10, 5, False), (7, 2, True)])
def test_widths_and_velocities(tmp_path, w, d, vel):
    raw = hand_file(45, 7, w * 10 + vel, w=w, d=d, vel=vel)
    check(tmp_path, raw)
    check(tmp_path, raw, chunk_bytes=1000)
    check(tmp_path, raw, frames=[6, 0, 3, 3])


def test_fields_outside_the_fast_paths(tmp_path):
    from moleculekit_b200 import gro

    toks = ["  1.5e-3", " -2.5E+2", "     nan", "    -nan", "     inf", "   +1.25", "   .5   ", "  -0.000", "0012.500",
            "-1.00001", "1.234567", "       7", "  -.1234", "  12.345"]
    rows = ["%5d%-5s%5s%5d%8.3f%8.3f%8.3f%8.4f%8.4f%8.4f" % (1, "A", "B", 1, 1, 2, 3, 0.1, 0.2, 0.3)]
    for a in range(1, 60):
        f = [toks[(a + k * 5) % len(toks)] for k in range(6)]
        rows.append("%5d%-5s%5s%5d%s" % (a, "A", "B", a, "".join(f)))

    def wrap(r):
        return ("t\n%5d\n" % len(r) + "\n".join(r) + "\n   1.0 2.0 3.0\n").encode()

    check(tmp_path, wrap(rows), host_lines=0)
    # an underscore, which float() takes: the host decides the line
    rows[3] = rows[3][:28] + "   1_0.5" + rows[3][36:]
    check(tmp_path, wrap(rows), host_lines=1)
    # a byte >= 0x80 in a velocity field: the host decides, and float() rejects it
    raw = wrap(rows).replace(rows[9].encode(), rows[9][:52].encode() + b"  1.5\xc3\xa9 " + rows[9][60:].encode())
    with pytest.raises(ValueError, match=r"frame 0, line 12, column 53: the vy field b'  1.5\\xc3\\xa9 ' is not a "
                                         r"number"):
        gro.read_gro_device(put(tmp_path, raw), fields=("x", "v"))


def test_boxes_and_titles(tmp_path):
    for nine in (False, True):
        for title in (lambda f: "no time here", lambda f: f"t= {f} step= x {f}", lambda f: f" t= {f}.25",
                      lambda f: f"a step= {-f} b t= nan", lambda f: f"z t= 1_0 step= 0{f}", lambda f: " t= "):
            check(tmp_path, hand_file(5, 4, 3, nine=nine, title=title))


def test_line_endings_and_truncation(tmp_path, caplog):
    check(tmp_path, hand_file(20, 3, 4, vel=True, nl="\r\n"))
    check(tmp_path, hand_file(20, 3, 5).rstrip(b"\n"))  # a last line without a newline
    check(tmp_path, hand_file(20, 3, 5) + b"\n  \n\t\n")  # trailing blank lines
    raw = hand_file(20, 4, 6)
    cut = raw[:raw.index(b"\n", raw.index(b"frame 3") + 200) + 1]
    with caplog.at_level(logging.WARNING, logger="moleculekit_b200.gro"):
        info = check(tmp_path, cut)
    assert info["n_frames"] == 3 and "is dropped" in caplog.text


def test_chunks_frame_lists_and_out_slices(tmp_path):
    from moleculekit_b200 import gro

    N, F = 30, 12
    raw = hand_file(N, F, 7, vel=True)
    for chunk in (977, 1024, 4096, 1 << 20):  # lines and frames straddle chunk edges; a frame > a chunk
        check(tmp_path, raw, chunk_bytes=chunk)
    check(tmp_path, raw, frames=[11, 0, 3, 3, 7, 0], chunk_bytes=1100)
    with pytest.raises(IndexError):
        gro.read_gro_frames(put(tmp_path, raw), [0, 12])
    _, _, time, step = gro.read_gro_frames(put(tmp_path, raw), [5, 2])
    assert time.tolist() == [2.5, 1.0] and step.tolist() == [5, 2]
    # a frame slice of larger out tensors
    idx = gro.index_gro(put(tmp_path, raw))
    s, e = int(idx["offsets"][4]), int(idx["offsets"][5])
    dev = torch.device("cuda")
    buf = torch.zeros((e - s + 31) // 16 * 16, dtype=torch.uint8, device=dev)
    buf[:e - s] = torch.frombuffer(bytearray(raw[s:e]), dtype=torch.uint8).to(dev)
    big, bigv = torch.full((N, 3, 20), -1.0, device=dev), torch.full((N, 3, 20), -1.0, device=dev)
    gro.decode_gro_device(buf[:e - s], 1, [0, 0], N, 8, True, out=big[:, :, 7:9], vout=bigv[:, :, 7:9])
    want = og.read(raw)
    assert np.array_equal(bits(big[:, :, 8].cpu().numpy()), bits(want["coords"][4]))
    assert np.array_equal(bits(bigv[:, :, 7].cpu().numpy()), bits(want["vels"][4]))
    assert (big[:, :, 9] == -1).all() and (bigv[:, :, 6] == -1).all()


def test_error_messages(tmp_path):
    from moleculekit_b200 import gro

    N = 4
    lines = hand_file(N, 3, 8, vel=True).decode().split("\n")
    P = N + 3

    def read(ls):
        return gro.read_gro(put(tmp_path, "\n".join(ls).encode()))

    for n in (N - 1, N + 1):
        bad = list(lines)
        bad[P + 1] = "%5d" % n
        with pytest.raises(ValueError, match=rf"frame 1, line {P + 2}, column 5: the atom count is {n}, frame 0 has "
                                             f"{N}"):
            read(bad)
    short = list(lines)
    short[2 * P + 3] = short[2 * P + 3][:60]
    with pytest.raises(ValueError, match=rf"frame 2, line {2 * P + 4}, column 61: the atom line has 60 columns, an "
                                         r"atom line of this file needs 68"):
        read(short)
    crlf = [ln + "\r" for ln in lines[:-1]] + [""]
    crlf[P + 2] = crlf[P + 2][:44] + "\r"
    with pytest.raises(ValueError, match=rf"frame 1, line {P + 3}, column 45: the atom line has 44 columns"):
        read(crlf)
    reject = list(lines)
    reject[P + 4] = reject[P + 4][:28] + "  1.2.3 " + reject[P + 4][36:]
    with pytest.raises(ValueError, match=rf"frame 1, line {P + 5}, column 29: the y field b'  1.2.3 ' is not a number"):
        read(reject)
    box4 = list(lines)
    box4[P + N + 2] = "1.0 2.0 3.0 4.0"
    with pytest.raises(ValueError, match=rf"frame 1, line {P + N + 3}, column 1: the box line holds 4 values, a GRO "
                                         r"box line holds 3 or 9"):
        read(box4)
    spacing = list(lines)
    spacing[2] = spacing[2][:20] + "   1.000  2.000    3.000" + spacing[2][44:]
    with pytest.raises(ValueError, match=r"frame 0, line 3, column 21: the decimal points of the first atom line are "
                                         r"not equally spaced \(inconsistent precision\)"):
        read(spacing)
    lone = "\n".join(lines).replace("\n" + lines[P], "\r" + lines[P], 1)
    with pytest.raises(ValueError, match=rf"line {P}, column {len(lines[P - 1]) + 1}: a CR that is not followed by LF"):
        gro.read_gro(put(tmp_path, lone.encode()))
    with pytest.raises(ValueError, match="has no velocities"):
        gro.read_gro_device(put(tmp_path, hand_file(3, 2, 1)), fields=("v",))


def boxes(F, seed, nine):
    rng = np.random.default_rng(seed)
    b = np.zeros((3, 3, F), np.float32)
    for i in range(3):
        b[i, i] = rng.uniform(0.5, 999.99, F)
    if nine:
        b[1, 0] = rng.uniform(-99.99, 999.9, F)
        b[2, 1] = rng.uniform(-99.99, 999.9, F)
    return b


def test_writer_matches_the_oracle(tmp_path):
    from moleculekit_b200 import gro

    for N, F, seed, nine, vel, ts in ((1, 3, 0, False, False, False), (33, 5, 1, True, True, True),
                                      (257, 40, 2, True, False, True), (100, 3, 3, False, True, False)):
        top = og.random_topology(N, seed)
        rng = np.random.default_rng(seed)
        x = rng.uniform(-999.999, 9999.999, size=(N, 3, F)).astype(np.float32)
        x[0, 0, 0] = -0.0
        x[min(1, N - 1), 1, 0] = np.float32(-0.0004)
        x[0, 2, -1] = np.float32(-999.999)
        x[N - 1, 0, -1] = np.float32(9999.999)
        x[N // 2, 1, F // 2] = np.float32(0.0005)  # a tie in the float32's exact value rounds as printf does
        v = None
        if vel:
            v = rng.uniform(-99.9999, 999.9999, size=(N, 3, F)).astype(np.float32)
            v[0, 0, 0], v[0, 1, -1], v[N - 1, 2, 0] = -0.0, np.float32(-99.9999), np.float32(999.9999)
            v[N // 2, 0, F // 2] = np.float32(-0.00004)
        b = boxes(F, seed, nine)
        b[0, 0, 0] = np.float32(999.9999)  # the ends of the box range a float32 holds
        if nine:
            b[1, 0, 0], b[2, 1, -1] = np.float32(-99.99999), -0.0
        time = rng.uniform(-5, 1e5, F) if ts else None
        step = rng.integers(0, 10 ** 9, F) if ts else None
        want = og.write(list(x.transpose(2, 0, 1)), top, list(b.transpose(2, 0, 1)), title="title", times=time,
                        steps=step, velocities=None if v is None else list(v.transpose(2, 0, 1)))
        for chunk in (1 << 20, 5000):
            assert gro.gro_bytes(x, top, b, time, step, "title", v, chunk_bytes=chunk) == want, (N, F, chunk)
        d = torch.from_numpy(x).cuda()
        dv = None if v is None else torch.from_numpy(v).cuda()
        assert bytes(gro.encode_gro_device(d, top, b, time, step, "title", dv).cpu().numpy()) == want
        fn = put(tmp_path, b"", "w.gro")
        gro.write_gro(fn, d, top, b, time, step, "title", dv)
        back, bb, tt, ss = gro.read_gro(fn)
        exp = np.float32([[[float("%8.3f" % q) for q in row] for row in fr] for fr in x.astype(np.float64)])
        assert np.array_equal(bits(back), bits(exp))
        assert np.array_equal(bits(bb), bits(np.float32(np.vectorize(lambda q: float("%10.5f" % q))(b))))
        if ts:
            assert np.array_equal(tt, np.float64(["%.5f" % t for t in time]))
            assert ss.tolist() == step.tolist()


def test_nan_leaves_no_file(tmp_path):
    from moleculekit_b200 import gro

    x = np.zeros((4, 3, 2), np.float32)
    x[2, 1, 1] = np.nan
    fn = tmp_path / "nan.gro"
    with pytest.raises(ValueError, match="frame 1, atom 2, axis y"):
        gro.write_gro(str(fn), torch.from_numpy(x).cuda(), og.random_topology(4, 0), boxes(2, 0, False))
    assert not fn.exists()


def test_more_than_65535_frame_tiles(tmp_path):
    from moleculekit_b200 import gro

    N, F = 1, 2097153  # 65 537 tiles of 32 frames
    xs = np.random.default_rng(9).uniform(-999, 9999, size=(N, 3, F)).astype(np.float32)
    b = np.zeros((3, 3, F), np.float32)
    b[0, 0], b[1, 1], b[2, 2] = 3.0, 4.0, np.arange(F, dtype=np.float32) % 900
    top = og.random_topology(N, 9)
    raw = gro.gro_bytes(xs, top, b)
    assert len(raw) == F * (7 + 45 + 31)
    assert raw[-83 * 3:] == og.write(list(xs[:, :, -3:].transpose(2, 0, 1)), top, list(b[:, :, -3:].transpose(2, 0, 1)))
    back, bb, _, _ = gro.read_gro(put(tmp_path, raw))
    want = np.float32(np.round(xs.astype(np.float64) * 1000) / 1000)
    assert back.shape[2] == F and np.array_equal(bits(back), bits(want))
    assert np.array_equal(bb, b)


def test_box_and_velocity_layouts_for_one_frame_chunks(tmp_path):
    """the encoder reads the box's (3, 3) part and the velocities through the strides it checks, for one frame too:
    a transposed one-frame CUDA box, a permuted multi-frame box written in one-frame chunks, a one-frame position slice
    beside contiguous velocities"""
    from moleculekit_b200 import gro

    N = 5
    top = og.random_topology(N, 11)
    rng = np.random.default_rng(11)
    x = torch.from_numpy(rng.uniform(-9, 99, size=(N, 3, 4)).astype(np.float32)).cuda()
    v = torch.from_numpy(rng.uniform(-9, 9, size=(N, 3, 4)).astype(np.float32)).cuda()
    m = np.float32([[4.0, 0.5, 0.25], [1.5, 5.0, -0.75], [0.125, 2.0, 6.0]])  # rows: box vectors

    def want(xs, vs, bs):
        return og.write(list(xs.cpu().numpy().transpose(2, 0, 1)), top, list(np.asarray(bs).transpose(2, 0, 1)),
                        velocities=None if vs is None else list(vs.cpu().numpy().transpose(2, 0, 1)))

    one = torch.from_numpy(m).cuda().T.contiguous().T.unsqueeze(2)  # strides (1, 3, 1)
    assert one.stride()[:2] == (1, 3)
    assert gro.gro_bytes(x[:, :, :1], top, one) == want(x[:, :, :1], None, m[:, :, None])
    many = torch.from_numpy(np.stack([m + f for f in range(4)], 2)).cuda()
    perm = many.permute(1, 0, 2).contiguous().permute(1, 0, 2)  # the same values, strides (4, 12, 1)
    assert perm.stride(0) != 3 * perm.stride(1)
    S = gro.frame_bytes(N, 1 + 6, False, True)
    for chunk in (S, 2 * S - 1, 1 << 20):  # one-frame chunks, then all frames at once
        assert gro.gro_bytes(x, top, perm, chunk_bytes=chunk) == want(x, None, many.cpu().numpy())
    big = torch.from_numpy(rng.uniform(-9, 99, size=(N, 3, 9)).astype(np.float32)).cuda()
    assert gro.gro_bytes(big[:, :, 4:5], top, one, velocities=v[:, :, :1].contiguous()) == \
        want(big[:, :, 4:5], v[:, :, :1], m[:, :, None])


def test_titles_boxes_and_count_lines_are_decided_on_the_device(tmp_path):
    """on well-formed frames mkb_gro_index and mkb_gro_head leave nothing to the host"""
    from moleculekit_b200 import _lib, gro

    N, F = 7, 40
    raw = hand_file(N, F, 12, vel=True, nine=True, title=lambda f: f"run {f} t= {f * 0.25:.5f} step= {-f * 1000}") + \
        hand_file(N, F, 13, vel=True, title=lambda f: f"plain {f}")
    want = og.read(raw)
    dev = _lib.device(None)
    buf = torch.zeros(len(raw) + 16, dtype=torch.uint8, device=dev)
    buf[:len(raw)] = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
    state = torch.tensor([0, gro.INT64_MAX, 0], dtype=torch.int64, device=dev)
    frame_off = torch.zeros(2 * F + 1, dtype=torch.int64, device=dev)
    status = torch.full((2 * F,), 7, dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_gro_index", _lib.ptr(buf), len(raw), len(raw), 0, N, _lib.ptr(state), _lib.ptr(frame_off),
              _lib.ptr(status), 2 * F)
    assert state.cpu().tolist() == [2 * F * (N + 3), gro.INT64_MAX, 0]
    assert not status.any()
    at = np.append(frame_off.cpu().numpy()[:2 * F], len(raw))
    at[0] = 0
    box, time, step, st = gro._head_device(buf, at, dev)
    assert not st.any()
    nine = box.view(-1, 9).cpu().numpy()
    for t, (i, j) in enumerate(og.ORDER):
        assert np.array_equal(bits(nine[:, t]), bits(want["box"][:, i, j]))
    assert np.array_equal(bits(time.cpu().numpy()), bits(want["time"]))
    assert step.cpu().tolist() == want["step"].tolist()


def test_bytes_0x1c_to_0x1f_are_not_whitespace(tmp_path):
    """float(), int() and bytes.split() do not take 0x1c-0x1f as whitespace, so neither does the device"""
    from moleculekit_b200 import gro

    N = 4
    lines = hand_file(N, 3, 14).decode().split("\n")
    P = N + 3

    def read(ls):
        return gro.read_gro_device(put(tmp_path, "\n".join(ls).encode()))

    field = list(lines)
    field[P + 3] = field[P + 3][:20] + " 1.5\x1c   " + field[P + 3][28:]
    with pytest.raises(ValueError, match=rf"frame 1, line {P + 4}, column 21: the x field b' 1.5\\x1c   ' is not a "
                                         r"number"):
        read(field)
    box = list(lines)
    box[P + N + 2] = "1.0\x1f2.0 3.0 4.0"
    with pytest.raises(ValueError, match=rf"frame 1, line {P + N + 3}, column 1: the box value b'1.0\\x1f2.0' is "
                                         r"not a number"):
        read(box)  # bytes.split() sees one token "1.0\x1f2.0": 3 values, the first not a number
    box[P + N + 2] = "1.0\x1f 2.0 3.0"
    with pytest.raises(ValueError, match=rf"frame 1, line {P + N + 3}, column 1: the box value b'1.0\\x1f' is not a "
                                         r"number"):
        read(box)
    count = list(lines)
    count[2 * P + 1] = "\x1c%4d" % N
    with pytest.raises(ValueError, match=rf"frame 2, line {2 * P + 2}, column 1: the atom count line"):
        read(count)
    title = list(lines)
    title[P] = "x t= 1.5\x1d step= 7\x1e"
    _, _, info = read(title)
    assert np.isnan(info["time"][1]) and info["step"][1] == -1 and info["time"][2] == 1.0


def test_first_error_in_file_order(tmp_path):
    """a bad box line and a bad atom line: the one earlier in the file is named, whichever kind it is"""
    from moleculekit_b200 import gro

    N = 4
    lines = hand_file(N, 6, 15).decode().split("\n")
    P = N + 3
    atom, box = 1 * P + 3, 4 * P + N + 2  # an atom line of frame 1, the box line of frame 4
    bad = list(lines)
    bad[atom] = bad[atom][:28] + "  1.2.3 " + bad[atom][36:]
    bad[box] = "1 2"
    with pytest.raises(ValueError, match=rf"frame 1, line {atom + 1}, column 29: the y field"):
        gro.read_gro(put(tmp_path, "\n".join(bad).encode()))
    atom, box = 4 * P + 3, 1 * P + N + 2
    bad = list(lines)
    bad[atom] = bad[atom][:28] + "  1.2.3 " + bad[atom][36:]
    bad[box] = "1 2"
    with pytest.raises(ValueError, match=rf"frame 1, line {box + 1}, column 1: the box line holds 2 values"):
        gro.read_gro(put(tmp_path, "\n".join(bad).encode()), chunk_bytes=500)


def test_steps_past_2_pow_53(tmp_path):
    from moleculekit_b200 import gro

    steps = np.int64([2 ** 53 + 1, 2 ** 62 + 3])
    x = np.zeros((2, 3, 2), np.float32)
    b = np.zeros((3, 3, 2), np.float32)
    b[0, 0] = b[1, 1] = b[2, 2] = 2.0
    top = og.random_topology(2, 16)
    raw = gro.gro_bytes(x, top, b, step=steps)
    assert raw == og.write(list(x.transpose(2, 0, 1)), top, list(b.transpose(2, 0, 1)), steps=steps.tolist())
    _, _, _, got = gro.read_gro(put(tmp_path, raw))
    assert got.tolist() == steps.tolist()
