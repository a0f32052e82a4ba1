"""K28 on the GPU: PDB files indexed and parsed on the device bit for bit as the oracle reader (np.float32(float(field))
of columns 31-54, NaN signs included), records between atoms, MODEL-less files, CRYST1 placement, line endings,
chunking and frame lists, the lines left to the host, every error message, the writer byte for byte Python's '%'
formatting, and more than 65 535 frames in one decode and one encode."""
import logging

import numpy as np
import pytest
import torch

from oracle import pdb_format as of

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def put(tmp_path, raw, name="t.pdb"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def check(tmp_path, raw, host_lines=0, frames=None, **kw):
    from moleculekit_b200 import pdb as pp

    got, info = pp.read_pdb_device(put(tmp_path, raw), frames=frames, **kw)
    want = of.read(raw)
    sel = slice(None) if frames is None else np.asarray(frames)
    assert np.array_equal(bits(got.cpu().numpy()), bits(want["coords"].transpose(1, 2, 0)[:, :, sel]))
    assert np.array_equal(bits(info["box"]), bits(want["box"].T[:, sel]))
    assert np.array_equal(bits(info["boxangles"]), bits(want["boxangles"].T[:, sel]))
    if host_lines is not None:
        assert info["host_lines"] == host_lines
    return info


def hand_file(N, F, seed, cryst="header", extra=True, model=True, nl="\n", fmt="%8.3f"):
    """a file written line by line: REMARK / TER / ANISOU / HETATM records between atoms, CRYST1 in the header or per
    model"""
    rng = np.random.default_rng(seed)
    xs = rng.normal(0, 40, size=(F, N, 3))
    out = ["REMARK   1 generated", "HEADER    TEST"]
    if cryst == "header":
        out.append("CRYST1   50.000   60.000   70.000  90.00 100.00 110.00 P 1           1")
    for f in range(F):
        if model:
            out.append("MODEL     %4d" % (f + 1))
        if cryst == "model":
            out.append("CRYST1%9.3f%9.3f%9.3f%7.2f%7.2f%7.2f P 1           1" % (40 + f, 41.5, 42.25, 90, 90 - f % 7, 60))
        for a in range(N):
            rec = "HETATM" if a % 5 == 4 else "ATOM  "
            coords = "".join(fmt % v for v in xs[f, a])
            out.append("%s%5d  CA  ALA A%4d    %s  1.00 %5.2f           C" % (rec, a + 1, a, coords, a % 50))
            if extra and a % 7 == 3:
                out.append("ANISOU%5d  CA  ALA A%4d     1234   5678   9012   3456   7890   1234       C" % (a + 1, a))
            if extra and a % 11 == 10:
                out.append("TER   %5d      ALA A%4d" % (a + 2, a))
                out.append("REMARK 350 between atoms")
        if model:
            out.append("ENDMDL")
    out.append("CONECT    1    2")
    out.append("MASTER        0    0    0    0    0    0    0    0    5    0    5    0")
    out.append("END")
    return (nl.join(out) + nl).encode()


@pytest.mark.parametrize("cryst", ["header", "model", None])
def test_models_with_records_between_atoms(tmp_path, cryst):
    info = check(tmp_path, hand_file(37, 9, 1, cryst=cryst))
    assert info["natoms"] == 37 and info["n_frames"] == 9
    t = info["topology"]
    assert list(t["record"][:5]) == ["ATOM"] * 4 + ["HETATM"] and list(t["serial"][:3]) == [1, 2, 3]
    assert list(t["name"][:2]) == ["CA", "CA"] and t["resname"][0] == "ALA" and t["chain"][0] == "A"
    assert list(t["resid"][:3]) == [0, 1, 2] and t["element"][0] == "C" and float(t["beta"][3]) == 3.0


def test_no_model_records_crlf_and_trimmed_lines(tmp_path):
    check(tmp_path, hand_file(40, 1, 2, model=False))
    check(tmp_path, hand_file(40, 5, 3, nl="\r\n"))
    check(tmp_path, hand_file(40, 1, 4, model=False, cryst="header", nl="\r\n"))
    # atom lines trimmed to 54 columns, and a last line without a newline
    rows = ["ATOM  %5d  C   X   X   1    %8.3f%8.3f%8.3f" % (a, a * 1.5, -a, 0.25) for a in range(20)]
    check(tmp_path, "\n".join(rows).encode())
    check(tmp_path, ("MODEL 1\n" + "\n".join(rows) + "\nENDMDL\nMODEL 2\n" + "\n".join(rows)).encode())


def test_fields_outside_f83(tmp_path):
    toks = ["%8.2f" % 12.345, "%8.4f" % -1.23456, "%8.1f" % 3.25, "  1.5e-3", " -2.5E+2", "     nan", "    -nan",
            "     inf", "-1.00001", "   .5   ", "  -0.000", "+123.456", "0012.500", "1.234567", "       7"]
    rows = []
    for a in range(60):
        f = [toks[(a + d * 5) % len(toks)] for d in range(3)]
        rows.append("ATOM  %5d  C   X   X   1    %s%s%s  1.00  0.00" % (a, *f))
    raw = ("MODEL 1\n" + "\n".join(rows) + "\nENDMDL\n").encode()
    check(tmp_path, raw, host_lines=0)
    # an underscore, which float() takes: the host decides the line
    rows[3] = rows[3][:30] + "   1_0.5" + rows[3][38:]
    raw = ("MODEL 1\n" + "\n".join(rows) + "\nENDMDL\n").encode()
    check(tmp_path, raw, host_lines=1)
    # a byte >= 0x80 in a field: the host decides, and float() rejects it
    raw = raw.replace(rows[9].encode(), rows[9][:30].encode() + b"  1.5\xc3\xa9 " + rows[9][38:].encode())
    from moleculekit_b200 import pdb as pp

    with pytest.raises(ValueError, match=r"frame 0, line 11, column 31: the x field b'  1.5\\xc3\\xa9 '"):
        pp.read_pdb(put(tmp_path, raw))


def test_chunks_frame_lists_and_out_slices(tmp_path):
    from moleculekit_b200 import pdb as pp

    N, F = 50, 12
    top = of.random_topology(N, 5)
    xs = frames(N, F, 6)
    boxes = [np.float32([30 + f, 31, 32]) for f in range(F)]
    raw = of.write(xs, top, boxes, [np.float32([90, 80, 70])] * F)
    for chunk in (977, 4096, 8192, 1 << 20):  # lines, records and frames straddle chunk edges; a frame > a chunk
        check(tmp_path, raw, chunk_bytes=chunk)
    check(tmp_path, raw, frames=[11, 0, 3, 3, 7, 0], chunk_bytes=9000)
    with pytest.raises(IndexError):
        pp.read_pdb_frames(put(tmp_path, raw), [0, 12])
    got, info = pp.read_pdb_frames(put(tmp_path, raw), [5, 2])
    assert info["frames"].tolist() == [5, 2]
    for k in ("name", "resname", "segid", "element", "chain"):
        assert list(info["topology"][k]) == top[k], k
    assert list(info["topology"]["serial"]) == [s % 100000 for s in top["serial"]]
    # a frame slice of a larger out tensor
    idx = pp.index_pdb(put(tmp_path, raw))
    dev = torch.device("cuda")
    big = torch.full((N, 3, 20), -1.0, device=dev)
    fn = put(tmp_path, raw)
    with open(fn, "rb") as fh:
        span = fh.read()
    s, e = int(idx["start"][4]), int(idx["end"][4])
    buf = torch.zeros((e - s + 31) // 16 * 16, dtype=torch.uint8, device=dev)
    buf[:e - s] = torch.frombuffer(bytearray(span[s:e]), dtype=torch.uint8).to(dev)
    pp.decode_pdb_device(buf[:e - s], 1, [0, 0], N, out=big[:, :, 7:9])
    want = of.read(raw)["coords"][4]
    assert np.array_equal(bits(big[:, :, 7].cpu().numpy()), bits(want)) and (big[:, :, 9] == -1).all()


def test_many_frames_of_a_few_atoms(tmp_path):
    N, F = 3, 70000  # more than 65 535 frames of one atom tile
    xs = np.random.default_rng(7).uniform(-999, 9999, size=(N, 3, F)).astype(np.float32)
    from moleculekit_b200 import pdb as pp

    top = of.random_topology(N, 8)
    raw = pp.pdb_bytes(xs, top)
    back, info = pp.read_pdb(put(tmp_path, raw))
    want = np.float32(np.round(xs.astype(np.float64) * 1000) / 1000)
    assert info["n_frames"] == F and np.array_equal(bits(back), bits(want))
    assert raw[-30:] == of.write([xs[:, :, -1]], top)[-30:]


def test_model_count_errors(tmp_path):
    from moleculekit_b200 import pdb as pp

    raw = hand_file(12, 4, 9, extra=False)
    lines = raw.decode().split("\n")
    models = [i for i, ln in enumerate(lines) if ln.startswith("MODEL")]
    fewer = lines[:models[2] + 3] + lines[models[2] + 4:]  # frame 2 loses an atom line
    with pytest.raises(ValueError, match=rf"frame 2 \(MODEL 3, line {models[2] + 1}\): 11 atom records, frame 0 has 12"):
        pp.read_pdb(put(tmp_path, "\n".join(fewer).encode()))
    more = lines[:models[1] + 3] + [lines[models[1] + 3]] + lines[models[1] + 3:]
    with pytest.raises(ValueError, match=rf"frame 1 \(MODEL 2, line {models[1] + 1}\): 13 atom records"):
        pp.read_pdb(put(tmp_path, "\n".join(more).encode()))


def test_line_errors(tmp_path):
    from moleculekit_b200 import pdb as pp

    rows = ["ATOM  %5d  C   X   X   1    %8.3f%8.3f%8.3f  1.00  0.00" % (a, a, -a, 0.5) for a in range(10)]

    def model_file(r):
        return ("REMARK x\nMODEL 1\n" + "\n".join(r) + "\nENDMDL\nMODEL 2\n" + "\n".join(rows) + "\nENDMDL\n").encode()

    short = list(rows)
    short[4] = short[4][:50]
    with pytest.raises(ValueError, match=r"frame 0, line 7, column 51: the atom line has 50 columns"):
        pp.read_pdb(put(tmp_path, model_file(short)))
    crlf_short = list(rows)
    crlf_short[2] = crlf_short[2][:53] + "\r"
    with pytest.raises(ValueError, match=r"frame 0, line 5, column 54: the atom line has 53 columns"):
        pp.read_pdb(put(tmp_path, model_file(crlf_short)))
    bad = list(rows)
    bad[6] = bad[6][:38] + "  1.2.3 " + bad[6][46:]
    with pytest.raises(ValueError, match=r"frame 0, line 9, column 39: the y field b'  1.2.3 ' is not a number"):
        pp.read_pdb(put(tmp_path, model_file(bad)))
    blank = list(rows)
    blank[0] = blank[0][:46] + " " * 8 + blank[0][54:]
    with pytest.raises(ValueError, match=r"frame 0, line 3, column 47: the z field"):
        pp.read_pdb(put(tmp_path, model_file(blank)))
    lone = model_file(rows).replace(b"ENDMDL\nMODEL 2", b"ENDMDL\rMODEL 2")
    with pytest.raises(ValueError, match=r"line 13, column 7: a CR that is not followed by LF"):
        pp.read_pdb(put(tmp_path, lone))


def test_truncated_last_model_is_dropped(tmp_path, caplog):
    from moleculekit_b200 import pdb as pp

    raw = hand_file(20, 5, 11, extra=False)
    cut = raw[:raw.index(b"\n", raw.rindex(b"MODEL") + 300) + 1]  # the last model stops after a whole line
    with caplog.at_level(logging.WARNING, logger="moleculekit_b200.pdb"):
        info = check(tmp_path, cut)
    assert info["n_frames"] == 4 and "is dropped" in caplog.text


def test_writer_matches_the_oracle(tmp_path):
    from moleculekit_b200 import pdb as pp

    for N, F, seed, with_box in ((1, 3, 0, False), (33, 5, 1, True), (257, 40, 2, True), (1000, 3, 3, False)):
        top = of.random_topology(N, seed)
        x = np.random.default_rng(seed).uniform(-999.999, 9999.999, size=(N, 3, F)).astype(np.float32)
        x[0, 0, 0] = -0.0
        x[min(1, N - 1), 1, 0] = np.float32(-0.0004)
        x[0, 2, -1] = np.float32(-999.999)
        x[N - 1, 0, -1] = np.float32(9999.999)
        x[N // 2, 1, F // 2] = np.float32(0.0005)  # a tie in the float32's exact value rounds as printf does
        box = ang = None
        if with_box:
            box = np.random.default_rng(seed).uniform(-9999.999, 99999.99, size=(3, F)).astype(np.float32)
            ang = np.random.default_rng(seed + 1).uniform(-999.99, 9999.99, size=(3, F)).astype(np.float32)
            box[0, 0], ang[1, 0] = -0.0, -0.0
        want = of.write(list(x.transpose(2, 0, 1)), top, None if box is None else list(box.T),
                        None if ang is None else list(ang.T))
        for chunk in (1 << 20, 5000):
            assert pp.pdb_bytes(x, top, box, ang, chunk_bytes=chunk) == want, (N, F, chunk)
        d = torch.from_numpy(x).cuda()
        assert bytes(pp.encode_pdb_device(d, top, box, ang).cpu().numpy()) == want[:-4]
        fn = put(tmp_path, b"", "w.pdb")
        pp.write_pdb(fn, d, top, box, ang)
        back, info = pp.read_pdb(fn)
        exp = np.float32([[[float("%8.3f" % v) for v in row] for row in fr] for fr in x.astype(np.float64)])
        assert np.array_equal(bits(back), bits(exp))
        if with_box:
            assert np.array_equal(bits(info["box"]), bits(np.float32(np.vectorize(lambda v: float("%9.3f" % v))(box))))


def test_nan_leaves_no_file(tmp_path):
    from moleculekit_b200 import pdb as pp

    x = np.zeros((4, 3, 2), np.float32)
    x[2, 1, 1] = np.nan
    fn = tmp_path / "nan.pdb"
    with pytest.raises(ValueError, match="frame 1, atom 2, axis y"):
        pp.write_pdb(str(fn), torch.from_numpy(x).cuda(), of.random_topology(4, 0))
    assert not fn.exists()
