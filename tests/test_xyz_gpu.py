"""K26 on the GPU: XYZ files indexed and parsed on the device bit for bit as the oracle reader (np.float32(float(field)),
NaN signs included), a million random tokens against float(), separators, line endings, chunking and frame lists, the
lines left to the host, every error message, the writer byte for byte Python's '%' formatting, and more than 65 535
frame tiles in one decode and one encode."""
import logging
import random

import numpy as np
import pytest
import torch

from oracle import xyz_format as of

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def want_from(raw):
    return of.read(raw)["coords"].transpose(1, 2, 0)


def put(tmp_path, raw, name="t.xyz"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def lines_file(rows, natoms, comment="c", nl="\n"):
    """rows: per atom line its text; natoms per frame -> bytes"""
    out = []
    for f in range(0, len(rows), natoms):
        out += [str(natoms), comment] + rows[f:f + natoms]
    return (nl.join(out) + nl).encode("utf-8")


def check(tmp_path, raw, host_lines=0, **kw):
    from moleculekit_b200 import xyz as px

    got, info = px.read_xyz_device(put(tmp_path, raw), **kw)
    want = want_from(raw)
    if kw.get("frames") is not None:
        want = want[:, :, np.asarray(kw["frames"])]
    assert np.array_equal(bits(got.cpu().numpy()), bits(want))
    if host_lines is not None:
        assert info["host_lines"] == host_lines
    return info


TOKENS = ["%f" % 1.2345678, "%.3f" % -3.14159, "%15.8f" % 12.5, "%22.15f" % 0.1, "%22.15f" % -123.456, repr(0.1),
          repr(-2.0 / 3), "%e" % 6.02214076e23, "%E" % -1.5e-7, "1.5E+02", "+7.25", "+.5", ".5", "5.", "-5.", "0.0",
          "-0.0", "+0.0", "1e-45", "1.4e-45", "-7e-46", "3e-39", "1.1754942e-38", "1e39", "-1e39", "3.4028236e38",
          "nan", "-nan", "NaN", "Infinity", "-inf", "+INF", "1.00000005960464477539062500001", "00012.500",
          "12345678901234567890123", "0.000000000000000000000000000001234", "1e-400", "1e400", "-0e5"]


def test_token_forms(tmp_path):
    rows = ["X %s %s %s" % (TOKENS[i % len(TOKENS)], TOKENS[(i + 7) % len(TOKENS)], TOKENS[(i + 13) % len(TOKENS)])
            for i in range(len(TOKENS) * 2)]
    check(tmp_path, lines_file(rows, len(TOKENS)))


def test_double_rounding_and_nan_signs(tmp_path):
    from moleculekit_b200 import xyz as px

    raw = b"1\n\nH 1.00000005960464477539062500001 -nan nan\n"
    got, info = px.read_xyz_device(put(tmp_path, raw))
    assert bits(got.cpu().numpy()).ravel().tolist() == [0x3f800000, 0xffc00000, 0x7fc00000]
    assert info["host_lines"] == 0


def test_a_million_random_tokens(tmp_path):
    rng = random.Random(2026)
    toks = []
    for _ in range(1_000_002):
        d = "".join(rng.choice("0123456789") for _ in range(rng.randint(1, 25)))
        if rng.random() < 0.4:
            k = rng.randint(0, len(d))
            d = d[:k] + "." + d[k:]
        toks.append(rng.choice(["", "", "-", "+"]) + d +
                    (rng.choice("eE") + str(rng.randint(-330, 310)) if rng.random() < 0.6 else ""))
    N = 1000
    rows = ["C %s %s %s" % tuple(toks[3 * i:3 * i + 3]) for i in range(len(toks) // 3)]
    F = len(rows) // N
    rows = rows[:F * N]
    raw = lines_file(rows, N)
    from moleculekit_b200 import xyz as px

    got, info = px.read_xyz_device(put(tmp_path, raw), chunk_bytes=16 << 20)
    with np.errstate(over="ignore"):
        want = np.array([float(t) for t in toks[:3 * F * N]]).astype(np.float32).reshape(F, N, 3).transpose(1, 2, 0)
    assert np.array_equal(bits(got.cpu().numpy()), bits(want))
    # only tokens of more than 19 digits whose rounding the truncated digits leave open go to the host
    assert 0 < info["host_lines"] < 2000


def test_separators_and_line_endings(tmp_path):
    rows = ["  C\t1.5 \t -2.25\x1c3.0 extra columns 7", "\x1fO\x1d.5\x1e\x1f-1e1 +2 q", "H 1 2 3\x0b\x0c",
            "\tN 4. 5.0e0 6"]
    for nl in ("\n", "\r\n"):
        check(tmp_path, lines_file(rows * 3, 4, nl=nl))
    raw = lines_file(rows * 2, 4)
    check(tmp_path, raw[:-1])  # no newline at the end
    check(tmp_path, raw + b"\n\n  \t\n \r\n")  # trailing blank lines
    check(tmp_path, raw[:-1] + b"\r\n\r\n")


def test_truncated_last_frame_is_dropped(tmp_path, caplog):
    rows = ["C %d %d %d" % (i, -i, 2 * i) for i in range(15)]
    raw = lines_file(rows, 5)
    with caplog.at_level(logging.WARNING, logger="moleculekit_b200.xyz"):
        info = check(tmp_path, raw + b"5\ncomment\nC 1 2 3\n")
    assert info["n_frames"] == 3 and "frame 3" in caplog.text


def test_chunks_and_frame_lists(tmp_path):
    from moleculekit_b200 import xyz as px

    rng = np.random.default_rng(3)
    N, F = 37, 41
    rows = ["%s %r %.3f %22.15f" % (("C", "Hg")[i % 2], float(rng.normal(0, 30)), rng.normal(0, 5), rng.normal())
            for i in range(N * F)]
    raw = lines_file(rows, N, comment="frame comment")
    fn = put(tmp_path, raw)
    whole = want_from(raw)
    idx = None
    for chunk in (100, 1000, 1500, 7777, 1 << 20):  # smaller than a frame, frames split across chunks, one chunk
        i = px.index_xyz(fn, chunk_bytes=chunk)
        if idx is None:
            idx = i
            assert i["natoms"] == N and i["n_frames"] == F and i["comment"] == "frame comment"
            assert i["element"] == ["C", "Hg"] * (N // 2) + ["C"]
            assert i["offsets"][0] == 0 and i["offsets"][-1] == len(raw) - 1 and len(i["offsets"]) == F + 1
        assert np.array_equal(i["offsets"], idx["offsets"])
    sel = [40, 3, 3, 0, 17, 40, 5, 6, 7, 3]
    for chunk in (100, 3000, 1 << 20):
        got, info = px.read_xyz_device(fn, frames=sel, chunk_bytes=chunk)
        assert np.array_equal(bits(got.cpu().numpy()), bits(whole[:, :, sel])) and info["host_lines"] == 0
        assert list(info["frames"]) == sel
        got, _ = px.read_xyz_device(fn, frames=sel, index=idx, chunk_bytes=chunk)
        assert np.array_equal(bits(got.cpu().numpy()), bits(whole[:, :, sel]))
    got, info = px.read_xyz_frames(fn, [-1, 0])
    assert np.array_equal(bits(got), bits(whole[:, :, [40, 0]]))
    with pytest.raises(IndexError):
        px.read_xyz_device(fn, frames=[41])
    assert px.read_xyz_device(fn, frames=[])[0].shape == (N, 3, 0)


def test_lines_left_to_the_host(tmp_path):
    base = ["C 1.0 2.0 3.0", "O -1.5 0.25 7"]
    for odd, n in (("C 1_000.5 2 3", 1), ("C 1.5e1_0 2 3", 1), ("\u00d6 1 2 3", 1), ("C 1 2 3 ", 0),
                   ("C 1 2 3 4 x", 0), ("C 9007199254740993.00000000001 2 3", 1), ("C \u0661 2 3", 1),
                   ("C\u00a01 2 3", 1), ("C 1 2 3 \u00e9", 0)):
        rows = base * 2 + [odd] + base
        raw = lines_file(rows, 7)
        check(tmp_path, raw, host_lines=n)
        check(tmp_path, raw, host_lines=2 * n, frames=[0, 0])


def test_error_messages(tmp_path):
    from moleculekit_b200 import xyz as px

    ok = b"2\nc\nC 1 2 3\nC 1 2 3\n2\nc\nC 1 2 3\nC 1 2 3\n"
    assert ok[20:22] == b"2\n"
    cases = [
        (ok[:20] + b" 3" + ok[21:], r"frame 1, line 5, column 2: the atom count is 3, frame 0 has 2 \(the atom count "
                                    r"must not change between frames\)"),
        (ok[:20] + b"two" + ok[21:], r"frame 1, line 5, column 1: the atom count line 'two' does not start with an "
                                     r"integer"),
        (lines_file(["C 1 2 3", "C 1 2 3", "C 1 2 3", "C 1 2"], 2),
         r"frame 1, line 8, column 6: the atom line has 3 field\(s\), an atom line needs four \(element x y z\)"),
        (lines_file(["C 1 2 3", "C 1 2 3", "C 1 x2 3", "C 1 2"], 2), r"frame 1, line 7, column 5: the y field 'x2' is "
                                                                     r"not a number"),
        (lines_file(["C 1 2 3", "C 1 2 3", "C 1 2 3 1.2.3", "C 1 2 1e"], 2), r"frame 1, line 8, column 7: the z field "
                                                                             r"'1e' is not a number"),
        (ok.replace(b"C 1 2 3\n", b"C 1 2 3\rC", 1), r"frame 0, line 3, column 8: a CR that is not followed by LF ends "
                                                     r"a line; lone CR line endings are not supported"),
    ]
    for raw, match in cases:
        fn = put(tmp_path, raw)
        with pytest.raises(ValueError, match=match) as e:
            px.read_xyz_device(fn)
        assert str(e.value).startswith(f"XYZ file {fn}, ")


def test_writer_matches_python_formatting(tmp_path):
    from moleculekit_b200 import xyz as px

    rng = np.random.default_rng(7)
    N, F = 45, 70
    x = rng.normal(0, 200, size=(N, 3, F)).astype(np.float32)
    x[0, :, 0] = [999999.9375, -99999.9921875, -0.0]
    x[1, :, 0] = [0.000000005, -0.000000005, 0.000000015]  # float32 neighbours of ties
    x[2, :, 0] = [1e-30, -1e-30, 5e-9]
    el = [("C", "Hg", "N", "Xyzzy")[i % 4] for i in range(N)]
    want = of.write(list(x.transpose(2, 0, 1)), el, comment="written on the GPU")
    for chunk in (1, 5000, 1 << 20):
        assert px.xyz_bytes(x, el, comment="written on the GPU", chunk_bytes=chunk) == want
    xd = torch.from_numpy(x).cuda()
    big = torch.zeros((N, 3, F + 9), device="cuda")
    big[:, :, 4:4 + F] = xd
    assert px.xyz_bytes(big[:, :, 4:4 + F], el, comment="written on the GPU") == want
    assert bytes(px.encode_xyz_device(xd, el, "written on the GPU").cpu().numpy()) == want
    fn = str(tmp_path / "w.xyz")
    px.write_xyz(fn, xd, el, comment="written on the GPU", chunk_bytes=7000)
    assert open(fn, "rb").read() == want
    back, info = px.read_xyz_device(fn)
    rounded = (np.rint(x.astype(np.float64) * 1e8) / 1e8).astype(np.float32)
    assert np.array_equal(bits(back.cpu().numpy()), bits(rounded)) and info["host_lines"] == 0
    assert info["element"] == el and info["comment"] == "written on the GPU"


def test_more_than_65535_frame_tiles(tmp_path):
    from moleculekit_b200 import xyz as px

    F = 65535 * 32 + 37
    x = torch.arange(F, dtype=torch.float32, device="cuda").mul_(0.37).remainder_(997.0).sub_(400.0).view(1, 1, F)
    x = torch.cat([x, -x * 0.5, x + 0.125], 1)
    fn = str(tmp_path / "long.xyz")
    px.write_xyz(fn, x, ["H"], chunk_bytes=1 << 30)  # one encode call
    back, info = px.read_xyz_device(fn, chunk_bytes=1 << 30)  # one index and one decode call
    assert info["n_frames"] == F and info["host_lines"] == 0
    want = (torch.round(x.double() * 1e8) / 1e8).float()
    bad = torch.nonzero(back.view(torch.int32) != want.view(torch.int32))
    assert len(bad) == 0, bad[:5].tolist()
    with open(fn, "rb") as fh:
        head = fh.read(3 * 53)
    assert head == of.write(list(x[:, :, :3].cpu().numpy().transpose(2, 0, 1)), ["H"])
