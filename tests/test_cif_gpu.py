"""K30 on the GPU: mmCIF files indexed and parsed on the device bit for bit as the oracle reader (np.float32(float(token))
of the Cartn tokens), column orders, comment lines and CRLF, chunk edges and frame lists, tokens outside the fast path,
the rows left to the host, every error message, the writer byte for byte Python's '%' formatting, ids and model numbers
past PDB's columns, more than 65 535 models in one decode and one encode, and one trajectory through PDB and mmCIF."""
import logging

import numpy as np
import pytest
import torch

from oracle import cif_format as of

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def put(tmp_path, raw, name="t.cif"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def check(tmp_path, raw, host_lines=0, frames=None, **kw):
    from moleculekit_b200 import cif as pc

    got, info = pc.read_cif_device(put(tmp_path, raw), frames=frames, **kw)
    want = of.read(raw)
    sel = slice(None) if frames is None else np.asarray(frames)
    assert np.array_equal(bits(got.cpu().numpy()), bits(want["coords"].transpose(1, 2, 0)[:, :, sel]))
    n = got.shape[2]
    assert np.array_equal(bits(info["box"]), bits(np.repeat(want["box"][:, None], n, 1)))
    assert np.array_equal(bits(info["boxangles"]), bits(np.repeat(want["boxangles"][:, None], n, 1)))
    assert np.array_equal(info["model"], want["model"][sel])
    for k, v in want["topology"].items():
        assert list(info["topology"][k]) == list(np.asarray(v, dtype=info["topology"][k].dtype)), k
    if host_lines is not None:
        assert info["host_lines"] == host_lines
    return info


def model_first(tags):
    return ["pdbx_PDB_model_num"] + [t for t in tags if t != "pdbx_PDB_model_num"]


REST = [t for t in of.TAGS if not t.startswith("Cartn")]
ORDERS = dict(rcsb=of.TAGS,
              coords_first=["Cartn_x", "Cartn_y", "Cartn_z"] + REST,
              coords_last_z_first=model_first(REST) + ["Cartn_z", "Cartn_x", "Cartn_y"],
              no_model=[t for t in of.TAGS if t != "pdbx_PDB_model_num"],
              label_only=["id", "label_atom_id", "label_comp_id", "Cartn_x", "label_asym_id", "Cartn_y",
                          "label_seq_id", "Cartn_z", "pdbx_PDB_model_num", "type_symbol"])


@pytest.mark.parametrize("order", list(ORDERS))
def test_column_orders(tmp_path, order):
    top = of.random_topology(37, 2)
    raw = of.rcsb(frames(37, 6, 1), top, tags=ORDERS[order], box=[40, 41.5, 42.25, 90, 80, 70], model_base=3)
    info = check(tmp_path, raw)
    F = 1 if order == "no_model" else 6
    assert info["n_frames"] == F and info["natoms"] == 37 * 6 // F


def test_comments_crlf_chunks_and_frame_lists(tmp_path):
    from moleculekit_b200 import cif as pc

    N, F = 50, 12
    top = of.random_topology(N, 5)
    raw = of.rcsb(frames(N, F, 6), top, box=[30, 31, 32, 90, 90, 90], nl="\r\n")
    for chunk in (977, 4096, 8192, 1 << 20):  # rows, marks and frames straddle chunk edges; a frame > a chunk
        check(tmp_path, raw, chunk_bytes=chunk)
    # comment and blank lines between frames and inside them; models not in order, repeated model numbers
    lines = of.rcsb(frames(N, F, 7), top).split(b"\n")
    body = [i for i, ln in enumerate(lines) if ln.startswith((b"ATOM", b"HETATM"))]
    for i in reversed(body[::17]):
        lines[i:i] = [b"# between rows", b"", b"  \t", b"#"]
    raw = b"\n".join(lines)
    raw = raw.replace(b" 2 \n", b" 9 \n").replace(b" 4 \n", b" 1 \n")  # models 1, 9, 3, 1, 5, ...
    info = check(tmp_path, raw, chunk_bytes=5000)
    assert info["model"][:5].tolist() == [1, 9, 3, 1, 5]
    check(tmp_path, raw, frames=[11, 0, 3, 3, 7, 0], chunk_bytes=9000)
    with pytest.raises(IndexError):
        pc.read_cif_frames(put(tmp_path, raw), [0, 12])
    got, info = pc.read_cif_frames(put(tmp_path, raw), [5, 2])
    assert info["frames"].tolist() == [5, 2] and info["model"].tolist() == [6, 3]
    # a frame slice of a larger out tensor
    fn = put(tmp_path, raw)
    idx = pc.index_cif(fn)
    dev = torch.device("cuda")
    big = torch.full((N, 3, 20), -1.0, device=dev)
    s, e = int(idx["start"][4]), int(idx["end"][4])
    buf = torch.zeros((e - s + 31) // 16 * 16, dtype=torch.uint8, device=dev)
    buf[:e - s] = torch.frombuffer(bytearray(raw[s:e]), dtype=torch.uint8).to(dev)
    pc.decode_cif_device(buf[:e - s], 1, [0, 0], N, pc._cartn(idx["tags"]), out=big[:, :, 7:9])
    want = of.read(raw)["coords"][4]
    assert np.array_equal(bits(big[:, :, 7].cpu().numpy()), bits(want)) and (big[:, :, 9] == -1).all()


def table(rows, tags=("id", "Cartn_x", "Cartn_y", "Cartn_z", "pdbx_PDB_model_num"), tail=b"#\n"):
    head = b"data_t\nloop_\n" + b"".join(b"_atom_site.%s\n" % t.encode() for t in tags)
    return head + b"".join(r.encode("latin-1") + b"\n" for r in rows) + tail


def test_tokens_outside_the_fast_path(tmp_path):
    toks = ["12.345", "-1.23456", "3.25", "1.5e-3", "-2.5E+2", "nan", "-nan", "inf", "-Infinity", ".5", "5.", "-0.000",
            "+123.456", "0012.500", "7", "+0", "1e38", "-3.4e-45", "0.1234567890123456789012345",
            "12345678901234567890123.5", "-99999999999999999999.99"]
    rows = ["%d %s %s %s 1" % (a, *(toks[(a + 7 * d) % len(toks)] for d in range(3))) for a in range(60)]
    check(tmp_path, table(rows), host_lines=None)
    check(tmp_path, table(rows[:14]), host_lines=0)


def test_host_lines(tmp_path):
    rows = ["%d C%d %.3f %.3f %.3f 1" % (a, a, a * 1.5, -a, 0.25) for a in range(40)]
    tags = ("id", "label_atom_id", "Cartn_x", "Cartn_y", "Cartn_z", "pdbx_PDB_model_num")
    rows[3] = "3 C3 '1.5' 2 3 1"
    rows[5] = "5 C5 4 \"-2.25\" 3 1"
    rows[8] = "8 C8 1.5(2) 2 -3.25(13) 1"
    rows[11] = "11 C\xe9 1 2 3 1"
    rows[12] = "12 'C\xe9 x' 1 2 3 1"
    info = check(tmp_path, table(rows, tags), host_lines=5)
    assert info["topology"]["name"][11] == "C\xe9"
    # a byte >= 0x80 after the coordinates is the device's
    rows = ["%d %.3f %.3f %.3f 1 C\xe9" % (a, a, -a, 0.5) for a in range(40)]
    check(tmp_path, table(rows, ("id", "Cartn_x", "Cartn_y", "Cartn_z", "pdbx_PDB_model_num", "type_symbol")),
          host_lines=0)


def test_errors(tmp_path):
    from moleculekit_b200 import cif as pc

    N = 10
    rows = ["%d %.3f %.3f %.3f %d" % (f * N + a, a, -a, 0.5, f + 1) for f in range(3) for a in range(N)]
    first = 8  # the 1-based line of rows[0] in table()

    def fails(r, match, **kw):
        with pytest.raises(ValueError, match=match):
            pc.read_cif(put(tmp_path, table(r, **kw)))

    fewer = rows[:2 * N + 3] + rows[2 * N + 4:]  # frame 2 loses a row; another category follows, so it is no truncation
    fails(fewer, rf"frame 2 \(model 3, line {first + 2 * N}\): 9 rows, frame 0 has 10", tail=b"#\nloop_\n_other.x\n1\n")
    more = rows[:N + 2] + [rows[N + 2]] + rows[N + 2:]
    fails(more, rf"frame 1 \(model 2, line {first + N}\): 11 rows")
    toks = list(rows)
    toks[4] = "4 1.0 2.0 3.0"
    fails(toks, rf"line {first + 4}: the _atom_site row holds 4 tokens, the loop has 5 tags; rows must be one line each")
    span = list(rows)
    span[6:7] = ["6 1.0 2.0", "3.0 1"]  # a row that spans lines
    fails(span, rf"line {first + 6}: the _atom_site row holds 3 tokens")
    text = list(rows)
    text[5:6] = ["5 1.0 2.0 3.0", ";a text field", ";"]
    fails(text, rf"line {first + 5}: the _atom_site row holds 4 tokens")
    text = rows[:5] + [";a text field", ";"] + rows[5:]
    fails(text, rf"line {first + 5}: the _atom_site row holds 0 tokens and starts a ';' text field")
    quote = list(rows)
    quote[2] = "2 '1.0 2.0 3.0 1"
    fails(quote, rf"line {first + 2}: the _atom_site row holds 1 tokens and a quoted token that does not close")
    lone = list(rows)
    lone[8] = lone[8] + "\r\r"
    fails(lone, rf"line {first + 8}, column \d+: a CR that is not followed by LF")
    null = list(rows)
    null[13] = "13 1.0 ? 3.0 2"
    fails(null, rf"frame 1, line {first + 13}, column 3: the Cartn_y token b'\?' is a null value")
    nan = list(rows)
    nan[1] = "1 1.2.3 2 3 1"
    fails(nan, rf"frame 0, line {first + 1}, column 2: the Cartn_x token b'1.2.3' is not a number")
    model = list(rows)
    model[17] = "17 1 2 3 2.0"
    fails(model, rf"line {first + 17}: the pdbx_PDB_model_num token b'2.0' is not an integer")
    model[17] = "17 1 2 3 '2'"
    fails(model, rf"line {first + 17}: the pdbx_PDB_model_num token b'2' is not an integer")


def test_truncated_last_model_is_dropped(tmp_path, caplog):
    from moleculekit_b200 import cif as pc

    raw = pc.cif_bytes(np.stack(frames(20, 5, 11), axis=2), of.random_topology(20, 11))
    at = raw.index(b" 5\n")  # the first row of the last model
    for _ in range(3):
        at = raw.index(b"\n", at + 1)
    cut = raw[:at + 1]  # the last model stops after a whole row
    with caplog.at_level(logging.WARNING, logger="moleculekit_b200.cif"):
        info = check(tmp_path, cut)
    assert info["n_frames"] == 4 and "is dropped" in caplog.text


def test_writer_matches_the_oracle(tmp_path):
    from moleculekit_b200 import cif as pc

    for N, F, seed, with_box in ((1, 3, 0, False), (33, 5, 1, True), (257, 40, 2, True), (1000, 3, 3, False)):
        top = of.random_topology(N, seed)
        x = np.random.default_rng(seed).uniform(-99999.99, 999999.9, size=(N, 3, F)).astype(np.float32)
        x[0, 0, 0] = -0.0
        x[min(1, N - 1), 1, 0] = np.float32(-0.0004)
        x[0, 2, -1] = np.float32(-99999.99)
        x[N - 1, 0, -1] = np.float32(999999.9)
        x[N // 2, 1, F // 2] = np.float32(0.0005)  # a tie in the float32's exact value rounds as printf does
        box = ang = None
        if with_box:
            box = np.repeat(np.float32([[12.5], [1e5], [0.001]]), F, 1)
            ang = np.repeat(np.float32([[90], [-0.0], [109.471]]), F, 1)
        want = of.write(list(x.transpose(2, 0, 1)), top, None if box is None else box[:, 0],
                        None if ang is None else ang[:, 0], title="t%d" % N)
        for chunk in (1 << 20, 5000):
            assert pc.cif_bytes(x, top, box, ang, title="t%d" % N, chunk_bytes=chunk) == want, (N, F, chunk)
        d = torch.from_numpy(x).cuda()
        head = pc._header("t%d" % N, None if box is None else box[:, 0], None if ang is None else ang[:, 0])
        assert bytes(pc.encode_cif_device(d, top).cpu().numpy()) == want[len(head):-2]
        fn = put(tmp_path, b"", "w.cif")
        pc.write_cif(fn, d, top, box, ang, title="t%d" % N)
        back, info = pc.read_cif(fn)
        exp = np.float32([[[float("%.3f" % v) for v in row] for row in fr] for fr in x.astype(np.float64)])
        assert np.array_equal(bits(back), bits(exp))
        if with_box:
            assert np.array_equal(bits(info["box"]), bits(np.float32([[float("%.3f" % v)] * F for v in box[:, 0]])))


def test_ids_and_models_past_pdb_columns(tmp_path):
    from moleculekit_b200 import cif as pc

    N, F = 12, 10001  # ids past 99 999, models past 9 999
    x = np.random.default_rng(3).uniform(-50, 50, size=(N, 3, F)).astype(np.float32)
    top = of.random_topology(N, 4)
    raw = pc.cif_bytes(x, top)
    assert raw == of.write(list(x.transpose(2, 0, 1)), top)
    back, info = pc.read_cif(put(tmp_path, raw))
    assert info["n_frames"] == F and info["model"][-1] == F and info["model"][:3].tolist() == [1, 2, 3]
    assert np.array_equal(bits(back), bits(np.float32(np.round(x.astype(np.float64) * 1000) / 1000)))
    assert raw[-len(b"10001\n#\n"):] == b"10001\n#\n" and b" 120012 " in raw


def test_many_models_of_a_few_atoms(tmp_path):
    from moleculekit_b200 import cif as pc

    N, F = 3, 70000  # more than 65 535 frames of one atom tile
    xs = np.random.default_rng(7).uniform(-99999, 999999, size=(N, 3, F)).astype(np.float32)
    top = of.random_topology(N, 8)
    raw = pc.cif_bytes(xs, top)
    back, info = pc.read_cif(put(tmp_path, raw))
    want = np.float32(np.round(xs.astype(np.float64) * 1000) / 1000)
    assert info["n_frames"] == F and np.array_equal(bits(back), bits(want))
    last = raw.split(b"\n")[-3].split()  # the last row: id, coordinates and model number of the last frame
    assert last[1] == b"%d" % (N * F) and last[-1] == b"%d" % F
    assert [b"%.3f" % v for v in xs[-1, :, -1].astype(np.float64)] == last[10:13]


def test_one_trajectory_through_pdb_and_cif(tmp_path):
    from moleculekit_b200 import cif as pc
    from moleculekit_b200 import pdb as pp
    from oracle import pdb_format

    N, F = 64, 7
    top = pdb_format.random_topology(N, 30)
    top["serial"] = list(range(1, N + 1))
    x = np.random.default_rng(30).uniform(-999, 9999, size=(N, 3, F)).astype(np.float32)
    box = np.repeat(np.float32([[50.5], [60.25], [70.125]]), F, 1)
    ang = np.repeat(np.float32([[90], [100.5], [110.25]]), F, 1)
    pp.write_pdb(put(tmp_path, b"", "x.pdb"), x, top, box, ang)
    pc.write_cif(put(tmp_path, b"", "x.cif"), x, top, box, ang)
    a, ia = pp.read_pdb(str(tmp_path / "x.pdb"))
    b, ib = pc.read_cif(str(tmp_path / "x.cif"))
    assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(bits(ia["box"]), bits(ib["box"])) and np.array_equal(bits(ia["boxangles"]),
                                                                                bits(ib["boxangles"]))
    for k in pp.FIELDS:
        assert np.array_equal(np.asarray(ia["topology"][k]), np.asarray(ib["topology"][k])), k


def test_nan_leaves_no_file(tmp_path):
    from moleculekit_b200 import cif as pc

    x = np.zeros((4, 3, 2), np.float32)
    x[2, 1, 1] = np.nan
    fn = tmp_path / "nan.cif"
    with pytest.raises(ValueError, match="frame 1, atom 2, axis y"):
        pc.write_cif(str(fn), torch.from_numpy(x).cuda(), of.random_topology(4, 0))
    assert not fn.exists()
