"""The host side of multi-model PDB reading and writing (moleculekit_b200/pdb.py; K28 indexes, parses and formats on
the device): the independent oracle's round trip, the host template builder against the oracle writer's PDB 3.3
columns, the writer's checks that run before the file is opened, the reader's checks that run before the device, and
the C-ABI symbols."""
import os

import numpy as np
import pytest

from oracle import pdb_format as of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def test_oracle_round_trip():
    for N, box in ((1, False), (3, True), (17, True)):
        top = of.random_topology(N, N)
        xs = frames(N, 4, N)
        boxes = [np.float32([10 + f, 20.5, 99999.99]) for f in range(4)] if box else None
        angles = [np.float32([90, 60 + f, 120.25]) for f in range(4)] if box else None
        raw = of.write(xs, top, boxes, angles)
        got = of.read(raw)
        assert got["natoms"] == N
        want = np.float32([[[float("%8.3f" % v) for v in row] for row in x] for x in xs])
        assert np.array_equal(got["coords"].view(np.uint32), want.view(np.uint32))
        for k in ("record", "name", "altloc", "resname", "chain", "insertion", "segid", "element", "resid", "charge"):
            assert got["topology"][k] == [type(got["topology"][k][0])(v) for v in top[k]], k
        assert got["topology"]["serial"] == [s % 100000 for s in top["serial"]]
        assert np.array_equal(np.float32(got["topology"]["beta"]), np.float32(["%6.2f" % v for v in top["beta"]]))
        if box:
            assert np.array_equal(got["box"], np.float32([[float("%9.3f" % v) for v in b] for b in boxes]))
            assert np.array_equal(got["boxangles"], np.float32([[float("%7.2f" % v) for v in a] for a in angles]))
        else:
            assert not got["box"].any() and (got["boxangles"] == 90).all()
        # the file's own values come back unchanged
        assert of.write(list(got["coords"]), got["topology"], list(got["box"]) if box else None,
                        list(got["boxangles"]) if box else None) == raw


def test_atom_line_columns_by_hand():
    top = dict(record=["ATOM", "HETATM", "ATOM", "ATOM"], serial=[1, 123456, 99999, 100000], name=["CA", "FE", "OXT",
               "HG21"], altloc=["", "A", "", ""], resname=["ALA", "HEM", "NME", "POPC"], chain=["A", "", "B", "C"],
               resid=[1, -999, 9999, 42], insertion=["", "B", "", ""], occupancy=[1, 0.5, 0, 12.345],
               beta=[0, 999.99, -99.99, 1.005], segid=["P1", "", "SEGA", "L"], element=["C", "FE", "O", "H"],
               charge=[0, 2, -1, 0])
    xyz = np.float32([[1.5, -2.0005, 0], [-0.0, 9999.999, -999.999], [12.3456, 0.0004, -0.0004], [1, 2, 3]])
    raw = of.write([xyz], top)
    lines = raw.decode().split("\n")
    # record, serial, ' ', name, altloc, resname, chain, resid, insertion, '   ', x y z, occupancy, beta, 6 spaces,
    # segid, element, charge
    want = ["ATOM  " + "    1" + " " + " CA " + " " + "ALA " + "A" + "   1" + " " + "   " + "   1.500  -2.000   0.000" +
            "  1.00" + "  0.00" + " " * 6 + "P1  " + " C" + "  ",
            "HETATM" + "23456" + " " + "FE  " + "A" + "HEM " + " " + "-999" + "B" + "   " + "  -0.0009999.999-999.999" +
            "  0.50" + "999.99" + " " * 6 + "    " + "FE" + "2+",
            "ATOM  " + "99999" + " " + " OXT" + " " + "NME " + "B" + "9999" + " " + "   " + "  12.346   0.000  -0.000" +
            "  0.00" + "-99.99" + " " * 6 + "SEGA" + " O" + "1-",
            "ATOM  " + "    0" + " " + "HG21" + " " + "POPC" + "C" + "  42" + " " + "   " + "   1.000   2.000   3.000" +
            " 12.35" + "  1.00" + " " * 6 + "L   " + " H" + "  "]
    assert lines[0] == "MODEL        1"
    assert lines[1:5] == want
    assert all(len(ln) == 80 for ln in want)
    assert lines[5:] == ["ENDMDL", "END", ""]
    from moleculekit_b200 import pdb as pp

    got = pp._template(pp._fields(top, 4), 4)
    assert len(got) == 4 * 81
    rows = got.reshape(4, 81)
    for i in range(4):
        w = bytearray(want[i].encode() + b"\n")
        w[30:54] = b" " * 24
        assert bytes(rows[i]) == bytes(w), (i, bytes(rows[i]), bytes(w))


def test_template_matches_the_oracle_writer():
    for N, seed in ((1, 0), (5, 1), (333, 2), (2000, 3)):
        top = of.random_topology(N, seed)
        from moleculekit_b200 import pdb as pp

        rows = pp._template(pp._fields(top, N), N)[:N * 81].reshape(N, 81)
        assert len(pp._template(pp._fields(top, N), N)) % 4 == 0
        lines = of.write([np.zeros((N, 3), np.float32)], top).split(b"\n")[1:1 + N]
        for i, ln in enumerate(lines):
            want = bytearray(ln + b"\n")
            want[30:54] = b" " * 24
            assert bytes(rows[i]) == bytes(want), (N, seed, i)
    assert pp.frame_bytes(3, True) == 15 + 71 + 3 * 81 + 7
    raw = of.write([np.zeros((3, 3), np.float32)], of.random_topology(3, 0), [np.ones(3)], [np.full(3, 90.0)])
    assert len(raw) == pp.frame_bytes(3, True) + 4


def test_default_topology_fields():
    from moleculekit_b200 import pdb as pp

    t = pp._fields(dict(name=["CA", "N"], element=["C", "N"]), 2)
    assert list(t["serial"]) == [1, 2] and list(t["record"]) == ["ATOM", "ATOM"]
    assert list(t["resid"]) == [0, 0] and list(t["segid"]) == ["", ""] and list(t["charge"]) == [0, 0]

    class Mol:
        name = np.array(["CA"], object)
        element = np.array(["C"], object)
        resname = np.array(["GLY"], object)
        resid = np.array([7])

    rows = pp._template(pp._fields(Mol(), 1), 1)[:81]
    want = ("ATOM  " + "    1" + " " + " CA " + " " + "GLY " + " " + "   7" + " " + "   " + " " * 24 + "  0.00" + "  0.00" +
            " " * 6 + "    " + " C" + "  " + "\n")
    assert bytes(rows) == want.encode()


def test_writer_checks_before_the_file(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import pdb as pp

    N, F = 6, 4
    c = np.zeros((N, 3, F), np.float32)
    top = of.random_topology(N, 7)
    top["resid"] = [1] * N

    def huge(v, at=(5, 1, 2)):
        x = c.copy()
        x[at] = v
        return x

    def t_with(k, v, a=3):
        t = {kk: list(vv) for kk, vv in top.items()}
        t[k][a] = v
        return t

    box = np.full((3, F), 10.0, np.float32)
    cases = [((c[:, :2], top), {}), ((c[0], top), {}), ((np.zeros((0, 3, 4), np.float32), top), {}),
             ((c, dict(name=["C"] * 5)), {}), ((c, top), dict(chunk_bytes=0)),
             ((c, top), dict(boxangles=box)), ((c, top), dict(box=box[:, :3])),
             ((c, top), dict(box=box, boxangles=box[:2]))]
    for k, v in (("name", "CAXXX"), ("resname", "ABCDE"), ("segid", "ABCDE"), ("chain", "AB"), ("element", "FEX"),
                 ("altloc", "AB"), ("insertion", "AB"), ("record", "ATOMS"), ("name", "é"), ("name", "C\n"),
                 ("resid", 10000), ("resid", -1000), ("resid", 1.5), ("charge", 10), ("charge", 0.5),
                 ("occupancy", 1000.0), ("occupancy", -100.0), ("beta", np.nan), ("beta", np.inf),
                 ("serial", 1.5)):
        cases.append(((c, t_with(k, v)), dict(match=f"atom 3, field {k}")))
    for v in (np.nan, np.inf, -np.inf, 10000.0, np.float32(-1000.0), np.float32(-999.9996)):
        cases.append(((huge(v), top), dict(match="coords at frame 2, atom 5, axis y")))
    x = huge(1e7, (4, 0, 1))
    x[3, 2, 1] = np.nan
    x[0, 0, 3] = -5e5
    cases.append(((x, top), dict(match="frame 1, atom 3, axis z")))
    b = box.copy()
    b[1, 2] = 100000.0
    cases.append(((c, top), dict(box=b, match="box at frame 2, axis b")))
    b = box.copy()
    b[2, 1] = np.nan
    cases.append(((huge(np.nan, (0, 0, 1)), top), dict(box=b, match="box at frame 1, axis c")))
    ang = np.full((3, F), 90.0, np.float32)
    ang[0, 0] = 10000.0
    cases.append(((c, top), dict(box=box, boxangles=ang, match="boxangles at frame 0, axis a")))
    for args, kw in cases:
        match = kw.pop("match", None)
        with pytest.raises(ValueError, match=match):
            pp.pdb_bytes(*args, **kw)
        fn = tmp_path / "untouched.pdb"
        with pytest.raises(ValueError, match=match):
            pp.write_pdb(str(fn), *args, **kw)
        assert not fn.exists()
    # the range rule's edges pass the checks: only the missing device stops the call
    edge = huge(np.float32(9999.999), (0, 0, 0))
    edge[1, 1, 1] = np.float32(-999.999)
    edge[2, 2, 2] = np.float32(-0.0)
    ok_box = np.full((3, F), 99999.99, np.float32)
    ok_ang = np.full((3, F), -999.99, np.float32)
    ok_ang[1] = 9999.99
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pp.pdb_bytes(edge, top, box=ok_box, boxangles=ok_ang)
        fn = tmp_path / "t.pdb"
        fn.write_bytes(of.write(frames(3, 2, 0), of.random_topology(3, 0)))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pp.read_pdb_device(str(fn))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pp.decode_pdb_device(torch.zeros(16, dtype=torch.uint8), 1, np.zeros(0), 3)
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pp.encode_pdb_device(torch.zeros((6, 3, 4)), top)
    # no frames: just END, no device needed
    assert pp.pdb_bytes(np.zeros((5, 3, 0), np.float32), of.random_topology(5, 1)) == b"END\n"


def test_reader_rejects_before_the_device(tmp_path):
    from moleculekit_b200 import pdb as pp

    for raw, match in ((b"", "empty"), (b"REMARK 1\nTER\nEND\n", "no ATOM or HETATM"), (b"\n\n", "no ATOM"),
                       (b"ATOM\n", "no ATOM"), (b"MODEL 1\nHETAT 1\nENDMDL\n", "no ATOM")):
        fn = tmp_path / "r.pdb"
        fn.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            pp.index_pdb(str(fn))
    with pytest.raises(ValueError, match="chunk_bytes"):
        pp.index_pdb(str(fn), chunk_bytes=0)


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_pdb_index", 9), ("mkb_pdb_decode", 13), ("mkb_pdb_cell", 6), ("mkb_pdb_encode", 13)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
