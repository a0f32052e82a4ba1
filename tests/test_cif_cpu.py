"""The host side of multi-model PDBx/mmCIF reading and writing (moleculekit_b200/cif.py; K30 indexes, parses and formats
on the device): the independent oracle's round trip, the host tokenizer against the oracle's, the search for the
_atom_site loop header, the topology mapping, the host row template against the oracle writer, the writer's checks
that run before the file is opened, and the C-ABI symbols."""
import os

import numpy as np
import pytest

from oracle import cif_format as of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def test_oracle_round_trip():
    for N, box in ((1, False), (3, True), (40, True)):
        top = of.random_topology(N, N)
        xs = frames(N, 4, N)
        cell = ([10.5, 20.25, 99999.99], [90, 60, 120.25]) if box else (None, None)
        raw = of.write(xs, top, *cell)
        got = of.read(raw)
        assert got["natoms"] == N and got["model"].tolist() == [1, 2, 3, 4]
        want = np.float32([[[float("%10.3f" % v) for v in row] for row in x] for x in xs])
        assert np.array_equal(got["coords"].view(np.uint32), want.view(np.uint32))
        for k in ("record", "name", "altloc", "resname", "chain", "insertion", "segid", "element", "resid", "charge"):
            assert got["topology"][k] == [type(got["topology"][k][0])(v) for v in top[k]], k
        assert got["topology"]["serial"] == list(range(1, N + 1))
        if box:
            assert np.array_equal(got["box"], np.float32([float("%.3f" % v) for v in cell[0]]))
            assert np.array_equal(got["boxangles"], np.float32([float("%.2f" % v) for v in cell[1]]))
        else:
            assert not got["box"].any() and (got["boxangles"] == 90).all()
        # an RCSB-style file of the same frames reads back the same
        rc = of.read(of.rcsb(xs, top, box=None if not box else [*cell[0], *cell[1]], fmt="%10.3f"))
        assert np.array_equal(rc["coords"], got["coords"]) and rc["topology"]["name"] == got["topology"]["name"]


@pytest.mark.parametrize("line", [
    b"ATOM 1 C \"O5'\" . DA A 1 1.0 2.0 3.0",
    b"ATOM 2 C 'C 1' . 'A B' A 1 1.0 2.0 3.0 ",
    b"HETATM 3 O O5' . \"x'y z\" . 1 -1.5 2 3\r",
    b"  'it''s' \"a\"b\" x'y 'loop_' data_x \t 'stop_'\v? .",
    b"'a' 'b'c' \"\" '' 'x ' ",
    b"A 'unclosed",
    b";text field",
    b"  ;x",
])
def test_host_tokenizer_matches_the_oracle(line):
    from moleculekit_b200 import cif as pc

    toks, complete = pc._tokens(line)
    try:
        want = of.tokens(line)
    except ValueError:
        assert not complete
        return
    assert complete and toks == want


def test_cif_token_quoting():
    from moleculekit_b200 import cif as pc

    for s in ("CA", "O5'", "C 1", "_X", "#1", "$y", "[x]", "]x", ";z", "'q", '"q', ".", "?", "loop_", "LOOP_", "data_x",
              "Save_1", "global_", "stop_", "a\"b", "it's"):
        tok = pc.cif_token(s)
        assert tok == of.quote(s), s
        assert pc._tokens(tok.encode())[0] == [(s.encode(), tok != s)], s
    assert pc.cif_token("") == "."
    for s in ("'a \" b", "é", "a\tb", "a\nb"):
        assert pc.cif_token(s) is None


def test_template_matches_the_oracle_writer():
    from moleculekit_b200 import cif as pc

    for N, F, seed, box in ((1, 1, 0, False), (5, 12, 1, True), (333, 3, 2, False), (2000, 1, 3, True)):
        top = of.random_topology(N, seed)
        tmpl, R, c_id, w_id, c_x, c_model, w_model = pc._layout(pc._fields(top, N), N, F)
        assert len(tmpl) % 4 == 0 and w_id == len(str(N * F)) and w_model == len(str(F))
        cell = ([10, 20, 30], [90, 90, 120]) if box else (None, None)
        raw = of.write([np.zeros((N, 3), np.float32)] * F, top, *cell)
        head = pc._header("trajectory", *(np.float32(c) if c is not None else None for c in cell))
        assert raw.startswith(head) and raw.endswith(b"#\n")
        assert len(raw) == len(head) + F * pc.frame_bytes(N, R) + 2
        rows = raw[len(head):].split(b"\n")
        for i in range(N):
            want = bytearray(rows[i] + b"\n")
            for a, w in ((c_id, w_id), (c_x, 32), (c_model, w_model)):
                want[a:a + w] = b" " * w
            assert bytes(tmpl[i * R:(i + 1) * R]) == bytes(want), (N, i)


def _scan(tmp_path, raw):
    from moleculekit_b200 import cif as pc

    fn = tmp_path / "h.cif"
    fn.write_bytes(raw)
    with open(fn, "rb") as fh:
        return pc._scan(str(fn), fh.fileno(), 0, len(raw), True)


def test_header_search(tmp_path):
    xs, top = frames(6, 2, 0), of.random_topology(6, 0)
    raw = of.rcsb(xs, top, box=[10, 20, 30, 90, 90, 90])
    h = _scan(tmp_path, raw)
    assert h["tags"] == [t.lower() for t in of.TAGS]
    assert raw[h["body"]:].startswith(b"HETATM 1 ") or raw[h["body"]:].startswith(b"ATOM 1 ")
    assert h["cell"] == dict(length_a=10.0, length_b=20.0, length_c=30.0, angle_alpha=90.0, angle_beta=90.0,
                             angle_gamma=90.0)
    # the loop after megabytes of other categories (a loop with many rows and a text field), and an
    # _atom_site_anisotrop loop before it
    filler = b"loop_\n_pdbx_filler.id\n_pdbx_filler.text\n" + b"".join(b"%d 'row of filler text'\n" % i
                                                                      for i in range(150000))
    decoy = b"#\nloop_\n_atom_site_anisotrop.id\n_atom_site_anisotrop.U[1][1]\n1 0.5\n#\n"
    k = raw.index(b"loop_\n_atom_site.")
    big = raw[:k] + filler + decoy + b"_struct.pdbx_descriptor\n;\nloop_\n_atom_site.id\n;\n" + raw[k:]
    assert len(big) > 3 << 20
    h = _scan(tmp_path, big)
    assert h["body"] == raw.index(b"\n", raw.index(b"_atom_site.pdbx_PDB_model_num")) + 1 + len(big) - len(raw)
    # tags in mixed case
    mixed = raw.replace(b"_atom_site.Cartn_x", b"_ATOM_SITE.CARTN_X").replace(b"_atom_site.id", b"_Atom_Site.ID")
    h = _scan(tmp_path, mixed)
    assert h["tags"][1] == "id" and "cartn_x" in h["tags"]


def test_header_errors(tmp_path):
    from moleculekit_b200 import cif as pc

    raw = of.rcsb(frames(4, 1, 1), of.random_topology(4, 1))
    cases = [(b"", "the file is empty"),
             (raw.replace(b"_atom_site.Cartn_z", b"_atom_site.Cartn_q"), "no _atom_site.Cartn_z tag"),
             (raw.replace(b"loop_\n_atom_site.", b"loop_\n_atom_sitex."), "no _atom_site loop"),
             (b"data_x\n#\n_entry.id x\n", "no _atom_site loop"),
             (b"data_a\n_entry.id a\ndata_b\n" + raw[raw.index(b"loop_\n_atom_site."):], "no _atom_site loop"),
             (b"data_x\n_atom_site.id 1\n_atom_site.Cartn_x 1\n", "not a loop")]
    for data, match in cases:
        fn = tmp_path / "e.cif"
        fn.write_bytes(data)
        with pytest.raises(ValueError, match=match):
            pc.index_cif(str(fn))
    with pytest.raises(ValueError, match="chunk_bytes"):
        pc.index_cif(str(fn), chunk_bytes=0)


def test_topology_mapping(tmp_path):
    from moleculekit_b200 import cif as pc

    top = of.random_topology(30, 5)
    raw = of.write(frames(30, 1, 5), top)
    fn = tmp_path / "t.cif"
    fn.write_bytes(raw)
    h = _scan(tmp_path, raw)
    with open(fn, "rb") as fh:
        t = pc._topology(str(fn), fh.fileno(), h["tags"], raw[h["body"]:], h["body"])
    want = of.read(raw)["topology"]
    for k in pc.FIELDS:
        assert list(t[k]) == list(np.asarray(want[k], dtype=t[k].dtype)), k
    # the label_* fallbacks, missing tags, '?' and '.' blanks, and a standard uncertainty on a number
    tags = ["label_atom_id", "label_comp_id", "label_asym_id", "label_seq_id", "Cartn_x", "Cartn_y", "Cartn_z",
            "occupancy", "pdbx_formal_charge"]
    rows = b"CA ALA B 7 1 2 3 0.5(1) -1\n'O5''' ? . ? 1 2 3 . ?\n"
    body = b"data_x\nloop_\n" + b"".join(b"_atom_site.%s\n" % t.encode() for t in tags) + rows
    fn.write_bytes(body)
    with open(fn, "rb") as fh:
        t = pc._topology(str(fn), fh.fileno(), [x.lower() for x in tags], rows, len(body) - len(rows))
    assert list(t["name"]) == ["CA", "O5''"] and list(t["resname"]) == ["ALA", ""]
    assert list(t["chain"]) == ["B", ""] and list(t["segid"]) == ["B", ""] and list(t["resid"]) == [7, 0]
    assert list(t["occupancy"]) == [0.5, 0.0] and list(t["charge"]) == [-1.0, 0.0]
    assert list(t["record"]) == ["", ""] and list(t["serial"]) == [0, 0] and list(t["beta"]) == [0.0, 0.0]
    bad = body.replace(b"B 7 1", b"B 7x 1")
    fn.write_bytes(bad)
    with open(fn, "rb") as fh, pytest.raises(ValueError, match=r"frame 0, line 12, column 4: the label_seq_id token "
                                                                r"b'7x' is not an integer"):
        pc._topology(str(fn), fh.fileno(), [x.lower() for x in tags], rows.replace(b"7", b"7x", 1),
                     len(bad) - len(rows) - 1)


def test_writer_checks_before_the_file(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import cif as pc

    N, F = 6, 4
    c = np.zeros((N, 3, F), np.float32)
    top = of.random_topology(N, 7)

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
             ((c, top), dict(box=box, boxangles=box[:2])), ((c, top), dict(title="a b")),
             ((c, top), dict(title="")), ((c, dict(name=["x" * 800] * N)), dict(match="768"))]
    for k, v in (("name", "a'b \""), ("resname", "é"), ("segid", "A\tB"), ("chain", "x\n"), ("element", "x\x01"),
                 ("resid", 1.5), ("resid", np.nan), ("charge", 0.5), ("occupancy", np.inf), ("beta", np.nan)):
        cases.append(((c, t_with(k, v)), dict(match=f"atom 3, field {k}")))
    for v in (np.nan, np.inf, -np.inf, 1e6, np.float32(-100000.0), np.float32(-99999.9996)):
        cases.append(((huge(v), top), dict(match="coords at frame 2, atom 5, axis y")))
    x = huge(1e7, (4, 0, 1))
    x[3, 2, 1] = np.nan
    x[0, 0, 3] = -5e5
    cases.append(((x, top), dict(match="frame 1, atom 3, axis z")))
    b = box.copy()
    b[1, 2] = 11.0
    cases.append(((c, top), dict(box=b, match="the box of frame 2 differs")))
    ang = np.full((3, F), 90.0, np.float32)
    ang[0, 3] = 60.0
    cases.append(((c, top), dict(box=box, boxangles=ang, match="the box of frame 3 differs")))
    b = box.copy()
    b[2, 1] = np.nan
    cases.append(((c, top), dict(box=b, match="box at frame 1, axis c")))
    for args, kw in cases:
        match = kw.pop("match", None)
        with pytest.raises(ValueError, match=match):
            pc.cif_bytes(*args, **kw)
        fn = tmp_path / "untouched.cif"
        with pytest.raises(ValueError, match=match):
            pc.write_cif(str(fn), *args, **kw)
        assert not fn.exists()
    # the range rule's edges pass the checks: only the missing device stops the call
    edge = huge(np.float32(999999.9), (0, 0, 0))
    edge[1, 1, 1] = np.float32(-99999.99)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pc.cif_bytes(edge, top, box=box)
        fn = tmp_path / "t.cif"
        fn.write_bytes(of.write(frames(3, 2, 0), of.random_topology(3, 0)))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pc.read_cif_device(str(fn))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pc.decode_cif_device(torch.zeros(16, dtype=torch.uint8), 1, np.zeros(0), 3, (0, 1, 2))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pc.encode_cif_device(torch.zeros((6, 3, 4)), top)
    # no frames: the header and the last '#', no device needed
    raw = pc.cif_bytes(np.zeros((5, 3, 0), np.float32), of.random_topology(5, 1), title="empty")
    assert raw == of.write([], of.random_topology(5, 1), title="empty")


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_cif_index", 12), ("mkb_cif_decode", 16), ("mkb_cif_encode", 16)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
