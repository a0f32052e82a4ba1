"""The host side of BinaryCIF reading and writing (moleculekit_b200/bcif.py; K31 decodes and encodes on the device): the
independent oracle's encoders against its decoders on the packing limits and int32 wrap, the size formula against the
packed lengths, the classifier's tie order, the container errors raised before any device call, every writer check
before the file is opened, and the C-ABI symbols."""
import os

import msgpack
import numpy as np
import pytest

from oracle import bcif_format as of
from oracle import cif_format as cf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMITS = [127, -128, 255, 32767, -32768, 65535, 2**31 - 1, -(2**31 - 1), 0, 128, -129, 256, 65536, -32769, 7, 7, 7]


def wrap32(v):
    return [((int(x) + 2**31) % 2**32) - 2**31 for x in v]


@pytest.mark.parametrize("v", [LIMITS, [5] * 40, list(range(-300, 300, 7)), [2**31 - 1, -(2**31 - 1), 2**31 - 1],
                               [0], [1000, 1001, 1003, 1003, 1003, 990]])
def test_oracle_chains_round_trip(v):
    for data, enc in of.chains(v):
        assert of.decode(data, enc).tolist() == wrap32(v), enc
    x = np.float32([x for x in v if abs(x) < 2**30] or [0]) / np.float32(1000)
    data, enc = of.encode_fixed(x, 1000)
    assert np.array_equal(of.decode(data, enc), np.float32(np.rint(x.astype(np.float64) * 1000) / 1000))


def test_delta_wraps_int32():
    v = [2**31 - 1, -(2**31 - 1), 5, 2**31 - 1]
    d = of.deltas(v)
    assert d[1] == 2 and all(-2**31 <= x < 2**31 for x in d)
    enc = [{"kind": "Delta", "origin": v[0], "srcType": 3}, {"kind": "ByteArray", "type": 3}]
    assert of.decode(np.int32(d).tobytes(), enc).tolist() == v
    # d[0] != 0 and a non-zero origin; narrowing to Int8
    enc = [{"kind": "Delta", "origin": 100, "srcType": 1}, {"kind": "ByteArray", "type": 3}]
    assert of.decode(np.int32([27, 1, 5]).tobytes(), enc).tolist() == [127, -128, -123]


def test_size_formula_matches_the_packed_lengths():
    rng = np.random.default_rng(1)
    for v in (LIMITS, rng.integers(-70000, 70000, 200).tolist(), rng.integers(0, 300, 200).tolist()):
        for unsigned in ((False, True) if min(v) >= 0 else (False,)):
            for w, lims in ((1, (0xFF, 0xFF) if unsigned else (0x7F, 0x80)), (2, (0xFFFF, 0xFFFF) if unsigned
                                                                                 else (0x7FFF, 0x8000))):
                want = sum(abs(x) // (lims[0] if x >= 0 else lims[1]) + 1 for x in v)
                assert len(of.elements(v, w, unsigned)) == want


def test_classifier_choices_and_tie_order():
    # (a) wins on random small values, (b) on long runs, (c) on a ramp, (d) on a staircase of equal steps
    rng = np.random.default_rng(2)
    cases = {0: rng.integers(0, 100, 300).tolist(), 1: [7] * 100 + [9] * 100,
             2: (np.cumsum(rng.integers(-3, 4, 300)) + 10**6).tolist(), 3: list(range(10**6, 10**6 + 300))}
    for c, v in cases.items():
        sizes = [len(d) for d, _ in of.chains(v)]
        assert int(np.argmin(sizes)) == c, (c, sizes)
        assert of.encode_int(v) == of.chains(v)[c]
    # a tie goes to the earlier chain: one value, every chain's payload is one byte or the RunLength pair
    v = [3]
    sizes = [len(d) for d, _ in of.chains(v)]
    assert sizes[0] == min(sizes) and of.encode_int(v) == of.chains(v)[0]
    assert of.encode_int([0, 0]) == of.chains([0, 0])[0]  # (a) 2 bytes ties (c) 2 bytes
    # each packing width: Int32 for huge values, 2 bytes, 1 byte
    assert of.packing([2**30, -2**30])[0] == 4 and of.packing([300, -300, 1000])[0] == 2
    assert of.packing([1, 2, 3])[:2] == (1, True) and of.packing([-1, 2])[:2] == (1, False)


def _doc(cats, blocks=None):
    return msgpack.packb({"version": "0.3.0", "encoder": "t",
                          "dataBlocks": blocks if blocks is not None else [{"header": "x", "categories": cats}]},
                         use_bin_type=True)


@pytest.mark.parametrize("raw,match", [
    (b"", "not a \\(gzip\\) MessagePack"),
    (b"\xc1garbage", "not a \\(gzip\\) MessagePack"),
    # gzip of b"\xc1" written out with a zero timestamp, so the test id is the same on every run and every Python
    (b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x02\xff;\x08\x00\xab\x1da>\x01\x00\x00\x00", "not a \\(gzip\\) MessagePack"),
    (msgpack.packb([1, 2, 3]), "not shaped as a BinaryCIF document"),
    (_doc(None, blocks=[]), "not shaped"),
    (_doc([{"name": "_atom_site", "columns": [{"name": 3, "data": {}}], "rowCount": 1}]), "not shaped"),
    (_doc([{"name": "_entry", "columns": [], "rowCount": 1}]), "no _atom_site category"),
    (_doc([{"name": "atom_site", "columns": [], "rowCount": 1}]), "no Cartn_x column"),
])
def test_container_errors_before_any_device_call(tmp_path, raw, match):
    from moleculekit_b200 import bcif as pb

    fn = tmp_path / "bad.bcif"
    fn.write_bytes(raw)
    with pytest.raises(ValueError, match=match) as e:
        pb.index_bcif(str(fn))
    assert str(fn) in str(e.value)


def test_chain_errors_before_any_device_call():
    from moleculekit_b200 import bcif as pb

    ba = {"kind": "ByteArray", "type": 3}
    for data, enc, match in [
        (b"\0" * 6, [ba], "not a whole number of 4-byte values"),
        (b"\0" * 4, [{"kind": "Huffman"}, ba], "kind 'Huffman' is not supported"),
        (b"\0" * 4, [{"kind": "Delta", "origin": 0, "srcType": 3}], "not a ByteArray"),
        (b"\0" * 4, [{"kind": "Delta", "origin": 0, "srcType": 3}, {"kind": "ByteArray", "type": 32}], "over floats"),
        (b"\0" * 4, [{"kind": "IntegerPacking", "byteCount": 1, "isUnsigned": False, "srcSize": 5},
                     {"kind": "ByteArray", "type": 1}], "another number of values"),
        (b"\0" * 12, [{"kind": "RunLength", "srcType": 3, "srcSize": 1}, ba], "pairs"),
        (b"\0" * 4, [{"kind": "Delta"}, ba], "malformed"),
    ]:
        with pytest.raises(ValueError, match=match) as e:
            pb._chain("f.bcif", "Cartn_x", data, enc)
        assert "f.bcif, column Cartn_x" in str(e.value)


def test_writer_checks_before_the_file(tmp_path):
    from moleculekit_b200 import bcif as pb

    N, F = 6, 4
    c = np.zeros((N, 3, F), np.float32)
    top = cf.random_topology(N, 7)

    def t_with(k, v, a=3):
        t = {kk: list(vv) for kk, vv in top.items()}
        t[k][a] = v
        return t

    def huge(v, at=(5, 1, 2)):
        x = c.copy()
        x[at] = v
        return x

    box = np.full((3, F), 10.0, np.float32)
    cases = [((c[:, :2], top), {}), ((c[0], top), {}), ((np.zeros((0, 3, 4), np.float32), top), {}),
             ((np.zeros((3, 3, 0), np.float32), top), {}), ((c, dict(name=["C"] * 5)), {}),
             ((c, top), dict(boxangles=box)), ((c, top), dict(box=box[:, :3])),
             ((c, top), dict(box=box, boxangles=box[:2])), ((c, top), dict(title="")), ((c, top), dict(title=3))]
    for k, v in (("name", "é"), ("segid", "Å"), ("resid", 1.5), ("resid", 2.0**31), ("charge", np.nan),
                 ("occupancy", np.inf), ("beta", 3e7)):
        cases.append(((c, t_with(k, v)), dict(match=f"atom 3, field {k}")))
    for v in (np.nan, np.inf, -np.inf, 2.2e6, -2.2e6):
        cases.append(((huge(v), top), dict(match="coords at frame 2, atom 5, axis y")))
    b = box.copy()
    b[1, 2] = 11.0
    cases.append(((c, top), dict(box=b, match="the box of frame 2 differs")))
    b = box.copy()
    b[2, 1] = np.nan
    cases.append(((c, top), dict(box=b, match="box at frame 1, axis c")))
    for args, kw in cases:
        match = kw.pop("match", None)
        with pytest.raises(ValueError, match=match):
            pb.bcif_bytes(*args, **kw)
        fn = tmp_path / "untouched.bcif"
        with pytest.raises(ValueError, match=match):
            pb.write_bcif(str(fn), *args, **kw)
        assert not fn.exists()


def test_without_a_device_nothing_falls_back(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import bcif as pb

    if torch.cuda.is_available():
        pytest.skip("a device is present")
    top = cf.random_topology(3, 0)
    fn = tmp_path / "t.bcif"
    fn.write_bytes(of.write([np.zeros((3, 3), np.float32)], top))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pb.read_bcif_device(str(fn))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pb.bcif_bytes(np.zeros((3, 3, 1), np.float32), top)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pb.encode_bcif_device(torch.zeros(4, dtype=torch.int32))


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_bcif_decode", 13), ("mkb_bcif_quantize", 9), ("mkb_bcif_sizes", 7),
                        ("mkb_bcif_emit", 12)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
