"""K31 on the GPU: BinaryCIF columns decoded bit for bit as the oracle's sequential decoders for every coordinate chain,
RCSB-shaped files (extra categories, a second data block, column orders, bare category names, masks, gzip), model
numbers that do not start at 1, frame lists, every error message, the writer byte for byte the oracle's writer with
every chain and packing width chosen, the round trip, one trajectory through mmCIF and BinaryCIF, and more than 65 535
models in one decode and one encode."""
import msgpack
import numpy as np
import pytest
import torch

from oracle import bcif_format as of
from oracle import cif_format as cf

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def put(tmp_path, raw, name="t.bcif"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def check(tmp_path, raw, sel=None):
    from moleculekit_b200 import bcif as pb

    got, info = pb.read_bcif_device(put(tmp_path, raw), frames=sel)
    want = of.read(raw)
    s = slice(None) if sel is None else np.asarray(sel, dtype=np.int64)
    assert np.array_equal(bits(got.cpu().numpy()), bits(want["coords"].transpose(1, 2, 0)[:, :, s]))
    assert np.array_equal(info["model"], want["model"][s])
    n = got.shape[2]
    assert np.array_equal(bits(info["box"]), bits(np.repeat(want["box"][:, None], n, 1)))
    assert np.array_equal(bits(info["boxangles"]), bits(np.repeat(want["boxangles"][:, None], n, 1)))
    for k, v in want["topology"].items():
        assert list(info["topology"][k]) == list(np.asarray(v, dtype=info["topology"][k].dtype)), k
    return info


def fixed_then(chain, w=None, unsigned=None):
    """a coordinate encoder: FixedPoint(1000) over one forced chain (0 to 3) of the oracle"""
    def enc(x):
        q = [int(np.rint(np.float64(v) * 1000)) for v in x]
        data, e = of.chains(q)[chain]
        if w is not None:
            assert e[-2]["kind"] == "IntegerPacking" and e[-2]["byteCount"] == w and e[-2]["isUnsigned"] == unsigned, e
        return data, [{"kind": "FixedPoint", "factor": 1000, "srcType": 32}] + e
    return enc


def float_bytes(t):
    return lambda x: of.byte_array(np.asarray(x, np.float64 if t == 33 else np.float32), t)


def interval(x):
    lo, hi, steps = -100.0, 100.0, 2**20
    q = np.clip(np.rint((np.float64(x) - lo) / ((hi - lo) / (steps - 1))), 0, steps - 1).astype(np.int32)
    data, e = of.encode_int(q)
    return data, [{"kind": "IntervalQuantization", "min": lo, "max": hi, "numSteps": steps, "srcType": 32}] + e


def delta_origin(x):
    """Delta with a non-zero origin and d[0] != 0: origin 5, d[0] = q[0] - 5"""
    q = [int(np.rint(np.float64(v) * 1000)) for v in x]
    d = [q[0] - 5] + [q[i] - q[i - 1] for i in range(1, len(q))]
    data, e = of.pack(d)
    return data, [{"kind": "FixedPoint", "factor": 1000, "srcType": 32}, {"kind": "Delta", "origin": 5,
                                                                          "srcType": 3}] + e


@pytest.mark.parametrize("name,coord,scale", [
    ("float32", float_bytes(32), 30.0), ("float64", float_bytes(33), 30.0), ("fixed_int32", fixed_then(0), 1e5),
    ("delta_pack1_signed", fixed_then(2, 1, False), 0.02), ("delta_pack2_signed", fixed_then(2, 2, False), 3.0),
    ("pack1_unsigned", fixed_then(0, 1, True), -1), ("pack2_unsigned", fixed_then(0, 2, True), -2),
    ("runs", fixed_then(1), 30.0), ("delta_runs", fixed_then(3), 30.0), ("interval", interval, 30.0),
    ("delta_origin", delta_origin, 30.0)])
def test_coordinate_chains_match_the_oracle(tmp_path, name, coord, scale):
    N, F = 37, 5
    if scale == -1:  # non-negative quanta below 255 and limits: 1-byte unsigned packing
        xs = [np.float32(np.random.default_rng(f).choice([0, 0.254, 0.255, 0.256, 0.1], (N, 3))) for f in range(F)]
    elif scale == -2:
        xs = [np.float32(np.random.default_rng(f).uniform(40, 60, (N, 3))) for f in range(F)]
    else:
        xs = frames(N, F, 3, scale)
    top = cf.random_topology(N, 4)
    check(tmp_path, of.rcsb(xs, top, box=[10, 20, 30], angles=[90, 80, 70], coord=coord))


@pytest.mark.parametrize("bare,gz,order,base", [(False, False, None, 1), (True, True, list(reversed(of.TAGS)), 5),
                                                (False, True, of.TAGS[10:] + of.TAGS[:10], -3)])
def test_rcsb_shaped_files(tmp_path, bare, gz, order, base):
    xs = frames(23, 6, 7)
    raw = of.rcsb(xs, cf.random_topology(23, 8), box=[50, 60, 70], model_base=base, order=order, bare=bare, gz=gz)
    info = check(tmp_path, raw)
    assert info["model"].tolist() == list(range(base, base + 6))
    check(tmp_path, raw, sel=[5, 0, 0, 3])


def test_frame_lists_and_errors(tmp_path):
    from moleculekit_b200 import bcif as pb

    xs = frames(9, 4, 11)
    raw = of.write(xs, cf.random_topology(9, 11))
    check(tmp_path, raw, sel=[3, 1, 1, 2])
    check(tmp_path, raw, sel=[])
    with pytest.raises(IndexError):
        pb.read_bcif_frames(put(tmp_path, raw), [4])

    doc = msgpack.unpackb(raw, raw=False)
    cols = {c["name"]: c for c in doc["dataBlocks"][0]["categories"][-1]["columns"]}

    def variant(name, **kw):
        d = msgpack.unpackb(raw, raw=False)
        site = d["dataBlocks"][0]["categories"][-1]
        for c in site["columns"]:
            if c["name"] == name:
                c.update(kw)
        return put(tmp_path, msgpack.packb(d, use_bin_type=True), "v.bcif")

    # a masked coordinate: frame 2, atom 4
    m = [0] * 36
    m[2 * 9 + 4] = 2
    with pytest.raises(ValueError, match=r"frame 2, atom 4, column Cartn_y: a masked"):
        pb.read_bcif(variant("Cartn_y", mask=dict(zip(("data", "encoding"), of.encode_int(m)))))
    # a frame of another row count
    model = [1] * 9 + [2] * 8 + [3] * 10 + [4] * 9
    with pytest.raises(ValueError, match=r"frame 1 \(model 2, row 9\): 8 rows, frame 0 has 9"):
        pb.index_bcif(variant("pdbx_PDB_model_num", data=dict(zip(("data", "encoding"), of.encode_int(model)))))
    # device-found errors: a packing that ends inside a value, counts that do not sum to srcSize
    pk = {"kind": "IntegerPacking", "byteCount": 1, "isUnsigned": False, "srcSize": 36}
    mid = dict(data=np.int8([1] * 35 + [127]).tobytes(), encoding=[pk, {"kind": "ByteArray", "type": 1}])
    with pytest.raises(ValueError, match="column id: an IntegerPacking ends inside a value"):
        pb.index_bcif(variant("id", data=mid))
    few = dict(data=np.int8([1] * 37).tobytes(), encoding=[pk, {"kind": "ByteArray", "type": 1}])
    with pytest.raises(ValueError, match="column id: an IntegerPacking holds another number"):
        pb.index_bcif(variant("id", data=few))
    rl = dict(data=np.int32([1, 35]).tobytes(), encoding=[{"kind": "RunLength", "srcType": 3, "srcSize": 36},
                                                           {"kind": "ByteArray", "type": 3}])
    with pytest.raises(ValueError, match="column pdbx_PDB_model_num: the RunLength counts do not sum"):
        pb.index_bcif(variant("pdbx_PDB_model_num", data=rl))
    short = dict(zip(("data", "encoding"), of.encode_int([1] * 35)))
    with pytest.raises(ValueError, match="column id: decodes to 35 values, the category has 36 rows"):
        pb.index_bcif(variant("id", data=short))
    ints = dict(zip(("data", "encoding"), of.encode_int([1] * 36)))
    with pytest.raises(ValueError, match="column Cartn_z: a coordinate column that does not decode to floats"):
        pb.read_bcif(variant("Cartn_z", data=ints))
    huff = dict(data=b"\0" * 4, encoding=[{"kind": "Huffman"}, {"kind": "ByteArray", "type": 3}])
    with pytest.raises(ValueError, match="column Cartn_x: the encoding kind 'Huffman' is not supported"):
        pb.read_bcif(variant("Cartn_x", data=huff))
    assert cols["Cartn_x"]["data"]["encoding"][0]["kind"] == "FixedPoint"


def encodings(raw):
    """every (chain, width) the writer chose in a file"""
    out = set()

    def walk(enc):
        kinds = [e["kind"] for e in enc]
        if kinds[0] == "StringArray":
            walk(enc[0]["dataEncoding"])
            walk(enc[0]["offsetEncoding"])
            return
        kinds = [k for k in kinds if k != "FixedPoint"]
        chain = {("ByteArray",): 0, ("IntegerPacking", "ByteArray"): 0, ("RunLength",): 1, ("Delta",): 2,
                 ("Delta", "RunLength"): 3}
        head = tuple(k for k in kinds if k in ("Delta", "RunLength")) or tuple(kinds)
        w = next((e["byteCount"] for e in enc if e["kind"] == "IntegerPacking"), 4)
        out.add((chain.get(head, chain.get(tuple(kinds))), w))

    for cat in msgpack.unpackb(raw, raw=False)["dataBlocks"][0]["categories"]:
        for c in cat["columns"]:
            walk(c["data"]["encoding"])
            if c["mask"]:
                walk(c["mask"]["encoding"])
    return out


def test_writer_matches_the_oracle_byte_for_byte(tmp_path):
    from moleculekit_b200 import bcif as pb

    seen = set()
    for N, F, seed, scale, box in ((1, 1, 0, 30.0, False), (40, 3, 1, 30.0, True), (300, 7, 2, 1e4, True),
                                   (64, 20, 3, 0.05, False), (5, 200, 4, 300.0, True)):
        xs = np.float32(frames(N, F, seed, scale))
        if seed == 3:  # a slow drift: deltas of one byte
            xs = np.float32(np.cumsum(xs, axis=0))
        top = cf.random_topology(N, seed)
        bx = np.repeat(np.float32([[12.5], [30], [99.999]]), F, 1) if box else None
        raw = pb.bcif_bytes(xs.transpose(1, 2, 0), top, bx, title="t%d" % seed)
        want = of.write(list(xs), top, None if bx is None else bx[:, 0], title="t%d" % seed)
        assert raw == want
        seen |= encodings(raw)
        back, info = pb.read_bcif(put(tmp_path, raw))
        q = np.float32(np.rint(xs.transpose(1, 2, 0).astype(np.float64) * 1000) / 1000) + np.float32(0)  # no -0.0
        assert np.array_equal(bits(back), bits(q))
        assert info["model"].tolist() == list(range(1, F + 1))
    assert {c for c, _ in seen} >= {0, 1, 2, 3} and {w for _, w in seen} >= {1, 2, 4}, seen


def test_encode_device_level():
    from moleculekit_b200 import bcif as pb

    for v in ([127, -128, 255, 32767, -32768, 65535, 2**31 - 1, -(2**31 - 1)], [3], [7] * 99 + [8],
              list(range(10**6, 10**6 + 500))):
        enc, data = pb.encode_bcif_device(torch.tensor(v, dtype=torch.int32, device="cuda"))
        assert (bytes(data.cpu().numpy()), enc) == of.encode_int(v)
        back = pb.decode_bcif_device(dict(data=bytes(data.cpu().numpy()), encoding=enc), rows=len(v))
        assert back.cpu().tolist() == v
    x = torch.tensor([1.2345, -7.0005, 3.0], device="cuda")
    enc, data = pb.encode_bcif_device(x, 1000)
    assert (bytes(data.cpu().numpy()), enc) == of.encode_fixed(x.cpu().numpy(), 1000)


def test_one_trajectory_through_mmcif_and_bcif(tmp_path):
    from moleculekit_b200 import bcif as pb
    from moleculekit_b200 import cif as pc

    N, F = 57, 6
    x = np.float32(np.rint(np.float64(np.float32(frames(N, F, 21, 40.0))) * 1000) / 1000).transpose(1, 2, 0)
    x = np.ascontiguousarray(x) + np.float32(0)  # -0.0 has no quantum of its own: BinaryCIF reads it as +0.0
    top = cf.random_topology(N, 21)
    box = np.repeat(np.float32([[31.5], [42.25], [53.125]]), F, 1)
    ang = np.repeat(np.float32([[90], [100.5], [120]]), F, 1)
    fc, fb = str(tmp_path / "t.cif"), str(tmp_path / "t.bcif")
    pc.write_cif(fc, x, top, box, ang)
    pb.write_bcif(fb, x, top, box, ang)
    a, ia = pc.read_cif(fc)
    b, ib = pb.read_bcif(fb)
    assert np.array_equal(bits(a), bits(b)) and np.array_equal(bits(b), bits(x))
    assert np.array_equal(ia["model"], ib["model"])
    for k in ("box", "boxangles"):
        assert np.array_equal(bits(ia[k]), bits(ib[k]))
    for k, v in ia["topology"].items():
        if k != "serial":
            assert list(v) == list(ib["topology"][k]), k


def test_more_than_65535_models(tmp_path):
    from moleculekit_b200 import bcif as pb

    N, F = 3, 70000
    x = np.random.default_rng(5).normal(0, 20, (N, 3, F)).astype(np.float32)
    fn = str(tmp_path / "big.bcif")
    pb.write_bcif(fn, torch.from_numpy(x).cuda(), cf.random_topology(N, 5))
    got, info = pb.read_bcif_device(fn)
    assert info["n_frames"] == F and info["model"][-1] == F
    want = np.float32(np.rint(x.astype(np.float64) * 1000) / 1000) + np.float32(0)  # a quantum of 0 reads as +0.0
    assert np.array_equal(bits(got.cpu().numpy()), bits(want))
    sel = [F - 1, 0, 65536]
    part, _ = pb.read_bcif_frames(fn, sel, index=pb.index_bcif(fn))
    assert np.array_equal(bits(part), bits(got.cpu().numpy()[:, :, sel]))
