"""An independent restatement of BinaryCIF in numpy and ``msgpack``: sequential decoders of every encoding, the writer's
classifier and encoders, a writer of multi-model ``_atom_site`` files and a reader.  Test infrastructure: the tests hold
moleculekit_b200/bcif.py and K31 to it, so it shares no code with them.  ``rcsb`` writes files shaped as the PDB's:
extra categories before and after ``_atom_site``, a second data block, any column order, category names with or
without the leading ``_``, masks, and gzip.

Encodings (the list gives the steps in the order they were applied; decoding runs it backwards):
ByteArray{type} (Int8 1, Int16 2, Int32 3, Uint8 4, Uint16 5, Uint32 6, Float32 32, Float64 33, little-endian),
IntegerPacking{byteCount, isUnsigned, srcSize}, Delta{origin, srcType}, RunLength{srcType, srcSize},
FixedPoint{factor, srcType}, IntervalQuantization{min, max, numSteps, srcType} and StringArray{dataEncoding, stringData,
offsetEncoding, offsets}.

The writer: every integer array takes the smallest of (a) IntegerPacking, (b) RunLength -> IntegerPacking, (c)
Delta(origin = v[0], d[0] = 0) -> IntegerPacking and (d) Delta -> RunLength -> IntegerPacking (ties to the earlier);
the packing is unsigned when no value is negative, and with size1 / size2 the element counts at 1 / 2 bytes it is none
(ByteArray Int32) when 4 n < 2 size2, else 2 bytes when 2 size2 < size1, else 1 byte.
"""
from __future__ import annotations

import gzip

import msgpack
import numpy as np

TAGS = ["group_PDB", "id", "type_symbol", "label_atom_id", "label_alt_id", "label_comp_id", "label_asym_id",
        "label_entity_id", "label_seq_id", "pdbx_PDB_ins_code", "Cartn_x", "Cartn_y", "Cartn_z", "occupancy",
        "B_iso_or_equiv", "pdbx_formal_charge", "auth_seq_id", "auth_comp_id", "auth_asym_id", "auth_atom_id",
        "pdbx_PDB_model_num"]
DTYPE = {1: "<i1", 2: "<i2", 3: "<i4", 4: "<u1", 5: "<u2", 6: "<u4", 32: "<f4", 33: "<f8"}
WRAP = {1: np.int8, 2: np.int16, 3: np.int32, 4: np.uint8, 5: np.uint16, 6: np.uint32}
CELL = ["length_a", "length_b", "length_c", "angle_alpha", "angle_beta", "angle_gamma"]


# ------------------------------------------------------------------------------------------------------------ decoding
def _wrap(vals, src_type):
    return np.array([int(v) for v in vals], dtype=np.int64).astype(np.uint64).astype(WRAP[src_type]) \
        if len(vals) else np.zeros(0, WRAP[src_type])


def decode(data, encoding):
    """one encoded array -> numpy array (StringArray -> list of str)"""
    for e in reversed(encoding):
        k = e["kind"]
        if k == "ByteArray":
            data = np.frombuffer(data, DTYPE[e["type"]]).copy()
        elif k == "IntegerPacking":
            w, u = e["byteCount"], e["isUnsigned"]
            hi, lo = ((0xFF, None) if w == 1 else (0xFFFF, None)) if u else ((0x7F, -0x80) if w == 1 else (0x7FFF, -0x8000))
            out, i, n = [], 0, len(data)
            while i < n:
                t = 0
                v = int(data[i])
                while v == hi or v == lo:
                    t += v
                    i += 1
                    if i == n:
                        raise ValueError("IntegerPacking ends inside a value")
                    v = int(data[i])
                out.append(t + v)
                i += 1
            if len(out) != e["srcSize"]:
                raise ValueError("IntegerPacking holds another number of values")
            data = _wrap(out, 3)
        elif k == "Delta":
            out, acc = [], int(e["origin"])
            for d in data:
                acc = (acc + int(d)) & 0xFFFFFFFF
                out.append(acc)
            data = _wrap(out, e["srcType"])
        elif k == "RunLength":
            out = []
            for j in range(0, len(data), 2):
                out += [int(data[j])] * int(data[j + 1])
            if len(out) != e["srcSize"]:
                raise ValueError("RunLength counts do not sum to srcSize")
            data = _wrap(out, e["srcType"])
        elif k == "FixedPoint":
            data = np.array([np.float32(float(int(q)) / float(e["factor"])) for q in data], np.float32)
        elif k == "IntervalQuantization":
            step = (float(e["max"]) - float(e["min"])) / (float(e["numSteps"]) - 1.0)
            data = np.array([np.float32(float(e["min"]) + step * float(int(q))) for q in data], np.float32)
        elif k == "StringArray":
            idx = decode(data, e["dataEncoding"])
            off = decode(e["offsets"], e["offsetEncoding"])
            strings = [e["stringData"][off[j]:off[j + 1]] for j in range(len(off) - 1)]
            return [strings[int(i)] for i in idx]
        else:
            raise ValueError(f"unknown encoding {k}")
    if data.dtype == np.float64:
        data = data.astype(np.float32)
    return data


# ------------------------------------------------------------------------------------------------------------ encoding
def byte_array(v, type_):
    return np.asarray(v).astype(DTYPE[type_]).tobytes(), [{"kind": "ByteArray", "type": type_}]


def elements(v, w, unsigned):
    """the elements IntegerPacking writes for each value"""
    out = []
    for x in (int(x) for x in v):
        if unsigned or x >= 0:
            lim = (0xFF if w == 1 else 0xFFFF) if unsigned else (0x7F if w == 1 else 0x7FFF)
            while x >= lim:
                out.append(lim)
                x -= lim
        else:
            lim = -0x80 if w == 1 else -0x8000
            while x <= lim:
                out.append(lim)
                x -= lim
        out.append(x)
    return out


def packing(v):
    """(width 1, 2 or 4, unsigned, payload bytes) of the classifier's packing choice"""
    n = len(v)
    unsigned = bool(min(int(x) for x in v) >= 0)
    size1, size2 = len(elements(v, 1, unsigned)), len(elements(v, 2, unsigned))
    if 4 * n < 2 * size2:
        return 4, unsigned, 4 * n
    if 2 * size2 < size1:
        return 2, unsigned, 2 * size2
    return 1, unsigned, size1


def pack(v):
    """(payload, encoding list) of the packing step alone"""
    w, u, _ = packing(v)
    if w == 4:
        return byte_array(v, 3)
    e = elements(v, w, u)
    t = {(1, False): 1, (2, False): 2, (1, True): 4, (2, True): 5}[(w, u)]
    data, enc = byte_array(e, t)
    return data, [{"kind": "IntegerPacking", "byteCount": w, "isUnsigned": u, "srcSize": len(v)}] + enc


def deltas(v):
    v = [int(x) for x in v]
    return [0] + [((v[i] - v[i - 1] + 2**31) % 2**32) - 2**31 for i in range(1, len(v))]


def runs(v):
    out = []
    for x in (int(x) for x in v):
        if out and out[-2] == x:
            out[-1] += 1
        else:
            out += [x, 1]
    return out


def chains(v):
    """the four candidate chains of an integer array -> [(payload, encoding list)] for (a) to (d)"""
    v = [int(x) for x in v]
    n = len(v)
    rl = {"kind": "RunLength", "srcType": 3, "srcSize": n}
    de = {"kind": "Delta", "origin": v[0], "srcType": 3}
    out = []
    for pre, arr in (([], v), ([rl], runs(v)), ([de], deltas(v)), ([de, rl], runs(deltas(v)))):
        data, enc = pack(arr)
        out.append((data, pre + enc))
    return out


def encode_int(v):
    """the classifier's choice: the fewest payload bytes, ties to the earlier chain"""
    best = None
    for data, enc in chains(v):
        if best is None or len(data) < len(best[0]):
            best = (data, enc)
    return best


def encode_fixed(x, factor):
    q = [int(np.rint(np.float64(v) * factor)) for v in np.asarray(x, np.float32).reshape(-1)]
    data, enc = encode_int(q)
    return data, [{"kind": "FixedPoint", "factor": factor, "srcType": 32}] + enc


def encode_strings(vals):
    """(column dict) of a text column: unique strings in order of first appearance, '' masked as '.'"""
    uniq = {}
    for s in vals:
        uniq.setdefault(s, len(uniq))
    strings = list(uniq)
    off = [0]
    for s in strings:
        off.append(off[-1] + len(s))
    idx = [uniq[s] for s in vals]
    idata, ienc = encode_int(idx)
    odata, oenc = encode_int(off)
    col = {"data": idata, "encoding": [{"kind": "StringArray", "dataEncoding": ienc, "stringData": "".join(strings),
                                        "offsetEncoding": oenc, "offsets": odata}]}
    mask = None
    if "" in uniq:
        m = [1 if s == "" else 0 for s in vals]
        mdata, menc = encode_int(m)
        mask = {"data": mdata, "encoding": menc}
    return col, mask


def column(name, data_enc, mask=None):
    return {"name": name, "data": {"data": data_enc[0], "encoding": data_enc[1]} if isinstance(data_enc, tuple)
            else data_enc, "mask": mask}


def write(frames, topology: dict, box=None, angles=None, title: str = "trajectory") -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays; ``topology``: per-atom sequences (record, name, altloc, resname,
    chain, resid, insertion, occupancy, beta, segid, element, charge); ``box`` / ``angles`` the one cell -> bytes"""
    t = topology
    n, F = len(t["name"]), len(frames)
    xyz = np.asarray(frames, np.float32).reshape(F, n, 3)

    def text(name, key):
        col, mask = encode_strings([str(s) for s in t[key]] * F if key else [""] * (n * F))
        return column(name, col, mask)

    def ints(name, v):
        return column(name, encode_int([int(x) for x in v]))

    resid = [int(v) for v in t["resid"]] * F
    cols = {"group_PDB": text("group_PDB", "record"), "id": ints("id", range(1, n * F + 1)),
            "type_symbol": text("type_symbol", "element"), "label_atom_id": text("label_atom_id", "name"),
            "label_alt_id": text("label_alt_id", "altloc"), "label_comp_id": text("label_comp_id", "resname"),
            "label_asym_id": text("label_asym_id", "segid"), "label_entity_id": text("label_entity_id", None),
            "label_seq_id": ints("label_seq_id", resid), "pdbx_PDB_ins_code": text("pdbx_PDB_ins_code", "insertion"),
            "occupancy": column("occupancy", encode_fixed(list(t["occupancy"]) * F, 100)),
            "B_iso_or_equiv": column("B_iso_or_equiv", encode_fixed(list(t["beta"]) * F, 100)),
            "pdbx_formal_charge": ints("pdbx_formal_charge", [int(c) for c in t["charge"]] * F),
            "auth_seq_id": ints("auth_seq_id", resid), "auth_comp_id": text("auth_comp_id", "resname"),
            "auth_asym_id": text("auth_asym_id", "chain"), "auth_atom_id": text("auth_atom_id", "name"),
            "pdbx_PDB_model_num": ints("pdbx_PDB_model_num", np.repeat(np.arange(1, F + 1), n))}
    for d, c in enumerate(("Cartn_x", "Cartn_y", "Cartn_z")):
        cols[c] = column(c, encode_fixed(xyz[:, :, d].reshape(-1), 1000))
    cats = []
    if box is not None:
        ang = angles if angles is not None else (90.0, 90.0, 90.0)
        cats.append({"name": "_cell", "columns": [column(k, encode_fixed([v], 1000 if k.startswith("length") else 100))
                                                  for k, v in zip(CELL, [*box, *ang])], "rowCount": 1})
        sg, _ = encode_strings(["P 1"])
        cats.append({"name": "_symmetry", "columns": [column("space_group_name_H-M", sg)], "rowCount": 1})
    cats.append({"name": "_atom_site", "columns": [cols[k] for k in TAGS], "rowCount": n * F})
    doc = {"version": "0.3.0", "encoder": "moleculekit_b200", "dataBlocks": [{"header": title, "categories": cats}]}
    return msgpack.packb(doc, use_bin_type=True)


def read(data: bytes) -> dict:
    """the reader's rules, sequentially -> dict(coords (F, natoms, 3) float32, model, natoms, box, boxangles, topology)"""
    if data[:2] == b"\x1f\x8b":
        data = gzip.decompress(data)
    doc = msgpack.unpackb(data, raw=False)
    cats = {c["name"].lower().lstrip("_"): c for c in doc["dataBlocks"][0]["categories"]}
    site = cats["atom_site"]
    cols = {c["name"].lower(): c for c in site["columns"]}

    def values(c):
        v = decode(c["data"]["data"], c["data"]["encoding"])
        m = decode(c["mask"]["data"], c["mask"]["encoding"]) if c.get("mask") else None
        return v, m

    rows = site["rowCount"]
    model = values(cols["pdbx_pdb_model_num"])[0].astype(np.int64) if "pdbx_pdb_model_num" in cols else \
        np.zeros(rows, np.int64)
    starts = [0] + [i for i in range(1, rows) if model[i] != model[i - 1]]
    N, F = (starts[1] if len(starts) > 1 else rows), len(starts)
    xyz = np.stack([values(cols[c])[0] for c in ("cartn_x", "cartn_y", "cartn_z")], axis=1)

    def pick(*names):
        for k in names:
            if k in cols:
                v, m = values(cols[k])
                return v[:N], (m[:N] if m is not None else np.zeros(N))
        return None, None

    def text(*names):
        v, m = pick(*names)
        return [""] * N if v is None else ["" if m[i] else str(v[i]) for i in range(N)]

    def number(kind, *names):
        v, m = pick(*names)
        return [kind(0)] * N if v is None else [kind(0) if m[i] else kind(v[i]) for i in range(N)]

    top = dict(record=text("group_pdb"), serial=number(int, "id"), name=text("auth_atom_id", "label_atom_id"),
               altloc=text("label_alt_id"), resname=text("auth_comp_id", "label_comp_id"),
               chain=text("auth_asym_id", "label_asym_id"), resid=number(int, "auth_seq_id", "label_seq_id"),
               insertion=text("pdbx_pdb_ins_code"), occupancy=number(float, "occupancy"),
               beta=number(float, "b_iso_or_equiv"), segid=text("label_asym_id"), element=text("type_symbol"),
               charge=number(int, "pdbx_formal_charge"))
    box, ang = np.zeros(3, np.float32), np.full(3, 90.0, np.float32)
    if "cell" in cats:
        cc = {c["name"].lower(): c for c in cats["cell"]["columns"]}
        for j, k in enumerate(CELL):
            if k in cc:
                (box if j < 3 else ang)[j % 3] = values(cc[k])[0][0]
    return dict(coords=xyz.reshape(F, N, 3), model=model[starts], natoms=N, box=box, boxangles=ang, topology=top)


def rcsb(frames, topology: dict, box=None, angles=None, model_base: int = 1, order=None, bare: bool = False,
         gz: bool = False, coord=None) -> bytes:
    """A file shaped as the PDB's: ``_entry`` and ``_struct`` categories before ``_atom_site``, ``_atom_type`` after it,
    a second data block, the columns in ``order`` (tag names), category names without '_' with ``bare``, model numbers
    from ``model_base``, every empty text field masked, gzip with ``gz``; ``coord``: (payload, encoding) per axis from
    the frames' (F * natoms,) values, in place of encode_fixed(x, 1000)"""
    doc = msgpack.unpackb(write(frames, topology, box, angles), raw=False)
    cats = doc["dataBlocks"][0]["categories"]
    site = cats[-1]
    cols = {c["name"]: c for c in site["columns"]}
    n, F = len(topology["name"]), len(frames)
    cols["pdbx_PDB_model_num"] = column("pdbx_PDB_model_num",
                                        encode_int(np.repeat(np.arange(model_base, model_base + F), n)))
    if coord is not None:
        xyz = np.asarray(frames, np.float32).reshape(F, n, 3)
        for d, c in enumerate(("Cartn_x", "Cartn_y", "Cartn_z")):
            cols[c] = column(c, coord(xyz[:, :, d].reshape(-1)))
    site["columns"] = [cols[k] for k in (order or TAGS)]
    extra = [{"name": "_entry", "columns": [column("id", encode_strings(["1ABC"])[0])], "rowCount": 1},
             {"name": "_struct", "columns": [column("title", encode_strings(["a test"])[0]),
                                             column("pdbx_descriptor", encode_strings(["x"])[0])], "rowCount": 1}]
    after = [{"name": "_atom_type", "columns": [column("symbol", encode_strings(["C", "N"])[0])], "rowCount": 2}]
    cats[:] = extra + cats + after
    if bare:
        for c in cats:
            c["name"] = c["name"].lstrip("_").upper()
    doc["dataBlocks"].append({"header": "second", "categories": [dict(after[0])]})
    raw = msgpack.packb(doc, use_bin_type=True)
    return gzip.compress(raw) if gz else raw
