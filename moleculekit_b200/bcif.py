"""Multi-model BinaryCIF trajectories read and written on the GPU (K31).

BinaryCIF (``.bcif``, often ``.bcif.gz``) is the ``_atom_site`` table of PDBx/mmCIF stored column by column in a
MessagePack document, each column an encoded byte array; the PDB serves every entry in it and Mol* reads and writes it.
Coordinates are fixed-point deltas packed into small integers, so an ensemble takes a fraction of its mmCIF size.
Decoding a column is a chain of prefix scans and encoding one is count passes, a scan and an emit pass, all on the
device (``mkb_bcif_decode``, ``mkb_bcif_quantize``, ``mkb_bcif_sizes``, ``mkb_bcif_emit``).  The MessagePack container
is read and written on the host with the ``msgpack`` package; strings are resolved on the host from frame 0's rows.
Names and return shapes mirror :mod:`moleculekit_b200.cif`, and a trajectory moves between the two forms unchanged.

Reader contract:

1. Container.  A MessagePack map ``{dataBlocks: [{header, categories: [{name, columns: [{name, data: {data, encoding},
   mask}], rowCount}]}]}``; a gzip file (magic 1f 8b) is decompressed first.  The first data block is read.  Category
   and column names compare case-insensitively, a category's leading ``_`` is optional, and ``_atom_site`` may be in
   any position.  A file that is not MessagePack of this shape raises ValueError naming the file.
2. Encodings: ByteArray, IntegerPacking, Delta, RunLength, FixedPoint, IntervalQuantization and StringArray, as the
   BinaryCIF specification states them; integers wrap modulo 2^32; a Float64 column is read as float32.  Another kind,
   a payload whose length is not a multiple of its type, a packing that ends inside a value, run counts or a packing
   that do not give srcSize values, or a column that decodes to another length than ``rowCount`` raises ValueError
   naming the file and the column.  A mask (0 a value, 1 ``.``, 2 ``?``) is decoded the same way.
3. Frames.  ``Cartn_x``, ``Cartn_y`` and ``Cartn_z`` are required and must decode to floats.  A frame is a maximal run of
   equal ``pdbx_PDB_model_num``; without that column the table is one frame.  Every frame holds frame 0's row count N,
   else ValueError naming the frame, its model number and its first row.  A masked coordinate anywhere in the table
   raises ValueError naming the file, frame, atom and column.
4. Topology, from frame 0's rows with ``pdb.FIELDS`` keys and :mod:`cif`'s mapping (``auth_*`` before ``label_*``); a
   masked or missing value reads as "" for text, 0 for numbers.
5. Cell.  The ``_cell`` category's length_a/b/c and angle_alpha/beta/gamma (row 0), repeated over every frame; without
   it the box is zeros and the angles 90.

The writer's file: ``{version, encoder, dataBlocks: [{header: title, categories}]}`` with, for a box, a one-row
``_cell`` and ``_symmetry`` (space group 'P 1'), then ``_atom_site`` with the 21 tags of :data:`cif.TAGS` in RCSB's
order, the rows of :func:`cif.write_cif` (id = f N + a + 1, pdbx_PDB_model_num = f + 1, label_entity_id ``.``).
Coordinates and cell lengths are FixedPoint(1000), occupancy, beta and cell angles FixedPoint(100), q = rint(x * factor)
half to even.  Every integer array (the quanta, integer columns, string indices and offsets, masks) takes the fewest
bytes of (a) IntegerPacking, (b) RunLength -> IntegerPacking, (c) Delta -> IntegerPacking and (d) Delta -> RunLength ->
IntegerPacking, ties to the earlier; the packing is unsigned without negative values, and none (ByteArray Int32) when
4 n < 2 size2, else 2 bytes when 2 size2 < size1, else 1 byte (size1, size2: the elements at 1 and 2 bytes).  Text
columns are StringArrays of the unique strings in order of first appearance, "" masked as ``.``.  Not supported:
writing gzip, categories other than ``_atom_site``, ``_cell`` and ``_symmetry``, per-model topology differences, and
columns that do not fit in device memory (a column is decoded whole: a delta needs every earlier row).
"""
from __future__ import annotations

import ctypes as C
import gzip

import numpy as np
import torch

from . import _lib, _trajio
from .cif import CELL, TAGS
from .pdb import FIELDS, topology_fields

TYPE_BYTES = {1: 1, 2: 2, 3: 4, 4: 1, 5: 2, 6: 4, 32: 4, 33: 8}
INT_TYPES = (1, 2, 3, 4, 5, 6)
K_BYTES, K_PACKING, K_DELTA, K_RUN_LENGTH, K_FIXED, K_INTERVAL = 1, 2, 3, 4, 5, 6
MODE_ROWS, MODE_FRAMES, MODE_RUNS = 0, 1, 2
MAX_LEN = 2**31 - 2  # values of one array on the device
INT32 = (-2**31, 2**31 - 1)
STATUS = {1: "an IntegerPacking ends inside a value", 2: "an IntegerPacking holds another number of values than its "
          "srcSize", 3: "the RunLength counts do not sum to its srcSize", 4: "a RunLength count is negative"}
CARTN = ("cartn_x", "cartn_y", "cartn_z")


def _msgpack():
    import msgpack  # only this module needs it

    return msgpack


def _err(fn, col, why) -> ValueError:
    return ValueError(f"BinaryCIF file {fn}, column {col}: {why}")


# ------------------------------------------------------------------------------------------------------------ reading
def _load(fn) -> dict:
    """the first data block's categories -> {normalised name: category}"""
    with open(fn, "rb") as f:
        raw = f.read()
    try:
        if raw[:2] == b"\x1f\x8b":
            raw = gzip.decompress(raw)
        doc = _msgpack().unpackb(raw, raw=False, strict_map_key=False)
    except Exception as e:
        raise ValueError(f"BinaryCIF file {fn}: not a (gzip) MessagePack document: {e}") from None
    try:
        cats = {}
        for c in doc["dataBlocks"][0]["categories"]:
            name = c["name"].lower()
            name = name[1:] if name.startswith("_") else name
            cols = {}
            for col in c["columns"]:
                if not isinstance(col["name"], str) or not isinstance(col["data"], dict):
                    raise TypeError
                cols[col["name"].lower()] = col
            if not isinstance(c["rowCount"], int) or c["rowCount"] < 0:
                raise TypeError
            cats.setdefault(name, dict(columns=cols, rows=c["rowCount"]))
    except (KeyError, IndexError, TypeError, AttributeError):
        raise ValueError(f"BinaryCIF file {fn}: not shaped as a BinaryCIF document (dataBlocks[0].categories with "
                         "name, columns and rowCount)") from None
    return cats


def _chain(fn, col: str, data, encoding) -> tuple:
    """(payload, steps float64 (k, 6) in decode order, decoded length, floats) of one encoded array; an encoding
    outside the supported kinds or a malformed step raises ValueError"""
    if not isinstance(data, (bytes, bytearray)) or not isinstance(encoding, list) or not encoding:
        raise _err(fn, col, "the data is not a byte array with an encoding list")
    enc = list(reversed(encoding))
    steps, m, floats = [], 0, False
    try:
        for j, e in enumerate(enc):
            k = e["kind"]
            if j == 0:
                if k != "ByteArray" or e["type"] not in TYPE_BYTES:
                    raise _err(fn, col, f"the last encoding is {k}, not a ByteArray of a known type")
                size = TYPE_BYTES[e["type"]]
                if len(data) % size:
                    raise _err(fn, col, f"{len(data)} bytes are not a whole number of {size}-byte values")
                steps.append([K_BYTES, e["type"], 0, 0, 0, 0])
                m, floats = len(data) // size, e["type"] >= 32
                continue
            if floats:
                raise _err(fn, col, f"a {k} encoding over floats")
            if k == "IntegerPacking":
                if e["byteCount"] not in (1, 2) or not 0 <= e["srcSize"]:
                    raise _err(fn, col, "IntegerPacking byteCount must be 1 or 2")
                if e["srcSize"] > m:
                    raise _err(fn, col, STATUS[2])
                steps.append([K_PACKING, e["byteCount"], 1 if e["isUnsigned"] else 0, e["srcSize"], 0, 0])
                m = e["srcSize"]
            elif k == "Delta":
                if e["srcType"] not in INT_TYPES:
                    raise _err(fn, col, "Delta srcType must be an integer type")
                steps.append([K_DELTA, int(e["origin"]), e["srcType"], 0, 0, 0])
            elif k == "RunLength":
                if e["srcType"] not in INT_TYPES or m % 2 or not 0 <= e["srcSize"] <= MAX_LEN:
                    raise _err(fn, col, "RunLength needs (value, count) pairs, an integer srcType and a srcSize")
                steps.append([K_RUN_LENGTH, e["srcType"], e["srcSize"], 0, 0, 0])
                m = e["srcSize"]
            elif k == "FixedPoint":
                if not float(e["factor"]):
                    raise _err(fn, col, "FixedPoint factor 0")
                steps.append([K_FIXED, float(e["factor"]), e.get("srcType", 32), 0, 0, 0])
                floats = True
            elif k == "IntervalQuantization":
                if not e["numSteps"] >= 2:
                    raise _err(fn, col, "IntervalQuantization numSteps must be at least 2")
                steps.append([K_INTERVAL, float(e["min"]), float(e["max"]), float(e["numSteps"]), 0, 0])
                floats = True
            else:
                raise _err(fn, col, f"the encoding kind {k!r} is not supported")
    except (KeyError, TypeError):
        raise _err(fn, col, f"a malformed encoding {e!r}") from None
    if m > MAX_LEN:
        raise _err(fn, col, f"{m} values, at most {MAX_LEN} are decoded")
    return bytes(data), np.asarray(steps, np.float64), m, floats


def _decode(dev, payload: bytes, steps, mode: int, out, n_out: int, frames=None, natoms: int = 0, atom_stride: int = 0):
    """one mkb_bcif_decode call -> status (device int64 (2,)); nothing is synchronised"""
    buf = torch.empty(max(16, (len(payload) + 15) & ~15), dtype=torch.uint8)
    buf[:len(payload)] = torch.frombuffer(bytearray(payload), dtype=torch.uint8) if payload else buf[:0]
    buf = buf.to(dev)
    status = torch.zeros(2, dtype=torch.int64, device=dev)
    steps = np.ascontiguousarray(steps, np.float64)
    fr = None if frames is None else np.ascontiguousarray(frames, np.int64)
    _lib.call(dev, "mkb_bcif_decode", _lib.ptr(buf), len(payload), steps.ctypes.data_as(C.c_void_p), len(steps), mode,
              _lib.ptr(out), int(n_out), None if fr is None else fr.ctypes.data_as(C.c_void_p), int(natoms),
              int(atom_stride), _lib.ptr(status))
    return status, (buf, steps, fr)


def _check(fn, col, status) -> np.ndarray:
    st = status.cpu().numpy()
    if st[0]:
        raise _err(fn, col, STATUS[int(st[0])])
    return st


def _array(fn, col: str, data: dict, rows: int, dev, n_out: int | None = None):
    """an encoded array (a column's data or mask) decoded on the device -> the first n_out values (numpy int32 or
    float32; a StringArray -> list of str)"""
    try:
        payload, encoding = data["data"], data["encoding"]
    except (KeyError, TypeError):
        raise _err(fn, col, "the data is not a {data, encoding} map") from None
    if isinstance(encoding, list) and len(encoding) == 1 and isinstance(encoding[0], dict) and \
            encoding[0].get("kind") == "StringArray":
        e = encoding[0]
        try:
            idx = _array(fn, col, dict(data=payload, encoding=e["dataEncoding"]), rows, dev, n_out)
            offs = dict(data=e["offsets"], encoding=e["offsetEncoding"])
            off = _array(fn, col, offs, None, dev)
            text = e["stringData"]
        except (KeyError, TypeError):
            raise _err(fn, col, "a malformed StringArray") from None
        strings = [text[int(off[j]):int(off[j + 1])] for j in range(len(off) - 1)]
        if len(idx) and (idx.min() < 0 or idx.max() >= len(strings)):
            raise _err(fn, col, "a string index outside the strings")
        return [strings[i] for i in idx.tolist()]
    payload, steps, m, floats = _chain(fn, col, payload, encoding)
    if rows is not None and m != rows:
        raise _err(fn, col, f"decodes to {m} values, the category has {rows} rows")
    n = m if n_out is None else min(n_out, m)
    out = torch.empty(max(n, 1), dtype=torch.float32 if floats else torch.int32, device=dev)
    status, keep = _decode(dev, payload, steps, MODE_ROWS, out, n)
    _check(fn, col, status)
    return out[:n].cpu().numpy()


def _runs(fn, col: str, data: dict, rows: int, dev) -> np.ndarray:
    """the runs of equal values of an integer array -> (R, 2) int64 (first row, value) in row order"""
    payload, steps, m, floats = _chain(fn, col, data.get("data"), data.get("encoding"))
    if m != rows:
        raise _err(fn, col, f"decodes to {m} values, the category has {rows} rows")
    if floats:
        raise _err(fn, col, "does not decode to integers")
    cap = 4096
    while True:
        out = torch.empty(2 * cap, dtype=torch.int64, device=dev)
        status, keep = _decode(dev, payload, steps, MODE_RUNS, out, cap)
        st = _check(fn, col, status)
        if st[1] <= cap:
            r = out[:2 * int(st[1])].view(-1, 2).cpu().numpy()
            return r[np.argsort(r[:, 0], kind="stable")]
        cap = int(st[1])


def _text(v, mask, n) -> np.ndarray:
    if v is None:
        return np.full(n, "", dtype=object)
    vals = v if isinstance(v, list) else [str(x) for x in v.tolist()]
    return np.array(["" if mask is not None and mask[i] else vals[i] for i in range(n)], dtype=object)


def _number(fn, col, v, mask, n, dtype, integer: bool) -> np.ndarray:
    out = np.zeros(n, dtype)
    if v is None:
        return out
    for i in range(n):
        if mask is not None and mask[i]:
            continue
        x = v[i]
        try:
            out[i] = (int(x) if integer else float(x)) if isinstance(x, str) else (int(x) if integer else x)
        except ValueError:
            raise _err(fn, col, f"row {i}: {x!r} is not {'an integer' if integer else 'a number'}") from None
    return out


def _topology(fn, cols: dict, rows: int, N: int, dev) -> dict:
    def pick(*names):
        for k in names:
            if k.lower() in cols:
                c = cols[k.lower()]
                v = _array(fn, c["name"], c["data"], rows, dev, N)
                m = _array(fn, c["name"] + " mask", c["mask"], rows, dev, N) if c.get("mask") else None
                return v, m, c["name"]
        return None, None, None

    def text(*names):
        v, m, _ = pick(*names)
        return _text(v, m, N)

    def number(dtype, integer, *names):
        v, m, name = pick(*names)
        return _number(fn, name, v, m, N, dtype, integer)

    return dict(record=text("group_PDB"), serial=number(np.int64, True, "id"),
                name=text("auth_atom_id", "label_atom_id"), altloc=text("label_alt_id"),
                resname=text("auth_comp_id", "label_comp_id"), chain=text("auth_asym_id", "label_asym_id"),
                resid=number(np.int64, True, "auth_seq_id", "label_seq_id"), insertion=text("pdbx_PDB_ins_code"),
                occupancy=number(np.float32, False, "occupancy"), beta=number(np.float32, False, "B_iso_or_equiv"),
                segid=text("label_asym_id"), element=text("type_symbol"),
                charge=number(np.float32, True, "pdbx_formal_charge"))


def index_bcif(filename, device=None) -> dict:
    """Read a BinaryCIF file's container and find its frames on the device -> dict(natoms, n_frames, model ((F,) int64:
    each frame's pdbx_PDB_model_num, 0 without the column), topology (frame 0's rows, ``pdb.FIELDS`` keys), box and
    boxangles ((3,) float32: the file's one cell), columns (the ``_atom_site`` columns by lower-case name, as read),
    rows (its rowCount)).  Errors: see the module docstring."""
    fn = _trajio.name(filename)
    cats = _load(fn)
    if "atom_site" not in cats:
        raise ValueError(f"BinaryCIF file {fn}: no _atom_site category in the first data block")
    site = cats["atom_site"]
    cols, rows = site["columns"], site["rows"]
    for c in CARTN:
        if c not in cols:
            raise ValueError(f"BinaryCIF file {fn}: the _atom_site category has no Cartn_{c[-1]} column")
    if rows == 0:
        raise ValueError(f"BinaryCIF file {fn}: the _atom_site category holds no rows")
    dev = _lib.device(device)
    if "pdbx_pdb_model_num" in cols:
        c = cols["pdbx_pdb_model_num"]
        r = _runs(fn, c["name"], c["data"], rows, dev)
        start, model = r[:, 0], r[:, 1]
    else:
        start, model = np.zeros(1, np.int64), np.zeros(1, np.int64)
    count = np.diff(np.append(start, rows))
    N, F = int(count[0]), len(count)
    bad = np.flatnonzero(count != N)
    if len(bad):
        f = int(bad[0])
        raise ValueError(f"BinaryCIF file {fn}, frame {f} (model {int(model[f])}, row {int(start[f])}): {int(count[f])} "
                         f"rows, frame 0 has {N} (every model must hold the same atoms)")
    topology = _topology(fn, cols, rows, N, dev)
    box, angles = np.zeros(3, np.float32), np.full(3, 90.0, np.float32)
    if "cell" in cats:
        cc, crow = cats["cell"]["columns"], cats["cell"]["rows"]
        for j, k in enumerate(CELL):
            if k in cc and crow:
                v = _array(fn, cc[k]["name"], cc[k]["data"], crow, dev, 1)
                (box if j < 3 else angles)[j % 3] = float(v[0])
    return dict(natoms=N, n_frames=F, model=model.astype(np.int64), topology=topology, box=box, boxangles=angles,
                columns=cols, rows=rows)


def decode_bcif_device(data: dict, rows: int | None = None, device=None) -> torch.Tensor:
    """K31 on the device: one encoded array ``data`` ({"data": bytes, "encoding": [...]}, a column's data or mask, not a
    StringArray) -> CUDA tensor of its values in row order (int32, or float32 after a float ByteArray, FixedPoint or
    IntervalQuantization).  ``rows``: the length it must decode to.  Errors raise ValueError."""
    dev = _lib.device(device)
    payload, steps, m, floats = _chain("<memory>", "<array>", data.get("data"), data.get("encoding"))
    if rows is not None and m != rows:
        raise _err("<memory>", "<array>", f"decodes to {m} values, expected {rows}")
    out = torch.empty(max(m, 1), dtype=torch.float32 if floats else torch.int32, device=dev)
    status, keep = _decode(dev, payload, steps, MODE_ROWS, out, m)
    _check("<memory>", "<array>", status)
    return out[:m]


def _read(filename, frames, index, device):
    fn = _trajio.name(filename)
    idx = index if index is not None else index_bcif(fn, device)
    N, F, rows = int(idx["natoms"]), int(idx["n_frames"]), int(idx["rows"])
    sel = _trajio.select(F, frames)
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((N, 3, n), dtype=torch.float32, device=dev)
    for d, c in enumerate(CARTN):
        col = idx["columns"][c]
        name = col["name"]
        if col.get("mask"):
            r = _runs(fn, name + " mask", col["mask"], rows, dev)
            hit = np.flatnonzero(r[:, 1] != 0)
            if len(hit):
                row = int(r[hit[0], 0])
                raise ValueError(f"BinaryCIF file {fn}, frame {row // N}, atom {row % N}, column {name}: a masked "
                                 "('.' or '?') coordinate; every atom needs coordinates")
        payload, steps, m, floats = _chain(fn, name, col["data"].get("data"), col["data"].get("encoding"))
        if m != rows:
            raise _err(fn, name, f"decodes to {m} values, the category has {rows} rows")
        if not floats:
            raise _err(fn, name, "a coordinate column that does not decode to floats")
        if n:
            out = coords[:, d, :]
            status, keep = _decode(dev, payload, steps, MODE_FRAMES, out, n, sel, N, out.stride(0))
            _check(fn, name, status)
    info = dict(natoms=N, n_frames=F, frames=sel, topology=idx["topology"],
                box=np.repeat(np.asarray(idx["box"], np.float32).reshape(3, 1), n, axis=1),
                boxangles=np.repeat(np.asarray(idx["boxangles"], np.float32).reshape(3, 1), n, axis=1),
                model=np.asarray(idx["model"], np.int64)[sel])
    return coords, info


def read_bcif_device(filename, frames=None, index: dict | None = None, device=None):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    (coords CUDA (natoms, 3, F) float32 [Angstrom], info) with the trajectory left on the GPU.  ``index`` (what
    :func:`index_bcif` returned for this file) skips reading the file again.  ``info`` holds natoms, n_frames, frames,
    box and boxangles ((3, F) float32), topology and model, as :func:`cif.read_cif_device`'s."""
    return _read(filename, frames, index, device)


def read_bcif(filename, index: dict | None = None, device=None):
    """Every frame -> (coords (natoms, 3, F) float32 numpy [Angstrom], info as :func:`read_bcif_device`)."""
    coords, info = _read(filename, None, index, device)
    return coords.cpu().numpy(), info


def read_bcif_frames(filename, frames, index: dict | None = None, device=None):
    """:func:`read_bcif` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, info = _read(filename, frames, index, device)
    return coords.cpu().numpy(), info


# ------------------------------------------------------------------------------------------------------------ writing
def _encode_ints(v: torch.Tensor, n: int, step: int = 0) -> tuple:
    """K31's classifier and encoder over the int32 CUDA array ``v`` repeated to n values (value i = v[i % len(v)] +
    (i // len(v)) * step) -> (payload bytes, encoding list)"""
    dev = v.device
    period = int(v.numel())
    sizes = (C.c_int64 * 25)()
    _lib.call(dev, "mkb_bcif_sizes", _lib.ptr(v), period, int(step), int(n), sizes)
    best = None
    for c in range(4):
        ln, mn, s1u, s2u, s1s, s2s = sizes[1 + 6 * c: 7 + 6 * c]
        u = mn >= 0
        s1, s2 = (s1u, s2u) if u else (s1s, s2s)
        w, nb = (4, 4 * ln) if 4 * ln < 2 * s2 else (2, 2 * s2) if 2 * s2 < s1 else (1, s1)
        if best is None or nb < best[0]:
            best = (nb, c, w, u, ln)
    nb, c, w, u, ln = best
    out = torch.empty(max(4, (nb + 3) & ~3), dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_bcif_emit", _lib.ptr(v), period, int(step), int(n), c, w, int(u), int(ln), _lib.ptr(out), nb)
    if w == 4:
        pack = [{"kind": "ByteArray", "type": 3}]
    else:
        pack = [{"kind": "IntegerPacking", "byteCount": w, "isUnsigned": bool(u), "srcSize": int(ln)},
                {"kind": "ByteArray", "type": {(1, False): 1, (2, False): 2, (1, True): 4, (2, True): 5}[(w, bool(u))]}]
    rl = {"kind": "RunLength", "srcType": 3, "srcSize": int(n)}
    de = {"kind": "Delta", "origin": int(sizes[0]), "srcType": 3}
    pre = ([], [rl], [de], [de, rl])[c]
    return out[:nb].cpu().numpy().tobytes(), pre + pack


def encode_bcif_device(values: torch.Tensor, factor: int | None = None) -> tuple:
    """K31 on the device: one 1-D CUDA array -> (encoding list, payload uint8 CUDA tensor) as the writer encodes it:
    int32 ``values`` with the classifier's chain, or float32 ``values`` with ``factor`` as FixedPoint(factor) of
    q = rint(x * factor) (finite, q inside int32: checked)."""
    dev = _lib.tensor_device(values, "encode_bcif_device")
    if values.ndim != 1 or values.numel() == 0 or values.numel() > MAX_LEN:
        raise ValueError(f"values must be a 1-D array of 1 to {MAX_LEN} values, got {tuple(values.shape)}")
    if factor is None:
        if values.dtype != torch.int32:
            raise ValueError("integer values must be int32; floats need a factor")
        data, enc = _encode_ints(values.contiguous(), values.numel())
    else:
        x = values.to(torch.float32)
        bad = _trajio.first_bad(x.reshape(1, 1, -1), *INT32, factor)
        if bad is not None:
            raise ValueError(f"values[{bad[0]}] = {bad[3]!r}: rint(x * {factor}) must be a finite int32")
        q = torch.empty(x.numel(), dtype=torch.int32, device=dev)
        _lib.call(dev, "mkb_bcif_quantize", _lib.ptr(x), 1, 0, x.numel(), 1, float(factor), _lib.ptr(q))
        data, enc = _encode_ints(q, q.numel())
        enc = [{"kind": "FixedPoint", "factor": factor, "srcType": 32}] + enc
    return enc, torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev) if data else \
        torch.empty(0, dtype=torch.uint8, device=dev)


def _strings(vals, n_rows: int, dev) -> tuple:
    """(column data, mask or None) of a text column repeated to n_rows from the per-atom ``vals``"""
    uniq = {}
    for s in vals:
        uniq.setdefault(s, len(uniq))
    strings = list(uniq)
    off = np.zeros(len(strings) + 1, np.int32)
    off[1:] = np.cumsum([len(s) for s in strings])
    idx = torch.tensor([uniq[s] for s in vals], dtype=torch.int32, device=dev)
    idata, ienc = _encode_ints(idx, n_rows)
    odata, oenc = _encode_ints(torch.from_numpy(off).to(dev), len(off))
    data = {"data": idata, "encoding": [{"kind": "StringArray", "dataEncoding": ienc, "stringData": "".join(strings),
                                         "offsetEncoding": oenc, "offsets": odata}]}
    mask = None
    if "" in uniq:
        m = torch.tensor([1 if s == "" else 0 for s in vals], dtype=torch.int32, device=dev)
        mdata, menc = _encode_ints(m, n_rows)
        mask = {"data": mdata, "encoding": menc}
    return data, mask


def _column(name, data_enc, mask=None) -> dict:
    data = {"data": data_enc[0], "encoding": data_enc[1]} if isinstance(data_enc, tuple) else data_enc
    return {"name": name, "data": data, "mask": mask}


def _quanta(v, factor) -> tuple:
    """host values -> (quanta rint(float64(x) * factor), whether each is finite and inside int32)"""
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.rint(np.asarray(v, np.float64) * factor)
    ok = np.isfinite(q) & (q >= INT32[0]) & (q <= INT32[1])
    return q, ok


def _prepare(coords, topology, box, boxangles, title, device):
    """every check -> (coords on the device, natoms, F, topology fields, cell values or None, title)"""
    coords = _trajio.writer_coords(coords, "write_bcif")
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if natoms < 1 or F < 1 or natoms * F > 2**31 - 1:
        raise ValueError(f"a BinaryCIF file written here holds 1 or more atoms and frames with natoms * F < 2^31 (id is "
                         f"an int32), got {natoms} atoms x {F} frames")
    title = "trajectory" if title is None else title
    if not isinstance(title, str) or not title:
        raise ValueError(f"title must be a non-empty string (it names the data block), got {title!r}")
    if box is None and boxangles is not None:
        raise ValueError("boxangles needs a box")
    cell = []
    for name, v in (("box", box), ("boxangles", boxangles)):
        if v is None:
            cell.append(None)
            continue
        v = _trajio.host(v).astype(np.float32)
        if v.shape != (3, F):
            raise ValueError(f"{name} must be (3, F) = {(3, F)}, got {tuple(v.shape)}")
        cell.append(v)
    box, angles = cell
    if box is not None and angles is None:
        angles = np.full((3, F), 90.0, np.float32)
    t = topology_fields(topology, natoms)
    bad = []
    for k in ("record", "name", "altloc", "resname", "chain", "insertion", "segid", "element"):
        vals = t[k].tolist()
        for a, s in enumerate(vals):
            if not isinstance(s, str) or not s.isascii():
                bad.append((a, k, f"{s!r}: an ASCII string"))
                break
    for k in ("resid", "charge"):
        v = t[k].astype(np.float64)
        with np.errstate(invalid="ignore"):
            hit = np.flatnonzero(~(np.isfinite(v) & (v == np.round(v)) & (v >= INT32[0]) & (v <= INT32[1])))
        if len(hit):
            bad.append((int(hit[0]), k, f"{t[k].tolist()[hit[0]]!r}: an int32 integer"))
    for k in ("occupancy", "beta"):
        _, ok = _quanta(t[k], 100)
        if not ok.all():
            a = int(np.argmin(ok))
            bad.append((a, k, f"{t[k].tolist()[a]!r}: finite with rint(x * 100) inside int32"))
    if bad:
        a, k, why = min(bad)
        raise ValueError(f"topology at atom {a}, field {k} is {why}")
    b = _trajio.first_bad(coords, *INT32, 1000)
    if b is not None:
        f, atom, axis, v = b
        raise ValueError(f"coords at frame {f}, atom {atom}, axis {'xyz'[axis]} is {v!r}: FixedPoint(1000) holds "
                         "finite values with rint(x * 1000) inside int32")
    values = None
    if box is not None:
        for name, v, factor in (("box", box, 1000), ("boxangles", angles, 100)):
            _, ok = _quanta(v, factor)
            if not ok.all():
                f, axis = np.unravel_index(np.argmax(~ok.T), (F, 3))
                raise ValueError(f"{name} at frame {f}, axis {'abc'[axis]} is {v[axis, f]!r}: not finite, or "
                                 f"rint(x * {factor}) outside int32")
        same = (box == box[:, :1]).all(axis=0) & (angles == angles[:, :1]).all(axis=0)
        if not same.all():
            f = int(np.argmin(same))
            raise ValueError(f"the box of frame {f} differs from frame 0's: a BinaryCIF data block holds one cell")
        values = [*box[:, 0], *angles[:, 0]]
    return _trajio.on_device(coords, device), natoms, F, t, values, title


def bcif_bytes(coords, topology, box=None, boxangles=None, title=None, device=None) -> bytes:
    """The file :func:`write_bcif` writes, as a ``bytes`` object."""
    x, N, F, t, cell, title = _prepare(coords, topology, box, boxangles, title, device)
    dev = x.device
    n = N * F

    def text(name, key):
        return _column(name, *_strings(t[key].tolist() if key else [""] * N, n, dev))

    def ints(name, v, step=0):
        return _column(name, _encode_ints(torch.as_tensor(np.asarray(v, np.int64).astype(np.int32)).to(dev), n, step))

    def fixed(name, v, factor, rows):
        q, _ = _quanta(v, factor)
        data, enc = _encode_ints(torch.from_numpy(q.astype(np.int32)).to(dev), rows)
        return _column(name, (data, [{"kind": "FixedPoint", "factor": factor, "srcType": 32}] + enc))

    resid = t["resid"].astype(np.float64).astype(np.int64)
    cols = {"group_PDB": text("group_PDB", "record"), "id": ints("id", np.arange(1, N + 1), N),
            "type_symbol": text("type_symbol", "element"), "label_atom_id": text("label_atom_id", "name"),
            "label_alt_id": text("label_alt_id", "altloc"), "label_comp_id": text("label_comp_id", "resname"),
            "label_asym_id": text("label_asym_id", "segid"), "label_entity_id": text("label_entity_id", None),
            "label_seq_id": ints("label_seq_id", resid), "pdbx_PDB_ins_code": text("pdbx_PDB_ins_code", "insertion"),
            "occupancy": fixed("occupancy", t["occupancy"], 100, n),
            "B_iso_or_equiv": fixed("B_iso_or_equiv", t["beta"], 100, n),
            "pdbx_formal_charge": ints("pdbx_formal_charge", t["charge"].astype(np.float64).astype(np.int64)),
            "auth_seq_id": ints("auth_seq_id", resid), "auth_comp_id": text("auth_comp_id", "resname"),
            "auth_asym_id": text("auth_asym_id", "chain"), "auth_atom_id": text("auth_atom_id", "name"),
            "pdbx_PDB_model_num": ints("pdbx_PDB_model_num", np.ones(N), 1)}
    xf = _trajio.frame_minor(x)
    q = torch.empty(n, dtype=torch.int32, device=dev)
    for d, c in enumerate(("Cartn_x", "Cartn_y", "Cartn_z")):
        v = xf[:, d, :]
        _lib.call(dev, "mkb_bcif_quantize", _lib.ptr(v), int(v.stride(0)), int(v.stride(1)), N, F, 1000.0, _lib.ptr(q))
        data, enc = _encode_ints(q, n)
        cols[c] = _column(c, (data, [{"kind": "FixedPoint", "factor": 1000, "srcType": 32}] + enc))
    cats = []
    if cell is not None:
        cats.append({"name": "_cell", "columns": [fixed(k, [v], 1000 if k.startswith("length") else 100, 1)
                                                  for k, v in zip(CELL, cell)], "rowCount": 1})
        cats.append({"name": "_symmetry", "columns": [_column("space_group_name_H-M", *_strings(["P 1"], 1, dev))],
                     "rowCount": 1})
    cats.append({"name": "_atom_site", "columns": [cols[k] for k in TAGS], "rowCount": n})
    doc = {"version": "0.3.0", "encoder": "moleculekit_b200", "dataBlocks": [{"header": title, "categories": cats}]}
    return _msgpack().packb(doc, use_bin_type=True)


def write_bcif(filename, coords, topology, box=None, boxangles=None, title=None, device=None) -> None:
    """Write a multi-model BinaryCIF file with every column encoded on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is).  ``topology``, ``box``,
    ``boxangles`` and ``title`` as :func:`cif.write_cif`'s.  Checked before the file is opened, each failure a
    ValueError naming the first frame, atom and field: at least one atom and frame, natoms * F < 2^31; coords finite
    with rint(x * 1000) inside int32; box and angles likewise (1000, 100) and equal in every frame; text ASCII strings;
    resid and charge int32 integers; occupancy and beta finite with rint(x * 100) inside int32.  The layout is in the
    module docstring.  The file is created or truncated."""
    fn = _trajio.name(filename)
    raw = bcif_bytes(coords, topology, box, boxangles, title, device)
    with open(fn, "wb") as fh:
        fh.write(raw)


__all__ = ["index_bcif", "read_bcif", "read_bcif_frames", "read_bcif_device", "decode_bcif_device", "write_bcif",
           "bcif_bytes", "encode_bcif_device", "FIELDS", "TAGS"]
