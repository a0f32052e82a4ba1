"""AMBER NetCDF trajectories read and written on the GPU (K23).

AMBER's default trajectory format is netCDF-3 (classic CDF-1 or 64-bit offset CDF-2) under the AMBER convention 1.0:
every frame is one record holding ``time``, ``coordinates`` (frame, atom, spatial) as big-endian float32 and, with a
box, ``cell_lengths`` / ``cell_angles`` as float64 (plus optional ``velocities``, ``forces``, ``remd_*``).  The host
parses the header (``index_netcdf``) and reads the small per-frame variables through strided views of the mapped file;
only the coordinate slabs of the listed frames travel to the device, where ``mkb_netcdf_decode`` byte-swaps and
transposes them into the frame-minor ``(natoms, 3, F)`` layout the other kernels consume.  ``mkb_netcdf_encode`` is the
same transposition the other way round and writes finished records.  Coordinates move as 32-bit words: bit-identical in
both directions, NaN payloads, signalling NaNs and -0.0 included.

Reading gathers the listed frames' slabs into two pinned staging buffers of at most ``chunk_bytes`` (one ``preadv``
per run of up to 512 nearby slabs, the bytes between them going to a scratch buffer) and decodes one chunk while the
other fills: only coordinate bytes cross PCIe, and the device holds the output plus two chunks.  Writing builds the header on the host, encodes chunk by chunk and writes each while the next encodes.
The writer lays the file out as ``scipy.io.netcdf_file`` does for the same definitions (non-record variables first,
larger shapes first, then the record variables in definition order), byte for byte.

Not supported (rejected with an error naming them): netCDF-4/HDF5 and CDF-5 files, AMBER restart files
(``AMBERRESTART``: non-record double coordinates), double-precision coordinates.  ``velocities``, ``forces`` and other
record variables are skipped through the record layout, never read.

Not confirmed against moleculekit (its NetCDF sources and a file written by AMBER were not at hand):

- the names and signatures of moleculekit's NetCDF reader, and whether it writes NetCDF at all (``read_netcdf`` /
  ``write_netcdf`` here follow the XTC and DCD modules' shape);
- whether ``Molecule.time`` is the file's ``time`` (ps) times 1000 (here ``info["time"]`` is the file's value in ps);
- the box it gives a file without cell variables (here the DCD module's defaults: zeros, angles 90);
- how it handles a truncated file or ``numrecs`` = STREAMING (here: the whole records present are read, a partial
  record is dropped with a warning, and STREAMING takes the count from the file size);
- the AMBER writer's exact attribute and variable order: ours is restated from the published convention, not from
  AMBER's source or a file AMBER wrote.
"""
from __future__ import annotations

import ctypes as C
import io
import logging
import os
import struct

import numpy as np
import torch

from . import __version__, _lib, _trajio

logger = logging.getLogger(__name__)

NC_DIMENSION, NC_VARIABLE, NC_ATTRIBUTE = 10, 11, 12
NC_BYTE, NC_CHAR, NC_SHORT, NC_INT, NC_FLOAT, NC_DOUBLE = 1, 2, 3, 4, 5, 6
NC_DTYPE = {NC_BYTE: "i1", NC_CHAR: "S1", NC_SHORT: ">i2", NC_INT: ">i4", NC_FLOAT: ">f4", NC_DOUBLE: ">f8"}
STREAMING = 0xFFFFFFFF  # numrecs of a file still being written: the count comes from the file size
MAX_ATOMS = (2**31 - 1) // 12  # a coordinate slab of 12 * natoms bytes must fit a 32-bit vsize
MAX_FRAMES = 2**31 - 1  # numrecs is a non-negative int32 in a classic file
DEFAULT_TITLE = "written by moleculekit_b200"
CHUNK_BYTES = 256 << 20
# the host-built part of a record, in file byte order: time, then (with a box) cell_lengths and cell_angles
EXTRA_BOX = np.dtype([("time", ">f4"), ("lengths", ">f8", (3,)), ("angles", ">f8", (3,))], align=False)
EXTRA_NOBOX = np.dtype([("time", ">f4")])
assert EXTRA_BOX.itemsize == 52 and EXTRA_NOBOX.itemsize == 4


def _malformed(msg):
    return RuntimeError(f"Malformed NetCDF file: {msg}")


def _pad4(n: int) -> int:
    return n + (-n % 4)


class _Cursor:
    """Big-endian reader over the header bytes; running out of bytes raises EOFError."""

    def __init__(self, b, version: int):
        self.b, self.pos, self.version = b, 4, version

    def take(self, n: int) -> bytes:
        if n < 0 or self.pos + n > len(self.b):
            raise EOFError
        out = bytes(self.b[self.pos:self.pos + n])
        self.pos += n
        return out

    def int32(self) -> int:
        return struct.unpack(">i", self.take(4))[0]

    def uint32(self) -> int:
        return struct.unpack(">I", self.take(4))[0]

    def begin(self) -> int:
        return struct.unpack(">i" if self.version == 1 else ">q", self.take(4 if self.version == 1 else 8))[0]

    def name(self) -> str:
        n = self.int32()
        s = self.take(n)
        self.take(-n % 4)
        return s.decode("latin-1")

    def list_header(self, tag: int, what: str) -> int:
        t, n = self.int32(), self.int32()
        if t not in (0, tag) or n < 0 or (t == 0 and n != 0):
            raise _malformed(f"bad {what} list header (tag {t}, {n} entries)")
        return n

    def attributes(self) -> dict:
        out = {}
        for _ in range(self.list_header(NC_ATTRIBUTE, "attribute")):
            name = self.name()
            t, n = self.int32(), self.int32()
            if t not in NC_DTYPE or n < 0:
                raise _malformed(f"attribute {name!r} has type {t} and {n} values")
            size = np.dtype(NC_DTYPE[t]).itemsize
            raw = self.take(n * size)
            self.take(-(n * size) % 4)
            out[name] = raw.rstrip(b"\x00").decode("latin-1") if t == NC_CHAR else np.frombuffer(raw, NC_DTYPE[t])
        return out


def _parse(b) -> dict:
    """The header of a netCDF-3 byte buffer: version, numrecs, dims [(name, length)], globals, variables (name ->
    dict(dims, type, shape, slab, vsize, begin, record)), header_end.  Structure only; sizes and offsets are checked by
    index_netcdf."""
    head = bytes(b[:4])
    if head.startswith(b"\x89HDF"):
        raise ValueError("netCDF-4 / HDF5 files are not supported: only netCDF-3 (CDF-1, CDF-2) AMBER trajectories")
    if head == b"CDF\x05":
        raise ValueError("CDF-5 (64-bit data) netCDF files are not supported: only netCDF-3 (CDF-1, CDF-2)")
    if len(head) < 4 or head[:3] != b"CDF" or head[3] not in (1, 2):
        raise _malformed("the file does not start with the netCDF-3 magic CDF\\x01 or CDF\\x02")
    cur = _Cursor(b, head[3])
    try:
        numrecs = cur.uint32()
        dims = []
        for _ in range(cur.list_header(NC_DIMENSION, "dimension")):
            name, length = cur.name(), cur.int32()
            if length < 0:
                raise _malformed(f"dimension {name!r} has length {length}")
            dims.append((name, length))
        if sum(1 for _, n in dims if n == 0) > 1:
            raise _malformed("more than one unlimited (record) dimension")
        gatts = cur.attributes()
        variables = {}
        for _ in range(cur.list_header(NC_VARIABLE, "variable")):
            name = cur.name()
            nd = cur.int32()
            if nd < 0:
                raise _malformed(f"variable {name!r} has {nd} dimensions")
            ids = [cur.int32() for _ in range(nd)]
            if any(not 0 <= i < len(dims) for i in ids):
                raise _malformed(f"variable {name!r} refers to a dimension that does not exist")
            atts = cur.attributes()
            t, vsize, begin = cur.int32(), cur.uint32(), cur.begin()
            if t not in NC_DTYPE:
                raise _malformed(f"variable {name!r} has type {t}")
            shape = [dims[i][1] for i in ids]
            if 0 in shape[1:]:
                raise _malformed(f"variable {name!r}: only its first dimension may be the record dimension")
            record = bool(shape) and shape[0] == 0
            slab = int(np.prod(shape[1:] if record else shape, dtype=np.int64)) * np.dtype(NC_DTYPE[t]).itemsize
            variables[name] = dict(dims=[dims[i][0] for i in ids], type=t, shape=shape, slab=slab, vsize=vsize,
                                   begin=begin, record=record, attributes=atts)
    except (EOFError, struct.error):
        raise _malformed("the header is truncated") from None
    return dict(version=head[3], numrecs=numrecs, dims=dims, attributes=gatts, variables=variables, header_end=cur.pos)


def index_netcdf(buf) -> dict:
    """Parse an AMBER NetCDF trajectory in a byte buffer (bytes, memoryview or a read-only np.memmap of the file).

    Returns dict(natoms, n_frames, numrecs (the header's count; -1 for STREAMING), version (1 or 2), recsize,
    record_start (the first record's byte offset), begin (frame 0's coordinate bytes; frame k's are at
    begin + k * recsize), time ((F,) float32 ps, zeros without a ``time`` variable), box / boxangles ((3, F) float32 from
    ``cell_lengths`` / ``cell_angles`` rounded from float64; zeros and 90 without them), title / application / program /
    programVersion / Conventions / ConventionVersion (str or None), attributes (every global attribute), variables
    (names in header order)).  The frame count is numrecs capped by the whole records present; a partial record, or a
    numrecs larger than the data, is dropped with a warning."""
    b = np.frombuffer(buf, dtype=np.uint8)
    h = _parse(b)
    n = len(b)
    V = h["variables"]
    rec = [v for v in V.values() if v["record"]]
    for name, v in V.items():
        padded = _pad4(v["slab"])
        ok = (padded, v["slab"]) + ((0xFFFFFFFF,) if padded >= 2**32 - 4 else ()) + \
            ((0,) if v["record"] and h["numrecs"] == 0 else ())  # scipy writes 0 for the record variables of an empty file
        if v["vsize"] not in ok:
            raise _malformed(f"variable {name!r}: vsize {v['vsize']} in the header, {padded} from its shape and type")
    # one record variable: its slabs follow each other unpadded; more: each is padded to 4 bytes
    recsize = rec[0]["slab"] if len(rec) == 1 else sum(_pad4(v["slab"]) for v in rec)
    record_start = min((v["begin"] for v in rec), default=n)
    for name, v in V.items():
        # a record variable's data may lie past the end of the file: the frame count below covers what is present
        if v["begin"] < h["header_end"] or (not v["record"] and v["begin"] + v["slab"] > n):
            raise _malformed(f"variable {name!r} of {v['slab']} bytes begins at {v['begin']}, outside the file's data "
                             f"({h['header_end']}..{n})")
    for name, v in V.items():
        if v["record"] and v["begin"] - record_start + v["slab"] > recsize:
            raise _malformed(f"record variable {name!r} at {v['begin']} does not fit the record of {recsize} bytes "
                             f"from {record_start}")

    c = V.get("coordinates")
    if c is None:
        raise ValueError("the NetCDF file has no 'coordinates' variable: it is not an AMBER trajectory")
    if not c["record"]:
        raise ValueError("'coordinates' is not a record variable (frame, atom, spatial): an AMBER restart file "
                         f"(Conventions {h['attributes'].get('Conventions')!r}; AMBERRESTART) holds one frame and is "
                         "not supported, only AMBER trajectories")
    if c["type"] != NC_FLOAT:
        raise ValueError(f"'coordinates' has netCDF type {c['type']}: only NC_FLOAT ({NC_FLOAT}) coordinates are "
                         "supported")
    if len(c["shape"]) != 3 or c["shape"][2] != 3:
        raise ValueError(f"'coordinates' has dimensions {c['dims']}: expected (frame, atom, spatial = 3)")
    natoms = c["shape"][1]

    present = max(0, (n - record_start) // recsize) if recsize else 0
    numrecs = h["numrecs"]
    if numrecs == STREAMING:
        F = present
        rest = n - record_start - F * recsize
        if rest > 0:
            logger.warning("NetCDF file (numrecs STREAMING): %d trailing bytes after %d whole records are dropped",
                           rest, F)
    else:
        F = min(numrecs, present)
        if numrecs > present:
            logger.warning("NetCDF file: numrecs is %d but the file holds %d whole records; the rest is dropped",
                           numrecs, present)

    def per_frame(name, cols, types=(NC_FLOAT, NC_DOUBLE)):
        v = V.get(name)
        if v is None:
            return None
        if not v["record"] or v["type"] not in types or v["shape"][1:] != ([cols] if cols else []):
            raise ValueError(f"{name!r} has dimensions {v['dims']} and netCDF type {v['type']}: expected a float or "
                             f"double record variable{f' of {cols} values' if cols else ''}")
        dt = np.dtype(NC_DTYPE[v["type"]])
        if F == 0:
            return np.zeros((0, cols or 1), np.float32)
        view = np.ndarray((F, cols or 1), dtype=dt, buffer=b, offset=v["begin"], strides=(recsize, dt.itemsize))
        return view.astype(np.float32)

    t = per_frame("time", 0)
    lengths = per_frame("cell_lengths", 3)
    angles = per_frame("cell_angles", 3)
    g = h["attributes"]

    def text(key):
        val = g.get(key)
        return val if isinstance(val, str) else None

    return dict(natoms=int(natoms), n_frames=int(F), numrecs=-1 if numrecs == STREAMING else int(numrecs),
                version=int(h["version"]), recsize=int(recsize), record_start=int(record_start),
                begin=int(c["begin"]),
                time=np.zeros(F, np.float32) if t is None else np.ascontiguousarray(t[:, 0]),
                box=np.zeros((3, F), np.float32) if lengths is None else np.ascontiguousarray(lengths.T),
                boxangles=np.full((3, F), 90, np.float32) if angles is None else np.ascontiguousarray(angles.T),
                title=text("title"), application=text("application"), program=text("program"),
                programVersion=text("programVersion"), Conventions=text("Conventions"),
                ConventionVersion=text("ConventionVersion"), attributes=g, variables=list(V))


def decode_netcdf_device(buf: torch.Tensor, offsets, natoms: int, out: torch.Tensor | None = None) -> torch.Tensor:
    """K23 on the device: ``buf`` (uint8 CUDA tensor of staged file bytes), ``offsets`` (int64 per listed frame: the byte
    offset in ``buf`` of its 12 * natoms big-endian coordinate bytes) -> coords (natoms, 3, len(offsets)) float32.
    ``out`` may be a frame slice of a larger (natoms, 3, F) tensor."""
    dev = _lib.tensor_device(buf, "decode_netcdf_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    offsets = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    F = int(offsets.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    if F == 0 or natoms == 0:
        return out
    _lib.call(dev, "mkb_netcdf_decode", _lib.ptr(buf), int(buf.numel()), offsets.ctypes.data_as(C.c_void_p), F,
              int(natoms), _lib.ptr(out), stride)
    return out


def read_netcdf_device(filename, frames=None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Whole file (or the frames listed: any order, repeats allowed; out of range raises IndexError) -> (coords CUDA
    (natoms, 3, F) float32 [Angstrom], box (3, F) float32, boxangles (3, F) float32, info dict) with the trajectory left
    on the GPU.  ``info`` holds natoms, n_frames (the frames present in the file), numrecs, version, time (the listed
    frames' ``time`` in ps) and the global attributes title / application / program / programVersion / Conventions /
    ConventionVersion.  Only the listed frames' coordinate bytes are read and cross PCIe."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    if os.path.getsize(filename) == 0:
        raise _malformed("the file is empty")
    mm = np.memmap(filename, dtype=np.uint8, mode="r")
    idx = index_netcdf(mm)
    F, natoms = idx["n_frames"], idx["natoms"]
    sel = _trajio.select(F, frames)
    info = {k: idx[k] for k in ("natoms", "n_frames", "numrecs", "version", "title", "application", "program",
                                "programVersion", "Conventions", "ConventionVersion")}
    info["time"] = idx["time"][sel]
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((natoms, 3, n), dtype=torch.float32, device=dev)
    if n == 0:
        return coords, idx["box"][:, sel], idx["boxangles"][:, sel], info
    del mm  # the slabs are read with preadv: a copy from the page cache, without a page fault per 4 KiB
    slab = 12 * natoms
    chunks = _trajio.chunks(sel, np.full(F, slab, np.int64), int(chunk_bytes))
    with open(filename, "rb") as fh:
        def stage(c, host):
            uniq = chunks[c][2]
            used = len(uniq) * slab
            _trajio.gather_slabs(fh.fileno(), idx["begin"] + uniq * idx["recsize"], slab,
                                 host[:used].reshape(len(uniq), slab), "NetCDF")
            return used

        def consume(c, buf):
            k0, k1, uniq = chunks[c]
            decode_netcdf_device(buf, np.searchsorted(uniq, sel[k0:k1]) * slab, natoms, out=coords[:, :, k0:k1])

        _trajio.upload(dev, len(chunks), max(len(u) for _, _, u in chunks) * slab, stage, consume)
    return coords, idx["box"][:, sel], idx["boxangles"][:, sel], info


def read_netcdf(filename, device=None, chunk_bytes: int = CHUNK_BYTES):
    """(coords (natoms, 3, F) float32 [Angstrom], box (3, F), boxangles (3, F), info) as numpy arrays."""
    coords, box, angles, info = read_netcdf_device(filename, device=device, chunk_bytes=chunk_bytes)
    return coords.cpu().numpy(), box, angles, info


def read_netcdf_frames(filename, frames, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_netcdf` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, box, angles, info = read_netcdf_device(filename, frames=np.asarray(frames), device=device,
                                                   chunk_bytes=chunk_bytes)
    return coords.cpu().numpy(), box, angles, info


# ------------------------------------------------------------------------------------------------------------ writing
def _record_layout(natoms: int, with_box: bool) -> tuple[int, int]:
    """(record_bytes, coord_offset): time, coordinates, then with a box cell_lengths and cell_angles"""
    return 4 + 12 * natoms + (48 if with_box else 0), 4


def netcdf_header(natoms: int, n_frames: int, with_box: bool = False, title=None) -> bytes:
    """The bytes before the first record of the CDF-2 file :func:`write_netcdf` writes: the header and the non-record
    variables.  AMBER convention 1.0: dimensions frame (unlimited), spatial, atom and, with a box, cell_spatial, label,
    cell_angular; globals title, application, program, programVersion, Conventions = "AMBER", ConventionVersion = "1.0";
    variables spatial, time [picosecond], coordinates [angstrom] and, with a box, cell_spatial, cell_angular,
    cell_lengths [angstrom], cell_angles [degree].  In the file the non-record variables come first, larger shapes
    first, then the record variables in that order."""
    title = DEFAULT_TITLE if title is None else title
    dims = [("frame", 0), ("spatial", 3), ("atom", natoms)]
    if with_box:
        dims += [("cell_spatial", 3), ("label", 5), ("cell_angular", 3)]
    dim_id = {name: i for i, (name, _) in enumerate(dims)}
    gatts = [("title", title), ("application", "moleculekit_b200"), ("program", "moleculekit_b200"),
             ("programVersion", __version__), ("Conventions", "AMBER"), ("ConventionVersion", "1.0")]
    # (name, dims, units, type, data of a non-record variable / slab bytes of a record variable)
    nonrec = ([("cell_angular", ("cell_angular", "label"), None, NC_CHAR, b"alphabeta gamma")] if with_box else []) + \
        [("spatial", ("spatial",), None, NC_CHAR, b"xyz")] + \
        ([("cell_spatial", ("cell_spatial",), None, NC_CHAR, b"abc")] if with_box else [])
    recs = [("time", ("frame",), "picosecond", NC_FLOAT, 4),
            ("coordinates", ("frame", "atom", "spatial"), "angstrom", NC_FLOAT, 12 * natoms)]
    if with_box:
        recs += [("cell_lengths", ("frame", "cell_spatial"), "angstrom", NC_DOUBLE, 24),
                 ("cell_angles", ("frame", "cell_angular"), "degree", NC_DOUBLE, 24)]

    def name(s: str) -> bytes:
        raw = s.encode("ascii")
        return struct.pack(">i", len(raw)) + raw + b"\x00" * (-len(raw) % 4)

    def text_att(key: str, val: str) -> bytes:
        raw = val.encode("ascii")
        return name(key) + struct.pack(">ii", NC_CHAR, len(raw)) + raw + b"\x00" * (-len(raw) % 4)

    def header(begins) -> bytes:
        out = [b"CDF\x02", struct.pack(">i", n_frames), struct.pack(">ii", NC_DIMENSION, len(dims))]
        out += [name(d) + struct.pack(">i", n) for d, n in dims]
        out += [struct.pack(">ii", NC_ATTRIBUTE, len(gatts))] + [text_att(k, v) for k, v in gatts]
        out.append(struct.pack(">ii", NC_VARIABLE, len(nonrec) + len(recs)))
        for (vname, vdims, units, t, data), begin in zip(nonrec + recs, begins):
            size = len(data) if isinstance(data, bytes) else data
            out.append(name(vname) + struct.pack(">i", len(vdims)) + b"".join(struct.pack(">i", dim_id[d]) for d in vdims))
            out.append(struct.pack(">ii", NC_ATTRIBUTE, 1) + text_att("units", units) if units else b"\x00" * 8)
            out.append(struct.pack(">iiq", t, _pad4(size), begin))
        return b"".join(out)

    pos = len(header([0] * (len(nonrec) + len(recs))))
    begins = []
    for v in nonrec:
        begins.append(pos)
        pos += _pad4(len(v[4]))
    for v in recs:
        begins.append(pos)
        pos += _pad4(v[4])
    return header(begins) + b"".join(v[4] + b"\x00" * (-len(v[4]) % 4) for v in nonrec)


def _writer_args(coords, box, boxangles, time, title):
    """shapes and ranges checked before any device work; returns (natoms, F)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"a NetCDF trajectory holds 1 to {MAX_ATOMS} atoms (a dimension of length 0 would be the "
                         f"record dimension), got {natoms}")
    if F > MAX_FRAMES:
        raise ValueError(f"{F} frames do not fit the int32 record count of a netCDF-3 file")
    if box is None and boxangles is not None:
        raise ValueError("boxangles need a box")
    for name, v, shape in (("box", box, (3, F)), ("boxangles", boxangles, (3, F)), ("time", time, (F,))):
        if v is not None and tuple(v.shape) != shape:
            raise ValueError(f"{name} must be {shape}, got {tuple(v.shape)}")
    if title is not None and (not isinstance(title, str) or not title.isascii()):
        raise ValueError("title must be an ASCII string")
    return natoms, F


def _extra(F: int, box, boxangles, time) -> np.ndarray:
    """(F, 4 or 52) uint8: each record's time, cell_lengths and cell_angles in file byte order"""
    e = np.zeros(F, EXTRA_NOBOX if box is None else EXTRA_BOX)
    e["time"] = np.arange(F, dtype=np.float32) if time is None else np.asarray(time, np.float32)
    if box is not None:
        e["lengths"] = np.asarray(box, np.float32).T
        e["angles"] = 90.0 if boxangles is None else np.asarray(boxangles, np.float32).T
    return e.view(np.uint8).reshape(F, -1)


def _encode(coords, extra, natoms: int, F: int, with_box: bool, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = coords.device
    record_bytes, coord_offset = _record_layout(natoms, with_box)
    if out is None:
        out = torch.empty(F * record_bytes, dtype=torch.uint8, device=dev)
    if F == 0:
        return out[:0]
    coords = _trajio.frame_minor(coords)
    _lib.call(dev, "mkb_netcdf_encode", _lib.ptr(coords), max(int(coords.stride(1)), F), F, natoms, record_bytes,
              coord_offset, _lib.ptr(extra), _lib.ptr(out), int(out.numel()))
    return out[:F * record_bytes]


def encode_netcdf_device(coords: torch.Tensor, box=None, boxangles=None, time=None) -> torch.Tensor:
    """K23 on the device: ``coords`` (CUDA (natoms, 3, F) float32, frame-minor; a frame slice of a larger tensor is used
    in place) -> uint8 CUDA tensor of the F records of :func:`write_netcdf`'s file back to back: time, coordinates and,
    when ``box`` (3, F) is given, cell_lengths and cell_angles (``boxangles`` (3, F), 90 by default).  ``time`` (F,)
    in ps defaults to the frame index."""
    dev = _lib.tensor_device(coords, "encode_netcdf_device")
    if coords.dtype != torch.float32:
        raise ValueError(f"coords must be float32, got {coords.dtype}")
    box, boxangles, time = _trajio.host(box), _trajio.host(boxangles), _trajio.host(time)
    natoms, F = _writer_args(coords, box, boxangles, time, None)
    extra = torch.from_numpy(_extra(F, box, boxangles, time)).to(dev)
    return _encode(coords, extra, natoms, F, box is not None)


def _prepare(coords, box, boxangles, time, title, device, chunk_bytes):
    """every check, then (header, coords and the host-built record bytes as CUDA tensors or None without frames,
    natoms, F, with_box)"""
    coords = _trajio.writer_coords(coords, "write_netcdf")
    box, boxangles, time = _trajio.host(box), _trajio.host(boxangles), _trajio.host(time)
    natoms, F = _writer_args(coords, box, boxangles, time, title)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    with_box = box is not None
    header = netcdf_header(natoms, F, with_box, title)
    if F == 0:
        return header, None, None, natoms, F, with_box
    x = _trajio.on_device(coords, device)
    extra = torch.from_numpy(_extra(F, box, boxangles, time)).to(x.device)
    return header, x, extra, natoms, F, with_box


def _emit(fh, header, x, extra, natoms: int, F: int, with_box: bool, chunk_bytes) -> None:
    fh.write(header)
    if F == 0:
        return
    _trajio.write_encoded(fh, x.device, F, _record_layout(natoms, with_box)[0], chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], extra[f0:f1], natoms, f1 - f0, with_box,
                                                      out=out))


def netcdf_bytes(coords, box=None, boxangles=None, time=None, title=None, device=None,
                 chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_netcdf` writes, as a ``bytes`` object."""
    prep = _prepare(coords, box, boxangles, time, title, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, *prep, chunk_bytes)
    return fh.getvalue()


def write_netcdf(filename, coords, box=None, boxangles=None, time=None, title=None, device=None,
                 chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write an AMBER NetCDF trajectory (CDF-2, AMBER convention 1.0) with the records built on the GPU.  ``coords``
    (natoms, 3, F) float32 in Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a
    frame slice is fine).  ``box`` (3, F) [A, B, C] given means every frame carries cell_lengths and cell_angles, the
    angles from ``boxangles`` (3, F) [alpha, beta, gamma] (90 by default).  ``time`` (F,) in ps defaults to the frame
    index (0, 1, 2, ... ps), since the trajectory carries no time step.  ``title``: an ASCII string.  The frames are
    encoded in chunks of at most ``chunk_bytes`` and each chunk is written while the next one encodes.  The file is
    created or truncated; arguments are checked before it is opened."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    prep = _prepare(coords, box, boxangles, time, title, device, chunk_bytes)
    with open(filename, "wb") as fh:
        _emit(fh, *prep, chunk_bytes)
