"""GROMACS TRR trajectories read and written on the GPU (K24).

TRR is GROMACS's full-precision trajectory format, and the common format that stores velocities and forces.  A file
is a run of frames, each an XDR (big-endian) header -- magic 1993, the string "GMX_trn_file", the byte sizes of the
ir / e / box / vir / pres / top / sym / x / v / f blocks, natoms, step, nre, t and lambda -- then the blocks whose
size is not zero, in the order box, vir, pres, x, v, f.  Reals are float32, or float64 when a double-precision GROMACS
build wrote the file; the width follows xdrfile's nFloatSize (box_size / 9, else x_size, v_size or f_size over
3 natoms).  GROMACS writes x, v and f at independent intervals, so one file can mix x-only, v-only and x+v+f frames:
the word for a frame here is a *record*, and every record says which blocks it carries.

The host walks the headers (``index_trr``: only the header bytes and the 9-real box are read, through a memory map);
only the requested blocks of the listed records travel to the device, where ``mkb_trr_decode`` byte-swaps and
transposes them into the frame-minor ``(natoms, 3, F)`` layout the other kernels consume.  Float32 values move as
32-bit words (bit-identical, NaN payloads, signalling NaNs and -0.0 included); float64 values are rounded to float32
on the device exactly as numpy's ``astype(np.float32)`` rounds them on x86-64 (NaNs included).  ``mkb_trr_encode``
writes single-precision records (header and box built on the host, x and optionally v and f transposed on the device).

Reading gathers the listed records' blocks into two pinned staging buffers of at most ``chunk_bytes`` (one ``preadv``
per run of nearby blocks) and decodes one chunk while the other fills: only the requested blocks cross PCIe, and the
device holds the output plus two chunks.  Each block gets its own staging row of 3 natoms reals, so float64 blocks,
which lie on 4-byte boundaries in the file, are 8-byte aligned on the device.  Writing encodes chunk by chunk and writes
each chunk while the next one encodes.

Not supported (rejected with an error naming them): non-zero ir, e, top or sym blocks (xdrfile reads none of them), a
change of natoms or of precision between records, and writing double precision.  A truncated last record is dropped
with a warning.  Units are the file's: nm, ps, kJ mol^-1 nm^-1 (``scale`` multiplies x only, e.g. 10 for Angstrom).

Not confirmed (no TRR file written by GROMACS, no xdrfile or GROMACS source and no moleculekit checkout were at hand;
the layout is restated from xdrfile's published frame layout):

- the names and signatures of moleculekit's TRR functions (``trr.pyx``), and whether it returns velocities and forces
  or writes TRR at all (``read_trr`` / ``write_trr`` here follow the XTC module's shape);
- its units: nm here, like ``read_xtc``;
- what it does with records that carry no x, or with a file that has no box (here: ``read_trr`` returns the records
  with x, and a record without a box has a zero box);
- byte-for-byte agreement of the written header with a file GROMACS wrote.
"""
from __future__ import annotations

import ctypes as C
import io
import logging
import os
import struct

import numpy as np
import torch

from . import _lib, _trajio

logger = logging.getLogger(__name__)

MAGIC = 1993
NAME = b"GMX_trn_file"
CORE = 76  # header bytes before t and lambda: magic, 13, the XDR string, 11 sizes and natoms, step, nre
FIELDS = ("x", "v", "f")
MAX_ATOMS = (2**31 - 1) // 12  # x_size = 12 * natoms is an int32
CHUNK_BYTES = 256 << 20
# what the writer's host builds per record, in file byte order: the 84-byte single-precision header and the box
HEAD = np.dtype([("magic", ">i4"), ("slen", ">i4"), ("nlen", ">u4"), ("name", "S12"), ("sizes", ">i4", (10,)),
                 ("natoms", ">i4"), ("step", ">i4"), ("nre", ">i4"), ("t", ">f4"), ("lambda", ">f4"),
                 ("box", ">f4", (9,))], align=False)
assert HEAD.itemsize == 84 + 36


def _malformed(msg):
    return RuntimeError(f"Malformed TRR file: {msg}")


def index_trr(buf) -> dict:
    """Walk the records of a TRR file in a byte buffer (bytes, memoryview or a read-only np.memmap of the file), reading
    only their headers and boxes.

    Returns dict(natoms, double (float64 reals), n_records, and per record: offset (int64 byte offset), step (int32),
    time and lambda (float64: exact in both precisions), has_box / has_x / has_v / has_f (bool), x_offset / v_offset /
    f_offset (int64 byte offsets of the blocks, -1 where absent), box ((3, 3, R) float32, the box vectors as rows,
    zeros for a record without a box)).  A truncated last record is dropped with a warning."""
    b = np.frombuffer(buf, dtype=np.uint8)
    n, pos = len(b), 0
    natoms = w = None
    rows, boxes = [], []
    while pos < n:
        r = len(rows)
        where = f"record {r} at byte {pos}"
        if pos + CORE > n:
            logger.warning("TRR file: the last record (%s) is cut inside its header; it is dropped", where)
            break
        magic, slen, nlen = struct.unpack_from(">iiI", b, pos)
        if magic != MAGIC:
            raise _malformed(f"{where}: magic {magic}, expected {MAGIC}")
        if slen != 13 or nlen != 12:
            raise _malformed(f"{where}: version string lengths {slen} and {nlen}, expected 13 and 12")
        ir, e, box, vir, pres, top, sym, x, v, f, nat = struct.unpack_from(">11i", b, pos + 24)
        for name, size in (("ir", ir), ("e", e), ("top", top), ("sym", sym)):
            if size:
                raise ValueError(f"TRR {where}: {name}_size is {size}; ir, e, top and sym blocks are not supported "
                                 "(xdrfile reads none of them)")
        if nat < 0:
            raise _malformed(f"{where}: natoms is {nat}")
        for size, per in ((box, 9), (x, 3 * nat), (v, 3 * nat), (f, 3 * nat)):
            if size:
                rw = size // per if per > 0 else 0
                break
        else:
            raise _malformed(f"{where}: box_size, x_size, v_size and f_size are all 0")
        if rw not in (4, 8):
            raise _malformed(f"{where}: the sizes give {rw}-byte reals, expected 4 or 8")
        for name, size, per in (("box", box, 9), ("vir", vir, 9), ("pres", pres, 9), ("x", x, 3 * nat),
                                ("v", v, 3 * nat), ("f", f, 3 * nat)):
            if size not in (0, per * rw):
                raise _malformed(f"{where}: {name}_size is {size}, expected 0 or {per * rw} ({per} {rw}-byte reals)")
        if natoms is None:
            natoms, w = nat, rw
        elif nat != natoms:
            raise ValueError(f"TRR {where}: natoms changes from {natoms} to {nat}; a changing atom count is not "
                             "supported")
        elif rw != w:
            raise ValueError(f"TRR {where}: {rw}-byte reals after {w}-byte ones; a change of precision is not "
                             "supported")
        data = pos + CORE + 2 * w
        end = data + box + vir + pres + x + v + f
        if end > n:
            logger.warning("TRR file: the last record (%s) needs %d bytes, %d are left; it is dropped", where,
                           end - pos, n - pos)
            break
        t, lam = struct.unpack_from(">dd" if w == 8 else ">ff", b, pos + CORE)
        xo = data + box + vir + pres
        rows.append((pos, struct.unpack_from(">i", b, pos + 68)[0], t, lam, box > 0, x > 0, v > 0, f > 0,
                     xo if x else -1, xo + x if v else -1, xo + x + v if f else -1))
        boxes.append(np.frombuffer(b, ">f8" if w == 8 else ">f4", 9, data).astype(np.float32) if box else
                     np.zeros(9, np.float32))
        pos = end
    R = len(rows)
    cols = list(zip(*rows)) if R else [()] * 11
    out = dict(natoms=int(natoms or 0), double=w == 8, n_records=R,
               offset=np.array(cols[0], np.int64), step=np.array(cols[1], np.int32),
               time=np.array(cols[2], np.float64), **{"lambda": np.array(cols[3], np.float64)},
               has_box=np.array(cols[4], bool), has_x=np.array(cols[5], bool), has_v=np.array(cols[6], bool),
               has_f=np.array(cols[7], bool), x_offset=np.array(cols[8], np.int64),
               v_offset=np.array(cols[9], np.int64), f_offset=np.array(cols[10], np.int64))
    out["box"] = np.ascontiguousarray(np.array(boxes, np.float32).reshape(R, 3, 3).transpose(1, 2, 0))
    return out


def decode_trr_device(buf: torch.Tensor, offsets, natoms: int, value_bytes: int,
                      out: torch.Tensor | None = None) -> torch.Tensor:
    """K24 on the device: ``buf`` (uint8 CUDA tensor of staged file bytes), ``offsets`` (int64 per listed record: the
    byte offset in ``buf`` of its block of 3 * natoms big-endian reals, ``value_bytes`` 4 or 8 each, a multiple of
    ``value_bytes``) -> (natoms, 3, len(offsets)) float32.  ``out`` may be a frame slice of a larger (natoms, 3, F)
    tensor."""
    dev = _lib.tensor_device(buf, "decode_trr_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    offsets = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    F = int(offsets.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    if F == 0 or natoms == 0:
        return out
    _lib.call(dev, "mkb_trr_decode", _lib.ptr(buf), int(buf.numel()), offsets.ctypes.data_as(C.c_void_p), F,
              int(natoms), int(value_bytes), _lib.ptr(out), stride)
    return out


def _fields(fields) -> tuple:
    fields = (fields,) if isinstance(fields, str) else tuple(fields)
    if not fields or any(f not in FIELDS for f in fields) or len(set(fields)) != len(fields):
        raise ValueError(f"fields must be distinct names among {FIELDS}, got {fields!r}")
    return fields


def _read(filename, select, fields, scale, device, chunk_bytes):
    """The records ``select(index)`` picks -> ({field: CUDA (natoms, 3, F)}, box (3, 3, F), info)"""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    fields = _fields(fields)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    mm = np.memmap(filename, dtype=np.uint8, mode="r") if os.path.getsize(filename) else b""
    idx = index_trr(mm)
    R, natoms = idx["n_records"], idx["natoms"]
    sel = select(idx)
    for f in fields:
        missing = ~idx[f"has_{f}"][sel]
        if missing.any():
            raise ValueError(f"TRR record {int(sel[np.argmax(missing)])} has no {f} block")
    info = dict(natoms=natoms, n_records=R, double=idx["double"], records=sel, step=idx["step"][sel],
                time=idx["time"][sel], **{"lambda": idx["lambda"][sel]})
    box = np.ascontiguousarray(idx["box"][:, :, sel])
    dev = _lib.device(device)
    n = len(sel)
    out = {f: torch.empty((natoms, 3, n), dtype=torch.float32, device=dev) for f in fields}
    if n == 0 or natoms == 0:
        return out, box, info
    del mm  # the blocks are read with preadv: a copy from the page cache, without a page fault per 4 KiB
    w = 8 if idx["double"] else 4
    slab = 3 * natoms * w
    order = [f for f in FIELDS if f in fields]  # file order: ascending offsets within a record
    nf = len(order)
    chunks = _trajio.chunks(sel, np.full(R, nf * slab, np.int64), int(chunk_bytes))
    with open(filename, "rb") as fh:
        def stage(c, host):
            uniq = chunks[c][2]
            used = len(uniq) * nf * slab
            starts = np.stack([idx[f"{f}_offset"][uniq] for f in order], axis=1).reshape(-1)
            _trajio.gather_slabs(fh.fileno(), starts, slab, host[:used].reshape(len(uniq) * nf, slab), "TRR")
            return used

        def consume(c, buf):
            k0, k1, uniq = chunks[c]
            row = np.searchsorted(uniq, sel[k0:k1]) * nf
            for j, f in enumerate(order):
                decode_trr_device(buf, (row + j) * slab, natoms, w, out=out[f][:, :, k0:k1])

        _trajio.upload(dev, len(chunks), max(len(u) for _, _, u in chunks) * nf * slab, stage, consume)
    s = np.float32(scale)
    if "x" in out and s != 1:
        out["x"].mul_(float(s))  # one float32 multiply of the rounded value
    return out, box, info


def read_trr_device(filename, frames=None, fields=("x",), scale: float = 1.0, device=None,
                    chunk_bytes: int = CHUNK_BYTES):
    """Every record that carries all of ``fields`` (or the records listed in ``frames``: record indices, any order,
    repeats allowed; out of range raises IndexError, a listed record without a requested field ValueError) ->
    ({field: CUDA (natoms, 3, F) float32}, box (3, 3, F) float32, info) with the trajectory left on the GPU.
    ``fields`` names blocks among "x", "v", "f".  ``scale`` multiplies x only, as one float32 multiply after the
    rounding to float32 (10: Angstrom from nm); with ``scale == 1`` the values are not touched.  ``info`` holds natoms,
    n_records (records in the file), double, records (the record index of each returned frame), and the returned
    frames' step (int32), time and lambda (float64).  Only the requested blocks of the listed records are read and
    cross PCIe."""
    def select(idx):
        R = idx["n_records"]
        if frames is None:
            have = np.ones(R, bool)
            for f in _fields(fields):
                have &= idx[f"has_{f}"]
            return np.flatnonzero(have).astype(np.int64)
        return _trajio.select(R, frames)

    return _read(filename, select, fields, scale, device, chunk_bytes)


def read_trr(filename, device=None, chunk_bytes: int = CHUNK_BYTES):
    """The records that carry x -> (coords (natoms, 3, F) float32 [nm], box (3, 3, F), time (F,) float32, step (F,)
    int32) as numpy arrays, the return shape of ``read_xtc``."""
    out, box, info = read_trr_device(filename, device=device, chunk_bytes=chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"].astype(np.float32), info["step"].copy()


def read_trr_frames(filename, frames, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_trr` for the listed frames, numbered as :func:`read_trr` numbers them: frame k is the k-th record
    that carries x (any order, repeats allowed; out of range raises IndexError)."""
    frames = np.asarray(frames, np.int64).ravel()
    out, box, info = _read(filename, lambda idx: np.flatnonzero(idx["has_x"]).astype(np.int64)[frames], ("x",), 1.0,
                           device, chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"].astype(np.float32), info["step"].copy()


# ------------------------------------------------------------------------------------------------------------ writing
def _writer_args(coords, box, time, step, lambd, velocities, forces, scale, chunk_bytes):
    """shapes and values checked before any device work; returns (natoms, F)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"a TRR frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    for name, v, shape in (("box", box, (3, 3, F)), ("time", time, (F,)), ("step", step, (F,)),
                           ("lambd", lambd, (F,))):
        if v is not None and tuple(v.shape) != shape:
            raise ValueError(f"{name} must be {shape}, got {tuple(v.shape)}")
    if box is None or time is None or step is None:
        raise ValueError("box, time and step are required")
    for name, v in (("velocities", velocities), ("forces", forces)):
        if v is None:
            continue
        if tuple(v.shape) != (natoms, 3, F):
            raise ValueError(f"{name} must be {(natoms, 3, F)} like coords, got {tuple(v.shape)}")
        if isinstance(v, torch.Tensor):
            if v.dtype != torch.float32:
                raise ValueError(f"{name} must be float32, got {v.dtype}")
            _lib.tensor_device(v, "write_trr")
    if isinstance(coords, torch.Tensor) and coords.dtype != torch.float32:
        raise ValueError(f"coords must be float32, got {coords.dtype}")
    if not np.isfinite(np.float32(scale)):
        raise ValueError(f"scale must be finite, got {scale}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    return natoms, F


def _heads(natoms: int, F: int, box, time, step, lambd, with_v: bool, with_f: bool) -> np.ndarray:
    """(F, 120) uint8: each record's single-precision header and box, in file byte order"""
    h = np.zeros(F, HEAD)
    h["magic"], h["slen"], h["nlen"], h["name"], h["natoms"] = MAGIC, 13, 12, NAME, natoms
    h["sizes"] = [0, 0, 36, 0, 0, 0, 0, 12 * natoms, 12 * natoms if with_v else 0, 12 * natoms if with_f else 0]
    h["step"] = np.asarray(step).astype(np.int64).astype(np.int32)  # wraps like the writer's C int
    h["t"] = np.asarray(time, np.float32)
    h["lambda"] = 0 if lambd is None else np.asarray(lambd, np.float32)
    h["box"] = np.asarray(box, np.float32).transpose(2, 0, 1).reshape(F, 9)
    return h.view(np.uint8).reshape(F, HEAD.itemsize)


def _encode(x, v, f, head, natoms: int, F: int, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = x.device
    arrs = [_trajio.frame_minor(a) for a in (x, v, f) if a is not None]
    if len({max(int(a.stride(1)), F) for a in arrs}) > 1:  # the entry point takes one frame stride for all three
        arrs = [a.contiguous() for a in arrs]
    record_bytes = HEAD.itemsize + 12 * natoms * len(arrs)
    if out is None:
        out = torch.empty(F * record_bytes, dtype=torch.uint8, device=dev)
    if F == 0:
        return out[:0]
    x, v, f = arrs[0], (arrs[1] if v is not None else None), (arrs[-1] if f is not None else None)
    _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), _lib.ptr(v), _lib.ptr(f), max(int(x.stride(1)), F), F, natoms,
              _lib.ptr(head), HEAD.itemsize, _lib.ptr(out), int(out.numel()))
    return out[:F * record_bytes]


def _scaled(x, scale):
    s = np.float32(scale)
    return x if s == 1 else x * float(s)  # one float32 multiply


def encode_trr_device(coords: torch.Tensor, box, time, step, lambd=None, velocities=None, forces=None,
                      scale: float = 1.0) -> torch.Tensor:
    """K24 on the device: ``coords`` (CUDA (natoms, 3, F) float32, frame-minor; a frame slice of a larger tensor is
    used in place) -> uint8 CUDA tensor of the F records of :func:`write_trr`'s file back to back."""
    dev = _lib.tensor_device(coords, "encode_trr_device")
    box, time, step, lambd = (_trajio.host(a) for a in (box, time, step, lambd))
    natoms, F = _writer_args(coords, box, time, step, lambd, velocities, forces, scale, 1)
    head = torch.from_numpy(_heads(natoms, F, box, time, step, lambd, velocities is not None,
                                   forces is not None)).to(dev)
    return _encode(_scaled(coords, scale), _trajio.on_device(velocities, dev), _trajio.on_device(forces, dev), head,
                   natoms, F)


def _prepare(coords, box, time, step, lambd, velocities, forces, scale, device, chunk_bytes):
    """every check, then (x, v, f and the host-built headers as CUDA tensors or None without frames, natoms, F)"""
    coords = _trajio.writer_coords(coords, "write_trr")
    box, time, step, lambd = (_trajio.host(a) for a in (box, time, step, lambd))
    natoms, F = _writer_args(coords, box, time, step, lambd, velocities, forces, scale, chunk_bytes)
    if F == 0:
        return None, None, None, None, natoms, F
    dev = coords.device if isinstance(coords, torch.Tensor) else _lib.device(device)
    for name, a in (("velocities", velocities), ("forces", forces)):
        if isinstance(a, torch.Tensor) and a.device != dev:
            raise ValueError(f"{name} are on {a.device}, coords on {dev}")
    x, v, f = (_trajio.on_device(a, dev) for a in (coords, velocities, forces))
    head = torch.from_numpy(_heads(natoms, F, box, time, step, lambd, v is not None, f is not None)).to(dev)
    return _scaled(x, scale), v, f, head, natoms, F


def _emit(fh, x, v, f, head, natoms: int, F: int, chunk_bytes) -> None:
    if F == 0:
        return
    record_bytes = HEAD.itemsize + 12 * natoms * (1 + (v is not None) + (f is not None))

    def part(a, f0, f1):
        return None if a is None else a[:, :, f0:f1]

    _trajio.write_encoded(fh, x.device, F, record_bytes, chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], part(v, f0, f1), part(f, f0, f1), head[f0:f1],
                                                      natoms, f1 - f0, out=out))


def trr_bytes(coords, box, time, step, lambd=None, velocities=None, forces=None, scale: float = 1.0, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_trr` writes, as a ``bytes`` object."""
    prep = _prepare(coords, box, time, step, lambd, velocities, forces, scale, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, *prep, chunk_bytes)
    return fh.getvalue()


def write_trr(filename, coords, box, time, step, lambd=None, velocities=None, forces=None, scale: float = 1.0,
              device=None, chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a single-precision GROMACS TRR trajectory with the records built on the GPU.  ``coords`` (natoms, 3, F)
    float32 in nm: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``box`` (3, 3, F) (the box vectors as rows, nm), ``time`` (F,) ps, ``step`` (F,), ``lambd`` (F,) (0 by default):
    host arrays.  ``velocities`` / ``forces`` (natoms, 3, F), given, are written into every record after x.  ``scale``
    multiplies x only, as one float32 multiply (0.1 undoes the ``scale=10`` of :func:`read_trr_device`).  Every record
    carries the header, the box and x (ir, e, vir, pres, top, sym and nre are 0).  The records are encoded in chunks of
    at most ``chunk_bytes`` and each chunk is written while the next one encodes.  The file is created or truncated;
    arguments are checked before it is opened."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    prep = _prepare(coords, box, time, step, lambd, velocities, forces, scale, device, chunk_bytes)
    with open(filename, "wb") as fh:
        _emit(fh, *prep, chunk_bytes)
