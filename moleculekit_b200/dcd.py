"""DCD trajectories (CHARMM / NAMD / OpenMM) read and written on the GPU (K22).

Mirrors the VMD molfile DCD plugin that moleculekit wraps (moleculekit/fileformats/dcd/{dcd.pyx,src/dcdplugin.c}):
``read_dcdheader`` / ``read_next_timestep`` for reading, ``write_dcdheader`` / ``write_dcdstep`` for writing.  The host
walks the small headers and the record markers; the frame records travel to the device as they are in the file, and
``mkb_dcd_decode`` turns them straight into the frame-minor ``(natoms, 3, F)`` layout the other kernels consume -- no
per-frame interleave and no transposition on the host.  ``mkb_dcd_encode`` is the same transposition the other way
round.  Coordinates move as 32-bit words: bit-identical in both directions, NaN payloads and -0.0 included.

Reading streams the listed frames' byte ranges through two pinned staging buffers of at most ``chunk_bytes``: the device
holds the output plus two chunks, and a frame subset reads only its frames from disk.  Writing encodes chunk by chunk
and writes each while the next one encodes.

Not confirmed against moleculekit (its DCD sources and a DCD written by it were not at hand):

- the names and signatures of moleculekit's DCD reader and writer (``read_dcd`` / ``write_dcd`` here follow the XTC
  module's shape);
- how ``Molecule`` fills ``time`` and ``step`` from ISTART / NSAVC / DELTA (returned in ``info``, not turned into times);
- the box it returns for files without a unit cell (here the plugin's defaults: zeros, angles 90);
- whether it writes a zero box as a unit cell (here: a unit cell is written exactly when ``box`` is given);
- the writer's default ISTART / NSAVC / DELTA and title (the plugin writes a date line, so its files are not
  reproducible byte for byte; here 0 / 1 / 1.0 and one fixed line);
- what it does with a truncated last frame (here: dropped with a warning);
- whether it accepts 64-bit record markers (here: read, never written);
- two details of the plugin's writer restated from its published layout and not checked against its source: the value
  it leaves in ICNTRL[3] (here ISTART + NSET * NSAVC) and the padding of the title lines (here spaces).
"""
from __future__ import annotations

import ctypes as C
import io
import logging
import math
import os
import struct

import numpy as np
import torch

from . import _lib, _trajio

logger = logging.getLogger(__name__)

# numpy mirror of `mkb_dcd_frame` (32 bytes)
FRAME_DESC = np.dtype([("offset", "<i8", (3,)), ("count", "<i8")], align=False)
assert FRAME_DESC.itemsize == 32
M_PI_2 = 1.57079632679489661923
MAX_ATOMS = (2**31 - 1) // 4  # a record of 4 * natoms bytes must fit the int32 marker
DEFAULT_TITLE = ("REMARKS written by moleculekit_b200",)
CHUNK_BYTES = 256 << 20


def _malformed(msg):
    return RuntimeError(f"Malformed DCD file: {msg}")


class _Records:
    """Record walker over a byte buffer of known byte order (``e``) and marker width (``mw``)."""

    def __init__(self, b, e: str, mw: int):
        self.b, self.e, self.mw = b, e, mw
        self.mfmt = e + ("i" if mw == 4 else "q")

    def marker(self, pos: int) -> int:
        if pos + self.mw > len(self.b):
            raise EOFError
        return struct.unpack_from(self.mfmt, self.b, pos)[0]

    def record(self, pos: int, what: str, length: int | None = None) -> tuple[int, int]:
        """(start of the data, position after the trailing marker); checks both markers (and ``length``)"""
        n = self.marker(pos)
        if n < 0 or (length is not None and n != length):
            raise _malformed(f"{what} record has length {n}" + (f", expected {length}" if length is not None else ""))
        end = pos + self.mw + n
        if self.marker(end) != n:
            raise _malformed(f"{what} record: the trailing marker does not match the leading one ({n})")
        return pos + self.mw, end + self.mw


def _detect(b) -> tuple[str, int]:
    """byte order and marker width, as read_dcdheader decides them"""
    if len(b) < 12:
        raise _malformed("too short for a header")
    for e in "<>":
        m0, m1 = struct.unpack_from(e + "ii", b, 0)
        if m0 + m1 == 84 and bytes(b[8:12]) == b"CORD":
            return e, 8
        if m0 == 84 and bytes(b[4:8]) == b"CORD":
            return e, 4
    raise _malformed("the file does not start with the 84-byte CORD record")


def _frame_layout(r: _Records, start: int, count: int, extra: bool, four_d: bool, f: int) -> dict:
    """Walk one frame record set at ``start``: size, the offsets of the X / Y / Z data relative to ``start``, and of the
    unit cell (None unless the extra block is 48 bytes long).  Raises EOFError when the bytes end inside the frame."""
    pos, cell = start, None
    if extra:
        n = r.marker(pos)
        data, pos = r.record(pos, f"frame {f}: unit-cell")
        if n == 48:
            cell = data - start
    xyz = []
    for axis in "XYZ":
        data, pos = r.record(pos, f"frame {f}: {axis}", 4 * count)
        xyz.append(data - start)
    if four_d:
        _, pos = r.record(pos, f"frame {f}: 4D")
    if pos > len(r.b):
        raise EOFError
    return dict(size=pos - start, xyz=xyz, cell=cell, count=count)


def _check_markers(r: _Records, b, start: int, size: int, n: int, lay: dict, extra: bool, four_d: bool, first: int):
    """The leading and trailing markers of the ``n`` frames of ``size`` bytes at ``start``, vectorised over frames."""
    if n <= 0:
        return
    mdt = np.dtype(r.mfmt)

    def at(rel):  # the marker at ``rel`` in every frame
        return np.ndarray((n,), dtype=mdt, buffer=b, offset=start + rel, strides=(size,))

    checks = []
    pos = 0
    if extra:
        n_extra = int(at(0)[0])
        checks.append((0, n_extra, "unit-cell"))
        pos = 2 * r.mw + n_extra
    for axis in "XYZ":
        checks.append((pos, 4 * lay["count"], axis))
        pos += 2 * r.mw + 4 * lay["count"]
    if four_d:
        checks.append((pos, int(at(pos)[0]), "4D"))
    for rel, n_rec, what in checks:
        bad = (at(rel) != n_rec) | (at(rel + r.mw + n_rec) != n_rec)
        if bad.any():
            f = first + int(np.argmax(bad))
            raise _malformed(f"frame {f}: {what} record markers do not match ({n_rec} bytes expected)")


def unitcell_to_box(cells) -> tuple[np.ndarray, np.ndarray]:
    """(F, 6) float64 unit-cell records -> box (3, F) float32 [A, B, C], boxangles (3, F) float32 [alpha, beta, gamma],
    as read_next_timestep converts them: cosines through libm's asin when all three angle slots are within [-1, 1],
    degrees otherwise."""
    cells = np.asarray(cells, dtype=np.float64).reshape(-1, 6)
    F = cells.shape[0]
    box = np.zeros((3, F), np.float32)
    angles = np.zeros((3, F), np.float32)
    if F == 0:
        return box, angles
    # trajectories at constant volume convert one cell; rows are told apart by their bits (-0.0 is not 0.0 here)
    rows, inv = np.unique(np.ascontiguousarray(cells).view(np.int64), axis=0, return_inverse=True)
    table = np.zeros((len(rows), 6), np.float32)
    for i, uc in enumerate(rows.view(np.float64).tolist()):
        if all(-1.0 <= uc[j] <= 1.0 for j in (1, 3, 4)):
            ang = [90.0 - math.asin(uc[j]) * 90.0 / M_PI_2 for j in (4, 3, 1)]
        else:
            ang = [uc[4], uc[3], uc[1]]
        table[i] = [uc[0], uc[2], uc[5]] + ang
    table = table[np.asarray(inv).reshape(-1)]
    return np.ascontiguousarray(table[:, :3].T), np.ascontiguousarray(table[:, 3:].T)


def box_to_unitcell(box, boxangles=None) -> np.ndarray:
    """box (3, F) [A, B, C] and boxangles (3, F) [alpha, beta, gamma] (None: 90) -> (F, 6) float64 unit-cell records
    ``A, cos gamma, B, cos beta, cos alpha, C`` as the plugin's writer forms them from float32 values:
    ``cos x = sin((M_PI_2 / 90) * (90 - x))`` through libm's sin."""
    box = np.asarray(box, dtype=np.float32)
    F = box.shape[1]
    ang = np.full((3, F), 90.0, np.float32) if boxangles is None else np.asarray(boxangles, dtype=np.float32)
    vals = np.ascontiguousarray(np.concatenate([box, ang]).T.astype(np.float64))
    rows, inv = np.unique(vals.view(np.int64), axis=0, return_inverse=True)
    table = np.zeros((len(rows), 6), np.float64)
    for i, (a, b, c, alpha, beta, gamma) in enumerate(rows.view(np.float64).tolist()):
        table[i] = [a, math.sin((M_PI_2 / 90.0) * (90.0 - gamma)), b, math.sin((M_PI_2 / 90.0) * (90.0 - beta)),
                    math.sin((M_PI_2 / 90.0) * (90.0 - alpha)), c]
    return np.ascontiguousarray(table[np.asarray(inv).reshape(-1)])


def index_dcd(buf) -> dict:
    """Walk the header and the frame records of a DCD byte buffer (bytes, memoryview or a read-only np.memmap of the file),
    as read_dcdheader / read_next_timestep of the plugin do.

    Returns dict(natoms, n_frames, nset, istart, nsavc, delta, namnf, charmm, has_extra, has_4d, title (list of str),
    swap (the file is in the other byte order), marker_bytes (4 or 8), free (int32 0-based indices of the free atoms, None
    without fixed atoms), frames (FRAME_DESC per frame, absolute byte offsets), start / size (int64 per frame: the byte
    range of its records), unitcell ((F, 6) float64, zeros where a frame has none), box / boxangles ((3, F) float32)).
    The frame count comes from the bytes present: a trailing partial frame is dropped with a warning."""
    b = np.frombuffer(buf, dtype=np.uint8)
    e, mw = _detect(b)
    r = _Records(b, e, mw)
    try:
        data, pos = r.record(0, "CORD", 84)
        icntrl = struct.unpack_from(e + "20i", b, data + 4)
        charmm = icntrl[19] != 0
        if charmm:
            delta = float(struct.unpack_from(e + "f", b, data + 4 + 36)[0])
        else:
            delta = float(struct.unpack_from(e + "d", b, data + 4 + 36)[0])
        has_extra = charmm and icntrl[10] != 0
        has_4d = charmm and icntrl[11] == 1
        namnf = icntrl[8]
        n_title_bytes = r.marker(pos)
        ntitle = struct.unpack_from(e + "i", b, pos + mw)[0] if n_title_bytes >= 4 else -1
        if ntitle < 0 or n_title_bytes != 4 + 80 * ntitle:
            raise _malformed(f"title record of {n_title_bytes} bytes does not hold NTITLE = {ntitle} lines of 80")
        data, pos = r.record(pos, "title")
        title = [bytes(b[data + 4 + 80 * i: data + 84 + 80 * i]).decode("latin-1") for i in range(ntitle)]
        data, pos = r.record(pos, "NATOM", 4)
        natoms = struct.unpack_from(e + "i", b, data)[0]
        if natoms < 0:
            raise _malformed(f"NATOM = {natoms}")
        free = None
        n_free = natoms
        if namnf != 0:
            if not 0 < namnf < natoms:
                raise _malformed(f"NAMNF = {namnf} fixed atoms of {natoms}")
            n_free = natoms - namnf
            data, pos = r.record(pos, "free-atom index", 4 * n_free)
            free = np.frombuffer(b, dtype=e + "i4", count=n_free, offset=data).astype(np.int32) - 1
            if free.min() < 0 or free.max() >= natoms or len(np.unique(free)) != n_free:
                raise _malformed("the free-atom index record lists atoms outside 1..NATOM or twice")
    except (EOFError, struct.error):
        raise _malformed("the header is truncated") from None
    header_end = pos

    lay0 = lay1 = None
    try:
        lay0 = _frame_layout(r, header_end, natoms, has_extra, has_4d, 0)
        lay1 = _frame_layout(r, header_end + lay0["size"], n_free, has_extra, has_4d, 1)
    except EOFError:
        pass
    rest = len(b) - header_end
    if lay0 is None:
        F = 0
    elif lay1 is None:
        F = 1
    else:
        F = 1 + (rest - lay0["size"]) // lay1["size"]
    used = 0 if F == 0 else lay0["size"] + (F - 1) * (lay1["size"] if lay1 else 0)
    if rest > used:
        logger.warning("DCD file: %d trailing bytes after %d whole frames do not make a frame; they are ignored",
                       rest - used, F)
    if F > 1:
        _check_markers(r, b, header_end + lay0["size"], lay1["size"], F - 1, lay1, has_extra, has_4d, 1)

    start = np.zeros(F, np.int64)
    size = np.zeros(F, np.int64)
    frames = np.zeros(F, dtype=FRAME_DESC)
    cells = np.zeros((F, 6), np.float64)
    has_cell = np.zeros(F, bool)
    if F:
        start[0], size[0] = header_end, lay0["size"]
        start[1:] = header_end + lay0["size"] + np.arange(F - 1, dtype=np.int64) * (lay1["size"] if lay1 else 0)
        size[1:] = lay1["size"] if lay1 else 0
        for sl, lay in ((slice(0, 1), lay0), (slice(1, F), lay1)):
            if lay is None or sl.start >= F:
                continue
            frames["offset"][sl] = start[sl, None] + np.asarray(lay["xyz"], np.int64)[None, :]
            frames["count"][sl] = lay["count"]
            if lay["cell"] is not None:
                n = sl.stop - sl.start
                view = np.ndarray((n, 6), dtype=e + "f8", buffer=b, offset=int(start[sl.start]) + lay["cell"],
                                  strides=(int(lay["size"]), 8))
                cells[sl] = view
                has_cell[sl] = True
    defaults = np.array([0.0, 90.0, 0.0, 90.0, 90.0, 0.0])  # the plugin's values when a frame carries no unit cell
    box, angles = unitcell_to_box(np.where(has_cell[:, None], cells, defaults))
    return dict(natoms=int(natoms), n_frames=int(F), nset=int(icntrl[0]), istart=int(icntrl[1]), nsavc=int(icntrl[2]),
                delta=delta, namnf=int(namnf), charmm=bool(charmm), has_extra=bool(has_extra), has_4d=bool(has_4d),
                title=title, swap=e != "<", marker_bytes=mw, free=free, frames=frames, start=start, size=size,
                unitcell=cells, box=box, boxangles=angles)


def _slot_map(natoms: int, free) -> np.ndarray:
    slot = np.full(natoms, -1, np.int32)
    slot[free] = np.arange(len(free), dtype=np.int32)
    return slot


def decode_dcd_device(buf: torch.Tensor, frames: np.ndarray, natoms: int, swap: bool = False, slot=None, n_free: int = 0,
                      first_buf=None, first=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """K22 on the device: ``buf`` (uint8 CUDA tensor holding frame records; the whole file, or a part of it), ``frames``
    (FRAME_DESC, offsets into ``buf``, any subset / order) -> coords (natoms, 3, len(frames)) float32.  ``swap``: the
    records are in the other byte order.  Fixed atoms: ``slot`` (int32 CUDA (natoms,): position in the free list, -1
    for a fixed atom), ``n_free`` (the length of the free list), the file's first frame ``first_buf`` (uint8 CUDA) and
    its descriptor ``first`` (FRAME_DESC array of one, offsets into ``first_buf``).  ``out`` may be a frame slice of a larger (natoms, 3, F) tensor."""
    dev = _lib.tensor_device(buf, "decode_dcd_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    frames = np.ascontiguousarray(frames, dtype=FRAME_DESC)
    F = int(frames.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    if F == 0 or natoms == 0:
        return out
    first_arr = None
    if slot is not None:
        _lib.index_arg(slot, dev)
        assert first_buf is not None and first is not None and first_buf.device == dev and first_buf.dtype == torch.uint8
        first_arr = np.ascontiguousarray(first, dtype=FRAME_DESC).reshape(1)
    _lib.call(dev, "mkb_dcd_decode", _lib.ptr(buf), int(buf.numel()), frames.ctypes.data_as(C.c_void_p), F, int(natoms),
              _lib.ptr(slot), int(n_free), _lib.ptr(first_buf), int(first_buf.numel()) if first_buf is not None else 0,
              first_arr.ctypes.data_as(C.c_void_p) if first_arr is not None else None, int(bool(swap)), _lib.ptr(out),
              stride)
    return out


def read_dcd_device(filename, frames=None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Whole file (or the frames listed: any order, repeats allowed) -> (coords CUDA (natoms, 3, F) float32 [Angstrom],
    box (3, F) float32, boxangles (3, F) float32, info dict) with the trajectory left on the GPU.  ``info`` holds istart,
    nsavc, delta, natoms, nset (the header's frame count), charmm / has_extra / has_4d / namnf, title and n_frames (the
    frames present in the file)."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    if os.path.getsize(filename) == 0:
        raise _malformed("the file is empty")
    idx = index_dcd(np.memmap(filename, dtype=np.uint8, mode="r"))
    F, natoms = idx["n_frames"], idx["natoms"]
    sel = _trajio.select(F, frames)
    info = {k: idx[k] for k in ("istart", "nsavc", "delta", "natoms", "nset", "charmm", "has_extra", "has_4d", "namnf",
                                "title", "n_frames")}
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((natoms, 3, n), dtype=torch.float32, device=dev)
    if n == 0 or natoms == 0:
        return coords, idx["box"][:, sel], idx["boxangles"][:, sel], info
    start, size, fdesc = idx["start"], idx["size"], idx["frames"]
    with open(filename, "rb") as fh:
        slot = first_buf = first = None
        if idx["free"] is not None:  # the first frame stays resident: it holds the fixed atoms of every frame
            fh.seek(int(start[0]))
            first_buf = torch.frombuffer(bytearray(fh.read(int(size[0]))), dtype=torch.uint8).to(dev)
            first = fdesc[:1].copy()
            first["offset"] -= start[0]
            slot = torch.from_numpy(_slot_map(natoms, idx["free"])).to(dev)

        def decode(buf, at, frame_of, k0, k1):
            desc = fdesc[sel[k0:k1]].copy()
            desc["offset"] += (at[frame_of] - start[sel[k0:k1]])[:, None]
            decode_dcd_device(buf, desc, natoms, idx["swap"], slot, natoms - idx["namnf"], first_buf, first,
                              out=coords[:, :, k0:k1])

        _trajio.read_frames(fh.fileno(), dev, sel, start, size, chunk_bytes, "DCD", decode)
    return coords, idx["box"][:, sel], idx["boxangles"][:, sel], info


def read_dcd(filename, device=None, chunk_bytes: int = CHUNK_BYTES):
    """(coords (natoms, 3, F) float32 [Angstrom], box (3, F), boxangles (3, F), info) as numpy arrays."""
    coords, box, angles, info = read_dcd_device(filename, device=device, chunk_bytes=chunk_bytes)
    return coords.cpu().numpy(), box, angles, info


def read_dcd_frames(filename, frames, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_dcd` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, box, angles, info = read_dcd_device(filename, frames=np.asarray(frames), device=device, chunk_bytes=chunk_bytes)
    return coords.cpu().numpy(), box, angles, info


# ------------------------------------------------------------------------------------------------------------ writing
def dcd_header(natoms: int, n_frames: int, istart: int = 0, nsavc: int = 1, delta: float = 1.0, title=None,
               with_unitcell: bool = False) -> bytes:
    """The header write_dcdheader writes, with the frame count the per-frame updates leave: the 84-byte CORD record
    (NSET, ISTART, NSAVC, ICNTRL[3] = ISTART + NSET * NSAVC, DELTA as float32, the extra-block flag, CHARMM version 24),
    the title record (each line cut to or padded with spaces to 80 characters) and NATOM.  Little-endian, 4-byte
    markers."""
    lines = list(DEFAULT_TITLE if title is None else ([title] if isinstance(title, str) else title))
    icntrl = [0] * 20
    icntrl[0], icntrl[1], icntrl[2] = n_frames, istart, nsavc
    icntrl[3] = (istart + n_frames * nsavc + 2**31) % 2**32 - 2**31  # C int arithmetic
    icntrl[10], icntrl[19] = int(bool(with_unitcell)), 24
    cord = struct.pack("<i4s9i", 84, b"CORD", *icntrl[:9]) + struct.pack("<f", delta) + \
        struct.pack("<10ii", *icntrl[10:], 84)
    text = b"".join(line.encode("latin-1")[:80].ljust(80, b" ") for line in lines)
    n = 4 + len(text)
    return cord + struct.pack("<ii", n, len(lines)) + text + struct.pack("<iiii", n, 4, natoms, 4)


def _writer_args(coords, box, boxangles, istart, nsavc, title):
    """shapes and ranges checked before any device work; returns (natoms, F)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if natoms > MAX_ATOMS:
        raise ValueError(f"{natoms} atoms do not fit the int32 record markers of a DCD file (at most {MAX_ATOMS})")
    if box is None and boxangles is not None:
        raise ValueError("boxangles need a box")
    for name, v in (("box", box), ("boxangles", boxangles)):
        if v is not None and tuple(v.shape) != (3, F):
            raise ValueError(f"{name} must be (3, {F}), got {tuple(v.shape)}")
    for name, v in (("istart", istart), ("nsavc", nsavc)):
        if not -2**31 <= int(v) < 2**31:
            raise ValueError(f"{name} = {v} does not fit an int32")
    if title is not None and not isinstance(title, str) and not all(isinstance(t, str) for t in title):
        raise ValueError("title must be a string or a list of strings")
    return natoms, F


def encode_dcd_device(coords: torch.Tensor, box=None, boxangles=None) -> torch.Tensor:
    """K22 on the device: ``coords`` (CUDA (natoms, 3, F) float32, frame-minor; a frame slice of a larger tensor is used
    in place) -> uint8 CUDA tensor of the F frame records back to back: the unit-cell record when ``box`` (3, F) is
    given (angles from ``boxangles`` (3, F), 90 by default), then the X, Y and Z records."""
    dev = _lib.tensor_device(coords, "encode_dcd_device")
    if coords.dtype != torch.float32:
        raise ValueError(f"coords must be float32, got {coords.dtype}")
    box, boxangles = _trajio.host(box), _trajio.host(boxangles)
    natoms, F = _writer_args(coords, box, boxangles, 0, 1, None)
    cells = None if box is None else torch.from_numpy(box_to_unitcell(box, boxangles)).to(dev)
    return _encode(coords, cells, natoms, F)


def _frame_bytes(natoms: int, with_unitcell: bool) -> int:
    return (56 if with_unitcell else 0) + 3 * (8 + 4 * natoms)


def _encode(coords, cells, natoms: int, F: int, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = coords.device
    nbytes = F * _frame_bytes(natoms, cells is not None)
    if out is None:
        out = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    if F == 0:
        return out[:0]
    coords = _trajio.frame_minor(coords)
    stride = coords.stride(1) if natoms else F
    _lib.call(dev, "mkb_dcd_encode", _lib.ptr(coords) if natoms else None, max(int(stride), F), F, natoms,
              _lib.ptr(cells), _lib.ptr(out), int(out.numel()))
    return out[:nbytes]


def _prepare(coords, box, boxangles, istart, nsavc, delta, title, device, chunk_bytes):
    """every check, then (header, coords and unit cells as CUDA tensors or None without frames, natoms, F)"""
    coords = _trajio.writer_coords(coords, "write_dcd")
    box = None if box is None else np.asarray(box)
    boxangles = None if boxangles is None else np.asarray(boxangles)
    natoms, F = _writer_args(coords, box, boxangles, istart, nsavc, title)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    header = dcd_header(natoms, F, int(istart), int(nsavc), float(delta), title, box is not None)
    if F == 0:
        return header, None, None, natoms, F
    x = _trajio.on_device(coords, device)
    cells = None if box is None else torch.from_numpy(box_to_unitcell(box, boxangles)).to(x.device)
    return header, x, cells, natoms, F


def _emit(fh, header, x, cells, natoms: int, F: int, chunk_bytes) -> None:
    fh.write(header)
    if F == 0:
        return
    _trajio.write_encoded(fh, x.device, F, _frame_bytes(natoms, cells is not None), chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], None if cells is None else cells[f0:f1], natoms,
                                                      f1 - f0, out=out))


def dcd_bytes(coords, box=None, boxangles=None, istart: int = 0, nsavc: int = 1, delta: float = 1.0, title=None,
              device=None, chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_dcd` writes, as a ``bytes`` object."""
    prep = _prepare(coords, box, boxangles, istart, nsavc, delta, title, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, *prep, chunk_bytes)
    return fh.getvalue()


def write_dcd(filename, coords, box=None, boxangles=None, istart: int = 0, nsavc: int = 1, delta: float = 1.0,
              title=None, device=None, chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a CHARMM-style DCD file with the frame records built on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``box`` (3, F) [A, B, C] given means every frame carries a unit cell, with the angles of ``boxangles`` (3, F)
    [alpha, beta, gamma] (90 by default).  ``title``: a string or a list of lines.  The frames are encoded in chunks of
    at most ``chunk_bytes`` and each chunk is written while the next one encodes.  The file is created or truncated;
    arguments are checked before it is opened."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    prep = _prepare(coords, box, boxangles, istart, nsavc, delta, title, device, chunk_bytes)
    with open(filename, "wb") as fh:
        _emit(fh, *prep, chunk_bytes)
