"""AMBER ASCII trajectories (mdcrd / crd / trj, and mdvel) read and written on the GPU (K25).

The format sander / pmemd write with ioutfm=0 (and cpptraj): a title line, then frames of 3 natoms values atom-major
(x, y, z of atom 0, then atom 1, ...) as Fortran F8.3 fields, ten per line, each line ending in a newline, and with a
periodic box one more line of three F8.3 fields (A, B, C in Angstrom) per frame.  Every frame has the same size,
``S = 24 natoms + ceil(3 natoms / 10) + (25 with a box)`` bytes.  Velocity files (mdvel) share the layout.

It is the largest trajectory format on disk (about 24.3 bytes per atom-frame) and the slowest to read on the host,
where every field is converted on its own.  Here the host only finds the frames (``index_mdcrd`` reads the title and
the line after the first frame); the listed frames travel to the device in two pinned staging buffers of at most
``chunk_bytes`` (one frame per 16-byte-aligned staging row), and ``mkb_mdcrd_decode`` parses and transposes one chunk
into the frame-minor ``(natoms, 3, F)`` layout while the next one is read.  A field decodes bit for bit to
``np.float32(float(field))``; a malformed field or a misplaced newline raises ValueError naming the frame, line and
column.  Writing formats on the device (``mkb_mdcrd_encode``), byte for byte ``'%8.3f' % x``, chunk by chunk, each
chunk written while the next one encodes.

Writable values: ``rint(x * 1000)`` (in float64: exact, half to even, as '%8.3f' rounds) at most 9 999 999 for x >= 0
and at least -999 999 for x < 0, so that the field keeps 8 characters; anything else, NaN and +-inf included, is
rejected before the file is opened with an error naming the first offending frame, atom and axis.  A negative value
that rounds to zero, and -0.0, are written as ``-0.000``, as printf writes them.

Not supported: compressed (.gz / .bz2) files, REMD per-frame headers, CRLF line endings (the title line is checked and
the message says so; a CR inside a frame is a malformed field), AMBER restart / inpcrd files (12.7 fields) and a
changing atom count.  A truncated last frame is dropped with a warning.

Not confirmed (no moleculekit checkout was at hand; the contract here follows the format itself, with Python's
``float()`` and ``'%8.3f'`` as the arithmetic reference):

- the name and signature of moleculekit's mdcrd reader (``read_mdcrd`` here follows the other modules' shape, with the
  atom count as an argument: the file does not store it);
- whether moleculekit writes mdcrd at all;
- how it decides that a box line is present (here: a 24-character line after frame 0; with one atom, whose frame
  lines are also 24 characters, the file size decides, or ``box=`` must be given);
- the title the writer puts on line 1: here the given title padded to 80 columns, as sander's (a80) writes it.
"""
from __future__ import annotations

import ctypes as C
import io
import logging
import os

import numpy as np
import torch

from . import _lib, _trajio

logger = logging.getLogger(__name__)

CHUNK_BYTES = 256 << 20
MAX_ATOMS = (2**31 - 1) // 25  # a frame's bytes fit an int32
POS_MAX, NEG_MIN = 9999999, -999999  # the writable range of rint(x * 1000): "9999.999" and "-999.999"
INT64_MAX = 2**63 - 1
TITLE_WIDTH = 80


def frame_bytes(natoms: int, box: bool) -> int:
    """bytes of one frame: 3 natoms F8.3 fields, ten per line, and the box line"""
    return 24 * natoms + (3 * natoms + 9) // 10 + (25 if box else 0)


def _find_newline(b: np.ndarray, start: int = 0) -> int:
    """index of the first b'\\n' at or after ``start``, -1 when there is none (reads the buffer in windows)"""
    step = 1 << 16
    for w in range(start, len(b), step):
        i = bytes(b[w:w + step]).find(b"\n")
        if i >= 0:
            return w + i
    return -1


def index_mdcrd(buf, natoms: int, box: bool | None = None) -> dict:
    """Find the frames of an AMBER ASCII trajectory in a byte buffer (bytes, memoryview or a read-only np.memmap of the
    file), reading only the title line and the line after the first frame.

    ``box`` None detects the box line: a 24-character line after frame 0 is one.  With one atom a frame's line is also
    24 characters, so the file size decides: a box-less reading that ends on a whole frame where the boxed one would
    not, or no frame at all; otherwise ValueError asks for ``box=True`` or ``box=False``.
    Returns dict(title (str: the first line without its newline and trailing spaces), has_box, frame_bytes, offset (of
    the first frame), n_frames).  A truncated last frame is dropped with a warning."""
    natoms = int(natoms)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"natoms must be 1 to {MAX_ATOMS}, got {natoms}")
    b = np.frombuffer(buf, dtype=np.uint8)
    n = len(b)
    nl = _find_newline(b)
    if nl < 0:
        raise ValueError("AMBER mdcrd file: no title line (the file has no newline)")
    if nl > 0 and b[nl - 1] == 13:
        raise ValueError("AMBER mdcrd file: the title line ends in CR LF; CRLF line endings are not supported "
                         "(convert the file to LF line endings)")
    t0 = nl + 1
    rest = n - t0
    if box is None:
        if natoms == 1:
            if rest == 0 or rest % 50 == 25:
                has_box = False
            else:
                raise ValueError(f"AMBER mdcrd file with one atom: the {rest} bytes after the title fit frames with and "
                                 "without a box line alike (each line is 24 characters); pass box=True or box=False")
        else:
            after = t0 + frame_bytes(natoms, False)
            line = bytes(b[after:after + 25])
            has_box = len(line) == 25 and line[24] == 10 and b"\n" not in line[:24]
    else:
        has_box = bool(box)
    S = frame_bytes(natoms, has_box)
    F, cut = divmod(rest, S)
    if cut:
        logger.warning("AMBER mdcrd file: the last frame (frame %d) has %d of its %d bytes; it is dropped", F, cut, S)
    return dict(title=bytes(b[:nl]).decode("latin-1").rstrip(" "), has_box=has_box, frame_bytes=S, offset=t0,
                n_frames=int(F))


def decode_mdcrd_device(buf: torch.Tensor, offsets, natoms: int, with_box: bool, out: torch.Tensor | None = None,
                        box_out: torch.Tensor | None = None, bad: torch.Tensor | None = None):
    """K25 on the device: ``buf`` (uint8 CUDA tensor of staged frames, 16-byte aligned), ``offsets`` (int64 per listed
    frame: its byte offset in ``buf``, a multiple of 16) -> (coords (natoms, 3, F) float32, box (3, F) float32 or None,
    bad (1,) int64).  ``bad`` stays INT64_MAX on clean input, else holds the smallest k * S + b over the malformed bytes
    b of listed frame k (S = :func:`frame_bytes`).  ``out`` may be a frame slice of a larger (natoms, 3, F) tensor and
    ``box_out`` of a larger (3, F) one.  Nothing is synchronised."""
    dev = _lib.tensor_device(buf, "decode_mdcrd_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    offsets = np.ascontiguousarray(offsets, dtype=np.int64).reshape(-1)
    F = int(offsets.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    if box_out is None and with_box:
        box_out = torch.empty((3, F), dtype=torch.float32, device=dev)
    if bad is None:
        bad = torch.full((1,), INT64_MAX, dtype=torch.int64, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    box_stride = 1
    if with_box:
        assert box_out.shape == (3, F) and box_out.dtype == torch.float32 and box_out.device == dev
        assert F <= 1 or (box_out.stride(1) == 1 and box_out.stride(0) >= F), "box_out must be (3, F) frame-minor"
        box_stride = max(int(box_out.stride(0)), F, 1)
    assert bad.dtype == torch.int64 and bad.device == dev and bad.numel() >= 1
    if F == 0:
        return out, box_out, bad
    _lib.call(dev, "mkb_mdcrd_decode", _lib.ptr(buf), int(buf.numel()), offsets.ctypes.data_as(C.c_void_p), F,
              int(natoms), int(bool(with_box)), _lib.ptr(out), stride,
              _lib.ptr(box_out if with_box else None), box_stride, _lib.ptr(bad))
    return out, box_out, bad


def _malformed(filename, idx, natoms: int, frame: int, b: int) -> ValueError:
    """the error for byte ``b`` of file frame ``frame``: its 1-based line and column and the field, re-read from the
    file"""
    n = 3 * natoms
    L = (n + 9) // 10
    body = 24 * natoms + L
    if b < body:
        li, col = divmod(b, 81)
        width = 80 if li < L - 1 else 8 * (n - 10 * (L - 1))
    else:
        li, col, width = L, b - body, 24
    line = 2 + frame * (L + idx["has_box"]) + li
    start = idx["offset"] + frame * idx["frame_bytes"] + (li * 81 if b < body else body)  # the line's first byte
    with open(filename, "rb") as fh:
        if col == width:
            what = f"expected the newline that ends the line, found {os.pread(fh.fileno(), 1, start + col)!r}"
        else:
            col -= col % 8
            what = f"malformed field {os.pread(fh.fileno(), 8, start + col)!r} in columns {col + 1}-{col + 8}"
    return ValueError(f"AMBER mdcrd file {filename}, frame {frame} (natoms={natoms}, "
                      f"{'with' if idx['has_box'] else 'no'} box line), line {line}, column {col + 1}: {what}")


def _read(filename, natoms, frames, box, device, chunk_bytes):
    """The frames :func:`_trajio.select` picks -> (coords CUDA (natoms, 3, F), box (3, F) numpy, info)"""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    natoms = int(natoms)
    mm = np.memmap(filename, dtype=np.uint8, mode="r") if os.path.getsize(filename) else b""
    idx = index_mdcrd(mm, natoms, box)
    F, S, hb = idx["n_frames"], idx["frame_bytes"], idx["has_box"]
    sel = _trajio.select(F, frames)
    info = dict(title=idx["title"], has_box=hb, natoms=natoms, n_frames=F, frames=sel)
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((natoms, 3, n), dtype=torch.float32, device=dev)
    if n == 0:
        return coords, np.zeros((3, 0), np.float32), info
    del mm  # the frames are read with preadv: a copy from the page cache, without a page fault per 4 KiB
    row = (S + 15) & ~15  # every staged frame starts on a 16-byte boundary
    chunks = _trajio.chunks(sel, np.full(F, row, np.int64), int(chunk_bytes))
    box_d = torch.zeros((3, n), dtype=torch.float32, device=dev)
    bad = torch.full((len(chunks),), INT64_MAX, dtype=torch.int64, device=dev)  # one slot per chunk: no sync per chunk
    with open(filename, "rb") as fh:
        def stage(c, host):
            uniq = chunks[c][2]
            used = len(uniq) * row
            rows = host[:used].reshape(len(uniq), row)[:, :S]
            _trajio.gather_slabs(fh.fileno(), idx["offset"] + uniq * S, S, rows, "AMBER mdcrd")
            return used

        def consume(c, buf):
            k0, k1, uniq = chunks[c]
            decode_mdcrd_device(buf, np.searchsorted(uniq, sel[k0:k1]) * row, natoms, hb, out=coords[:, :, k0:k1],
                                box_out=box_d[:, k0:k1] if hb else None, bad=bad[c:c + 1])

        _trajio.upload(dev, len(chunks), max(len(u) for _, _, u in chunks) * row, stage, consume)
    worst = bad.cpu().numpy()
    box_h = box_d.cpu().numpy()
    hit = np.flatnonzero(worst != INT64_MAX)
    if len(hit):
        c = int(hit[0])
        k, b = divmod(int(worst[c]), S)
        raise _malformed(filename, idx, natoms, int(sel[chunks[c][0] + k]), b)
    return coords, box_h, info


def read_mdcrd_device(filename, natoms: int, frames=None, box: bool | None = None, device=None,
                      chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    (coords CUDA (natoms, 3, F) float32 [Angstrom], box (3, F) float32 numpy (A, B, C; zeros without a box line),
    info) with the trajectory left on the GPU.  ``box`` None detects the box line (see :func:`index_mdcrd`).  ``info``
    holds title, has_box, natoms, n_frames (frames in the file) and frames (the file frame of each returned frame).
    A malformed field or a misplaced newline raises ValueError naming the frame, the 1-based line and column and the
    field's bytes."""
    return _read(filename, natoms, frames, box, device, chunk_bytes)


def read_mdcrd(filename, natoms: int, box: bool | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (coords (natoms, 3, F) float32 [Angstrom], box (3, F) float32) as numpy arrays."""
    coords, bx, _ = _read(filename, natoms, None, box, device, chunk_bytes)
    return coords.cpu().numpy(), bx


def read_mdcrd_frames(filename, natoms: int, frames, box: bool | None = None, device=None,
                      chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_mdcrd` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, bx, _ = _read(filename, natoms, frames, box, device, chunk_bytes)
    return coords.cpu().numpy(), bx


# ------------------------------------------------------------------------------------------------------------ writing
def _title_line(title) -> bytes:
    if not isinstance(title, str):
        raise ValueError(f"title must be a str, got {type(title).__name__}")
    if not title.isascii() or "\n" in title or "\r" in title or len(title) > TITLE_WIDTH:
        raise ValueError(f"title must be ASCII, without a line break, at most {TITLE_WIDTH} characters: {title!r}")
    return (title.ljust(TITLE_WIDTH) + "\n").encode("ascii")


def _writer_args(coords, box, title, chunk_bytes):
    """shapes and the title checked before any device work; returns (natoms, F)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"an mdcrd frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    if box is not None:
        if tuple(box.shape) != (3, F):
            raise ValueError(f"box must be (3, F) = {(3, F)}, got {tuple(box.shape)}")
        if isinstance(box, torch.Tensor) and box.dtype != torch.float32:
            raise ValueError(f"box must be float32, got {box.dtype}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    _title_line(title)
    return natoms, F


def _check_range(a, name: str) -> None:
    """ValueError naming the first value of ``a`` ((natoms, 3, F) coords or (3, F) box) in file order that '%8.3f'
    cannot write in 8 characters"""
    bad = _trajio.first_bad(a, NEG_MIN, POS_MAX, 1000)
    if bad is not None:
        f, atom, axis, v = bad
        where = f"frame {f}, atom {atom}, axis {'xyz'[axis]}" if atom is not None else f"frame {f}, axis {'ABC'[axis]}"
        raise ValueError(f"{name} at {where} is {v!r}: an mdcrd field (%8.3f) holds -999.999 to 9999.999 and no NaN "
                         "or infinity")


def _prepare(coords, box, title, device, chunk_bytes):
    """every check, then (coords, box) as CUDA tensors (a CUDA tensor used where it is, numpy uploaded), natoms, F"""
    coords = _trajio.writer_coords(coords, "write_mdcrd")
    if box is not None and not isinstance(box, torch.Tensor):
        box = np.asarray(box, dtype=np.float32)
    natoms, F = _writer_args(coords, box, title, chunk_bytes)
    _check_range(coords, "coords")
    if box is not None:
        _check_range(box, "box")
    if F == 0:
        return None, None, natoms, F
    x = _trajio.on_device(coords, device)
    if box is not None:
        box = box.to(x.device) if isinstance(box, torch.Tensor) else _trajio.on_device(box, x.device)
    return x, box, natoms, F


def _encode(x, box, natoms: int, F: int, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = x.device
    x = _trajio.frame_minor(x)
    if box is not None and F > 1 and (box.stride(1) != 1 or box.stride(0) < F):
        box = box.contiguous()
    S = frame_bytes(natoms, box is not None)
    if out is None:
        out = torch.empty(F * S, dtype=torch.uint8, device=dev)
    if F == 0:
        return out[:0]
    _lib.call(dev, "mkb_mdcrd_encode", _lib.ptr(x), max(int(x.stride(1)), F), F, natoms, _lib.ptr(box),
              max(int(box.stride(0)), F) if box is not None else 1, _lib.ptr(out), int(out.numel()))
    return out[:F * S]


def encode_mdcrd_device(coords: torch.Tensor, box=None) -> torch.Tensor:
    """K25 on the device: ``coords`` (CUDA (natoms, 3, F) float32, frame-minor; a frame slice of a larger tensor is
    used in place), ``box`` (3, F) or None -> uint8 CUDA tensor of the F frames of :func:`write_mdcrd`'s file back to
    back (no title line).  Values outside the writable range raise ValueError."""
    _lib.tensor_device(coords, "encode_mdcrd_device")
    x, b, natoms, F = _prepare(coords, box, "", None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    return _encode(x, b, natoms, F)


def _emit(fh, x, box, natoms: int, F: int, title, chunk_bytes) -> None:
    fh.write(_title_line(title))
    if F == 0:
        return
    _trajio.write_encoded(fh, x.device, F, frame_bytes(natoms, box is not None), chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], None if box is None else box[:, f0:f1], natoms,
                                                      f1 - f0, out=out))


def mdcrd_bytes(coords, box=None, title: str = "", device=None, chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_mdcrd` writes, as a ``bytes`` object."""
    x, b, natoms, F = _prepare(coords, box, title, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, x, b, natoms, F, title, chunk_bytes)
    return fh.getvalue()


def write_mdcrd(filename, coords, box=None, title: str = "", device=None, chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write an AMBER ASCII trajectory with the frames formatted on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``box`` (3, F) (A, B, C in Angstrom) or None for frames without a box line.  ``title`` (ASCII, no line break, at
    most 80 characters) is padded to 80 columns on line 1.  Every value is written as '%8.3f' ten per line; the range
    rule and the error are in the module docstring.  The frames are encoded in chunks of at most ``chunk_bytes`` and
    each chunk is written while the next one encodes.  The file is created or truncated; arguments and values are
    checked before it is opened."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    x, b, natoms, F = _prepare(coords, box, title, device, chunk_bytes)
    with open(filename, "wb") as fh:
        _emit(fh, x, b, natoms, F, title, chunk_bytes)
