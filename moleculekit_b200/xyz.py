"""Multi-frame XYZ trajectories read and written on the GPU (K26).

The text format QM and ML-potential tools write (ASE, CP2K, ORCA, xtb, i-PI, the LAMMPS xyz dump): per frame a line
holding the atom count N, a comment line, and N lines ``element x y z [more fields]`` in Angstrom, fields separated by
whitespace and of no fixed width.  The reference reads it line by line with ``split()`` and ``float()``; here:

- ``index_xyz`` streams the file through two pinned and two device buffers.  ``mkb_xyz_index`` finds every newline on
  the device, keeps a running line count there, and records where each frame starts (frame f is lines [f (N + 2),
  (f + 1)(N + 2))) and whether its count line is N.  The host reads only frame 0 (N, the comment and the elements), the
  content end of the file, and the O(F) frame offsets.
- ``read_xyz_device`` stages the listed frames (any order, repeats allowed) whole, chunk by chunk, and
  ``mkb_xyz_decode`` indexes their lines and parses fields 1-3 of every atom line into the frame-minor ``(N, 3, F)``
  float32 layout.  Every coordinate is bit for bit ``np.float32(float(field))``: the decimal is rounded correctly to
  double, then to float32.  A line the device leaves open (a byte >= 0x80, an underscore, any field outside the plain
  decimal / nan / inf grammar, fewer than four fields, or a rounding the 128-bit product cannot decide) is re-read on
  the host with ``split()`` and ``float()``; ``info["host_lines"]`` counts them.
- ``write_xyz`` formats on the device (``mkb_xyz_encode``): per frame ``"%d\\n" % N``, the comment line, and per atom
  ``"%-*s %15.8f %15.8f %15.8f\\n"`` with the element column as wide as the longest element, byte for byte Python's
  ``%`` formatting.

Errors (ValueError naming the file, frame, 1-based line and column): a count line that is not N (the atom count must
not change), an atom line with fewer than four fields, a field ``float()`` rejects, and a lone CR line ending (CRLF is
read; a CR not followed by LF is not supported).  Lines after the last whole frame that hold only whitespace are
ignored; other trailing lines (a truncated last frame) are dropped with a warning.  A last line without a newline is
read.  Not supported: extended-XYZ ``Lattice=`` / ``Properties=`` parsing, per-frame comments (``comment`` is frame
0's), compressed files and an atom count that changes between frames.
"""
from __future__ import annotations

import ctypes as C
import io
import logging
import os
import re

import numpy as np
import torch

from . import _lib, _trajio

logger = logging.getLogger(__name__)

CHUNK_BYTES = 256 << 20
LOOKAHEAD = 64  # bytes past a chunk the index pass may read (a count line starting in the chunk)
MAX_ATOMS = (2**31 - 1) // 3
MAX_ELEMENT = 256  # widest element column the writer takes
FLAG_CAP = 1 << 20  # host lines recorded by position per read; past it every atom line of the listed frames is re-read
INT64_MAX = 2**63 - 1
POS_MAX, NEG_MIN = 99999999999999, -9999999999999  # rint(x * 1e8) that '%15.8f' writes in 15 characters
_FIELD = re.compile(r"\S+")


def _where(fn, frame: int, line: int, col: int) -> str:
    return f"XYZ file {fn}, frame {frame}, line {line}, column {col}"


def _text(fn, raw: bytes, frame: int, line: int) -> str:
    try:
        return raw.decode("utf-8")
    except UnicodeDecodeError as e:
        raise ValueError(f"{_where(fn, frame, line, e.start + 1)}: the line is not UTF-8 text") from None


def _count(fn, raw: bytes, frame: int, line: int, natoms: int | None) -> int:
    """int() of the count line's first field; with ``natoms`` it must equal it"""
    text = _text(fn, raw, frame, line)
    m = _FIELD.search(text)
    try:
        v = int(m.group())
    except (AttributeError, ValueError):
        raise ValueError(f"{_where(fn, frame, line, m.start() + 1 if m else 1)}: the atom count line {text!r} does "
                         "not start with an integer") from None
    if natoms is not None and v != natoms:
        raise ValueError(f"{_where(fn, frame, line, m.start() + 1)}: the atom count is {v}, frame 0 has {natoms} (the "
                         "atom count must not change between frames)")
    return v


def _atom(fn, raw: bytes, frame: int, line: int) -> np.ndarray:
    """fields 1-3 of an atom line as the reference reads them: np.float32(float(field))"""
    text = _text(fn, raw, frame, line)
    fields = list(_FIELD.finditer(text))
    if len(fields) < 4:
        col = len(text.rstrip("\r")) + 1
        raise ValueError(f"{_where(fn, frame, line, col)}: the atom line has {len(fields)} field(s), an atom line needs "
                         f"four (element x y z): {text!r}")
    out = np.empty(3, np.float32)
    for d in range(3):
        tok = fields[1 + d].group()
        try:
            out[d] = np.float32(float(tok))
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line, fields[1 + d].start() + 1)}: the {'xyz'[d]} field {tok!r} is "
                             "not a number") from None
    return out


def _frame0(fn, fh, E: int) -> tuple[int, str, list]:
    """natoms, comment and elements from the lines of frame 0"""
    fh.seek(0)
    natoms = _count(fn, fh.readline().removesuffix(b"\n"), 0, 1, None)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"{_where(fn, 0, 1, 1)}: the atom count must be 1 to {MAX_ATOMS}, got {natoms}")
    comment = _text(fn, fh.readline().removesuffix(b"\n"), 0, 2).removesuffix("\r")
    element = []
    for a in range(natoms):
        if fh.tell() >= E:
            break
        m = _FIELD.search(_text(fn, fh.readline(), 0, 3 + a))
        element.append(m.group() if m else "")
    return natoms, comment, element


def index_xyz(filename, device=None, chunk_bytes: int = CHUNK_BYTES) -> dict:
    """Find the frames of a multi-frame XYZ file on the device -> dict(natoms, n_frames, offsets ((F + 1,) int64: the
    file offset of each frame and the end of the last), element (list of str: field 0 of frame 0's atom lines), comment
    (str: frame 0's comment line)).  The file goes through the device in chunks of ``chunk_bytes`` with one host sync at
    the end.  Count-line mismatches and lone CR line endings raise ValueError (see the module docstring)."""
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    B = (int(chunk_bytes) + 15) & ~15
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        E = _trajio.content_end(fd, os.fstat(fd).st_size)
        if E == 0:
            raise ValueError(f"XYZ file {fn}: no frames (the file is empty or blank)")
        natoms, comment, element = _frame0(fn, fh, E)
        P = natoms + 2
        cap = E // (8 * natoms + 3) + 2  # frames of lines of at least 2, 1 and 8 bytes
        dev = _lib.device(device)
        state = torch.tensor([0, INT64_MAX, 0], dtype=torch.int64, device=dev)
        frame_off = torch.zeros(cap + 1, dtype=torch.int64, device=dev)  # + 1: the end of the last frame, set below
        status = torch.zeros(cap, dtype=torch.uint8, device=dev)

        def stage(c, host):
            n_read = min(B + LOOKAHEAD, E - c * B)
            _trajio.read_exact(fd, host[:n_read], c * B, "XYZ")
            return n_read

        def consume(c, buf):
            _lib.call(dev, "mkb_xyz_index", _lib.ptr(buf), min(B, E - c * B), int(buf.numel()), c * B, natoms,
                      _lib.ptr(state), _lib.ptr(frame_off), _lib.ptr(status), cap)

        _trajio.upload(dev, -(-E // B), min(B, E) + LOOKAHEAD, stage, consume)
        lines, lone_cr, past = (int(v) for v in state.cpu())
        lines += 1  # the last line ends at E, without a newline
        F, rest = divmod(lines, P)
        if past:
            _short_atom_line(fn, fd, natoms, E)  # only lines too short for four fields pack frames this densely
        offsets = frame_off[:F + 1].cpu().numpy().copy()
        offsets[0] = 0
        if rest == 0:
            offsets[F] = E
        flagged = np.flatnonzero(status[1:F].cpu().numpy()) + 1
        errors = []
        if lone_cr != INT64_MAX:
            line, col = _trajio.line_col(fd, lone_cr)
            errors.append((lone_cr, ValueError(f"{_where(fn, line // P, line + 1, col)}: a CR that is not followed by "
                                               "LF ends a line; lone CR line endings are not supported")))
        for f in flagged.tolist():
            try:
                _count(fn, _trajio.line_at(fd, int(offsets[f]), E), f, f * P + 1, natoms)
            except ValueError as e:
                errors.append((int(offsets[f]), e))
                break
        if errors:
            raise min(errors, key=lambda t: t[0])[1]
    if rest:
        logger.warning("XYZ file %s: the last frame (frame %d) has %d of its %d lines; it is dropped", fn, F, rest, P)
    return dict(natoms=natoms, n_frames=int(F), offsets=offsets.astype(np.int64), element=element, comment=comment)


def _short_atom_line(fn, fd: int, natoms: int, E: int) -> None:
    """raise the error of the first atom line with fewer than four fields (a host scan of the file's newlines)"""
    P, line, pos, step = natoms + 2, 0, 0, 64 << 20
    for w in range(0, E, step):
        b = np.frombuffer(os.pread(fd, min(step, E - w), w), np.uint8)
        ends = np.concatenate([w + np.flatnonzero(b == 10), [E] if w + len(b) == E else []]).astype(np.int64)
        for e in ends.tolist():
            if line % P >= 2 and e - pos < 8:
                raw = os.pread(fd, e - pos, pos)
                if len(raw.split()) < 4:
                    _atom(fn, raw, line // P, line + 1)
            line, pos = line + 1, e + 1
    raise RuntimeError(f"XYZ file {fn}: the frame index overflowed without a short atom line")


def decode_xyz_device(buf: torch.Tensor, n_staged: int, frame_of, natoms: int, out: torch.Tensor | None = None,
                      flags: torch.Tensor | None = None, frame_base: int = 0, flag_cap: int = FLAG_CAP):
    """K26 on the device: ``buf`` (uint8 CUDA tensor, 16-byte aligned: ``n_staged`` whole frames back to back, each
    ending in a newline except possibly the last), ``frame_of`` (int per listed frame: its staged frame) -> (coords
    (natoms, 3, F) float32, flags int64 (1 + 2 flag_cap,)).  flags[0] counts the lines left to the host; flags[1 + 2 j],
    flags[2 + 2 j] hold ((frame_base + k) * natoms + a, the line's byte offset from its frame's start) for the first
    flag_cap of them.  ``out`` may be a frame slice of a larger (natoms, 3, F) tensor.  Nothing is synchronised."""
    dev = _lib.tensor_device(buf, "decode_xyz_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    frame_of = np.ascontiguousarray(frame_of, dtype=np.int32).reshape(-1)
    F = int(frame_of.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    if flags is None:
        flags = torch.zeros(1 + 2 * flag_cap, dtype=torch.int64, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    assert flags.dtype == torch.int64 and flags.device == dev and flags.numel() >= 1 + 2 * flag_cap
    if F == 0:
        return out, flags
    _lib.call(dev, "mkb_xyz_decode", _lib.ptr(buf), int(buf.numel()), int(n_staged),
              frame_of.ctypes.data_as(C.c_void_p), F, int(natoms), _lib.ptr(out), stride, int(frame_base),
              _lib.ptr(flags), int(flag_cap))
    return out, flags


def _read(filename, frames, index, device, chunk_bytes):
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    idx = index if index is not None else index_xyz(fn, device, chunk_bytes)
    N, F, offs = int(idx["natoms"]), int(idx["n_frames"]), np.asarray(idx["offsets"], np.int64)
    sel = _trajio.select(F, frames)
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((N, 3, n), dtype=torch.float32, device=dev)
    info = dict(natoms=N, n_frames=F, frames=sel, element=list(idx["element"]), comment=idx["comment"], host_lines=0)
    if n == 0:
        return coords, info
    flags = torch.zeros(1 + 2 * FLAG_CAP, dtype=torch.int64, device=dev)
    with open(fn, "rb") as fh:
        fd = fh.fileno()

        def decode(buf, at, frame_of, k0, k1):
            decode_xyz_device(buf, len(at) - 1, frame_of, N, out=coords[:, :, k0:k1], flags=flags, frame_base=k0)

        _trajio.read_frames(fd, dev, sel, offs[:-1], np.diff(offs), chunk_bytes, "XYZ", decode)
        k, a, rel = _trajio.flagged(flags, n, N, FLAG_CAP, 2)
        if len(k):
            _host_lines(fn, fd, offs, sel, N, k, a, rel, coords)
            info["host_lines"] = len(k)
    return coords, info


def _host_lines(fn, fd, offs, sel, N, k, a, rel, coords) -> None:
    """re-read atom lines (listed frame k, atom a; rel = byte offset from the frame start, None: find it) on the host
    and write their coordinates; the first bad line in file order raises"""
    order = np.lexsort((a, sel[k]))
    vals = np.empty((len(k), 3), np.float32)
    frame_lines = {}
    for j in order.tolist():
        f, at = int(sel[k[j]]), int(a[j])
        if rel is None:
            if f not in frame_lines:
                frame_lines = {f: os.pread(fd, int(offs[f + 1] - offs[f]), int(offs[f])).split(b"\n")}
            raw = frame_lines[f][2 + at]
        else:
            raw = _trajio.line_at(fd, int(offs[f] + rel[j]), int(offs[f + 1]))
        vals[j] = _atom(fn, raw, f, f * (N + 2) + 3 + at)
    dev = coords.device
    coords[torch.from_numpy(a).to(dev), :, torch.from_numpy(k).to(dev)] = torch.from_numpy(vals).to(dev)


def read_xyz_device(filename, frames=None, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    (coords CUDA (natoms, 3, F) float32 [Angstrom], info) with the trajectory left on the GPU.  ``index`` (what
    :func:`index_xyz` returned for this file) skips the index pass.  ``info`` holds natoms, n_frames (frames in the
    file), frames (the file frame of each returned frame), element and comment (frame 0's) and host_lines (the atom
    lines re-read on the host).  Errors: see the module docstring."""
    return _read(filename, frames, index, device, chunk_bytes)


def read_xyz(filename, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (coords (natoms, 3, F) float32 numpy [Angstrom], info as :func:`read_xyz_device`)."""
    coords, info = _read(filename, None, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


def read_xyz_frames(filename, frames, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_xyz` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, info = _read(filename, frames, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


# ------------------------------------------------------------------------------------------------------------ writing
def _writer_args(coords, element, comment, chunk_bytes):
    """shapes, elements and the comment checked before any device work -> (natoms, F, head bytes, element column)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"an XYZ frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    if isinstance(element, str) or len(element) != natoms:
        raise ValueError(f"element must be a sequence of {natoms} strings (one per atom)")
    for a, e in enumerate(element):
        if not isinstance(e, str) or not e or not e.isascii() or e.split() != [e] or len(e) > MAX_ELEMENT:
            raise ValueError(f"element of atom {a} is {e!r}: an element must be a non-empty ASCII string without "
                             f"whitespace, at most {MAX_ELEMENT} characters")
    if not isinstance(comment, str):
        raise ValueError(f"comment must be a str, got {type(comment).__name__}")
    if not comment.isascii() or "\n" in comment or "\r" in comment:
        raise ValueError(f"comment must be ASCII, without a line break: {comment!r}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    width = max(len(e) for e in element)
    column = np.frombuffer("".join(e.ljust(width) for e in element).encode("ascii"), np.uint8)
    return natoms, F, f"{natoms}\n{comment}\n".encode("ascii"), column


def _check_range(a) -> None:
    """ValueError naming the first value of (natoms, 3, F) ``a`` in file order that '%15.8f' cannot write in 15
    characters"""
    bad = _trajio.first_bad(a, NEG_MIN, POS_MAX, 1e8)
    if bad is not None:
        f, atom, axis, v = bad
        raise ValueError(f"coords at frame {f}, atom {atom}, axis {'xyz'[axis]} is {v!r}: an XYZ field (%15.8f) holds "
                         "-99999.99999999 to 999999.99999999 and no NaN or infinity")


def _prepare(coords, element, comment, device, chunk_bytes):
    """every check, then (coords as a CUDA tensor or None without frames, natoms, F, head, column)"""
    coords = _trajio.writer_coords(coords, "write_xyz")
    natoms, F, head, column = _writer_args(coords, element, comment, chunk_bytes)
    _check_range(coords)
    if F == 0:
        return None, natoms, F, head, column
    return _trajio.on_device(coords, device), natoms, F, head, column


def frame_bytes(natoms: int, head: bytes, width: int) -> int:
    """bytes of one written frame: the head, then per atom the element column, three 16-byte fields and a newline"""
    return len(head) + natoms * (width + 49)


def _encode(x, natoms: int, F: int, head_d, column_d, width: int, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = x.device
    x = _trajio.frame_minor(x)
    S = int(head_d.numel()) + natoms * (width + 49)
    if out is None:
        out = torch.empty(F * S, dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_xyz_encode", _lib.ptr(x), max(int(x.stride(1)), F), F, natoms, _lib.ptr(head_d),
              int(head_d.numel()), _lib.ptr(column_d), width, _lib.ptr(out), int(out.numel()))
    return out[:F * S]


def _device_text(head, column, dev):
    return torch.frombuffer(bytearray(head), dtype=torch.uint8).to(dev), torch.from_numpy(column.copy()).to(dev)


def encode_xyz_device(coords: torch.Tensor, element, comment: str = "") -> torch.Tensor:
    """K26 on the device: ``coords`` (CUDA (natoms, 3, F) float32; a frame slice of a larger tensor is used in place)
    -> uint8 CUDA tensor of the F frames of :func:`write_xyz`'s file.  Values outside the writable range raise
    ValueError."""
    _lib.tensor_device(coords, "encode_xyz_device")
    x, natoms, F, head, column = _prepare(coords, element, comment, None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    width = len(column) // natoms
    return _encode(x, natoms, F, *_device_text(head, column, x.device), width)


def _emit(fh, x, natoms: int, F: int, head, column, chunk_bytes) -> None:
    if F == 0:
        return
    width = len(column) // natoms
    head_d, column_d = _device_text(head, column, x.device)
    _trajio.write_encoded(fh, x.device, F, frame_bytes(natoms, head, width), chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], natoms, f1 - f0, head_d, column_d, width,
                                                      out=out))


def xyz_bytes(coords, element, comment: str = "", device=None, chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_xyz` writes, as a ``bytes`` object."""
    x, natoms, F, head, column = _prepare(coords, element, comment, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, x, natoms, F, head, column, chunk_bytes)
    return fh.getvalue()


def write_xyz(filename, coords, element, comment: str = "", device=None, chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a multi-frame XYZ file with the frames formatted on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``element``: one non-empty ASCII string without whitespace per atom; ``comment``: one ASCII line for every frame.
    Per frame: ``"%d\\n" % natoms``, the comment, and per atom ``"%-*s %15.8f %15.8f %15.8f\\n"`` with the element
    column as wide as the longest element.  A value whose field would pass 15 characters (above 999999.99999999, below
    -99999.99999999), NaN or +-inf is rejected with an error naming the first offending frame, atom and axis.  The
    frames are encoded in chunks of at most ``chunk_bytes`` and each chunk is written while the next one encodes.  The
    file is created or truncated; arguments and values are checked before it is opened."""
    fn = _trajio.name(filename)
    x, natoms, F, head, column = _prepare(coords, element, comment, device, chunk_bytes)
    with open(fn, "wb") as fh:
        _emit(fh, x, natoms, F, head, column, chunk_bytes)
