"""Multi-frame GROMACS GRO trajectories read and written on the GPU (K29).

GROMACS's text format: ``confout.gro`` (a run's last frame, with velocities), ``gmx trjconv -o traj.gro`` (many frames,
often with velocities) and equilibration snapshots.  A frame is N + 3 lines:

1. a title, free text; GROMACS writes ``... t= <time> step= <step>`` into it;
2. the atom count N, a free-format integer;
3. N atom lines ``"%5d%-5s%5s%5d"`` (resid, resname, atom name, serial), then three position fields of width w in nm,
   optionally followed by three velocity fields of width w in nm/ps.  GROMACS writes ``%8.3f`` and ``%8.4f`` by
   default; ``-ndec d`` writes width d + 5 with d decimals for positions and d + 1 for velocities;
4. a box line, free format: 3 values ``v1x v2y v3z`` or 9 values ``v1x v2y v3z v1y v1z v2x v2z v3x v3y``, in nm.

The reference reads it line by line with column slices and ``float()``; here:

- ``index_gro`` reads frame 0 on the host (N, w, the velocity flag, the topology: O(N) bytes) and streams the file
  through two pinned and two device buffers.  ``mkb_gro_index`` finds every newline on the device, keeps a running line
  count there, records where each frame starts (frame f is lines f (N + 3) ... f (N + 3) + N + 2) and checks each
  count line against N.
- ``read_gro_device`` stages the listed frames (any order, repeats allowed) whole, chunk by chunk; ``mkb_gro_decode``
  indexes their lines and parses the position (and velocity) fields of every atom line into the frame-minor
  ``(N, 3, F)`` float32 layout, and ``mkb_gro_head`` parses each frame's box line and title.
- ``write_gro`` formats on the device (``mkb_gro_encode``) from per-atom 20-byte prefixes and per-frame title and count
  lines built on the host.

Reader rules:

- N comes from frame 0's count line; every frame's count line must read N (its first field, ``int()``), else
  ValueError names the file, the frame and the 1-based line.
- Frame 0's first atom line decides the field width and the velocities, as GROMACS does: w is the distance between the
  first '.' at or after column 21 and the next '.', and a third '.' must follow at the same distance (else ValueError:
  inconsistent decimal spacing).  The file has velocities when that line holds 20 + 6w characters before its line end.
  Every atom line of every frame must then hold 20 + 3w (or 20 + 6w) characters, else ValueError naming the frame, line
  and column.  GROMACS instead drops the velocities of the whole file when a line lacks them; this reader is stricter.
- Every position and velocity is bit for bit ``np.float32(float(field))`` of its w-character column slice, in the
  file's units (nm, nm/ps); ``scale`` multiplies the positions only, as one float32 multiply.  A field ``float()``
  rejects raises ValueError naming frame, line and column.  A line the device leaves open (a byte >= 0x80, an
  underscore, a short line, an undecided rounding) is re-read on the host; ``info["host_lines"]`` counts them.
- The box line is split on ASCII whitespace and must hold 3 or 9 values, each ``np.float32(float(token))``; the box
  comes back as ``(3, 3, F)`` box vectors (rows), zeros where a 3-value line has none.
- ``info["time"]`` (float64, ps) is ``float()`` of the token after the first " t= " of the frame's title, NaN without
  one (or when ``float()`` rejects it); ``info["step"]`` (int64) is ``int()`` of the token after the first " step= ",
  -1 without one.
- The topology comes from frame 0: resid [0:5], resname [5:10], name [10:15], serial [15:20], text stripped.
- CRLF is read; a CR not followed by LF is an error.  Trailing whitespace-only lines are ignored; a last frame cut
  short by the end of the file is dropped with a warning.  A last line without a newline is read.

Writer rules: the title line is ``title``, then ``" t= %*.5f"`` with ``time`` and ``" step= %*d"`` with ``step``, the
widths fixed per file by the widest value (this writer's choice: every frame then has the same size and the encode is
data-parallel); ``"%5d\\n" % N``; per atom ``"%5d%-5s%5s%5d"`` with resid and serial modulo 100 000 (GROMACS's own
wrap), ``%8.3f`` positions and optionally ``%8.4f`` velocities; a box line of three ``%10.5f``, or nine in GRO order
when any off-diagonal component of any frame is non-zero (again one choice per file).  Positions are written with 3
decimals only.  Not supported: other ``-ndec`` precisions in written files, per-frame topology changes, a changing atom
count, compressed files and ``.g96``.
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
LOOKAHEAD = 64  # bytes past a chunk the index pass may read (a count line starting in the chunk)
FLAG_CAP = 1 << 20  # host lines recorded per read; past it every atom line of the listed frames is re-read
MAX_ATOMS = (2**31 - 1) // 69
MAX_WIDTH = 32  # widest field the decoder takes
INT64_MAX = 2**63 - 1
COORD = (-999999, 9999999)  # rint(x * 1000) that '%8.3f' writes in 8 characters
VELOCITY = (-999999, 9999999)  # rint(v * 10^4), '%8.4f'
BOX = (-9999999, 99999999)  # rint(b * 10^5): '%10.5f' with a leading space, so the box line splits into its values
ORDER = ((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 0), (1, 2), (2, 0), (2, 1))  # GRO's box fields as (vector, axis)
FIELD_NAMES = ("x", "y", "z", "vx", "vy", "vz")
WS = b" \t\n\v\f\r"  # the whitespace bytes.split(), int() and float() take (not 0x1c-0x1f, unlike str.split())


def _where(fn, frame: int, line: int, col: int) -> str:
    return f"GRO file {fn}, frame {frame}, line {line}, column {col}"


def _strip_cr(raw: bytes) -> bytes:
    return raw[:-1] if raw.endswith(b"\r") else raw


def _count(fn, raw: bytes, frame: int, line: int, natoms: int | None) -> int:
    """int() of the count line's first field; with ``natoms`` it must equal it"""
    toks = raw.split()
    col = len(raw) - len(raw.lstrip(WS)) + 1
    try:
        v = int(toks[0])
    except (IndexError, ValueError):
        raise ValueError(f"{_where(fn, frame, line, col)}: the atom count line {raw!r} does not start with an "
                         "integer") from None
    if natoms is not None and v != natoms:
        raise ValueError(f"{_where(fn, frame, line, col)}: the atom count is {v}, frame 0 has {natoms} (the atom count "
                         "must not change between frames)")
    return v


def _atom(fn, raw: bytes, frame: int, line: int, w: int, nf: int) -> np.ndarray:
    """the nf fields of width w after column 20 of an atom line as the reference reads them"""
    raw = _strip_cr(raw)
    cols = 20 + nf * w
    if len(raw) < cols:
        raise ValueError(f"{_where(fn, frame, line, len(raw) + 1)}: the atom line has {len(raw)} columns, an atom line "
                         f"of this file needs {cols} ({nf} fields of width {w} after column 20): {raw!r}")
    out = np.empty(nf, np.float32)
    for d in range(nf):
        tok = raw[20 + w * d:20 + w * (d + 1)]
        try:
            out[d] = np.float32(float(tok))
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line, 21 + w * d)}: the {FIELD_NAMES[d]} field {tok!r} is not a "
                             "number") from None
    return out


def _box(fn, raw: bytes, frame: int, line: int) -> np.ndarray:
    """the box line as (9,) float32 in GRO order (zeros past a 3-value line)"""
    toks = raw.split()
    if len(toks) not in (3, 9):
        raise ValueError(f"{_where(fn, frame, line, 1)}: the box line holds {len(toks)} values, a GRO box line holds "
                         f"3 or 9: {_strip_cr(raw)!r}")
    out = np.zeros(9, np.float32)
    for t, tok in enumerate(toks):
        try:
            out[t] = np.float32(float(tok))
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line, raw.find(tok) + 1)}: the box value {tok!r} is not a "
                             "number") from None
    return out


def _after(title: bytes, key: bytes):
    i = title.find(key)
    if i < 0:
        return None
    rest = title[i + len(key):].split()
    return rest[0] if rest else None


def _time(title: bytes) -> float:
    tok = _after(title, b" t= ")
    try:
        return float(tok) if tok is not None else float("nan")
    except ValueError:
        return float("nan")


def _step(title: bytes) -> int:
    tok = _after(title, b" step= ")
    try:
        return int(tok) if tok is not None else -1
    except ValueError:
        return -1


def _frame0(fn, fh, E: int) -> dict:
    """natoms, field width, velocity flag, title and topology from the lines of frame 0"""
    fh.seek(0)
    title = _strip_cr(fh.readline().removesuffix(b"\n"))
    natoms = _count(fn, _strip_cr(fh.readline().removesuffix(b"\n")), 0, 2, None)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"{_where(fn, 0, 2, 1)}: the atom count must be 1 to {MAX_ATOMS}, got {natoms}")
    rows = []
    for a in range(natoms):
        if fh.tell() >= E:
            break
        rows.append(_strip_cr(fh.readline().removesuffix(b"\n")))
    if not rows:
        raise ValueError(f"GRO file {fn}: frame 0 has no atom lines")
    first = rows[0]
    i = first.find(b".", 20)
    j = first.find(b".", i + 1) if i >= 0 else -1
    w = j - i
    if i < 0 or j < 0 or first.find(b".", j + 1) != j + w:
        raise ValueError(f"{_where(fn, 0, 3, 21)}: the decimal points of the first atom line are not equally spaced "
                         f"(inconsistent precision): {first!r}")
    if w > MAX_WIDTH:
        raise ValueError(f"{_where(fn, 0, 3, 21)}: fields of width {w}, at most {MAX_WIDTH} are read")
    velocities = len(first) >= 20 + 6 * w

    def num(a, row, b0, b1, what):
        s = row[b0:b1].strip()
        try:
            return int(s)
        except ValueError:
            raise ValueError(f"{_where(fn, 0, 3 + a, b0 + 1)}: the {what} {s!r} is not an integer") from None

    topology = dict(resid=np.array([num(a, r, 0, 5, "resid") for a, r in enumerate(rows)], np.int64),
                    resname=np.array([r[5:10].decode("latin-1").strip() for r in rows], dtype=object),
                    name=np.array([r[10:15].decode("latin-1").strip() for r in rows], dtype=object),
                    serial=np.array([num(a, r, 15, 20, "serial") for a, r in enumerate(rows)], np.int64))
    return dict(natoms=natoms, width=w, velocities=velocities, title=title.decode("latin-1"), topology=topology)


def _index(fn, fd, E: int, head: dict, dev, B: int) -> dict:
    natoms, w = head["natoms"], head["width"]
    P = natoms + 3
    cap = E // (natoms * (21 + 3 * w) + 9) + 2  # frames of lines of at least 1, 2, 21 + 3w and 6 bytes
    while True:
        state = torch.tensor([0, INT64_MAX, 0], dtype=torch.int64, device=dev)
        frame_off = torch.zeros(cap + 1, dtype=torch.int64, device=dev)  # + 1: the end of the last frame, set below
        status = torch.zeros(cap, dtype=torch.uint8, device=dev)

        def stage(c, host):
            n_read = min(B + LOOKAHEAD, E - c * B)
            _trajio.read_exact(fd, host[:n_read], c * B, "GRO")
            return n_read

        def consume(c, buf):
            _lib.call(dev, "mkb_gro_index", _lib.ptr(buf), min(B, E - c * B), int(buf.numel()), c * B, natoms,
                      _lib.ptr(state), _lib.ptr(frame_off), _lib.ptr(status), cap)

        _trajio.upload(dev, -(-E // B), min(B, E) + LOOKAHEAD, stage, consume)
        lines, lone_cr, past = (int(v) for v in state.cpu())
        if not past:
            break
        cap = past  # frames shorter than the shortest valid ones (short atom lines): index again with room for all
    lines += 1  # the last line ends at E, without a newline
    F, rest = divmod(lines, P)
    offsets = frame_off[:F + 1].cpu().numpy().copy()
    offsets[0] = 0
    if rest == 0:
        offsets[F] = E
    flagged = np.flatnonzero(status[1:F].cpu().numpy()) + 1
    errors = []
    if lone_cr != INT64_MAX:
        line, col = _trajio.line_col(fd, lone_cr)
        errors.append((lone_cr, ValueError(f"{_where(fn, line // P, line + 1, col)}: a CR that is not followed by LF "
                                           "ends a line; lone CR line endings are not supported")))
    for f in flagged.tolist():
        title = _trajio.line_at(fd, int(offsets[f]), E)
        pos = int(offsets[f]) + len(title) + 1
        try:
            _count(fn, _strip_cr(_trajio.line_at(fd, pos, E)), f, f * P + 2, natoms)
        except ValueError as e:
            errors.append((pos, e))
            break
    if errors:
        raise min(errors, key=lambda t: t[0])[1]
    if rest:
        logger.warning("GRO file %s: the last frame (frame %d) has %d of its %d lines; it is dropped", fn, F, rest, P)
    return dict(head, n_frames=int(F), offsets=offsets.astype(np.int64))


def index_gro(filename, device=None, chunk_bytes: int = CHUNK_BYTES) -> dict:
    """Find the frames of a GRO file on the device -> dict(natoms, n_frames, offsets ((F + 1,) int64: the file offset of
    each frame and the end of the last), width (the field width w), velocities (bool), title (frame 0's) and topology
    (frame 0's resid, resname, name and serial)).  The file goes through the device in chunks of ``chunk_bytes`` with
    one host sync at the end.  Count-line mismatches, inconsistent decimal spacing and lone CR line endings raise
    ValueError (see the module docstring)."""
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    with open(fn, "rb") as fh:
        E = _trajio.content_end(fh.fileno(), os.fstat(fh.fileno()).st_size)
        if E == 0:
            raise ValueError(f"GRO file {fn}: no frames (the file is empty or blank)")
        return _index(fn, fh.fileno(), E, _frame0(fn, fh, E), _lib.device(device), (int(chunk_bytes) + 15) & ~15)


def decode_gro_device(buf: torch.Tensor, n_staged: int, frame_of, natoms: int, width: int, velocities: bool,
                      out: torch.Tensor | None = None, vout: torch.Tensor | None = None, want_v: bool = False,
                      flags: torch.Tensor | None = None, frame_base: int = 0, flag_cap: int = FLAG_CAP):
    """K29 on the device: ``buf`` (uint8 CUDA tensor, 16-byte aligned: ``n_staged`` whole frames back to back, each
    ending in a newline except possibly the last), ``frame_of`` (int per listed frame: its staged frame), the file's
    field ``width`` and velocity flag -> (positions (natoms, 3, F) float32, velocities (natoms, 3, F) float32 or None,
    flags int64 (1 + flag_cap,)).  Velocities are decoded when ``vout`` is given or ``want_v``.  flags[0] counts the
    lines left to the host; flags[1 + j] holds (frame_base + k) * natoms + a for the first flag_cap of them.  ``out``
    and ``vout`` may be frame slices of larger (natoms, 3, F) tensors with the same strides.  Nothing is
    synchronised."""
    dev = _lib.tensor_device(buf, "decode_gro_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    frame_of = np.ascontiguousarray(frame_of, dtype=np.int32).reshape(-1)
    F = int(frame_of.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    if vout is None and want_v:
        vout = torch.empty_like(out)
    if vout is not None and not velocities:
        raise ValueError("velocities requested from a file without velocities")
    if flags is None:
        flags = torch.zeros(1 + flag_cap, dtype=torch.int64, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out, vout)
    assert flags.dtype == torch.int64 and flags.device == dev and flags.numel() >= 1 + flag_cap
    if F == 0:
        return out, vout, flags
    _lib.call(dev, "mkb_gro_decode", _lib.ptr(buf), int(buf.numel()), int(n_staged),
              frame_of.ctypes.data_as(C.c_void_p), F, int(natoms), int(width), int(bool(velocities)), _lib.ptr(out),
              _lib.ptr(vout), stride, int(frame_base), _lib.ptr(flags), int(flag_cap))
    return out, vout, flags


def _head_device(buf, at: np.ndarray, dev):
    """mkb_gro_head over the staged frames at staging offsets ``at`` -> device (box9, time, step, status)"""
    n = len(at) - 1
    # from pinned memory without a sync, so the upload loop keeps staging the next chunk meanwhile
    at_d = torch.from_numpy(np.ascontiguousarray(at, np.int64)).pin_memory().to(dev, non_blocking=True)
    box = torch.zeros(9 * n, dtype=torch.float32, device=dev)
    time = torch.empty(n, dtype=torch.float64, device=dev)
    step = torch.empty(n, dtype=torch.int64, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    _lib.call(dev, "mkb_gro_head", _lib.ptr(buf), _lib.ptr(at_d), n, _lib.ptr(box), _lib.ptr(time), _lib.ptr(step),
              _lib.ptr(status))
    return box, time, step, status


def _check_fields(fields) -> tuple:
    fields = (fields,) if isinstance(fields, str) else tuple(fields)
    if not fields or any(f not in ("x", "v") for f in fields) or len(set(fields)) != len(fields):
        raise ValueError(f"fields must name distinct blocks among 'x' and 'v', got {fields!r}")
    return fields


def _read(filename, frames, fields, scale, index, device, chunk_bytes):
    fn = _trajio.name(filename)
    fields = _check_fields(fields)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    s = np.float32(scale)
    if not np.isfinite(s):
        raise ValueError(f"scale must be finite, got {scale}")
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        if index is None:
            E = _trajio.content_end(fd, os.fstat(fd).st_size)
            if E == 0:
                raise ValueError(f"GRO file {fn}: no frames (the file is empty or blank)")
            head = _frame0(fn, fh, E)
            if "v" in fields and not head["velocities"]:
                raise ValueError(f"GRO file {fn} has no velocities")
            dev = _lib.device(device)
            idx = _index(fn, fd, E, head, dev, (int(chunk_bytes) + 15) & ~15)
        else:
            idx = index
            if "v" in fields and not idx["velocities"]:
                raise ValueError(f"GRO file {fn} has no velocities")
            dev = _lib.device(device)
        N, F, w, vel = int(idx["natoms"]), int(idx["n_frames"]), int(idx["width"]), bool(idx["velocities"])
        offs = np.asarray(idx["offsets"], np.int64)
        sel = _trajio.select(F, frames)
        n = len(sel)
        x = torch.empty((N, 3, n), dtype=torch.float32, device=dev)
        v = torch.empty((N, 3, n), dtype=torch.float32, device=dev) if "v" in fields else None
        box = np.zeros((3, 3, n), np.float32)
        info = dict(natoms=N, n_frames=F, frames=sel, width=w, velocities=vel, time=np.full(n, np.nan),
                    step=np.full(n, -1, np.int64), topology=idx["topology"], host_lines=0)
        out = {k: t for k, t in (("x", x), ("v", v)) if k in fields}
        if n == 0:
            return out, box, info
        flags = torch.zeros(1 + FLAG_CAP, dtype=torch.int64, device=dev)
        heads = []

        def decode(buf, at, frame_of, k0, k1):
            decode_gro_device(buf, len(at) - 1, frame_of, N, w, vel, out=x[:, :, k0:k1],
                              vout=None if v is None else v[:, :, k0:k1], flags=flags, frame_base=k0)
            heads.append(_head_device(buf, at, dev))

        chunks = _trajio.read_frames(fd, dev, sel, offs[:-1], np.diff(offs), chunk_bytes, "GRO", decode)
        box9 = np.empty((n, 9), np.float32)
        errors = []  # (1-based line, ValueError): the first bad box line and the first bad atom line
        for (k0, k1, uniq), (b_d, t_d, s_d, st_d) in zip(chunks, heads):
            row = np.searchsorted(uniq, sel[k0:k1])
            box9[k0:k1] = b_d.view(-1, 9).cpu().numpy()[row]
            info["time"][k0:k1] = t_d.cpu().numpy()[row]
            info["step"][k0:k1] = s_d.cpu().numpy()[row]
            status = st_d.cpu().numpy()[row]
            for j in np.flatnonzero(status).tolist():  # the host decides, and names a bad box line
                f = int(sel[k0 + j])
                raw = os.pread(fd, int(offs[f + 1] - offs[f]), int(offs[f])).split(b"\n")
                if status[j] & 1:
                    line = f * (N + 3) + N + 3
                    try:
                        box9[k0 + j] = _box(fn, raw[N + 2], f, line)
                    except ValueError as e:
                        errors.append((line, e))
                if status[j] & 2:
                    info["time"][k0 + j] = _time(_strip_cr(raw[0]))
                if status[j] & 4:
                    info["step"][k0 + j] = _step(_strip_cr(raw[0]))
        for t, (i, j) in enumerate(ORDER):
            box[i, j] = box9[:, t]
        k, a, _ = _trajio.flagged(flags, n, N, FLAG_CAP, 1)
        if len(k):
            bad = _host_lines(fn, fd, offs, sel, N, w, 6 if vel else 3, k, a, x, v)
            if bad is not None:
                errors.append(bad)
            info["host_lines"] = len(k)
        if errors:
            raise min(errors, key=lambda t: t[0])[1]
    if s != 1:
        x.mul_(float(s))  # one float32 multiply of the rounded value
    return out, box, info


def _host_lines(fn, fd, offs, sel, N, w, nf, k, a, x, v):
    """re-read atom lines (listed frame k, atom a) on the host and write their values -> None, or (1-based line,
    ValueError) of the first bad line in file order"""
    order = np.lexsort((a, sel[k]))
    vals = np.empty((len(k), nf), np.float32)
    frame_lines = {}
    for j in order.tolist():
        f, at = int(sel[k[j]]), int(a[j])
        if f not in frame_lines:
            frame_lines = {f: os.pread(fd, int(offs[f + 1] - offs[f]), int(offs[f])).split(b"\n")}
        line = f * (N + 3) + 3 + at
        try:
            vals[j] = _atom(fn, frame_lines[f][2 + at], f, line, w, nf)
        except ValueError as e:
            return line, e
    dev = x.device
    ai, ki = torch.from_numpy(a).to(dev), torch.from_numpy(k).to(dev)
    x[ai, :, ki] = torch.from_numpy(vals[:, :3].copy()).to(dev)
    if v is not None:
        v[ai, :, ki] = torch.from_numpy(vals[:, 3:].copy()).to(dev)
    return None


def read_gro_device(filename, frames=None, fields=("x",), scale: float = 1.0, index: dict | None = None, device=None,
                    chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    ({"x": positions, "v": velocities} for the blocks named in ``fields``, each CUDA (natoms, 3, F) float32 [nm, nm/ps],
    box (3, 3, F) float32 numpy [nm, box vectors as rows], info) with the trajectory left on the GPU.  ``scale``
    multiplies the positions only, as one float32 multiply (10: Angstrom from nm).  Asking for "v" from a file without
    velocities is a ValueError.  ``index`` (what :func:`index_gro` returned for this file) skips the index pass.
    ``info`` holds natoms, n_frames (frames in the file), frames (the file frame of each returned frame), width,
    velocities, time ((F,) float64), step ((F,) int64), topology (frame 0's) and host_lines (the atom lines re-read on
    the host).  Errors: see the module docstring."""
    return _read(filename, frames, fields, scale, index, device, chunk_bytes)


def read_gro(filename, scale: float = 1.0, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (positions (natoms, 3, F) float32 [nm, times ``scale``], box (3, 3, F) float32, time (F,) float64
    [ps, NaN without one], step (F,) int64 [-1 without one]) as numpy arrays, the return shape of ``read_trr`` (GRO
    titles carry time and step at full precision, hence float64 and int64).  The topology and the other details are in
    the ``info`` of :func:`read_gro_device`."""
    out, box, info = _read(filename, None, ("x",), scale, index, device, chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"], info["step"]


def read_gro_frames(filename, frames, scale: float = 1.0, index: dict | None = None, device=None,
                    chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_gro` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    out, box, info = _read(filename, frames, ("x",), scale, index, device, chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"], info["step"]


# ------------------------------------------------------------------------------------------------------------ writing
def _fields(topology, natoms: int) -> dict:
    """``topology`` (a Molecule / MolLite-like object or a dict) -> resid, resname, name, serial as natoms-long arrays;
    a missing resid is 1, a missing serial counts from 1, missing text is empty"""
    def get(k):
        v = topology.get(k) if isinstance(topology, dict) else getattr(topology, k, None)
        return None if v is None else np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v)

    out = {}
    for k in ("resid", "resname", "name", "serial"):
        v = get(k)
        if v is None:
            v = {"resid": np.ones(natoms, np.int64), "serial": np.arange(1, natoms + 1)}.get(k, np.full(natoms, "",
                                                                                                      object))
        v = np.asarray(v).reshape(-1) if np.ndim(v) else np.full(natoms, v)
        if len(v) != natoms:
            raise ValueError(f"topology field {k} has {len(v)} entries, coords have {natoms} atoms")
        out[k] = v
    return out


def _prefix(t: dict, natoms: int) -> np.ndarray:
    """ValueError for the first atom whose topology the GRO columns cannot hold, else the 20-byte "%5d%-5s%5s%5d"
    prefix of every atom as uint8 (natoms * 20,)"""
    bad = []
    for k in ("resname", "name"):
        for a, s in enumerate(t[k].tolist()):
            if not isinstance(s, str) or not s.isascii() or len(s) > 5 or s.split() != ([s] if s else []):
                bad.append((a, k, f"{s!r}: at most 5 ASCII characters without whitespace"))
                break
    for k in ("resid", "serial"):
        r = t[k].astype(np.float64)
        with np.errstate(invalid="ignore"):
            ok = np.isfinite(r) & (r == np.round(r)) & ((r >= 0) if k == "resid" else True)
        hit = np.flatnonzero(~ok)
        if len(hit):
            bad.append((int(hit[0]), k, f"{t[k].tolist()[hit[0]]!r}: " + ("a non-negative integer" if k == "resid"
                                                                          else "an integer")))
    if bad:
        a, k, why = min(bad)
        raise ValueError(f"topology at atom {a}, field {k} is {why}")
    rows = np.char.add(np.char.add(np.char.rjust(np.char.mod("%d", t["resid"].astype(np.int64) % 100000), 5),
                                   np.char.ljust(np.asarray(t["resname"], dtype=str), 5)),
                       np.char.add(np.char.rjust(np.asarray(t["name"], dtype=str), 5),
                                   np.char.rjust(np.char.mod("%d", t["serial"].astype(np.int64) % 100000), 5)))
    b = np.char.encode(np.asarray(rows, dtype="U20"), "ascii")
    assert b.dtype.itemsize == 20
    return np.frombuffer(b.tobytes(), np.uint8).copy()


def _per_frame(v, F: int, name: str, dtype):
    """``v`` (None, a scalar or one value per frame) -> (F,) float64, or int64 for ``dtype`` int; integer input is
    taken as int64 as it is, so steps past 2^53 keep every digit"""
    if v is None:
        return None
    v = np.asarray(_trajio.host(v))
    v = v.reshape(-1) if v.ndim else np.full(F, v)
    if len(v) != F:
        raise ValueError(f"{name} must hold one value per frame ({F}), got {len(v)}")
    if dtype is int and v.dtype.kind in "iu":
        if v.dtype.kind == "u" and len(v) and v.max() > np.iinfo(np.int64).max:
            raise ValueError(f"{name} at frame {int(np.argmax(v > np.iinfo(np.int64).max))} is past the int64 range")
        return v.astype(np.int64)
    v = v.astype(np.float64)
    if not np.isfinite(v).all():
        raise ValueError(f"{name} at frame {int(np.flatnonzero(~np.isfinite(v))[0])} is not finite")
    if dtype is int:
        if not (v == np.round(v)).all():
            raise ValueError(f"{name} at frame {int(np.flatnonzero(v != np.round(v))[0])} is not an integer")
        if not (np.abs(v) < 2.0 ** 63).all():
            raise ValueError(f"{name} at frame {int(np.flatnonzero(np.abs(v) >= 2.0 ** 63)[0])} is past the int64 "
                             "range")
        return v.astype(np.int64)
    return v


def _prepare(coords, topology, box, time, step, title, velocities, device, chunk_bytes):
    """every check, then (x, v, box as CUDA tensors or None without frames, natoms, F, head rows, prefix, box9)"""
    coords = _trajio.writer_coords(coords, "write_gro")
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"a GRO frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    if velocities is not None:
        velocities = _trajio.writer_coords(velocities, "write_gro")
        if tuple(velocities.shape) != (natoms, 3, F):
            raise ValueError(f"velocities must be (natoms, 3, F) = {(natoms, 3, F)}, got {tuple(velocities.shape)}")
        if isinstance(velocities, torch.Tensor) != isinstance(coords, torch.Tensor) or \
                (isinstance(coords, torch.Tensor) and velocities.device != coords.device):
            raise ValueError("velocities must be on the device of coords")
    if box is None:
        raise ValueError("box is required: (3, 3, F) box vectors in nm")
    if isinstance(box, torch.Tensor):
        if box.dtype != torch.float32:
            raise ValueError(f"box must be float32, got {box.dtype}")
    else:
        box = np.asarray(box, dtype=np.float32)
    if tuple(box.shape) != (3, 3, F):
        raise ValueError(f"box must be (3, 3, F) = {(3, 3, F)}, got {tuple(box.shape)}")
    if not isinstance(title, str) or not title.isascii() or "\n" in title or "\r" in title:
        raise ValueError(f"title must be an ASCII str without a line break: {title!r}")
    times = _per_frame(time, F, "time", float)
    steps = _per_frame(step, F, "step", int)
    t = _fields(topology, natoms)
    prefix = _prefix(t, natoms)
    bad = [(b, what) for b, what in ((_trajio.first_bad(coords, *COORD, 1000), "coords"),
                                     (_trajio.first_bad(velocities, *VELOCITY, 10000) if velocities is not None
                                      else None, "velocities"),
                                     (_trajio.first_bad(box, *BOX, 100000), "box")) if b is not None]
    if bad:
        (f, atom, axis, v), what = min(bad, key=lambda e: (e[0][0], e[1] != "coords", e[1] == "box"))
        field = dict(coords="'%8.3f' (-999.999 to 9999.999)", velocities="'%8.4f' (-99.9999 to 999.9999)",
                     box="'%10.5f' with a separating space (-99.99999 to 999.99999)")[what]
        at = (f"frame {f}, vector {atom}, axis {'xyz'[axis]}" if what == "box"
              else f"frame {f}, atom {atom}, axis {'xyz'[axis]}")
        raise ValueError(f"{what} at {at} is {v!r}: a GRO field {field} holds no such value, NaN or infinity")
    bh = _trajio.host(box)
    box9 = bool(F) and any(bool(np.any(bh[i, j] != 0)) for i, j in ORDER[3:])
    heads = _head_rows(title, times, steps, natoms, F)
    if F == 0:
        return None, None, None, natoms, F, heads, prefix, box9
    x = _trajio.on_device(coords, device)
    v = _trajio.on_device(velocities, x.device) if velocities is not None else None
    b = box.to(x.device) if isinstance(box, torch.Tensor) else _trajio.on_device(box, x.device)
    return x, v, b, natoms, F, heads, prefix, box9


def _head_rows(title: str, times, steps, natoms: int, F: int) -> np.ndarray:
    """the title and count lines of every frame, all of one length, as uint8 (F, H)"""
    rows = np.full(F, title, dtype=object)
    if times is not None:
        txt = np.char.mod("%.5f", times)
        rows = rows + " t= " + np.char.rjust(txt, max(np.char.str_len(txt).max(initial=0), 0)).astype(object)
    if steps is not None:
        txt = np.char.mod("%d", steps)
        rows = rows + " step= " + np.char.rjust(txt, max(np.char.str_len(txt).max(initial=0), 0)).astype(object)
    rows = rows + ("\n%5d\n" % natoms)
    H = len(rows[0]) if F else len(title) + 1 + len("%5d\n" % natoms)
    b = np.char.encode(np.asarray(rows.tolist(), dtype=f"U{H}"), "ascii") if F else np.zeros(0, f"S{H}")
    return np.frombuffer(b.tobytes(), np.uint8).reshape(F, H).copy()


def frame_bytes(natoms: int, head_bytes: int, velocities: bool, box9: bool) -> int:
    """bytes of one written frame: title and count lines, the atom lines and the box line"""
    return head_bytes + natoms * (69 if velocities else 45) + (91 if box9 else 31)


def _box_minor(b, F):
    """``b`` as it is when component (i, j) of frame k lies at (3 i + j) * b.stride(1) + k (what mkb_gro_encode reads),
    else a contiguous copy; the (3, 3) part is checked for one frame too"""
    if not (b.stride(0) == 3 * b.stride(1) and b.stride(1) >= F and (F == 1 or b.stride(2) == 1)):
        b = b.contiguous()
    return b


def _encode(x, v, box, natoms: int, F: int, head_d, prefix_d, box9: bool, out=None) -> torch.Tensor:
    dev = x.device
    x = _trajio.frame_minor(x)
    if v is not None:
        v = _trajio.frame_minor(v)
        if v.stride(1) != x.stride(1):  # the kernel reads both with one stride, for one frame too
            x, v = x.contiguous(), v.contiguous()
    box = _box_minor(box, F)
    H = int(head_d.shape[1])
    S = frame_bytes(natoms, H, v is not None, box9)
    if out is None:
        out = torch.empty(F * S, dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_gro_encode", _lib.ptr(x), _lib.ptr(v), max(int(x.stride(1)), F), F, natoms, _lib.ptr(head_d),
              H, _lib.ptr(prefix_d), _lib.ptr(box), int(box.stride(1)), int(box9), _lib.ptr(out),
              int(out.numel()))
    return out[:F * S]


def encode_gro_device(coords: torch.Tensor, topology, box, time=None, step=None, title: str = "",
                      velocities=None) -> torch.Tensor:
    """K29 on the device: ``coords`` (CUDA (natoms, 3, F) float32 in nm; a frame slice of a larger tensor is used in
    place) -> uint8 CUDA tensor of :func:`write_gro`'s file.  Values outside the writable range raise ValueError."""
    _lib.tensor_device(coords, "encode_gro_device")
    x, v, b, natoms, F, heads, prefix, box9 = _prepare(coords, topology, box, time, step, title, velocities, None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    return _encode(x, v, b, natoms, F, torch.from_numpy(heads).to(x.device), torch.from_numpy(prefix).to(x.device),
                   box9)


def _emit(fh, x, v, b, natoms: int, F: int, heads, prefix, box9, chunk_bytes) -> None:
    if F == 0:
        return
    head_d, prefix_d = torch.from_numpy(heads).to(x.device), torch.from_numpy(prefix).to(x.device)
    _trajio.write_encoded(fh, x.device, F, frame_bytes(natoms, heads.shape[1], v is not None, box9), chunk_bytes,
                          lambda f0, f1, out: _encode(x[:, :, f0:f1], None if v is None else v[:, :, f0:f1],
                                                      b[:, :, f0:f1], natoms, f1 - f0, head_d[f0:f1], prefix_d, box9,
                                                      out=out))


def gro_bytes(coords, topology, box, time=None, step=None, title: str = "", velocities=None, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_gro` writes, as a ``bytes`` object."""
    prep = _prepare(coords, topology, box, time, step, title, velocities, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, *prep, chunk_bytes)
    return fh.getvalue()


def write_gro(filename, coords, topology, box, time=None, step=None, title: str = "", velocities=None, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a multi-frame GRO file with the frames formatted on the GPU.  ``coords`` (natoms, 3, F) float32 in nm: a
    numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine); ``velocities`` the
    same in nm/ps, or None.  ``topology``: a Molecule / MolLite-like object or a dict with any of resid, resname, name
    and serial (a missing resid is 1, serials count from 1).  ``box`` (3, 3, F): box vectors as rows, in nm (required,
    as in ``write_trr``).  ``time`` (ps) and ``step``: one value per frame, or None to leave them out of the titles.
    The layout is in the module docstring.  Checked before the file is opened, each failure a ValueError naming the
    first offender: rint(x * 1000) and rint(v * 10^4) in [-999 999, 9 999 999]; rint(b * 10^5) in [-9 999 999,
    99 999 999], a '%10.5f' field that keeps a leading space, so that the free-format box line splits into its values
    (a box of 1 000 nm would fill all 10 columns and run into its neighbour); no NaN or infinity anywhere; resname and
    name at most 5 ASCII characters without whitespace; resid >= 0; the title ASCII without a line break; integer
    steps within int64.  The frames are encoded in chunks of at most ``chunk_bytes`` and each chunk is written while
    the next one encodes.  The file is created or truncated."""
    fn = _trajio.name(filename)
    prep = _prepare(coords, topology, box, time, step, title, velocities, device, chunk_bytes)
    with open(fn, "wb") as fh:
        _emit(fh, *prep, chunk_bytes)
