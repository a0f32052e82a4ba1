"""LAMMPS dump trajectories (``.lammpstrj``) read and written on the GPU (K32).

The text LAMMPS writes with ``dump atom`` and ``dump custom``: per frame the items ITEM: TIME (optional), ITEM:
TIMESTEP, ITEM: NUMBER OF ATOMS, ITEM: BOX BOUNDS (three bound lines, with tilts for a restricted-triclinic box) and
ITEM: ATOMS followed by one line per atom whose columns are named in that item's header.  Frame 0 may start with ITEM:
UNITS.  Atoms come in any order within a frame (each MPI rank's in turn unless ``dump_modify sort id``).

- ``index_lammpstrj`` parses frame 0 on the host (items, columns, ids and topology) and streams the file through the
  device: ``mkb_lammpstrj_index`` finds every newline, records where each frame starts (every frame after the first
  has frame 0's line count P) and checks each frame's ITEM lines against frame 0's and its atom count against N;
  ``mkb_lammpstrj_head`` parses TIMESTEP, TIME and the box lines of every frame.  A frame the device does not decide
  is checked on the host.
- ``read_lammpstrj_device`` stages the listed frames (any order, repeats allowed) and ``mkb_lammpstrj_decode`` parses
  the columns it needs, chosen by name, places each atom line in its row by id (rows in ascending id order of frame
  0; line order without an id column) and converts scaled (xs, xsu) coordinates and image flags through the frame's
  box: x = ((xlo + xs lx) + ys xy) + zs xz, y = (ylo + ys ly) + zs yz, z = zlo + zs lz, and with ``unwrap`` x += (ix lx +
  iy xy) + iz xz, y += iy ly + iz yz, z += iz lz, in float64 from float() of each token, rounded to float32 once.  With
  ``x`` and no unwrap every value is np.float32(float(token)).  The box comes back as (3, 3, F) float32 vectors a =
  (lx, 0, 0), b = (xy, ly, 0), c = (xz, yz, lz) with xlo = xlo_bound - min(0, xy, xz, xy + xz), xhi = xhi_bound - max(0,
  xy, xz, xy + xz), ylo = ylo_bound - min(0, yz), yhi = yhi_bound - max(0, yz).  A frame with an atom line outside the
  device grammar (a byte >= 0x80, an underscore, a token the 128-bit product cannot decide, a short line) is re-read on
  the host with split() / float() / int(); ``info["host_lines"]`` counts the lines re-read.
- ``write_lammpstrj`` writes each frame's header on the host as ``dump custom`` does and formats the atom lines
  ``"%d %d %.9g %.9g %.9g"`` on the device (``mkb_lammpstrj_encode``): a length pass, a scan and an emit pass.  '%.9g'
  is the shortest %g precision that round-trips every float32, so a written file reads back to the same bits (LAMMPS's
  own default, %g, keeps 6 digits).

Errors (ValueError naming the file, frame, 1-based line and column): a changed atom count (dynamic groups are not
supported), item order or ATOMS header; a duplicate, missing or unknown id; a field float() or int() rejects; a lone
CR line ending (CRLF is read); a general-triclinic box (BOX BOUNDS abc origin).  Whitespace-only trailing lines are
ignored and a truncated last frame is dropped with a warning.  Not supported: gzip and binary dumps, dump local,
atom counts that change between frames and custom ``dump_modify format`` strings in the writer.
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
MAX_ATOMS = (2**31 - 1) // 3
INT64_MAX = 2**63 - 1
G9_MAX = 15  # longest '%.9g' of a float32
STYLES = ("x", "xu", "xs", "xsu")
TRIPLES = {"x": ("x", "y", "z"), "xu": ("xu", "yu", "zu"), "xs": ("xs", "ys", "zs"), "xsu": ("xsu", "ysu", "zsu")}
BLOCKS = {"v": ("vx", "vy", "vz"), "f": ("fx", "fy", "fz")}
ROLE_ID, ROLE_POS, ROLE_IMG, ROLE_VEL, ROLE_FRC = 1, 2, 5, 8, 11
_FIELD = re.compile(r"\S+")


def _where(fn, frame: int, line: int, col: int) -> str:
    return f"LAMMPS dump file {fn}, frame {frame}, line {line}, column {col}"


def _text(fn, raw: bytes, frame: int, line: int) -> str:
    try:
        return raw.decode("utf-8").rstrip("\r")
    except UnicodeDecodeError as e:
        raise ValueError(f"{_where(fn, frame, line, e.start + 1)}: the line is not UTF-8 text") from None


class _Lines:
    """the lines of a file from a byte offset, without their '\\n' (not past ``end``)"""

    def __init__(self, fd: int, pos: int, end: int):
        self.fd, self.pos, self.end, self.buf = fd, pos, end, b""

    def next(self) -> bytes | None:
        while True:
            i = self.buf.find(b"\n")
            if i >= 0:
                out, self.buf = self.buf[:i], self.buf[i + 1:]
                return out
            if self.pos >= self.end:
                out, self.buf = self.buf, b""
                return out if out else None
            b = os.pread(self.fd, min(1 << 20, self.end - self.pos), self.pos)
            self.pos += len(b)
            self.buf += b


def _int(fn, text: str, frame: int, line: int, what: str) -> int:
    m = _FIELD.search(text)
    try:
        if m is None or m.end() != len(text.rstrip()):
            raise ValueError
        return int(m.group())
    except ValueError:
        raise ValueError(f"{_where(fn, frame, line, m.start() + 1 if m else 1)}: the {what} line {text!r} is not an "
                         "integer") from None


def _floats(fn, text: str, frame: int, line: int, n: tuple, what: str) -> list:
    toks = list(_FIELD.finditer(text))
    if len(toks) not in n:
        raise ValueError(f"{_where(fn, frame, line, 1)}: the {what} line holds {len(toks)} values, it must hold "
                         f"{' or '.join(map(str, n))}: {text!r}")
    out = []
    for m in toks:
        try:
            out.append(float(m.group()))
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line, m.start() + 1)}: the {what} value {m.group()!r} is not a "
                             "number") from None
    return out


def _header(fn, lines: _Lines, frame: int, line0: int, natoms: int | None) -> dict:
    """the header items of one frame (lines read from ``lines``, the first being 1-based file line ``line0``) -> dict
    (items, rows (the header lines without trailing whitespace), natoms, step, time, bounds (3, 3), tilt, columns and
    the line numbers of the values)"""
    h = dict(items=[], rows=[], time=np.nan, step_line=-1, time_line=-1, count_line=-1, box_line=-1)
    j = 0

    def get():
        nonlocal j
        raw = lines.next()
        if raw is None:
            raise ValueError(f"{_where(fn, frame, line0 + j, 1)}: the frame ends inside its header")
        t = _text(fn, raw, frame, line0 + j).rstrip()
        h["rows"].append(t)
        j += 1
        return t

    while True:
        item = get()
        if not item.startswith("ITEM: "):
            raise ValueError(f"{_where(fn, frame, line0 + j - 1, 1)}: {item!r} is not an ITEM line")
        name = item[6:]
        if name == "TIME":
            h["items"].append("TIME")
            h["time_line"] = j
            h["time"] = _floats(fn, get(), frame, line0 + j - 1, (1,), "TIME")[0]
        elif name == "TIMESTEP":
            h["items"].append("TIMESTEP")
            h["step_line"] = j
            h["step"] = _int(fn, get(), frame, line0 + j - 1, "TIMESTEP")
        elif name == "NUMBER OF ATOMS":
            h["items"].append("NUMBER OF ATOMS")
            h["count_line"] = j
            h["natoms"] = n = _int(fn, get(), frame, line0 + j - 1, "NUMBER OF ATOMS")
            if natoms is not None and n != natoms:
                raise ValueError(f"{_where(fn, frame, line0 + j - 1, 1)}: the atom count is {n}, frame 0 has {natoms} "
                                 "(the atom count must not change between frames: dynamic groups are not supported)")
        elif name.startswith("BOX BOUNDS"):
            words = name.split()[2:]
            if "abc" in words or "origin" in words:
                raise ValueError(f"{_where(fn, frame, line0 + j - 1, 1)}: a general triclinic box ({item!r}) is not "
                                 "supported, only orthogonal and restricted-triclinic bounds")
            h["items"].append("BOX BOUNDS")
            h["tilt"] = tilt = words[:3] == ["xy", "xz", "yz"]
            h["box_line"] = j
            b = np.zeros((3, 3))
            for d in range(3):
                v = _floats(fn, get(), frame, line0 + j - 1, (3,) if tilt else (2,), "box bound")
                b[d, :len(v)] = v
            h["bounds"] = b
        elif name.startswith("ATOMS"):
            h["items"].append("ATOMS")
            h["columns"] = name.split()[1:]
            h["H"] = j
            break
        else:
            raise ValueError(f"{_where(fn, frame, line0 + j - 1, 1)}: the item {item!r} is not read here (TIME, "
                             "TIMESTEP, NUMBER OF ATOMS, BOX BOUNDS and ATOMS are)")
    for need in ("TIMESTEP", "NUMBER OF ATOMS", "BOX BOUNDS"):
        if need not in h["items"]:
            raise ValueError(f"{_where(fn, frame, line0, 1)}: the frame has no ITEM: {need}")
    return h


def _same_layout(fn, h: dict, h0: dict, frame: int, line0: int) -> None:
    if h["items"] != h0["items"]:
        raise ValueError(f"{_where(fn, frame, line0, 1)}: the items are {h['items']}, frame 0 has {h0['items']} (the "
                         "item order must not change)")
    for j, (a, b) in enumerate(zip(h["rows"], h0["rows"])):
        if b.startswith("ITEM:") and a != b:
            raise ValueError(f"{_where(fn, frame, line0 + j, 1)}: the header line {a!r} differs from frame 0's {b!r} "
                             "(the ATOMS header and the other ITEM lines must not change)")


def _roles(columns, style: str, fields, unwrap: bool) -> np.ndarray:
    """the int8 role of each column up to the last one read"""
    role = np.zeros(len(columns), np.int8)
    if "id" in columns:
        role[columns.index("id")] = ROLE_ID
    if "x" in fields:
        for d, c in enumerate(TRIPLES[style]):
            role[columns.index(c)] = ROLE_POS + d
        if unwrap:
            for d, c in enumerate(("ix", "iy", "iz")):
                role[columns.index(c)] = ROLE_IMG + d
    for key, base in (("v", ROLE_VEL), ("f", ROLE_FRC)):
        if key in fields:
            for d, c in enumerate(BLOCKS[key]):
                role[columns.index(c)] = base + d
    return role[:int(np.flatnonzero(role)[-1]) + 1] if role.any() else role[:1]


def _atoms(fn, lines, frame: int, line0: int, columns, natoms: int, want: dict) -> tuple:
    """the atom lines of a frame on the host -> (ids (N,) int64 in line order, {column: values}); ``want`` maps a
    column name to int or float"""
    idx = {c: columns.index(c) for c in want}
    last = max(idx.values()) if idx else 0
    vals = {c: [] for c in want}
    for a in range(natoms):
        raw = lines[a] if isinstance(lines, list) else lines.next()
        if raw is None:
            raise ValueError(f"{_where(fn, frame, line0 + a, 1)}: the frame ends after {a} of its {natoms} atom lines")
        text = _text(fn, raw, frame, line0 + a)
        toks = list(_FIELD.finditer(text))
        if len(toks) <= last:
            raise ValueError(f"{_where(fn, frame, line0 + a, len(text) + 1)}: the atom line has {len(toks)} field(s), "
                             f"the ATOMS header names {len(columns)}: {text!r}")
        for c, kind in want.items():
            m = toks[idx[c]]
            try:
                vals[c].append(kind(m.group()))
            except ValueError:
                raise ValueError(f"{_where(fn, frame, line0 + a, m.start() + 1)}: the {c} field {m.group()!r} is not "
                                 f"{'an integer' if kind is int else 'a number'}") from None
    return vals


def _frame0(fn, fd: int, E: int) -> dict:
    """frame 0's header, columns, ids and topology"""
    lines = _Lines(fd, 0, E)
    first = lines.next()
    units, u, skip = None, 0, 0
    if first is not None and _text(fn, first, 0, 1).rstrip() == "ITEM: UNITS":
        raw = lines.next()
        units = _text(fn, raw or b"", 0, 2).strip()
        u, skip = 2, len(first) + 1 + len(raw or b"") + 1
    else:
        lines = _Lines(fd, 0, E)
    h = _header(fn, lines, 0, 1 + u, None)
    N, cols = h["natoms"], h["columns"]
    if not 1 <= N <= MAX_ATOMS:
        raise ValueError(f"{_where(fn, 0, 1 + u + h['count_line'], 1)}: the atom count must be 1 to {MAX_ATOMS}, got {N}")
    if len(set(cols)) != len(cols) or not cols:
        raise ValueError(f"{_where(fn, 0, u + h['H'], 1)}: the ATOMS header {cols!r} must name distinct columns")
    want = {c: int for c in ("id", "type", "mol") if c in cols}
    if "element" in cols:
        want["element"] = str
    line0 = 1 + u + h["H"]
    vals = _atoms(fn, lines, 0, line0, cols, N, want)
    if "id" in cols:
        ids = np.array(vals["id"], np.int64)
        order = np.argsort(ids, kind="stable")
        dup = np.flatnonzero(np.diff(ids[order]) == 0)
        if len(dup):
            a = int(max(order[dup[0]], order[dup[0] + 1]))
            raise ValueError(f"{_where(fn, 0, line0 + a, 1)}: the id {int(ids[a])} appears twice in the frame")
    else:
        ids, order = np.arange(1, N + 1, dtype=np.int64), np.arange(N)
    topo = dict(ids=ids[order])
    for c in ("type", "mol"):
        if c in vals:
            topo[c] = np.array(vals[c], np.int64)[order]
    topo.setdefault("type", np.ones(N, np.int64))
    if "element" in vals:
        topo["element"] = [vals["element"][i] for i in order.tolist()]
    h.update(units=units, units_lines=u, skip=skip, topology=topo, natoms=N)
    return h


def _params(bounds: np.ndarray) -> np.ndarray:
    """(F, 3, 3) bound lines -> (F, 9) float64 xlo ylo zlo lx ly lz xy xz yz, each a float64 step in the stated order"""
    out = np.empty((len(bounds), 9))
    for f, b in enumerate(bounds.tolist()):
        (xlb, xhb, xy), (ylb, yhb, xz), (zlb, zhb, yz) = b
        xlo = xlb - min(0.0, xy, xz, xy + xz)
        xhi = xhb - max(0.0, xy, xz, xy + xz)
        ylo = ylb - min(0.0, yz)
        yhi = yhb - max(0.0, yz)
        out[f] = (xlo, ylo, zlb, xhi - xlo, yhi - ylo, zhb - zlb, xy, xz, yz)
    return out


def _index(fn, fd: int, E: int, h0: dict, dev, B: int) -> dict:
    N, H, u = h0["natoms"], h0["H"], h0["units_lines"]
    P = H + N
    tmpl = ("\n".join(h0["rows"]) + "\n").encode("utf-8")
    item_bytes = sum(len(r) + 1 for r in h0["rows"] if r.startswith("ITEM:"))
    min_frame = item_bytes + 2 * (H - sum(r.startswith("ITEM:") for r in h0["rows"])) + 2 * N
    cap = E // min_frame + 2
    lookahead = max(4096, 4 * len(tmpl))
    ntilt = 1 if h0["tilt"] else 0
    state = torch.tensor([-u, INT64_MAX, 0, 0], dtype=torch.int64, device=dev)
    frame_off = torch.zeros(cap + 1, dtype=torch.int64, device=dev)
    status = torch.zeros(cap, dtype=torch.uint8, device=dev)
    step = torch.zeros(cap, dtype=torch.int64, device=dev)
    time = torch.zeros(cap, dtype=torch.float64, device=dev)
    bounds = torch.zeros(9 * cap, dtype=torch.float64, device=dev)
    hstatus = torch.zeros(cap, dtype=torch.uint8, device=dev)
    tmpl_d = torch.frombuffer(bytearray(tmpl), dtype=torch.uint8).to(dev)

    def stage(c, host):
        n_read = min(B + lookahead, E - c * B)
        _trajio.read_exact(fd, host[:n_read], c * B, "LAMMPS dump")
        return n_read

    def consume(c, buf):
        n = min(B, E - c * B)
        _lib.call(dev, "mkb_lammpstrj_index", _lib.ptr(buf), n, int(buf.numel()), c * B, P, N, _lib.ptr(tmpl_d), H,
                  h0["count_line"], _lib.ptr(state), _lib.ptr(frame_off), _lib.ptr(status), cap)
        _lib.call(dev, "mkb_lammpstrj_head", _lib.ptr(buf), n, int(buf.numel()), c * B, P, _lib.ptr(state),
                  _lib.ptr(frame_off), cap, h0["step_line"], h0["time_line"], h0["box_line"], ntilt, _lib.ptr(step),
                  _lib.ptr(time), _lib.ptr(bounds), _lib.ptr(hstatus))

    _trajio.upload(dev, -(-E // B), min(B, E) + lookahead, stage, consume)
    lines, lone_cr, past = (int(v) for v in state[:3].cpu())
    F, rest = divmod(lines + 1, P)  # the last line ends at E, without a newline
    if past:
        raise ValueError(f"LAMMPS dump file {fn}: frames of {P} lines take fewer bytes than frame 0's items allow (blank "
                         "or cut atom lines)")
    offsets = frame_off[:F + 1].cpu().numpy().copy()
    offsets[0] = h0["skip"]
    if rest == 0:
        offsets[F] = E
    steps = step[:F].cpu().numpy().copy()
    times = time[:F].cpu().numpy().copy() if h0["time_line"] >= 0 else np.full(F, np.nan)
    bnd = bounds[:9 * F].view(-1, 3, 3).cpu().numpy().copy()
    steps[0], times[0], bnd[0] = h0["step"], h0["time"], h0["bounds"]
    errors = []
    if lone_cr != INT64_MAX:
        line, col = _trajio.line_col(fd, lone_cr)
        errors.append((lone_cr, ValueError(f"{_where(fn, max(0, (line - u) // P), line + 1, col)}: a CR that is not "
                                           "followed by LF ends a line; lone CR line endings are not supported")))
    flagged = np.flatnonzero(status[1:F].cpu().numpy() | hstatus[1:F].cpu().numpy()) + 1
    for f in flagged.tolist():
        line0 = 1 + u + f * P
        try:
            h = _header(fn, _Lines(fd, int(offsets[f]), E), f, line0, N)
            _same_layout(fn, h, h0, f, line0)
        except ValueError as e:
            errors.append((int(offsets[f]), e))
            break
        steps[f], times[f], bnd[f] = h["step"], h["time"], h["bounds"]
    if errors:
        raise min(errors, key=lambda t: t[0])[1]
    if rest:
        logger.warning("LAMMPS dump file %s: the last frame (frame %d) has %d of its %d lines; it is dropped", fn, F,
                       rest, P)
    t = h0["topology"]
    return dict(natoms=N, n_frames=int(F), offsets=offsets.astype(np.int64), columns=list(h0["columns"]),
                units=h0["units"], H=H, header=h0, step=steps, time=times, bounds=bnd, ids=t["ids"], type=t["type"],
                **{k: t[k] for k in ("mol", "element") if k in t})


def index_lammpstrj(filename, device=None, chunk_bytes: int = CHUNK_BYTES) -> dict:
    """Find and check the frames of a LAMMPS dump file on the device -> dict(natoms, n_frames, offsets ((F + 1,) int64:
    the file offset of each frame and the end of the last), columns, units, step (F,) int64, time (F,) float64 (NaN
    without ITEM: TIME), bounds (F, 3, 3) float64 (the raw bound lines), ids, type (and mol, element when present:
    frame 0's, in ascending id order)).  Errors: see the module docstring."""
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        E = _trajio.content_end(fd, os.fstat(fd).st_size)
        if E == 0:
            raise ValueError(f"LAMMPS dump file {fn}: no frames (the file is empty or blank)")
        h0 = _frame0(fn, fd, E)
        return _index(fn, fd, E, h0, _lib.device(device), (int(chunk_bytes) + 15) & ~15)


def _choose(fn, columns, fields, style, unwrap) -> tuple:
    """the coordinate style read and whether image flags are added"""
    fields = tuple(fields)
    if not fields or any(f not in ("x", "v", "f") for f in fields) or len(set(fields)) != len(fields):
        raise ValueError(f"fields must name distinct blocks among 'x', 'v' and 'f', got {fields!r}")
    if style is not None and style not in STYLES:
        raise ValueError(f"style must be None or one of {STYLES}, got {style!r}")
    for key in ("v", "f"):
        if key in fields and not all(c in columns for c in BLOCKS[key]):
            raise ValueError(f"LAMMPS dump file {fn} has no {' '.join(BLOCKS[key])} columns")
    if style is None:
        style = next((s for s in STYLES if all(c in columns for c in TRIPLES[s])), None)
        if style is None and "x" in fields:
            raise ValueError(f"LAMMPS dump file {fn} has no coordinate columns (x y z, xu yu zu, xs ys zs or xsu ysu "
                             "zsu)")
    elif not all(c in columns for c in TRIPLES[style]):
        raise ValueError(f"LAMMPS dump file {fn} has no {' '.join(TRIPLES[style])} columns")
    add = bool(unwrap) and style in ("x", "xs")
    if add and not all(c in columns for c in ("ix", "iy", "iz")):
        raise ValueError(f"LAMMPS dump file {fn}: unwrap=True needs the ix iy iz columns with {style} coordinates")
    return fields, style, add


def _host_frame(fn, fd, offs, f: int, idx: dict, style: str, add: bool, fields, params) -> dict:
    """listed frame f re-read on the host -> {block: (N, 3) float32 in row order}; the first bad line raises"""
    h0, N, cols = idx["header"], idx["natoms"], idx["columns"]
    P, u = idx["H"] + N, h0["units_lines"]
    line0 = 1 + u + f * P + idx["H"]
    raw = os.pread(fd, int(offs[f + 1] - offs[f]), int(offs[f])).split(b"\n")[idx["H"]:]
    want = {}
    if "id" in cols:
        want["id"] = int
    if "x" in fields:
        want.update({c: float for c in TRIPLES[style]})
        if add:
            want.update({c: int for c in ("ix", "iy", "iz")})
    for key in ("v", "f"):
        if key in fields:
            want.update({c: float for c in BLOCKS[key]})
    vals = _atoms(fn, raw, f, line0, cols, N, want)
    if "id" in cols:
        ids = np.array(vals["id"], np.int64)
        row = np.searchsorted(idx["ids"], ids)
        seen = np.zeros(N, bool)
        for a, (i, r) in enumerate(zip(ids.tolist(), row.tolist())):
            if r >= N or idx["ids"][r] != i:
                raise ValueError(f"{_where(fn, f, line0 + a, 1)}: the id {i} is not an id of frame 0")
            if seen[r]:
                raise ValueError(f"{_where(fn, f, line0 + a, 1)}: the id {i} appears twice in the frame")
            seen[r] = True
    else:
        row = np.arange(N)
    out = {}
    if "x" in fields:
        xlo, ylo, zlo, lx, ly, lz, xy, xz, yz = params.tolist()
        x = np.empty((N, 3), np.float32)
        cx, cy, cz = (vals[c] for c in TRIPLES[style])
        for a in range(N):
            px, py, pz = cx[a], cy[a], cz[a]
            if style in ("xs", "xsu"):
                px, py, pz = ((xlo + px * lx) + py * xy) + pz * xz, (ylo + py * ly) + pz * yz, zlo + pz * lz
            if add:
                ix, iy, iz = (float(vals[c][a]) for c in ("ix", "iy", "iz"))
                px, py, pz = px + ((ix * lx + iy * xy) + iz * xz), py + (iy * ly + iz * yz), pz + iz * lz
            x[row[a]] = (px, py, pz)
        out["x"] = x
    for key in ("v", "f"):
        if key in fields:
            b = np.empty((N, 3), np.float32)
            b[row] = np.stack([np.array(vals[c], np.float64) for c in BLOCKS[key]], 1)
            out[key] = b
    return out


def decode_lammpstrj_device(buf: torch.Tensor, n_staged: int, frame_of, natoms: int, H: int, role, ids=None,
                            params=None, scaled: bool = False, unwrap: bool = False, out=None, vout=None, fout=None,
                            fstat=None):
    """K32 on the device: ``buf`` (uint8 CUDA tensor, 16-byte aligned: ``n_staged`` whole frames of H + natoms lines
    back to back), ``frame_of`` (int per listed frame: its staged frame), ``role`` (int8 per column, see
    ``mkb_lammpstrj_decode``), ``ids`` (None: ids 1..natoms, else frame 0's ascending int64 ids on the device),
    ``params`` ((F, 9) float64 CUDA: xlo ylo zlo lx ly lz xy xz yz per listed frame) -> (coords, vels, forces (natoms,
    3, F) float32 or None, fstat uint8 (F rounded up to 4,): bit 0 a line left to the host, bit 1 an id error).
    ``out`` / ``vout`` / ``fout`` may be frame slices of larger tensors.  Nothing is synchronised."""
    dev = _lib.tensor_device(buf, "decode_lammpstrj_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    frame_of = np.ascontiguousarray(frame_of, dtype=np.int32).reshape(-1)
    F = int(frame_of.shape[0])
    role = torch.as_tensor(np.asarray(role, np.int8)).to(dev)
    if fstat is None:
        fstat = torch.zeros(max(4, (F + 3) & ~3), dtype=torch.uint8, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out, vout, fout)
    if F == 0:
        return out, vout, fout, fstat
    _lib.call(dev, "mkb_lammpstrj_decode", _lib.ptr(buf), int(buf.numel()), int(n_staged),
              frame_of.ctypes.data_as(C.c_void_p), F, int(natoms), int(H), _lib.ptr(role), int(role.numel()),
              _lib.ptr(ids) if ids is not None else None, _lib.ptr(params) if params is not None else None,
              int(scaled), int(unwrap), _lib.ptr(out) if out is not None else None,
              _lib.ptr(vout) if vout is not None else None, _lib.ptr(fout) if fout is not None else None, stride,
              _lib.ptr(fstat))
    return out, vout, fout, fstat


def _read(filename, frames, fields, style, unwrap, scale, index, device, chunk_bytes):
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    s = np.float32(scale)
    if not np.isfinite(s):
        raise ValueError(f"scale must be finite, got {scale}")
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        dev = _lib.device(device)
        if index is None:
            E = _trajio.content_end(fd, os.fstat(fd).st_size)
            if E == 0:
                raise ValueError(f"LAMMPS dump file {fn}: no frames (the file is empty or blank)")
            h0 = _frame0(fn, fd, E)
            fields, style, add = _choose(fn, h0["columns"], fields, style, unwrap)
            idx = _index(fn, fd, E, h0, dev, (int(chunk_bytes) + 15) & ~15)
        else:
            idx = index
            fields, style, add = _choose(fn, idx["columns"], fields, style, unwrap)
        N, F, H = int(idx["natoms"]), int(idx["n_frames"]), int(idx["H"])
        offs = np.asarray(idx["offsets"], np.int64)
        sel = _trajio.select(F, frames)
        n = len(sel)
        out = {k: torch.empty((N, 3, n), dtype=torch.float32, device=dev) for k in fields}
        bounds = np.asarray(idx["bounds"])[sel]
        params = _params(bounds)
        box = np.zeros((3, 3, n), np.float32)
        for t, (i, j) in enumerate(((0, 0), (1, 1), (2, 2), (1, 0), (2, 0), (2, 1))):
            box[i, j] = params[:, 3 + t].astype(np.float32)
        info = dict(natoms=N, n_frames=F, frames=sel, style=style, columns=list(idx["columns"]), units=idx["units"],
                    time=np.asarray(idx["time"])[sel], step=np.asarray(idx["step"])[sel], bounds=bounds,
                    origin=params[:, :3].copy(), ids=idx["ids"], type=idx["type"], host_lines=0,
                    **{k: idx[k] for k in ("mol", "element") if k in idx})
        if n == 0:
            return out, box, info
        cols = idx["columns"]
        role = _roles(cols, style, fields, add)
        dense = "id" not in cols or np.array_equal(idx["ids"], np.arange(1, N + 1))
        ids_d = None if dense else torch.from_numpy(np.ascontiguousarray(idx["ids"], np.int64)).to(dev)
        params_d = torch.from_numpy(params).to(dev)
        stats = []

        def decode(buf, at, frame_of, k0, k1):
            _, _, _, st = decode_lammpstrj_device(
                buf, len(at) - 1, frame_of, N, H, role, ids_d, params_d[k0:k1], style in ("xs", "xsu"), add,
                *(out[k][:, :, k0:k1] if k in out else None for k in ("x", "v", "f")))
            stats.append(st)

        chunks = _trajio.read_frames(fd, dev, sel, offs[:-1], np.diff(offs), chunk_bytes, "LAMMPS dump", decode)
        fst = np.concatenate([st.cpu().numpy()[:k1 - k0] for st, (k0, k1, _) in zip(stats, chunks)])
        redo = np.flatnonzero(fst)
        if len(redo):
            done = {}
            for k in sorted(redo.tolist(), key=lambda k: int(sel[k])):  # file order: the first bad line raises
                f = int(sel[k])
                if f not in done:
                    done[f] = _host_frame(fn, fd, offs, f, idx, style, add, fields, params[k])
                for key, val in done[f].items():
                    out[key][:, :, k] = torch.from_numpy(val).to(dev)
            info["host_lines"] = N * len(redo)
    if s != 1 and "x" in out:
        out["x"].mul_(float(s))  # one float32 multiply of the rounded value
    return out, box, info


def read_lammpstrj_device(filename, frames=None, fields=("x",), style=None, unwrap: bool = False, scale: float = 1.0,
                          index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    ({"x": positions, "v": velocities, "f": forces} for the blocks named in ``fields``, each CUDA (natoms, 3, F)
    float32, rows in ascending id order of frame 0; box (3, 3, F) float32 numpy [box vectors as rows]; info) with the
    trajectory left on the GPU.  ``style`` (None: the first of x, xu, xs, xsu present) names the coordinate columns;
    ``unwrap`` adds the ix iy iz image flags to wrapped coordinates (a no-op for xu / xsu).  ``scale`` multiplies the
    positions only, as one float32 multiply (1: real and metal units are Angstrom already).  ``index`` (what
    :func:`index_lammpstrj` returned for this file) skips the index pass.  ``info`` holds natoms, n_frames, frames,
    style, columns, units, time (float64), step (int64), bounds ((F, 3, 3) float64 raw bound lines), origin ((F, 3)
    float64 xlo ylo zlo), ids, type (and mol, element when present) and host_lines.  Errors: see the module
    docstring."""
    return _read(filename, frames, fields, style, unwrap, scale, index, device, chunk_bytes)


def read_lammpstrj(filename, style=None, unwrap: bool = False, scale: float = 1.0, index: dict | None = None,
                   device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (positions (natoms, 3, F) float32, box (3, 3, F) float32, time (F,) float64 [NaN without ITEM:
    TIME], step (F,) int64) as numpy arrays, the return shape of ``read_gro``.  The topology and the other details are
    in the ``info`` of :func:`read_lammpstrj_device`."""
    out, box, info = _read(filename, None, ("x",), style, unwrap, scale, index, device, chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"], info["step"]


def read_lammpstrj_frames(filename, frames, style=None, unwrap: bool = False, scale: float = 1.0,
                          index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_lammpstrj` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    out, box, info = _read(filename, frames, ("x",), style, unwrap, scale, index, device, chunk_bytes)
    return out["x"].cpu().numpy(), box, info["time"], info["step"]


# ------------------------------------------------------------------------------------------------------------ writing
def _bound_rows(box: np.ndarray, origin: np.ndarray) -> np.ndarray:
    """(3, 3) float32 vectors and (3,) float64 origin -> (3, 3) float64 bound lines (lo_bound, hi_bound, tilt)"""
    lx, xy, ly, xz, yz, lz = (float(box[0, 0]), float(box[1, 0]), float(box[1, 1]), float(box[2, 0]), float(box[2, 1]),
                              float(box[2, 2]))
    ox, oy, oz = (float(v) for v in origin)
    return np.array([[ox + min(0.0, xy, xz, xy + xz), ox + lx + max(0.0, xy, xz, xy + xz), xy],
                     [oy + min(0.0, yz), oy + ly + max(0.0, yz), xz],
                     [oz, oz + lz, yz]])


def _ints(v, natoms: int, name: str, default) -> np.ndarray:
    if v is None:
        return default
    a = np.asarray(_trajio.host(v))
    if a.shape != (natoms,) or a.dtype.kind not in "iu":
        raise ValueError(f"{name} must be {natoms} integers (one per atom), got shape {a.shape} and dtype {a.dtype}")
    if a.dtype.kind == "u" and len(a) and a.max() > INT64_MAX:
        raise ValueError(f"{name} holds a value past the int64 range")
    return a.astype(np.int64)


def _per_frame(v, F: int, name: str, kind):
    if v is None:
        return None
    a = np.asarray(_trajio.host(v))
    a = a.reshape(-1) if a.ndim else np.full(F, a)
    if len(a) != F:
        raise ValueError(f"{name} must hold one value per frame ({F}), got {len(a)}")
    if kind is int:
        if a.dtype.kind not in "iu":
            f64 = a.astype(np.float64)
            bad = ~np.isfinite(f64) | (f64 != np.round(f64)) | (np.abs(f64) >= 2.0 ** 63)
            if bad.any():
                raise ValueError(f"{name} at frame {int(np.flatnonzero(bad)[0])} is not an int64 integer")
        return a.astype(np.int64)
    a = a.astype(np.float64)
    if not np.isfinite(a).all():
        raise ValueError(f"{name} at frame {int(np.flatnonzero(~np.isfinite(a))[0])} is not finite")
    return a


def _prepare(coords, box, step, time, ids, types, velocities, origin, units, device, chunk_bytes):
    """every check, then (x, v as CUDA tensors or None without frames, natoms, F, headers, ids, types)"""
    coords = _trajio.writer_coords(coords, "write_lammpstrj")
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"a LAMMPS dump frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    if velocities is not None:
        velocities = _trajio.writer_coords(velocities, "write_lammpstrj")
        if tuple(velocities.shape) != (natoms, 3, F):
            raise ValueError(f"velocities must be (natoms, 3, F) = {(natoms, 3, F)}, got {tuple(velocities.shape)}")
        if isinstance(velocities, torch.Tensor) != isinstance(coords, torch.Tensor) or \
                (isinstance(coords, torch.Tensor) and velocities.device != coords.device):
            raise ValueError("velocities must be on the device of coords")
    if box is None:
        raise ValueError("box is required: (3, 3, F) box vectors")
    if isinstance(box, torch.Tensor) and box.dtype != torch.float32:
        raise ValueError(f"box must be float32, got {box.dtype}")
    bh = np.asarray(_trajio.host(box), dtype=np.float32)
    if bh.shape != (3, 3, F):
        raise ValueError(f"box must be (3, 3, F) = {(3, 3, F)}, got {tuple(bh.shape)}")
    if not np.isfinite(bh).all():
        raise ValueError(f"box at frame {int(np.flatnonzero(~np.isfinite(bh).all((0, 1)))[0])} is not finite")
    upper = (bh[0, 1] != 0) | (bh[0, 2] != 0) | (bh[1, 2] != 0)
    if upper.any():
        raise ValueError(f"box at frame {int(np.flatnonzero(upper)[0])} is not restricted-triclinic: a LAMMPS box has "
                         "a = (lx, 0, 0), b = (xy, ly, 0), c = (xz, yz, lz)")
    if origin is None:
        org = np.zeros((F, 3))
    else:
        org = np.asarray(_trajio.host(origin), dtype=np.float64)
        org = np.broadcast_to(org, (F, 3)) if org.shape == (3,) else org
        if org.shape != (F, 3) or not np.isfinite(org).all():
            raise ValueError(f"origin must be (3,) or (F, 3) = {(F, 3)} finite values, got shape {org.shape}")
    steps = _per_frame(step, F, "step", int)
    times = _per_frame(time, F, "time", float)
    idv = _ints(ids, natoms, "ids", np.arange(1, natoms + 1, dtype=np.int64))
    tv = _ints(types, natoms, "types", np.ones(natoms, np.int64))
    if units is not None and (not isinstance(units, str) or not units.isascii() or not units or
                              units.split() != [units]):
        raise ValueError(f"units must be one ASCII word (real, metal, lj, ...), got {units!r}")
    vel = velocities is not None
    heads = []
    for f in range(F):
        h = []
        if units is not None and f == 0:
            h.append("ITEM: UNITS\n%s\n" % units)
        if times is not None:
            h.append("ITEM: TIME\n%.16g\n" % float(times[f]))
        h.append("ITEM: TIMESTEP\n%d\n" % (f if steps is None else int(steps[f])))
        h.append("ITEM: NUMBER OF ATOMS\n%d\n" % natoms)
        b = _bound_rows(bh[:, :, f], org[f])
        if b[0, 2] == 0 and b[1, 2] == 0 and b[2, 2] == 0:
            h.append("ITEM: BOX BOUNDS pp pp pp\n")
            h.extend("%-1.16e %-1.16e\n" % (r[0], r[1]) for r in b)
        else:
            h.append("ITEM: BOX BOUNDS xy xz yz pp pp pp\n")
            h.extend("%-1.16e %-1.16e %-1.16e\n" % tuple(r) for r in b)
        h.append("ITEM: ATOMS id type x y z%s\n" % (" vx vy vz" if vel else ""))
        heads.append("".join(h).encode("ascii"))
    if F == 0:
        return None, None, natoms, F, heads, idv, tv
    x = _trajio.on_device(coords, device)
    v = _trajio.on_device(velocities, x.device) if vel else None
    return x, v, natoms, F, heads, idv, tv


def _line_max(idv, tv, vel: bool) -> int:
    w = lambda a: max(len(str(int(a.min()))), len(str(int(a.max()))))
    return w(idv) + 1 + w(tv) + (6 if vel else 3) * (G9_MAX + 1) + 1


def _encode(x, v, natoms: int, f0: int, f1: int, heads, ids_d, types_d, line_max: int, out=None):
    """frames [f0, f1) -> (the uint8 device buffer, a device int64 holding the bytes written)"""
    dev = x.device
    xs = _trajio.frame_minor(x[:, :, f0:f1])
    vs = None if v is None else v[:, :, f0:f1]
    if vs is not None and vs.stride() != xs.stride():
        xs, vs = xs.contiguous(), vs.contiguous()
    F = f1 - f0
    hb = b"".join(heads[f0:f1])
    head_off = torch.from_numpy(np.concatenate([[0], np.cumsum([len(h) for h in heads[f0:f1]])]).astype(np.int64))
    head_d = torch.frombuffer(bytearray(hb), dtype=torch.uint8).to(dev) if hb else None
    cap = len(hb) + F * natoms * line_max
    if out is None:
        out = torch.empty(cap, dtype=torch.uint8, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    _lib.call(dev, "mkb_lammpstrj_encode", _lib.ptr(xs), _lib.ptr(vs) if vs is not None else None,
              max(int(xs.stride(1)), F), F, natoms, _lib.ptr(ids_d), _lib.ptr(types_d), line_max,
              _lib.ptr(head_d) if head_d is not None else None, _lib.ptr(head_off.to(dev)), len(hb), _lib.ptr(out),
              int(out.numel()), _lib.ptr(total))
    return out, total


def encode_lammpstrj_device(coords: torch.Tensor, box, step=None, time=None, ids=None, types=None, velocities=None,
                            origin=None, units=None) -> torch.Tensor:
    """K32 on the device: ``coords`` (CUDA (natoms, 3, F) float32) -> uint8 CUDA tensor of :func:`write_lammpstrj`'s
    file.  Arguments as :func:`write_lammpstrj`."""
    _lib.tensor_device(coords, "encode_lammpstrj_device")
    x, v, natoms, F, heads, idv, tv = _prepare(coords, box, step, time, ids, types, velocities, origin, units, None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    ids_d, types_d = torch.from_numpy(idv).to(x.device), torch.from_numpy(tv).to(x.device)
    out, total = _encode(x, v, natoms, 0, F, heads, ids_d, types_d, _line_max(idv, tv, v is not None))
    return out[:int(total.item())]


def _emit(fh, x, v, natoms: int, F: int, heads, idv, tv, chunk_bytes) -> None:
    if F == 0:
        return
    ids_d, types_d = torch.from_numpy(idv).to(x.device), torch.from_numpy(tv).to(x.device)
    lm = _line_max(idv, tv, v is not None)
    frame_max = max(len(h) for h in heads) + natoms * lm

    def encode(f0, f1, out):
        _, total = _encode(x, v, natoms, f0, f1, heads, ids_d, types_d, lm, out=out)
        return int(total.item())

    _trajio.write_encoded(fh, x.device, F, frame_max, chunk_bytes, encode)


def lammpstrj_bytes(coords, box, step=None, time=None, ids=None, types=None, velocities=None, origin=None, units=None,
                    device=None, chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_lammpstrj` writes, as a ``bytes`` object."""
    args = _prepare(coords, box, step, time, ids, types, velocities, origin, units, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, *args, chunk_bytes)
    return fh.getvalue()


def write_lammpstrj(filename, coords, box, step=None, time=None, ids=None, types=None, velocities=None, origin=None,
                    units=None, device=None, chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a LAMMPS dump file with the atom lines formatted on the GPU.  ``coords`` (natoms, 3, F) float32: a numpy
    array (uploaded to ``device``) or a CUDA tensor (used where it is).  ``box`` (3, 3, F) float32 box vectors as rows,
    restricted-triclinic (a = (lx, 0, 0), b = (xy, ly, 0), c = (xz, yz, lz)); ``origin`` (3,) or (F, 3) xlo ylo zlo
    (default 0).  ``step`` (default the frame index) and ``time`` (None: no ITEM: TIME) per frame; ``ids`` (default
    1..N) and ``types`` (default 1) per atom; ``velocities`` adds vx vy vz columns; ``units`` writes ITEM: UNITS before
    frame 0.  Each frame's header is written as LAMMPS's dump custom does (bounds '%-1.16e', tilts only for a tilted
    box) and each atom line is ``"%d %d %.9g %.9g %.9g[ %.9g %.9g %.9g]\\n"``, byte for byte Python's ``%`` of
    float(np.float32(v)) (NaN and infinities as Python spells them).  The frames are encoded in chunks of at most
    ``chunk_bytes`` and each chunk is written while the next one encodes.  The file is created or truncated; every
    argument is checked before it is opened."""
    fn = _trajio.name(filename)
    args = _prepare(coords, box, step, time, ids, types, velocities, origin, units, device, chunk_bytes)
    with open(fn, "wb") as fh:
        _emit(fh, *args, chunk_bytes)
