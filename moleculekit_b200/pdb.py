"""Multi-model PDB trajectories read and written on the GPU (K28).

The format of NMR ensembles and of the trajectories VMD, PyMOL, mdtraj, OpenMM's PDBReporter and cpptraj export: fixed
columns, about 81 bytes per atom-frame, each frame a MODEL of ATOM / HETATM records.  The reference reads it line by
line and calls ``float()`` on three column slices per atom; here:

- ``index_pdb`` streams the file through two pinned and two device buffers.  ``mkb_pdb_index`` classifies every line
  start on the device, keeps a running atom record count there, and lists each MODEL, ENDMDL, END and CRYST1 record with
  the number of atom records before it.  The host derives the frames from that O(F) list and parses the topology from
  frame 0's bytes; it never reads the coordinate columns of later frames.
- ``read_pdb_device`` stages the listed frames (any order, repeats allowed) whole, chunk by chunk, and
  ``mkb_pdb_decode`` ranks the atom records of every staged frame and parses columns 31-54 of each into the frame-minor
  ``(N, 3, F)`` float32 layout.  ``mkb_pdb_cell`` parses the frames' CRYST1 records.
- ``write_pdb`` builds each atom's 81-byte line once on the host and formats the coordinates, the MODEL serials and the
  CRYST1 records on the device (``mkb_pdb_encode``).

Frame rules:

- An atom record is a line whose first six bytes are ``ATOM  `` or ``HETATM``.  Every other record is skipped (TER,
  ANISOU, REMARK, HETNAM, CONECT, MASTER, blank lines, ...).
- With MODEL records (``MODEL`` then a space or the line's end), each MODEL starts a frame that runs to the next MODEL,
  ENDMDL or END record, or to the end of the file; atom records outside such a frame belong to none.  Without MODEL
  records the file is one frame of the atom records before the first ENDMDL / END.  N is the atom record count of frame
  0, and every other frame must hold exactly N: otherwise ValueError names the frame, its MODEL serial and the 1-based
  line of its MODEL record.  A last model cut short by the end of the file (no ENDMDL / END after it) is dropped with a
  warning.
- A coordinate is bit for bit ``np.float32(float(line[30:38]))``, then ``[38:46]`` and ``[46:54]``: rounded once to
  double and once to float32.  The device tries the F8.3 fast path, then K26's general grammar within the field; a line
  it cannot decide goes to the host, and ``info["host_lines"]`` counts those.  An atom line shorter than 54 columns or
  a field ``float()`` rejects raises ValueError naming the file, frame, 1-based line and column.  CRLF is read; a CR not
  followed by LF is an error.
- A frame's cell is the last CRYST1 record before its first atom record (a, b, c in columns 7-33, alpha, beta, gamma in
  34-54), so one CRYST1 in the header applies to every frame.  Without one the box is zeros and the angles 90.
- The topology comes from frame 0's atom records with the PDB 3.3 columns: record 1-6, serial 7-11, name 13-16, altloc
  17, resname 18-21, chain 22, resid 23-26, insertion 27, occupancy 55-60, beta 61-66, segid 73-76, element 77-78 and
  charge 79-80 (``2+`` / ``1-``).  Blank columns read as "" for text, 0 for serial, resid and charge, and 0.0 for
  occupancy and beta.

The writer's per-frame layout is ``"MODEL %8d\\n"``, with a box ``"CRYST1%9.3f%9.3f%9.3f%7.2f%7.2f%7.2f P 1           1
\\n"``, N atom lines of 80 columns and ``"ENDMDL\\n"``; the file ends with ``"END\\n"``.  A name of 4 characters starts in
column 13, a shorter one in column 14 when the element has one letter, else in column 13; a resname of 4 characters
fills columns 18-21, a shorter one is right-justified in 18-20.  Serials are written modulo 100 000, this writer's choice
so that systems of any size can be written.  Not supported: CONECT / bonds, hybrid-36 serials, compressed files,
per-model topology differences and TER records in written files.
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
LOOKAHEAD = 16  # bytes past a chunk the index pass may read (the record name of a line starting at its end)
FLAG_CAP = 1 << 20  # host lines recorded per read; past it every atom line of the listed frames is re-read
MAX_ATOMS = (2**31 - 1) // 81
MAX_MODELS = 99999999  # the largest serial "MODEL %8d" writes
INT64_MAX = 2**63 - 1
REC_MODEL, REC_ENDMDL, REC_END, REC_CRYST1 = 2, 3, 4, 5
CELL_ROW = 64
ATOM_RECORDS = (b"ATOM  ", b"HETATM")
FIELDS = ("record", "serial", "name", "altloc", "resname", "chain", "resid", "insertion", "occupancy", "beta", "segid",
          "element", "charge")
TEXT = dict(record=6, name=4, altloc=1, resname=4, chain=1, insertion=1, segid=4, element=2)  # widest value
COORD = (-999999, 9999999)  # rint(x * 1000) that '%8.3f' writes in 8 characters
LENGTH = (-9999999, 99999999)  # rint(x * 1000), '%9.3f'
ANGLE = (-99999, 999999)  # rint(x * 100), '%7.2f'
OCCUPANCY = (-9999, 99999)  # rint(x * 100), '%6.2f'


def _where(fn, frame: int, line: int, col: int) -> str:
    return f"PDB file {fn}, frame {frame}, line {line}, column {col}"


def _is_atom(line: bytes) -> bool:
    return line[:6] in ATOM_RECORDS


def _first_atom(fn, fd: int, size: int) -> None:
    """ValueError for a file without an atom record (the host reads up to the first one)"""
    if size == 0:
        raise ValueError(f"PDB file {fn}: the file is empty")
    pos, carry, step = 0, b"\n", 1 << 20
    while pos < size:
        b = carry + os.pread(fd, min(step, size - pos), pos)
        if b"\nATOM  " in b or b"\nHETATM" in b:
            return
        carry = b[-7:]
        pos += step
    raise ValueError(f"PDB file {fn}: no ATOM or HETATM record")


def _marks(fn, fd: int, E: int, dev, B: int):
    """the index pass -> (sorted marks (M, 2) int64: file offset * 8 + kind, atom records before; total atom records;
    the file offset of the first lone CR or INT64_MAX)"""
    cap = 4096 + E // 2048
    while True:
        state = torch.tensor([0, INT64_MAX, 0], dtype=torch.int64, device=dev)
        marks = torch.empty(2 * cap, dtype=torch.int64, device=dev)

        def stage(c, host):
            n_read = min(B + LOOKAHEAD, E - c * B)
            _trajio.read_exact(fd, host[:n_read], c * B, "PDB")
            return n_read

        def consume(c, buf):
            _lib.call(dev, "mkb_pdb_index", _lib.ptr(buf), min(B, E - c * B), int(buf.numel()), c * B,
                      _lib.ptr(state), _lib.ptr(marks), cap)

        _trajio.upload(dev, -(-E // B), min(B, E) + LOOKAHEAD, stage, consume)
        total, lone_cr, n = (int(v) for v in state.cpu())
        if n <= cap:
            m = marks[:2 * n].view(n, 2).cpu().numpy()
            return m[np.argsort(m[:, 0], kind="stable")], total, lone_cr
        cap = n  # more records than the first guess: index again with room for all of them


def index_pdb(filename, device=None, chunk_bytes: int = CHUNK_BYTES) -> dict:
    """Find the frames of a PDB file on the device -> dict(natoms, n_frames, start, end ((F,) int64: the file bytes
    [start, end) of each frame, from its MODEL record to the record that ends it), cell ((F,) int64: the file offset of
    each frame's CRYST1 record, -1 without one), topology (frame 0's atom records, see the module docstring)).  The file
    goes through the device in chunks of ``chunk_bytes`` with one host sync at the end.  Frames whose atom count is not
    frame 0's and lone CR line endings raise ValueError (see the module docstring)."""
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    B = (int(chunk_bytes) + 15) & ~15
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        E = os.fstat(fd).st_size
        _first_atom(fn, fd, E)
        m, total, lone_cr = _marks(fn, fd, E, _lib.device(device), B)
        off, kind, before = m[:, 0] >> 3, m[:, 0] & 7, m[:, 1]
        bound = kind != REC_CRYST1
        b_off, b_kind, b_before = off[bound], kind[bound], before[bound]
        mi = np.flatnonzero(b_kind == REC_MODEL)
        if len(mi) == 0:  # one frame: from the file's start to the first ENDMDL / END
            start, a0 = np.zeros(1, np.int64), np.zeros(1, np.int64)
            nxt = np.zeros(1, np.int64)
        else:
            start, a0, nxt = b_off[mi], b_before[mi], mi + 1
        closed = nxt < len(b_off)
        end = np.where(closed, b_off[np.minimum(nxt, len(b_off) - 1)] if len(b_off) else E, E).astype(np.int64)
        a1 = np.where(closed, b_before[np.minimum(nxt, len(b_off) - 1)] if len(b_off) else total, total)
        count = (a1 - a0).astype(np.int64)
        errors = []
        if lone_cr != INT64_MAX:
            line, col = _trajio.line_col(fd, lone_cr)
            errors.append((lone_cr, ValueError(f"PDB file {fn}, line {line + 1}, column {col}: a CR that is not "
                                               "followed by LF ends a line; lone CR line endings are not supported")))
        N = int(count[0])
        if N == 0:
            line = _trajio.line_col(fd, int(start[0]))[0] + 1
            errors.append((int(start[0]), ValueError(f"PDB file {fn}: frame 0 (line {line}) holds no ATOM or HETATM "
                                                     "record")))
        F = len(count)
        if F > 1 and not closed[-1] and count[-1] < N:
            F -= 1
            logger.warning("PDB file %s: the last model (frame %d) has %d of its %d atom records; it is dropped", fn,
                           F, int(count[-1]), N)
        bad = np.flatnonzero(count[:F] != N)
        if len(bad) and N:
            f = int(bad[0])
            line, _ = _trajio.line_col(fd, int(start[f]))
            serial = _trajio.line_at(fd, int(start[f]), E)[6:].strip().decode("latin-1")
            errors.append((int(start[f]), ValueError(
                f"PDB file {fn}, frame {f} (MODEL {serial}, line {line + 1}): {int(count[f])} atom records, frame 0 "
                f"has {N} (every model must hold the same atoms)")))
        if errors:
            raise min(errors, key=lambda t: t[0])[1]
        c_off, c_before = off[kind == REC_CRYST1], before[kind == REC_CRYST1]
        ci = np.searchsorted(c_before, a0[:F], side="right") - 1
        cell = np.where(ci >= 0, c_off[np.maximum(ci, 0)] if len(c_off) else -1, -1).astype(np.int64)
        raw0 = os.pread(fd, int(end[0] - start[0]), int(start[0]))
        topology = _topology(fn, raw0, int(start[0]), fd)
    return dict(natoms=N, n_frames=int(F), start=start[:F].astype(np.int64), end=end[:F], cell=cell,
                topology=topology)


def _int_field(fn, fd, pos, line: bytes, a: int, b: int, what: str) -> int:
    s = line[a:b].strip()
    if not s:
        return 0
    try:
        return int(s)
    except ValueError:
        raise ValueError(f"{_where(fn, 0, _trajio.line_col(fd, pos)[0] + 1, a + 1)}: the {what} {s!r} is not an "
                         "integer") from None


def _float_field(fn, fd, pos, line: bytes, a: int, b: int, what: str) -> float:
    s = line[a:b].strip()
    if not s:
        return 0.0
    try:
        return float(s)
    except ValueError:
        raise ValueError(f"{_where(fn, 0, _trajio.line_col(fd, pos)[0] + 1, a + 1)}: the {what} {s!r} is not a "
                         "number") from None


def _charge(fn, fd, pos, line: bytes) -> float:
    s = line[78:80].strip()
    if not s:
        return 0.0
    try:
        return float(int(s[:-1]) * (-1 if s[-1:] == b"-" else 1)) if s[-1:] in (b"+", b"-") else float(int(s))
    except ValueError:
        raise ValueError(f"{_where(fn, 0, _trajio.line_col(fd, pos)[0] + 1, 79)}: the charge {s!r} is not an integer "
                         "with an optional trailing sign") from None


def _topology(fn, raw: bytes, base: int, fd: int) -> dict:
    """frame 0's atom records (the bytes ``raw`` at file offset ``base``) -> dict of per-atom arrays"""
    rows, pos = [], base
    for ln in raw.split(b"\n"):
        if _is_atom(ln):
            rows.append((pos, ln[:-1] if ln.endswith(b"\r") else ln))
        pos += len(ln) + 1

    def text(a, b):
        return np.array([ln[a:b].decode("latin-1").strip() for _, ln in rows], dtype=object)

    return dict(record=text(0, 6),
                serial=np.array([_int_field(fn, fd, p, ln, 6, 11, "serial") for p, ln in rows], np.int64),
                name=text(12, 16), altloc=text(16, 17), resname=text(17, 21), chain=text(21, 22),
                resid=np.array([_int_field(fn, fd, p, ln, 22, 26, "resid") for p, ln in rows], np.int64),
                insertion=text(26, 27),
                occupancy=np.array([_float_field(fn, fd, p, ln, 54, 60, "occupancy") for p, ln in rows], np.float32),
                beta=np.array([_float_field(fn, fd, p, ln, 60, 66, "beta") for p, ln in rows], np.float32),
                segid=text(72, 76), element=text(76, 78),
                charge=np.array([_charge(fn, fd, p, ln) for p, ln in rows], np.float32))


def decode_pdb_device(buf: torch.Tensor, n_staged: int, frame_of, natoms: int, out: torch.Tensor | None = None,
                      flags: torch.Tensor | None = None, frame_base: int = 0, flag_cap: int = FLAG_CAP):
    """K28 on the device: ``buf`` (uint8 CUDA tensor, 16-byte aligned: ``n_staged`` whole frames back to back, each
    starting a line and holding exactly ``natoms`` atom records), ``frame_of`` (int per listed frame: its staged frame)
    -> (coords (natoms, 3, F) float32, flags int64 (1 + flag_cap,)).  flags[0] counts the lines left to the host;
    flags[1 + j] holds (frame_base + k) * natoms + a for the first flag_cap of them.  ``out`` may be a frame slice of a
    larger (natoms, 3, F) tensor.  Nothing is synchronised."""
    dev = _lib.tensor_device(buf, "decode_pdb_device")
    assert buf.dtype == torch.uint8 and buf.is_contiguous()
    frame_of = np.ascontiguousarray(frame_of, dtype=np.int32).reshape(-1)
    F = int(frame_of.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    if flags is None:
        flags = torch.zeros(1 + flag_cap, dtype=torch.int64, device=dev)
    stride = _trajio.decode_outputs(dev, natoms, F, out)
    assert flags.dtype == torch.int64 and flags.device == dev and flags.numel() >= 1 + flag_cap
    if F == 0:
        return out, flags
    _lib.call(dev, "mkb_pdb_decode", _lib.ptr(buf), int(buf.numel()), int(n_staged),
              frame_of.ctypes.data_as(C.c_void_p), F, int(natoms), _lib.ptr(out), stride, int(frame_base),
              _lib.ptr(flags), int(flag_cap))
    return out, flags


def _atom_coords(fn, line: bytes, frame: int, line_no) -> np.ndarray:
    """columns 31-54 of an atom line as the reference reads them; ``line_no()`` gives its 1-based line for errors"""
    line = line[:-1] if line.endswith(b"\r") else line
    if len(line) < 54:
        raise ValueError(f"{_where(fn, frame, line_no(), len(line) + 1)}: the atom line has {len(line)} columns, an "
                         f"atom line needs 54 (x, y, z in columns 31-54): {line!r}")
    out = np.empty(3, np.float32)
    for d in range(3):
        tok = line[30 + 8 * d:38 + 8 * d]
        try:
            out[d] = np.float32(float(tok))
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line_no(), 31 + 8 * d)}: the {'xyz'[d]} field {tok!r} is not a "
                             "number") from None
    return out


def _host_lines(fn, fd, start, end, sel, N, k, a, coords) -> None:
    """re-read atom records (listed frame k, atom a) on the host and write their coordinates; the first bad line in
    file order raises"""
    order = np.lexsort((a, sel[k]))
    vals = np.empty((len(k), 3), np.float32)
    cached = (-1, None)
    for j in order.tolist():
        f, at = int(sel[k[j]]), int(a[j])
        if cached[0] != f:
            raw = os.pread(fd, int(end[f] - start[f]), int(start[f]))
            rows, pos = [], int(start[f])
            for ln in raw.split(b"\n"):
                if _is_atom(ln):
                    rows.append((pos, ln))
                pos += len(ln) + 1
            cached = (f, rows)
        pos, ln = cached[1][at]
        vals[j] = _atom_coords(fn, ln, f, lambda: _trajio.line_col(fd, pos)[0] + 1)
    dev = coords.device
    coords[torch.from_numpy(a).to(dev), :, torch.from_numpy(k).to(dev)] = torch.from_numpy(vals).to(dev)


def _cells(fn, fd, E: int, cell: np.ndarray, dev):
    """the (3, n) box and angles of the listed frames' CRYST1 offsets ``cell`` (-1: none), parsed on the device"""
    n = len(cell)
    box = np.zeros((3, n), np.float32)
    angles = np.full((3, n), 90.0, np.float32)
    uniq, inv = np.unique(cell, return_inverse=True)
    have = uniq >= 0
    if not have.any():
        return box, angles
    pos = uniq[have]
    rows = np.full((len(pos), CELL_ROW), 10, np.uint8)
    for i, p in enumerate(pos.tolist()):
        b = os.pread(fd, min(CELL_ROW, E - p), p)
        rows[i, :len(b)] = np.frombuffer(b, np.uint8)
    rows_d = torch.from_numpy(rows.reshape(-1)).to(dev)
    cells_d = torch.empty(6 * len(pos), dtype=torch.float32, device=dev)
    bad_d = torch.empty(len(pos), dtype=torch.int32, device=dev)
    _lib.call(dev, "mkb_pdb_cell", _lib.ptr(rows_d), len(pos), _lib.ptr(cells_d), _lib.ptr(bad_d))
    cells = cells_d.cpu().numpy().reshape(-1, 6)
    for i in np.flatnonzero(bad_d.cpu().numpy()).tolist():  # the host decides, and names a bad field
        line = _trajio.line_at(fd, int(pos[i]), E)
        line = line[:-1] if line.endswith(b"\r") else line
        line_no = _trajio.line_col(fd, int(pos[i]))[0] + 1
        if len(line) < 54:
            raise ValueError(f"PDB file {fn}, line {line_no}, column {len(line) + 1}: the CRYST1 record has "
                             f"{len(line)} columns, it needs 54: {line!r}")
        for d, (a, b) in enumerate(((6, 15), (15, 24), (24, 33), (33, 40), (40, 47), (47, 54))):
            try:
                cells[i, d] = np.float32(float(line[a:b]))
            except ValueError:
                raise ValueError(f"PDB file {fn}, line {line_no}, column {a + 1}: the CRYST1 field {line[a:b]!r} is "
                                 "not a number") from None
    full = np.zeros((len(uniq), 6), np.float32)
    full[:, 3:] = 90.0
    full[have] = cells
    picked = full[inv.reshape(-1)]
    return np.ascontiguousarray(picked[:, :3].T), np.ascontiguousarray(picked[:, 3:].T)


def _read(filename, frames, index, device, chunk_bytes):
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    idx = index if index is not None else index_pdb(fn, device, chunk_bytes)
    N, F = int(idx["natoms"]), int(idx["n_frames"])
    start, end = np.asarray(idx["start"], np.int64), np.asarray(idx["end"], np.int64)
    sel = _trajio.select(F, frames)
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((N, 3, n), dtype=torch.float32, device=dev)
    info = dict(natoms=N, n_frames=F, frames=sel, topology=idx["topology"], host_lines=0,
                box=np.zeros((3, n), np.float32), boxangles=np.full((3, n), 90.0, np.float32))
    if n == 0:
        return coords, info
    flags = torch.zeros(1 + FLAG_CAP, dtype=torch.int64, device=dev)
    with open(fn, "rb") as fh:
        fd = fh.fileno()

        def decode(buf, at, frame_of, k0, k1):
            decode_pdb_device(buf, len(at) - 1, frame_of, N, out=coords[:, :, k0:k1], flags=flags, frame_base=k0)

        _trajio.read_frames(fd, dev, sel, start, end - start, chunk_bytes, "PDB", decode)
        E = os.fstat(fd).st_size
        info["box"], info["boxangles"] = _cells(fn, fd, E, np.asarray(idx["cell"], np.int64)[sel], dev)
        k, a, _ = _trajio.flagged(flags, n, N, FLAG_CAP, 1)
        if len(k):
            _host_lines(fn, fd, start, end, sel, N, k, a, coords)
            info["host_lines"] = len(k)
    return coords, info


def read_pdb_device(filename, frames=None, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    (coords CUDA (natoms, 3, F) float32 [Angstrom], info) with the trajectory left on the GPU.  ``index`` (what
    :func:`index_pdb` returned for this file) skips the index pass.  ``info`` holds natoms, n_frames (frames in the
    file), frames (the file frame of each returned frame), box and boxangles ((3, F) float32 numpy), topology (frame
    0's atom records) and host_lines (the atom lines re-read on the host).  Errors: see the module docstring."""
    return _read(filename, frames, index, device, chunk_bytes)


def read_pdb(filename, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (coords (natoms, 3, F) float32 numpy [Angstrom], info as :func:`read_pdb_device`)."""
    coords, info = _read(filename, None, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


def read_pdb_frames(filename, frames, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_pdb` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, info = _read(filename, frames, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


# ------------------------------------------------------------------------------------------------------------ writing
def topology_fields(topology, natoms: int) -> dict:
    """``topology`` (a Molecule / MolLite-like object or a dict) -> a dict of the FIELDS as natoms-long arrays; a
    missing field takes the reader's blank default (serial: 1 ... natoms)"""
    def get(k):
        v = topology.get(k) if isinstance(topology, dict) else getattr(topology, k, None)
        return None if v is None else np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v)

    out = {}
    for k in FIELDS:
        v = get(k)
        if v is None:
            v = {"record": np.full(natoms, "ATOM", object), "serial": np.arange(1, natoms + 1),
                 "resid": np.zeros(natoms, np.int64), "occupancy": np.zeros(natoms), "beta": np.zeros(natoms),
                 "charge": np.zeros(natoms)}.get(k, np.full(natoms, "", object))
        v = np.asarray(v).reshape(-1) if np.ndim(v) else np.full(natoms, v)
        if len(v) != natoms:
            raise ValueError(f"topology field {k} has {len(v)} entries, coords have {natoms} atoms")
        out[k] = v
    return out


_fields = topology_fields  # the name bench_pdb.py, bench_cif.py and the tests build writer templates with


def _check_topology(t: dict, natoms: int) -> None:
    """ValueError naming the first atom and field that the PDB columns cannot hold"""
    bad = []  # (atom, field, reason)
    for k, width in TEXT.items():
        for a, s in enumerate(t[k].tolist()):
            if not isinstance(s, str) or not s.isascii() or len(s) > width or any(c in s for c in "\n\r"):
                bad.append((a, k, f"{s!r}: at most {width} ASCII characters"))
                break
            if k == "record" and s not in ("ATOM", "HETATM"):
                bad.append((a, k, f"{s!r}: ATOM or HETATM"))
                break

    def first(k, ok, reason):
        with np.errstate(invalid="ignore", over="ignore"):
            hit = np.flatnonzero(~ok)
        if len(hit):
            bad.append((int(hit[0]), k, f"{t[k].tolist()[hit[0]]!r}: {reason}"))

    for k in ("serial", "resid", "charge"):
        v = t[k].astype(np.float64)
        first(k, np.isfinite(v) & (v == np.round(v)), "an integer")
    r = t["resid"].astype(np.float64)
    first("resid", (r >= -999) & (r <= 9999), "within '%4d' (-999 to 9999)")
    c = t["charge"].astype(np.float64)
    first("charge", (c >= -9) & (c <= 9), "-9 to 9")
    for k in ("occupancy", "beta"):
        with np.errstate(invalid="ignore", over="ignore"):
            q = np.rint(t[k].astype(np.float64) * 100)
        first(k, (q >= OCCUPANCY[0]) & (q <= OCCUPANCY[1]), "within '%6.2f' (-99.99 to 999.99)")
    if bad:
        a, k, why = min(bad)
        raise ValueError(f"topology at atom {a}, field {k} is {why}")


def _template(t: dict, natoms: int) -> np.ndarray:
    """the 81-byte line of every atom with columns 31-54 left blank, as uint8 (natoms * 81 rounded up to 4,)"""
    line = np.full((natoms, 81), ord(" "), np.uint8)
    line[:, 80] = 10

    def put(col, strs, width):
        b = np.char.encode(np.asarray(strs, dtype=f"U{width}"), "ascii")
        assert b.dtype.itemsize == width
        line[:, col:col + width] = np.frombuffer(b.tobytes(), np.uint8).reshape(natoms, width)

    def s(k):
        return np.asarray(t[k], dtype=str)

    el, name, rn = s("element"), s("name"), s("resname")
    put(0, np.char.ljust(s("record"), 6), 6)
    put(6, np.char.rjust(np.char.mod("%d", t["serial"].astype(np.int64) % 100000), 5), 5)
    nlen = np.char.str_len(name)
    put(12, np.where(nlen == 4, name, np.where(np.char.str_len(el) == 1, np.char.add(" ", np.char.ljust(name, 3)),
                                                np.char.ljust(name, 4))), 4)
    put(16, np.char.ljust(s("altloc"), 1), 1)
    put(17, np.where(np.char.str_len(rn) == 4, rn, np.char.add(np.char.rjust(rn, 3), " ")), 4)
    put(21, np.char.ljust(s("chain"), 1), 1)
    put(22, np.char.rjust(np.char.mod("%d", t["resid"].astype(np.int64)), 4), 4)
    put(26, np.char.ljust(s("insertion"), 1), 1)
    put(54, np.char.mod("%6.2f", t["occupancy"].astype(np.float64)), 6)
    put(60, np.char.mod("%6.2f", t["beta"].astype(np.float64)), 6)
    put(72, np.char.ljust(s("segid"), 4), 4)
    put(76, np.char.rjust(el, 2), 2)
    ch = t["charge"].astype(np.int64)
    put(78, np.where(ch == 0, "  ", np.char.add(np.char.mod("%d", np.abs(ch)), np.where(ch > 0, "+", "-"))), 2)
    out = np.zeros((natoms * 81 + 3) & ~3, np.uint8)
    out[:natoms * 81] = line.reshape(-1)
    return out


def _prepare(coords, topology, box, boxangles, device, chunk_bytes):
    """every check, then (coords, box, angles as CUDA tensors or None without frames, natoms, F, template)"""
    coords = _trajio.writer_coords(coords, "write_pdb")
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= MAX_ATOMS:
        raise ValueError(f"a PDB frame written here holds 1 to {MAX_ATOMS} atoms, got {natoms}")
    if F > MAX_MODELS:
        raise ValueError(f"a PDB file written here holds at most {MAX_MODELS} models, got {F}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    if box is None and boxangles is not None:
        raise ValueError("boxangles needs a box")
    cell = []
    for name, v in (("box", box), ("boxangles", boxangles)):
        if v is None:
            cell.append(None)
            continue
        if isinstance(v, torch.Tensor):
            if v.dtype != torch.float32:
                raise ValueError(f"{name} must be float32, got {v.dtype}")
        else:
            v = np.asarray(v, dtype=np.float32)
        if tuple(v.shape) != (3, F):
            raise ValueError(f"{name} must be (3, F) = {(3, F)}, got {tuple(v.shape)}")
        cell.append(v)
    box, angles = cell
    if box is not None and angles is None:
        angles = np.full((3, F), 90.0, np.float32)
    t = topology_fields(topology, natoms)
    _check_topology(t, natoms)
    bad = [(b, what) for b, what in ((_trajio.first_bad(coords, *COORD, 1000), "coords"),) if b is not None]
    if box is not None:
        bad += [(b, what) for b, what in ((_trajio.first_bad(box, *LENGTH, 1000), "box"),
                                          (_trajio.first_bad(angles, *ANGLE, 100), "boxangles")) if b is not None]
    if bad:
        (f, atom, axis, v), what = min(bad, key=lambda e: (e[0][0], e[1] == "coords"))
        field = dict(coords="'%8.3f' (-999.999 to 9999.999)", box="'%9.3f' (-9999.999 to 99999.999)",
                     boxangles="'%7.2f' (-999.99 to 9999.99)")[what]
        at = f"frame {f}, atom {atom}, axis {'xyz'[axis]}" if atom is not None else f"frame {f}, axis {'abc'[axis]}"
        raise ValueError(f"{what} at {at} is {v!r}: a PDB field {field} holds no such value, NaN or infinity")
    tmpl = _template(t, natoms)
    if F == 0:
        return None, None, None, natoms, F, tmpl
    x = _trajio.on_device(coords, device)
    if box is not None:
        box = box.to(x.device) if isinstance(box, torch.Tensor) else _trajio.on_device(box, x.device)
        angles = angles.to(x.device) if isinstance(angles, torch.Tensor) else _trajio.on_device(angles, x.device)
    return x, box, angles, natoms, F, tmpl


def frame_bytes(natoms: int, box: bool) -> int:
    """bytes of one written frame: MODEL, CRYST1 (with a box), the atom lines and ENDMDL"""
    return 15 + (71 if box else 0) + 81 * natoms + 7


def _cell_minor(v, F):
    if v is not None and F > 1 and (v.stride(1) != 1 or v.stride(0) < F):
        v = v.contiguous()
    return v


def _encode(x, box, angles, natoms: int, F: int, tmpl_d, model0: int = 0, out=None) -> torch.Tensor:
    dev = x.device
    x = _trajio.frame_minor(x)
    if box is not None:  # box and angles share one stride
        box, angles = _cell_minor(box, F), _cell_minor(angles, F)
        if box.stride(0) != angles.stride(0):
            box, angles = box.contiguous(), angles.contiguous()
    S = frame_bytes(natoms, box is not None)
    if out is None:
        out = torch.empty(F * S, dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_pdb_encode", _lib.ptr(x), max(int(x.stride(1)), F), F, natoms, _lib.ptr(tmpl_d),
              _lib.ptr(box), _lib.ptr(angles), max(int(box.stride(0)), F) if box is not None else 1, int(model0),
              _lib.ptr(out), int(out.numel()))
    return out[:F * S]


def encode_pdb_device(coords: torch.Tensor, topology, box=None, boxangles=None) -> torch.Tensor:
    """K28 on the device: ``coords`` (CUDA (natoms, 3, F) float32; a frame slice of a larger tensor is used in place)
    -> uint8 CUDA tensor of the F frames of :func:`write_pdb`'s file (without the final END line).  Values outside the
    writable range raise ValueError."""
    _lib.tensor_device(coords, "encode_pdb_device")
    x, b, ang, natoms, F, tmpl = _prepare(coords, topology, box, boxangles, None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    return _encode(x, b, ang, natoms, F, torch.from_numpy(tmpl).to(x.device))


def _emit(fh, x, box, angles, natoms: int, F: int, tmpl, chunk_bytes) -> None:
    if F:
        tmpl_d = torch.from_numpy(tmpl).to(x.device)
        _trajio.write_encoded(fh, x.device, F, frame_bytes(natoms, box is not None), chunk_bytes,
                              lambda f0, f1, out: _encode(x[:, :, f0:f1], None if box is None else box[:, f0:f1],
                                                          None if box is None else angles[:, f0:f1], natoms, f1 - f0,
                                                          tmpl_d, f0, out=out))
    fh.write(b"END\n")


def pdb_bytes(coords, topology, box=None, boxangles=None, device=None, chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_pdb` writes, as a ``bytes`` object."""
    x, b, ang, natoms, F, tmpl = _prepare(coords, topology, box, boxangles, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, x, b, ang, natoms, F, tmpl, chunk_bytes)
    return fh.getvalue()


def write_pdb(filename, coords, topology, box=None, boxangles=None, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a multi-model PDB file with the frames formatted on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``topology``: a Molecule / MolLite-like object or a dict with any of record, serial, name, altloc, resname, chain,
    resid, insertion, occupancy, beta, segid, element and charge (missing fields take the reader's blank defaults, and
    serials count from 1).  ``box`` (3, F) a, b, c and ``boxangles`` (3, F) alpha, beta, gamma (90 when omitted) add a
    CRYST1 record to every model.  The layout, column rules and serial wrap are in the module docstring.  Checked
    before the file is opened, each failure a ValueError naming the first frame, atom and field: coords finite with
    rint(x * 1000) in [-999 999, 9 999 999]; box and angles finite and within '%9.3f' / '%7.2f'; name, resname and
    segid at most 4 characters, chain, altloc and insertion 1, element 2, record ATOM or HETATM; resid within '%4d';
    occupancy and beta within '%6.2f'; charge an integer from -9 to 9.  The frames are encoded in chunks of at most
    ``chunk_bytes`` and each chunk is written while the next one encodes.  The file is created or truncated."""
    fn = _trajio.name(filename)
    x, b, ang, natoms, F, tmpl = _prepare(coords, topology, box, boxangles, device, chunk_bytes)
    with open(fn, "wb") as fh:
        _emit(fh, x, b, ang, natoms, F, tmpl, chunk_bytes)
