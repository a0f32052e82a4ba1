"""Multi-model PDBx/mmCIF trajectories read and written on the GPU (K30).

The format the PDB distributes every entry in, and the only one that holds systems of more than 99 999 atoms faithfully:
NMR and integrative-model ensembles and MD snapshots of large systems are one ``_atom_site`` loop whose rows carry
``pdbx_PDB_model_num``.  The reference tokenizes every row and calls ``float()`` on three tokens per atom; here:

- ``index_cif`` finds the loop header on the host and streams the loop body through two pinned and two device buffers.
  ``mkb_cif_index`` classifies every line start on the device, tokenizes every row (its token count and its model
  number) and lists each row whose model number differs from the row before it.  The host derives the frames from that
  O(F) list and parses the topology from frame 0's rows; it never tokenizes the rows of later frames.
- ``read_cif_device`` stages the listed frames (any order, repeats allowed) whole, chunk by chunk, and
  ``mkb_cif_decode`` ranks the rows of every staged frame and parses their Cartn_x, Cartn_y and Cartn_z tokens into the
  frame-minor ``(N, 3, F)`` float32 layout.
- ``write_cif`` builds each atom's row once on the host, at a fixed width, and fills in ``id``, the coordinates and
  ``pdbx_PDB_model_num`` on the device (``mkb_cif_encode``).

Reader contract:

1. The loop.  The first ``data_`` block is read.  The coordinates come from the ``loop_`` whose tags start with
   ``_atom_site.`` (tags compare case-insensitively, as in CIF; ``_atom_site_anisotrop.`` is another category).
   ``Cartn_x``, ``Cartn_y`` and ``Cartn_z`` are required; without ``pdbx_PDB_model_num`` the file is one frame.  The
   host finds the header by reading the file in chunks up to the loop's first row.  No ``_atom_site`` loop, a missing
   ``Cartn_*`` tag or an empty file raises ValueError naming the file.
2. The body starts at the first line after the tags.  Blank lines and lines whose first non-blank byte is ``#`` (CIF
   comments) are skipped.  The body ends at the first line whose first token is a tag (``_...``), ``loop_``, ``stop_``,
   ``global_``, ``data_...`` or ``save_...`` (in any case), or at the end of the file.  Every other line is one row and
   holds exactly T tokens (T tags).  Blanks are space, tab, \\v, \\f and \\r (what ``bytes.split()`` splits on).  A token
   is a run of other bytes, or a ``'...'`` / ``"..."`` string that opens at the token's start and closes at the first
   matching quote followed by a blank or the line's end.  A row that spans lines, a ``;`` text field or a row of another
   token count raises ValueError naming the file, the 1-based line and the token count: rows must be one line each.
   CRLF is read; a CR not followed by LF inside the body is an error.
3. Frames.  A frame is a maximal run of consecutive rows with the same integer ``pdbx_PDB_model_num`` (an unquoted
   ``[+-]digits`` of at most 18 digits; anything else raises ValueError naming the line).  N is the row count of frame
   0; a later frame of another row count raises ValueError naming the frame, its model number and its first line.  A
   last frame cut short by the end of the file (the body runs to the end of the file) is dropped with a warning.
4. Coordinates.  Each is bit for bit ``np.float32(float(token))``.  The device decides unquoted tokens in K26's grammar;
   quoted tokens, ``?`` and ``.``, values with a standard uncertainty (``1.234(5)``: read as ``1.234``), a byte >= 0x80
   before the coordinates and undecided roundings are re-read on the host, and ``info["host_lines"]`` counts those rows.
   ``?`` or ``.`` for a coordinate, or a token ``float()`` rejects, raises ValueError naming the file, frame, line and
   column.
5. Topology, from frame 0's rows with ``pdb.FIELDS`` keys: record ``group_PDB``, serial ``id``, name ``auth_atom_id``
   (else ``label_atom_id``), altloc ``label_alt_id``, resname ``auth_comp_id`` (else ``label_comp_id``), chain
   ``auth_asym_id`` (else ``label_asym_id``), resid ``auth_seq_id`` (else ``label_seq_id``), insertion
   ``pdbx_PDB_ins_code``, occupancy ``occupancy``, beta ``B_iso_or_equiv``, segid ``label_asym_id``, element
   ``type_symbol`` and charge ``pdbx_formal_charge``.  An unquoted ``?`` or ``.`` and a missing tag read as "" for
   text, 0 for integers and 0.0 for floats.
6. Cell.  ``_cell.length_a/b/c`` and ``_cell.angle_alpha/beta/gamma``, key-value items anywhere in the block, give the
   one cell of the file, repeated over every frame.  Without them the box is zeros and the angles 90.

The writer's file is ``data_<title>``, ``#``, with a box the six ``_cell`` items and ``_symmetry.space_group_name_H-M
'P 1'``, ``#``, ``loop_`` and the 21 tags of :data:`TAGS` (RCSB's order), one row per atom and frame, and a last ``#``
line.  Every column is padded to its widest value over the file (text left-justified, numbers right-justified) and
separated by one space, so every frame has the same size; ``id`` = f N + a + 1 is unique across the file,
``pdbx_PDB_model_num`` = f + 1.  Not supported: rows that span lines and ``;`` text fields in the loop, data
blocks after the first, per-model topology differences, compressed files, and on write ``_atom_site_anisotrop``, bonds
and ``_chem_comp``.
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
from .pdb import FIELDS, topology_fields

_fields = topology_fields  # the name bench_cif.py and the tests build writer layouts with

logger = logging.getLogger(__name__)

CHUNK_BYTES = 256 << 20
LOOKAHEAD = 1 << 16  # bytes past a chunk the index pass may read: the longest row it reads whole at a chunk's end
HEAD_STEP = 1 << 20  # bytes per read of the header search
FLAG_CAP = 1 << 20  # host rows recorded per read; past it every row of the listed frames is re-read
INT64_MAX, INT64_MIN = 2**63 - 1, -2**63
MAX_ROW = 768  # the widest row the device writes, '\n' included
BLANKS = b" \t\v\f\r"
TAGS = ("group_PDB", "id", "type_symbol", "label_atom_id", "label_alt_id", "label_comp_id", "label_asym_id",
        "label_entity_id", "label_seq_id", "pdbx_PDB_ins_code", "Cartn_x", "Cartn_y", "Cartn_z", "occupancy",
        "B_iso_or_equiv", "pdbx_formal_charge", "auth_seq_id", "auth_comp_id", "auth_asym_id", "auth_atom_id",
        "pdbx_PDB_model_num")
CELL = ("length_a", "length_b", "length_c", "angle_alpha", "angle_beta", "angle_gamma")
COORD = (-99999999, 999999999)  # rint(x * 1000) that '%10.3f' writes in 10 characters
SKIP, ROW, TERM = 0, 1, 2
_SU = re.compile(rb"(.*[0-9.])\([0-9]+\)")  # a value with a standard uncertainty: 1.234(5)


def _where(fn, frame: int, line: int, col: int) -> str:
    return f"CIF file {fn}, frame {frame}, line {line}, column {col}"


def _tokens(line: bytes):
    """the tokens of a row (without its '\\n') -> (list of (value, quoted), complete); complete is False when a quoted
    token does not close before the line's end or the row starts a ';' text field"""
    if b"'" not in line and b'"' not in line and line.lstrip(BLANKS)[:1] != b";":
        return [(t, False) for t in line.split()], True
    out, i, n = [], 0, len(line)
    while True:
        while i < n and line[i] in BLANKS:
            i += 1
        if i == n:
            return out, True
        q = line[i]
        if q in b"'\"":
            j = i + 1
            while True:
                j = line.find(line[i:i + 1], j)
                if j < 0:
                    return out, False
                if j + 1 == n or line[j + 1] in BLANKS:
                    break
                j += 1
            out.append((line[i + 1:j], True))
            i = j + 1
        else:
            if q == ord(";") and not out:
                return out, False
            j = i
            while j < n and line[j] not in BLANKS:
                j += 1
            out.append((line[i:j], False))
            i = j


def _kind(line: bytes) -> int:
    s = line.lstrip(BLANKS)
    if not s or s[:1] == b"#":
        return SKIP
    if s[:1] == b"_":
        return TERM
    tok = s.split(None, 1)[0].lower()
    if tok in (b"loop_", b"stop_", b"global_") or tok[:5] in (b"data_", b"save_"):
        return TERM
    return ROW


def _lines(fd: int, pos: int, end: int):
    """(file offset, line without its '\\n') from ``pos`` to ``end``, read in HEAD_STEP pieces"""
    carry = b""
    while pos < end:
        b = os.pread(fd, min(HEAD_STEP, end - pos), pos)
        if not b:
            break
        pos += len(b)
        b = carry + b
        at = pos - len(b)
        lines = b.split(b"\n")
        carry = lines.pop()
        for ln in lines:
            yield at, ln
            at += len(ln) + 1
    if carry:
        yield pos - len(carry), carry


def _value(tok: bytes, quoted: bool):
    """a numeric token as float() reads it after its standard uncertainty is cut off; None for ? and ."""
    if not quoted:
        if tok in (b"?", b"."):
            return None
        m = _SU.fullmatch(tok)
        if m:
            tok = m.group(1)
    return float(tok)


def _scan(fn, fd: int, pos: int, E: int, find_loop: bool) -> dict:
    """the data block's lines from ``pos``: its cell items and, with ``find_loop``, the _atom_site loop header ->
    dict(cell {name: value}, tags [lower-case names after '_atom_site.'], body (file offset of the first line after the
    tags)); stops at the loop's first row, at the next data block or at the end of the file"""
    cell, tags, in_text, in_data, header = {}, None, False, not find_loop, None
    for at, ln in _lines(fd, pos, E):
        if in_text:  # a ';' text field runs to the next line starting with ';'
            in_text = ln[:1] != b";"
            continue
        if ln[:1] == b";":
            in_text = True
            continue
        s = ln.strip(BLANKS)
        low = s.lower()
        if header is not None:  # inside a loop header
            if low[:1] == b"_":
                header.append(low.split()[0])
                continue
            if not s or s[:1] == b"#":
                continue
            if find_loop and header and header[0].startswith(b"_atom_site."):
                tags = [t[len(b"_atom_site."):].decode("latin-1") for t in header]
                return dict(cell=cell, tags=tags, body=at)
            header = None
        if low.startswith(b"data_"):
            if in_data:
                break
            in_data = True
        elif not in_data:
            continue
        elif low.split(None, 1)[:1] == [b"loop_"]:
            header = []
        elif low.startswith(b"_cell."):
            parts, _ = _tokens(s)
            name = parts[0][0][6:].decode("latin-1").lower()
            if name in CELL and len(parts) > 1:
                try:
                    cell[name] = _value(*parts[1])
                except ValueError:
                    raise ValueError(f"CIF file {fn}, line {_trajio.line_col(fd, at)[0] + 1}: _cell.{name} "
                                     f"{parts[1][0]!r} is not a number") from None
        elif find_loop and low.startswith(b"_atom_site."):
            raise ValueError(f"CIF file {fn}, line {_trajio.line_col(fd, at)[0] + 1}: the _atom_site category is not a "
                             "loop; only a loop_ of atom rows is read")
    if find_loop and header and header[0].startswith(b"_atom_site."):  # a header that runs to the end of the file: no rows
        return dict(cell=cell, tags=[t[len(b"_atom_site."):].decode("latin-1") for t in header], body=E)
    return dict(cell=cell, tags=None, body=E)


def _marks(fd: int, body: int, E: int, dev, B: int, T: int, model_col: int):
    """the index pass over the body [body, E) -> (marks (M, 3) int64 in file order: file offset, rows before it, model
    number; the final state, see mkb_cif_index)"""
    span = E - body
    cap = 4096 + span // 4096
    while True:
        state = torch.tensor([0, INT64_MAX, 0, INT64_MAX, INT64_MAX, INT64_MIN, -1], dtype=torch.int64, device=dev)
        marks = torch.empty(3 * cap, dtype=torch.int64, device=dev)

        def stage(c, host):
            n_read = min(B + LOOKAHEAD, span - c * B)
            _trajio.read_exact(fd, host[:n_read], body + c * B, "CIF")
            return n_read

        def consume(c, buf):
            _lib.call(dev, "mkb_cif_index", _lib.ptr(buf), min(B, span - c * B), int(buf.numel()), body + c * B,
                      int(c == 0), T, model_col, _lib.ptr(state), _lib.ptr(marks), cap)

        _trajio.upload(dev, -(-span // B), min(B, span) + LOOKAHEAD, stage, consume)
        st = [int(v) for v in state.cpu()]
        n = st[2]
        if n <= cap:
            m = marks[:3 * n].view(n, 3).cpu().numpy()
            return m[np.argsort(m[:, 0], kind="stable")], st
        cap = n  # more marks than the first guess: index again with room for all of them


def _bad_row(fn, fd, pos: int, E: int, T: int, model_col: int) -> ValueError:
    """the error of the row the index pass flagged at file offset ``pos``"""
    line = _trajio.line_at(fd, pos, E)
    toks, complete = _tokens(line)
    no = _trajio.line_col(fd, pos)[0] + 1
    if complete and len(toks) == T:
        if model_col >= 0 and not (not toks[model_col][1] and re.fullmatch(rb"[+-]?[0-9]{1,18}", toks[model_col][0])):
            return ValueError(f"CIF file {fn}, line {no}: the pdbx_PDB_model_num token {toks[model_col][0]!r} is not "
                              "an integer of at most 18 digits")
        return ValueError(f"CIF file {fn}, line {no}: a row of {len(line)} bytes; rows longer than {LOOKAHEAD} bytes "
                          "are not read")
    text = " and starts a ';' text field" if line.lstrip(BLANKS)[:1] == b";" else \
        " and a quoted token that does not close" if not complete else ""
    return ValueError(f"CIF file {fn}, line {no}: the _atom_site row holds {len(toks)} tokens{text}, the loop has {T} "
                      "tags; rows must be one line each (rows that span lines and ';' text fields are not read)")


def index_cif(filename, device=None, chunk_bytes: int = CHUNK_BYTES) -> dict:
    """Find the frames of a PDBx/mmCIF file on the device -> dict(natoms, n_frames, start, end ((F,) int64: the file
    bytes [start, end) of each frame, from its first row to the next frame's first row, or for the last frame to the
    line that ends the loop or the end of the file), model ((F,) int64: each frame's pdbx_PDB_model_num, 0 without the
    tag), topology (frame 0's rows, with ``pdb.FIELDS`` keys), box and boxangles ((3,) float32: the file's one cell),
    tags (the loop's tags after '_atom_site.', lower case)).  The loop body goes through the device in chunks of
    ``chunk_bytes`` with one host sync at the end.  Errors: see the module docstring."""
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    B = (int(chunk_bytes) + 15) & ~15
    with open(fn, "rb") as fh:
        fd = fh.fileno()
        E = os.fstat(fd).st_size
        if E == 0:
            raise ValueError(f"CIF file {fn}: the file is empty")
        head = _scan(fn, fd, 0, E, True)
        tags = head["tags"]
        if tags is None:
            raise ValueError(f"CIF file {fn}: no _atom_site loop in the first data block")
        for c in ("cartn_x", "cartn_y", "cartn_z"):
            if c not in tags:
                raise ValueError(f"CIF file {fn}: the _atom_site loop has no _atom_site.{c[:1].upper()}{c[1:]} tag")
        T = len(tags)
        if T > 1 << 20:
            raise ValueError(f"CIF file {fn}: the _atom_site loop has {T} tags, at most {1 << 20} are read")
        model_col = tags.index("pdbx_pdb_model_num") if "pdbx_pdb_model_num" in tags else -1
        m, st = _marks(fd, head["body"], E, _lib.device(device), B, T, model_col)
        n_rows, lone_cr, _, bad, term, _, term_rank = st
        stop = term if term != INT64_MAX else E
        if term != INT64_MAX:
            n_rows = term_rank
        errors = []
        if lone_cr < stop:
            line, col = _trajio.line_col(fd, lone_cr)
            errors.append((lone_cr, ValueError(f"CIF file {fn}, line {line + 1}, column {col}: a CR that is not "
                                               "followed by LF ends a line; lone CR line endings are not supported")))
        if bad < stop:
            errors.append((bad, _bad_row(fn, fd, bad, E, T, model_col)))
        if errors:
            raise min(errors, key=lambda t: t[0])[1]
        if len(m) == 0:
            raise ValueError(f"CIF file {fn}: the _atom_site loop holds no rows")
        start, model = m[:, 0].copy(), m[:, 2].copy()
        count = np.diff(np.append(m[:, 1], n_rows)).astype(np.int64)
        N, F = int(count[0]), len(count)
        if F > 1 and term == INT64_MAX and count[-1] < N:
            F -= 1
            logger.warning("CIF file %s: the last model (frame %d, model %d) has %d of its %d rows; it is dropped", fn,
                           F, int(model[-1]), int(count[-1]), N)
        diff = np.flatnonzero(count[:F] != N)
        if len(diff):
            f = int(diff[0])
            raise ValueError(f"CIF file {fn}, frame {f} (model {int(model[f])}, line "
                             f"{_trajio.line_col(fd, int(start[f]))[0] + 1}): {int(count[f])} rows, frame 0 has {N} "
                             "(every model must hold the same atoms)")
        end = np.append(start[1:], stop).astype(np.int64)
        raw0 = os.pread(fd, int(end[0] - start[0]), int(start[0]))
        topology = _topology(fn, fd, tags, raw0, int(start[0]))
        cell = dict(head["cell"])
        if term < E:  # the block's items after the loop
            cell.update({k: v for k, v in _scan(fn, fd, term, E, False)["cell"].items() if k not in cell})
    box = np.float32([cell.get(k) or 0.0 for k in CELL[:3]])
    angles = np.float32([cell[k] if cell.get(k) is not None else 90.0 for k in CELL[3:]])
    return dict(natoms=N, n_frames=int(F), start=start[:F].astype(np.int64), end=end[:F], model=model[:F],
                topology=topology, box=box, boxangles=angles, tags=tags)


def _rows(raw: bytes, base: int) -> list:
    """the rows of a frame's bytes ``raw`` (at file offset ``base``) -> [(file offset, line)]"""
    rows, pos = [], base
    for ln in raw.split(b"\n"):
        if _kind(ln) == ROW:
            rows.append((pos, ln))
        pos += len(ln) + 1
    return rows


def _topology(fn, fd, tags, raw: bytes, base: int) -> dict:
    """frame 0's rows (the bytes ``raw`` at file offset ``base``) -> dict of per-atom arrays with pdb.FIELDS keys"""
    rows = _rows(raw, base)
    toks = [_tokens(ln)[0] for _, ln in rows]
    col = {t: i for i, t in enumerate(tags)}

    def pick(*names):
        for n in names:
            if n.lower() in col:
                return col[n.lower()]
        return None

    def text(*names):
        i = pick(*names)
        if i is None:
            return np.full(len(rows), "", dtype=object)
        return np.array(["" if not q and v in (b"?", b".") else v.decode("latin-1") for v, q in (t[i] for t in toks)],
                        dtype=object)

    def number(kind, dtype, *names):
        i = pick(*names)
        out = np.zeros(len(rows), dtype)
        if i is None:
            return out
        for r, t in enumerate(toks):
            v, q = t[i]
            try:
                x = _value(v, q)
                out[r] = 0 if x is None else (int(v) if kind is int else x)
            except ValueError:
                raise ValueError(f"{_where(fn, 0, _trajio.line_col(fd, rows[r][0])[0] + 1, i + 1)}: the {tags[i]} "
                                 f"token {v!r} is not {'an integer' if kind is int else 'a number'}") from None
        return out

    return dict(record=text("group_PDB"), serial=number(int, np.int64, "id"),
                name=text("auth_atom_id", "label_atom_id"), altloc=text("label_alt_id"),
                resname=text("auth_comp_id", "label_comp_id"), chain=text("auth_asym_id", "label_asym_id"),
                resid=number(int, np.int64, "auth_seq_id", "label_seq_id"), insertion=text("pdbx_PDB_ins_code"),
                occupancy=number(float, np.float32, "occupancy"), beta=number(float, np.float32, "B_iso_or_equiv"),
                segid=text("label_asym_id"), element=text("type_symbol"),
                charge=number(int, np.float32, "pdbx_formal_charge"))


def _cartn(tags) -> tuple:
    return tuple(tags.index(c) for c in ("cartn_x", "cartn_y", "cartn_z"))


def decode_cif_device(buf: torch.Tensor, n_staged: int, frame_of, natoms: int, cols, out: torch.Tensor | None = None,
                      flags: torch.Tensor | None = None, frame_base: int = 0, flag_cap: int = FLAG_CAP):
    """K30 on the device: ``buf`` (uint8 CUDA tensor, 16-byte aligned: ``n_staged`` whole frames back to back, each
    starting a line and holding exactly ``natoms`` rows), ``frame_of`` (int per listed frame: its staged frame),
    ``cols`` (the 0-based token columns of Cartn_x, Cartn_y, Cartn_z) -> (coords (natoms, 3, F) float32, flags int64
    (1 + flag_cap,)).  flags[0] counts the rows left to the host; flags[1 + j] holds (frame_base + k) * natoms + a for
    the first flag_cap of them.  ``out`` may be a frame slice of a larger (natoms, 3, F) tensor.  Nothing is
    synchronised."""
    dev = _lib.tensor_device(buf, "decode_cif_device")
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
    cx, cy, cz = (int(c) for c in cols)
    _lib.call(dev, "mkb_cif_decode", _lib.ptr(buf), int(buf.numel()), int(n_staged),
              frame_of.ctypes.data_as(C.c_void_p), F, int(natoms), cx, cy, cz, _lib.ptr(out), stride,
              int(frame_base), _lib.ptr(flags), int(flag_cap))
    return out, flags


def _row_coords(fn, line: bytes, cols, tags, frame: int, line_no) -> np.ndarray:
    """the Cartn tokens of a row as the reference reads them; ``line_no()`` gives its 1-based line for errors"""
    toks, complete = _tokens(line)
    if not complete or len(toks) != len(tags):
        raise ValueError(f"CIF file {fn}, frame {frame}, line {line_no()}: the _atom_site row holds {len(toks)} tokens, "
                         f"the loop has {len(tags)} tags")
    out = np.empty(3, np.float32)
    for d, i in enumerate(cols):
        v, q = toks[i]
        try:
            x = _value(v, q)
        except ValueError:
            raise ValueError(f"{_where(fn, frame, line_no(), i + 1)}: the Cartn_{'xyz'[d]} token {v!r} is not a "
                             "number") from None
        if x is None:
            raise ValueError(f"{_where(fn, frame, line_no(), i + 1)}: the Cartn_{'xyz'[d]} token {v!r} is a null "
                             "value; every atom needs coordinates")
        out[d] = np.float32(x)
    return out


def _host_rows(fn, fd, start, end, sel, N, k, a, cols, tags, coords) -> None:
    """re-read rows (listed frame k, atom a) on the host and write their coordinates; the first bad row in file order
    raises"""
    order = np.lexsort((a, sel[k]))
    vals = np.empty((len(k), 3), np.float32)
    cached = (-1, None)
    for j in order.tolist():
        f, at = int(sel[k[j]]), int(a[j])
        if cached[0] != f:
            cached = (f, _rows(os.pread(fd, int(end[f] - start[f]), int(start[f])), int(start[f])))
        pos, ln = cached[1][at]
        vals[j] = _row_coords(fn, ln, cols, tags, f, lambda: _trajio.line_col(fd, pos)[0] + 1)
    dev = coords.device
    coords[torch.from_numpy(a).to(dev), :, torch.from_numpy(k).to(dev)] = torch.from_numpy(vals).to(dev)


def _read(filename, frames, index, device, chunk_bytes):
    fn = _trajio.name(filename)
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    idx = index if index is not None else index_cif(fn, device, chunk_bytes)
    N, F = int(idx["natoms"]), int(idx["n_frames"])
    start, end = np.asarray(idx["start"], np.int64), np.asarray(idx["end"], np.int64)
    cols = _cartn(idx["tags"])
    sel = _trajio.select(F, frames)
    dev = _lib.device(device)
    n = len(sel)
    coords = torch.empty((N, 3, n), dtype=torch.float32, device=dev)
    info = dict(natoms=N, n_frames=F, frames=sel, topology=idx["topology"], host_lines=0,
                box=np.repeat(np.asarray(idx["box"], np.float32).reshape(3, 1), n, axis=1),
                boxangles=np.repeat(np.asarray(idx["boxangles"], np.float32).reshape(3, 1), n, axis=1),
                model=np.asarray(idx["model"], np.int64)[sel])
    if n == 0:
        return coords, info
    flags = torch.zeros(1 + FLAG_CAP, dtype=torch.int64, device=dev)
    with open(fn, "rb") as fh:
        fd = fh.fileno()

        def decode(buf, at, frame_of, k0, k1):
            decode_cif_device(buf, len(at) - 1, frame_of, N, cols, out=coords[:, :, k0:k1], flags=flags, frame_base=k0)

        _trajio.read_frames(fd, dev, sel, start, end - start, chunk_bytes, "CIF", decode)
        k, a, _ = _trajio.flagged(flags, n, N, FLAG_CAP, 1)
        if len(k):
            _host_rows(fn, fd, start, end, sel, N, k, a, cols, idx["tags"], coords)
            info["host_lines"] = len(k)
    return coords, info


def read_cif_device(filename, frames=None, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame (or the frames listed in ``frames``: any order, repeats allowed; out of range raises IndexError) ->
    (coords CUDA (natoms, 3, F) float32 [Angstrom], info) with the trajectory left on the GPU.  ``index`` (what
    :func:`index_cif` returned for this file) skips the index pass.  ``info`` holds natoms, n_frames (frames in the
    file), frames (the file frame of each returned frame), box and boxangles ((3, F) float32 numpy, the file's cell in
    every frame), topology (frame 0's rows), host_lines (the rows re-read on the host) and model (each returned frame's
    pdbx_PDB_model_num).  Errors: see the module docstring."""
    return _read(filename, frames, index, device, chunk_bytes)


def read_cif(filename, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """Every frame -> (coords (natoms, 3, F) float32 numpy [Angstrom], info as :func:`read_cif_device`)."""
    coords, info = _read(filename, None, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


def read_cif_frames(filename, frames, index: dict | None = None, device=None, chunk_bytes: int = CHUNK_BYTES):
    """:func:`read_cif` for the listed frames (any order, repeats allowed; out of range raises IndexError)."""
    coords, info = _read(filename, frames, index, device, chunk_bytes)
    return coords.cpu().numpy(), info


# ------------------------------------------------------------------------------------------------------------ writing
def cif_token(s: str) -> str | None:
    """text as one CIF token: "." for "", quoted with the quote character it does not contain when it holds a blank,
    starts with _ # $ ' " [ ] ;, is . or ? or a reserved word; None when it cannot be written (not printable ASCII, or
    both quote characters where quoting is needed)"""
    if s == "":
        return "."
    if not all(" " <= c <= "~" for c in s):
        return None
    low = s.lower()
    if not (" " in s or s[0] in "_#$'\"[];" or s in (".", "?") or low in ("loop_", "stop_", "global_")
            or low.startswith(("data_", "save_"))):
        return s
    if "'" not in s:
        return f"'{s}'"
    if '"' not in s:
        return f'"{s}"'
    return None


def _check(t: dict) -> dict:
    """the topology's text as tokens (ValueError naming the first atom and field that cannot be written)"""
    bad, toks = [], {}
    for k in ("record", "name", "altloc", "resname", "chain", "insertion", "segid", "element"):
        vals = t[k].tolist()
        uniq = {}
        for a, s in enumerate(vals):
            if s not in uniq:
                uniq[s] = cif_token(s) if isinstance(s, str) else None
            if uniq[s] is None:
                bad.append((a, k, f"{s!r}: printable ASCII, and not both quote characters where it must be quoted"))
                break
        toks[k] = np.array([uniq.get(s, "") for s in vals], dtype=object)

    def first(k, ok, reason):
        with np.errstate(invalid="ignore", over="ignore"):
            hit = np.flatnonzero(~ok)
        if len(hit):
            bad.append((int(hit[0]), k, f"{t[k].tolist()[hit[0]]!r}: {reason}"))

    for k in ("resid", "charge"):
        v = t[k].astype(np.float64)
        first(k, np.isfinite(v) & (v == np.round(v)) & (np.abs(v) < 2**53), "an integer")
    for k in ("occupancy", "beta"):
        first(k, np.isfinite(t[k].astype(np.float64)), "a finite number")
    if bad:
        a, k, why = min(bad)
        raise ValueError(f"topology at atom {a}, field {k} is {why}")
    return toks


def _layout(t: dict, natoms: int, F: int) -> tuple:
    """the fixed-width rows -> (template uint8 (natoms * R rounded up to 4,), R, col_id, id width, col_x, col_model,
    model width): every column padded to its widest value, text left-justified, numbers right-justified, id, Cartn and
    pdbx_PDB_model_num left blank"""
    toks = _check(t)

    def ints(v):
        return np.char.mod("%d", np.asarray(v, np.float64).astype(np.int64))

    resid, blank = ints(t["resid"]), np.full(natoms, "", dtype=object)
    cols = [(toks["record"], False), (blank, True), (toks["element"], False), (toks["name"], False),
            (toks["altloc"], False), (toks["resname"], False), (toks["segid"], False),
            (np.full(natoms, ".", dtype=object), False), (resid, True), (toks["insertion"], False),
            (blank, True), (blank, True), (blank, True),
            (np.char.mod("%.2f", t["occupancy"].astype(np.float64)), True),
            (np.char.mod("%.2f", t["beta"].astype(np.float64)), True), (ints(t["charge"]), True), (resid, True),
            (toks["resname"], False), (toks["chain"], False), (toks["name"], False), (blank, True)]
    id_w, model_w = len(str(F * natoms)), len(str(F))
    fixed = {1: id_w, 10: 10, 11: 10, 12: 10, 20: model_w}
    parts, at, offs = [], 0, []
    for i, (v, right) in enumerate(cols):
        v = np.asarray(v, dtype=str)
        w = fixed.get(i, int(np.char.str_len(v).max()))
        parts.append(np.char.rjust(v, w) if right else np.char.ljust(v, w))
        offs.append(at)
        at += w + 1
    R = at  # the last column's separator is the '\n'
    if R > MAX_ROW:
        raise ValueError(f"an _atom_site row of this topology takes {R} bytes; at most {MAX_ROW} are written")
    rows = parts[0]
    for p in parts[1:]:
        rows = np.char.add(np.char.add(rows, " "), p)
    b = np.char.encode(np.char.add(rows, "\n"), "ascii")
    assert b.dtype.itemsize == R
    out = np.zeros((natoms * R + 3) & ~3, np.uint8)
    out[:natoms * R] = np.frombuffer(b.tobytes(), np.uint8)
    return out, R, offs[1], id_w, offs[10], offs[20], model_w


def _header(title: str, box, angles) -> bytes:
    out = [f"data_{title}", "#"]
    if box is not None:
        for k, v in zip(CELL, [*box, *angles]):
            out.append(f"_cell.{k} " + ("%.3f" if k.startswith("length") else "%.2f") % float(v))
        out.append("_symmetry.space_group_name_H-M 'P 1'")
        out.append("#")
    out.append("loop_")
    out += [f"_atom_site.{t}" for t in TAGS]
    return ("\n".join(out) + "\n").encode("ascii")


def _prepare(coords, topology, box, boxangles, title, device, chunk_bytes):
    """every check, then (coords as a CUDA tensor or None without frames, natoms, F, header, layout)"""
    coords = _trajio.writer_coords(coords, "write_cif")
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if not 1 <= natoms <= (2**31 - 1) // 3:
        raise ValueError(f"a CIF frame written here holds 1 to {(2**31 - 1) // 3} atoms, got {natoms}")
    if chunk_bytes <= 0:
        raise ValueError(f"chunk_bytes must be positive, got {chunk_bytes}")
    title = "trajectory" if title is None else title
    if not isinstance(title, str) or not title or not all("!" <= c <= "~" for c in title):
        raise ValueError(f"title must be printable ASCII without blanks (it names the data block), got {title!r}")
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
    layout = _layout(t, natoms, F)
    bad = _trajio.first_bad(coords, *COORD, 1000)
    if bad is not None:
        f, atom, axis, v = bad
        raise ValueError(f"coords at frame {f}, atom {atom}, axis {'xyz'[axis]} is {v!r}: a '%10.3f' Cartn field "
                         "(-99999.999 to 999999.999) holds no such value, NaN or infinity")
    if box is not None and F:
        for name, v in (("box", box), ("boxangles", angles)):
            if not np.isfinite(v).all():
                f, axis = np.unravel_index(np.argmax(~np.isfinite(v.T)), (F, 3))
                raise ValueError(f"{name} at frame {f}, axis {'abc'[axis]} is {v[axis, f]!r}: not finite")
        same = (box == box[:, :1]).all(axis=0) & (angles == angles[:, :1]).all(axis=0)
        if not same.all():
            f = int(np.argmin(same))
            raise ValueError(f"the box of frame {f} differs from frame 0's: an mmCIF data block holds one cell")
    head = _header(title, None if box is None or not F else box[:, 0], None if box is None or not F else angles[:, 0])
    if F == 0:
        return None, natoms, F, head, layout
    return _trajio.on_device(coords, device), natoms, F, head, layout


def frame_bytes(natoms: int, row_bytes: int) -> int:
    """bytes of one written frame: natoms rows of ``row_bytes``"""
    return natoms * row_bytes


def _encode(x, natoms: int, F: int, tmpl_d, layout, frame0: int = 0, out=None) -> torch.Tensor:
    dev = x.device
    x = _trajio.frame_minor(x)
    _, R, col_id, id_w, col_x, col_model, model_w = layout
    S = frame_bytes(natoms, R)
    if out is None:
        out = torch.empty(F * S, dtype=torch.uint8, device=dev)
    _lib.call(dev, "mkb_cif_encode", _lib.ptr(x), max(int(x.stride(1)), F), F, natoms, _lib.ptr(tmpl_d), R, col_id,
              id_w, col_x, col_model, model_w, int(frame0), _lib.ptr(out), int(out.numel()))
    return out[:F * S]


def encode_cif_device(coords: torch.Tensor, topology) -> torch.Tensor:
    """K30 on the device: ``coords`` (CUDA (natoms, 3, F) float32; a frame slice of a larger tensor is used in place)
    -> uint8 CUDA tensor of the F frames' rows of :func:`write_cif`'s file (without its header and last '#' line).
    Values outside the writable range raise ValueError."""
    _lib.tensor_device(coords, "encode_cif_device")
    x, natoms, F, _, layout = _prepare(coords, topology, None, None, None, None, 1)
    if F == 0:
        return torch.empty(0, dtype=torch.uint8, device=coords.device)
    return _encode(x, natoms, F, torch.from_numpy(layout[0]).to(x.device), layout)


def _emit(fh, x, natoms: int, F: int, head: bytes, layout, chunk_bytes) -> None:
    fh.write(head)
    if F:
        tmpl_d = torch.from_numpy(layout[0]).to(x.device)
        _trajio.write_encoded(fh, x.device, F, frame_bytes(natoms, layout[1]), chunk_bytes,
                              lambda f0, f1, out: _encode(x[:, :, f0:f1], natoms, f1 - f0, tmpl_d, layout, f0, out=out))
    fh.write(b"#\n")


def cif_bytes(coords, topology, box=None, boxangles=None, title=None, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> bytes:
    """The file :func:`write_cif` writes, as a ``bytes`` object."""
    x, natoms, F, head, layout = _prepare(coords, topology, box, boxangles, title, device, chunk_bytes)
    fh = io.BytesIO()
    _emit(fh, x, natoms, F, head, layout, chunk_bytes)
    return fh.getvalue()


def write_cif(filename, coords, topology, box=None, boxangles=None, title=None, device=None,
              chunk_bytes: int = CHUNK_BYTES) -> None:
    """Write a multi-model PDBx/mmCIF file with the frames formatted on the GPU.  ``coords`` (natoms, 3, F) float32 in
    Angstrom: a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is; a frame slice is fine).
    ``topology``: a Molecule / MolLite-like object or a dict with any of pdb.FIELDS (missing fields take the reader's
    blank defaults; serial is not written: id counts the rows of the file from 1).  ``box`` (3, F) a, b, c and
    ``boxangles`` (3, F) alpha, beta, gamma (90 when omitted) write the ``_cell`` items; they must be the same in every
    frame.  ``title`` names the data block ("trajectory" by default).  The layout is in the module docstring.  Checked
    before the file is opened, each failure a ValueError naming the first frame, atom and field: coords finite with
    rint(x * 1000) in [-99 999 999, 999 999 999] ('%10.3f'); box and angles finite and equal in every frame; text
    printable ASCII that can be quoted; resid and charge integers; occupancy and beta finite; a row of at most 768
    bytes.  The frames are encoded in chunks of at most ``chunk_bytes`` and each chunk is written while the next one
    encodes.  The file is created or truncated."""
    fn = _trajio.name(filename)
    x, natoms, F, head, layout = _prepare(coords, topology, box, boxangles, title, device, chunk_bytes)
    with open(fn, "wb") as fh:
        _emit(fh, x, natoms, F, head, layout, chunk_bytes)


__all__ = ["index_cif", "read_cif", "read_cif_frames", "read_cif_device", "decode_cif_device", "write_cif", "cif_bytes",
           "encode_cif_device", "FIELDS", "TAGS"]
