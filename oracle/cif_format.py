"""An independent restatement of multi-model PDBx/mmCIF in pure Python: a writer that formats every row with ``%`` and a
reader that splits lines with ``bytes.split()``, a small quote rule and ``float()`` per token.  Test infrastructure: the
tests hold moleculekit_b200/cif.py and K30 to it, so it shares no code with them.  ``rcsb`` writes the files the PDB
distributes: other categories before and after ``_atom_site``, ``#`` separators, quoted primed atom names, any column
order, and an ``_atom_site_anisotrop`` loop after the coordinates.

A written file: ``data_<title>``, ``#``, with a box the six ``_cell`` items and ``_symmetry.space_group_name_H-M 'P 1'``
and ``#``, then ``loop_``, the 21 ``_atom_site`` tags in RCSB's order, one row per atom and frame, and ``#``.  Columns
are joined by one space and padded to their widest value in the file: text with ``%-*s``, numbers with ``%*s``;
Cartn_x, Cartn_y, Cartn_z are ``%10.3f``, occupancy and B_iso_or_equiv ``%.2f``; ``id`` = f N + a + 1 and
``pdbx_PDB_model_num`` = f + 1.
"""
from __future__ import annotations

import re

import numpy as np

TAGS = ["group_PDB", "id", "type_symbol", "label_atom_id", "label_alt_id", "label_comp_id", "label_asym_id",
        "label_entity_id", "label_seq_id", "pdbx_PDB_ins_code", "Cartn_x", "Cartn_y", "Cartn_z", "occupancy",
        "B_iso_or_equiv", "pdbx_formal_charge", "auth_seq_id", "auth_comp_id", "auth_asym_id", "auth_atom_id",
        "pdbx_PDB_model_num"]
RESERVED = re.compile(r"(?i)(data_.*|save_.*|loop_|stop_|global_)\Z")
# a token at a token start: a quoted string closed by its quote and a blank or the end, or a run of non-blanks
TOKEN = re.compile(rb"""'(.*?)'(?=[ \t\v\f\r]|\Z)|"(.*?)"(?=[ \t\v\f\r]|\Z)|([^ \t\v\f\r]+)""", re.S)


def quote(s: str) -> str:
    """text as a CIF value"""
    if s == "":
        return "."
    if " " in s or s[0] in "_#$'\"[];" or s in (".", "?") or RESERVED.match(s):
        q = "'" if "'" not in s else '"'
        assert q not in s
        return q + s + q
    return s


def write(frames, topology: dict, box=None, angles=None, title: str = "trajectory") -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays; ``topology``: a dict of per-atom sequences (record, name, altloc,
    resname, chain, resid, insertion, occupancy, beta, segid, element, charge); ``box`` / ``angles``: the one cell
    (a, b, c) / (alpha, beta, gamma), or None -> the file's bytes"""
    t = topology
    n, F = len(t["name"]), len(frames)
    text = {k: [quote(v) for v in t[k]] for k in ("record", "name", "altloc", "resname", "chain", "insertion", "segid",
                                                  "element")}
    static = [("L", text["record"]), None, ("L", text["element"]), ("L", text["name"]), ("L", text["altloc"]),
              ("L", text["resname"]), ("L", text["segid"]), ("L", ["."] * n), ("R", ["%d" % r for r in t["resid"]]),
              ("L", text["insertion"]), None, None, None, ("R", ["%.2f" % float(v) for v in t["occupancy"]]),
              ("R", ["%.2f" % float(v) for v in t["beta"]]), ("R", ["%d" % int(c) for c in t["charge"]]),
              ("R", ["%d" % r for r in t["resid"]]), ("L", text["resname"]), ("L", text["chain"]),
              ("L", text["name"]), None]
    width = [max(len(v) for v in c[1]) if c else 0 for c in static]
    wid, wmod = len("%d" % (F * n)), len("%d" % F)
    out = ["data_%s\n#\n" % title]
    if box is not None:
        a, b, c = (float(v) for v in box)
        al, be, ga = (float(v) for v in (angles if angles is not None else (90.0, 90.0, 90.0)))
        out.append("_cell.length_a %.3f\n_cell.length_b %.3f\n_cell.length_c %.3f\n" % (a, b, c))
        out.append("_cell.angle_alpha %.2f\n_cell.angle_beta %.2f\n_cell.angle_gamma %.2f\n" % (al, be, ga))
        out.append("_symmetry.space_group_name_H-M 'P 1'\n#\n")
    out.append("loop_\n" + "".join("_atom_site.%s\n" % tg for tg in TAGS))
    for f, xyz in enumerate(frames):
        xyz = np.asarray(xyz, np.float32).reshape(n, 3)
        for i in range(n):
            cells = []
            for c, col in enumerate(static):
                if c == 1:
                    cells.append("%*d" % (wid, f * n + i + 1))
                elif c in (10, 11, 12):
                    cells.append("%10.3f" % float(xyz[i, c - 10]))
                elif c == 20:
                    cells.append("%*d" % (wmod, f + 1))
                elif col[0] == "L":
                    cells.append("%-*s" % (width[c], col[1][i]))
                else:
                    cells.append("%*s" % (width[c], col[1][i]))
            out.append(" ".join(cells) + "\n")
    out.append("#\n")
    return "".join(out).encode("ascii")


def tokens(line: bytes) -> list:
    """a row's tokens as (value, quoted); ValueError for a quote that does not close or a text field"""
    if line.lstrip()[:1] == b";":
        raise ValueError("a text field")
    if b"'" not in line and b'"' not in line:
        return [(t, False) for t in line.split()]
    out, pos = [], 0
    while True:
        rest = line[pos:]
        stripped = rest.lstrip(b" \t\v\f\r")
        if not stripped:
            return out
        pos += len(rest) - len(stripped)
        m = TOKEN.match(line, pos)
        if line[pos:pos + 1] in (b"'", b'"') and m.group(3) is not None:
            raise ValueError("a quote that does not close")
        if m.group(3) is not None:
            out.append((m.group(3), False))
        else:
            out.append((m.group(1) if m.group(1) is not None else m.group(2), True))
        pos = m.end()


def _number(tok: bytes, quoted: bool):
    if not quoted and tok in (b"?", b"."):
        return None
    if not quoted and tok.endswith(b")") and b"(" in tok:
        tok = tok[:tok.rindex(b"(")]
    return float(tok)


def _is_end(line: bytes) -> bool:
    s = line.strip().lower()
    first = s.split()[0] if s else b""
    return first[:1] == b"_" or first in (b"loop_", b"stop_", b"global_") or first.startswith((b"data_", b"save_"))


def read(data: bytes) -> dict:
    """The file's bytes -> dict(natoms, coords (F, natoms, 3) float32, model (F,), box (3,), boxangles (3,),
    topology (frame 0's rows, a dict of lists with the pdb field names), tags).  The first data block's _atom_site
    loop; rows grouped into frames by pdbx_PDB_model_num; a last frame cut short by the end of the file is dropped."""
    lines = [ln[:-1] if ln.endswith(b"\r") else ln for ln in data.split(b"\n")]
    i, blocks, cell, tags, body = 0, 0, {}, None, None
    in_text = False
    while i < len(lines):
        ln = lines[i]
        if in_text or ln[:1] == b";":
            in_text = not in_text if ln[:1] == b";" else in_text
            i += 1
            continue
        low = ln.strip().lower()
        if low.startswith(b"data_"):
            blocks += 1
            if blocks > 1:
                break
        elif low.startswith(b"_cell."):
            key, val = tokens(ln)[:2]
            name = key[0][6:].decode().lower()
            if name.startswith(("length_", "angle_")):
                cell[name] = _number(*val)
        elif low == b"loop_" and tags is None and blocks == 1:
            j, head = i + 1, []
            while j < len(lines) and (lines[j].strip()[:1] in (b"_", b"#") or not lines[j].strip()):
                if lines[j].strip()[:1] == b"_":
                    head.append(lines[j].strip().decode().lower())
                j += 1
            if head and head[0].startswith("_atom_site."):
                tags = [h[len("_atom_site."):] for h in head]
                body = j
                while j < len(lines) and not _is_end(lines[j]):
                    j += 1
                rows = [ln for ln in lines[body:j] if ln.strip() and ln.strip()[:1] != b"#"]
                ended = j < len(lines)
                i = j
                continue
        i += 1
    if tags is None:
        raise ValueError("no _atom_site loop")
    col = {t: k for k, t in enumerate(tags)}
    frames, models, top = [], [], []
    for ln in rows:
        tk = tokens(ln)
        if len(tk) != len(tags):
            raise ValueError("a row of %d tokens" % len(tk))
        m = int(tk[col["pdbx_pdb_model_num"]][0]) if "pdbx_pdb_model_num" in col else 0
        if not models or models[-1] != m:
            models.append(m)
            frames.append([])
        xyz = [_number(*tk[col[c]]) for c in ("cartn_x", "cartn_y", "cartn_z")]
        if None in xyz:
            raise ValueError("a null coordinate")
        frames[-1].append(xyz)
        if len(frames) == 1:
            top.append(tk)
    natoms = len(frames[0]) if frames else 0
    if len(frames) > 1 and not ended and len(frames[-1]) < natoms:
        frames.pop()
        models.pop()
    for f, c in enumerate(frames):
        if len(c) != natoms:
            raise ValueError("frame %d (model %d): %d rows, frame 0 has %d" % (f, models[f], len(c), natoms))

    def field(kind, *names):
        for nm in names:
            if nm.lower() in col:
                k = col[nm.lower()]
                vals = []
                for tk in top:
                    v, q = tk[k]
                    blank = not q and v in (b"?", b".")
                    if kind == "text":
                        vals.append("" if blank else v.decode("latin-1"))
                    elif kind == "int":
                        vals.append(0 if blank else int(v))
                    else:
                        vals.append(0.0 if blank else _number(v, q))
                return vals
        return [{"text": "", "int": 0, "float": 0.0}[kind]] * natoms

    topology = dict(record=field("text", "group_PDB"), serial=field("int", "id"),
                    name=field("text", "auth_atom_id", "label_atom_id"), altloc=field("text", "label_alt_id"),
                    resname=field("text", "auth_comp_id", "label_comp_id"),
                    chain=field("text", "auth_asym_id", "label_asym_id"),
                    resid=field("int", "auth_seq_id", "label_seq_id"), insertion=field("text", "pdbx_PDB_ins_code"),
                    occupancy=field("float", "occupancy"), beta=field("float", "B_iso_or_equiv"),
                    segid=field("text", "label_asym_id"), element=field("text", "type_symbol"),
                    charge=[float(c) for c in field("int", "pdbx_formal_charge")])
    box = np.float32([cell.get(k) or 0.0 for k in ("length_a", "length_b", "length_c")])
    ang = np.float32([cell[k] if cell.get(k) is not None else 90.0 for k in ("angle_alpha", "angle_beta",
                                                                             "angle_gamma")])
    coords = np.array(frames, np.float64).astype(np.float32).reshape(len(frames), natoms, 3)
    return dict(natoms=natoms, coords=coords, model=np.array(models, np.int64), box=box, boxangles=ang,
                topology=topology, tags=tags)


def rcsb(frames, topology: dict, tags=None, box=None, model_base: int = 1, fmt: str = "%.3f", nl: str = "\n",
         title: str = "1ABC", comments: bool = True, anisotrop: bool = True) -> bytes:
    """A file in the shape the PDB distributes: entry, struct (with a ';' text field) and entity categories, the cell,
    '#' between categories, the _atom_site loop with the columns ``tags`` (any order and subset of TAGS that keeps the
    Cartn tags; label_* and auth_* both given), names with a prime written in double quotes, coordinates as ``fmt``,
    models numbered from ``model_base``, and an _atom_site_anisotrop loop after it."""
    t = topology
    tags = list(TAGS) if tags is None else list(tags)
    n = len(t["name"])

    def val(tag, f, i, xyz):
        name = t["name"][i]
        q = quote if "'" not in name else (lambda s: '"%s"' % s)
        v = {"group_PDB": lambda: quote(t["record"][i]), "id": lambda: "%d" % (f * n + i + 1),
             "type_symbol": lambda: quote(t["element"][i]), "label_atom_id": lambda: q(name),
             "label_alt_id": lambda: quote(t["altloc"][i]), "label_comp_id": lambda: quote(t["resname"][i]),
             "label_asym_id": lambda: quote(t["segid"][i]), "label_entity_id": lambda: "1",
             "label_seq_id": lambda: "%d" % t["resid"][i], "pdbx_PDB_ins_code": lambda: quote(t["insertion"][i]) if
             t["insertion"][i] else "?", "Cartn_x": lambda: fmt % xyz[i, 0], "Cartn_y": lambda: fmt % xyz[i, 1],
             "Cartn_z": lambda: fmt % xyz[i, 2], "occupancy": lambda: "%.2f" % t["occupancy"][i],
             "B_iso_or_equiv": lambda: "%.2f" % t["beta"][i], "pdbx_formal_charge": lambda: "%d" % t["charge"][i],
             "auth_seq_id": lambda: "%d" % t["resid"][i], "auth_comp_id": lambda: quote(t["resname"][i]),
             "auth_asym_id": lambda: quote(t["chain"][i]), "auth_atom_id": lambda: q(name),
             "pdbx_PDB_model_num": lambda: "%d" % (model_base + f)}[tag]
        return v()

    out = ["data_%s" % title, "#", "_entry.id   %s" % title, "#", "_struct.entry_id %s" % title, "_struct.title",
           ";Generated test entry", "loop_ inside a text field, and _atom_site.id too", ";", "#"]
    if box is not None:
        out += ["_cell.entry_id           %s" % title, "_cell.length_a           %.3f" % box[0],
                "_cell.length_b           %.3f" % box[1], "_cell.length_c           %.3f" % box[2],
                "_cell.angle_alpha        %.2f" % box[3], "_cell.angle_beta         %.2f" % box[4],
                "_cell.angle_gamma        %.2f" % box[5], "_cell.Z_PDB              1", "#"]
    out += ["loop_", "_entity.id", "_entity.type", "1 polymer", "2 water", "#", "loop_"]
    out += ["_atom_site.%s" % tg for tg in tags]
    for f, xyz in enumerate(frames):
        xyz = np.asarray(xyz, np.float64)
        for i in range(n):
            out.append(" ".join(val(tg, f, i, xyz) for tg in tags) + " ")
            if comments and f == 0 and i == 1:
                out += ["# a comment between rows", "", "   "]
    out.append("#")
    if anisotrop:
        out += ["loop_", "_atom_site_anisotrop.id", "_atom_site_anisotrop.type_symbol", "_atom_site_anisotrop.U[1][1]"]
        out += ["%d %s 0.1234" % (i + 1, quote(t["element"][i])) for i in range(min(n, 5))]
        out.append("#")
    out += ["loop_", "_pdbx_poly_seq_scheme.asym_id", "_pdbx_poly_seq_scheme.seq_id", "A 1", "A 2", "#"]
    return (nl.join(out) + nl).encode("ascii")


def random_topology(n: int, seed: int) -> dict:
    """A seeded topology of ``n`` atoms covering the quoting rules: primed names, names and residue names with a
    blank, one starting with '_' or '#', reserved words, '.' and '?' as text, blank fields, charges from -3 to 3 and
    resids past 9999"""
    rng = np.random.default_rng(seed)
    letters = "ABCDEFGHIJKLMNOPQRSTUVWXYZ"

    def word(lo, hi):
        return "".join(rng.choice(list(letters + "0123456789'"), size=int(rng.integers(lo, hi + 1))))

    odd = ["O5'", "C 1", "_X", "#1", "loop_", "data_x", ".", "?", "a\"b", "[x]", "$y", ";z", "Global_", "stop_"]
    name = [str(rng.choice(odd)) if rng.random() < 0.2 else word(1, 4) for _ in range(n)]
    return dict(record=[str(rng.choice(["ATOM", "HETATM"])) for _ in range(n)],
                serial=list(range(1, n + 1)),
                name=name,
                altloc=[str(rng.choice(["", "", "A", "B"])) for _ in range(n)],
                resname=[str(rng.choice(["ALA", "HOH", "POPC", "A B", "DA"])) for _ in range(n)],
                chain=[str(rng.choice(["", "A", "B", "AA"])) for _ in range(n)],
                resid=[int(v) for v in rng.integers(-999, 100000, n)],
                insertion=[str(rng.choice(["", "", "A"])) for _ in range(n)],
                occupancy=[float(np.float32(v)) for v in rng.choice([0.0, 1.0, 0.5, 12.34, -99.99, 999.99], n)],
                beta=[float(np.float32(v)) for v in rng.uniform(-99.99, 999.99, n)],
                segid=[str(rng.choice(["", "A", "SEG1", "B"])) for _ in range(n)],
                element=[str(rng.choice(["C", "N", "O", "H", "S", "FE", "CL", ""])) for _ in range(n)],
                charge=[float(v) for v in rng.integers(-3, 4, n)])
