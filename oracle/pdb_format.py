"""An independent restatement of the multi-model PDB format in pure Python: a writer that formats every line with ``%``
and a reader that walks the lines and slices columns, with ``float()`` per coordinate.  Test infrastructure: the tests
hold moleculekit_b200/pdb.py and K28 to it, so it shares no code with them.

A written file, per frame:

    MODEL %8d                  the 1-based model serial
    CRYST1 ...                 a, b, c as %9.3f, alpha, beta, gamma as %7.2f, " P 1           1" (with a box only)
    natoms ATOM / HETATM lines the PDB 3.3 columns, x y z as %8.3f in columns 31-54
    ENDMDL

and "END" after the last frame.
"""
from __future__ import annotations

import numpy as np

ATOM_LINE = "%-6s%5d %4s%1s%4s%1s%4d%1s   %8.3f%8.3f%8.3f%6.2f%6.2f      %-4s%2s%2s\n"


def _name_field(name: str, element: str) -> str:
    if len(name) == 4:
        return name
    if len(element) == 1:
        return " %-3s" % name
    return "%-4s" % name


def _resname_field(resname: str) -> str:
    return resname if len(resname) == 4 else "%3s " % resname


def _charge_field(charge) -> str:
    c = int(charge)
    if c == 0:
        return ""
    return "%d%s" % (abs(c), "+" if c > 0 else "-")


def write(frames, topology: dict, boxes=None, angles=None) -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays; ``topology``: a dict of per-atom sequences (record, serial, name,
    altloc, resname, chain, resid, insertion, occupancy, beta, segid, element, charge); ``boxes`` / ``angles``: one
    (a, b, c) / (alpha, beta, gamma) per frame, or None -> the file's bytes."""
    t = topology
    n = len(t["name"])
    out = []
    for f, xyz in enumerate(frames):
        xyz = np.asarray(xyz, np.float32).reshape(n, 3)
        out.append("MODEL %8d\n" % (f + 1))
        if boxes is not None:
            a, b, c = (float(v) for v in boxes[f])
            al, be, ga = (float(v) for v in (angles[f] if angles is not None else (90.0, 90.0, 90.0)))
            out.append("CRYST1%9.3f%9.3f%9.3f%7.2f%7.2f%7.2f P 1           1\n" % (a, b, c, al, be, ga))
        for i in range(n):
            x, y, z = (float(v) for v in xyz[i])
            out.append(ATOM_LINE % (t["record"][i], int(t["serial"][i]) % 100000,
                                    _name_field(t["name"][i], t["element"][i]), t["altloc"][i],
                                    _resname_field(t["resname"][i]), t["chain"][i], int(t["resid"][i]),
                                    t["insertion"][i], x, y, z, float(t["occupancy"][i]), float(t["beta"][i]),
                                    t["segid"][i], t["element"][i], _charge_field(t["charge"][i])))
        out.append("ENDMDL\n")
    out.append("END\n")
    return "".join(out).encode("ascii")


def _is(line: bytes, word: bytes) -> bool:
    """the record name is ``word``, followed by a space or the end of the line"""
    return line[:len(word)] == word and (len(line) == len(word) or line[len(word):len(word) + 1] == b" ")


def _atom(line: bytes) -> dict:
    def text(a, b):
        return line[a:b].decode("ascii").strip()

    def num(a, b, kind, default):
        s = line[a:b].strip()
        return kind(s) if s else default

    ch = line[78:80].strip().decode("ascii")
    charge = 0.0
    if ch:
        charge = float(int(ch[:-1]) * (-1 if ch[-1] == "-" else 1)) if ch[-1] in "+-" else float(int(ch))
    return dict(record=text(0, 6), serial=num(6, 11, int, 0), name=text(12, 16), altloc=text(16, 17),
                resname=text(17, 21), chain=text(21, 22), resid=num(22, 26, int, 0), insertion=text(26, 27),
                occupancy=num(54, 60, float, 0.0), beta=num(60, 66, float, 0.0), segid=text(72, 76),
                element=text(76, 78), charge=charge)


def read(data: bytes) -> dict:
    """The file's bytes -> dict(natoms, coords (F, natoms, 3) float32, box (F, 3) float32, boxangles (F, 3) float32,
    topology (frame 0's atom records, a dict of lists)).  Atom records are the lines starting "ATOM  " or "HETATM";
    with MODEL records each MODEL starts a frame that ENDMDL, END or the next MODEL ends, without them the file is one
    frame ended by ENDMDL / END; a frame's cell is the last CRYST1 before its first atom record (zeros and 90 without
    one); every coordinate is np.float32(float(line[30:38])) and so on.  A last frame cut short by the end of the file
    is dropped; any other frame whose atom count differs from frame 0's raises ValueError."""
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    lines = [ln[:-1] if ln.endswith(b"\r") else ln for ln in lines]
    has_model = any(_is(ln, b"MODEL") for ln in lines)
    frames = []  # (coords, cell, closed, first line)
    cell = None
    cur = [] if not has_model else None
    cur_cell, cur_line = None, 1
    top = []
    for i, ln in enumerate(lines):
        if _is(ln, b"MODEL"):
            if cur is not None:
                frames.append((cur, cur_cell, True, cur_line))
            cur, cur_cell, cur_line = [], None, i + 1
        elif _is(ln, b"ENDMDL") or _is(ln, b"END"):
            if cur is not None:
                frames.append((cur, cur_cell, True, cur_line))
            cur = None
        elif ln[:6] == b"CRYST1":
            cell = [float(ln[6 + 9 * d:15 + 9 * d]) for d in range(3)] + \
                   [float(ln[33 + 7 * d:40 + 7 * d]) for d in range(3)]
        elif ln[:6] in (b"ATOM  ", b"HETATM") and cur is not None:
            if len(ln) < 54:
                raise ValueError(f"line {i + 1}: an atom line of {len(ln)} columns")
            if not cur:
                cur_cell = cell
            cur.append([float(ln[30:38]), float(ln[38:46]), float(ln[46:54])])
            if not frames:
                top.append(_atom(ln))
    if cur is not None:
        frames.append((cur, cur_cell, False, cur_line))
    natoms = len(frames[0][0]) if frames else 0
    if frames and len(frames) > 1 and not frames[-1][2] and len(frames[-1][0]) < natoms:
        frames.pop()
    for f, (c, _, _, line) in enumerate(frames):
        if len(c) != natoms:
            raise ValueError(f"frame {f} (line {line}): {len(c)} atom records, frame 0 has {natoms}")
    F = len(frames)
    coords = np.array([c for c, _, _, _ in frames], np.float32).reshape(F, natoms, 3)
    cells = np.array([cl if cl is not None else [0, 0, 0, 90, 90, 90] for _, cl, _, _ in frames],
                     np.float32).reshape(F, 6)
    topology = {k: [a[k] for a in top] for k in ("record", "serial", "name", "altloc", "resname", "chain", "resid",
                                                 "insertion", "occupancy", "beta", "segid", "element", "charge")}
    return dict(natoms=natoms, coords=coords, box=cells[:, :3], boxangles=cells[:, 3:], topology=topology)


def random_topology(n: int, seed: int) -> dict:
    """A seeded topology of ``n`` atoms covering the column rules: names of 1-4 characters with 1- and 2-letter
    elements, blank and set altlocs / chains / insertions / segids, 3- and 4-character resnames, charges from -3 to 3,
    serials past 99 999 and resids over the whole '%4d' range."""
    rng = np.random.default_rng(seed)
    letters = "ABCDEFGHIJKLMNOPQRSTUVWXYZ"

    def word(lo, hi):
        return "".join(rng.choice(list(letters + "0123456789'"), size=int(rng.integers(lo, hi + 1))))

    element = [str(rng.choice(["C", "N", "O", "H", "S", "FE", "CL", "NA", "ZN", ""])) for _ in range(n)]
    return dict(record=[str(rng.choice(["ATOM", "HETATM"])) for _ in range(n)],
                serial=[int(v) for v in rng.integers(0, 250000, n)],
                name=[word(1, 4) for _ in range(n)],
                altloc=[str(rng.choice(["", "", "A", "B"])) for _ in range(n)],
                resname=[word(1, 4) for _ in range(n)],
                chain=[str(rng.choice(["", "A", "B", "z"])) for _ in range(n)],
                resid=[int(v) for v in rng.integers(-999, 10000, n)],
                insertion=[str(rng.choice(["", "", "A"])) for _ in range(n)],
                occupancy=[float(np.float32(v)) for v in rng.choice([0.0, 1.0, 0.5, 12.34, -99.99, 999.99], n)],
                beta=[float(np.float32(v)) for v in rng.uniform(-99.99, 999.99, n)],
                segid=[word(0, 4) for _ in range(n)],
                element=element,
                charge=[float(v) for v in rng.integers(-3, 4, n)])
