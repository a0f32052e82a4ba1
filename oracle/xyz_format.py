"""An independent restatement of the multi-frame XYZ format in pure Python: a writer that formats every line with
``%`` and a reader that restates the reference's loop (text mode, ``split()``, ``int()`` and ``float()`` per line).
Test infrastructure: the tests hold moleculekit_b200/xyz.py and K26 to it, so it shares no code with them.

A file, per frame:

    natoms                    the atom count, "%d"
    comment                   one line
    natoms atom lines         element x y z [more fields], whitespace separated, x y z in Angstrom
"""
from __future__ import annotations

import io

import numpy as np


def write(frames, element, comment: str = "") -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays; ``element``: natoms strings -> the file's bytes, per atom
    ``"%-*s %15.8f %15.8f %15.8f\\n"`` with the element column as wide as the longest element."""
    w = max((len(e) for e in element), default=0)
    out = []
    for xyz in frames:
        xyz = np.asarray(xyz, np.float32).reshape(len(element), 3)
        out.append("%d\n%s\n" % (len(element), comment))
        out.extend("%-*s %15.8f %15.8f %15.8f\n" % (w, e, float(x), float(y), float(z))
                   for e, (x, y, z) in zip(element, xyz))
    return "".join(out).encode("ascii")


def read(data: bytes) -> dict:
    """The file's bytes -> dict(natoms, element (frame 0's field 0), comment (frame 0's), coords (F, natoms, 3)
    float32).  The reference's loop: text mode (universal newlines), ``int(line.split()[0])`` for the count,
    ``np.float32(float(field))`` for fields 1-3 of every atom line.  Blank lines after the last frame are skipped and an
    incomplete last frame is dropped, as the reader under test does."""
    lines = io.TextIOWrapper(io.BytesIO(data), encoding="utf-8", newline=None).read().split("\n")
    if lines and lines[-1] == "":
        lines.pop()  # the newline that ends the last line
    while lines and not lines[-1].split():
        lines.pop()
    natoms = int(lines[0].split()[0])
    element = [ln.split()[0] for ln in lines[2:2 + natoms]]
    comment = lines[1]
    frames = []
    pos = 0
    while pos + natoms + 2 <= len(lines):
        n = int(lines[pos].split()[0])
        if n != natoms:
            raise ValueError(f"line {pos + 1}: atom count {n}, frame 0 has {natoms}")
        frames.append(np.float32([[float(v) for v in ln.split()[1:4]] for ln in lines[pos + 2:pos + 2 + natoms]]))
        pos += natoms + 2
    F = len(frames)
    return dict(natoms=natoms, element=element, comment=comment,
                coords=np.array(frames, np.float32).reshape(F, natoms, 3))
