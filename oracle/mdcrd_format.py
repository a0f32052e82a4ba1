"""An independent restatement of AMBER's ASCII trajectory format (mdcrd / crd / trj, and mdvel) in pure Python: a writer
that formats every value with ``'%8.3f'`` and a reader that converts every field with ``float()``.  Test
infrastructure: the tests hold moleculekit_b200/mdcrd.py and K25 to it, so it shares no code with them.

A file, as sander / pmemd write it with ioutfm=0:

    title line                                           the title padded to 80 columns, then a newline
    per frame: 3 natoms values, atom-major (x y z of atom 0, then atom 1, ...), Fortran F8.3, ten per line, each line
               ending in a newline (the last one after the frame's last value)
               [with a periodic box: one line of three F8.3 fields, A B C, and a newline]
"""
from __future__ import annotations

import numpy as np


def _lines(values):
    vals = ["%8.3f" % float(v) for v in values]
    return "".join("".join(vals[i:i + 10]) + "\n" for i in range(0, len(vals), 10))


def write(frames, boxes=None, title: str = "") -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays; ``boxes``: None or one (3,) array per frame -> the file's bytes.
    Values are formatted as they are; a value that '%8.3f' prints wider than 8 characters is the caller's problem."""
    out = [title.ljust(80) + "\n"]
    for k, xyz in enumerate(frames):
        out.append(_lines(np.asarray(xyz, np.float32).reshape(-1)))
        if boxes is not None:
            out.append(_lines(np.asarray(boxes[k], np.float32).reshape(3)))
    return "".join(out).encode("ascii")


def read(data: bytes, natoms: int, box: bool) -> dict:
    """The file's bytes -> dict(title (the first line without its newline), coords (F, natoms, 3) float32, box (F, 3)
    float32 or None, trailing: the bytes after the last whole frame).  Every field goes through ``float()``; a line
    whose length is not what the layout says raises ValueError."""
    text = data.decode("ascii")
    end = text.index("\n")
    title, pos = text[:end], end + 1
    n = 3 * natoms
    widths = [80] * (n // 10) + ([8 * (n % 10)] if n % 10 else [])
    if box:
        widths.append(24)
    frame_len = sum(w + 1 for w in widths)
    coords, boxes = [], []
    while pos + frame_len <= len(text):
        vals = []
        for w in widths:
            line = text[pos:pos + w]
            if text[pos + w] != "\n" or "\n" in line:
                raise ValueError(f"line at byte {pos} is not {w} characters long")
            vals += [float(line[c:c + 8]) for c in range(0, w, 8)]
            pos += w + 1
        coords.append(np.float32(vals[:n]).reshape(natoms, 3))
        if box:
            boxes.append(np.float32(vals[n:]))
    F = len(coords)
    return dict(title=title, coords=np.array(coords, np.float32).reshape(F, natoms, 3),
                box=np.array(boxes, np.float32).reshape(F, 3) if box else None, trailing=len(text) - pos)
