"""An independent restatement of the multi-frame GROMACS GRO format in pure Python: a writer that formats every line
with ``%`` and a reader that slices columns and splits the free-format lines, with ``float()`` per value.  Test
infrastructure: the tests hold moleculekit_b200/gro.py and K29 to it, so it shares no code with them.

A frame is N + 3 lines:

    title                      free text; GROMACS writes "t= <time> step= <step>" into it
    N                          the atom count
    N atom lines               "%5d%-5s%5s%5d" (resid, resname, name, serial), three position fields of width w (nm),
                               optionally three velocity fields of width w (nm/ps)
    box                        3 values v1x v2y v3z or 9 values v1x v2y v3z v1y v1z v2x v2z v3x v3y (nm)

The reader takes w as the distance between the first '.' at or after column 21 of frame 0's first atom line and the
next '.', and velocities when that line holds 20 + 6w characters.
"""
from __future__ import annotations

import numpy as np

ORDER = ((0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 0), (1, 2), (2, 0), (2, 1))  # GRO's box fields as (vector, axis)


def write(frames, topology: dict, boxes, title: str = "", times=None, steps=None, velocities=None) -> bytes:
    """``frames``: a sequence of (natoms, 3) arrays in nm; ``topology``: a dict of per-atom resid, resname, name and
    serial; ``boxes``: one (3, 3) array of box vectors (rows) per frame; ``times`` / ``steps``: one value per frame or
    None; ``velocities``: a sequence of (natoms, 3) arrays or None -> the file's bytes.  The time and step fields are
    as wide as the widest value in the file; the box has 9 fields when any frame has a non-zero off-diagonal."""
    t = topology
    n = len(t["name"])
    boxes = [np.asarray(b, np.float32).reshape(3, 3) for b in boxes]
    nine = any(float(b[i, j]) != 0.0 for b in boxes for i, j in ORDER[3:])
    wt = max(len("%.5f" % float(v)) for v in times) if times is not None else 0
    ws = max(len("%d" % int(v)) for v in steps) if steps is not None else 0
    out = []
    for f, xyz in enumerate(frames):
        xyz = np.asarray(xyz, np.float32).reshape(n, 3)
        head = title
        if times is not None:
            head += " t= %*.5f" % (wt, float(times[f]))
        if steps is not None:
            head += " step= %*d" % (ws, int(steps[f]))
        out.append(head + "\n")
        out.append("%5d\n" % n)
        vel = None if velocities is None else np.asarray(velocities[f], np.float32).reshape(n, 3)
        for i in range(n):
            line = "%5d%-5s%5s%5d" % (int(t["resid"][i]) % 100000, t["resname"][i], t["name"][i],
                                     int(t["serial"][i]) % 100000)
            line += "%8.3f%8.3f%8.3f" % tuple(float(v) for v in xyz[i])
            if vel is not None:
                line += "%8.4f%8.4f%8.4f" % tuple(float(v) for v in vel[i])
            out.append(line + "\n")
        b = boxes[f]
        out.append("".join("%10.5f" % float(b[i, j]) for i, j in (ORDER if nine else ORDER[:3])) + "\n")
    return "".join(out).encode("ascii")


def _after(title: bytes, key: bytes):
    i = title.find(key)
    if i < 0:
        return None
    rest = title[i + len(key):].split()
    return rest[0] if rest else b""


def read(data: bytes) -> dict:
    """The file's bytes -> dict(natoms, width, velocities, coords (F, natoms, 3) float32, vels (F, natoms, 3) float32 or
    None, box (F, 3, 3) float32, time (F,) float64, step (F,) int64, topology (frame 0's resid, resname, name, serial
    as lists)).  Trailing whitespace-only lines are ignored and a last frame cut short is dropped; a count line that is
    not N, a short atom line, a box line of other than 3 or 9 values, or a field float() rejects raises ValueError."""
    if b"\r" in data.replace(b"\r\n", b""):
        raise ValueError("a lone CR")
    lines = data.rstrip(b" \t\n\v\f\r\x1c\x1d\x1e\x1f").split(b"\n")
    lines = [ln[:-1] if ln.endswith(b"\r") else ln for ln in lines]
    N = int(lines[1].split()[0])
    first = lines[2]
    i = first.find(b".", 20)
    j = first.find(b".", i + 1)
    w = j - i
    if i < 0 or j < 0 or first.find(b".", j + 1) != j + w:
        raise ValueError("inconsistent decimal spacing")
    vel = len(first) >= 20 + 6 * w
    cols = 20 + (6 if vel else 3) * w
    P = N + 3
    F = len(lines) // P
    coords = np.zeros((F, N, 3), np.float32)
    vels = np.zeros((F, N, 3), np.float32) if vel else None
    box = np.zeros((F, 3, 3), np.float32)
    time = np.full(F, np.nan)
    step = np.full(F, -1, np.int64)
    for f in range(F):
        ls = lines[f * P:(f + 1) * P]
        if int(ls[1].split()[0]) != N:
            raise ValueError(f"frame {f}: the atom count is not {N}")
        for a in range(N):
            ln = ls[2 + a]
            if len(ln) < cols:
                raise ValueError(f"frame {f}, atom {a}: a short atom line")
            for d in range(3):
                coords[f, a, d] = np.float32(float(ln[20 + w * d:20 + w * (d + 1)]))
                if vel:
                    vels[f, a, d] = np.float32(float(ln[20 + w * (3 + d):20 + w * (4 + d)]))
        toks = ls[N + 2].split()
        if len(toks) not in (3, 9):
            raise ValueError(f"frame {f}: the box line holds {len(toks)} values")
        for (bi, bj), tok in zip(ORDER, toks):
            box[f, bi, bj] = np.float32(float(tok))
        tt = _after(ls[0], b" t= ")
        if tt is not None:
            try:
                time[f] = float(tt)
            except ValueError:
                pass
        st = _after(ls[0], b" step= ")
        if st is not None:
            try:
                step[f] = int(st)
            except ValueError:
                pass
    top = lines[2:2 + N]
    topology = dict(resid=[int(ln[0:5]) for ln in top], resname=[ln[5:10].decode("ascii").strip() for ln in top],
                    name=[ln[10:15].decode("ascii").strip() for ln in top], serial=[int(ln[15:20]) for ln in top])
    return dict(natoms=N, width=w, velocities=vel, coords=coords, vels=vels, box=box, time=time, step=step,
                topology=topology)


def random_topology(n: int, seed: int) -> dict:
    """A seeded topology of ``n`` atoms: resnames and names of 1-5 characters, resids and serials past 99 999."""
    rng = np.random.default_rng(seed)
    letters = list("ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789'*")

    def word():
        return "".join(rng.choice(letters, size=int(rng.integers(1, 6))))

    return dict(resid=[int(v) for v in rng.integers(0, 250000, n)], resname=[word() for _ in range(n)],
                name=[word() for _ in range(n)], serial=[int(v) for v in rng.integers(0, 250000, n)])
