"""An independent restatement of the DCD format in pure Python / numpy: a writer and a reader written from the record
layout of the VMD molfile DCD plugin (moleculekit/fileformats/dcd/src/dcdplugin.c: read_dcdheader, read_charmm_timestep,
read_next_timestep, write_dcdheader, write_dcdstep).  Test infrastructure: the tests hold moleculekit_b200/dcd.py and
K22 to it, so it shares no code with them.

The writer covers more than the product writes: both byte orders, 4- and 8-byte record markers, CHARMM and X-PLOR
headers, unit cells stored as cosines or in degrees (or an extra block of another length), the 4D record, fixed atoms,
an explicit title, and any NSET in the header.  Coordinates are (F, N, 3) float32 here, the plugin's frame-major layout.

A file:

    [84] "CORD" ICNTRL[20] [84]          ICNTRL: 0 NSET, 1 ISTART, 2 NSAVC, 3 ISTART + NSET * NSAVC, 8 NAMNF,
                                         9 DELTA (float32; X-PLOR: float64 over 9..10), 10 extra block, 11 4D, 19 version
    [4 + 80 NTITLE] NTITLE lines [..]
    [4] NATOM [4]
    [4 NFREE] free atoms (1-based) [..]  only when NAMNF > 0
    per frame: [len] extra block [len]   CHARMM with ICNTRL[10] != 0; a unit cell when len = 48 (6 float64)
               [4 n] X [4 n]  [4 n] Y [4 n]  [4 n] Z [4 n]      n = NATOM in the first frame, NFREE in later ones
               [len] 4D record [len]     CHARMM with ICNTRL[11] == 1
"""
from __future__ import annotations

import math
import struct

import numpy as np

HALF_PI = 1.57079632679489661923


def cosine_cell(a, b, c, alpha, beta, gamma) -> list:
    """the plugin writer's unit cell from float32 lengths and angles: A, cos(gamma), B, cos(beta), cos(alpha), C"""
    a, b, c, alpha, beta, gamma = (float(np.float32(v)) for v in (a, b, c, alpha, beta, gamma))
    k = HALF_PI / 90.0
    return [a, math.sin(k * (90.0 - gamma)), b, math.sin(k * (90.0 - beta)), math.sin(k * (90.0 - alpha)), c]


def cell_to_box(uc) -> tuple:
    """the plugin reader's (A, B, C, alpha, beta, gamma) as float32 from one 6-double unit cell"""
    uc = [float(v) for v in uc]
    if -1.0 <= uc[1] <= 1.0 and -1.0 <= uc[3] <= 1.0 and -1.0 <= uc[4] <= 1.0:
        alpha = 90.0 - math.asin(uc[4]) * 90.0 / HALF_PI
        beta = 90.0 - math.asin(uc[3]) * 90.0 / HALF_PI
        gamma = 90.0 - math.asin(uc[1]) * 90.0 / HALF_PI
    else:
        alpha, beta, gamma = uc[4], uc[3], uc[1]
    return tuple(np.float32(v) for v in (uc[0], uc[2], uc[5], alpha, beta, gamma))


def write(coords, *, endian: str = "<", marker: int = 4, charmm: bool = True, cells=None, four_d: bool = False,
          free=None, title=("REMARKS oracle",), istart: int = 0, nsavc: int = 1, delta: float = 1.0, nset=None,
          icntrl3=None, pad: bytes = b" ") -> bytes:
    """coords (F, N, 3) float32 -> a DCD file.  ``cells``: (F, k) float64 extra blocks (k = 6: unit cells; CHARMM only);
    ``free``: 1-based indices of the free atoms (their count sets NAMNF = N - len(free)); ``nset`` / ``icntrl3``: header
    values other than the frame count and ISTART + NSET * NSAVC."""
    coords = np.asarray(coords, dtype=np.float32)
    F, N = coords.shape[0], coords.shape[1]
    i32, f32, f64 = endian + "i", endian + "f4", endian + "f8"

    def rec(payload: bytes) -> bytes:
        m = struct.pack(endian + ("i" if marker == 4 else "q"), len(payload))
        return m + payload + m

    ic = [0] * 20
    ic[0] = F if nset is None else nset
    ic[1], ic[2] = istart, nsavc
    ic[3] = (istart + ic[0] * nsavc) if icntrl3 is None else icntrl3
    ic[8] = 0 if free is None else N - len(free)
    body = b"CORD" + b"".join(struct.pack(i32, v) for v in ic[:9])
    if charmm:
        ic[10] = 0 if cells is None else 1
        ic[11] = 1 if four_d else 0
        ic[19] = 24
        body += struct.pack(endian + "f", delta) + b"".join(struct.pack(i32, v) for v in ic[10:])
    else:
        body += struct.pack(endian + "d", delta) + b"".join(struct.pack(i32, v) for v in ic[11:])
    assert len(body) == 84
    out = [rec(body)]
    lines = [t.encode("latin-1")[:80].ljust(80, pad) for t in title]
    out.append(rec(struct.pack(i32, len(lines)) + b"".join(lines)))
    out.append(rec(struct.pack(i32, N)))
    if free is not None:
        out.append(rec(np.asarray(free, dtype=i32).tobytes()))
    for f in range(F):
        if charmm and cells is not None:
            out.append(rec(np.asarray(cells[f], dtype=f64).tobytes()))
        xyz = coords[f] if (free is None or f == 0) else coords[f][np.asarray(free) - 1]
        for d in range(3):
            out.append(rec(np.ascontiguousarray(xyz[:, d]).astype(f32).tobytes()))
        if charmm and four_d:
            out.append(rec(np.full(len(xyz), 0.5, dtype=f32).tobytes()))
    return b"".join(out)


class Malformed(Exception):
    pass


def read(data: bytes) -> dict:
    """A DCD file -> dict(natoms, nset, istart, nsavc, icntrl3, delta, namnf, charmm, extra, four_d, title, free (1-based
    or None), endian, marker, coords (F, N, 3) float32, cells (F, 6) float64 (zeros where a frame has none),
    box (F, 3) and angles (F, 3) float32).  Reads frame after frame and stops before an incomplete one; a marker that
    does not match raises Malformed."""
    a, b = struct.unpack_from("<ii", data, 0)
    if a + b == 84 and data[8:12] == b"CORD":
        endian, marker = "<", 8
    elif a == 84 and data[4:8] == b"CORD":
        endian, marker = "<", 4
    else:
        a, b = struct.unpack_from(">ii", data, 0)
        if a + b == 84 and data[8:12] == b"CORD":
            endian, marker = ">", 8
        elif a == 84 and data[4:8] == b"CORD":
            endian, marker = ">", 4
        else:
            raise Malformed("not a DCD file")
    mfmt = endian + ("i" if marker == 4 else "q")
    pos = 0

    def next_record(expect=None):
        nonlocal pos
        if pos + marker > len(data):
            raise EOFError
        (n,) = struct.unpack_from(mfmt, data, pos)
        if expect is not None and n != expect:
            raise Malformed(f"record at {pos}: length {n}, expected {expect}")
        if pos + 2 * marker + n > len(data):
            raise EOFError
        (m,) = struct.unpack_from(mfmt, data, pos + marker + n)
        if m != n:
            raise Malformed(f"record at {pos}: markers {n} and {m}")
        payload = data[pos + marker:pos + marker + n]
        pos += 2 * marker + n
        return payload

    head = next_record(84)
    ic = struct.unpack(endian + "20i", head[4:84])
    charmm = ic[19] != 0
    delta = struct.unpack(endian + ("f" if charmm else "d"), head[40:44] if charmm else head[40:48])[0]
    extra = charmm and ic[10] != 0
    four_d = charmm and ic[11] == 1
    t = next_record()
    ntitle = struct.unpack(endian + "i", t[:4])[0]
    if len(t) != 4 + 80 * ntitle:
        raise Malformed("title record")
    title = [t[4 + 80 * i:84 + 80 * i].decode("latin-1") for i in range(ntitle)]
    natoms = struct.unpack(endian + "i", next_record(4))[0]
    namnf = ic[8]
    free = None
    if namnf > 0:
        free = np.frombuffer(next_record(4 * (natoms - namnf)), dtype=endian + "i4").astype(np.int64)
    frames, cells = [], []
    while True:
        start = pos
        try:
            cell = np.zeros(6)
            if extra:
                blk = next_record()
                if len(blk) == 48:
                    cell = np.frombuffer(blk, dtype=endian + "f8").astype(np.float64)
            n = natoms if (free is None or not frames) else len(free)
            xyz = [np.frombuffer(next_record(4 * n), dtype=endian + "f4").astype(np.float32) for _ in range(3)]
            if four_d:
                next_record()
        except EOFError:
            pos = start
            break
        fr = np.stack(xyz, axis=1)
        if free is not None and frames:
            full = frames[0].copy()
            full[free - 1] = fr
            fr = full
        frames.append(fr)
        cells.append(cell)
    F = len(frames)
    coords = np.stack(frames) if F else np.zeros((0, natoms, 3), np.float32)
    cells = np.array(cells, dtype=np.float64).reshape(F, 6)
    box = np.zeros((F, 3), np.float32)
    angles = np.full((F, 3), 90.0, np.float32)
    for f in range(F):
        if extra and cells[f].any():
            v = cell_to_box(cells[f])
            box[f], angles[f] = v[:3], v[3:]
    return dict(natoms=natoms, nset=ic[0], istart=ic[1], nsavc=ic[2], icntrl3=ic[3], delta=delta, namnf=namnf,
                charmm=charmm, extra=extra, four_d=four_d, title=title, free=free, endian=endian, marker=marker,
                coords=coords, cells=cells, box=box, angles=angles, trailing=len(data) - pos)
