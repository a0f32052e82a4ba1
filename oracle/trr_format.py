"""An independent restatement of the GROMACS TRR format in pure Python / numpy: a writer and a reader written from the
frame layout of xdrfile (xdrfile_trr.c: do_trnheader, do_htrn, nFloatSize), which moleculekit vendors under
moleculekit/fileformats/xtc/.  Test infrastructure: the tests hold moleculekit_b200/trr.py and K24 to it, so it shares no
code with them.

The writer covers more than the product writes: both precisions, and any per-frame mix of box, vir, pres, x, v and f,
with step, time and lambda.  Arrays are (natoms, 3) per frame here, xdrfile's layout.

A frame, every value big-endian XDR:

    int32 1993, int32 13, uint32 12, "GMX_trn_file"
    int32 ir_size, e_size, box_size, vir_size, pres_size, top_size, sym_size, x_size, v_size, f_size, natoms
    int32 step, int32 nre
    real t, real lambda                                       real = float32 or float64 (the precision w, 4 or 8)
    [box 9 reals] [vir 9 reals] [pres 9 reals] [x 3N reals] [v 3N reals] [f 3N reals]   each when its size is not 0

w is box_size / 9, or else x_size / 3N, v_size / 3N, f_size / 3N: the first of them that is not 0.
"""
from __future__ import annotations

import struct

import numpy as np

MAGIC = 1993
BLOCKS = ("box", "vir", "pres", "x", "v", "f")


def frame(natoms: int, step: int = 0, time: float = 0.0, lambd: float = 0.0, **blocks) -> dict:
    """one frame for :func:`write`: ``blocks`` maps box / vir / pres to (3, 3) and x / v / f to (natoms, 3) arrays"""
    bad = set(blocks) - set(BLOCKS)
    assert not bad, bad
    return dict(natoms=natoms, step=step, time=time, lambd=lambd, **{k: blocks.get(k) for k in BLOCKS})


def write(frames, double: bool = False) -> bytes:
    """A list of :func:`frame` dicts -> a TRR file in one precision (float64 reals when ``double``)."""
    w = 8 if double else 4
    real = ">d" if double else ">f"
    out = []
    for fr in frames:
        n = fr["natoms"]
        sizes = {k: 0 if fr[k] is None else (9 if k in ("box", "vir", "pres") else 3 * n) * w for k in BLOCKS}
        head = struct.pack(">ii", MAGIC, 13) + struct.pack(">I", 12) + b"GMX_trn_file"
        head += struct.pack(">11i", 0, 0, sizes["box"], sizes["vir"], sizes["pres"], 0, 0, sizes["x"], sizes["v"],
                            sizes["f"], n)
        head += struct.pack(">ii", fr["step"], 0)
        head += struct.pack(real, fr["time"]) + struct.pack(real, fr["lambd"])
        out.append(head)
        for k in BLOCKS:
            if fr[k] is not None:
                out.append(np.asarray(fr[k], dtype=real).reshape(-1).tobytes())
    return b"".join(out)


class Malformed(Exception):
    pass


def read(data: bytes) -> dict:
    """A TRR file -> dict(double, natoms, frames: a list of dict(step, time, lambd, offset, and box / vir / pres (3, 3)
    / x / v / f (natoms, 3) arrays in the file's precision, native byte order, bits unchanged, or None), trailing: the
    bytes of an incomplete last frame).  Every frame must have the precision and atom count of the first."""
    pos, frames, double, natoms = 0, [], None, None
    while pos < len(data):
        start = pos
        if pos + 76 > len(data):
            break
        magic, slen, n12 = struct.unpack_from(">iiI", data, pos)
        if magic != MAGIC or slen != 13 or n12 != 12:
            raise Malformed(f"frame at {pos}: header {magic} {slen} {n12}")
        v = struct.unpack_from(">11i", data, pos + 24)
        sizes = dict(ir=v[0], e=v[1], box=v[2], vir=v[3], pres=v[4], top=v[5], sym=v[6], x=v[7], v=v[8], f=v[9])
        n = v[10]
        step, _nre = struct.unpack_from(">ii", data, pos + 68)
        if sizes["box"]:
            w = sizes["box"] // 9
        elif sizes["x"]:
            w = sizes["x"] // (3 * n)
        elif sizes["v"]:
            w = sizes["v"] // (3 * n)
        elif sizes["f"]:
            w = sizes["f"] // (3 * n)
        else:
            raise Malformed(f"frame at {pos}: no box, x, v or f")
        if w not in (4, 8) or any(sizes[k] for k in ("ir", "e", "top", "sym")):
            raise Malformed(f"frame at {pos}: sizes {sizes}")
        for k in BLOCKS:
            if sizes[k] not in (0, (9 if k in ("box", "vir", "pres") else 3 * n) * w):
                raise Malformed(f"frame at {pos}: {k} size {sizes[k]}")
        if double is None:
            double, natoms = w == 8, n
        elif double != (w == 8) or natoms != n:
            raise Malformed(f"frame at {pos}: precision or atom count changes")
        real = ">d" if w == 8 else ">f"
        hsize = 76 + 2 * w
        if pos + hsize > len(data):
            break
        t, lam = struct.unpack_from(">dd" if w == 8 else ">ff", data, pos + 76)
        pos += hsize
        fr = dict(step=step, time=t, lambd=lam, offset=start)
        complete = True
        for k in BLOCKS:
            if sizes[k] == 0:
                fr[k] = None
                continue
            if pos + sizes[k] > len(data):
                complete = False
                break
            a = np.frombuffer(data, dtype=real, count=sizes[k] // w, offset=pos).astype(np.float64 if w == 8 else np.float32)
            fr[k] = a.reshape(3, 3) if k in ("box", "vir", "pres") else a.reshape(n, 3)
            pos += sizes[k]
        if not complete:
            pos = start
            break
        frames.append(fr)
    return dict(double=bool(double), natoms=natoms or 0, frames=frames, trailing=len(data) - pos)
