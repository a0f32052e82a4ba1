"""Independent reference for K32 (LAMMPS dump trajectories): a ``%`` writer, a ``split()`` / ``float()`` / ``int()``
reader, and hand-made test files.

No LAMMPS-written file is available here, so the layouts of ``make_file`` are restated from the LAMMPS documentation
of ``dump atom`` / ``dump custom`` and ``dump_modify`` (items UNITS, TIME, TIMESTEP, NUMBER OF ATOMS, BOX BOUNDS and
ATOMS; orthogonal and restricted-triclinic bounds; the x / xs / xu / xsu coordinate columns and ix iy iz image flags;
atoms in any order unless ``dump_modify sort id``).  The box rules are LAMMPS's restricted-triclinic ones:
xlo = xlo_bound - min(0, xy, xz, xy + xz), xhi = xhi_bound - max(0, xy, xz, xy + xz), ylo = ylo_bound - min(0, yz),
yhi = yhi_bound - max(0, yz), l = hi - lo, every step a float64 operation in that order."""
from __future__ import annotations

import numpy as np

STYLES = ("x", "xu", "xs", "xsu")
TRIPLES = {"x": ("x", "y", "z"), "xu": ("xu", "yu", "zu"), "xs": ("xs", "ys", "zs"), "xsu": ("xsu", "ysu", "zsu")}


def lohi(bounds):
    """(3, 3) float64 bound lines (lo_bound, hi_bound, tilt) -> (xlo, ylo, zlo, lx, ly, lz, xy, xz, yz)"""
    (xlb, xhb, xy), (ylb, yhb, xz), (zlb, zhb, yz) = (tuple(float(v) for v in r) for r in bounds)
    xlo = xlb - min(0.0, xy, xz, xy + xz)
    xhi = xhb - max(0.0, xy, xz, xy + xz)
    ylo = ylb - min(0.0, yz)
    yhi = yhb - max(0.0, yz)
    return xlo, ylo, zlb, xhi - xlo, yhi - ylo, zhb - zlb, xy, xz, yz


def bound_lines(box, origin):
    """(3, 3) float32 box vectors (rows a, b, c, lower-triangular) and origin (3,) -> (3, 3) float64 bound lines"""
    lx, xy, ly, xz, yz, lz = (float(box[0, 0]), float(box[1, 0]), float(box[1, 1]), float(box[2, 0]), float(box[2, 1]),
                              float(box[2, 2]))
    ox, oy, oz = (float(v) for v in origin)
    return np.array([[ox + min(0.0, xy, xz, xy + xz), ox + lx + max(0.0, xy, xz, xy + xz), xy],
                     [oy + min(0.0, yz), oy + ly + max(0.0, yz), xz],
                     [oz, oz + lz, yz]])


def write(coords, box, step=None, time=None, ids=None, types=None, velocities=None, origin=None, units=None) -> bytes:
    """coords: list of (N, 3) float32 frames; box: list of (3, 3) float32 vectors -> the file's bytes"""
    N = len(coords[0])
    ids = range(1, N + 1) if ids is None else [int(v) for v in ids]
    types = [1] * N if types is None else [int(v) for v in types]
    out = []
    for f, x in enumerate(coords):
        if units is not None and f == 0:
            out.append("ITEM: UNITS\n%s\n" % units)
        if time is not None:
            out.append("ITEM: TIME\n%.16g\n" % float(time[f]))
        out.append("ITEM: TIMESTEP\n%d\n" % (f if step is None else int(step[f])))
        out.append("ITEM: NUMBER OF ATOMS\n%d\n" % N)
        b = bound_lines(box[f], (0.0, 0.0, 0.0) if origin is None else origin[f])
        if b[0, 2] == 0 and b[1, 2] == 0 and b[2, 2] == 0:
            out.append("ITEM: BOX BOUNDS pp pp pp\n")
            out.extend("%-1.16e %-1.16e\n" % (r[0], r[1]) for r in b)
        else:
            out.append("ITEM: BOX BOUNDS xy xz yz pp pp pp\n")
            out.extend("%-1.16e %-1.16e %-1.16e\n" % tuple(r) for r in b)
        v = None if velocities is None else velocities[f]
        out.append("ITEM: ATOMS id type x y z%s\n" % ("" if v is None else " vx vy vz"))
        for a in range(N):
            vals = [float(np.float32(t)) for t in x[a]] + ([] if v is None else [float(np.float32(t)) for t in v[a]])
            out.append("%d %d " % (ids[a], types[a]) + " ".join("%.9g" % t for t in vals) + "\n")
    return "".join(out).encode("ascii")


def read(raw: bytes, style=None, unwrap=False):
    """the file's bytes -> dict(coords (F, N, 3) float32, v / f (F, N, 3) float32 or None, box (F, 3, 3) float32 rows,
    bounds (F, 3, 3), origin (F, 3), step, time, ids (frame 0's, ascending), type, columns, units)"""
    lines = raw.decode("utf-8").replace("\r\n", "\n").split("\n")
    while lines and not lines[-1].strip():
        lines.pop()
    i, units, frames = 0, None, []
    if lines[0].strip() == "ITEM: UNITS":
        units, i = lines[1].strip(), 2
    while i < len(lines):
        fr = {"time": np.nan}
        while True:
            item = lines[i].strip()
            i += 1
            if item == "ITEM: TIME":
                fr["time"] = float(lines[i]); i += 1
            elif item == "ITEM: TIMESTEP":
                fr["step"] = int(lines[i]); i += 1
            elif item == "ITEM: NUMBER OF ATOMS":
                fr["n"] = int(lines[i]); i += 1
            elif item.startswith("ITEM: BOX BOUNDS"):
                tilt = item.split()[3:6] == ["xy", "xz", "yz"]
                b = np.zeros((3, 3))
                for d in range(3):
                    b[d, :3 if tilt else 2] = [float(t) for t in lines[i + d].split()]
                fr["bounds"] = b
                i += 3
            elif item.startswith("ITEM: ATOMS"):
                fr["columns"] = item.split()[2:]
                fr["rows"] = [lines[i + a].split() for a in range(fr["n"])]
                i += fr["n"]
                break
        frames.append(fr)
    cols = frames[0]["columns"]
    style = style or next(s for s in STYLES if all(c in cols for c in TRIPLES[s]))
    pos = [cols.index(c) for c in TRIPLES[style]]
    img = [cols.index(c) for c in ("ix", "iy", "iz")] if unwrap and style in ("x", "xs") else None
    key = (lambda r: int(r[cols.index("id")])) if "id" in cols else None
    ids0 = sorted(key(r) for r in frames[0]["rows"]) if key else None
    F, N = len(frames), frames[0]["n"]
    out = dict(coords=np.empty((F, N, 3), np.float32), box=np.zeros((F, 3, 3), np.float32), bounds=np.empty((F, 3, 3)),
               origin=np.empty((F, 3)), step=np.array([fr["step"] for fr in frames], np.int64),
               time=np.array([fr["time"] for fr in frames]), columns=cols, units=units, v=None, f=None)
    for name, c3 in (("v", ("vx", "vy", "vz")), ("f", ("fx", "fy", "fz"))):
        if all(c in cols for c in c3):
            out[name] = np.empty((F, N, 3), np.float32)
    for f, fr in enumerate(frames):
        xlo, ylo, zlo, lx, ly, lz, xy, xz, yz = lohi(fr["bounds"])
        out["bounds"][f], out["origin"][f] = fr["bounds"], (xlo, ylo, zlo)
        out["box"][f] = np.float32([[lx, 0, 0], [xy, ly, 0], [xz, yz, lz]])
        rows = sorted(fr["rows"], key=key) if key else fr["rows"]
        for a, r in enumerate(rows):
            x, y, z = (float(r[c]) for c in pos)
            if style in ("xs", "xsu"):
                x, y, z = ((xlo + x * lx) + y * xy) + z * xz, (ylo + y * ly) + z * yz, zlo + z * lz
            if img is not None:
                ix, iy, iz = (float(int(r[c])) for c in img)
                x, y, z = x + ((ix * lx + iy * xy) + iz * xz), y + (iy * ly + iz * yz), z + iz * lz
            out["coords"][f, a] = np.float32([x, y, z])
            for name, c3 in (("v", ("vx", "vy", "vz")), ("f", ("fx", "fy", "fz"))):
                if out[name] is not None:
                    out[name][f, a] = [np.float32(float(r[cols.index(c)])) for c in c3]
    out["ids"] = np.array(ids0 if ids0 else range(1, N + 1), np.int64)
    rows0 = sorted(frames[0]["rows"], key=key) if key else frames[0]["rows"]
    out["type"] = np.array([int(r[cols.index("type")]) for r in rows0], np.int64) if "type" in cols else None
    return out


def make_file(rng, N: int, F: int, columns, triclinic=False, shuffle=False, ids=None, units=None, time=False,
              crlf=False, trailing=False, fmt="%.9g") -> bytes:
    """a dump custom file in the layout the LAMMPS documentation describes: ``columns`` names the ATOMS columns (id,
    type, mol, element, q, x y z, xs ys zs, xu yu zu, xsu ysu zsu, ix iy iz, vx vy vz, fx fy fz, c_* / v_*), atoms in
    a random order per frame with ``shuffle``, bound lines with tilts with ``triclinic``"""
    ids = np.arange(1, N + 1) if ids is None else np.asarray(ids)
    out = []
    eol = "\r\n" if crlf else "\n"
    pad = "  " if trailing else ""
    for f in range(F):
        lx, ly, lz = rng.uniform(20, 40, 3)
        xy, xz, yz = rng.uniform(-5, 5, 3) if triclinic else (0.0, 0.0, 0.0)
        o = rng.uniform(-10, 10, 3)
        b = bound_lines(np.float32([[lx, 0, 0], [xy, ly, 0], [xz, yz, lz]]), o)
        if units is not None and f == 0:
            out.append("ITEM: UNITS" + pad + eol + units + eol)
        if time:
            out.append("ITEM: TIME" + eol + repr(float(f) * 0.5 + 0.125) + eol)
        out.append("ITEM: TIMESTEP" + pad + eol + "%d" % (1000 * f) + pad + eol)
        out.append("ITEM: NUMBER OF ATOMS" + eol + "%d" % N + eol)
        if triclinic:
            out.append("ITEM: BOX BOUNDS xy xz yz pp pp pp" + pad + eol)
            out.extend("%-1.16e %-1.16e %-1.16e" % tuple(r) + pad + eol for r in b)
        else:
            out.append("ITEM: BOX BOUNDS pp pp pp" + pad + eol)
            out.extend("%-1.16e %-1.16e" % (r[0], r[1]) + pad + eol for r in b)
        out.append("ITEM: ATOMS " + " ".join(columns) + pad + eol)
        order = rng.permutation(N) if shuffle else np.arange(N)
        for a in order:
            row = []
            for c in columns:
                if c == "id":
                    row.append("%d" % ids[a])
                elif c in ("type", "mol"):
                    row.append("%d" % (1 + (a * 7 + (c == "mol")) % 5))
                elif c == "element":
                    row.append(("C", "N", "O", "H")[a % 4])
                elif c in ("ix", "iy", "iz"):
                    row.append("%d" % rng.integers(-3, 4))
                elif c in ("xs", "ys", "zs", "xsu", "ysu", "zsu"):
                    row.append(fmt % rng.uniform(-0.5, 1.5))
                else:
                    row.append(fmt % rng.normal(0, 15))
            out.append(" ".join(row) + pad + eol)
    return "".join(out).encode("ascii")
