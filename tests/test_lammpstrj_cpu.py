"""K32 (LAMMPS dump trajectories) without a GPU: the frame-0 header and column parsing, the box-bound conversions in
both directions, the writer's argument checks (each fires before the file exists), the C-ABI symbols, the oracle's
round trip, and K32's '%.9g' formatter (csrc/lammpstrj_g9.cuh) built with the host compiler against Python's %."""
import os
import shutil
import subprocess
import sys
from decimal import Decimal, getcontext

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from moleculekit_b200 import lammpstrj  # noqa: E402
from oracle import lammpstrj_format as lf  # noqa: E402


def _write(tmp_path, raw, name="t.lammpstrj"):
    p = tmp_path / name
    p.write_bytes(raw)
    return str(p)


def test_frame0_header_and_columns(tmp_path):
    rng = np.random.default_rng(0)
    raw = lf.make_file(rng, 5, 2, ["id", "type", "mol", "element", "q", "xs", "ys", "zs", "ix", "iy", "iz"],
                       triclinic=True, shuffle=True, ids=[10, 3, 7, 40, 2], units="real", time=True, trailing=True)
    fn = _write(tmp_path, raw)
    with open(fn, "rb") as fh:
        h = lammpstrj._frame0(fn, fh.fileno(), len(raw.rstrip()))
    assert h["units"] == "real" and h["units_lines"] == 2
    assert h["items"] == ["TIME", "TIMESTEP", "NUMBER OF ATOMS", "BOX BOUNDS", "ATOMS"]
    assert h["columns"] == ["id", "type", "mol", "element", "q", "xs", "ys", "zs", "ix", "iy", "iz"]
    assert h["H"] == 11 and h["count_line"] == 5 and h["step_line"] == 3 and h["time_line"] == 1
    assert h["box_line"] == 7 and h["tilt"] and h["time"] == 0.125 and h["step"] == 0
    assert h["topology"]["ids"].tolist() == [2, 3, 7, 10, 40]
    want = lf.read(raw)
    assert h["topology"]["type"].tolist() == want["type"].tolist()
    role = lammpstrj._roles(h["columns"], "xs", ("x",), True)
    assert role.tolist() == [1, 0, 0, 0, 0, 2, 3, 4, 5, 6, 7]
    assert lammpstrj._roles(h["columns"], "xs", ("x",), False).tolist() == [1, 0, 0, 0, 0, 2, 3, 4]


def test_choose_style_and_unwrap_checks():
    cols = ["id", "type", "xs", "ys", "zs", "xu", "yu", "zu"]
    assert lammpstrj._choose("f", cols, ("x",), None, False)[1] == "xu"
    assert lammpstrj._choose("f", cols, ("x",), "xs", False)[1] == "xs"
    with pytest.raises(ValueError, match="no x y z columns"):
        lammpstrj._choose("f", cols, ("x",), "x", False)
    with pytest.raises(ValueError, match="unwrap=True needs the ix iy iz"):
        lammpstrj._choose("f", cols, ("x",), "xs", True)
    assert lammpstrj._choose("f", cols, ("x",), "xu", True)[2] is False  # a no-op for unwrapped styles
    with pytest.raises(ValueError, match="no vx vy vz"):
        lammpstrj._choose("f", cols, ("x", "v"), None, False)


def test_general_triclinic_box_raises(tmp_path):
    raw = (b"ITEM: TIMESTEP\n0\nITEM: NUMBER OF ATOMS\n1\nITEM: BOX BOUNDS abc origin pp pp pp\n1 0 0 0\n0 1 0 0\n"
           b"0 0 1 0\nITEM: ATOMS id type x y z\n1 1 0 0 0\n")
    fn = _write(tmp_path, raw)
    with open(fn, "rb") as fh, pytest.raises(ValueError, match="general triclinic"):
        lammpstrj._frame0(fn, fh.fileno(), len(raw.rstrip()))


@pytest.mark.parametrize("tilt", [(0.0, 0.0, 0.0), (1.5, -2.25, 0.75), (-3.0, -1.0, -0.5), (2.0, 3.0, -4.0)])
def test_box_bounds_both_directions(tilt):
    xy, xz, yz = tilt
    box = np.float32([[21.5, 0, 0], [xy, 30.25, 0], [xz, yz, 17.0]])
    origin = np.array([-3.5, 2.0, 0.25])
    b = lammpstrj._bound_rows(box, origin)
    assert np.array_equal(b, lf.bound_lines(box, origin))
    xlo, ylo, zlo, lx, ly, lz, pxy, pxz, pyz = lammpstrj._params(b[None])[0]
    assert (xlo, ylo, zlo) == tuple(origin)
    assert np.float32(lx) == box[0, 0] and np.float32(ly) == box[1, 1] and np.float32(lz) == box[2, 2]
    assert (pxy, pxz, pyz) == (float(box[1, 0]), float(box[2, 0]), float(box[2, 1]))
    assert lammpstrj._params(b[None])[0].tolist() == list(lf.lohi(b))


def test_oracle_round_trip():
    rng = np.random.default_rng(3)
    N, F = 7, 3
    x = [rng.normal(0, 20, (N, 3)).astype(np.float32) for _ in range(F)]
    v = [rng.normal(0, 1, (N, 3)).astype(np.float32) for _ in range(F)]
    box = [np.float32([[30, 0, 0], [1.5 * f, 31, 0], [0, -0.5, 29]]) for f in range(F)]
    raw = lf.write(x, box, step=[5, 10, 15], time=[0.0, 0.5, 1.0], ids=range(11, 11 + N), types=[2] * N,
                   velocities=v, units="metal")
    got = lf.read(raw)
    assert np.array_equal(got["coords"].view(np.uint32), np.stack(x).view(np.uint32))
    assert np.array_equal(got["v"].view(np.uint32), np.stack(v).view(np.uint32))
    assert np.array_equal(got["box"], np.stack(box)) and got["step"].tolist() == [5, 10, 15]
    assert got["units"] == "metal" and got["ids"].tolist() == list(range(11, 11 + N))


def _ok_args():
    x = np.zeros((2, 3, 2), np.float32)
    box = np.zeros((3, 3, 2), np.float32)
    box[0, 0] = box[1, 1] = box[2, 2] = 10
    return x, box


@pytest.mark.parametrize("kw,msg", [
    (dict(coords=np.zeros((2, 2, 2), np.float32)), "coords must be"),
    (dict(box=None), "box is required"),
    (dict(box=np.zeros((3, 3), np.float32)), "box must be"),
    (dict(box="upper"), "restricted-triclinic"),
    (dict(box="nan"), "not finite"),
    (dict(step=[1]), "step must hold"),
    (dict(step=[1.5, 2]), "not an int64"),
    (dict(time=[0.0, np.inf]), "time at frame 1"),
    (dict(ids=[1]), "ids must be"),
    (dict(types=[1.0, 2.0]), "types must be"),
    (dict(velocities=np.zeros((2, 3, 3), np.float32)), "velocities must be"),
    (dict(origin=np.zeros(2)), "origin must be"),
    (dict(units="two words"), "units must be"),
    (dict(chunk_bytes=0), "chunk_bytes"),
])
def test_writer_checks_before_file(tmp_path, kw, msg):
    x, box = _ok_args()
    if isinstance(kw.get("box"), str):
        box = box.copy()
        if kw["box"] == "upper":
            box[0, 1, 1] = 1.0
        else:
            box[2, 2, 1] = np.nan
        kw = dict(kw, box=box)
    args = dict(coords=x, box=box)
    args.update(kw)
    p = tmp_path / "w.lammpstrj"
    with pytest.raises(ValueError, match=msg):
        lammpstrj.write_lammpstrj(str(p), **args)
    assert not p.exists()


def test_symbols_present():
    from moleculekit_b200 import _lib
    lib = _lib.load()
    for s in ("mkb_lammpstrj_index", "mkb_lammpstrj_head", "mkb_lammpstrj_decode", "mkb_lammpstrj_encode"):
        assert hasattr(lib, s) and s in _lib.EXPORTS


_G9_SRC = r"""
#include <cstdio>
#include <cstring>
#include "lammpstrj_g9.cuh"
int main() {
    unsigned v;
    unsigned char d[32];
    while (scanf("%x", &v) == 1) {
        float f;
        memcpy(&f, &v, 4);
        int n = mkb::g9_format(f, d);
        fwrite(d, 1, n, stdout);
        putchar('\n');
    }
    return 0;
}
"""


def _edge_patterns() -> np.ndarray:
    """binade edges, the 9.99999995e k rounding boundaries, exact decimal ties, subnormals, zeros, the largest float,
    NaN and infinities, and each pattern's neighbours"""
    getcontext().prec = 60
    pats = [0, 1, 2, 0x7fffff, 0x800000, 0x7f7fffff, 0x7f800000, 0x7fc00000, 0x7f800001, 0x3f800000]
    pats += [e << 23 for e in range(1, 255)] + [(e << 23) | 0x7fffff for e in range(0, 255)]
    for k in range(-46, 40):
        for s in ("9.99999995e%d", "1e%d", "5e%d", "1.000000005e%d", "2.5e%d"):
            pats.append(int(np.float32(float(s % k)).view(np.uint32)) if -46 <= k < 38 else 0)
    # exact decimal ties: m 2^-k whose exact decimal has ten significant digits, the last a 5
    for m in range(1, 1 << 13, 2):
        for k in range(1, 60):
            d = Decimal(m) / (Decimal(2) ** k)
            if len(d.normalize().as_tuple().digits) == 10:
                pats.append(int(np.float32(m * 2.0 ** -k).view(np.uint32)))
    p = np.array(pats, np.int64) & 0x7fffffff
    p = np.concatenate([p, p + 1, np.maximum(p - 1, 0)]) & 0x7fffffff
    p = np.concatenate([p, p | 0x80000000])
    return np.unique(p).astype(np.uint32)


def _g9_exe(tmp_path):
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    src = tmp_path / "g9.cpp"
    src.write_text(_G9_SRC)
    exe = tmp_path / "g9"
    subprocess.run([cxx, "-O2", "-std=c++17", f"-I{os.path.join(ROOT, 'moleculekit_b200', 'csrc')}", str(src), "-o",
                    str(exe)], check=True)
    return exe


def test_g9_matches_python(tmp_path):
    exe = _g9_exe(tmp_path)
    rng = np.random.default_rng(32)
    pats = np.concatenate([_edge_patterns(), rng.integers(0, 2**32, 3_000_000, dtype=np.uint64).astype(np.uint32)])
    out = subprocess.run([str(exe)], input="\n".join("%x" % u for u in pats.tolist()) + "\n", capture_output=True,
                         text=True, check=True).stdout.split("\n")[:-1]
    assert len(out) == len(pats)
    vals = pats.view(np.float32).tolist()
    bad = [(hex(int(u)), o) for u, v, o in zip(pats.tolist(), vals, out) if o != "%.9g" % v]
    assert not bad, bad[:10]
