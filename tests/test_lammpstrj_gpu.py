"""K32 (LAMMPS dump trajectories) on the GPU: every read bit for bit against oracle/lammpstrj_format.py's split() /
float() reader, the writer byte for byte against its % writer, the round trip, and every error."""
import logging
import os
import sys
import zlib

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from moleculekit_b200 import lammpstrj  # noqa: E402
from oracle import lammpstrj_format as lf  # noqa: E402

pytestmark = pytest.mark.gpu

COLS = {"x": ["x", "y", "z"], "xs": ["xs", "ys", "zs"], "xu": ["xu", "yu", "zu"], "xsu": ["xsu", "ysu", "zsu"]}


def _file(tmp_path, raw, name="t.lammpstrj"):
    p = tmp_path / name
    p.write_bytes(raw)
    return str(p)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _check(fn, raw, frames=None, fields=("x",), style=None, unwrap=False, **kw):
    out, box, info = lammpstrj.read_lammpstrj_device(fn, frames=frames, fields=fields, style=style, unwrap=unwrap,
                                                     **kw)
    want = lf.read(raw, style, unwrap)
    sel = np.arange(len(want["step"])) if frames is None else np.asarray(frames)
    for key, wk in (("x", "coords"), ("v", "v"), ("f", "f")):
        if key in fields:
            assert np.array_equal(_bits(out[key].cpu().numpy()), _bits(want[wk][sel].transpose(1, 2, 0))), key
    assert np.array_equal(_bits(box), _bits(want["box"][sel].transpose(1, 2, 0)))
    assert np.array_equal(info["step"], want["step"][sel])
    assert np.array_equal(info["time"], want["time"][sel], equal_nan=True)
    assert np.array_equal(info["bounds"], want["bounds"][sel])
    assert np.array_equal(info["ids"], want["ids"])
    return out, box, info


@pytest.mark.parametrize("style", ["x", "xs", "xu", "xsu"])
@pytest.mark.parametrize("images", [False, True])
@pytest.mark.parametrize("triclinic", [False, True])
def test_styles_boxes_and_images(tmp_path, style, images, triclinic):
    rng = np.random.default_rng(zlib.crc32(f"{style}{images}{triclinic}".encode()))
    cols = ["id", "type", "q"] + COLS[style] + (["ix", "iy", "iz"] if images else []) + ["c_pe"]
    raw = lf.make_file(rng, 300, 7, cols, triclinic=triclinic, shuffle=True)
    fn = _file(tmp_path, raw)
    _check(fn, raw, style=style)
    if images or style in ("xu", "xsu"):
        _check(fn, raw, style=style, unwrap=True)
    else:
        with pytest.raises(ValueError, match="unwrap=True needs the ix iy iz"):
            lammpstrj.read_lammpstrj_device(fn, style=style, unwrap=True)


@pytest.mark.parametrize("ids", ["dense", "sparse"])
@pytest.mark.parametrize("shuffle", [False, True])
def test_ids_order(tmp_path, ids, shuffle):
    rng = np.random.default_rng(5)
    N = 257
    idv = None if ids == "dense" else rng.choice(10**12, N, replace=False) + 5
    raw = lf.make_file(rng, N, 9, ["id", "type", "x", "y", "z"], shuffle=shuffle, ids=idv)
    _, _, info = _check(_file(tmp_path, raw), raw)
    assert np.array_equal(info["type"], lf.read(raw)["type"])


def test_no_id_column_is_line_order(tmp_path):
    rng = np.random.default_rng(6)
    raw = lf.make_file(rng, 40, 3, ["type", "x", "y", "z"])
    _check(_file(tmp_path, raw), raw)


@pytest.mark.parametrize("crlf", [False, True])
def test_time_units_crlf_trailing_spaces(tmp_path, crlf):
    rng = np.random.default_rng(7)
    raw = lf.make_file(rng, 50, 6, ["id", "type", "mol", "element", "x", "y", "z"], triclinic=True, shuffle=True,
                       units="real", time=True, crlf=crlf, trailing=True)
    fn = _file(tmp_path, raw + b"\n  \n\t\n")
    _, _, info = _check(fn, raw)
    assert info["units"] == "real" and info["host_lines"] == 0
    idx = lammpstrj.index_lammpstrj(fn)
    assert idx["element"][:4] == ["C", "N", "O", "H"] and len(idx["mol"]) == 50


def test_exponent_nan_inf_and_host_tokens(tmp_path):
    rng = np.random.default_rng(8)
    raw = lf.make_file(rng, 64, 4, ["id", "type", "x", "y", "z", "vx", "vy", "vz", "fx", "fy", "fz"], fmt="%.6e")
    lines = raw.split(b"\n")
    lines[9] = b"1 1 nan -inf +1.5E+3 1 2 3 4 5 6"
    lines[10] = b"2 1 Infinity -NaN 0.000000000000000000000000000000000001 1 2 3 4 5 6"
    bad = [b"3 1 1_0.5 2 3 1 2 3 4 5 6", b"4 1 0.123456789012345678901234567 2 3 1 2 3 4 5 6"]
    lines[11], lines[12] = bad
    raw = b"\n".join(lines)
    out, _, info = _check(_file(tmp_path, raw), raw, fields=("x", "v", "f"))
    assert info["host_lines"] == 64  # the frame holding the two host lines is re-read


def test_frame_lists_and_chunks(tmp_path):
    rng = np.random.default_rng(9)
    raw = lf.make_file(rng, 500, 12, ["id", "type", "xs", "ys", "zs"], triclinic=True, shuffle=True, time=True)
    fn = _file(tmp_path, raw)
    frames = [11, 0, 3, 3, 7, 0, 11, 5]
    _check(fn, raw, frames=frames)
    _check(fn, raw, frames=frames, chunk_bytes=4096)  # a frame larger than a chunk
    _check(fn, raw, chunk_bytes=50000)
    idx = lammpstrj.index_lammpstrj(fn, chunk_bytes=3000)
    _check(fn, raw, frames=frames, index=idx)
    x, box, t, s = lammpstrj.read_lammpstrj_frames(fn, frames, index=idx)
    assert x.shape == (500, 3, len(frames)) and t.dtype == np.float64 and s.dtype == np.int64
    with pytest.raises(IndexError):
        lammpstrj.read_lammpstrj_frames(fn, [12])


def test_scale_multiplies_positions(tmp_path):
    rng = np.random.default_rng(10)
    raw = lf.make_file(rng, 20, 2, ["id", "type", "x", "y", "z"])
    fn = _file(tmp_path, raw)
    x, _, _, _ = lammpstrj.read_lammpstrj(fn, scale=0.1)
    assert np.array_equal(_bits(x), _bits(lf.read(raw)["coords"].transpose(1, 2, 0) * np.float32(0.1)))


def test_70000_one_atom_frames(tmp_path):
    F = 70000
    rng = np.random.default_rng(11)
    x = rng.normal(0, 5, (1, 3, F)).astype(np.float32)
    box = np.zeros((3, 3, F), np.float32)
    box[0, 0], box[1, 1], box[2, 2] = 10, 11, 12
    box[1, 0] = rng.uniform(-1, 1, F).astype(np.float32)
    raw = lammpstrj.lammpstrj_bytes(x, box)
    assert raw == lf.write(list(x.transpose(2, 0, 1)), list(box.transpose(2, 0, 1)))
    fn = _file(tmp_path, raw)
    got, gbox, _, step = lammpstrj.read_lammpstrj(fn)
    assert np.array_equal(_bits(got), _bits(x)) and np.array_equal(_bits(gbox), _bits(box))
    assert np.array_equal(step, np.arange(F))


def _values(rng, N, F):
    x = rng.normal(0, 30, (N, 3, F)).astype(np.float32)
    flat = x.reshape(-1)
    special = np.float32([np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -3.4028235e38, 1e-8, 123456789.0, 5e-5])
    flat[:len(special)] = special
    return x


@pytest.mark.parametrize("triclinic", [False, True])
@pytest.mark.parametrize("vel", [False, True])
def test_writer_bytes_and_round_trip(tmp_path, triclinic, vel):
    rng = np.random.default_rng(12)
    N, F = 333, 5
    x = _values(rng, N, F)
    v = rng.normal(0, 1, (N, 3, F)).astype(np.float32) if vel else None
    box = np.zeros((3, 3, F), np.float32)
    box[0, 0], box[1, 1], box[2, 2] = 40, 41, 42
    if triclinic:
        box[1, 0], box[2, 0], box[2, 1] = 2.5, -1.25, 0.5
    origin = rng.uniform(-5, 5, (F, 3))
    ids = rng.choice(10**9, N, replace=False) + 1
    types = rng.integers(1, 5, N)
    step, time = np.arange(F) * 1000 + 7, np.arange(F) * 0.5
    kw = dict(step=step, time=time, ids=ids, types=types, velocities=v, origin=origin, units="metal")
    raw = lammpstrj.lammpstrj_bytes(x, box, chunk_bytes=20000, **kw)
    want = lf.write(list(x.transpose(2, 0, 1)), list(box.transpose(2, 0, 1)), step=step, time=time, ids=ids,
                    types=types, velocities=None if v is None else list(v.transpose(2, 0, 1)), origin=origin,
                    units="metal")
    assert raw == want
    fn = str(tmp_path / "w.lammpstrj")
    lammpstrj.write_lammpstrj(fn, torch.from_numpy(x).cuda(), box, **dict(kw, velocities=None if v is None else
                                                                          torch.from_numpy(v).cuda()))
    assert open(fn, "rb").read() == want
    dev = lammpstrj.encode_lammpstrj_device(torch.from_numpy(x).cuda(), box, **dict(
        kw, velocities=None if v is None else torch.from_numpy(v).cuda()))
    assert bytes(dev.cpu().numpy()) == want
    out, gbox, info = lammpstrj.read_lammpstrj_device(fn, fields=("x", "v") if vel else ("x",))
    order = np.argsort(ids)
    assert np.array_equal(_bits(out["x"].cpu().numpy()), _bits(x[order]))
    if vel:
        assert np.array_equal(_bits(out["v"].cpu().numpy()), _bits(v[order]))
    assert np.array_equal(_bits(gbox), _bits(box))
    assert np.array_equal(info["step"], step) and np.array_equal(info["time"], time)


def _lines(rng, **kw):
    return lf.make_file(rng, 30, 4, ["id", "type", "x", "y", "z"], **kw).split(b"\n")


def _raises(tmp_path, lines, match):
    fn = _file(tmp_path, b"\n".join(lines))
    with pytest.raises(ValueError, match=match):
        lammpstrj.read_lammpstrj(fn)


def test_id_errors(tmp_path):
    rng = np.random.default_rng(13)
    P = 9 + 30
    lines = _lines(rng)
    lines[2 * P + 9] = b"7 " + lines[2 * P + 9].split(b" ", 1)[1]  # frame 2: a second id 7 (and id 1 goes missing)
    _raises(tmp_path, lines, f"frame 2, line {2 * P + 16}, column 1: the id 7 appears twice")
    lines = _lines(rng)
    lines[P + 9 + 4] = b"99 " + lines[P + 9 + 4].split(b" ", 1)[1]
    _raises(tmp_path, lines, f"frame 1, line {P + 9 + 5}, column 1: the id 99 is not an id of frame 0")


def test_structure_errors(tmp_path, caplog):
    rng = np.random.default_rng(14)
    P = 9 + 30
    lines = _lines(rng)
    lines[2 * P + 3] = b"31"
    _raises(tmp_path, lines, f"frame 2, line {2 * P + 4}, column 1: the atom count is 31, frame 0 has 30 .*dynamic")
    lines = _lines(rng)
    lines[P + 8] = b"ITEM: ATOMS id type x y zz"
    _raises(tmp_path, lines, f"frame 1, line {P + 9}, column 1: the header line")
    lines = _lines(rng)
    lines[P], lines[P + 1], lines[P + 2], lines[P + 3] = lines[P + 2], lines[P + 3], lines[P], lines[P + 1]
    _raises(tmp_path, lines, "frame 1, .*the items are")
    lines = _lines(rng)
    lines[3 * P + 12] = b"13 1 0.5 abc 2"
    _raises(tmp_path, lines, f"frame 3, line {3 * P + 13}, column 10: the y field 'abc' is not a number")
    lines = _lines(rng)
    lines[P + 20] = lines[P + 20] + b"\r 1"
    _raises(tmp_path, lines, "lone CR")
    lines = _lines(rng)
    fn = _file(tmp_path, b"\n".join(lines[:3 * P + 20]))
    with caplog.at_level(logging.WARNING):
        x, _, _, _ = lammpstrj.read_lammpstrj(fn)
    assert x.shape[2] == 3 and "frame 3" in caplog.text and "dropped" in caplog.text
    raw = (b"ITEM: TIMESTEP\n0\nITEM: NUMBER OF ATOMS\n1\nITEM: BOX BOUNDS abc origin pp pp pp\n1 0 0 0\n0 1 0 0\n"
           b"0 0 1 0\nITEM: ATOMS id type x y z\n1 1 0 0 0\n")
    with pytest.raises(ValueError, match="general triclinic"):
        lammpstrj.read_lammpstrj(_file(tmp_path, raw))
