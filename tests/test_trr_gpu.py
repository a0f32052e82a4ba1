"""K24 on the device: GROMACS TRR x, v and f decoded into (natoms, 3, F) and encoded back, bit for bit against
oracle/trr_format.py, an independent restatement of the format, and float64 blocks rounded exactly as numpy's
astype(np.float32) rounds them on x86-64."""
import ctypes
import os
import warnings

import numpy as np
import pytest

from oracle import trr_format as tf
from test_trr_cpu import _box, _xyz, mixed

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOT_REQUANTISABLE = {"wide_x", "wide_xyz"}  # tests/test_xtc_encode_cpu.py::test_which_golden_files_requantise


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _f32(a):
    """the float32 numpy gives for an array of the file's precision (float64 rounded on the host, warnings quiet)"""
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        return np.asarray(a).astype(np.float32)


def _special32(x):
    """x with -0.0, quiet NaNs with a payload, negative signalling NaNs and the smallest subnormal sprinkled in"""
    bits = x.view(np.uint32)
    bits.flat[::5] = 0x80000000
    bits.flat[1::7] = 0x7FC12345
    bits.flat[2::11] = 0xFF800001
    bits.flat[3::13] = 0x00000001
    return x


# float64 bit patterns and what numpy's astype(np.float32) gives for them on x86-64
F64_TABLE = [
    (0x47EFFFFFF0000000, None),  # halfway between FLT_MAX and 2^128: ties to even, to +inf
    (0x47EFFFFFE0000000, None),  # FLT_MAX exactly
    (0x47EFFFFFEFFFFFFF, None),  # just below the tie: FLT_MAX
    (0x7FEFFFFFFFFFFFFF, None),  # DBL_MAX: +inf
    (0x36A0000000000000, None),  # 2^-149, the smallest float32 subnormal
    (0x3690000000000000, None),  # 2^-150: the tie with 0 goes to even, +0
    (0x36A8000000000000, None),  # 3 * 2^-150: the tie between 2^-149 and 2^-148 goes to even, 2^-148
    (0xB6A8000000000000, None),  # -3 * 2^-150
    (0x3690000000000001, None),  # just above 2^-150: 2^-149
    (0x0000000000000001, None),  # the smallest double subnormal: +0
    (0x800FFFFFFFFFFFFF, None),  # the largest negative double subnormal: -0
    (0x380FFFFFFFFFFFFF, None),  # just below FLT_MIN: rounds up to FLT_MIN
    (0x3810000000000000, None),  # FLT_MIN
    (0x3FF0000010000000, None),  # 1 + 2^-24: a tie, to even (1)
    (0x3FF0000030000000, None),  # 1 + 3 * 2^-24: a tie, to even (1 + 2^-22)
    (0x8000000000000000, None),  # -0.0
    (0x7FF0000000000000, None),  # +inf
    (0xFFF0000000000000, None),  # -inf
    (0xFFF4000020000000, 0xFFE00001),  # signalling NaN, payload in the high and low mantissa bits
    (0x7FF0000000000001, 0x7FC00000),  # signalling NaN, payload in the lowest bit only: lost
    (0x7FF8000000000000, 0x7FC00000),  # the default quiet NaN
    (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFF),  # every mantissa bit set
    (0x7FF80000E0000000, 0x7FC00007),  # quiet NaN, low-word payload bits 31..29
    (0x7FF00000_1FFFFFFF, 0x7FC00000),  # signalling NaN whose payload lies below bit 29 only
]


def _special64(x):
    bits = x.view(np.uint64)
    pats = np.array([p for p, _ in F64_TABLE], np.uint64)
    bits.flat[::3] = pats[np.arange(bits.size)[::3] % len(pats)]
    return x


def _file(tmp_path, raw, name="t.trr"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return str(fn)


def _want(raw, key, records):
    """the oracle's (N, 3, len(records)) float32 of block ``key``"""
    o = tf.read(raw)
    fr = o["frames"]
    if not len(records):
        return np.zeros((o["natoms"], 3, 0), np.float32)
    return np.ascontiguousarray(np.stack([_f32(fr[r][key]) for r in records], axis=2))


def test_float64_table_against_numpy(tmp_path):
    from moleculekit_b200 import trr as pt

    pats = np.array([p for p, _ in F64_TABLE], np.uint64)
    N = len(pats)
    x = pats.view(np.float64).reshape(N, 1).repeat(3, axis=1)
    raw = tf.write([tf.frame(N, box=np.eye(3), x=x)], double=True)
    got = pt.read_trr(_file(tmp_path, raw))[0][:, :, 0].view(np.uint32)
    want = _f32(x).view(np.uint32)
    assert np.array_equal(got, want), [(hex(p), hex(g), hex(w)) for p, g, w in zip(pats, got[:, 0], want[:, 0])
                                       if g != w]
    for (p, expect), w in zip(F64_TABLE, want[:, 0]):
        if expect is not None:  # numpy's own answer on x86-64, stated by hand
            assert w == expect, hex(p)


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("N", [1, 31, 33, 97])
@pytest.mark.parametrize("F", [1, 31, 33, 97])
def test_decoding_is_bit_identical_off_the_tile(tmp_path, double, N, F):
    from moleculekit_b200 import trr as pt

    rng = np.random.default_rng(N * 1000 + F)
    dt = np.float64 if double else np.float32
    special = _special64 if double else _special32
    fr = []
    for k in range(F):
        x = special(rng.normal(0, 5, size=(N, 3)).astype(dt))
        v = special(rng.normal(0, 1, size=(N, 3)).astype(dt)) if k % 2 == 0 else None
        fr.append(tf.frame(N, step=k, time=0.5 * k, box=_box(k), x=x, v=v, f=x[::-1].copy() if k % 3 == 0 else None))
    raw = tf.write(fr, double=double)
    fn = _file(tmp_path, raw)
    coords, box, time, step = pt.read_trr(fn)
    assert coords.shape == (N, 3, F) and np.array_equal(_bits(coords), _bits(_want(raw, "x", range(F))))
    assert np.array_equal(box, np.stack([_f32(f["box"]) for f in tf.read(raw)["frames"]], axis=2))
    assert np.array_equal(step, np.arange(F)) and np.array_equal(time, np.float32(0.5) * np.arange(F, dtype=np.float32))
    out, _, info = pt.read_trr_device(fn, fields=("v", "x", "f"))
    rec = [k for k in range(F) if k % 6 == 0]
    assert info["records"].tolist() == rec and info["double"] == double
    for key in ("x", "v", "f"):
        assert np.array_equal(_bits(out[key].cpu().numpy()), _bits(_want(raw, key, rec))), key


def test_frame_lists_repeats_and_errors(tmp_path):
    from moleculekit_b200 import trr as pt

    N = 40
    for double in (False, True):
        fr = mixed(N, seed=5)
        raw = tf.write(fr, double=double)
        fn = _file(tmp_path, raw)
        idx = pt.index_trr(raw)
        xs = np.flatnonzero(idx["has_x"])
        rng = np.random.default_rng(3)
        for sel in (rng.choice(xs, size=20), np.concatenate([xs[::-1], xs[:2]]), xs[-1:]):
            out, box, info = pt.read_trr_device(fn, frames=sel)
            assert np.array_equal(_bits(out["x"].cpu().numpy()), _bits(_want(raw, "x", sel)))
            assert np.array_equal(box, idx["box"][:, :, sel]) and np.array_equal(info["records"], sel)
            assert np.array_equal(info["time"], idx["time"][sel]) and np.array_equal(info["lambda"], idx["lambda"][sel])
            assert np.array_equal(info["step"], idx["step"][sel])
        # read_trr_frames numbers the frames as read_trr returns them: the records with x
        c, b, t, s = pt.read_trr_frames(fn, [3, 0, 3])
        assert np.array_equal(_bits(c), _bits(_want(raw, "x", xs[[3, 0, 3]]))) and np.array_equal(s, idx["step"][xs[[3, 0, 3]]])
        with pytest.raises(IndexError):
            pt.read_trr_device(fn, frames=[len(fr)])
        with pytest.raises(ValueError, match="record 7 has no x"):
            pt.read_trr_device(fn, frames=[0, 7])
        with pytest.raises(ValueError, match="record 2 has no v"):
            pt.read_trr_device(fn, frames=[1, 2], fields="v")


def test_velocities_and_forces_on_mixed_files(tmp_path):
    from moleculekit_b200 import trr as pt

    N = 70
    for double in (False, True):
        fr = mixed(N, seed=8)
        raw = tf.write(fr, double=double)
        fn = _file(tmp_path, raw)
        for fields in (("v",), ("f",), ("x", "v"), ("f", "v"), ("x", "v", "f")):
            out, _, info = pt.read_trr_device(fn, fields=fields, chunk_bytes=3 * 12 * N)
            rec = [r for r, a in enumerate(fr) if all(a[k] is not None for k in fields)]
            assert rec and info["records"].tolist() == rec and set(out) == set(fields)
            for key in fields:
                assert np.array_equal(_bits(out[key].cpu().numpy()), _bits(_want(raw, key, rec))), (fields, key)
        # scale multiplies x only, one float32 multiply
        out, _, _ = pt.read_trr_device(fn, fields=("x", "v"), scale=10)
        rec = [r for r, a in enumerate(fr) if a["x"] is not None and a["v"] is not None]
        assert np.array_equal(_bits(out["x"].cpu().numpy()), _bits(_want(raw, "x", rec) * np.float32(10)))
        assert np.array_equal(_bits(out["v"].cpu().numpy()), _bits(_want(raw, "v", rec)))


def test_large_trajectory_and_many_chunks(tmp_path):
    from moleculekit_b200 import trr as pt

    F, N = 2000, 5000
    rng = np.random.default_rng(5)
    x = rng.normal(0, 3, size=(F, N, 3)).astype(np.float32)
    v = rng.normal(0, 1, size=(F, N, 3)).astype(np.float32)
    raw = tf.write([tf.frame(N, step=k, time=k, box=_box(k % 7), x=x[k], v=v[k] if k % 2 else None)
                    for k in range(F)])
    fn = _file(tmp_path, raw)
    want = np.ascontiguousarray(x.transpose(1, 2, 0))
    one = pt.read_trr_device(fn)[0]["x"]
    assert np.array_equal(_bits(one.cpu().numpy()), _bits(want))
    slab = 12 * N
    many = pt.read_trr_device(fn, chunk_bytes=37 * slab)[0]["x"]  # 55 chunks
    assert np.array_equal(_bits(many.cpu().numpy()), _bits(want))
    sel = np.random.default_rng(9).integers(0, F, size=3001) | 1
    part, pbox, info = pt.read_trr_device(fn, frames=sel, fields=("v", "x"), chunk_bytes=100 * 2 * slab)
    assert np.array_equal(_bits(part["x"].cpu().numpy()), _bits(want[:, :, sel]))
    assert np.array_equal(_bits(part["v"].cpu().numpy()), _bits(np.ascontiguousarray(v.transpose(1, 2, 0))[:, :, sel]))
    assert np.array_equal(info["step"], sel)


@pytest.mark.parametrize("F,N", [(1, 1), (5, 33), (67, 100), (300, 2)])
def test_writer_matches_the_oracle(tmp_path, F, N):
    import torch
    from moleculekit_b200 import trr as pt

    rng = np.random.default_rng(F + N)
    x = _special32(rng.normal(0, 3, size=(N, 3, F)).astype(np.float32))
    v = _special32(rng.normal(0, 1, size=(N, 3, F)).astype(np.float32))
    f = rng.normal(0, 100, size=(N, 3, F)).astype(np.float32)
    box = rng.uniform(1, 9, size=(3, 3, F)).astype(np.float32)
    time = rng.uniform(0, 1e4, size=F).astype(np.float32)
    step = rng.integers(-5, 10**6, size=F)
    lambd = rng.uniform(0, 1, size=F).astype(np.float32)
    for vel, frc, lam in ((None, None, None), (v, None, lambd), (None, f, None), (v, f, lambd)):
        want = tf.write([tf.frame(N, step=int(step[k]), time=float(time[k]), lambd=0.0 if lam is None else float(lam[k]),
                                  box=box[:, :, k], x=x[:, :, k], v=None if vel is None else vel[:, :, k],
                                  f=None if frc is None else frc[:, :, k]) for k in range(F)])
        kw = dict(lambd=lam, velocities=vel, forces=frc)
        assert pt.trr_bytes(x, box, time, step, **kw) == want
        R = len(want) // F
        # device tensors with a frame stride (the middle F frames of wider trajectories) and small chunks
        wide = {}
        for name, a in (("x", x), ("v", vel), ("f", frc)):
            if a is not None:
                t = torch.zeros((N, 3, F + 7), dtype=torch.float32, device="cuda")
                t[:, :, 3:3 + F] = torch.from_numpy(a).cuda()
                wide[name] = t[:, :, 3:3 + F]
        dkw = dict(lambd=lam, velocities=wide.get("v"), forces=frc)  # forces stay on the host: uploaded
        assert pt.trr_bytes(wide["x"], box, time, step, chunk_bytes=2 * R + 1, **dkw) == want
        fn = str(tmp_path / "w.trr")
        pt.write_trr(fn, wide["x"], box, time, step, chunk_bytes=R, **dkw)
        assert open(fn, "rb").read() == want
        fields = ("x",) + (("v",) if vel is not None else ()) + (("f",) if frc is not None else ())
        back, bbox, info = pt.read_trr_device(fn, fields=fields, chunk_bytes=5000)
        src = dict(x=x, v=vel, f=frc)
        for name in fields:
            assert np.array_equal(_bits(back[name].cpu().numpy()), _bits(src[name])), name
        assert np.array_equal(bbox, box) and np.array_equal(info["step"], step.astype(np.int32))
        dev = pt.encode_trr_device(wide["x"], box, time, step, **dkw)
        assert bytes(dev.cpu().numpy()) == want


def test_writer_scale_multiplies_x_only():
    from moleculekit_b200 import trr as pt

    N, F = 9, 4
    rng = np.random.default_rng(1)
    x = rng.normal(0, 30, size=(N, 3, F)).astype(np.float32)
    v = rng.normal(0, 1, size=(N, 3, F)).astype(np.float32)
    box, time, step = np.ones((3, 3, F), np.float32), np.zeros(F), np.arange(F)
    assert pt.trr_bytes(x, box, time, step, velocities=v, scale=0.1) == \
        pt.trr_bytes(x * np.float32(0.1), box, time, step, velocities=v)


def test_xtc_goldens_through_trr(tmp_path):
    import torch
    from moleculekit_b200 import trr as pt
    from moleculekit_b200 import xtc as px

    gold = os.path.join(ROOT, "tests", "golden", "xtc")
    names = sorted(f[:-4] for f in os.listdir(gold) if f.endswith(".xtc"))
    assert len(names) == 9
    for name in names:
        fn = os.path.join(gold, name + ".xtc")
        coords, box, time, step = px.read_xtc_device(fn)
        out = str(tmp_path / (name + ".trr"))
        pt.write_trr(out, coords, box, time, step)
        back, bbox, btime, bstep = pt.read_trr(out)
        assert np.array_equal(_bits(back), _bits(coords.cpu().numpy())), name
        assert np.array_equal(bbox, np.asarray(box, np.float32)) and np.array_equal(btime, np.asarray(time, np.float32))
        assert np.array_equal(bstep, np.asarray(step).astype(np.int64).astype(np.int32))
        if name not in NOT_REQUANTISABLE:  # the trajectory comes back from TRR as the same XTC file
            assert px.xtc_bytes(back, bbox, btime, bstep) == open(fn, "rb").read(), name
        dev, _, _ = pt.read_trr_device(out)
        assert torch.equal(dev["x"].view(torch.int32), coords.view(torch.int32))


def _at(t, offset):
    """a pointer ``offset`` bytes into a tensor"""
    return ctypes.c_void_p(t.data_ptr() + offset)


def test_abi_argument_checks():
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import trr as pt

    dev = torch.device("cuda", 0)
    x = torch.zeros((10, 3, 4), device=dev)
    head = torch.zeros(4 * 120, dtype=torch.uint8, device=dev)
    R = 120 + 3 * 120
    out = torch.empty(4 * R, dtype=torch.uint8, device=dev)
    with pytest.raises(_lib.MkbCapacity, match=str(4 * R)):
        _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 4, 4, 10, _lib.ptr(head), 120,
                  _lib.ptr(out), 4 * R - 4)
    with pytest.raises(_lib.MkbCapacity, match=str(4 * (120 + 240))):
        _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), None, _lib.ptr(x), 4, 4, 10, _lib.ptr(head), 120,
                  _lib.ptr(out), 4 * (120 + 240) - 1)
    with pytest.raises(_lib.MkbError, match="multiple of 4"):
        _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), None, None, 4, 4, 10, _lib.ptr(head), 118, _lib.ptr(out), 4 * R)
    with pytest.raises(_lib.MkbError, match="4-byte aligned"):
        _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), None, None, 4, 4, 10, _lib.ptr(head), 120, _at(out, 2), 4 * R)
    with pytest.raises(_lib.MkbError, match="frame stride"):
        _lib.call(dev, "mkb_trr_encode", _lib.ptr(x), None, None, 3, 4, 10, _lib.ptr(head), 120, _lib.ptr(out), 4 * R)
    buf = torch.zeros(1024, dtype=torch.uint8, device=dev)
    for vb, offsets in ((4, [0, 1000]), (4, [2]), (4, [-4]), (4, [1024 - 120 + 4]), (8, [4]), (8, [1024 - 240 + 8]),
                        (8, [0, 12])):
        with pytest.raises(_lib.MkbError, match="offset"):
            pt.decode_trr_device(buf, np.array(offsets), 10, vb)
    for vb in (0, 2, 16):
        with pytest.raises(_lib.MkbError, match="value_bytes"):
            pt.decode_trr_device(buf, np.array([0]), 10, vb)
    with pytest.raises(_lib.MkbError, match="8-byte aligned"):
        _lib.call(dev, "mkb_trr_decode", _at(buf, 4), 1000, np.zeros(1, np.int64).ctypes.data_as(ctypes.c_void_p),
                  1, 10, 8, _lib.ptr(x), 4)
    ok = pt.decode_trr_device(buf, np.array([1024 - 240, 0]), 10, 8)
    assert ok.shape == (10, 3, 2) and not ok.any()
    ok = pt.decode_trr_device(buf, np.array([1024 - 120, 4]), 10, 4)
    assert ok.shape == (10, 3, 2) and not ok.any()
