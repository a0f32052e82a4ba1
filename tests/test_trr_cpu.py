"""The host side of GROMACS TRR reading and writing (moleculekit_b200/trr.py; K24 moves x, v and f on the device):
the independent oracle's round trip and a frame written out byte by byte, index_trr against the oracle on mixed files,
the truncated-record warning, every rejection, the argument checks that run before any device work, and the C-ABI
symbols."""
import logging
import os
import struct

import numpy as np
import pytest

from oracle import trr_format as tf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _xyz(N, seed):
    return np.random.default_rng(seed).normal(0, 3, size=(N, 3)).astype(np.float32)


def _box(seed):
    return np.diag(np.random.default_rng(seed).uniform(2, 9, size=3)) + np.triu(np.full((3, 3), 0.25), 1)


def mixed(N, seed=0):
    """x-only, v-only, x+v+f, box-less, vir / pres, lambda: the records a GROMACS run with different nstxout, nstvout
    and nstfout produces, and more"""
    fr = []
    for r in range(9):
        s = seed * 100 + r
        kw = {}
        if r % 3 != 1:
            kw["x"] = _xyz(N, s)
        if r % 2 == 1 or r in (4, 8):
            kw["v"] = _xyz(N, s + 50)
        if r in (4, 8):
            kw["f"] = _xyz(N, s + 70)
        if r != 5 and r != 1:
            kw["box"] = _box(s)
        if r == 4:
            kw["vir"], kw["pres"] = _box(s + 1), _box(s + 2)
        if r == 7:
            kw = dict(f=_xyz(N, s))
        fr.append(tf.frame(N, step=10 * r - 5, time=0.002 * 10 * r + 0.1, lambd=r / 8, **kw))
    return fr


def _as32(a):
    return None if a is None else np.asarray(a).astype(np.float32)


def test_oracle_round_trip():
    for double in (False, True):
        fr = mixed(7, seed=3)
        got = tf.read(tf.write(fr, double=double))
        assert got["double"] == double and got["natoms"] == 7 and got["trailing"] == 0 and len(got["frames"]) == 9
        for a, b in zip(fr, got["frames"]):
            assert (a["step"], a["lambd"]) == (b["step"], b["lambd"])
            assert b["time"] == (a["time"] if double else float(np.float32(a["time"])))
            for k in tf.BLOCKS:
                assert (a[k] is None) == (b[k] is None), k
                if a[k] is not None:
                    want = np.asarray(a[k], np.float64 if double else np.float32)
                    assert np.array_equal(b[k], want), k


def test_first_frame_of_a_one_atom_file_byte_by_byte():
    x = np.float32([[1.0, -2.0, 0.5]])
    box = np.diag([3.0, 4.0, 5.0])
    raw = tf.write([tf.frame(1, step=7, time=0.25, lambd=0.0, box=box, x=x)])
    want = bytes.fromhex(
        "000007c9"                              # magic 1993
        "0000000d"                              # 13 = strlen("GMX_trn_file") + 1
        "0000000c" "474d585f74726e5f66696c65"  # XDR string: length 12, "GMX_trn_file"
        "00000000" "00000000"                   # ir_size, e_size
        "00000024"                              # box_size 36
        "00000000" "00000000" "00000000" "00000000"  # vir, pres, top, sym
        "0000000c" "00000000" "00000000"        # x_size 12, v_size, f_size
        "00000001"                              # natoms
        "00000007" "00000000"                   # step, nre
        "3e800000" "00000000"                   # t = 0.25, lambda = 0
        "40400000" "00000000" "00000000"        # box row 0
        "00000000" "40800000" "00000000"        # box row 1
        "00000000" "00000000" "40a00000"        # box row 2
        "3f800000" "c0000000" "3f000000")       # x of atom 0
    assert raw == want and len(raw) == 84 + 36 + 12


def _check_index(idx, fr, double):
    w = 8 if double else 4
    assert idx["n_records"] == len(fr) and idx["double"] == double
    raw_frames = tf.read(tf.write(fr, double=double))["frames"]
    for r, (a, b) in enumerate(zip(fr, raw_frames)):
        assert idx["offset"][r] == b["offset"]
        assert idx["step"][r] == a["step"]
        assert idx["time"][r] == b["time"] and idx["lambda"][r] == b["lambd"]
        for k in ("box", "x", "v", "f"):
            assert idx[f"has_{k}"][r] == (a[k] is not None), (r, k)
        want_box = np.zeros((3, 3), np.float32) if a["box"] is None else b["box"].astype(np.float32)
        assert np.array_equal(idx["box"][:, :, r], want_box)
        # the block offsets: header, box, vir, pres, then x, v, f
        pos = b["offset"] + 76 + 2 * w + sum(9 * w for k in ("box", "vir", "pres") if a[k] is not None)
        for k in ("x", "v", "f"):
            if a[k] is None:
                assert idx[f"{k}_offset"][r] == -1
            else:
                assert idx[f"{k}_offset"][r] == pos
                pos += 3 * a["natoms"] * w


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("N", [1, 31, 33])
def test_index_matches_the_oracle(double, N):
    from moleculekit_b200 import trr as pt

    fr = mixed(N, seed=N)
    raw = tf.write(fr, double=double)
    idx = pt.index_trr(raw)
    assert idx["natoms"] == N
    _check_index(idx, fr, double)
    # a memory map of the file gives the same index
    assert pt.index_trr(np.frombuffer(raw, np.uint8))["offset"].tolist() == idx["offset"].tolist()
    # every record's block really is where the index says
    w = 8 if double else 4
    for r, a in enumerate(fr):
        for k in ("x", "v", "f"):
            if a[k] is not None:
                got = np.frombuffer(raw, ">f8" if double else ">f4", 3 * N, idx[f"{k}_offset"][r])
                assert np.array_equal(got.reshape(N, 3), np.asarray(a[k], np.float64 if double else np.float32))
    assert w in (4, 8)


def test_empty_buffer_has_no_records():
    from moleculekit_b200 import trr as pt

    idx = pt.index_trr(b"")
    assert idx["n_records"] == 0 and idx["natoms"] == 0 and idx["box"].shape == (3, 3, 0)


def test_truncated_last_record_is_dropped_with_a_warning(caplog):
    from moleculekit_b200 import trr as pt

    for double in (False, True):
        fr = mixed(5, seed=1)
        raw = tf.write(fr, double=double)
        full = pt.index_trr(raw)
        last = int(full["offset"][-1])
        for cut in (1, 3, 40, len(raw) - last - 80, len(raw) - last - 1):
            with caplog.at_level(logging.WARNING, logger="moleculekit_b200.trr"):
                caplog.clear()
                idx = pt.index_trr(raw[:len(raw) - cut])
                assert idx["n_records"] == len(fr) - 1 and caplog.records, cut
                assert np.array_equal(idx["offset"], full["offset"][:-1])
        with caplog.at_level(logging.WARNING, logger="moleculekit_b200.trr"):
            caplog.clear()
            assert pt.index_trr(raw[:last])["n_records"] == len(fr) - 1 and not caplog.records


def _patch(raw, at, value, fmt=">i"):
    return raw[:at] + struct.pack(fmt, value) + raw[at + struct.calcsize(fmt):]


SIZE_AT = {k: 24 + 4 * i for i, k in enumerate(("ir", "e", "box", "vir", "pres", "top", "sym", "x", "v", "f", "natoms"))}


def test_rejections():
    from moleculekit_b200 import trr as pt

    N = 4
    one = tf.write([tf.frame(N, box=_box(0), x=_xyz(N, 0), v=_xyz(N, 1))])
    two = one + one
    with pytest.raises(RuntimeError, match="Malformed TRR file: .*magic 1995"):
        pt.index_trr(_patch(one, 0, 1995))
    with pytest.raises(RuntimeError, match="Malformed TRR file: record 1 .*magic"):
        pt.index_trr(_patch(two, len(one), 0))
    for at, v in ((4, 12), (4, 14), (8, 13), (8, 0)):
        with pytest.raises(RuntimeError, match="Malformed TRR file: .*string lengths"):
            pt.index_trr(_patch(one, at, v))
    for field, v in (("box", 40), ("box", 72), ("x", 12 * N + 4), ("v", 24 * N), ("vir", 36 + 4), ("pres", 8),
                     ("f", 11), ("box", -36)):
        with pytest.raises(RuntimeError, match="Malformed TRR file"):
            pt.index_trr(_patch(one, SIZE_AT[field], v))
    with pytest.raises(RuntimeError, match="Malformed TRR file: .*v_size is 24"):
        pt.index_trr(_patch(one, SIZE_AT["v"], 24))
    with pytest.raises(RuntimeError, match="Malformed TRR file: .*all 0"):
        zero = one
        for field in ("box", "x", "v"):
            zero = _patch(zero, SIZE_AT[field], 0)
        pt.index_trr(zero)
    with pytest.raises(RuntimeError, match="Malformed TRR file: .*8-byte reals|Malformed TRR file"):
        pt.index_trr(_patch(one, SIZE_AT["natoms"], -1))
    for field in ("ir", "e", "top", "sym"):
        with pytest.raises(ValueError, match=f"{field}_size is 8"):
            pt.index_trr(_patch(one, SIZE_AT[field], 8))
    dbl = tf.write([tf.frame(N, box=_box(0), x=_xyz(N, 0))], double=True)
    with pytest.raises(ValueError, match="change of precision"):
        pt.index_trr(one + dbl)
    with pytest.raises(ValueError, match="change of precision"):
        pt.index_trr(dbl + one)
    other = tf.write([tf.frame(N + 1, box=_box(0), x=_xyz(N + 1, 0))])
    with pytest.raises(ValueError, match="natoms changes from 4 to 5"):
        pt.index_trr(one + other)


def test_writer_heads_match_the_oracle():
    from moleculekit_b200 import trr as pt

    N, F = 3, 4
    rng = np.random.default_rng(2)
    box = rng.uniform(1, 5, size=(3, 3, F)).astype(np.float32)
    time = np.float32([0.0, 0.5, 1.25, 1e6])
    step = np.array([0, 5, 2**31 - 1, -3])
    lambd = np.float32([0, 0.25, 0.5, 1])
    for with_v, with_f in ((False, False), (True, False), (False, True), (True, True)):
        heads = pt._heads(N, F, box, time, step, lambd, with_v, with_f)
        zeros = np.zeros((N, 3), np.float32)
        want = tf.write([tf.frame(N, step=int(step[k]), time=float(time[k]), lambd=float(lambd[k]), box=box[:, :, k],
                                  x=zeros, v=zeros if with_v else None, f=zeros if with_f else None)
                         for k in range(F)])
        R = 120 + 12 * N * (1 + with_v + with_f)
        recs = np.frombuffer(want, np.uint8).reshape(F, R)
        assert np.array_equal(recs[:, :120], heads)
    # lambda defaults to 0
    assert np.array_equal(pt._heads(N, F, box, time, step, None, False, False)[:, 80:84], np.zeros((F, 4), np.uint8))


def test_arguments_are_checked_before_the_device_is_touched(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import trr as pt

    c = np.zeros((12, 3, 4), np.float32)
    box, time, step = np.ones((3, 3, 4), np.float32), np.zeros(4), np.zeros(4, np.int32)
    good = dict(box=box, time=time, step=step)
    for args, kw in (((c[:, :2],), good), ((c[0],), good), ((c,), dict(good, box=box[:, :, :3])),
                     ((c,), dict(good, box=box[:2])), ((c,), dict(good, time=np.zeros(3))),
                     ((c,), dict(good, step=np.zeros(5))), ((c,), dict(good, lambd=np.zeros(2))),
                     ((c,), dict(good, velocities=c[:, :, :3])), ((c,), dict(good, forces=c[:5])),
                     ((c,), dict(good, velocities=torch.zeros((12, 3, 4), dtype=torch.float64))),
                     ((c,), dict(good, box=None)), ((c,), dict(good, chunk_bytes=0)),
                     ((c,), dict(good, scale=float("nan"))), ((np.zeros((0, 3, 4), np.float32),), good),
                     ((np.broadcast_to(np.float32(0), (pt.MAX_ATOMS + 1, 3, 4)),), good)):
        with pytest.raises(ValueError):
            pt.trr_bytes(*args, **kw)
        fn = tmp_path / "untouched.trr"
        with pytest.raises(ValueError):
            pt.write_trr(str(fn), *args, **kw)
        assert not fn.exists()
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pt.encode_trr_device(torch.zeros((12, 3, 4)), box, time, step)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pt.trr_bytes(torch.zeros((12, 3, 4)), box, time, step)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pt.decode_trr_device(torch.zeros(16, dtype=torch.uint8), np.zeros(0, np.int64), 4, 4)
    # no frames: an empty file, no device needed
    assert pt.trr_bytes(np.zeros((5, 3, 0), np.float32), np.zeros((3, 3, 0)), np.zeros(0), np.zeros(0)) == b""
    fn = tmp_path / "t.trr"
    fn.write_bytes(tf.write(mixed(5)))
    for bad in ([9], [-10], [0, 70]):
        with pytest.raises(IndexError):
            pt.read_trr_device(str(fn), frames=bad)
    with pytest.raises(IndexError):
        pt.read_trr_frames(str(fn), [6])  # six records carry x
    with pytest.raises(ValueError, match="record 1 has no x"):
        pt.read_trr_device(str(fn), frames=[0, 1])
    with pytest.raises(ValueError, match="record 0 has no v"):
        pt.read_trr_device(str(fn), frames=[3, 0], fields=("x", "v"))
    for fields in ((), ("x", "x"), ("q",), ("x", "pos")):
        with pytest.raises(ValueError, match="fields"):
            pt.read_trr_device(str(fn), fields=fields)
    with pytest.raises(ValueError):
        pt.read_trr_device(str(fn), chunk_bytes=0)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pt.trr_bytes(c, **good)
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pt.read_trr(str(fn))


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_trr_decode", 10), ("mkb_trr_encode", 12)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
