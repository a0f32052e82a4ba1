"""The host side of AMBER ASCII trajectory reading and writing (moleculekit_b200/mdcrd.py; K25 parses and formats on
the device): the independent oracle's round trip and a small file written out byte by byte, every index_mdcrd rule
(box detection, one atom, truncation, CRLF), the writer's argument and range checks that run before the file is opened,
and the C-ABI symbols."""
import logging
import os

import numpy as np
import pytest

from oracle import mdcrd_format as of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(N, F, seed, scale=30.0):
    """F (N, 3) float32 frames well inside the writable range"""
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def boxes(F, seed):
    return [b for b in np.random.default_rng(seed).uniform(20, 90, size=(F, 3)).astype(np.float32)]


def test_oracle_round_trip():
    for N in (1, 2, 3, 4, 7):
        for with_box in (False, True):
            xs = frames(N, 5, N)
            bx = boxes(5, N) if with_box else None
            raw = of.write(xs, bx, title="round trip")
            got = of.read(raw, N, with_box)
            assert got["title"] == "round trip".ljust(80) and got["trailing"] == 0
            want = np.float32([[float("%8.3f" % v) for v in x.reshape(-1)] for x in xs]).reshape(5, N, 3)
            assert np.array_equal(got["coords"], want)
            if with_box:
                assert np.array_equal(got["box"], np.float32([[float("%8.3f" % v) for v in b] for b in bx]))
            # the file's own values come back unchanged
            assert of.write(list(got["coords"]), None if bx is None else list(got["box"]), "round trip") == raw


def test_two_atoms_two_frames_with_a_box_byte_by_byte():
    xs = [np.float32([[1.0, -2.5, 0.0625], [1234.5678, -0.0004, 9999.999]]),
          np.float32([[-999.999, 0.5, -0.0], [3.14159, 2.71828, -12.3456]])]
    bx = [np.float32([30.0, 40.5, 50.25]), np.float32([31.0, 41.5, 51.25])]
    want = (b"t".ljust(80) + b"\n"
            b"   1.000  -2.500   0.0621234.568  -0.0009999.999\n"
            b"  30.000  40.500  50.250\n"
            b"-999.999   0.500  -0.000   3.142   2.718 -12.346\n"
            b"  31.000  41.500  51.250\n")
    assert of.write(xs, bx, title="t") == want
    from moleculekit_b200 import mdcrd as pm

    assert pm.frame_bytes(2, True) == 49 + 25 and len(want) == 81 + 2 * 74
    idx = pm.index_mdcrd(want, 2)
    assert idx == dict(title="t", has_box=True, frame_bytes=74, offset=81, n_frames=2)


def test_index_detects_the_box_line():
    from moleculekit_b200 import mdcrd as pm

    for N in (2, 3, 4, 31, 33, 97):
        for with_box in (False, True):
            for F in (1, 2, 5):
                raw = of.write(frames(N, F, N), boxes(F, N) if with_box else None, title="x")
                idx = pm.index_mdcrd(raw, N)
                assert idx["has_box"] == with_box and idx["n_frames"] == F, (N, with_box, F)
                assert idx["frame_bytes"] == pm.frame_bytes(N, with_box) and idx["offset"] == 81
                assert pm.index_mdcrd(np.frombuffer(raw, np.uint8), N) == idx
                # the caller's word wins: the other layout reads the same bytes as other frames
                assert pm.index_mdcrd(raw, N, box=not with_box)["has_box"] == (not with_box)


def test_index_with_one_atom():
    from moleculekit_b200 import mdcrd as pm

    for F in (1, 3):
        raw = of.write(frames(1, F, 1), None)  # 25 F bytes: odd multiples of 25 only fit frames without a box
        assert pm.index_mdcrd(raw, 1) == dict(title="", has_box=False, frame_bytes=25, offset=81, n_frames=F)
    for F in (2, 4):
        raw = of.write(frames(1, F, 1), None)  # 50 k bytes: k boxed frames or 2 k plain ones
        with pytest.raises(ValueError, match="box=True or box=False"):
            pm.index_mdcrd(raw, 1)
        assert pm.index_mdcrd(raw, 1, box=False)["n_frames"] == F
        assert pm.index_mdcrd(raw, 1, box=True)["n_frames"] == F // 2
    raw = of.write(frames(1, 3, 1), boxes(3, 1))  # 150 bytes: ambiguous as well
    with pytest.raises(ValueError, match="box=True"):
        pm.index_mdcrd(raw, 1)
    assert pm.index_mdcrd(raw, 1, box=True)["n_frames"] == 3
    with pytest.raises(ValueError, match="box=True"):
        pm.index_mdcrd(raw[:-7], 1)  # neither reading ends on a whole frame
    assert pm.index_mdcrd(of.write([], None), 1)["n_frames"] == 0


def test_truncated_last_frame_is_dropped_with_a_warning(caplog):
    from moleculekit_b200 import mdcrd as pm

    for N, with_box in ((5, False), (5, True), (40, True)):
        raw = of.write(frames(N, 4, N), boxes(4, N) if with_box else None)
        S = pm.frame_bytes(N, with_box)
        for cut in (1, 2, 25, S - 1):
            with caplog.at_level(logging.WARNING, logger="moleculekit_b200.mdcrd"):
                caplog.clear()
                idx = pm.index_mdcrd(raw[:len(raw) - cut], N, box=with_box)
                assert idx["n_frames"] == 3 and caplog.records, cut
        with caplog.at_level(logging.WARNING, logger="moleculekit_b200.mdcrd"):
            caplog.clear()
            assert pm.index_mdcrd(raw[:len(raw) - S], N)["n_frames"] == 3 and not caplog.records


def test_index_rejections():
    from moleculekit_b200 import mdcrd as pm

    raw = of.write(frames(4, 2, 0), None, title="crlf")
    with pytest.raises(ValueError, match="CRLF"):
        pm.index_mdcrd(raw.replace(b"\n", b"\r\n"), 4)
    with pytest.raises(ValueError, match="no title line"):
        pm.index_mdcrd(b"   1.000   2.000", 4)
    for bad in (0, -1, pm.MAX_ATOMS + 1):
        with pytest.raises(ValueError, match="natoms"):
            pm.index_mdcrd(raw, bad)
    assert pm.index_mdcrd(b"title only\n", 4)["n_frames"] == 0


def test_writer_argument_checks(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import mdcrd as pm

    c = np.zeros((12, 3, 4), np.float32)

    def huge(v, at=(5, 1, 2)):
        x = c.copy()
        x[at] = v
        return x

    cases = [((c[:, :2],), {}), ((c[0],), {}), ((np.zeros((0, 3, 4), np.float32),), {}),
             ((c,), dict(box=np.ones((3, 3), np.float32))), ((c,), dict(box=np.ones((2, 4), np.float32))),
             ((c,), dict(title="x" * 81)), ((c,), dict(title="a\nb")), ((c,), dict(title="café")),
             ((c,), dict(title=b"bytes")), ((c,), dict(chunk_bytes=0))]
    for v, where in ((np.nan, "frame 2, atom 5, axis y"), (np.inf, "frame 2, atom 5, axis y"),
                     (-np.inf, "frame 2, atom 5, axis y"), (10000.0, "frame 2, atom 5, axis y"),
                     (np.nextafter(np.float32(9999.999), np.float32(np.inf)), "frame 2, atom 5, axis y"),
                     (-1000.0, "frame 2, atom 5, axis y"), (np.float32(-999.9995), "frame 2, atom 5, axis y")):
        cases.append(((huge(v),), dict(match=where)))
    # the first offender in file order: frame, then atom, then axis
    x = huge(1e5, (7, 0, 1))
    x[3, 2, 1] = np.nan
    x[0, 0, 3] = -5000
    cases.append(((x,), dict(match="frame 1, atom 3, axis z")))
    cases.append(((c,), dict(box=np.float32([[1, 2, 3, 4], [5, 6, np.inf, 8], [9, 10, 11, 1e4]]),
                             match="box at frame 2, axis B")))
    for args, kw in cases:
        match = kw.pop("match", None)
        with pytest.raises(ValueError, match=match):
            pm.mdcrd_bytes(*args, **kw)
        fn = tmp_path / "untouched.mdcrd"
        with pytest.raises(ValueError, match=match):
            pm.write_mdcrd(str(fn), *args, **kw)
        assert not fn.exists()
    # the range rule's edges are accepted: the checks pass and only the missing device stops the call
    edge = huge(np.float32(9999.999), (0, 0, 0))
    edge[1, 1, 1] = np.float32(-999.999)
    edge[2, 2, 2] = np.float32(-0.0)
    edge[3, 0, 0] = np.float32(-0.0004)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pm.mdcrd_bytes(edge)
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            pm.read_mdcrd_device(str(_write(tmp_path, of.write(frames(3, 2, 0), None))), 3)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pm.encode_mdcrd_device(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pm.mdcrd_bytes(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        pm.decode_mdcrd_device(torch.zeros(16, dtype=torch.uint8), np.zeros(0, np.int64), 4, False)
    # no frames: the title line alone, no device needed
    assert pm.mdcrd_bytes(np.zeros((5, 3, 0), np.float32), title="empty") == b"empty".ljust(80) + b"\n"
    assert pm.mdcrd_bytes(np.zeros((5, 3, 0), np.float32), box=np.zeros((3, 0))) == b" " * 80 + b"\n"


def _write(tmp_path, raw, name="t.mdcrd"):
    fn = tmp_path / name
    fn.write_bytes(raw)
    return fn


def test_reader_arguments(tmp_path):
    from moleculekit_b200 import mdcrd as pm

    fn = str(_write(tmp_path, of.write(frames(3, 5, 0), None)))
    for bad in ([5], [-6], [0, 70]):
        with pytest.raises(IndexError):
            pm.read_mdcrd_device(fn, 3, frames=bad)
    with pytest.raises(ValueError, match="chunk_bytes"):
        pm.read_mdcrd_device(fn, 3, chunk_bytes=0)


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_mdcrd_decode", 13), ("mkb_mdcrd_encode", 10)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs
