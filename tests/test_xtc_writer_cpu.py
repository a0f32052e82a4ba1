"""The Python XTC writer and integer reader (oracle/xtc_writer.py) against the reference's files, and the C oracle's XTC
decoder against exact expectations on generated streams (oracle/xtc_cases.py).

The writer is trusted because it reproduces, byte for byte, the nine files the reference's own write_xtc wrote
(tests/golden/xtc/).  The generated streams then reach the decoder paths those nine files never take; the coverage guard
at the end fails if an edit to the generator drops one of them.
"""
import functools
import os

import numpy as np
import pytest

from oracle import xtc_cases as xc
from oracle import xtc_writer as xw


@functools.lru_cache(maxsize=None)
def _case(name):
    return xc.build(name)


def _golden(g, name):
    return open(os.path.join(g["_dir"], name + ".xtc"), "rb").read()


def _assert_bits(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert not len(bad), f"{what}: {len(bad)} values differ, first at (atom, axis, frame) {tuple(bad[0])}: " \
                         f"{got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}"


def test_bit_primitives_round_trip():
    """send_bits / send_ints and the reader's take / take_ints are inverses, up to 72-bit mixed-radix values"""
    rng = np.random.default_rng(5)
    w, fields = xw.BitWriter(), []
    for _ in range(3000):
        if rng.random() < 0.5:
            n = int(rng.integers(0, 33))
            v = int(rng.integers(0, 1 << n)) if n else 0
            w.send_bits(n, v)
            fields.append((n, v))
        else:
            sizes = [int(s) for s in rng.integers(1, 0x1000000, size=3)]
            nums = [int(rng.integers(0, s)) for s in sizes]
            w.send_ints(xw.sizeofints(sizes), sizes, nums)
            fields.append((sizes, nums))
    r = xw.BitReader(w.tobytes())
    for f, v in fields:
        got = r.take(f) if isinstance(f, int) else r.take_ints(xw.sizeofints(f), f)
        assert got == v
    assert len(w.tobytes()) == (w.nbits + 7) // 8
    with pytest.raises(ValueError):
        w.send_ints(8, (16, 16, 16), (15, 15, 15))  # 4095 needs 12 bits


def test_read_ints_matches_reference_goldens(g_xtc):
    """The integer reader on the nine committed files: (float)int · (float)(1/precision) is what the reference's
    read_xtc returned, bit for bit, and the headers agree with the golden arrays and the package's header walk."""
    from moleculekit_b200 import xtc as px

    for name in g_xtc["names"].tolist():
        raw = _golden(g_xtc, name)
        frames = xw.read_ints(raw)
        _assert_bits(xw.coords(frames), g_xtc[f"{name}_coords"], name)
        assert np.array_equal(np.stack([f.box for f in frames], axis=2), g_xtc[f"{name}_box"])
        assert np.array_equal([f.time for f in frames], g_xtc[f"{name}_time"])
        assert np.array_equal([f.step for f in frames], g_xtc[f"{name}_step"])
        idx = px.index_xtc(raw)["frames"]
        for fr, d in zip(frames, idx):
            if fr.ints is not None:
                assert (fr.precision, fr.minint, fr.maxint, fr.smallidx) == \
                       (d["precision"], tuple(d["minint"]), tuple(d["maxint"]), d["smallidx"])


def test_writer_reproduces_reference_files_byte_for_byte(g_xtc):
    """The integers (and headers) of each committed file, written again, give the reference writer's bytes: every
    choice of xdrfile_compress_coord_float (small range, swaps, runs, flags, adaptation, byte count, padding) agrees."""
    for name in g_xtc["names"].tolist():
        raw = _golden(g_xtc, name)
        frames = [xw.Frame(step=f.step, time=f.time, box=f.box, precision=f.precision, ints=f.ints, xyz=f.xyz)
                  for f in xw.read_ints(raw)]
        out = xw.write_frames(frames)
        assert len(out) == len(raw) and out == raw, name


def test_writer_matches_live_reference(refmods, tmp_path):
    """The float -> int step: write_xtc equals the reference's write_xtc byte for byte on seeded floats."""
    if refmods is None or len(refmods) < 6:
        pytest.skip("oracle/_ref not built")
    xr = refmods[5]
    rng = np.random.default_rng(91)
    for t, (N, F, sd) in enumerate([(5, 2, 1.0), (9, 2, 1.0), (10, 3, 0.5), (300, 3, 0.05), (400, 2, 2.0),
                                    (200, 2, 40.0), (1000, 2, 1.5)]):
        xyz = (rng.normal(0, sd, size=(N, 3, F)) + rng.normal(0, 3, 3)[None, :, None]).astype(np.float32)
        xyz[::7] = -xyz[::7]  # both signs of the ± 0.5 rounding
        box = rng.uniform(0, 5, size=(3, 3, F)).astype(np.float32)
        time = (np.arange(F) * 0.25).astype(np.float32)
        step = np.arange(F, dtype=np.uint32) * 100
        fn = str(tmp_path / f"w{t}.xtc")
        xr.write_xtc(fn.encode(), np.ascontiguousarray(xyz), box, time, step)
        assert open(fn, "rb").read() == xw.write_xtc(xyz, box, time, step), (N, F, sd)


def test_writer_refuses_what_the_reference_cannot_write():
    # initial small range 65: the reference reads magicints[73], one past its table
    far = np.arange(12)[:, None] * np.array([[3_000_000, 0, 0]])
    with pytest.raises(ValueError, match="past its table"):
        xw.compress_frame(far, 1000.0)
    # a range of 2^31: the reference prints "Internal overflow" and writes a corrupt stream
    with pytest.raises(ValueError, match="Internal overflow"):
        xw.compress_frame(np.array([[-(2**30), 0, 0]] * 6 + [[2**30 + 10, 0, 0]] * 6), 1000.0)
    with pytest.raises(ValueError, match="Internal overflow"):
        xw.to_lattice(np.array([[3e6, 0, 0]], np.float32), 1000.0)
    # a flag-less group repeats the previous run: asking for another one is refused
    blk = xw.Block([0, 0, 0], [100, 100, 100], 12)
    blk.group([50, 50, 50], [[51, 51, 51]])
    with pytest.raises(ValueError, match="repeats the last run"):
        blk.group([10, 10, 10], [], 0, flag=False)


@pytest.mark.parametrize("name", xc.NAMES)
def test_oracle_decodes_generated_streams_exactly(oracle, name):
    """oracle_xtc_decode_block and the integer reader on every generated stream: exact expectation, bit for bit."""
    from moleculekit_b200 import xtc as px

    c = _case(name)
    coords, box, time, step = oracle.read_xtc(c.raw)
    _assert_bits(coords, c.expected(), name)
    assert np.array_equal(box, np.stack([f.box for f in c.frames], axis=2))
    assert np.array_equal(time, [f.time for f in c.frames]) and np.array_equal(step, [f.step for f in c.frames])
    back = xw.read_ints(c.raw)
    for a, b in zip(back, c.frames):
        assert np.array_equal(a.ints if a.ints is not None else a.xyz, b.ints if b.ints is not None else b.xyz), name
    idx = px.index_xtc(c.raw)  # the package's header walk finds every block where the writer put it
    assert idx["natoms"] == coords.shape[0] and len(idx["frames"]) == len(c.frames)
    assert np.array_equal(idx["frames"]["smallidx"], [-1 if f.smallidx is None else f.smallidx for f in back])


def test_generated_streams_cover_every_decoder_branch():
    """The union of what the generated streams drive covers every decoder path no committed file reaches."""
    cover = set().union(*(_case(n).cover for n in xc.NAMES))

    def values(key):
        return {k[1] for k in cover if k[0] == key}

    # paths the committed files never take
    assert ">64" in values("full_bits")                        # full-range triple > 64 bits, sizes <= 2^24
    assert set(range(65, 73)) <= values("run_smallidx")         # run triples at small ranges 65..72
    assert min(values("adapted_to")) == 9 and max(values("adapted_to")) == 72
    assert values("precision") - {1000.0}                       # precision other than 1000
    assert {1, 63, 64, 65, 300} <= values("frames")              # more than one 64-thread block of frames
    assert {"precision", "ranges", "smallidx"} <= values("mixed")  # frames of one file with different headers
    assert set(range(27, 32)) <= values("run_code")              # runs of 9 and 10 atoms
    assert ("range_overflows_int",) in cover                    # maxint - minint + 1 > INT_MAX
    assert max(values("natoms")) >= 50_000                      # large frames
    # and every branch a decoder has
    assert {1, 2, 3} <= values("wide_axes")                      # bitsize == 0 with one, two, three wide axes
    assert {"<=32", "33-64", ">64"} <= values("full_bits")
    assert {2**32 - 1, 2**32, 2**64 - 1, 2**64} <= values("full_value")
    assert {("flagless_run",), ("plain",), ("negative_minint",)} <= cover
