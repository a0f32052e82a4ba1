"""K11 (xtc_decode_kernel) on generated XTC streams: every decoded coordinate equals (float)int · (float)(1/precision)
of the integers the stream was written from, bit for bit, with no tolerance.

The streams (oracle/xtc_cases.py) sweep the precision, the plain / compressed boundary at 9-11 atoms, 1-300 frames
(several 64-thread blocks), the wide-range branch on one to three axes, full-range triples of 65-72 bits and values on
both sides of 2^32 and 2^64, runs of 9 and 10 atoms, runs at small ranges 65-72, the small range walked from 9 to 72,
ranges of 2^31 or more, one file with mixed headers and one of 50 000 atoms x 8 frames.  tests/test_xtc_writer_cpu.py
checks the writer against the reference's own files and the C oracle on the same streams.
"""
import functools

import numpy as np
import pytest

from oracle import xtc_cases as xc

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _case(name):
    return xc.build(name)


def _file(tmp_path, name):
    fn = tmp_path / f"{name}.xtc"
    fn.write_bytes(_case(name).raw)
    return str(fn)


def _assert_bits(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert not len(bad), f"{what}: {len(bad)} values differ, first at (atom, axis, frame) {tuple(bad[0])}: " \
                         f"{got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}"


@pytest.mark.parametrize("name", xc.NAMES)
def test_decode_is_exact(tmp_path, name):
    from moleculekit_b200 import xtc as px

    c = _case(name)
    coords, box, time, step = px.read_xtc(_file(tmp_path, name))
    _assert_bits(coords, c.expected(), name)
    assert np.array_equal(box, np.stack([f.box for f in c.frames], axis=2))
    assert np.array_equal(time, [f.time for f in c.frames]) and np.array_equal(step, [f.step for f in c.frames])


def test_frame_subsets_in_any_order(tmp_path):
    """read_xtc_frames with a shuffled, repeating frame list over 300 frames (five 64-thread blocks)"""
    from moleculekit_b200 import xtc as px

    c = _case("frames_300")
    rng = np.random.default_rng(3)
    sel = np.concatenate([rng.permutation(300), rng.integers(0, 300, 77), [299, 0, 64, 63, 64]]).astype(np.int32)
    coords, box, time, step = px.read_xtc_frames(_file(tmp_path, "frames_300"), sel)
    _assert_bits(coords, c.expected()[:, :, sel], "frames_300 subset")
    assert np.array_equal(step, np.array([f.step for f in c.frames])[sel])
    assert np.array_equal(box, np.stack([f.box for f in c.frames], axis=2)[:, :, sel])


@pytest.mark.parametrize("name", ["frames_65", "mixed_headers", "range_2_31", "high_smallidx", "precision_333.3"])
def test_angstrom_scale_is_a_second_float32_multiplication(tmp_path, name):
    """read_xtc_device(scale=10): the reference's coords *= 10 after the decode, as its own float32 rounding"""
    from moleculekit_b200 import xtc as px

    d, _, _, _ = px.read_xtc_device(_file(tmp_path, name), scale=10.0)
    assert d.is_cuda and d.is_contiguous()
    want = _case(name).expected() * np.float32(10)
    _assert_bits(d.cpu().numpy(), want, name)
