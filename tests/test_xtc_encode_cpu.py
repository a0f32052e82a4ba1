"""The host side of the XTC writer (moleculekit_b200/xtc.py; K21 does the compression on the device): the frame headers
it puts between ready-made coordinate blocks, the argument checks that run before any device work, the C-ABI symbol,
and which of the reference's nine files survive the float -> int step again after decoding (tests/test_xtc_encode_gpu.py
compares exactly those with the committed bytes)."""
import os

import numpy as np
import pytest

from oracle import xtc_cases as xc
from oracle import xtc_writer as xw

# decoded coordinates of these two files (lattice values of 2^24 and more) do not return to the stored integers:
# (float)int * (float)(1/precision) * precision is no longer within half a step of int
NOT_REQUANTISABLE = {"wide_x", "wide_xyz"}


def _blocks(frames):
    """the coordinate blocks of oracle frames, packed as K21 packs them: (bytes, offsets, lengths)"""
    blocks = [xw.frame_bytes(fr)[56:] for fr in frames]
    lengths = np.array([len(b) for b in blocks], np.int32)
    offsets = np.concatenate([[0], np.cumsum(lengths[:-1])]).astype(np.int64)
    return np.frombuffer(b"".join(blocks), np.uint8), offsets, lengths


@pytest.mark.parametrize("name", ["water", "atoms_9", "atoms_10", "frames_65", "mixed_headers", "range_2_31"])
def test_headers_are_interleaved_as_the_oracle_writes_them(name):
    from moleculekit_b200 import xtc as px

    frames = xc.build(name).frames
    for f, fr in enumerate(frames):  # steps beyond int32 wrap as the reference's C int does
        fr.step = [2**31 + 5, -7, 2**32 + 3][f % 3] + f
    want = xw.write_frames(frames)
    blocks, offsets, lengths = _blocks(frames)
    box = np.stack([fr.box for fr in frames], axis=2)
    time = np.array([fr.time for fr in frames], np.float32)
    step = np.array([fr.step for fr in frames], np.int64)
    got = b"".join(px.frame_pieces(blocks, offsets, lengths, frames[0].natoms, box, time, step))
    assert got == want
    idx = px.index_xtc(got)  # and the package's own header walk finds every block again
    assert idx["natoms"] == frames[0].natoms and np.array_equal(idx["box"], box) and np.array_equal(idx["time"], time)
    assert np.array_equal(idx["step"], step.astype(np.int32))


def test_arguments_are_checked_before_the_device_is_touched(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import xtc as px

    c = np.zeros((12, 3, 4), np.float32)
    box, time, step = np.zeros((3, 3, 4), np.float32), np.zeros(4, np.float32), np.zeros(4, np.int32)
    for bad in ((c[:, :2], box, time, step), (c[0], box, time, step), (c, box[:, :, :3], time, step),
                (c, box[:2], time, step), (c, box, time[:3], step), (c, box, time, np.zeros(5, np.int32)),
                (c, box, np.zeros((4, 1), np.float32), step)):
        with pytest.raises(ValueError):
            px.xtc_bytes(*bad)
    fn = tmp_path / "untouched.xtc"
    with pytest.raises(ValueError):
        px.write_xtc(str(fn), c, box[:, :, :3], time, step)
    assert not fn.exists()
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        px.encode_xtc_device(torch.zeros((12, 3, 4)))
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        px.xtc_bytes(torch.zeros((12, 3, 4)), box, time, step)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            px.xtc_bytes(c, box, time, step)


def test_nothing_to_compress_needs_no_device(tmp_path):
    from moleculekit_b200 import xtc as px

    empty = np.zeros((30, 3, 0), np.float32)
    assert px.xtc_bytes(empty, np.zeros((3, 3, 0)), np.zeros(0), np.zeros(0)) == b""
    fn = tmp_path / "empty.xtc"
    fn.write_bytes(b"stale")
    px.write_xtc(str(fn), empty, np.zeros((3, 3, 0)), np.zeros(0), np.zeros(0))
    assert fn.read_bytes() == b""  # created or truncated
    box = np.arange(18, dtype=np.float32).reshape(3, 3, 2)
    got = px.xtc_bytes(np.zeros((0, 3, 2), np.float32), box, np.array([1.5, 2.5]), np.array([3, 4]))
    assert got == xw.write_xtc(np.zeros((0, 3, 2), np.float32), box, [1.5, 2.5], [3, 4])


def test_abi_symbol():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    assert "mkb_xtc_encode" in _lib.EXPORTS and hasattr(lib, "mkb_xtc_encode")
    assert len(lib.mkb_xtc_encode.argtypes) == 13
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mkb200.h")).read()
    for name, code in (("MKB_XTC_ENC_COORD_OVERFLOW", -1), ("MKB_XTC_ENC_RANGE_OVERFLOW", -2),
                       ("MKB_XTC_ENC_SMALLIDX_RANGE", -3)):
        assert f"#define {name} ({code})" in hdr
    from moleculekit_b200 import xtc as px

    assert set(px.ENCODE_STATUS) == {-1, -2, -3}


def test_which_golden_files_requantise(g_xtc):
    """Decoded coordinates re-enter the float -> int step when they are written again.  For seven of the reference's
    nine files that returns the stored integers (so the GPU writer must reproduce the committed bytes from the golden
    coordinates); for the two wide-range files it does not, and the oracle writer on the same floats is the yardstick."""
    for name in g_xtc["names"].tolist():
        raw = open(os.path.join(g_xtc["_dir"], name + ".xtc"), "rb").read()
        coords = g_xtc[f"{name}_coords"]
        same = all(fr.ints is None or np.array_equal(xw.to_lattice(coords[:, :, f], fr.precision), fr.ints)
                   for f, fr in enumerate(xw.read_ints(raw)))
        assert same == (name not in NOT_REQUANTISABLE), name
        again = xw.write_xtc(coords, g_xtc[f"{name}_box"], g_xtc[f"{name}_time"], g_xtc[f"{name}_step"])
        assert (again == raw) == same, name
