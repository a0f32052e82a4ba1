"""The host plumbing the trajectory modules share (moleculekit_b200/_trajio.py): the slab gather, the whole-frame
stager, and the rule that every writer checks its arguments before it opens, and so creates or truncates, its file."""
import importlib

import numpy as np
import pytest

C = np.zeros((12, 3, 4), np.float32)
BOX = np.ones((3, 4), np.float32)
NAN = C.copy()
NAN[5, 1, 2] = np.nan

# what each writer is given besides the file name: arguments it accepts, then changes to them it rejects
WRITERS = {
    "dcd": dict(coords=C),
    "netcdf": dict(coords=C),
    "trr": dict(coords=C, box=np.ones((3, 3, 4), np.float32), time=np.zeros(4), step=np.zeros(4, np.int32)),
    "mdcrd": dict(coords=C),
    "xyz": dict(coords=C, element=["C"] * 12),
}
REJECTED = {
    "dcd": [dict(coords=C[:, :2]), dict(box=BOX[:, :3]), dict(boxangles=BOX), dict(box=BOX, boxangles=BOX[:2]),
            dict(istart=2**31), dict(nsavc=-2**31 - 1), dict(title=[1, 2]), dict(chunk_bytes=0)],
    "netcdf": [dict(coords=C[:, :2]), dict(coords=np.zeros((0, 3, 4), np.float32)), dict(box=BOX[:2]),
               dict(boxangles=BOX), dict(time=np.zeros(3)), dict(title="café"), dict(chunk_bytes=0)],
    "trr": [dict(coords=C[0]), dict(box=None), dict(time=np.zeros(3)), dict(step=np.zeros(5)),
            dict(lambd=np.zeros(2)), dict(velocities=C[:, :, :3]), dict(forces=C[:5]), dict(scale=float("nan")),
            dict(chunk_bytes=0)],
    "mdcrd": [dict(coords=C[:, :2]), dict(box=np.ones((2, 4), np.float32)), dict(title="x" * 81), dict(coords=NAN),
              dict(box=np.full((3, 4), 1e4, np.float32)), dict(chunk_bytes=0)],
    "xyz": [dict(coords=C[:, :2]), dict(element=["C"] * 11), dict(element=["C"] * 11 + ["C a"]),
            dict(comment="a\nb"), dict(coords=NAN), dict(chunk_bytes=0)],
}


@pytest.mark.parametrize("fmt", list(WRITERS))
def test_rejected_arguments_leave_an_existing_file_alone(tmp_path, fmt):
    write = getattr(importlib.import_module(f"moleculekit_b200.{fmt}"), f"write_{fmt}")
    fn = tmp_path / f"precious.{fmt}"
    for change in REJECTED[fmt]:
        fn.write_bytes(b"precious")
        with pytest.raises(ValueError):
            write(str(fn), **dict(WRITERS[fmt], **change))
        assert fn.read_bytes() == b"precious", change


def test_slab_gather_reads_only_the_slabs(tmp_path):
    from moleculekit_b200 import _trajio

    rng = np.random.default_rng(4)
    raw = rng.integers(0, 256, size=300000, dtype=np.uint8)
    fn = tmp_path / "bytes"
    fn.write_bytes(raw.tobytes())
    slab = 96
    for starts in (np.arange(0, 200000, 100), np.arange(0, 290000, 96), np.array([8, 104, 5000, 5096, 299900 - 96]),
                   np.sort(rng.choice(2000, size=700, replace=False)) * 140 + 4, np.arange(0, 1100 * 200, 200)):
        out = np.zeros((len(starts), slab), np.uint8)
        with open(fn, "rb") as fh:
            _trajio.gather_slabs(fh.fileno(), starts.astype(np.int64), slab, out, "NetCDF")
        assert np.array_equal(out, raw[starts[:, None] + np.arange(slab)[None, :]])
    with open(fn, "rb") as fh, pytest.raises(RuntimeError, match="changed while it was read"):
        _trajio.gather_slabs(fh.fileno(), np.array([299990], np.int64), slab, np.zeros((1, slab), np.uint8), "NetCDF")


@pytest.mark.parametrize("piece", [1 << 30, 1000])
def test_stage_frames_reads_whole_frames_back_to_back(tmp_path, monkeypatch, piece):
    from moleculekit_b200 import _trajio

    monkeypatch.setattr(_trajio, "PREADV_BYTES", piece)  # 1000: every run longer than that takes several reads
    rng = np.random.default_rng(5)
    raw = rng.integers(0, 256, size=300000, dtype=np.uint8)
    fn = tmp_path / "bytes"
    fn.write_bytes(raw.tobytes())
    size = rng.integers(1, 290, size=1000)  # uneven frames back to back from byte 17
    start = 17 + np.concatenate([[0], np.cumsum(size[:-1])])
    for uniq in (np.arange(1000), np.array([0]), np.array([999]), np.array([3, 4, 5, 9, 10, 500, 998, 999]),
                 np.sort(rng.choice(1000, size=300, replace=False))):
        want = np.concatenate([raw[start[j]:start[j] + size[j]] for j in uniq])
        out = np.zeros(len(want) + 5, np.uint8)
        with open(fn, "rb") as fh:
            at = _trajio.stage_frames(fh.fileno(), start, size, uniq, out, "Test")
        assert at.tolist() == [0] + np.cumsum(size[uniq]).tolist()
        assert np.array_equal(out[:len(want)], want) and not out[len(want):].any()
    with open(fn, "rb") as fh, pytest.raises(RuntimeError, match="Malformed Test file: the file changed while it was"):
        _trajio.stage_frames(fh.fileno(), np.array([299000, 299500]), np.array([500, 501]), np.array([0, 1]),
                             np.zeros(1001, np.uint8), "Test")
