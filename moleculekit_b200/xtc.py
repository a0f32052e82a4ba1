"""XTC trajectories decoded on the GPU (K11, SURVEY 8f row 4, second half).

Mirrors ``moleculekit.xtc.read_xtc`` / ``read_xtc_frames`` (moleculekit/fileformats/xtc/xtc.pyx:34-87) and the unit handling of
``XTCread`` (moleculekit/readers.py:1830-1866).  The host only walks the XDR frame headers (a few words per frame); the
compressed coordinate blocks travel to the device as they are in the file (about a third of the float32 size) and
``mkb_xtc_decode`` expands them straight into the frame-minor ``(natoms, 3, nframes)`` layout the distance / wrapping kernels
consume -- no float32 trajectory on the host, no transposition pass.  Bit-identical to the reference reader.
"""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np
import torch

from . import _lib

XTC_MAGIC = 1995
# numpy mirror of `mkb_xtc_frame` (48 bytes)
FRAME_DESC = np.dtype([("data_offset", "<i8"), ("nbytes", "<i4"), ("natoms", "<i4"), ("precision", "<f4"),
                       ("minint", "<i4", (3,)), ("maxint", "<i4", (3,)), ("smallidx", "<i4")], align=False)
assert FRAME_DESC.itemsize == 48


def index_xtc(buf) -> dict:
    """Walk the frame headers of an XTC byte buffer (xdrfile_xtc.cpp:29-67 header, xdrfile.cpp:773-858 block header).
    Returns dict(frames=FRAME_DESC array, natoms, step (F,) int32, time (F,) float32, box (3,3,F) float32 in nm)."""
    mv = memoryview(buf)
    n = len(mv)
    pos = 0
    descs, steps, times, boxes = [], [], [], []
    natoms0 = None
    while pos + 16 <= n:
        magic, natoms, step = struct.unpack_from(">iii", mv, pos)
        if magic != XTC_MAGIC:
            raise RuntimeError(f"Malformed XTC file: bad magic number {magic} at byte {pos}")
        (time,) = struct.unpack_from(">f", mv, pos + 12)
        box = struct.unpack_from(">9f", mv, pos + 16)
        (lsize,) = struct.unpack_from(">i", mv, pos + 52)
        pos += 56
        if natoms0 is None:
            natoms0 = natoms
        if natoms != natoms0 or lsize != natoms:
            raise RuntimeError("Malformed XTC file: the number of atoms changes between frames")
        if lsize <= 9:  # xdrfile.cpp:802-806: three atoms or fewer... stored as plain floats (the test is on `size`)
            nbytes = 12 * lsize
            descs.append((pos, nbytes, natoms, 0.0, (0, 0, 0), (0, 0, 0), -1))
            pos += nbytes
        else:
            (precision,) = struct.unpack_from(">f", mv, pos)
            ints = struct.unpack_from(">8i", mv, pos + 4)
            nbytes = ints[7]
            if nbytes < 0 or pos + 36 + nbytes > n:
                raise RuntimeError("Malformed XTC file: truncated coordinate block")
            descs.append((pos + 36, nbytes, natoms, precision, ints[0:3], ints[3:6], ints[6]))
            pos += 36 + ((nbytes + 3) // 4) * 4
        steps.append(step); times.append(time); boxes.append(box)
    F = len(descs)
    frames = np.zeros(F, dtype=FRAME_DESC)
    for f, d in enumerate(descs):
        frames[f] = d
    box = np.zeros((3, 3, F), dtype=np.float32)
    if F:
        box[:] = np.asarray(boxes, dtype=np.float32).reshape(F, 3, 3).transpose(1, 2, 0)
    return dict(frames=frames, natoms=int(natoms0 or 0), step=np.asarray(steps, dtype=np.int32),
                time=np.asarray(times, dtype=np.float32), box=box)


def decode_xtc_device(file_bytes: torch.Tensor, frames: np.ndarray, natoms: int, scale: float = 1.0,
                      out: torch.Tensor | None = None) -> torch.Tensor:
    """K11 on the device: ``file_bytes`` (uint8 CUDA tensor holding the file), ``frames`` from :func:`index_xtc` (any
    subset / order of frames) -> coords (natoms, 3, len(frames)) float32, in nm (``scale=1``) or with the reference's
    ``coords *= 10`` applied (``scale=10``: Angstrom)."""
    dev = file_bytes.device
    assert file_bytes.is_cuda and file_bytes.dtype == torch.uint8 and file_bytes.is_contiguous()
    frames = np.ascontiguousarray(frames, dtype=FRAME_DESC)
    F = int(frames.shape[0])
    if out is None:
        out = torch.empty((natoms, 3, F), dtype=torch.float32, device=dev)
    assert out.shape == (natoms, 3, F) and out.dtype == torch.float32 and out.is_contiguous()
    status = torch.zeros(max(F, 1), dtype=torch.int32, device=dev)
    _lib.call(dev, "mkb_xtc_decode", _lib.ptr(file_bytes), int(file_bytes.numel()), frames.ctypes.data_as(C.c_void_p), F,
              int(natoms), _lib.ptr(out), max(F, 1), float(scale), _lib.ptr(status))
    bad = torch.nonzero(status[:F]).flatten()
    if bad.numel():
        raise RuntimeError(f"Malformed XTC file: frame {int(bad[0])} could not be decoded (status {int(status[bad[0]])})")
    return out


def _load(filename) -> bytes:
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    with open(filename, "rb") as f:
        return f.read()


def read_xtc_device(filename, frames=None, scale: float = 1.0, device=None):
    """Whole file (or the frames listed) -> (coords CUDA (natoms,3,F) float32, box (3,3,F), time, step) with the trajectory left on
    the GPU."""
    raw = _load(filename)
    idx = index_xtc(raw)
    sel = slice(None) if frames is None else np.asarray(frames, dtype=np.int64)
    dev = _lib.device(device)
    # (+4 zero bytes: the kernel reads whole 32-bit words, and a file cut right after its last block has no XDR padding)
    d_bytes = torch.frombuffer(bytearray(raw) + bytearray(4), dtype=torch.uint8).to(dev)
    coords = decode_xtc_device(d_bytes, idx["frames"][sel], idx["natoms"], scale=scale)
    return coords, idx["box"][:, :, sel], idx["time"][sel], idx["step"][sel]


def read_xtc(filename, device=None):
    """Drop-in for xtc.pyx:34-55: (coords (natoms,3,F) float32 [nm], box (3,3,F), time (F,), step (F,)) as numpy arrays."""
    coords, box, time, step = read_xtc_device(filename, device=device)
    return coords.cpu().numpy(), box.copy(), time.copy(), step.copy()


def read_xtc_frames(filename, frames, device=None):
    """Drop-in for xtc.pyx:59-87 (frames: int32 array of frame numbers)."""
    coords, box, time, step = read_xtc_device(filename, frames=np.asarray(frames), device=device)
    return coords.cpu().numpy(), np.ascontiguousarray(box), time.copy(), step.copy()
