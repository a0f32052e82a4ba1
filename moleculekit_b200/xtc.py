"""XTC trajectories decoded (K11, SURVEY 8f row 4, second half) and written (K21) on the GPU.

Mirrors ``moleculekit.xtc.read_xtc`` / ``read_xtc_frames`` (moleculekit/fileformats/xtc/xtc.pyx:34-87) and the unit handling of
``XTCread`` (moleculekit/readers.py:1830-1866).  The host only walks the XDR frame headers (a few words per frame); the
compressed coordinate blocks travel to the device as they are in the file (about a third of the float32 size) and
``mkb_xtc_decode`` expands them straight into the frame-minor ``(natoms, 3, nframes)`` layout the distance / wrapping kernels
consume -- no float32 trajectory on the host, no transposition pass.  Bit-identical to the reference reader.

The writer is the same trade the other way round (``write_xtc`` of xtc.pyx): ``mkb_xtc_encode`` compresses a trajectory
that is already on the device, the packed coordinate blocks are all that comes back over PCIe, and the host only puts
the 56-byte frame headers between them.  Byte-identical to the reference writer.
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
# one frame header of the file (xdrfile_xtc.cpp): magic, natoms, step, time, the box row by row, natoms again
FRAME_HEAD = np.dtype([("magic", ">i4"), ("natoms", ">i4"), ("step", ">i4"), ("time", ">f4"), ("box", ">f4", (9,)),
                       ("natoms2", ">i4")], align=False)
assert FRAME_HEAD.itemsize == 56
ENCODE_STATUS = {-1: "Internal overflow compressing coordinates", -2: "Internal overflow compressing coordinates",
                 -3: "consecutive atoms are further apart than the format's table of small ranges allows"}


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


# ------------------------------------------------------------------------------------------------------------ writing
def encode_xtc_device(coords: torch.Tensor, precision: float = 1000.0, scale: float = 1.0):
    """K21 on the device: ``coords`` (contiguous CUDA (natoms, 3, F) float32) -> (blocks, offsets, lengths).  ``blocks``
    is a uint8 CUDA tensor holding every frame's coordinate block -- what follows the second atom count in the file --
    back to back; frame f's is ``blocks[offsets[f] : offsets[f] + lengths[f]]`` (int64 / int32 CUDA tensors of F).
    ``precision <= 0`` means 1000 (the reference's rule); ``scale`` multiplies every coordinate first, as a float32
    operation of its own (1: the input is in nm; 0.1 undoes the ``scale=10`` of :func:`read_xtc_device`).  A frame the
    format cannot hold raises RuntimeError naming the first one."""
    dev = _lib.tensor_device(coords, "encode_xtc_device")
    if coords.dtype != torch.float32 or coords.ndim != 3 or coords.shape[1] != 3 or not coords.is_contiguous():
        raise ValueError(f"coords must be a contiguous (natoms, 3, F) float32 tensor, got {coords.dtype} {tuple(coords.shape)}")
    natoms, _, F = coords.shape
    offsets = torch.zeros(F + 1, dtype=torch.int64, device=dev)
    lengths = torch.zeros(F, dtype=torch.int32, device=dev)
    status = torch.zeros(max(F, 1), dtype=torch.int32, device=dev)
    # The lengths are known only after the library's size pass.  Start from 6 bytes per atom, half the float32 size
    # (solvated systems at precision 1000 take 4 to 5) and, when that is not enough, come back once with the size the
    # library reports.
    capacity = F * (36 + 6 * natoms)
    while True:
        blocks = torch.empty(capacity, dtype=torch.uint8, device=dev)
        try:
            _lib.call(dev, "mkb_xtc_encode", _lib.ptr(coords), max(F, 1), F, natoms, float(precision), float(scale),
                      _lib.ptr(blocks), capacity, _lib.ptr(offsets), _lib.ptr(lengths), _lib.ptr(status))
            break
        except _lib.MkbCapacity:
            capacity = int(offsets[F])
    bad = torch.nonzero(status[:F]).flatten()
    if bad.numel():
        code = int(status[bad[0]])
        raise RuntimeError(f"{ENCODE_STATUS.get(code, 'XTC encode failed')}: frame {int(bad[0])} (status {code})")
    return blocks[:int(offsets[F])], offsets[:F], lengths


def _frame_args(coords, box, time, step):
    """shapes and lengths of the writer's arguments, checked before any device work; returns (natoms, F)"""
    if coords.ndim != 3 or coords.shape[1] != 3:
        raise ValueError(f"coords must be (natoms, 3, F), got {tuple(coords.shape)}")
    natoms, _, F = (int(v) for v in coords.shape)
    if tuple(box.shape) != (3, 3, F):
        raise ValueError(f"box must be (3, 3, {F}), got {tuple(box.shape)}")
    if tuple(time.shape) != (F,) or tuple(step.shape) != (F,):
        raise ValueError(f"time and step must be ({F},), got {tuple(time.shape)} and {tuple(step.shape)}")
    return natoms, F


def frame_pieces(blocks, offsets, lengths, natoms: int, box, time, step) -> list:
    """The file as a list of buffers: for every frame its 56-byte header (magic 1995, natoms, step, time, the nine box
    floats, natoms), then its coordinate block ``blocks[offsets[f] : offsets[f] + lengths[f]]`` (host arrays)."""
    F = len(lengths)
    head = np.zeros(F, dtype=FRAME_HEAD)
    head["magic"], head["natoms"], head["natoms2"] = XTC_MAGIC, natoms, natoms
    head["step"] = np.asarray(step).astype(np.int64).astype(np.int32)  # wraps like the reference's C int
    head["time"] = np.asarray(time, dtype=np.float32)
    head["box"] = np.asarray(box, dtype=np.float32).transpose(2, 0, 1).reshape(F, 9)
    hv, bv = memoryview(head).cast("B"), memoryview(np.ascontiguousarray(blocks, dtype=np.uint8))
    pieces = []
    for f, (o, n) in enumerate(zip(np.asarray(offsets).tolist(), np.asarray(lengths).tolist())):
        pieces += [hv[56 * f:56 * f + 56], bv[o:o + n]]
    return pieces


def _pieces(coords, box, time, step, precision, scale, device) -> list:
    box, time, step = np.asarray(box), np.asarray(time), np.asarray(step)
    if isinstance(coords, torch.Tensor):
        natoms, F = _frame_args(coords, box, time, step)
        dev = _lib.tensor_device(coords, "write_xtc")
    else:
        coords = np.ascontiguousarray(coords, dtype=np.float32)
        natoms, F = _frame_args(coords, box, time, step)
        dev = _lib.device(device) if F and natoms else None
    if F == 0 or natoms == 0:  # nothing to compress: the headers alone
        return frame_pieces(np.zeros(0, np.uint8), np.zeros(F, np.int64), np.zeros(F, np.int32), natoms, box, time, step)
    if not isinstance(coords, torch.Tensor):
        coords = torch.from_numpy(coords).to(dev)
    blocks, offsets, lengths = encode_xtc_device(coords, precision, scale)
    return frame_pieces(blocks.cpu().numpy(), offsets.cpu().numpy(), lengths.cpu().numpy(), natoms, box, time, step)


def xtc_bytes(coords, box, time, step, precision: float = 1000.0, scale: float = 1.0, device=None) -> bytes:
    """The file :func:`write_xtc` writes, as a ``bytes`` object."""
    return b"".join(_pieces(coords, box, time, step, precision, scale, device))


def write_xtc(filename, coords, box, time, step, precision: float = 1000.0, scale: float = 1.0, device=None) -> None:
    """The reference's ``write_xtc(filename, coords, box, time, step)`` (xtc.pyx) with the compression on the GPU:
    ``coords`` (natoms, 3, F) float32, a numpy array (uploaded to ``device``) or a CUDA tensor (used where it is), in nm;
    ``box`` (3, 3, F), ``time`` (F,), ``step`` (F,) host arrays.  Every frame is written at ``precision``.  Only the
    compressed blocks cross PCIe; the host interleaves the frame headers and writes the file.

    The file is created or truncated.  Whether the reference appends to an existing file could not be established
    (its sources were not at hand), and neither could the unit handling of its ``Molecule``-level writer:
    ``scale=0.1`` undoes the ``scale=10`` of :func:`read_xtc_device`, and no more is claimed."""
    if isinstance(filename, bytes):
        filename = filename.decode("UTF-8")
    pieces = _pieces(coords, box, time, step, precision, scale, device)
    with open(filename, "wb") as f:
        f.writelines(pieces)
