"""Host plumbing shared by the trajectory file modules that decode and encode frames on the device (``dcd``,
``netcdf``, ``trr``, ``mdcrd``, ``xyz``, ``pdb``, ``gro``, ``cif``, ``lammpstrj``): the frame selection, the chunk planner of a frame list, the slab
gather and the whole-frame stager into staging buffers, the double-buffered read -> copy -> decode loop, the writers'
coords intake, the frame-minor layout check, and the double-buffered encode -> copy -> write loop."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib

IOV_MAX = 1024  # buffers per preadv call (Linux)
PREADV_BYTES = 1 << 30  # slab bytes per preadv call, well below the 2 GiB a single read returns at most


def select(n: int, frames) -> np.ndarray:
    """The frames a reader returns: all ``n`` for None, else ``frames`` (any order, repeats allowed) as int64 indices
    into range(n); one out of range raises IndexError."""
    every = np.arange(n, dtype=np.int64)
    return every if frames is None else every[np.asarray(frames, np.int64).ravel()]


def chunks(sel: np.ndarray, size: np.ndarray, chunk_bytes: int) -> list:
    """Cut the listed frames, in order, into chunks whose distinct frames take at most ``chunk_bytes`` (one frame at
    least): [(k0, k1, sorted distinct frames)]."""
    out, k0, seen, used = [], 0, set(), 0
    for k, j in enumerate(sel.tolist()):
        if j in seen:
            continue
        if seen and used + size[j] > chunk_bytes:
            out.append((k0, k, np.array(sorted(seen), np.int64)))
            k0, seen, used = k, set(), 0
        seen.add(j)
        used += int(size[j])
    if len(sel):
        out.append((k0, len(sel), np.array(sorted(seen), np.int64)))
    return out


def gather_slabs(fd: int, starts: np.ndarray, slab: int, out: np.ndarray, fmt: str) -> None:
    """Read the ``slab`` bytes at each file offset of ``starts`` (ascending) into the rows of ``out`` (len(starts), slab).
    A run of slabs whose gaps are small is one ``preadv``: the slabs land in their rows, the bytes between them (the
    record's other variables) in a scratch buffer, so the page cache is copied once and no gap reaches ``out``.  A short
    read raises RuntimeError("Malformed ``fmt`` file: ...")."""
    junk = memoryview(bytearray(max(slab, 1 << 20)))
    n, k = len(starts), 0
    while k < n:
        iov, j = [memoryview(out[k])], k
        while j + 1 < n and len(iov) + 2 <= IOV_MAX and (j + 2 - k) * slab <= PREADV_BYTES:
            gap = int(starts[j + 1] - starts[j]) - slab
            if not 0 <= gap <= len(junk):
                break
            if gap:
                iov.append(junk[:gap])
            iov.append(memoryview(out[j + 1]))
            j += 1
        want = sum(len(v) for v in iov)
        if os.preadv(fd, iov, int(starts[k])) != want:
            raise RuntimeError(f"Malformed {fmt} file: the file changed while it was read")
        k = j + 1


def read_exact(fd: int, buf, pos: int, fmt: str) -> None:
    """Fill ``buf`` with the bytes at file offset ``pos``, in ``preadv`` calls of at most PREADV_BYTES.  A short read
    raises RuntimeError("Malformed ``fmt`` file: ...")."""
    mv = memoryview(buf)
    for a in range(0, len(mv), PREADV_BYTES):
        part = mv[a:a + PREADV_BYTES]
        if os.preadv(fd, [part], pos + a) != len(part):
            raise RuntimeError(f"Malformed {fmt} file: the file changed while it was read")


def stage_frames(fd: int, start: np.ndarray, size: np.ndarray, uniq: np.ndarray, out: np.ndarray,
                 fmt: str) -> np.ndarray:
    """Read the whole frames ``uniq`` (ascending; frame j is the ``size[j]`` bytes at file offset ``start[j]``, and
    frame j + 1 follows it in the file) back to back into ``out``, a run of consecutive frames in one read.  Returns
    the staging offsets: frame uniq[k] lands at [at[k], at[k + 1]).  A short read raises RuntimeError as
    :func:`read_exact` does."""
    at = np.concatenate([[0], np.cumsum(size[uniq])]).astype(np.int64)
    breaks = np.flatnonzero(np.diff(uniq) != 1) + 1
    for a, z in zip(np.concatenate([[0], breaks]), np.concatenate([breaks, [len(uniq)]])):
        read_exact(fd, out[int(at[a]):int(at[z])], int(start[uniq[a]]), fmt)
    return at


def upload(dev, n_chunks: int, capacity: int, stage, consume) -> None:
    """Move ``n_chunks`` chunks of at most ``capacity`` bytes to ``dev``: ``stage(c, host)`` fills the pinned uint8
    array ``host`` with chunk ``c`` and returns the bytes it used, ``consume(c, buf)`` enqueues the work on them, the
    uint8 device tensor ``buf``, on the current stream.  Two pinned and two device buffers: a chunk is staged while
    the one before it copies and decodes.  Each buffer has 16 bytes past ``capacity``, so a kernel that loads 16-byte
    words stays inside it."""
    n_buf = min(2, n_chunks)
    pinned = [torch.empty(capacity + 16, dtype=torch.uint8, pin_memory=True) for _ in range(n_buf)]
    devb = [torch.empty(capacity + 16, dtype=torch.uint8, device=dev) for _ in range(n_buf)]
    copied = [None] * n_buf
    stream = torch.cuda.current_stream(dev)
    for c in range(n_chunks):
        i = c % n_buf
        if copied[i] is not None:
            copied[i].synchronize()  # the upload out of pinned[i] has left the host buffer
        used = stage(c, pinned[i].numpy())
        devb[i][:used].copy_(pinned[i][:used], non_blocking=True)
        copied[i] = torch.cuda.Event()
        copied[i].record(stream)
        consume(c, devb[i][:used])


def host(v):
    """``v`` (None, a tensor anywhere or anything numpy takes) as a numpy array"""
    return None if v is None else np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v)


def writer_coords(coords, caller: str):
    """A writer's ``coords`` before its checks: a tensor must be a float32 CUDA tensor and is used where it is
    (``caller`` names the writer in the error); anything else becomes a float32 numpy array, uploaded by
    :func:`on_device` once every check has passed."""
    if isinstance(coords, torch.Tensor):
        _lib.tensor_device(coords, caller)
        if coords.dtype != torch.float32:
            raise ValueError(f"coords must be float32, got {coords.dtype}")
        return coords
    return np.asarray(coords, dtype=np.float32)


def on_device(a, device):
    """``a`` (None passes) as a CUDA tensor: a tensor as it is, anything else uploaded to ``device`` as float32"""
    if a is None or isinstance(a, torch.Tensor):
        return a
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(_lib.device(device))


def frame_minor(coords: torch.Tensor) -> torch.Tensor:
    """``coords`` as it is when it is (natoms, 3, F) frame-minor (a frame slice included), else a contiguous copy"""
    N, _, F = coords.shape
    s_atom, s_axis, s_frame = coords.stride()
    if N and F and not (s_atom == 3 * s_axis and (F == 1 or s_frame == 1) and s_axis >= F):
        coords = coords.contiguous()
    return coords


def write_encoded(fh, dev, n_frames: int, frame_bytes: int, chunk_bytes: int, encode) -> None:
    """Write ``n_frames`` records of ``frame_bytes`` each (at most, for records of variable size) to ``fh``, encoded on
    ``dev`` in chunks of at most ``chunk_bytes`` (one frame at least): ``encode(f0, f1, out)`` enqueues frames [f0, f1)
    into the uint8 device buffer ``out`` on the current stream; an int it returns is the bytes it wrote, anything else
    means the records fill (f1 - f0) * frame_bytes bytes.  Two device and two pinned buffers: each chunk is copied to the host and
    written while the next one encodes."""
    S = frame_bytes
    per = max(1, min(n_frames, int(chunk_bytes) // S))
    spans = [(f0, min(n_frames, f0 + per)) for f0 in range(0, n_frames, per)]
    n_buf = min(2, len(spans))
    devb = [torch.empty(per * S, dtype=torch.uint8, device=dev) for _ in range(n_buf)]
    host = [torch.empty(per * S, dtype=torch.uint8, pin_memory=True) for _ in range(n_buf)]
    done = [None] * n_buf
    stream = torch.cuda.current_stream(dev)
    pending = None  # (buffer, bytes) copied to the host but not yet written
    for c, (f0, f1) in enumerate(spans):
        i = c % n_buf
        used = encode(f0, f1, devb[i])
        nbytes = used if isinstance(used, int) else (f1 - f0) * S
        host[i][:nbytes].copy_(devb[i][:nbytes], non_blocking=True)
        done[i] = torch.cuda.Event()
        done[i].record(stream)
        if pending is not None:  # write the previous chunk while this one encodes and copies
            j, nb = pending
            done[j].synchronize()
            fh.write(memoryview(host[j].numpy())[:nb])
        pending = (i, nbytes)
    j, nb = pending
    done[j].synchronize()
    fh.write(memoryview(host[j].numpy())[:nb])
