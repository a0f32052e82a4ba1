"""Host plumbing shared by the trajectory file modules that transpose frame records on the device (``dcd``, ``netcdf``,
``trr``): the chunk planner of a frame list, the slab gather into staging rows, the frame-minor layout check, and the
double-buffered encode -> copy -> write loop."""
from __future__ import annotations

import os

import numpy as np
import torch

IOV_MAX = 1024  # buffers per preadv call (Linux)
PREADV_BYTES = 1 << 30  # slab bytes per preadv call, well below the 2 GiB a single read returns at most


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


def frame_minor(coords: torch.Tensor) -> torch.Tensor:
    """``coords`` as it is when it is (natoms, 3, F) frame-minor (a frame slice included), else a contiguous copy"""
    N, _, F = coords.shape
    s_atom, s_axis, s_frame = coords.stride()
    if N and F and not (s_atom == 3 * s_axis and (F == 1 or s_frame == 1) and s_axis >= F):
        coords = coords.contiguous()
    return coords


def write_encoded(fh, dev, n_frames: int, frame_bytes: int, chunk_bytes: int, encode) -> None:
    """Write ``n_frames`` records of ``frame_bytes`` each to ``fh``, encoded on ``dev`` in chunks of at most
    ``chunk_bytes`` (one frame at least): ``encode(f0, f1, out)`` enqueues frames [f0, f1) into the uint8 device buffer
    ``out`` on the current stream.  Two device and two pinned buffers: each chunk is copied to the host and written
    while the next one encodes."""
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
        encode(f0, f1, devb[i])
        nbytes = (f1 - f0) * S
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
