"""Host plumbing shared by the trajectory file modules that transpose frame records on the device (``dcd``, ``netcdf``):
the chunk planner of a frame list, the frame-minor layout check, and the double-buffered encode -> copy -> write loop."""
from __future__ import annotations

import numpy as np
import torch


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
