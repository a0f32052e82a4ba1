"""Host plumbing shared by the trajectory file modules that decode and encode frames on the device (``dcd``,
``netcdf``, ``trr``, ``mdcrd``, ``xyz``, ``pdb``, ``gro``, ``cif``, ``bcif``, ``lammpstrj``): the text files' line
lookups, the frame selection, the chunk planner of a frame list, the slab gather and the whole-frame stager into
staging buffers, the double-buffered read -> copy -> decode loop and the staged-frame read on top of it, the readback of
the lines a decode left to the host, the decode outputs' check, the writers' coords intake and writable-range search,
the frame-minor layout check, and the double-buffered encode -> copy -> write loop."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import _lib

IOV_MAX = 1024  # buffers per preadv call (Linux)
PREADV_BYTES = 1 << 30  # slab bytes per preadv call, well below the 2 GiB a single read returns at most
WS = b" \t\n\v\f\r\x1c\x1d\x1e\x1f"  # the ASCII bytes str.split() splits on


def name(filename) -> str:
    """a file name given as str, bytes (UTF-8) or a path, as str"""
    return filename.decode("UTF-8") if isinstance(filename, bytes) else str(filename)


def content_end(fd: int, size: int) -> int:
    """one past the last byte of the ``size``-byte file that is not ASCII whitespace (0 for a blank file)"""
    end, step = size, 1 << 16
    while end > 0:
        lo = max(0, end - step)
        tail = os.pread(fd, end - lo, lo).rstrip(WS)
        if tail:
            return lo + len(tail)
        end = lo
    return 0


def line_at(fd: int, pos: int, end: int) -> bytes:
    """the bytes of the line starting at file offset ``pos``, without its '\\n' (not past ``end``)"""
    out, step = b"", 4096
    while pos < end:
        b = os.pread(fd, min(step, end - pos), pos)
        if not b:
            break
        i = b.find(b"\n")
        if i >= 0:
            return out + b[:i]
        out += b
        pos += len(b)
        step *= 2
    return out


def line_col(fd: int, pos: int) -> tuple[int, int]:
    """0-based line and 1-based column of file offset ``pos`` (counts the newlines before it)"""
    lines, last, step = 0, -1, 64 << 20
    for w in range(0, pos, step):
        b = np.frombuffer(os.pread(fd, min(step, pos - w), w), np.uint8)
        nl = np.flatnonzero(b == 10)
        lines += len(nl)
        if len(nl):
            last = w + int(nl[-1])
    return lines, pos - last


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
    """Read the whole frames ``uniq`` (ascending; frame j is the ``size[j]`` bytes at file offset ``start[j]``) back to
    back into ``out``, a run of frames that touch in the file in one read.  Returns the staging offsets: frame uniq[k]
    lands at [at[k], at[k + 1]).  A short read raises RuntimeError as :func:`read_exact` does."""
    at = np.concatenate([[0], np.cumsum(size[uniq])]).astype(np.int64)
    breaks = np.flatnonzero(start[uniq[1:]] != start[uniq[:-1]] + size[uniq[:-1]]) + 1
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


def read_frames(fd: int, dev, sel: np.ndarray, start: np.ndarray, size: np.ndarray, chunk_bytes: int, fmt: str,
                decode) -> list:
    """Move the listed frames ``sel`` (frame j is the ``size[j]`` bytes at file offset ``start[j]``) to ``dev`` whole,
    in chunks whose distinct frames take at most ``chunk_bytes``, through :func:`upload`.  ``decode(buf, at, frame_of,
    k0, k1)`` enqueues the work on each chunk: ``buf`` holds the chunk's distinct frames staged by
    :func:`stage_frames`, ``at`` their staging offsets, and ``frame_of`` the staged frame of each listed frame k0 ...
    k1 - 1.  Returns the chunks, as :func:`chunks` plans them."""
    plan = chunks(sel, size, int(chunk_bytes))
    staged = {}

    def stage(c, host):
        staged[c] = stage_frames(fd, start, size, plan[c][2], host, fmt)
        return int(staged[c][-1])

    def consume(c, buf):
        k0, k1, uniq = plan[c]
        decode(buf, staged.pop(c), np.searchsorted(uniq, sel[k0:k1]), k0, k1)

    upload(dev, len(plan), max(int(size[u].sum()) for _, _, u in plan), stage, consume)
    return plan


def flagged(flags: torch.Tensor, n: int, natoms: int, flag_cap: int, width: int):
    """The atom lines a decode pass left to the host, from its ``flags`` (flags[0] counts them; entry j, ``width``
    int64 at 1 + width * j, starts with k * natoms + a for the first ``flag_cap``) -> (k, a, rel): each line's listed
    frame k and atom a, and with ``width`` 2 the entry's second value, the line's byte offset from its frame's start
    (None otherwise).  Past ``flag_cap`` lines they are every atom line of the ``n`` listed frames, and rel is None."""
    n_host = int(flags[0].item())
    if n_host > flag_cap:  # too many to list: every atom line of the listed frames
        k, a = np.divmod(np.arange(n * natoms, dtype=np.int64), natoms)
        return k, a, None
    ent = flags[1:1 + width * n_host].view(n_host, width).cpu().numpy()
    k, a = np.divmod(ent[:, 0], natoms)
    return k, a, ent[:, 1] if width == 2 else None


def _minor(N: int, F: int, stride) -> bool:
    """whether an (N, 3, F) tensor of ``stride`` is frame-minor: contiguous, or a frame slice of a contiguous one"""
    s_atom, s_axis, s_frame = stride
    return N == 0 or F == 0 or (s_atom == 3 * s_axis and (F == 1 or s_frame == 1) and s_axis >= F)


def decode_outputs(dev, natoms: int, F: int, *outs) -> int:
    """Assert that the decode outputs ``outs`` (None skipped) are (natoms, 3, F) float32 tensors on ``dev``,
    frame-minor, with one axis stride; returns the frame stride the entry point takes (F for no output)."""
    outs = [t for t in outs if t is not None]
    for t in outs:
        assert t.shape == (natoms, 3, F) and t.dtype == torch.float32 and t.device == dev
        assert _minor(natoms, F, t.stride()), \
            "out must be (natoms, 3, F) frame-minor (a frame slice of a contiguous tensor is fine)"
    axis = {int(t.stride(1)) for t in outs}
    assert not (natoms and F) or len(axis) <= 1, "the outputs must share one frame stride"
    return max(axis.pop() if axis else F, F, 1)


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
    if not _minor(N, F, coords.stride()):
        coords = coords.contiguous()
    return coords


def first_bad(a, lo: int, hi: int, scale: float):
    """the first (frame, atom-or-None, axis, value) of (natoms, 3, F) or (3, F) ``a`` (a tensor or a numpy array) in
    file order with rint(x * scale) outside [lo, hi] or not finite, else None; one min / max pass when every value is
    inside"""
    if a.numel() == 0 if isinstance(a, torch.Tensor) else a.size == 0:
        return None
    if isinstance(a, torch.Tensor):
        mn, mx = (float(v) for v in torch.stack(torch.aminmax(a)).cpu())
    else:
        with np.errstate(invalid="ignore"):
            mn, mx = a.min(), a.max()
    if np.rint(np.float64(mn) * scale) >= lo and np.rint(np.float64(mx) * scale) <= hi:
        return None
    x = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    with np.errstate(invalid="ignore", over="ignore"):
        k = np.rint(x.astype(np.float64) * scale)
        bad = ~((k >= lo) & (k <= hi))
    if x.ndim == 3:
        f, atom, axis = np.unravel_index(np.argmax(bad.transpose(2, 0, 1)), (x.shape[2], x.shape[0], 3))
        return int(f), int(atom), int(axis), float(x[atom, axis, f])
    f, axis = np.unravel_index(np.argmax(bad.T), (x.shape[1], 3))
    return int(f), None, int(axis), float(x[axis, f])


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
