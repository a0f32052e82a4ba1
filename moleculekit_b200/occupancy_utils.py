"""Host side of the occupancy kernels: mirror of ``moleculekit.occupancy_utils`` over libmkb200.

``calculate_occupancy(centers, coords, sigmas, results)`` keeps the reference's signature and in-place
max-accumulate contract (moleculekit/occupancy_utils/occupancy_utils.pyx:34-61); the batched regular-grid entry
points are what ``tools.voxeldescriptors`` and the benchmark drive.  PyTorch is only the device container.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

MAX_CHANNELS_PER_CALL = 32
# Channel sigmas with 0 < |sigma| < SIGMA_EXACT (Angstrom) are evaluated with the reference's float64 operations by the
# points kernel (SIGMA_EXACT in csrc/occupancy.cu, DESIGN.md K1b): there the reference's own 1 - exp(-x^12) is quantised
# to multiples of 2^-53, which no float32 evaluation reproduces.
SIGMA_EXACT = 0.7


def make_grid_descs(origins, voxelsizes, dims, atom_offsets, out_offsets=None) -> tuple[np.ndarray, np.ndarray]:
    """Pack per-grid descriptors (``mkb_grid_desc``) for a batch.

    origins (B,3) f64: centre of voxel (0,0,0); voxelsizes (B,) or scalar; dims (B,3) int; atom_offsets (B+1,)
    (grid b owns atom rows [off[b], off[b+1])) or a (B,2) array of explicit [begin, end) ranges.
    Returns (descs, out_offsets (B+1,) in voxels)."""
    origins = np.atleast_2d(np.asarray(origins, dtype=np.float64))
    B = origins.shape[0]
    dims = np.atleast_2d(np.asarray(dims)).astype(np.int64)
    vs = np.broadcast_to(np.asarray(voxelsizes, dtype=np.float64), (B,))
    ao = np.asarray(atom_offsets, dtype=np.int64)
    if ao.ndim == 1:
        begin, end = ao[:-1], ao[1:]
    else:
        begin, end = ao[:, 0], ao[:, 1]
    nvox = dims.prod(axis=1)
    if out_offsets is None:
        out_offsets = np.zeros(B + 1, dtype=np.int64)
        np.cumsum(nvox, out=out_offsets[1:])
    out_offsets = np.asarray(out_offsets, dtype=np.int64)
    d = np.zeros(B, dtype=_lib.GRID_DESC)
    d["origin"] = origins
    d["voxelsize"] = vs
    d["dims"] = dims
    d["atom_begin"] = begin
    d["atom_end"] = end
    d["out_offset"] = out_offsets[:B]
    return d, out_offsets


def _layout_flag(layout: str) -> int:
    if layout == "xyzc":
        return 0
    if layout == "cxyz":
        return _lib.OCC_LAYOUT_CXYZ
    raise ValueError("layout must be 'xyzc' (the reference's voxel-major order) or 'cxyz' (channel-major)")


def split_small_sigmas(sigmas: torch.Tensor | None, radii: torch.Tensor | None = None, chanmask: torch.Tensor | None = None,
                       n_channels: int | None = None):
    """None when no channel entry has 0 < |sigma| < SIGMA_EXACT; else (the sigmas -- or radii -- with those entries zeroed,
    for the grid kernels; an (N, C) float64 matrix holding only those entries).  With bit-mask channels a small radius
    moves the whole atom.  Reads one flag back to the host (synchronises torch's current stream)."""
    if sigmas is not None:
        small = (sigmas != 0) & (sigmas.abs() < SIGMA_EXACT)
        if not bool(small.any()):
            return None
        return sigmas.masked_fill(small, 0.0), torch.where(small, sigmas, torch.zeros_like(sigmas))
    Cn = int(n_channels)
    bits = ((chanmask[:, None] >> torch.arange(Cn, device=chanmask.device, dtype=torch.int32)) & 1).bool()
    atom = (radii != 0) & (radii.abs() < SIGMA_EXACT) & bits.any(dim=1)
    if not bool(atom.any()):
        return None
    small = bits & atom[:, None]
    return radii.masked_fill(atom, 0.0), torch.where(small, radii[:, None].expand(-1, Cn), torch.zeros((), dtype=radii.dtype, device=radii.device))


def _merge_small_sigmas(coords: torch.Tensor, small: torch.Tensor, descs: np.ndarray, out: torch.Tensor, layout: str) -> None:
    """Max-merge the float64 small-sigma values (points kernel on each grid's centres and own atoms) into the grid output;
    entries no small-sigma atom reaches keep their bits."""
    Cn = int(small.shape[1])
    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    has = np.concatenate([[0], np.cumsum(small.ne(0).any(dim=1).cpu().numpy())])
    flat = out.view(-1)
    for b in range(len(descs)):
        d = descs[b:b + 1].copy()
        a0, a1 = int(d["atom_begin"][0]), int(d["atom_end"][0])
        if has[a1] == has[a0]:
            continue
        M = int(np.prod(d["dims"][0]))
        o = int(d["out_offset"][0]) * Cn
        d["out_offset"] = 0
        val = torch.full((M, Cn), float("-inf"), dtype=torch.float32, device=out.device)
        occupancy_points(grid_centers(d, out.device), coords[a0:a1], small[a0:a1].contiguous(), val, accumulate=True)
        g = flat[o:o + M * Cn].view(M, Cn) if layout == "xyzc" else flat[o:o + M * Cn].view(Cn, M).t()
        g.copy_(torch.where(val > g, val, g))


def occupancy_grid_batch(coords: torch.Tensor, sigmas: torch.Tensor | None, descs: np.ndarray, out: torch.Tensor,
                         accumulate: bool = False, layout: str = "xyzc", radii: torch.Tensor | None = None,
                         chanmask: torch.Tensor | None = None, n_channels: int | None = None,
                         small_sigmas: bool | None = None) -> torch.Tensor:
    """Launch K2+K1 for a batch of regular grids.  coords (N,3) f32 cuda, out (sum M_b * C) f32 cuda (written in place),
    channels either as ``sigmas`` (N,C) f64 cuda -- the reference's matrix -- or, assembled on the device, as ``radii``
    (N,) f64 + ``chanmask`` (N,) int32 bit masks with ``n_channels`` (SURVEY 8f row 1).  ``layout="cxyz"`` stores every grid
    channel-major, [C][nx][ny][nz].  Stream-ordered on torch's current stream.

    Channel entries with 0 < |sigma| < SIGMA_EXACT are zeroed in the copy the grid kernels see and evaluated in float64 by
    the points kernel on the grid centres, then max-merged.  ``small_sigmas=False`` is the caller's word that there are
    none (no check, no host synchronisation: the batch takes the grid kernels alone); None checks on the device."""
    split = None
    if small_sigmas is not False:
        split = split_small_sigmas(sigmas, radii, chanmask, n_channels if sigmas is None else None)
    if split is not None:
        fast, small = split
        if sigmas is not None:
            occupancy_grid_batch(coords, fast, descs, out, accumulate, layout, small_sigmas=False)
        else:
            occupancy_grid_batch(coords, None, descs, out, accumulate, layout, radii=fast, chanmask=chanmask,
                                 n_channels=n_channels, small_sigmas=False)
        _merge_small_sigmas(coords, small, descs, out, layout)
        return out
    dev = out.device
    assert coords.is_cuda and out.is_cuda and coords.device == dev
    assert coords.dtype == torch.float32 and out.dtype == torch.float32
    assert coords.is_contiguous() and out.is_contiguous() and coords.ndim == 2 and coords.shape[1] == 3
    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    flags = (_lib.OCC_ACCUMULATE if accumulate else 0) | _layout_flag(layout)
    if sigmas is not None:
        assert sigmas.is_cuda and sigmas.device == dev and sigmas.dtype == torch.float64 and sigmas.is_contiguous()
        assert sigmas.ndim == 2 and sigmas.shape[0] == coords.shape[0]
        Cn = int(sigmas.shape[1])
    else:
        assert radii is not None and chanmask is not None and n_channels is not None
        assert radii.is_cuda and chanmask.is_cuda and radii.dtype == torch.float64 and chanmask.dtype == torch.int32
        assert radii.is_contiguous() and chanmask.is_contiguous()
        assert radii.shape == (coords.shape[0],) and chanmask.shape == (coords.shape[0],)
        Cn = int(n_channels)
    if Cn > MAX_CHANNELS_PER_CALL:
        raise ValueError(f"at most {MAX_CHANNELS_PER_CALL} channels per call; split the channel set")
    if sigmas is not None:
        _lib.call(dev, "mkb_occupancy_grid_batch", _lib.ptr(coords), _lib.ptr(sigmas), int(coords.shape[0]), Cn,
                  descs.ctypes.data_as(C.c_void_p), int(descs.shape[0]), _lib.ptr(out), flags)
    else:
        _lib.call(dev, "mkb_occupancy_grid_batch_masked", _lib.ptr(coords), _lib.ptr(radii), _lib.ptr(chanmask),
                  int(coords.shape[0]), Cn, descs.ctypes.data_as(C.c_void_p), int(descs.shape[0]), _lib.ptr(out), flags)
    return out


def occupancy_grid_batch_compact(coords: torch.Tensor, sigmas: torch.Tensor | None, descs: np.ndarray,
                                 radii: torch.Tensor | None = None, chanmask: torch.Tensor | None = None,
                                 records: torch.Tensor | None = None, blk_rank: torch.Tensor | None = None,
                                 small_sigmas: bool | None = None):
    """K2+K1 with the compact result of ``mkb_occupancy_grid_batch_compact`` (8 channels): returns (records, blk_rank),
    ``records`` float32 cuda with one 4 KB row [4 x][4 y][8 z][8 ch] per 4x4x8-voxel block that has an atom within 5 A
    (room for every block of the batch; only the first blk_rank[-1] rows are written) and ``blk_rank`` int32 (blocks + 1,)
    the exclusive count of such blocks.  :func:`expand_compact_host` rebuilds the dense host array."""
    if small_sigmas is not False and split_small_sigmas(sigmas, radii, chanmask, 8 if sigmas is None else None) is not None:
        raise _lib.MkbUnsupported("channel sigmas below SIGMA_EXACT need the dense route (occupancy_grid_batch)")
    dev = coords.device
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.is_contiguous() and coords.ndim == 2
    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    lib = _lib.load()
    nblk = int(lib.mkb_occupancy_compact_blocks(descs.ctypes.data_as(C.c_void_p), int(descs.shape[0])))
    if records is None:
        records = torch.empty((nblk, 1024), dtype=torch.float32, device=dev)
    if blk_rank is None:
        blk_rank = torch.empty(nblk + 1, dtype=torch.int32, device=dev)
    assert records.is_cuda and records.dtype == torch.float32 and records.is_contiguous() and records.numel() >= nblk * 1024
    assert blk_rank.is_cuda and blk_rank.dtype == torch.int32 and blk_rank.numel() >= nblk + 1
    if sigmas is not None:
        assert sigmas.is_cuda and sigmas.dtype == torch.float64 and sigmas.is_contiguous() and sigmas.shape == (coords.shape[0], 8)
    else:
        assert radii is not None and chanmask is not None and radii.dtype == torch.float64 and chanmask.dtype == torch.int32
    masked = sigmas is None
    _lib.call(dev, "mkb_occupancy_grid_batch_compact", _lib.ptr(coords), _lib.ptr(sigmas),
              _lib.ptr(radii if masked else None), _lib.ptr(chanmask if masked else None), int(coords.shape[0]),
              descs.ctypes.data_as(C.c_void_p), int(descs.shape[0]), _lib.ptr(records), _lib.ptr(blk_rank),
              int(blk_rank.numel()))
    return records, blk_rank


def occupancy_grid_batch_to_host(coords: torch.Tensor, sigmas: torch.Tensor | None, descs: np.ndarray, out_host: torch.Tensor,
                                 radii: torch.Tensor | None = None, chanmask: torch.Tensor | None = None,
                                 small_sigmas: bool | None = None):
    """K2+K1 storing the non-empty 4x4x8 blocks straight into ``out_host`` -- a PINNED host float32 tensor (sum M, 8), device
    accessible under UVA -- while the block index travels to the host ahead of the fill kernel
    (``mkb_occupancy_grid_batch_to_host``).  Returns the pinned int32 index (blocks + 1,); call :func:`wait_index`, zero-fill
    the empty blocks with :func:`expand_compact_host` (``records=None``) and synchronise the stream before reading."""
    if small_sigmas is not False and split_small_sigmas(sigmas, radii, chanmask, 8 if sigmas is None else None) is not None:
        raise _lib.MkbUnsupported("channel sigmas below SIGMA_EXACT need the dense route (occupancy_grid_batch)")
    dev = coords.device
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.is_contiguous() and coords.ndim == 2
    assert not out_host.is_cuda and out_host.is_pinned() and out_host.dtype == torch.float32 and out_host.is_contiguous()
    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    lib = _lib.load()
    nblk = int(lib.mkb_occupancy_compact_blocks(descs.ctypes.data_as(C.c_void_p), int(descs.shape[0])))
    blk_rank = torch.empty(nblk + 1, dtype=torch.int32, device=dev)
    host_rank = torch.empty(nblk + 1, dtype=torch.int32, pin_memory=True)
    if sigmas is not None:
        assert sigmas.is_cuda and sigmas.dtype == torch.float64 and sigmas.is_contiguous() and sigmas.shape == (coords.shape[0], 8)
    else:
        assert radii is not None and chanmask is not None and radii.dtype == torch.float64 and chanmask.dtype == torch.int32
    masked = sigmas is None
    _lib.call(dev, "mkb_occupancy_grid_batch_to_host", _lib.ptr(coords), _lib.ptr(sigmas),
              _lib.ptr(radii if masked else None), _lib.ptr(chanmask if masked else None), int(coords.shape[0]),
              descs.ctypes.data_as(C.c_void_p), int(descs.shape[0]), _lib.ptr(out_host), _lib.ptr(blk_rank),
              int(blk_rank.numel()), _lib.ptr(host_rank))
    return host_rank, blk_rank


def wait_index(device) -> None:
    """Block until the block index of the last ``occupancy_grid_batch_to_host`` call on this device has reached the host."""
    h = _lib.handle(torch.device(device).index if not isinstance(device, int) else device)
    _lib.check(_lib.load().mkb_occupancy_wait_index(h), h)


def default_host_threads() -> int:
    """Host threads for the compact-transfer expansion: the CPUs this process may use, shared fairly between the ranks of a
    one-process-per-GPU job on this host (torchrun's LOCAL_WORLD_SIZE), at most 32 -- beyond that the expansion is bound
    by memory bandwidth, and 8 ranks x 32 threads oversubscribe a 128-thread host.
    ``MKB_HOST_THREADS`` overrides."""
    import os

    if os.environ.get("MKB_HOST_THREADS"):
        return max(1, int(os.environ["MKB_HOST_THREADS"]))
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    ranks = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", "1")))
    share = max(1, (os.cpu_count() or n) // ranks)
    return max(1, min(32, n, share))


def expand_compact_host(descs: np.ndarray, g0: int, g1: int, blk_rank: np.ndarray, records: np.ndarray, rec0: int,
                        out: np.ndarray, n_threads: int = 0) -> None:
    """Host half of the compact transfer (``mkb_occupancy_expand_host``): grids [g0, g1) of the dense float32 (sum M, 8)
    array ``out`` from the 4 KB block records (``records[0]`` is record ``rec0``; ``records=None`` only zero-fills the blocks
    that have no record).  Multi-threaded, releases the GIL."""
    import os

    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    assert blk_rank.dtype in (np.int32, np.uint32) and blk_rank.flags["C_CONTIGUOUS"]
    assert records is None or (records.dtype == np.float32 and records.flags["C_CONTIGUOUS"])
    assert out.flags["C_CONTIGUOUS"] and out.dtype in (np.float32, np.float64)
    if n_threads <= 0:
        n_threads = default_host_threads()
    rc = _lib.load().mkb_occupancy_expand_host(descs.ctypes.data_as(C.c_void_p), int(g0), int(g1), blk_rank.ctypes.data_as(C.c_void_p),
                                               records.ctypes.data_as(C.c_void_p) if records is not None else C.c_void_p(0), int(rec0), out.ctypes.data_as(C.c_void_p),
                                               1 if out.dtype == np.float64 else 0, int(n_threads))
    if rc != 0:
        raise ValueError("mkb_occupancy_expand_host: bad arguments")


def grid_centers(descs: np.ndarray, device=None) -> torch.Tensor:
    """Voxel centres of a batch of grids on the device: (sum M_b, 3) float64 cuda, bit-identical to getCenters."""
    dev = _lib.device(device)
    descs = np.ascontiguousarray(descs, dtype=_lib.GRID_DESC)
    total = int((descs["out_offset"] + descs["dims"].astype(np.int64).prod(axis=1)).max()) if len(descs) else 0
    out = torch.empty((total, 3), dtype=torch.float64, device=dev)
    _lib.call(dev, "mkb_grid_centers", descs.ctypes.data_as(C.c_void_p), int(descs.shape[0]), _lib.ptr(out))
    return out


def rotate_coords_device(coords: torch.Tensor, atom_offsets: torch.Tensor, matrices: torch.Tensor, centers: torch.Tensor,
                         out_dtype=torch.float32) -> torch.Tensor:
    """Batched rotateCoordinates on CUDA tensors: coords (N,3) f32, atom_offsets (B+1,) int64, matrices (B,3,3,3) f64
    (x, y, z rotation of every molecule), centers (B,3) f64 -> rotated (N,3) float32 or float64."""
    dev = coords.device
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.is_contiguous() and coords.shape[1] == 3
    assert atom_offsets.dtype == torch.int64 and matrices.dtype == torch.float64 and centers.dtype == torch.float64
    assert atom_offsets.is_contiguous() and matrices.is_contiguous() and centers.is_contiguous()
    B = int(atom_offsets.numel()) - 1
    assert matrices.shape == (B, 3, 3, 3) and centers.shape == (B, 3)
    out = torch.empty(coords.shape, dtype=out_dtype, device=dev)
    _lib.call(dev, "mkb_rotate_coords", _lib.ptr(coords), int(coords.shape[0]), _lib.ptr(atom_offsets), B,
              _lib.ptr(matrices), _lib.ptr(centers), _lib.ptr(out if out_dtype == torch.float32 else None),
              _lib.ptr(out if out_dtype == torch.float64 else None))
    return out


def occupancy_points(centers: torch.Tensor, coords: torch.Tensor, sigmas: torch.Tensor, out: torch.Tensor,
                     accumulate: bool = False) -> torch.Tensor:
    """K1b: arbitrary centres (M,3) f64 cuda -> out (M,C) f32 cuda."""
    dev = out.device
    assert centers.is_cuda and coords.is_cuda and sigmas.is_cuda and out.is_cuda
    assert centers.dtype == torch.float64 and coords.dtype == torch.float32 and sigmas.dtype == torch.float64
    assert out.dtype == torch.float32
    assert centers.is_contiguous() and coords.is_contiguous() and sigmas.is_contiguous() and out.is_contiguous()
    Cn = int(sigmas.shape[1])
    if Cn > MAX_CHANNELS_PER_CALL:
        raise ValueError(f"at most {MAX_CHANNELS_PER_CALL} channels per call; split the channel set")
    _lib.call(dev, "mkb_occupancy_points", _lib.ptr(centers), int(centers.shape[0]), _lib.ptr(coords), _lib.ptr(sigmas),
              int(coords.shape[0]), Cn, _lib.ptr(out), _lib.OCC_ACCUMULATE if accumulate else 0)
    return out


def _channel_chunks(C_total: int):
    for s in range(0, C_total, MAX_CHANNELS_PER_CALL):
        yield s, min(C_total, s + MAX_CHANNELS_PER_CALL)


def calculate_occupancy(centers, coords, sigmas, results, device=None) -> None:
    """Drop-in for ``moleculekit.occupancy_utils.calculate_occupancy`` (occupancy_utils.pyx:34-61).

    centers (M,3) f64, coords (N,3) f32, sigmas (N,C) f64, results (M,C) f64 **accumulated in place**
    (results = max(results, value), NaN never stored) -- same dtype errors as the Cython memoryviews."""
    for name, arr, dt, nd in (("centers", centers, np.float64, 2), ("coords", coords, np.float32, 2),
                              ("sigmas", sigmas, np.float64, 2), ("results", results, np.float64, 2)):
        if not isinstance(arr, np.ndarray) or arr.dtype != dt:
            raise ValueError(f"Buffer dtype mismatch, expected '{np.dtype(dt).name}' for {name}")
        if arr.ndim != nd:
            raise ValueError(f"Buffer has wrong number of dimensions (expected {nd}, got {arr.ndim})")
    M, N, Cn = centers.shape[0], coords.shape[0], sigmas.shape[1]
    if results.shape[0] < M or results.shape[1] < Cn:
        raise ValueError("results buffer too small")
    if M == 0 or Cn == 0:
        return
    dev = _lib.device(device)
    d_centers = torch.from_numpy(np.ascontiguousarray(centers)).to(dev)
    d_coords = torch.from_numpy(np.ascontiguousarray(coords)).to(dev)
    for c0, c1 in _channel_chunks(Cn):
        d_sig = torch.from_numpy(np.ascontiguousarray(sigmas[:, c0:c1])).to(dev)
        # -inf marks the entries no atom with a non-zero sigma reached: the reference leaves those untouched, whatever
        # `results` holds there (a negative prefill included)
        d_out = torch.full((M, c1 - c0), float("-inf"), dtype=torch.float32, device=dev)
        occupancy_points(d_centers, d_coords, d_sig, d_out, accumulate=True)
        val = d_out.cpu().numpy().astype(np.float64)
        old = results[:M, c0:c1]
        # reference update rule `value > old ? value : old` (NaN in `old` sticks, never produced by us)
        np.copyto(old, val, where=val > old)
