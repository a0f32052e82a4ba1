"""Multi-GPU sharding of the two embarrassingly parallel axes of the hot path (SURVEY.md section 8e).

  occupancy : molecules / pockets of a batch are independent  -> contiguous blocks of the batch per rank
  distances : trajectory frames are independent               -> contiguous frame blocks per rank

One process per GPU (torch.distributed, NCCL on GPUs, gloo in the CPU tests).  The data path has NO collective:
every rank voxelises / projects its own shard and keeps the result resident.  A collective (all_gather of row
blocks) runs only when the caller asks for the assembled array on every rank -- and for grids that gather costs
~30x the compute (8e), so the default is to leave shards where they are.
"""
from __future__ import annotations

import os
from typing import Callable, Sequence

import numpy as np
import torch
import torch.distributed as dist


def partition(n_items: int, world: int) -> np.ndarray:
    """Offsets (world+1,) of contiguous, size-balanced blocks: block r = [off[r], off[r+1])."""
    base, rem = divmod(int(n_items), int(world))
    sizes = np.full(world, base, dtype=np.int64)
    sizes[:rem] += 1
    off = np.zeros(world + 1, dtype=np.int64)
    np.cumsum(sizes, out=off[1:])
    return off


def balanced_partition(costs: Sequence[float], world: int) -> np.ndarray:
    """Contiguous partition of items with per-item costs (e.g. voxels or atoms x hits) into `world` blocks with
    near-equal cost: cut where the running cost crosses k/world of the total.  Returns offsets (world+1,)."""
    c = np.asarray(costs, dtype=np.float64)
    n = len(c)
    off = np.zeros(world + 1, dtype=np.int64)
    off[-1] = n
    if n == 0:
        return off
    cum = np.cumsum(c)
    total = cum[-1]
    for r in range(1, world):
        if total <= 0:
            off[r] = partition(n, world)[r]
        else:
            off[r] = int(np.searchsorted(cum, total * r / world, side="left") + 1)
        off[r] = min(max(off[r], off[r - 1]), n)
    return off


def bind_to_gpu_numa(index: int):
    """Pin this process to the CPUs next to GPU ``index`` (NVML affinity mask).  Call it before the first pinned buffer is
    allocated (``tools.voxeldescriptors.pinned_array``), so the page-locked memory is first touched on the GPU's NUMA node:
    a result on the other socket makes every device-to-host copy cross the socket link.
    Returns a one-line description of what was done ("unbound ..." when NVML or the affinity call is unavailable)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (os.cpu_count() + 63) // 64)
        cpus = {64 * i + b for i, w in enumerate(words) for b in range(64) if (w >> b) & 1}
        cur = os.sched_getaffinity(0)
        want = cpus & cur
        if want:
            os.sched_setaffinity(0, want)
            return f"{len(want)} CPUs near GPU {index}"
    except Exception as e:  # NVML missing or affinity not permitted: run unbound
        return f"unbound ({type(e).__name__})"
    return "unbound"


def world_info(group=None) -> tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def gather_rows(local: torch.Tensor, counts: Sequence[int], group=None) -> torch.Tensor:
    """Assemble row blocks from all ranks: rank r contributes `local` with counts[r] rows (same trailing shape).
    Implemented as one all_gather of blocks padded to the largest count (NCCL and gloo both support it); equal
    shards -- the common case -- have no padding.  Returns the concatenated tensor on every rank."""
    world, rank = world_info(group)
    if world == 1:
        return local
    counts = [int(c) for c in counts]
    assert local.shape[0] == counts[rank], (local.shape, counts, rank)
    mx = max(counts)
    if local.shape[0] < mx:
        pad = torch.zeros((mx - local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        local = torch.cat([local, pad], dim=0)
    local = local.contiguous()
    bufs = [torch.empty_like(local) for _ in range(world)]
    dist.all_gather(bufs, local, group=group)
    return torch.cat([b[:c] for b, c in zip(bufs, counts)], dim=0)


def run_sharded(n_items: int, compute_fn: Callable[[int, int], torch.Tensor], *, rows_per_item=None, gather: bool = False,
                costs: Sequence[float] | None = None, group=None):
    """Run `compute_fn(begin, end)` on this rank's contiguous block of `n_items` independent items.

    Returns (local_result, (begin, end)) or, with gather=True, (assembled_result, (0, n_items)).  `rows_per_item`
    (scalar or per-item array) says how many result rows each item produces, needed only for the gather."""
    world, rank = world_info(group)
    off = balanced_partition(costs, world) if costs is not None else partition(n_items, world)
    b, e = int(off[rank]), int(off[rank + 1])
    local = compute_fn(b, e)
    if not gather or world == 1:
        return local, (b, e)
    if rows_per_item is None:
        rows_per_item = 1
    rpi = np.broadcast_to(np.asarray(rows_per_item, dtype=np.int64), (n_items,))
    cum = np.concatenate([[0], np.cumsum(rpi)])
    counts = [int(cum[off[r + 1]] - cum[off[r]]) for r in range(world)]
    return gather_rows(local, counts, group=group), (0, n_items)


# ------------------------------------------------------------------------------------------- product wrappers
def voxelize_sharded(coords, channels, *, boxsize=None, centers=None, buffer=0.0, voxelsize=1.0, device=None,
                     gather: bool = False, group=None):
    """Voxelise a batch (lists of per-item coords / sigma channels) across the ranks of `group`.

    Returns (features float32 CUDA tensor, voxel offsets, (begin, end)): this rank's shard by default; with
    gather=True the whole batch's (sum M, C) tensor on every rank (NCCL all_gather over NVLink)."""
    from .tools.voxeldescriptors import VoxelBatch

    n = len(coords)
    holder = {}

    def compute(b, e):
        ctr = None if centers is None else np.asarray(centers)[b:e]
        vb = VoxelBatch(coords[b:e], channels[b:e], boxsize=boxsize, centers=ctr, buffer=buffer, voxelsize=voxelsize)
        d_c, d_s = vb.to_device(device)
        holder["vb"] = vb
        return vb.run(d_c, d_s)

    costs = [len(c) for c in coords]
    if gather:
        # rows per item must be known on every rank: compute the grid sizes of the whole batch on the host
        full = VoxelBatch(coords, channels, boxsize=boxsize, centers=centers, buffer=buffer, voxelsize=voxelsize)
        rows = np.diff(full.out_offsets)
        out, rng = run_sharded(n, compute, rows_per_item=rows, gather=True, costs=costs, group=group)
        return out, full.out_offsets, rng
    out, rng = run_sharded(n, compute, costs=costs, group=group)
    return out, holder["vb"].out_offsets, rng


def project_sharded(projection, mol, *, gather: bool = True, group=None):
    """Project a trajectory with frames split across ranks (MetricDistance.project on each frame block).

    Returns the (F, P) numpy array on every rank when gather=True, else this rank's rows and its (f0, f1)."""
    world, rank = world_info(group)
    F = mol.numFrames
    off = partition(F, world)
    f0, f1 = int(off[rank]), int(off[rank + 1])
    view = mol.copy() if world == 1 else _frame_view(mol, f0, f1)
    local = projection.project(view)
    if not gather or world == 1:
        return (local, (f0, f1)) if not gather else local
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    t = torch.from_numpy(np.ascontiguousarray(local)).to(dev)
    if t.dtype == torch.bool:
        t = t.to(torch.uint8)
    full = gather_rows(t, [int(off[r + 1] - off[r]) for r in range(world)], group=group)
    res = full.cpu().numpy()
    return res.astype(bool) if local.dtype == bool else res


def wrap_sharded(mol, *, gather: bool = True, group=None, wrap_fn=None, **wrap_kwargs):
    """Molecule.wrap (moleculekit/molecule.py:1987-2090) with the frames split across ranks: frames are independent
    (wrapping.pyx loops over them outermost), so every rank wraps its block with `wrapping.wrap` (orthorhombic K9 or the
    triclinic K9b kernels, chosen by the box angles) and no data-path collective is needed.  gather=True leaves the fully
    wrapped (N, 3, F) array in ``mol.coords`` on every rank (all_gather of the (F_r, 3N) row blocks); gather=False wraps
    only this rank's frames of ``mol.coords`` in place and returns (f0, f1).  ``wrap_fn(view, **kwargs)`` defaults to
    `moleculekit_b200.wrapping.wrap` (the gloo tests pass a CPU stand-in)."""
    if wrap_fn is None:
        from .wrapping import wrap as wrap_fn
    world, rank = world_info(group)
    F = mol.coords.shape[2]
    off = partition(F, world)
    f0, f1 = int(off[rank]), int(off[rank + 1])
    view = _frame_view(mol, f0, f1)
    for name in ("boxangles", "boxvectors"):  # per-frame cell data follows the frames
        a = getattr(mol, name, None)
        if isinstance(a, np.ndarray) and a.shape[-1] == F:
            try:
                setattr(view, name, np.ascontiguousarray(a[..., f0:f1]))
            except AttributeError:  # a read-only property derived from box / boxangles
                pass
    if f1 > f0:
        wrap_fn(view, **wrap_kwargs)
    mol.coords[:, :, f0:f1] = view.coords
    if not gather or world == 1:
        return (f0, f1)
    N = mol.coords.shape[0]
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    rows = torch.from_numpy(np.ascontiguousarray(np.moveaxis(view.coords, 2, 0)).reshape(f1 - f0, 3 * N)).to(dev)
    full = gather_rows(rows, [int(off[r + 1] - off[r]) for r in range(world)], group=group)
    mol.coords[...] = np.moveaxis(full.cpu().numpy().reshape(F, N, 3), 0, 2)
    return (0, F)


def hbonds_sharded(mol, donors, acceptors, sel1="all", sel2=None, *, gather: bool = True, group=None, hbonds_fn=None,
                   **hb_kwargs):
    """hbonds_calculate (moleculekit/interactions/interactions.py:365-467) with the frames split across ranks.  Returns the
    per-frame list of (n, 3) arrays for all frames on every rank (gather=True; the ragged lists travel with
    all_gather_object, they are small) or this rank's frames and (f0, f1).  ``hbonds_fn`` defaults to
    `moleculekit_b200.interactions.hbonds_calculate`."""
    import torch.distributed as dist

    if hbonds_fn is None:
        from .interactions import hbonds_calculate as hbonds_fn
    world, rank = world_info(group)
    F = mol.coords.shape[2]
    off = partition(F, world)
    f0, f1 = int(off[rank]), int(off[rank + 1])
    view = _frame_view(mol, f0, f1)
    if hasattr(view, "numFrames") and not isinstance(getattr(type(view), "numFrames", None), property):
        view.numFrames = f1 - f0
    local = hbonds_fn(view, donors, acceptors, sel1, sel2, **hb_kwargs) if f1 > f0 else []
    if not gather or world == 1:
        return (local, (f0, f1)) if not gather else local
    parts = [None] * world
    dist.all_gather_object(parts, local, group=group)
    return [fr for part in parts for fr in part]


def _frame_view(mol, f0: int, f1: int):
    """A shallow copy of `mol` restricted to frames [f0, f1) (coords / box sliced, topology shared)."""
    import copy

    v = copy.copy(mol)
    v.coords = np.ascontiguousarray(mol.coords[:, :, f0:f1])
    v.box = np.ascontiguousarray(mol.box[:, f0:f1]) if mol.box is not None and mol.box.shape[1] == mol.coords.shape[2] \
        else mol.box
    return v
