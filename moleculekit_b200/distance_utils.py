"""Host side of the distance kernels: mirror of ``moleculekit.distance_utils`` over libmkb200.

Function names, argument order and in-place output contracts follow the reference's Cython module
(moleculekit/distance_utils/distance_utils.pyx); arrays are numpy on the host, moved to the GPU for the call
(only the selected atoms' rows travel).  ``*_device`` variants take CUDA tensors and leave results on the device.
Results are bit-identical to the reference binary (every float op individually rounded, see csrc/distance.cu).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _lib

_NAN = float("nan")


def n_columns(n1: int, n2: int, selfdist: bool) -> int:
    return (n1 * (n2 - 1)) // 2 if selfdist else n1 * n2


# ------------------------------------------------------------------------------------------------ device level
def dist_trajectory_device(coords, box, sel1, sel2, chains, selfdist: bool, pbc: bool, *, metric: str = "distances",
                           truncate: float | None = None, threshold: float = 8.0, out: torch.Tensor | None = None,
                           exact: bool = True):
    """K3 on CUDA tensors.  Returns (F, P) float32 distances or bool contacts (post-ops fused, util.py:74-84).
    ``exact=False`` (distances only): MKB_DIST_DISTANCES_FAST, within 4 ulp of the reference's float32 values instead of
    bit-identical (contact maps are always the reference's booleans)."""
    dev = coords.device
    F = coords.shape[2]
    P = n_columns(len(sel1), len(sel2), selfdist)
    mode = _lib.DIST_CONTACTS if metric == "contacts" else (_lib.DIST_DISTANCES if exact else _lib.DIST_DISTANCES_FAST)
    if out is None:
        out = torch.empty((F, P), dtype=torch.uint8 if mode == _lib.DIST_CONTACTS else torch.float32, device=dev)  # the kernel writes every element
    tr = _lib.traj(coords, box)
    _lib.call(dev, "mkb_dist_trajectory", C.byref(tr), _lib.ptr(sel1), len(sel1), _lib.ptr(sel2), len(sel2),
              _lib.ptr(chains), int(bool(selfdist)), int(bool(pbc)), mode, _NAN if truncate is None else float(truncate),
              float(threshold), _lib.ptr(out))
    return out.view(torch.bool) if mode == _lib.DIST_CONTACTS else out


def contacts_trajectory_device(coords, box, sel1, sel2, chains, selfdist: bool, pbc: bool, dist_threshold: float):
    """K4 on CUDA tensors.  Returns (frame_offsets (F+1,) int64 cuda, pairs (total, 2) uint32-as-int32 cuda)."""
    dev = coords.device
    F, n1 = coords.shape[2], len(sel1)
    tr = _lib.traj(coords, box)
    row_off = torch.empty(F * n1 + 1, dtype=torch.int64, device=dev)
    args = (C.byref(tr), _lib.ptr(sel1), n1, _lib.ptr(sel2), len(sel2), _lib.ptr(chains), int(bool(selfdist)),
            int(bool(pbc)), float(np.float32(dist_threshold)))
    (pairs,) = _lib.count_fill(dev, "mkb_contacts_count", "mkb_contacts_fill", args, row_off,
                               lambda total: (torch.empty((total, 2), dtype=torch.int32, device=dev),))
    frame_off = row_off[::n1] if n1 > 0 else torch.zeros(F + 1, dtype=torch.int64, device=dev)
    return frame_off.contiguous(), pairs


def shell_counts_device(coords, box, sel1, sel2, chains, selfdist: bool, pbc: bool, edges, truncate=None):
    """K8 on CUDA tensors: (F, n1, numshells) int32 counts of sel2 partners per radial shell around each sel1 atom."""
    dev = coords.device
    F, n1 = coords.shape[2], len(sel1)
    numshells = int(edges.shape[0]) - 1
    counts = torch.zeros((F, n1, numshells), dtype=torch.int32, device=dev)
    tr = _lib.traj(coords, box)
    _lib.call(dev, "mkb_shell_counts", C.byref(tr), _lib.ptr(sel1), n1, _lib.ptr(sel2), len(sel2), _lib.ptr(chains),
              int(bool(selfdist)), int(bool(pbc)), _NAN if truncate is None else float(truncate), _lib.ptr(edges),
              numshells, _lib.ptr(counts))
    return counts


def shell_counts(coords, box, sel1, sel2, digitized_chains, selfdist, pbc, edges, truncate=None, device=None):
    """Host form of K8: numpy in, (F, n1, numshells) int64 counts out."""
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    _check("sel1", sel1, np.uint32, 1); _check("sel2", sel2, np.uint32, 1)
    _check("digitized_chains", digitized_chains, np.uint32, 1)
    edges = np.ascontiguousarray(edges, dtype=np.float64)
    F = coords.shape[2]
    if F == 0 or len(sel1) == 0:
        return np.zeros((F, len(sel1), len(edges) - 1), dtype=np.int64)
    d_coords, d_box, remap, d_ch, _ = upload_selected(coords, box, [sel1, sel2], digitized_chains, device=device)
    dev = d_coords.device
    out = shell_counts_device(d_coords, d_box, _sel_dev(sel1, remap, dev), _sel_dev(sel2, remap, dev), d_ch, selfdist,
                              pbc, torch.from_numpy(edges).to(dev), truncate=truncate)
    return out.cpu().numpy().astype(np.int64)


def _groups_csr(groups, dev):
    off = np.zeros(len(groups) + 1, dtype=np.int64)
    if len(groups):
        np.cumsum([len(g) for g in groups], out=off[1:])
    flat = np.concatenate([np.asarray(g, dtype=np.int32) for g in groups]) if len(groups) and off[-1] else \
        np.zeros(0, np.int32)
    return torch.from_numpy(off).to(dev), torch.from_numpy(np.ascontiguousarray(flat, dtype=np.int32)).to(dev)


def dist_reduction_device(coords, box, groups1, groups2, gchains1, gchains2, selfdist, pbc, masses, red1, red2, *,
                          pairs: bool = False, metric: str = "distances", truncate=None, threshold: float = 8.0):
    """K5 on CUDA tensors (groups are python lists of index lists)."""
    dev = coords.device
    F = coords.shape[2]
    G1, G2 = len(groups1), len(groups2)
    P = G1 if pairs else n_columns(G1, G2, selfdist)
    mode = _lib.DIST_CONTACTS if metric == "contacts" else _lib.DIST_DISTANCES
    out = torch.zeros((F, P), dtype=torch.uint8 if mode else torch.float32, device=dev)
    o1, a1 = _groups_csr(groups1, dev)
    o2, a2 = _groups_csr(groups2, dev)
    tr = _lib.traj(coords, box)
    _lib.call(dev, "mkb_dist_reduction", C.byref(tr), _lib.ptr(o1), _lib.ptr(a1), G1, _lib.ptr(o2), _lib.ptr(a2), G2,
              _lib.ptr(gchains1), _lib.ptr(gchains2), int(bool(selfdist)), int(bool(pbc)), _lib.ptr(masses), int(red1),
              int(red2), int(bool(pairs)), mode, _NAN if truncate is None else float(truncate), float(threshold),
              _lib.ptr(out))
    return out.view(torch.bool) if mode else out


# ------------------------------------------------------------------------------------------------ host mirrors
def _check(name, arr, dtype, ndim):
    if not isinstance(arr, np.ndarray) or arr.dtype != dtype:
        raise ValueError(f"Buffer dtype mismatch, expected '{np.dtype(dtype).name}' for {name}")
    if arr.ndim != ndim:
        raise ValueError(f"Buffer has wrong number of dimensions (expected {ndim}, got {arr.ndim})")


def upload_selected(coords, box, index_sets, digitized_chains=None, masses=None, device=None):
    """Move only the atoms that the call touches to the GPU: returns (coords_dev (n_used,3,F), box_dev,
    remapped index arrays, chains_dev, masses_dev).  PCIe is the end-to-end bound of this path (SURVEY 8e)."""
    dev = _lib.device(device)
    used = np.unique(np.concatenate([np.asarray(s, dtype=np.int64).reshape(-1) for s in index_sets])) \
        if len(index_sets) else np.zeros(0, np.int64)
    if used.size and (used[0] < 0 or used[-1] >= coords.shape[0]):
        raise IndexError("atom index out of range")
    remap = np.full(coords.shape[0], -1, dtype=np.int64)
    remap[used] = np.arange(used.size)
    if used.size and used[-1] - used[0] + 1 == used.size and coords.flags["C_CONTIGUOUS"]:
        # the selected rows are one slab of the (N, 3, F) array: copy it where it lies (no host gather; asynchronous and
        # at full PCIe rate when the caller's array is page-locked, e.g. from tools.voxeldescriptors.pinned_array)
        d_coords = torch.from_numpy(coords[int(used[0]):int(used[-1]) + 1]).to(dev, non_blocking=True)
    else:
        sub = np.ascontiguousarray(coords[used]) if used.size != coords.shape[0] else np.ascontiguousarray(coords)
        d_coords = torch.from_numpy(sub).to(dev)
    d_box = torch.from_numpy(np.ascontiguousarray(box, dtype=np.float32)).to(dev)
    d_ch = None
    if digitized_chains is not None:
        d_ch = torch.from_numpy(np.ascontiguousarray(np.asarray(digitized_chains, dtype=np.uint32)[used]).view(np.int32)).to(dev)
    d_m = None
    if masses is not None:
        d_m = torch.from_numpy(np.ascontiguousarray(np.asarray(masses, dtype=np.float32)[used])).to(dev)
    return d_coords, d_box, remap, d_ch, d_m


def _sel_dev(sel, remap, dev):
    return torch.from_numpy(remap[np.asarray(sel, dtype=np.int64)].astype(np.int32)).to(dev)


def dist_trajectory(coords, box, sel1, sel2, digitized_chains, selfdist, pbc, results, device=None,
                    metric: str = "distances", truncate=None, threshold: float = 8.0, exact: bool = True):
    """Drop-in for distance_utils.pyx:126-155 (results (F, P) float32 filled in place).  The optional keywords fuse the
    post-ops of pp_calcDistances; with metric="contacts" a new bool array is returned instead.  ``exact=False``: distances
    within 4 ulp of the reference's float32 values (about twice the kernel throughput) instead of bit-identical."""
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    _check("sel1", sel1, np.uint32, 1); _check("sel2", sel2, np.uint32, 1)
    _check("digitized_chains", digitized_chains, np.uint32, 1)
    F = coords.shape[2]
    P = n_columns(len(sel1), len(sel2), bool(selfdist))
    if metric != "contacts":
        _check("results", results, np.float32, 2)
    if F == 0 or P <= 0:
        return results if metric != "contacts" else np.zeros((F, max(P, 0)), dtype=bool)
    d_coords, d_box, remap, d_ch, _ = upload_selected(coords, box, [sel1, sel2], digitized_chains, device=device)
    dev = d_coords.device
    out = dist_trajectory_device(d_coords, d_box, _sel_dev(sel1, remap, dev), _sel_dev(sel2, remap, dev), d_ch,
                                 selfdist, pbc, metric=metric, truncate=truncate, threshold=threshold, exact=exact)
    if metric == "contacts":
        # page-locked result (torch's caching host allocator recycles the block once the array is dropped): the (F, P)
        # map leaves the GPU at PCIe rate instead of through the driver's pageable staging
        host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
        host.copy_(out, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        return host.numpy()
    torch.from_numpy(results[:F, :P]).copy_(out) if results.flags["C_CONTIGUOUS"] and results.shape == (F, P) \
        else np.copyto(results[:F, :P], out.cpu().numpy())
    return results


def contacts_trajectory_arrays(coords, box, sel1, sel2, digitized_chains, selfdist, pbc, dist_threshold=5, device=None):
    """(frame_offsets (F+1,) int64, pairs (total, 2) uint32): the array form of contacts_trajectory."""
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    _check("sel1", sel1, np.uint32, 1); _check("sel2", sel2, np.uint32, 1)
    _check("digitized_chains", digitized_chains, np.uint32, 1)
    F = coords.shape[2]
    if F == 0 or len(sel1) == 0 or len(sel2) == 0:
        return np.zeros(F + 1, np.int64), np.zeros((0, 2), np.uint32)
    d_coords, d_box, remap, d_ch, _ = upload_selected(coords, box, [sel1, sel2], digitized_chains, device=device)
    dev = d_coords.device
    # the kernel emits sel1[i] / sel2[j] values: give it the ORIGINAL atom ids to write, remapped ids to read
    s1, s2 = _sel_dev(sel1, remap, dev), _sel_dev(sel2, remap, dev)
    off, pairs = contacts_trajectory_device(d_coords, d_box, s1, s2, d_ch, selfdist, pbc, dist_threshold)
    pairs = pairs.cpu().numpy().view(np.uint32)
    if pairs.size:
        used = np.flatnonzero(remap >= 0).astype(np.uint32)
        pairs = used[pairs]  # compact ids -> original atom indices
    return off.cpu().numpy(), pairs


def contacts_trajectory(coords, box, sel1, sel2, digitized_chains, selfdist, pbc, dist_threshold=5, device=None):
    """Drop-in for distance_utils.pyx:59-93: list (per frame) of flat lists [a0, b0, a1, b1, ...]."""
    off, pairs = contacts_trajectory_arrays(coords, box, sel1, sel2, digitized_chains, selfdist, pbc, dist_threshold,
                                            device=device)
    return [pairs[off[f]:off[f + 1]].reshape(-1).tolist() for f in range(len(off) - 1)]


def _reduction(coords, box, groups1, groups2, ch1, ch2, selfdist, pbc, masses, red1, red2, results, pairs, device,
               metric, truncate, threshold):
    _check("coords", coords, np.float32, 3); _check("box", box, np.float32, 2)
    _check("digitized_chains1", ch1, np.uint32, 1); _check("digitized_chains2", ch2, np.uint32, 1)
    _check("masses", masses, np.float32, 1)
    groups1 = [list(g) for g in groups1]
    groups2 = [list(g) for g in groups2]
    F = coords.shape[2]
    if F == 0 or not groups1 or not groups2:
        return results
    d_coords, d_box, remap, _, d_m = upload_selected(coords, box, groups1 + groups2, masses=masses, device=device)
    dev = d_coords.device
    g1 = [remap[np.asarray(g, dtype=np.int64)].tolist() for g in groups1]
    g2 = [remap[np.asarray(g, dtype=np.int64)].tolist() for g in groups2]
    d_c1 = torch.from_numpy(np.ascontiguousarray(ch1).view(np.int32)).to(dev)
    d_c2 = torch.from_numpy(np.ascontiguousarray(ch2).view(np.int32)).to(dev)
    out = dist_reduction_device(d_coords, d_box, g1, g2, d_c1, d_c2, selfdist, pbc, d_m, red1, red2, pairs=pairs,
                                metric=metric, truncate=truncate, threshold=threshold)
    if metric == "contacts":
        return out.cpu().numpy()
    np.copyto(results[:out.shape[0], :out.shape[1]], out.cpu().numpy())
    return results


def dist_trajectory_reduction(coords, box, groups1, groups2, digitized_chains1, digitized_chains2, selfdist, pbc,
                              masses, reduction1, reduction2, results, device=None, metric="distances", truncate=None,
                              threshold: float = 8.0):
    """Drop-in for distance_utils.pyx:211-281."""
    return _reduction(coords, box, groups1, groups2, digitized_chains1, digitized_chains2, selfdist, pbc, masses,
                      reduction1, reduction2, results, False, device, metric, truncate, threshold)


def dist_trajectory_reduction_pairs(coords, box, groups1, groups2, digitized_chains1, digitized_chains2, pbc, masses,
                                    reduction1, reduction2, results, device=None, metric="distances", truncate=None,
                                    threshold: float = 8.0):
    """Drop-in for distance_utils.pyx:286-350."""
    return _reduction(coords, box, groups1, groups2, digitized_chains1, digitized_chains2, False, pbc, masses,
                      reduction1, reduction2, results, True, device, metric, truncate, threshold)


def cdist(coords1, coords2, results, device=None):
    """Drop-in for distance_utils.pyx:355-383."""
    _check("coords1", coords1, np.float32, 2); _check("coords2", coords2, np.float32, 2)
    _check("results", results, np.float32, 2)
    n1, n2, D = coords1.shape[0], coords2.shape[0], coords1.shape[1]
    if n1 == 0 or n2 == 0:
        return
    dev = _lib.device(device)
    a = torch.from_numpy(np.ascontiguousarray(coords1)).to(dev)
    b = torch.from_numpy(np.ascontiguousarray(coords2)).to(dev)
    out = torch.empty((n1, n2), dtype=torch.float32, device=dev)
    for r0 in range(0, n1, 65535):
        r1 = min(n1, r0 + 65535)
        _lib.call(dev, "mkb_cdist", _lib.ptr(a[r0:r1]), r1 - r0, _lib.ptr(b), n2, D, _lib.ptr(out[r0:r1]))
    np.copyto(results[:n1, :n2], out.cpu().numpy())


def pdist(coords, results, device=None):
    """Drop-in for distance_utils.pyx:388-416."""
    _check("coords", coords, np.float32, 2); _check("results", results, np.float32, 1)
    n, D = coords.shape
    if n < 2:
        return
    dev = _lib.device(device)
    a = torch.from_numpy(np.ascontiguousarray(coords)).to(dev)
    out = torch.empty(n * (n - 1) // 2, dtype=torch.float32, device=dev)
    _lib.call(dev, "mkb_pdist", _lib.ptr(a), n, D, _lib.ptr(out))
    np.copyto(results[:out.shape[0]], out.cpu().numpy())


def squareform(distances, device=None):
    """Drop-in for distance_utils.pyx:421-435: n' = int((sqrt(8n + 1) + 1) / 2)."""
    _check("distances", distances, np.float32, 1)
    n = distances.shape[0]
    dim = int((math.sqrt(8 * n + 1) + 1) / 2)
    if dim == 0:
        return np.zeros((0, 0), dtype=np.float32)
    dev = _lib.device(device)
    d = torch.from_numpy(np.ascontiguousarray(distances)).to(dev)
    out = torch.empty((dim, dim), dtype=torch.float32, device=dev)
    _lib.call(dev, "mkb_squareform", _lib.ptr(d), n, dim, _lib.ptr(out))
    return out.cpu().numpy()


def get_collisions(coords1, coords2, dist_threshold, device=None):
    """Drop-in for distance_utils.pyx:98-121: flat list of LOCAL index pairs [i0, j0, i1, j1, ...]."""
    _check("coords1", coords1, np.float32, 2); _check("coords2", coords2, np.float32, 2)
    n1, n2 = coords1.shape[0], coords2.shape[0]
    if n1 == 0 or n2 == 0:
        return []
    dev = _lib.device(device)
    a = torch.from_numpy(np.ascontiguousarray(coords1[:, :3])).to(dev)
    b = torch.from_numpy(np.ascontiguousarray(coords2[:, :3])).to(dev)
    off = torch.empty(n1 + 1, dtype=torch.int64, device=dev)
    args = (_lib.ptr(a), n1, _lib.ptr(b), n2, float(np.float32(dist_threshold)))
    (pairs,) = _lib.count_fill(dev, "mkb_collisions_count", "mkb_collisions_fill", args, off,
                               lambda total: (torch.empty((total, 2), dtype=torch.int32, device=dev),))
    return pairs.cpu().numpy().view(np.uint32).reshape(-1).tolist()
