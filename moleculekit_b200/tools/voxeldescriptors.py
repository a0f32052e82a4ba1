"""Drop-in for the voxelisation entry points of ``moleculekit.tools.voxeldescriptors``.

``getCenters`` / ``getVoxelDescriptors`` keep the reference's signatures, defaults, return arity and error
messages (moleculekit/tools/voxeldescriptors.py:197-203,251-264,345-360); the occupancy fill runs on the GPU
through libmkb200 (no CPU path).  ``getVoxelDescriptorsBatch`` is the batched form the hardware wants: many
molecules / pockets per launch, optionally left on the device.

Out of scope here (inputs to the hot path, SURVEY.md section 2b): atom typing (``getChannels`` needs RDKit /
OpenBabel).  Pass ``userchannels`` (bool or float, (natoms, nchannels)); if the real ``moleculekit`` package is
importable we defer to its ``getChannels`` for the default-channel case.
"""
from __future__ import annotations

import functools
import logging
import os

import numpy as np
import torch

from .. import _lib as _lib_mod
from .. import occupancy_utils as _occ
from ..elements import vdw_radii_of

logger = logging.getLogger(__name__)

_order = ("hydrophobic", "aromatic", "hbond_acceptor", "hbond_donor", "positive_ionizable",
          "negative_ionizable", "metal", "occupancies")


# ----------------------------------------------------------------------------------------------- host geometry
def _mol_coords(mol):
    """(natoms, 3[, 1]) coordinates of the molecule's current frame, like ``mol.get("coords")``."""
    if hasattr(mol, "get"):
        return mol.get("coords")
    c = np.asarray(mol.coords)
    if c.ndim == 3:
        c = c[:, :, getattr(mol, "frame", 0)]
    return c


def _bounding_box(mol):
    """moleculekit/util.py:376-379 (min / max over atoms, dtype of the coordinates, i.e. float32)."""
    c = _mol_coords(mol)
    return np.squeeze(np.min(c, axis=0)), np.squeeze(np.max(c, axis=0))


def _grid_spec(mol, buffer, boxsize, center, voxelsize):
    """(bb_min, nvoxels) with the reference's arithmetic (voxeldescriptors.py:229-243): float32 bounding box in
    `buffer` mode, float64 ``center - boxsize/2`` in `boxsize` mode."""
    if boxsize is None:
        bb_min, bb_max = _bounding_box(mol)
        bb_min = np.array(bb_min, copy=True)
        bb_max = np.array(bb_max, copy=True)
        bb_min -= buffer  # in place: stays in the coordinate dtype (float32), like the reference
        bb_max += buffer
        nvoxels = np.ceil((bb_max - bb_min) / voxelsize).astype(int) + 1
    else:
        boxsize = np.array(boxsize)
        center = np.array(center)
        nvoxels = np.ceil(boxsize / voxelsize).astype(int)
        bb_min = center - (boxsize / 2)
    return bb_min, nvoxels


@functools.lru_cache(maxsize=10)
def _grid_offsets(nx: int, ny: int, nz: int, voxelsize: float) -> np.ndarray:
    """(nx, ny, nz, 3) float64 float64(i_d * voxelsize), cached per grid shape like the reference's _getGridCenters
    (voxeldescriptors.py:116-123, lru_cache(10))."""
    out = np.empty((nx, ny, nz, 3), dtype=np.float64)
    for d, n in enumerate((nx, ny, nz)):
        shape = [1, 1, 1]
        shape[d] = n
        out[..., d] = (np.arange(n) * voxelsize).astype(np.float64).reshape(shape)
    out.setflags(write=False)
    return out


def _centers_from_spec(bb_min, nvoxels, voxelsize) -> np.ndarray:
    """(prod(nvoxels), 3) float64 centres, bit-identical to voxeldescriptors.py:125-132,245-247:
    c[ix,iy,iz,d] = float64(i_d * voxelsize) + bb_min[d], z fastest."""
    nx, ny, nz = (int(v) for v in nvoxels)
    return (_grid_offsets(nx, ny, nz, float(voxelsize)) + np.asarray(bb_min, dtype=np.float64)).reshape(nx * ny * nz, 3)


def getCenters(mol=None, buffer: float = 0, boxsize: list | None = None, center: list | None = None,
               voxelsize: float = 1):
    """Get a set of centers for voxelization (reference: voxeldescriptors.py:197-248).

    Returns ``(centers (nvoxels, 3) float64, nvoxels (3,) int)``; see the reference docstring for the arguments."""
    bb_min, nvoxels = _grid_spec(mol, buffer, boxsize, center, voxelsize)
    return _centers_from_spec(bb_min, nvoxels, voxelsize), nvoxels


def _channels_to_sigmas(channels, elements):
    """bool channels -> per-channel sigmas = vdW radius * mask (voxeldescriptors.py:117-121,332-335)."""
    channels = np.asarray(channels)
    if channels.dtype == bool:
        sigmas = vdw_radii_of(elements)
        channels = sigmas[:, np.newaxis] * channels.astype(float)
    return channels


def rotationMatrix(axis, theta: float) -> np.ndarray:
    """Rotation by ``theta`` radians about ``axis`` from the unit quaternion (cos(t/2), -axis sin(t/2)) -- the formula of
    moleculekit/util.py:101-117, evaluated with the same scalar operations so the matrices are bit-identical."""
    from math import cos, sin, sqrt

    axis = np.asarray(axis)
    theta = np.asarray(theta)
    axis = axis / sqrt(np.dot(axis, axis))
    a = cos(theta / 2)
    b, c, d = -axis * sin(theta / 2)
    aa, bb, cc, dd = a * a, b * b, c * c, d * d
    bc, ad, ac, ab, bd, cd = b * c, a * d, a * c, a * b, b * d, c * d
    return np.array([[aa + bb - cc - dd, 2 * (bc + ad), 2 * (bd - ac)],
                     [2 * (bc - ad), aa + cc - bb - dd, 2 * (cd + ab)],
                     [2 * (bd + ac), 2 * (cd - ab), aa + dd - bb - cc]])


def rotation_matrices(rotations) -> np.ndarray:
    """(B, 3) angles [rx, ry, rz] -> (B, 3, 3, 3) float64: the x, y and z rotation matrices rotateCoordinates applies in
    that order (voxeldescriptors.py:106-113)."""
    rot = np.atleast_2d(np.asarray(rotations, dtype=np.float64))
    out = np.zeros((rot.shape[0], 3, 3, 3), dtype=np.float64)
    for b in range(rot.shape[0]):
        out[b, 0] = rotationMatrix([1, 0, 0], rot[b, 0])
        out[b, 1] = rotationMatrix([0, 1, 0], rot[b, 1])
        out[b, 2] = rotationMatrix([0, 0, 1], rot[b, 2])
    return out


def rotateCoordinates(coords: np.ndarray, rotations: list, center: list, device=None) -> np.ndarray:
    """Drop-in for voxeldescriptors.py:78-114: rotates (natoms, 3) coordinates about ``center`` by [rx, ry, rz] radians
    around x, then y, then z; returns float64 like the reference (numpy promotes there).  Runs mkb_rotate_coords."""
    c32 = np.ascontiguousarray(np.asarray(coords), dtype=np.float32)
    if c32.ndim != 2 or c32.shape[1] != 3:
        raise ValueError("coords must have shape (natoms, 3)")
    if not np.array_equal(c32, np.asarray(coords)):
        raise ValueError("rotateCoordinates on the GPU takes float32-representable coordinates (Molecule.coords)")
    dev = _lib_mod.device(device)
    d = _occ.rotate_coords_device(torch.from_numpy(c32).to(dev),
                                  torch.tensor([0, c32.shape[0]], dtype=torch.int64, device=dev),
                                  torch.from_numpy(rotation_matrices(list(rotations))).to(dev),
                                  torch.from_numpy(np.asarray(center, dtype=np.float64).reshape(1, 3)).to(dev),
                                  out_dtype=torch.float64)
    return d.cpu().numpy()


def getChannels(mol, aromaticNitrogen: bool = False, version: int = 2, validitychecks: bool = True):
    """Atom typing is an INPUT of the accelerated path (RDKit/OpenBabel chemistry, SURVEY.md 2b).  Defer to the
    real moleculekit when it is installed; otherwise ask for ``userchannels``."""
    try:
        from moleculekit.tools.voxeldescriptors import getChannels as _ref_getChannels  # type: ignore
    except Exception as e:  # pragma: no cover - depends on the environment
        raise RuntimeError(
            "Default channels need moleculekit's atom typing (getChannels), which is outside the GPU hot path. "
            "Pass userchannels=(natoms, nchannels) bool/float array.") from e
    return _ref_getChannels(mol, aromaticNitrogen, version, validitychecks)


# ----------------------------------------------------------------------------------------------- device drivers
_stage_buf: torch.Tensor | None = None


def _staging(n: int) -> torch.Tensor:
    """Grow-only page-locked float32 staging buffer for the single-call path (drop-in calls return pageable numpy)."""
    global _stage_buf
    if _stage_buf is None or _stage_buf.numel() < n:
        _stage_buf = torch.empty(max(n, 1 << 20), dtype=torch.float32, pin_memory=True)
    return _stage_buf[:n]


def _occupancy_grid(coords, sigmas, bb_min, nvoxels, voxelsize, device=None) -> np.ndarray:
    """One regular grid -> (M, C) float64 numpy (the `_getOccupancyC` of the reference, :515-533)."""
    coords = np.ascontiguousarray(np.asarray(coords).astype(np.float32))
    sigmas = np.ascontiguousarray(np.asarray(sigmas).astype(np.float64))
    dev = _lib_mod.device(device)
    M = int(np.prod(nvoxels))
    Cn = sigmas.shape[1]
    feats = np.empty((M, Cn), dtype=np.float64)
    if M == 0 or Cn == 0:
        return feats
    d_coords = torch.from_numpy(coords).to(dev)
    for c0, c1 in _occ._channel_chunks(Cn):
        d_sig = torch.from_numpy(np.ascontiguousarray(sigmas[:, c0:c1])).to(dev)
        descs, _ = _occ.make_grid_descs(np.asarray(bb_min, dtype=np.float64)[None, :], float(voxelsize),
                                        np.asarray(nvoxels)[None, :], np.array([0, coords.shape[0]]))
        d_out = torch.empty((M, c1 - c0), dtype=torch.float32, device=dev)
        _occ.occupancy_grid_batch(d_coords, d_sig, descs, d_out)
        stage = _staging(M * (c1 - c0)).view(M, c1 - c0)  # page-locked: the D2H runs at PCIe rate, then one upcast pass
        stage.copy_(d_out, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        feats[:, c0:c1] = stage.numpy()
    return feats


def _occupancy_points(coords, centers, sigmas, device=None) -> np.ndarray:
    coords = np.ascontiguousarray(np.asarray(coords).astype(np.float32))
    centers = np.ascontiguousarray(np.asarray(centers).astype(np.float64))
    sigmas = np.ascontiguousarray(np.asarray(sigmas).astype(np.float64))
    occus = np.zeros((centers.shape[0], sigmas.shape[1]))
    _occ.calculate_occupancy(centers, coords, sigmas, occus, device=device)
    return occus


def getVoxelDescriptors(mol, boxsize: list | None = None, voxelsize: float = 1, buffer: float = 0,
                        center: list | None = None, usercenters: np.ndarray | None = None,
                        userchannels: np.ndarray | None = None, usercoords: np.ndarray | None = None,
                        aromaticNitrogen: bool = False, method: str = "C", version: int = 2,
                        validitychecks: bool = True, device=None):
    """Calculate descriptors of atom properties for voxels in a grid bounding the molecule.

    Same arguments, return arity and errors as moleculekit/tools/voxeldescriptors.py:251-365:
    ``(features (M,C) f64, centers (M,3) f64[, nvoxels (3,)])`` -- nvoxels only when `usercenters` is None.
    The only addition is the keyword ``device`` (default: current CUDA device)."""
    channels = userchannels
    if channels is None:
        channels, mol = getChannels(mol, aromaticNitrogen, version, validitychecks)
    channels = np.asarray(channels)
    if channels.dtype == bool:
        channels = _channels_to_sigmas(channels, mol.element)

    nvoxels = None
    centers = usercenters
    spec = None
    if centers is None:
        bb_min, nvoxels = _grid_spec(mol, buffer, boxsize, center, voxelsize)
        spec = (bb_min, nvoxels)
        centers = _centers_from_spec(bb_min, nvoxels, voxelsize)

    coords = usercoords
    if coords is None:
        coords = _mol_coords(mol)
    coords = np.asarray(coords)
    if coords.ndim == 3:
        if coords.shape[2] != 1:
            raise RuntimeError(
                "Only a single set of coordinates should be passed for voxelixation. "
                "Make sure your coordinates are either 3D with a last dim of 1 or 2D."
            )
        coords = coords[:, :, 0]

    if method.upper() == "C":
        if spec is not None:
            features = _occupancy_grid(coords, channels, spec[0], spec[1], voxelsize, device=device)
        else:
            centers = np.asarray(centers)  # the reference docstring passes a list here
            features = _occupancy_points(coords, centers, channels, device=device)
    else:
        raise RuntimeError("As of moleculekit 0.9.2 we only support C implementation of voxelization")

    if nvoxels is None:
        return features, centers
    return features, centers, nvoxels


# ----------------------------------------------------------------------------------------------- batched API
class VoxelBatch:
    """A batch of molecules / pockets voxelised in one launch sequence.

    coords: list of (N_b, 3) arrays (or one concatenated (N, 3) array with `atom_offsets`)
    channels: list of (N_b, C) float sigma arrays (bool masks need `elements`), same C for all.
    Grids: either ``boxsize`` (+ per-item ``centers`` (B,3)) or ``buffer`` (bounding box of each item).
    """

    def __init__(self, coords, channels, *, boxsize=None, centers=None, buffer=0.0, voxelsize=1.0,
                 atom_offsets=None, elements=None, radii=None):
        if atom_offsets is None:
            counts = [len(c) for c in coords]
            atom_offsets = np.zeros(len(coords) + 1, dtype=np.int64)
            np.cumsum(counts, out=atom_offsets[1:])
            coords_cat = np.concatenate([np.asarray(c, dtype=np.float32).reshape(-1, 3) for c in coords]) \
                if len(coords) else np.zeros((0, 3), np.float32)
            masked = len(channels) > 0 and all(np.asarray(ch).dtype == bool for ch in channels) and \
                (elements is not None or radii is not None)
            if masked:
                if radii is None:
                    radii = [vdw_radii_of(el) for el in elements]
                radii = np.concatenate([np.asarray(r, dtype=np.float64).reshape(-1) for r in radii])
                chan_cat = np.concatenate([np.asarray(c, dtype=bool) for c in channels])
            else:
                if elements is not None:
                    channels = [_channels_to_sigmas(ch, el) for ch, el in zip(channels, elements)]
                chan_cat = np.concatenate([np.asarray(c, dtype=np.float64) for c in channels]) \
                    if len(channels) else np.zeros((0, 8), np.float64)
        else:
            atom_offsets = np.asarray(atom_offsets, dtype=np.int64)
            coords_cat = np.asarray(coords, dtype=np.float32).reshape(-1, 3)
            masked = radii is not None and np.asarray(channels).dtype == bool
            if masked:
                radii = np.asarray(radii, dtype=np.float64).reshape(-1)
                chan_cat = np.asarray(channels, dtype=bool)
            else:
                chan_cat = np.asarray(channels, dtype=np.float64)
        B = len(atom_offsets) - 1
        self.B = B
        self.atom_offsets = atom_offsets
        self.coords = np.ascontiguousarray(coords_cat)
        self.C = int(chan_cat.shape[1])
        if masked:
            # device-side channel assembly (SURVEY 8f row 1): sigma = radius on the channels of the mask; the (N, C) float64
            # matrix of voxeldescriptors.py:332-335 is never built
            if self.C > 32:
                raise ValueError("bit-mask channels support at most 32 channels; pass float sigmas instead")
            if radii.shape[0] != chan_cat.shape[0]:
                raise ValueError("radii and channels must have one row per atom")
            self.sigmas = None
            self.radii = np.ascontiguousarray(radii)
            bits = (chan_cat.astype(np.uint64) << np.arange(self.C, dtype=np.uint64)).sum(axis=1, dtype=np.uint64)
            self.chanmask = np.ascontiguousarray(bits.astype(np.uint32).view(np.int32))
        else:
            self.sigmas = np.ascontiguousarray(chan_cat)
            self.radii = self.chanmask = None
        self.voxelsize = float(voxelsize)
        origins = np.zeros((B, 3), dtype=np.float64)
        dims = np.zeros((B, 3), dtype=np.int64)
        if boxsize is not None:
            bs = np.array(boxsize, dtype=np.float64)
            ctr = np.asarray(centers, dtype=np.float64).reshape(B, 3)
            dims[:] = np.ceil(bs / voxelsize).astype(int)
            origins[:] = ctr - (bs / 2)
        else:
            for b in range(B):
                c = self.coords[atom_offsets[b]:atom_offsets[b + 1]]
                bb_min = np.min(c, axis=0) - np.float32(buffer)
                bb_max = np.max(c, axis=0) + np.float32(buffer)
                dims[b] = np.ceil((bb_max - bb_min) / voxelsize).astype(int) + 1
                origins[b] = bb_min
        self.origins, self.dims = origins, dims
        self.descs, self.out_offsets = _occ.make_grid_descs(origins, self.voxelsize, dims, atom_offsets)
        self.total_voxels = int(self.out_offsets[-1])

    def centers(self, b: int) -> np.ndarray:
        return _centers_from_spec(self.origins[b], self.dims[b], self.voxelsize)

    def to_device(self, device=None):
        """(coords, channels) on the device; channels = the sigma matrix, or the (radii, bit mask) pair."""
        dev = _lib_mod.device(device)
        d_coords = torch.from_numpy(self.coords).to(dev, non_blocking=True)
        if self.sigmas is not None:
            return d_coords, torch.from_numpy(self.sigmas).to(dev, non_blocking=True)
        return d_coords, (torch.from_numpy(self.radii).to(dev, non_blocking=True),
                          torch.from_numpy(self.chanmask).to(dev, non_blocking=True))

    def run(self, d_coords, d_channels, out: torch.Tensor | None = None, layout: str = "xyzc") -> torch.Tensor:
        """K2+K1 on resident inputs.  ``out`` is (total_voxels, C) float32; with ``layout="cxyz"`` the memory of grid b
        (rows [out_offsets[b], out_offsets[b+1])) holds that grid channel-major, see :meth:`as_cxyz`."""
        if out is None:
            out = torch.empty((self.total_voxels, self.C), dtype=torch.float32, device=d_coords.device)
        small = None if self.has_small_sigmas(d_channels) else False
        if isinstance(d_channels, tuple):
            return _occ.occupancy_grid_batch(d_coords, None, self.descs, out, layout=layout, radii=d_channels[0],
                                             chanmask=d_channels[1], n_channels=self.C, small_sigmas=small)
        return _occ.occupancy_grid_batch(d_coords, d_channels, self.descs, out, layout=layout, small_sigmas=small)

    def has_small_sigmas(self, d_channels) -> bool:
        """Whether some channel entry has 0 < |sigma| < occupancy_utils.SIGMA_EXACT (evaluated in float64 after the grid
        kernels).  Checked on the device once per channel tensor and remembered, so repeated runs on resident inputs
        never wait for the stream."""
        t = d_channels if isinstance(d_channels, tuple) else (d_channels,)
        key = tuple((x.data_ptr(), x.numel()) for x in t)
        if getattr(self, "_small_key", None) != key:
            if isinstance(d_channels, tuple):
                split = _occ.split_small_sigmas(None, d_channels[0], d_channels[1], self.C)
            else:
                split = _occ.split_small_sigmas(d_channels)
            self._small_key, self._small = key, split is not None
        return self._small

    def rotate(self, d_coords, rotations, rot_centers) -> torch.Tensor:
        """Random-rotation augmentation on the device: item b is rotated by rotations[b] = [rx, ry, rz] about
        rot_centers[b] (batched rotateCoordinates); returns new float32 coords for :meth:`run`."""
        dev = d_coords.device
        mats = torch.from_numpy(rotation_matrices(np.asarray(rotations, dtype=np.float64).reshape(self.B, 3))).to(dev)
        ctr = torch.from_numpy(np.ascontiguousarray(np.asarray(rot_centers, dtype=np.float64).reshape(self.B, 3))).to(dev)
        off = torch.from_numpy(np.ascontiguousarray(self.atom_offsets)).to(dev)
        return _occ.rotate_coords_device(d_coords, off, mats, ctr)

    def centers_device(self, device=None) -> torch.Tensor:
        """(total_voxels, 3) float64 voxel centres generated on the device (bit-identical to getCenters)."""
        return _occ.grid_centers(self.descs, device=device)

    def as_cxyz(self, feats, b: int | None = None):
        """View a ``layout="cxyz"`` result as (C, X, Y, Z) for item b, or (B, C, X, Y, Z) for a uniform batch."""
        if b is not None:
            nx, ny, nz = (int(v) for v in self.dims[b])
            return feats[self.out_offsets[b]:self.out_offsets[b + 1]].reshape(self.C, nx, ny, nz)
        if not (self.dims == self.dims[0]).all():
            raise ValueError("items have different grid sizes: ask for one item (b=...)")
        nx, ny, nz = (int(v) for v in self.dims[0])
        return feats.reshape(self.B, self.C, nx, ny, nz)

    def split(self, feats):
        """(sum M_b, C) -> list of per-item (M_b, C) views."""
        return [feats[self.out_offsets[b]:self.out_offsets[b + 1]] for b in range(self.B)]


def pinned_array(shape, dtype=np.float32) -> np.ndarray:
    """A numpy array backed by page-locked host memory (async H2D / D2H at full PCIe rate)."""
    t = torch.empty(tuple(int(x) for x in np.atleast_1d(shape)), dtype=getattr(torch, np.dtype(dtype).name),
                    pin_memory=True)
    return t.numpy()


def _direct_to_host(batch, d_coords, d_chan, dev, out):
    """Zero-copy route for a PINNED float32 result: the fill kernel stores the non-empty blocks straight into ``out`` over
    PCIe (~30 % of the bytes, no staging buffer, no host copy) while host threads zero-fill the empty blocks -- the block
    index reaches the host before the fill kernel starts."""
    t_out = torch.from_numpy(out)
    if isinstance(d_chan, tuple):
        h_rank_t, _keep = _occ.occupancy_grid_batch_to_host(d_coords, None, batch.descs, t_out, radii=d_chan[0], chanmask=d_chan[1],
                                                                small_sigmas=batch.has_small_sigmas(d_chan))
    else:
        h_rank_t, _keep = _occ.occupancy_grid_batch_to_host(d_coords, d_chan, batch.descs, t_out,
                                                                small_sigmas=batch.has_small_sigmas(d_chan))
    _occ.wait_index(dev)
    h_rank = h_rank_t.numpy()
    _occ.expand_compact_host(batch.descs, 0, batch.B, h_rank, None, 0, out)   # zeros for the blocks the GPU does not write
    torch.cuda.current_stream(dev).synchronize()
    LAST_TRANSFER.update(mode="direct", d2h_bytes=int(h_rank[-1]) * 4096 + int(h_rank.nbytes), records=int(h_rank[-1]),
                         blocks=int(len(h_rank) - 1))
    return out


def _compact_to_host(batch, d_coords, d_chan, dev, out, dtype, n_chunks: int = 0):
    """Compact transfer: block records + index over PCIe in chunks, dense array rebuilt by host threads meanwhile."""
    if isinstance(d_chan, tuple):
        recs, rank = _occ.occupancy_grid_batch_compact(d_coords, None, batch.descs, radii=d_chan[0], chanmask=d_chan[1],
                                                         small_sigmas=batch.has_small_sigmas(d_chan))
    else:
        recs, rank = _occ.occupancy_grid_batch_compact(d_coords, d_chan, batch.descs, small_sigmas=batch.has_small_sigmas(d_chan))
    cur = torch.cuda.current_stream(dev)
    h_rank_t = torch.empty(rank.shape, dtype=torch.int32, pin_memory=True)
    h_rank_t.copy_(rank, non_blocking=True)
    cur.synchronize()
    h_rank = h_rank_t.numpy()
    total = int(h_rank[-1])
    h_recs_t = torch.empty((max(total, 1), 1024), dtype=torch.float32, pin_memory=True)
    h_recs = h_recs_t.numpy()
    if out is not None:
        host = out
    else:  # page-locked result from torch's caching host allocator: a fresh 4 GB numpy array would spend the call in page faults
        host = torch.empty((batch.total_voxels, batch.C), dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True).numpy()
    # blocks per grid -> the record range of a chunk of grids
    dims = batch.dims.astype(np.int64)
    nblk = ((dims[:, 0] + 3) // 4) * ((dims[:, 1] + 3) // 4) * ((dims[:, 2] + 7) // 8)
    bbase = np.concatenate([[0], np.cumsum(nblk)])
    if n_chunks <= 0:  # chunks of >= 64 MB of dense output: enough of them to overlap the copy with the expansion
        n_chunks = int(max(1, min(8, host.nbytes // (64 << 20))))
    cuts = np.unique(np.linspace(0, batch.B, min(n_chunks, batch.B) + 1).astype(np.int64))
    side = _side_stream(dev)
    side.wait_stream(cur)
    events = []
    with torch.cuda.stream(side):
        for g0, g1 in zip(cuts[:-1], cuts[1:]):
            r0, r1 = int(h_rank[bbase[g0]]), int(h_rank[bbase[g1]])
            if r1 > r0:
                h_recs_t[r0:r1].copy_(recs[r0:r1], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
            events.append((int(g0), int(g1), r0, ev))
    for g0, g1, r0, ev in events:
        ev.synchronize()
        _occ.expand_compact_host(batch.descs, g0, g1, h_rank, h_recs[r0:] if total else h_recs, r0, host)
    recs.record_stream(side)
    LAST_TRANSFER.update(mode="compact", d2h_bytes=int(total) * 4096 + int(h_rank.nbytes), records=total, blocks=int(len(h_rank) - 1))
    return host


_SIDE = {}
LAST_TRANSFER = {}  # what the most recent getVoxelDescriptorsBatch moved device -> host (bench.py reports it)


def _side_stream(dev):
    key = (dev.index if isinstance(dev, torch.device) else int(dev))
    if key not in _SIDE:
        _SIDE[key] = torch.cuda.Stream(device=dev)
    return _SIDE[key]


def getVoxelDescriptorsBatch(coords, channels, *, boxsize=None, centers=None, buffer=0.0, voxelsize=1.0,
                             elements=None, radii=None, atom_offsets=None, device=None, return_tensor: bool = False,
                             dtype=np.float64, out: np.ndarray | None = None, layout: str = "xyzc",
                             rotations=None, rotation_centers=None, transfer: str = "auto"):
    """Voxelise a batch of molecules / pockets in one launch sequence (HOST arrays in, HOST arrays out).

    coords / channels: lists of per-item (N_b, 3) / (N_b, C) arrays, or concatenated arrays with ``atom_offsets``
    (B+1,).  Grids: ``boxsize`` + per-item ``centers`` (B, 3), or ``buffer`` around each item's bounding box.
    Boolean ``channels`` with ``elements`` (vdW radii looked up) or explicit per-atom ``radii`` are assembled into
    sigmas on the device.  ``rotations`` (B, 3) [rx, ry, rz] + ``rotation_centers`` (B, 3) rotate every item on the
    device first (rotateCoordinates semantics; the grids stay where ``centers`` / the unrotated bounding boxes put them).
    Returns ``(features, nvoxels)``: features is a list of (M_b, C) arrays -- float64 by default like the reference,
    ``dtype=np.float32`` skips the upcast, ``out`` (float32 (sum M_b, C), ideally from :func:`pinned_array`) receives
    the device result directly -- or, with ``return_tensor=True``, ``(tensor, nvoxels, voxel_offsets)`` with one
    float32 CUDA tensor left on the device (the layout per-GPU consumers keep resident).  ``layout="cxyz"`` stores
    each grid channel-major: the list entries / tensor slices are then (C, X, Y, Z) (tensor: (B, C, X, Y, Z) when all
    grids have the same size).  ``nvoxels`` is (B, 3).

    ``transfer``: how the grids cross PCIe.  "dense" copies the (sum M, C) float32 array; "direct" (chosen by "auto" when
    ``out`` is page-locked, e.g. from :func:`pinned_array`) lets the fill kernel store the non-empty blocks straight into
    ``out`` while host threads zero the others; "compact" (8 channels,
    voxel-major) copies only the 4x4x8-voxel blocks that have an atom within 5 A (~30 % of a protein pocket grid) plus a
    block index, in chunks, while host threads rebuild the dense array -- float32 or, upcast on the fly, the reference's
    float64 -- with identical bytes; "auto" takes the compact route when it applies."""
    batch = VoxelBatch(coords, channels, boxsize=boxsize, centers=centers, buffer=buffer, voxelsize=voxelsize,
                       elements=elements, radii=radii, atom_offsets=atom_offsets)
    dev = _lib_mod.device(device)
    d_coords, d_chan = batch.to_device(dev)
    if rotations is not None:
        if rotation_centers is None:
            raise ValueError("rotation_centers is required with rotations")
        d_coords = batch.rotate(d_coords, rotations, rotation_centers)
    cx = layout == "cxyz"
    if transfer not in ("auto", "dense", "compact", "direct"):
        raise ValueError("transfer must be 'auto', 'dense', 'compact' or 'direct'")
    if transfer == "direct" and (out is None or not torch.from_numpy(out).is_pinned()):
        raise ValueError("transfer='direct' needs a page-locked float32 `out` (tools.voxeldescriptors.pinned_array)")
    want_dtype = np.float32 if out is not None else (np.dtype(dtype) if dtype is not None else np.dtype(np.float32))
    compact_ok = (not return_tensor and not cx and batch.C == 8 and np.dtype(want_dtype) in (np.dtype(np.float32), np.dtype(np.float64))
                  and batch.total_voxels > 0)
    if transfer == "compact" and not compact_ok:
        raise ValueError("transfer='compact' needs 8 channels, the voxel-major layout and host float32 / float64 results")
    # "auto": the compact route pays a block-index round trip and a host-thread expansion; it wins once the dense copy
    # is long enough to hide them (large batches such as C3's 256 pockets, not 32), and on a host shared by many ranks the
    # expansion competes for the same memory bandwidth as the DMA it replaces, so "auto" keeps the dense copy there
    if transfer == "auto" and (batch.total_voxels * batch.C * 4 < (512 << 20) or int(os.environ.get("LOCAL_WORLD_SIZE", "1")) > 2):
        compact_ok = False
    if compact_ok and transfer != "dense":
        if out is not None and (out.dtype != np.float32 or out.shape != (batch.total_voxels, batch.C) or not out.flags["C_CONTIGUOUS"]):
            raise ValueError(f"out must be a C-contiguous float32 array of shape {(batch.total_voxels, batch.C)}")
        try:
            if transfer != "compact" and out is not None and torch.from_numpy(out).is_pinned():
                host = _direct_to_host(batch, d_coords, d_chan, dev, out)
            else:
                host = _compact_to_host(batch, d_coords, d_chan, dev, out, want_dtype)
            return batch.split(host), batch.dims.copy()
        except _lib_mod.MkbUnsupported:
            if transfer == "compact":
                raise
    d_out = batch.run(d_coords, d_chan, layout=layout)
    if return_tensor:
        if cx and (batch.dims == batch.dims[0]).all():
            d_out = batch.as_cxyz(d_out)
        return d_out, batch.dims.copy(), batch.out_offsets.copy()
    if out is not None:
        if out.dtype != np.float32 or out.shape != (batch.total_voxels, batch.C) or not out.flags["C_CONTIGUOUS"]:
            raise ValueError(f"out must be a C-contiguous float32 array of shape {(batch.total_voxels, batch.C)}")
        torch.from_numpy(out).copy_(d_out, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()
        host = out
        LAST_TRANSFER.update(mode="dense", d2h_bytes=int(out.nbytes), records=None, blocks=None)
    else:
        host = d_out.cpu().numpy()
        if dtype is not None and np.dtype(dtype) != np.float32:
            host = host.astype(dtype)
    if cx:
        return [batch.as_cxyz(host, b) for b in range(batch.B)], batch.dims.copy()
    return batch.split(host), batch.dims.copy()
