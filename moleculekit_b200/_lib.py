"""ctypes binding of libmkb200.so (include/mkb200.h) and the one path by which the modules call it with torch tensors
(:func:`call`, :func:`traj`, :func:`ptr`).  No CPU fallback: if the CUDA library is missing or no CUDA device is
present, every entry point raises."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "lib", "libmkb200.so")

MKB_OK = 0
OCC_ACCUMULATE = 1
OCC_LAYOUT_CXYZ = 2
DIST_DISTANCES = 0
DIST_CONTACTS = 1
DIST_DISTANCES_FAST = 4

# numpy mirror of `mkb_grid_desc` (72 bytes, no padding)
GRID_DESC = np.dtype(
    [("origin", "<f8", (3,)), ("voxelsize", "<f8"), ("dims", "<i4", (3,)), ("reserved", "<i4"),
     ("atom_begin", "<i8"), ("atom_end", "<i8"), ("out_offset", "<i8")], align=False)
assert GRID_DESC.itemsize == 72


class Traj(C.Structure):
    """mirror of `mkb_traj`"""
    _fields_ = [("coords", C.c_void_p), ("box", C.c_void_p), ("n_atoms", C.c_int64), ("n_frames", C.c_int64),
                ("frame_stride", C.c_int64), ("frame_stride_box", C.c_int64)]


EXPORTS = [
    "mkb_version", "mkb_create", "mkb_destroy", "mkb_last_error", "mkb_launch_count",
    "mkb_set_timing", "mkb_get_timing", "mkb_last_kernel",
    "mkb_occupancy_grid_batch_compact", "mkb_occupancy_compact_blocks", "mkb_occupancy_expand_host",
    "mkb_occupancy_grid_batch_to_host", "mkb_occupancy_wait_index",
    "mkb_occupancy_grid_batch", "mkb_occupancy_grid_batch_masked", "mkb_occupancy_points",
    "mkb_grid_centers", "mkb_rotate_coords",
    "mkb_dist_trajectory", "mkb_contacts_count", "mkb_contacts_fill", "mkb_dist_reduction",
    "mkb_cdist", "mkb_pdist", "mkb_squareform", "mkb_collisions_count", "mkb_collisions_fill",
    "mkb_bonds_count", "mkb_bonds_fill", "mkb_shell_counts", "mkb_wrap_box", "mkb_within_distance", "mkb_xtc_decode",
    "mkb_xtc_encode", "mkb_dcd_decode", "mkb_dcd_encode", "mkb_netcdf_decode", "mkb_netcdf_encode",
    "mkb_trr_decode", "mkb_trr_encode", "mkb_mdcrd_decode", "mkb_mdcrd_encode", "mkb_xyz_index",
    "mkb_xyz_decode", "mkb_xyz_encode", "mkb_pdb_index", "mkb_pdb_decode", "mkb_pdb_cell", "mkb_pdb_encode",
    "mkb_gro_index", "mkb_gro_decode", "mkb_gro_head", "mkb_gro_encode", "mkb_cif_index", "mkb_cif_decode",
    "mkb_cif_encode", "mkb_bcif_decode", "mkb_bcif_quantize", "mkb_bcif_sizes", "mkb_bcif_emit",
    "mkb_lammpstrj_index", "mkb_lammpstrj_head", "mkb_lammpstrj_decode", "mkb_lammpstrj_encode",
    "mkb_wrap_triclinic", "mkb_hbonds_count", "mkb_hbonds_fill", "mkb_ring_pairs_count", "mkb_ring_pairs_fill",
    "mkb_align_fit", "mkb_align_apply", "mkb_rmsd", "mkb_coordinates", "mkb_coord_sums", "mkb_fluctuation",
    "mkb_frame_moments", "mkb_dihedrals", "mkb_sasa", "mkb_sasa_chunk_frames", "mkb_dssp", "mkb_dssp_chunk_frames",
    "mkb_tmscore", "mkb_tmscore_max_pairs", "mkb_tmalign", "mkb_tmalign_max_residues", "mkb_tmalign_chunk_frames",
]

_lib = None
_handles: dict[int, C.c_void_p] = {}


class MkbError(RuntimeError):
    pass


class MkbUnsupported(MkbError):
    """MKB_ERR_UNSUPPORTED: a valid request outside the domain of the entry point (callers fall back to the general one)."""


class MkbCapacity(MkbError):
    """MKB_ERR_CAPACITY: an output buffer is too small (the entry point says where it left the size to come back with)."""


def load():
    """dlopen the library (works without a GPU; creating a handle does not)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("MKB200_LIB", LIB_PATH)  # tuning hook: an alternative in-tree build of the same sources
    if not os.path.isfile(path):
        raise ImportError(
            f"{path} not found: build the CUDA extension first (python -m moleculekit_b200.build). "
            "moleculekit_b200 has no CPU fallback.")
    lib = C.CDLL(path)
    vp, i32, i64, u32, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_float
    lib.mkb_version.restype = C.c_int
    lib.mkb_create.argtypes = [C.c_int, C.POINTER(vp)]
    lib.mkb_destroy.argtypes = [vp]
    lib.mkb_last_error.argtypes = [vp]
    lib.mkb_last_error.restype = C.c_char_p
    lib.mkb_launch_count.argtypes = [vp]
    lib.mkb_launch_count.restype = i64
    lib.mkb_set_timing.argtypes = [vp, C.c_int]
    lib.mkb_get_timing.argtypes = [vp, C.POINTER(f32), C.POINTER(f32)]
    lib.mkb_last_kernel.argtypes = [vp]
    lib.mkb_last_kernel.restype = C.c_char_p
    lib.mkb_occupancy_grid_batch.argtypes = [vp, vp, vp, vp, i64, i32, vp, i32, vp, u32]
    lib.mkb_occupancy_grid_batch_compact.argtypes = [vp, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp, i64]
    lib.mkb_occupancy_grid_batch_to_host.argtypes = [vp, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp, i64, vp]
    lib.mkb_occupancy_wait_index.argtypes = [vp]
    lib.mkb_occupancy_compact_blocks.argtypes = [vp, i32]
    lib.mkb_occupancy_compact_blocks.restype = i64
    lib.mkb_occupancy_expand_host.argtypes = [vp, i32, i32, vp, vp, i64, vp, i32, i32]
    lib.mkb_occupancy_points.argtypes = [vp, vp, vp, i64, vp, vp, i64, i32, vp, u32]
    lib.mkb_occupancy_grid_batch_masked.argtypes = [vp, vp, vp, vp, vp, i64, i32, vp, i32, vp, u32]
    lib.mkb_grid_centers.argtypes = [vp, vp, vp, i32, vp]
    lib.mkb_rotate_coords.argtypes = [vp, vp, vp, i64, vp, i32, vp, vp, vp, vp]
    tp = C.POINTER(Traj)
    lib.mkb_dist_trajectory.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, i32, i32, i32, f32, f32, vp]
    lib.mkb_contacts_count.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, i32, i32, f32, vp, C.POINTER(i64)]
    lib.mkb_contacts_fill.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, i32, i32, f32, vp, vp]
    lib.mkb_dist_reduction.argtypes = [vp, vp, tp, vp, vp, i64, vp, vp, i64, vp, vp, i32, i32, vp, i32, i32, i32,
                                       i32, f32, f32, vp]
    lib.mkb_cdist.argtypes = [vp, vp, vp, i64, vp, i64, i32, vp]
    lib.mkb_pdist.argtypes = [vp, vp, vp, i64, i32, vp]
    lib.mkb_squareform.argtypes = [vp, vp, vp, i64, i64, vp]
    lib.mkb_collisions_count.argtypes = [vp, vp, vp, i64, vp, i64, f32, vp, C.POINTER(i64)]
    lib.mkb_collisions_fill.argtypes = [vp, vp, vp, i64, vp, i64, f32, vp, vp]
    lib.mkb_shell_counts.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, i32, i32, f32, vp, i32, vp]
    lib.mkb_bonds_count.argtypes = [vp, vp, vp, vp, vp, i64, f32, vp, C.POINTER(i64)]
    lib.mkb_bonds_fill.argtypes = [vp, vp, vp, vp, vp, i64, f32, vp, vp]
    lib.mkb_within_distance.argtypes = [vp, vp, vp, i64, vp, i64, vp, i64, f32, vp]
    lib.mkb_xtc_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, i64, f32, vp]
    lib.mkb_xtc_encode.argtypes = [vp, vp, vp, i64, i64, i64, f32, f32, vp, i64, vp, vp, vp]
    lib.mkb_dcd_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, i64, vp, i64, vp, i32, vp, i64]
    lib.mkb_dcd_encode.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, i64]
    lib.mkb_netcdf_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, i64]
    lib.mkb_netcdf_encode.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, vp, vp, i64]
    lib.mkb_trr_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, i32, vp, i64]
    lib.mkb_trr_encode.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, vp, i64, vp, i64]
    lib.mkb_mdcrd_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, i32, vp, i64, vp, i64, vp]
    lib.mkb_mdcrd_encode.argtypes = [vp, vp, vp, i64, i64, i64, vp, i64, vp, i64]
    lib.mkb_xyz_index.argtypes = [vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, i64]
    lib.mkb_xyz_decode.argtypes = [vp, vp, vp, i64, i64, vp, i64, i64, vp, i64, i64, vp, i64]
    lib.mkb_xyz_encode.argtypes = [vp, vp, vp, i64, i64, i64, vp, i64, vp, i64, vp, i64]
    lib.mkb_pdb_index.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, i64]
    lib.mkb_pdb_decode.argtypes = [vp, vp, vp, i64, i64, vp, i64, i64, vp, i64, i64, vp, i64]
    lib.mkb_pdb_cell.argtypes = [vp, vp, vp, i64, vp, vp]
    lib.mkb_pdb_encode.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, vp, i64, i64, vp, i64]
    lib.mkb_gro_index.argtypes = [vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, i64]
    lib.mkb_gro_decode.argtypes = [vp, vp, vp, i64, i64, vp, i64, i64, i64, i32, vp, vp, i64, i64, vp, i64]
    lib.mkb_gro_head.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp, vp]
    lib.mkb_gro_encode.argtypes = [vp, vp, vp, vp, i64, i64, i64, vp, i64, vp, vp, i64, i32, vp, i64]
    lib.mkb_cif_index.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, i64, vp, vp, i64]
    lib.mkb_cif_decode.argtypes = [vp, vp, vp, i64, i64, vp, i64, i64, i64, i64, i64, vp, i64, i64, vp, i64]
    lib.mkb_cif_encode.argtypes = [vp, vp, vp, i64, i64, i64, vp, i64, i64, i64, i64, i64, i64, i64, vp, i64]
    dbl = C.c_double
    lib.mkb_bcif_decode.argtypes = [vp, vp, vp, i64, vp, i64, i64, vp, i64, vp, i64, i64, vp]
    lib.mkb_bcif_quantize.argtypes = [vp, vp, vp, i64, i64, i64, i64, dbl, vp]
    lib.mkb_bcif_sizes.argtypes = [vp, vp, vp, i64, i64, i64, vp]
    lib.mkb_bcif_emit.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, vp, i64]
    lib.mkb_lammpstrj_index.argtypes = [vp, vp, vp, i64, i64, i64, i64, i64, vp, i64, i64, vp, vp, vp, i64]
    lib.mkb_lammpstrj_head.argtypes = [vp, vp, vp, i64, i64, i64, i64, vp, vp, i64, i64, i64, i64, i64, vp, vp, vp, vp]
    lib.mkb_lammpstrj_decode.argtypes = [vp, vp, vp, i64, i64, vp, i64, i64, i64, vp, i64, vp, vp, i32, i32, vp, vp,
                                         vp, i64, vp]
    lib.mkb_lammpstrj_encode.argtypes = [vp, vp, vp, vp, i64, i64, i64, vp, vp, i64, vp, vp, i64, vp, i64, vp]
    lib.mkb_wrap_box.argtypes = [vp, vp, tp, vp, i64, vp, i64, C.POINTER(C.c_float)]
    lib.mkb_wrap_triclinic.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, i64, C.POINTER(C.c_float), i32]
    lib.mkb_hbonds_count.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp, f32, f32, i32, i32, vp, C.POINTER(i64)]
    lib.mkb_hbonds_fill.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp, f32, f32, i32, i32, vp, vp]
    lib.mkb_ring_pairs_count.argtypes = [vp, vp, i32, tp, vp, vp, i64, vp, i64, f32, f32, f32, f32, vp, C.POINTER(i64)]
    lib.mkb_ring_pairs_fill.argtypes = [vp, vp, i32, tp, vp, vp, i64, vp, i64, f32, f32, f32, f32, vp, vp, vp]
    lib.mkb_align_fit.argtypes = [vp, vp, tp, vp, tp, vp, i64, vp, i64, vp, vp]
    lib.mkb_align_apply.argtypes = [vp, vp, tp, vp, i64, vp, vp]
    lib.mkb_rmsd.argtypes = [vp, vp, tp, vp, tp, vp, i64, vp, i64, vp, vp]
    lib.mkb_coordinates.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp, i64]
    lib.mkb_coord_sums.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp]
    lib.mkb_fluctuation.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp, vp, i64, vp, i64]
    lib.mkb_frame_moments.argtypes = [vp, vp, tp, vp, i64, vp, i64, vp, vp, vp, i64, vp]
    lib.mkb_dihedrals.argtypes = [vp, vp, tp, vp, i64, vp, i64, i32, vp, i64]
    lib.mkb_sasa.argtypes = [vp, vp, tp, vp, i64, vp, vp, i64, vp, i64, vp, i32, vp, i64, vp, i64, vp]
    lib.mkb_sasa_chunk_frames.argtypes = [i64, i64, i64]
    lib.mkb_sasa_chunk_frames.restype = i64
    lib.mkb_dssp.argtypes = [vp, vp, tp, vp, vp, i64, C.c_double, vp, i64, vp, i64, vp, vp]
    lib.mkb_dssp_chunk_frames.argtypes = [i64]
    lib.mkb_dssp_chunk_frames.restype = i64
    lib.mkb_tmscore.argtypes = [vp, vp, tp, vp, tp, vp, i64, i64, C.c_double, C.c_double, vp, i32, vp, i64, vp, vp]
    lib.mkb_tmscore_max_pairs.argtypes = []
    lib.mkb_tmscore_max_pairs.restype = i64
    lib.mkb_tmalign.argtypes = [vp, vp, tp, vp, i64, tp, vp, i64, i32, vp, vp, i64, vp, vp, vp, vp, vp]
    lib.mkb_tmalign_max_residues.argtypes = []
    lib.mkb_tmalign_max_residues.restype = i64
    lib.mkb_tmalign_chunk_frames.argtypes = [i64, i64]
    lib.mkb_tmalign_chunk_frames.restype = i64
    for name in EXPORTS:
        if name in ("mkb_last_error", "mkb_launch_count", "mkb_version", "mkb_last_kernel", "mkb_occupancy_compact_blocks",
                    "mkb_sasa_chunk_frames", "mkb_dssp_chunk_frames", "mkb_tmscore_max_pairs",
                    "mkb_tmalign_max_residues", "mkb_tmalign_chunk_frames"):
            continue
        getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib


def handle(device: int = 0):
    """One engine handle per CUDA device, created on first use."""
    lib = load()
    device = int(device)
    h = _handles.get(device)
    if h is None:
        out = C.c_void_p()
        rc = lib.mkb_create(device, C.byref(out))
        if rc != MKB_OK or not out.value:
            raise MkbError(
                f"mkb_create(device={device}) failed (status {rc}): a CUDA device is required, there is no CPU fallback")
        h = out
        _handles[device] = h
    return h


def check(rc: int, h) -> None:
    if rc != MKB_OK:
        msg = load().mkb_last_error(h)
        raise {-5: MkbUnsupported, -4: MkbCapacity}.get(rc, MkbError)(f"libmkb200 status {rc}: {msg.decode() if msg else '?'}")


# ------------------------------------------------------------------------------------------ calls from torch tensors
def device(device):
    """The torch.device a host-level function runs on: ``device``, or torch's current CUDA device for None."""
    if device is None:
        if not torch.cuda.is_available():
            raise MkbError("moleculekit_b200 needs a CUDA device (there is no CPU fallback)")
        return torch.device("cuda", torch.cuda.current_device())
    d = torch.device(device)
    if d.type != "cuda":
        raise MkbError(f"moleculekit_b200 runs on CUDA devices only, got {d}")
    return torch.device("cuda", d.index if d.index is not None else torch.cuda.current_device())


def tensor_device(t, caller: str):
    """The device of ``t``, which must be a CUDA device: ``caller`` names the entry point in the error."""
    dev = t.device
    if dev.type != "cuda":
        raise MkbError(f"{caller} runs on CUDA tensors only, got {dev} (there is no CPU fallback)")
    return dev


def ptr(t) -> C.c_void_p:
    """The data pointer of a tensor; None gives NULL."""
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def stream(dev) -> C.c_void_p:
    """torch's current stream on ``dev``: every entry point is ordered on it."""
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def index_arg(t, dev, dtype=torch.int32, cols: int | None = None) -> None:
    """Assert that the index tensor ``t`` (None passes) is a contiguous ``dtype`` tensor on ``dev``, 1-D or, with
    ``cols``, (m, cols).  The library reads packed 32-bit indices: an int64 tensor would be read as pairs of words."""
    if t is None:
        return
    assert t.dtype == dtype and t.device == dev and t.is_contiguous(), \
        f"index tensors must be contiguous {dtype} on {dev}, got {t.dtype} on {t.device}"
    assert t.ndim == 1 if cols is None else (t.ndim == 2 and t.shape[1] == cols), f"bad index tensor shape {tuple(t.shape)}"


def traj(coords, box=None, writable: bool = False) -> Traj:
    """`mkb_traj` view of an (N, 3, F) float32 CUDA trajectory and its (3, F) float32 ``box`` (None: a NULL box).

    A frame-minor tensor -- contiguous, or a frame slice of a contiguous one -- is passed in place.  Any other layout is
    copied for reading, kept alive on the struct; with ``writable`` (an entry point that writes ``coords``) it raises
    ValueError instead, as the result would land in the copy."""
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.ndim == 3 and coords.shape[1] == 3
    N, _, F = coords.shape
    s_atom, s_axis, s_frame = coords.stride()
    if not (N == 0 or (s_atom == 3 * s_axis and (F <= 1 or s_frame == 1) and s_axis >= F)):
        if writable:
            raise ValueError("coords must be (N, 3, F) frame-minor (a frame slice of a contiguous trajectory is fine)")
        coords = coords.contiguous()
        s_axis = coords.stride(1)
    t = Traj()
    t.n_atoms, t.n_frames = N, F
    t.frame_stride = t.frame_stride_box = max(s_axis if N else F, F, 1)
    if box is not None:
        assert box.is_cuda and box.dtype == torch.float32 and box.ndim == 2 and box.shape[0] == 3
        if F <= 1:
            # the stride of a size-1 / empty dimension is meaningless (numpy views may carry 0): normalise
            box = box.contiguous()
            t.frame_stride_box = max(F, 1)
        else:
            s_box, s_unit = box.stride()
            assert s_unit == 1, "box must be (3, F) frame-minor (a frame slice of a contiguous one is fine)"
            t.frame_stride_box = s_box
        t.box = box.data_ptr()
    t.coords = coords.data_ptr()
    t._keepalive = (coords, box)  # a copy made here must outlive the launch
    return t


def call(dev, name: str, *args) -> None:
    """Run the entry point ``name`` as name(handle, stream, *args) on CUDA device ``dev`` and torch's current stream
    there; a failed status raises :class:`MkbError`."""
    h = handle(dev.index)
    with torch.cuda.device(dev):
        check(getattr(load(), name)(h, stream(dev), *args), h)


def count_fill(dev, count_name: str, fill_name: str, args: tuple, offsets, alloc) -> tuple:
    """The two-pass entry points: ``count_name(*args, offsets, &total)`` writes the row offsets and returns the total
    (read back: synchronises), ``alloc(total)`` returns the output tensors and, when total > 0,
    ``fill_name(*args, offsets, *outputs)`` fills them.  Returns the outputs."""
    total = C.c_int64(0)
    call(dev, count_name, *args, ptr(offsets), C.byref(total))
    outs = alloc(max(total.value, 0))
    if total.value > 0:
        call(dev, fill_name, *args, ptr(offsets), *map(ptr, outs))
    return outs


def launch_count(device: int = 0) -> int:
    return int(load().mkb_launch_count(handle(device)))


def set_timing(on: bool, device: int = 0) -> None:
    h = handle(device)
    check(load().mkb_set_timing(h, 1 if on else 0), h)


def get_timing(device: int = 0) -> tuple[float, float]:
    """(prep_ms, main_kernel_ms) of the most recent timed entry point on this device (synchronises)."""
    h = handle(device)
    a, b = C.c_float(), C.c_float()
    check(load().mkb_get_timing(h, C.byref(a), C.byref(b)), h)
    return float(a.value), float(b.value)


def last_fill_kernel(device: int = 0) -> str:
    """Name of the main kernel the most recent occupancy / distance call launched on this device."""
    return load().mkb_last_kernel(handle(device)).decode()


def destroy_all() -> None:
    for dev, h in list(_handles.items()):
        load().mkb_destroy(h)
        del _handles[dev]
