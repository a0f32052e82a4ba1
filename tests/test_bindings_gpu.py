"""The shared binding layer (_lib.traj, _lib.index_arg, _lib.call) on the device: index tensors the library would misread
are refused, frame slices are passed in place, and any other layout gives the same results as its contiguous copy."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _setup():
    import torch

    dev = torch.device("cuda:0")
    rng = np.random.default_rng(5)
    X = torch.from_numpy(rng.normal(0, 6, size=(40, 3, 12)).astype(np.float32)).to(dev)
    sel = torch.arange(0, 40, 3, dtype=torch.int32, device=dev)
    frames = torch.tensor([7, 2, 5], dtype=torch.int32, device=dev)
    return dev, X, sel, frames


def _calls():
    import torch
    from moleculekit_b200 import align as al
    from moleculekit_b200 import coords as co

    return {
        "superpose_device": lambda X, sel, frames: al.superpose_device(X, sel, X[:, :, :1], sel, frames),
        "rmsd_device": lambda X, sel, frames: al.rmsd_device(X, sel, X[:, :, :1], sel, frames=frames),
        "apply_device": lambda X, sel, frames: al.apply_device(
            X, torch.zeros((3, al.RECORD), dtype=torch.float64, device=X.device), frames),
        "coordinates_device": lambda X, sel, frames: co.coordinates_device(X, sel, frames=frames),
        "coord_sums_device": lambda X, sel, frames: co.coord_sums_device(X, sel, frames=frames),
        "fluctuation_device": lambda X, sel, frames: co.fluctuation_device(
            X, sel, torch.zeros((sel.numel(), 3), dtype=torch.float64, device=X.device), frames=frames),
    }


CASES = [(fn, arg, bad) for fn in ("superpose_device", "rmsd_device", "apply_device", "coordinates_device",
                                   "coord_sums_device", "fluctuation_device")
         for arg in ("sel", "frames") for bad in ("int64", "strided") if not (fn == "apply_device" and arg == "sel")]


@pytest.mark.parametrize("fn,arg,bad", CASES)
def test_index_tensors_must_be_contiguous_int32(fn, arg, bad):
    """An int64 index tensor reaches a uint32_t * parameter as pairs of words (sel = [5, 9] would read atoms 5, 0, 9,
    0); a strided one is read as if it were packed.  Both are refused before anything is launched."""
    import torch

    dev, X, sel, frames = _setup()
    call = _calls()[fn]
    call(X, sel, frames)  # the int32 form runs
    args = {"sel": sel, "frames": frames}
    t = args[arg]
    args[arg] = t.long() if bad == "int64" else torch.stack([t, t], 1).reshape(-1)[::2]
    assert torch.equal(args[arg].to(torch.int32), t)
    with pytest.raises(AssertionError):
        call(X, args["sel"], args["frames"])


def test_traj_views():
    """Frame slices are passed in place with the whole trajectory's frame stride; the box keeps its own stride; a
    transposed tensor is copied for reading and refused for writing."""
    import torch
    from moleculekit_b200 import _lib

    dev = torch.device("cuda:0")
    d = torch.randn((50, 3, 64), device=dev)
    box = torch.rand((3, 64), device=dev) + 10
    t = _lib.traj(d[:, :, 16:48], box[:, 16:48])
    assert (t.n_atoms, t.n_frames, t.frame_stride, t.frame_stride_box) == (50, 32, 64, 64)
    assert t.coords == d[:, :, 16:48].data_ptr() and t.box == box[:, 16:48].data_ptr()
    t = _lib.traj(d[:, :, 16:48], box[:, 16:48].contiguous())
    assert (t.frame_stride, t.frame_stride_box) == (64, 32)
    t = _lib.traj(d[:, :, 16:48])
    assert t.box is None and (t.frame_stride, t.frame_stride_box) == (64, 64)
    # one frame: the coordinates stay in place, the (3, 1) box is normalised to stride 1
    t = _lib.traj(d[:, :, 5:6], box[:, 5:6], writable=True)
    assert t.coords == d[:, :, 5:6].data_ptr() and (t.n_frames, t.frame_stride, t.frame_stride_box) == (1, 64, 1)
    assert t.box != box[:, 5:6].data_ptr() and t._keepalive[1].stride() == (1, 1)
    t = _lib.traj(d[:, :, 5:6].contiguous())
    assert (t.frame_stride, t.frame_stride_box) == (1, 1)
    # frame-major storage (F, N, 3) viewed as (N, 3, F)
    fm = torch.randn((64, 50, 3), device=dev).permute(1, 2, 0)
    t = _lib.traj(fm, box)
    assert t.coords != fm.data_ptr() and t._keepalive[0].is_contiguous() and t.frame_stride == 64
    with pytest.raises(ValueError, match="frame-minor"):
        _lib.traj(fm, box, writable=True)
    with pytest.raises(AssertionError):
        _lib.traj(d, box.t().contiguous().t())  # the box must be frame-minor too


def _frame_major(X, dev):
    """``X`` (N, 3, F) on the device with frame-major storage: not a frame slice of any frame-minor array"""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(np.transpose(X, (2, 0, 1)))).to(dev).permute(1, 2, 0)
    assert t.shape == X.shape and not t.is_contiguous()
    return t


def test_non_frame_minor_inputs_match_contiguous():
    """Read-only entry points copy any other layout: dihedrals, DSSP and distances (which used to refuse it for more
    than one frame) give the bits of the contiguous trajectory."""
    import torch
    import dssp_oracle
    from moleculekit_b200.dihedral import dihedrals_device
    from moleculekit_b200.distance_utils import dist_trajectory_device
    from moleculekit_b200.dssp import dssp_device

    dev = torch.device("cuda:0")
    rng = np.random.default_rng(9)
    helix = dssp_oracle.chain([-57] * 20, [-47] * 20).reshape(80, 3)
    X = (helix[:, :, None] + rng.normal(0, 0.15, size=(80, 3, 6))).astype(np.float32)
    fm, dc = _frame_major(X, dev), torch.from_numpy(X).to(dev)

    quads = torch.arange(0, 76, dtype=torch.int32, device=dev).reshape(19, 4)
    assert torch.equal(dihedrals_device(fm, quads, True), dihedrals_device(dc, quads, True))

    bb = torch.arange(80, dtype=torch.int32, device=dev).reshape(20, 4)
    flags = torch.zeros(20, dtype=torch.uint8, device=dev)
    got, want = dssp_device(fm, bb, flags), dssp_device(dc, bb, flags)
    assert torch.equal(got, want) and (want == 1).any()  # helix residues found

    box = torch.full((3, 6), 30.0, device=dev)
    s1 = torch.arange(0, 40, dtype=torch.int32, device=dev)
    s2 = torch.arange(40, 80, dtype=torch.int32, device=dev)
    ch = torch.zeros(80, dtype=torch.int32, device=dev)
    got = dist_trajectory_device(fm, box, s1, s2, ch, False, True)
    want = dist_trajectory_device(dc, box, s1, s2, ch, False, True)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_wrap_box_single_frame_slice_in_place(oracle):
    """wrap_box_device on a one-frame slice of a resident trajectory wraps that frame where it lies."""
    import torch
    from moleculekit_b200.wrapping import wrap_box_device

    dev = torch.device("cuda:0")
    rng = np.random.default_rng(13)
    coords = rng.normal(0, 30, size=(90, 3, 8)).astype(np.float32)
    box = np.full((3, 8), 20.0, np.float32)
    groups = np.arange(0, 91, 3, dtype=np.uint32)
    want = np.ascontiguousarray(coords[:, :, 5:6])
    oracle.wrap_box(groups, want, np.ascontiguousarray(box[:, 5:6]), np.zeros(0, np.uint32), np.zeros(3, np.float32))
    d = torch.from_numpy(coords).to(dev)
    out = wrap_box_device(d[:, :, 5:6], torch.from_numpy(box).to(dev)[:, 5:6],
                          torch.from_numpy(groups.view(np.int32)).to(dev), None)
    assert out.data_ptr() == d[:, :, 5:6].data_ptr()
    got = d.cpu().numpy()
    assert np.array_equal(got[:, :, 5:6].view(np.uint32), want.view(np.uint32))
    assert np.array_equal(np.delete(got, 5, axis=2), np.delete(coords, 5, axis=2))
    with pytest.raises(ValueError, match="frame-minor"):
        wrap_box_device(_frame_major(coords, dev), torch.from_numpy(box).to(dev),
                        torch.from_numpy(groups.view(np.int32)).to(dev), None)
