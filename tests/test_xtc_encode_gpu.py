"""K21 (xtc_encode_kernel) against the reference writer: the bytes of write_xtc / xtc_bytes equal, with no tolerance, the
reference's own files (tests/golden/xtc/), the Python restatement of its writer (oracle/xtc_writer.py) on generated
floats, and what K11 decodes from them returns to the lattice exactly."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import xtc_cases as xc
from oracle import xtc_writer as xw

pytestmark = pytest.mark.gpu

NOT_REQUANTISABLE = {"wide_x", "wide_xyz"}  # tests/test_xtc_encode_cpu.py::test_which_golden_files_requantise


def _stack(frames):
    return np.ascontiguousarray(np.stack([np.asarray(f, np.float32) for f in frames], axis=2))


def _headers(F, seed=0):
    rng = np.random.default_rng(seed)
    return (rng.uniform(0, 5, size=(3, 3, F)).astype(np.float32), (np.arange(F) * 0.25 + 1).astype(np.float32),
            np.arange(F, dtype=np.int32) * 100 + 7)


def _assert_same_file(got, want, what):
    if got != want:
        n = min(len(got), len(want))
        d = np.flatnonzero(np.frombuffer(got[:n], np.uint8) != np.frombuffer(want[:n], np.uint8))
        raise AssertionError(f"{what}: {len(got)} bytes against {len(want)}, first difference at byte "
                             f"{d[0] if len(d) else n}")


def _check(coords, precision=1000.0, what=""):
    from moleculekit_b200 import xtc as px

    box, time, step = _headers(coords.shape[2])
    got = px.xtc_bytes(coords, box, time, step, precision=precision)
    _assert_same_file(got, xw.write_xtc(coords, box, time, step, precision), what)
    return got


# ----------------------------------------------------------------------------------------- 1. the reference's own files
def test_reference_files_byte_for_byte(g_xtc):
    from moleculekit_b200 import xtc as px

    for name in g_xtc["names"].tolist():
        args = [g_xtc[f"{name}_{k}"] for k in ("coords", "box", "time", "step")]
        want = open(os.path.join(g_xtc["_dir"], name + ".xtc"), "rb").read()
        if name in NOT_REQUANTISABLE:  # the decoded floats do not return to the file's integers: the oracle on the same floats
            want = xw.write_xtc(*args)
        _assert_same_file(px.xtc_bytes(*args), want, name)


# ----------------------------------------------------------------------------------------- 2. the oracle on generated floats
def _paired(rng, hi, n):
    """(n, 3) floats uniform in [-hi, hi], every second one next to its predecessor (keeps the first small range low)"""
    a = rng.uniform(-hi, hi, size=(n, 3))
    a[1::2] = a[0::2] + rng.normal(0, 0.002, size=a[1::2].shape)
    return a


def _precision_case(rng):
    return _stack([np.concatenate([xc._water(rng, 40, 4.0), rng.normal(0, 1.5, size=(80, 3))]) - 1.0 for _ in range(3)])


@pytest.mark.parametrize("precision", [1, 10, 100, 1000, 1e4, 1e5, 1e6, 333.3, 0, -5])
def test_oracle_parity_precisions(precision):
    _check(_precision_case(np.random.default_rng(11)), precision, f"precision {precision}")


@pytest.mark.parametrize("natoms", [1, 3, 9, 10, 11, 64, 1000])
def test_oracle_parity_atom_counts(natoms):
    rng = np.random.default_rng(natoms)
    _check(_stack([rng.normal(0, 1, size=(natoms, 3)) for _ in range(3)]), what=f"{natoms} atoms")


@pytest.mark.parametrize("F", [1, 63, 64, 65, 300])
def test_oracle_parity_frame_counts(F):
    """several 64-thread blocks of frames and a partial one"""
    rng = np.random.default_rng(F)
    w = xc._water(rng, 8, 2.0) - 1.0
    _check(_stack([w + rng.normal(0, 0.05, size=w.shape) * np.sqrt(f + 1) for f in range(F)]), what=f"{F} frames")


def test_oracle_parity_water_and_chain():
    rng = np.random.default_rng(21)
    w = xc._water(rng, 150, 3.0)
    _check(_stack([w + rng.normal(0, 0.03, size=w.shape) for _ in range(4)]), what="water")
    n = 2000  # a chain whose bond length swells and shrinks: long runs, the small range stepping up and down
    scale = 0.004 * np.exp(2.5 * np.sin(np.linspace(0, 6 * np.pi, n)))[:, None]
    _check(_stack([np.cumsum(rng.normal(0, 1, size=(n, 3)) * scale, axis=0) - 1.0 for _ in range(3)]), what="chain")


@pytest.mark.parametrize("naxes", [1, 2, 3])
def test_oracle_parity_ranges_beyond_24_bits(naxes):
    rng = np.random.default_rng(30 + naxes)
    hi = np.array([2.5, 1.8, 3.0])
    hi[:naxes] = [21000.0, 40000.0, 17000.0][:naxes]
    got = _check(_stack([_paired(rng, hi, 80) for _ in range(2)]), what=f"{naxes} wide axes")
    fr = xw.read_ints(got)[0]
    assert sum(b - a + 1 > 0xFFFFFF for a, b in zip(fr.minint, fr.maxint)) == naxes


def test_oracle_parity_full_triples_of_65_to_72_bits():
    rng = np.random.default_rng(41)
    for half in (2700.0, 4200.0, 8388.0):
        got = _check(_stack([_paired(rng, np.full(3, half), 120)]), what=f"half range {half}")
        fr = xw.read_ints(got)[0]
        assert xw.sizeofints([b - a + 1 for a, b in zip(fr.minint, fr.maxint)]) > 64


def test_oracle_parity_corners():
    rng = np.random.default_rng(51)
    _check(np.full((20, 3, 2), 1.234, np.float32), what="all atoms identical")
    _check(-np.abs(_stack([rng.normal(0, 2, size=(200, 3)) for _ in range(2)])) - 0.3, what="negative coordinates")
    _check(_stack([rng.uniform(-2000, 2000, size=(50, 3)) for _ in range(2)]), what="first small range near the table's end")
    _check(_stack([rng.normal(0, 300, size=(300, 3)) for _ in range(2)]), 1e4, what="spread at precision 1e4")


def test_oracle_parity_large():
    """50 000 atoms x 8 frames of water in an 8 nm box"""
    rng = np.random.default_rng(61)
    w = np.concatenate([xc._water(rng, 16_666, 8.0), rng.uniform(0, 8, size=(2, 3))])
    _check(_stack([w + rng.normal(0, 0.02 * (f + 1), size=w.shape) for f in range(8)]), what="large")


# ----------------------------------------------------------------------------------------- 3. round trip through K11
def _lattice_floats(coords, precision):
    p = np.float32(precision)
    lf = coords * p
    ints = np.where(coords >= 0, lf + np.float32(0.5), lf - np.float32(0.5)).astype(np.float32).astype(np.int64)
    return ints.astype(np.float32) * np.float32(1.0 / np.float64(p))


def _water_trajectory(N, F, seed):
    """(N, 3, F) float32 on the device: three-atom waters in a 4 nm box, every molecule on a random walk of its own
    (0.01 nm per frame) with 0.005 nm of per-atom jitter"""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    nm = (N + 2) // 3
    o = torch.rand((nm, 1, 3), generator=g, device="cuda") * 4.0
    mol = torch.cat([o, o + 0.06 * torch.randn((nm, 2, 3), generator=g, device="cuda")], 1)
    walk = torch.cumsum(0.01 * torch.randn((nm, 1, 3, F), generator=g, device="cuda"), dim=3)
    jitter = 0.005 * torch.randn((nm, 3, 3, F), generator=g, device="cuda")
    return (mol[..., None] + walk + jitter).reshape(3 * nm, 3, F)[:N].contiguous()


@pytest.mark.parametrize("precision", [1000.0, 100.0])
def test_round_trip_and_idempotence(tmp_path, precision):
    from moleculekit_b200 import xtc as px

    rng = np.random.default_rng(71)
    w = xc._water(rng, 300, 4.0) - 2.0
    coords = _stack([w + rng.normal(0, 0.03, size=w.shape) * np.sqrt(f + 1) for f in range(70)])
    box, time, step = _headers(70)
    fn = str(tmp_path / "rt.xtc")
    px.write_xtc(fn, coords, box, time, step, precision=precision)
    back, box2, time2, step2 = px.read_xtc(fn)
    want = _lattice_floats(coords, precision)
    assert np.array_equal(back.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(box2, box) and np.array_equal(time2, time) and np.array_equal(step2, step)
    assert px.xtc_bytes(back, box, time, step, precision=precision) == open(fn, "rb").read()


def test_round_trip_at_trajectory_size(tmp_path):
    """5 000 atoms x 2 000 frames, generated on the device: too much for the Python oracle, so the checks are the exact
    round trip through K11, idempotence and the length table"""
    import torch
    from moleculekit_b200 import xtc as px

    N, F = 5000, 2000
    coords = _water_trajectory(N, F, seed=5)
    blocks, offsets, lengths = px.encode_xtc_device(coords)
    assert blocks.dtype == torch.uint8 and blocks.is_cuda and offsets.shape == lengths.shape == (F,)
    assert int(lengths.sum()) == blocks.numel()
    assert torch.equal(offsets, torch.cumsum(lengths.long(), 0) - lengths)
    assert blocks.numel() < 0.45 * coords.numel() * 4  # the writer finds the runs of a solvated system
    box, time, step = _headers(F)
    fn = str(tmp_path / "big.xtc")
    px.write_xtc(fn, coords, box, time, step)
    assert os.path.getsize(fn) == 56 * F + blocks.numel()
    back, _, _, step2 = px.read_xtc_device(fn)
    want = _lattice_floats(coords.cpu().numpy(), 1000.0)
    assert np.array_equal(back.cpu().numpy().view(np.uint32), want.view(np.uint32)) and np.array_equal(step2, step)
    again, _, lengths2 = px.encode_xtc_device(back)
    assert torch.equal(again, blocks) and torch.equal(lengths2, lengths)


# ----------------------------------------------------------------------------------------- 4. inputs and errors
def _small(F=5, seed=81):
    rng = np.random.default_rng(seed)
    w = xc._water(rng, 30, 3.0) * 10 - 15  # Angstrom-sized numbers, both signs
    return _stack([w + rng.normal(0, 0.4, size=w.shape) for _ in range(F)])


def test_tensor_and_numpy_inputs_agree_and_scale_is_a_first_multiplication():
    import torch
    from moleculekit_b200 import xtc as px

    c = _small()
    box, time, step = _headers(c.shape[2])
    ref = px.xtc_bytes(c, box, time, step)
    assert px.xtc_bytes(torch.from_numpy(c).cuda(), box, time, step) == ref == xw.write_xtc(c, box, time, step)
    scaled = px.xtc_bytes(c, box, time, step, scale=0.1)
    assert scaled == px.xtc_bytes(c * np.float32(0.1), box, time, step) != ref
    with pytest.raises(ValueError):  # (natoms, 3, F) is required of tensors as well
        px.xtc_bytes(torch.from_numpy(c).cuda()[:, :2], box, time, step)
    with pytest.raises(ValueError):
        px.encode_xtc_device(torch.from_numpy(c).cuda().double())


def test_a_frame_beyond_the_lattice_limit_raises_and_names_the_frame():
    from moleculekit_b200 import xtc as px

    c = _small()
    box, time, step = _headers(c.shape[2])
    good = px.xtc_bytes(c, box, time, step)
    bad = c.copy()
    bad[7, 1, 3] = 3e6  # 3e9 lattice steps
    with pytest.raises(RuntimeError, match="Internal overflow compressing coordinates: frame 3"):
        px.xtc_bytes(bad, box, time, step)
    bad = c.copy()
    bad[:45, 0, 2], bad[45:, 0, 2] = -1.0e6, 1.2e6  # each fits, their range does not
    with pytest.raises(RuntimeError, match="Internal overflow compressing coordinates: frame 2"):
        px.xtc_bytes(bad, box, time, step)
    bad = c.copy()
    bad[:, :, 4] = (np.arange(90)[:, None] * np.array([[3000.0, 0, 0]])).astype(np.float32)
    with pytest.raises(RuntimeError, match="frame 4"):  # the oracle refuses this one too ("past its table")
        px.xtc_bytes(bad, box, time, step)
    with pytest.raises(ValueError, match="past its table"):
        xw.write_xtc(bad[:, :, 4:], box[:, :, 4:], time[4:], step[4:])
    assert px.xtc_bytes(c, box, time, step) == good  # the next call is unaffected


def _abi_encode(coords_view, stride, natoms, F, capacity, precision=1000.0, scale=1.0):
    import torch
    from moleculekit_b200 import _lib

    dev = coords_view.device
    blocks = torch.full((capacity + 8,), 0xAB, dtype=torch.uint8, device=dev)
    offsets = torch.zeros(max(F, 0) + 1, dtype=torch.int64, device=dev)
    lengths = torch.zeros(max(F, 0), dtype=torch.int32, device=dev)
    status = torch.zeros(max(F, 0), dtype=torch.int32, device=dev)
    h = _lib.handle(dev.index)
    rc = _lib.load().mkb_xtc_encode(h, _lib.stream(dev), _lib.ptr(coords_view), stride, F, natoms, C.c_float(precision),
                                    C.c_float(scale), _lib.ptr(blocks), capacity, _lib.ptr(offsets), _lib.ptr(lengths),
                                    _lib.ptr(status))
    torch.cuda.synchronize()
    return rc, blocks, offsets, lengths, status, _lib.load().mkb_last_error(h).decode()


def test_abi_strided_view_capacity_and_argument_checks():
    import torch
    from moleculekit_b200 import xtc as px

    c = _small(F=9)
    N, _, F = c.shape
    want, woff, wlen = px.encode_xtc_device(torch.from_numpy(c).cuda())
    total = want.numel()
    wide = torch.full((N, 3, F + 7), 1e9, dtype=torch.float32, device="cuda")  # the frames beyond F would overflow
    wide[:, :, :F] = torch.from_numpy(c).cuda()
    rc, blocks, offsets, lengths, status, _ = _abi_encode(wide, F + 7, N, F, total)
    assert rc == 0 and int(status.abs().sum()) == 0 and int(offsets[F]) == total
    assert torch.equal(blocks[:total], want) and bool((blocks[total:] == 0xAB).all())  # nothing beyond the last block
    assert torch.equal(offsets[:F], woff) and torch.equal(lengths, wlen)
    # too small: MKB_ERR_CAPACITY, nothing written, the tables and the required size filled in
    for cap in (0, 8, total - 4):
        rc, blocks, offsets, lengths, status, msg = _abi_encode(wide, F + 7, N, F, cap)
        assert rc == -4 and str(total) in msg and int(offsets[F]) == total and torch.equal(lengths, wlen)
        assert bool((blocks == 0xAB).all())
    # argument checks
    assert _abi_encode(wide, F - 1, N, F, total)[0] == -1   # frame stride < n_frames
    assert _abi_encode(wide, F + 7, N, -1, total)[0] == -1  # negative size
    assert _abi_encode(wide, F + 7, -1, F, total)[0] == -1
    rc, blocks, _, _, _, _ = _abi_encode(wide, F + 7, N, 0, total)  # zero frames: MKB_OK, nothing touched
    assert rc == 0 and bool((blocks == 0xAB).all())
