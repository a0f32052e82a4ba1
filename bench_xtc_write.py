"""XTC writing on one GPU (K21).  Prints one JSON line.

Workload: a water-like trajectory built on the device from a seed -- three-atom molecules (O at random in a cubic box,
two H within ~0.1 nm, the recipe of oracle/xtc_cases.py::_water), every molecule on a random walk of its own plus a
small per-atom jitter, 5 000 atoms x 10 000 frames by default.  It compresses like a solvated system: the writer finds
its runs of three atoms.  A uniform random cloud would not exercise them.

Reported: the card's name and power limit; the two passes of mkb_xtc_encode from the library's CUDA events after
warm-up (size pass with the scan and the read-back of the total; write pass); encode_xtc_device end to end (both passes,
allocation, status check); compressed bytes and their ratio to the float32 array; the encode followed by the one copy of
the packed blocks to the host; write_xtc end to end to a file in --out (that, plus the frame headers and the file
system); beside them the plain coords.cpu() copy that this path avoids; and, from decoding the file again with
read_xtc_device, the largest distance to the input in lattice steps (must be <= 0.5).  There is no CPU reference time:
the reference writer is not available here and the Python oracle is not a fair baseline.

    python bench_xtc_write.py [--atoms 5000] [--frames 10000] [--reps 10] [--seed 21] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_align import gpu_info  # noqa: E402


def water_trajectory(dev, N: int, F: int, seed: int, L: float = 4.0):
    """(N, 3, F) float32 on dev, in nm"""
    g = torch.Generator(device=dev).manual_seed(seed)
    nm = (N + 2) // 3
    o = torch.rand((nm, 1, 3), generator=g, device=dev) * L
    mol = torch.cat([o, o + 0.06 * torch.randn((nm, 2, 3), generator=g, device=dev)], 1)
    out = torch.empty((3 * nm, 3, F), dtype=torch.float32, device=dev).view(nm, 3, 3, F)
    chunk = 1000  # frames at a time: the generator's temporaries stay small beside the trajectory
    pos = torch.zeros((nm, 1, 3, 1), device=dev)
    for f0 in range(0, F, chunk):
        n = min(chunk, F - f0)
        walk = pos + torch.cumsum(0.01 * torch.randn((nm, 1, 3, n), generator=g, device=dev), dim=3)
        out[..., f0:f0 + n] = mol[..., None] + walk + 0.005 * torch.randn((nm, 3, 3, n), generator=g, device=dev)
        pos = walk[..., -1:].clone()
    return out.view(3 * nm, 3, F)[:N].contiguous()


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(np.min(xs)), max=float(np.max(xs)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=5000)
    ap.add_argument("--frames", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=21)
    ap.add_argument("--precision", type=float, default=1000.0)
    ap.add_argument("--out", default=None, help="directory for the file write_xtc writes (default: a temporary one)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_xtc_write.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200 import xtc as px

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords = water_trajectory(dev, N, F, a.seed)
    raw_bytes = coords.numel() * 4
    box = np.repeat((np.eye(3, dtype=np.float32) * 4.0)[:, :, None], F, axis=2)
    tm, step = np.arange(F, dtype=np.float32) * 0.1, np.arange(F, dtype=np.int32) * 100

    _lib.set_timing(True, 0)
    size_ms, write_ms, e2e_ms = [], [], []
    for it in range(a.reps + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        blocks, offsets, lengths = px.encode_xtc_device(coords, precision=a.precision)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        s_ms, w_ms = _lib.get_timing(0)
        if it >= 2:
            size_ms.append(s_ms); write_ms.append(w_ms); e2e_ms.append((t1 - t0) * 1e3)
    _lib.set_timing(False, 0)
    comp_bytes = int(blocks.numel())

    # the device's share of write_xtc: both passes and the one copy of the packed blocks to the host
    to_host_s = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_blocks = px.encode_xtc_device(coords, precision=a.precision)[0].cpu()
        to_host_s.append(time.perf_counter() - t0)
    del host_blocks

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench_xtc_write.xtc")
    file_s, copy_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        px.write_xtc(fn, coords, box, tm, step, precision=a.precision)
        file_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = coords.cpu()
        copy_s.append(time.perf_counter() - t0)
    del host
    file_bytes = os.path.getsize(fn)

    back, _, _, step2 = px.read_xtc_device(fn)
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()
    err = float(((back - coords).abs().max() * a.precision).item())
    assert np.array_equal(step2, step) and file_bytes == comp_bytes + 56 * F
    assert err <= 0.505, f"decoded coordinates are {err} lattice steps from the input"

    line = dict(
        bench="XTC write (K21)", gpu=card,
        workload=dict(atoms=N, frames=F, precision=a.precision, seed=a.seed, float32_bytes=raw_bytes),
        reps=a.reps,
        size_pass_ms=stats(size_ms), write_pass_ms=stats(write_ms), encode_xtc_device_ms=stats(e2e_ms),
        compressed_bytes=comp_bytes, ratio_to_float32=comp_bytes / raw_bytes, bytes_per_atom_frame=comp_bytes / (N * F),
        atom_frames_per_s_both_passes=N * F / ((np.median(size_ms) + np.median(write_ms)) * 1e-3),
        encode_and_blocks_to_host_s=stats(to_host_s),
        write_xtc_to_file_s=stats(file_s), file_bytes=file_bytes,
        coords_cpu_copy_s=stats(copy_s),
        max_lattice_error=err,
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
