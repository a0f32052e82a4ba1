"""DCD reading and writing on one GPU (K22).  Prints one JSON line.

Workload: 100 000 atoms x 1 000 frames (1.2 GB of float32) of seeded random-walk motion with a unit cell that breathes
from frame to frame, built on the device.  A variant with every other atom fixed (the file layout of CHARMM / NAMD
runs with NAMNF > 0) exercises the gather path of the decoder: frame 0 holds all atoms, later frames the free half.

Reported: the card's name and power limit; the decode and encode kernels from the library's CUDA events (median of
--reps after 2 warm-up calls), the bytes they move per atom-frame (12 read, 12 written) and their share of 3.35 TB/s
(H100 SXM HBM3, data sheet); write_dcd and read_dcd_device end to end, the file having just been written, so it sits in
the page cache; and the host baseline: oracle/dcd_format.py's reader (a Python / numpy restatement of the plugin's
layout, not the reference's binary) plus the (F, N, 3) -> (N, 3, F) transposition on one core.

    python bench_dcd.py [--atoms 100000] [--frames 1000] [--reps 10] [--seed 22] [--out DIR] [--no-host]
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

HBM_BYTES_PER_S = 3.35e12


def random_walk(dev, N: int, F: int, seed: int, L: float = 100.0):
    """(N, 3, F) float32 on dev [Angstrom] and the box lengths (3, F) on the host"""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    pos = torch.rand((N, 3, 1), generator=g, device=dev) * L
    chunk = 100  # frames at a time: the generator's temporaries stay small beside the trajectory
    for f0 in range(0, F, chunk):
        n = min(chunk, F - f0)
        walk = pos + torch.cumsum(0.3 * torch.randn((N, 3, n), generator=g, device=dev), dim=2)
        out[:, :, f0:f0 + n] = walk
        pos = walk[:, :, -1:].clone()
    box = (L + np.sin(np.arange(F) / 50.0)[None, :] * np.array([[1.0], [0.5], [0.25]])).astype(np.float32)
    return out, box


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(np.min(xs)), max=float(np.max(xs)))


def kernel_ms(fn, reps: int):
    """main-kernel times (library CUDA events) of ``reps`` calls after 2 warm-up calls"""
    from moleculekit_b200 import _lib

    _lib.set_timing(True, 0)
    ms = []
    for it in range(reps + 2):
        fn()
        torch.cuda.synchronize()
        if it >= 2:
            ms.append(_lib.get_timing(0)[1])
    _lib.set_timing(False, 0)
    return ms


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=100000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=22)
    ap.add_argument("--out", default=None, help="directory for the file write_dcd writes (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dcd.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import dcd as pd
    from oracle import dcd_format

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, box = random_walk(dev, N, F, a.seed)
    af = N * F
    moved = 24 * af  # 12 bytes read and 12 written per atom-frame

    # encode: the whole trajectory into one device buffer of frame records
    cells = torch.from_numpy(pd.box_to_unitcell(box)).to(dev)
    enc = torch.empty(F * pd._frame_bytes(N, True), dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pd._encode(coords, cells, N, F, out=enc), a.reps)

    # decode from the encoded records (frame k at k * S, no header needed on the device)
    S = pd._frame_bytes(N, True)
    frames = np.zeros(F, pd.FRAME_DESC)
    frames["offset"] = np.arange(F)[:, None] * S + 56 + np.arange(3)[None, :] * (8 + 4 * N) + 4
    frames["count"] = N
    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    dec_ms = kernel_ms(lambda: pd.decode_dcd_device(enc, frames, N, out=dec), a.reps)
    assert torch.equal(dec.view(torch.int32), coords.view(torch.int32))

    # fixed atoms: every other atom fixed; frame 0 holds all atoms, later frames the free half (encoded separately)
    free = np.arange(0, N, 2)
    nf = len(free)
    first = pd._encode(coords[:, :, :1], None, N, 1)
    rest = pd._encode(coords[torch.from_numpy(free).to(dev)][:, :, 1:].contiguous(), None, nf, F - 1)
    fixed_buf = torch.cat([first, rest])
    ff = np.zeros(F, pd.FRAME_DESC)
    S0, S1 = pd._frame_bytes(N, False), pd._frame_bytes(nf, False)
    ff["offset"][0] = np.arange(3) * (8 + 4 * N) + 4
    ff["offset"][1:] = S0 + np.arange(F - 1)[:, None] * S1 + np.arange(3)[None, :] * (8 + 4 * nf) + 4
    ff["count"][0], ff["count"][1:] = N, nf
    slot = torch.from_numpy(pd._slot_map(N, free)).to(dev)
    fixed_dec_ms = kernel_ms(lambda: pd.decode_dcd_device(fixed_buf, ff, N, False, slot, nf, first, ff[:1], out=dec),
                             a.reps)
    want = coords.clone()
    fixed_mask = torch.ones(N, dtype=torch.bool, device=dev)
    fixed_mask[torch.from_numpy(free).to(dev)] = False
    want[fixed_mask] = coords[fixed_mask][:, :, :1]
    assert torch.equal(dec.view(torch.int32), want.view(torch.int32))
    del enc, fixed_buf, rest, want

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench_dcd.dcd")
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pd.write_dcd(fn, coords, box)
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, bbox, _, _ = pd.read_dcd_device(fn)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), coords.view(torch.int32)) and np.array_equal(bbox, box)
        del back
    file_bytes = os.path.getsize(fn)

    host = None
    if not a.no_host:
        t0 = time.perf_counter()
        with open(fn, "rb") as f:
            raw = f.read()
        o = dcd_format.read(raw)
        del raw
        t1 = time.perf_counter()
        x = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
        t2 = time.perf_counter()
        assert np.array_equal(x.view(np.int32), coords.cpu().numpy().view(np.int32))
        host = dict(what="oracle/dcd_format.py reader (a restatement in Python / numpy, not the reference's binary) "
                         "and the (F, N, 3) -> (N, 3, F) transposition, one core",
                    read_s=t1 - t0, transpose_s=t2 - t1, total_s=t2 - t0)
        del o, x
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()

    def share(ms):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="DCD read / write (K22)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, float32_bytes=12 * af, file_bytes=file_bytes,
                      fixed_variant=dict(free_atoms=nf, fixed_atoms=N - nf)),
        reps=a.reps, bytes_per_atom_frame=dict(read=12, written=12),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms),
        decode_fixed_atoms_kernel_ms=stats(fixed_dec_ms), decode_fixed_atoms_hbm_share=share(fixed_dec_ms),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_dcd_s=stats(write_s), read_dcd_device_s=stats(read_s),
        read_note="read_dcd_device right after write_dcd: the file sits in the page cache",
        host_baseline=host if host is not None else "not measured",
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
