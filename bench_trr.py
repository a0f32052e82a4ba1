"""GROMACS TRR reading and writing on one GPU (K24).  Prints one JSON line.

Workload: 100 000 atoms x 1 000 frames (1.2 GB of float32 per block) of seeded random-walk motion with a box that
breathes from frame to frame, built on the device (bench_dcd.random_walk, so the formats' kernels compare directly);
velocities and forces are derived from it on the device.

Reported: the card's name and power limit; from the library's CUDA events (median of --reps after 2 warm-up calls) the
single- and double-precision decode kernels and the encode kernel for x alone and for x+v+f, with the bytes they move
per atom-frame and block and their share of 3.35 TB/s (H100 SXM HBM3, data sheet); write_trr and read_trr_device end
to end for x alone and for x+v+f, each file having just been written, so it sits in the page cache; and the host
baseline: oracle/trr_format.py's reader (a Python / numpy restatement of xdrfile's layout, not the reference's binary)
plus the (F, N, 3) -> (N, 3, F) transposition on one core.

    python bench_trr.py [--atoms 100000] [--frames 1000] [--reps 10] [--seed 24] [--out DIR] [--no-host]
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
from bench_dcd import HBM_BYTES_PER_S, kernel_ms, random_walk, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=100000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=24)
    ap.add_argument("--out", default=None, help="directory for the files write_trr writes (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trr.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import trr as pt

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, lengths = random_walk(dev, N, F, a.seed)
    vel = coords * 0.5 - 25.0
    frc = coords * -2.0 + 7.0
    box = np.zeros((3, 3, F), np.float32)
    for d in range(3):
        box[d, d] = lengths[d]
    ftime, fstep = np.arange(F, dtype=np.float32) * 2.0, np.arange(F) * 1000
    af = N * F

    # encode: the whole trajectory into one device buffer of records, x alone and x+v+f
    enc_ms, recs = {}, {}
    for name, (v, f) in (("x", (None, None)), ("xvf", (vel, frc))):
        head = torch.from_numpy(pt._heads(N, F, box, ftime, fstep, None, v is not None, f is not None)).to(dev)
        R = pt.HEAD.itemsize + 12 * N * (1 if v is None else 3)
        enc = torch.empty(F * R, dtype=torch.uint8, device=dev)
        enc_ms[name] = kernel_ms(lambda: pt._encode(coords, v, f, head, N, F, out=enc), a.reps)
        recs[name] = (enc, R)

    # single-precision decode of x from the x-only records: frame k's x at k * R + 120
    enc, R = recs["x"]
    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    offsets = np.arange(F, dtype=np.int64) * R + pt.HEAD.itemsize
    dec4_ms = kernel_ms(lambda: pt.decode_trr_device(enc, offsets, N, 4, out=dec), a.reps)
    assert torch.equal(dec.view(torch.int32), coords.view(torch.int32))
    del recs, enc
    # double-precision decode: the same values as big-endian float64 blocks of 24 N bytes, one per frame
    be64 = coords.permute(2, 0, 1).contiguous().double().view(torch.uint8).reshape(-1, 8).flip(1).reshape(-1)
    offsets = np.arange(F, dtype=np.int64) * 24 * N
    dec8_ms = kernel_ms(lambda: pt.decode_trr_device(be64, offsets, N, 8, out=dec), a.reps)
    assert torch.equal(dec.view(torch.int32), coords.view(torch.int32))  # float32 -> float64 -> float32 is exact
    del be64, dec

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    write_s, read_s, file_bytes = {}, {}, {}
    for name, (v, f, fields) in (("x", (None, None, ("x",))), ("xvf", (vel, frc, ("x", "v", "f")))):
        fn = os.path.join(a.out, f"bench_trr_{name}.trr")
        write_s[name], read_s[name] = [], []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pt.write_trr(fn, coords, box, ftime, fstep, velocities=v, forces=f)
            write_s[name].append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            back, bbox, _ = pt.read_trr_device(fn, fields=fields)
            torch.cuda.synchronize()
            read_s[name].append(time.perf_counter() - t0)
            assert torch.equal(back["x"].view(torch.int32), coords.view(torch.int32)) and np.array_equal(bbox, box)
            del back
        file_bytes[name] = os.path.getsize(fn)
        if name == "x" and not a.no_host:
            from oracle import trr_format as tf

            t0 = time.perf_counter()
            with open(fn, "rb") as fh:
                frames = tf.read(fh.read())["frames"]
            xyz = np.stack([fr["x"] for fr in frames])
            t1 = time.perf_counter()
            x = np.ascontiguousarray(xyz.transpose(1, 2, 0))
            t2 = time.perf_counter()
            assert np.array_equal(x.view(np.int32), coords.cpu().numpy().view(np.int32))
            host = dict(what="oracle/trr_format.py read of the file (to native float32 (F, N, 3)) and the (F, N, 3) -> "
                             "(N, 3, F) transposition, one core", read_s=t1 - t0, transpose_s=t2 - t1, total_s=t2 - t0)
            del frames, xyz, x
        os.remove(fn)
    if tmp is not None:
        tmp.cleanup()

    def share(ms, moved):
        return moved * af / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="GROMACS TRR read / write (K24)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, float32_bytes_per_block=12 * af, file_bytes=file_bytes),
        reps=a.reps,
        bytes_per_atom_frame=dict(decode_single=dict(read=12, written=12), decode_double=dict(read=24, written=12),
                                  encode_x=dict(read=12, written=12), encode_xvf=dict(read=36, written=36)),
        decode_single_kernel_ms=stats(dec4_ms), decode_single_hbm_share=share(dec4_ms, 24),
        decode_double_kernel_ms=stats(dec8_ms), decode_double_hbm_share=share(dec8_ms, 36),
        encode_x_kernel_ms=stats(enc_ms["x"]), encode_x_hbm_share=share(enc_ms["x"], 24),
        encode_xvf_kernel_ms=stats(enc_ms["xvf"]), encode_xvf_hbm_share=share(enc_ms["xvf"], 72),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_trr_x_s=stats(write_s["x"]), read_trr_device_x_s=stats(read_s["x"]),
        write_trr_xvf_s=stats(write_s["xvf"]), read_trr_device_xvf_s=stats(read_s["xvf"]),
        read_note="read_trr_device right after write_trr: the file sits in the page cache",
        host_baseline=host if not a.no_host else "not measured",
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
