"""AMBER NetCDF reading and writing on one GPU (K23).  Prints one JSON line.

Workload: 100 000 atoms x 1 000 frames (1.2 GB of float32) of seeded random-walk motion with a unit cell that breathes
from frame to frame, built on the device: the shape of bench_dcd.py, so the two formats' kernels compare directly.

Reported: the card's name and power limit; the decode and encode kernels from the library's CUDA events (median of
--reps after 2 warm-up calls), the bytes they move per atom-frame (12 read, 12 written) and their share of 3.35 TB/s
(H100 SXM HBM3, data sheet); write_netcdf and read_netcdf_device end to end, the file having just been written, so it
sits in the page cache; and the host baseline: scipy.io.netcdf_file reading the coordinates plus the
(F, N, 3) -> (N, 3, F) transposition on one core.

    python bench_netcdf.py [--atoms 100000] [--frames 1000] [--reps 10] [--seed 23] [--out DIR] [--no-host]
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
    ap.add_argument("--seed", type=int, default=23)
    ap.add_argument("--out", default=None, help="directory for the file write_netcdf writes (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_netcdf.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import netcdf as pn

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, box = random_walk(dev, N, F, a.seed)
    af = N * F
    moved = 24 * af  # 12 bytes read and 12 written per atom-frame

    # encode: the whole trajectory into one device buffer of records (time, coordinates, cell_lengths, cell_angles)
    extra = torch.from_numpy(pn._extra(F, box, None, None)).to(dev)
    record_bytes, coord_offset = pn._record_layout(N, True)
    enc = torch.empty(F * record_bytes, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pn._encode(coords, extra, N, F, True, out=enc), a.reps)

    # decode from the encoded records: frame k's coordinates at k * record_bytes + coord_offset
    offsets = np.arange(F, dtype=np.int64) * record_bytes + coord_offset
    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    dec_ms = kernel_ms(lambda: pn.decode_netcdf_device(enc, offsets, N, out=dec), a.reps)
    assert torch.equal(dec.view(torch.int32), coords.view(torch.int32))
    del enc, dec

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench_netcdf.nc")
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pn.write_netcdf(fn, coords, box)
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, bbox, _, _ = pn.read_netcdf_device(fn)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), coords.view(torch.int32)) and np.array_equal(bbox, box)
        del back
    file_bytes = os.path.getsize(fn)

    host = None
    if not a.no_host:
        from scipy.io import netcdf_file

        t0 = time.perf_counter()
        f = netcdf_file(fn, "r", mmap=False)
        xyz = np.asarray(f.variables["coordinates"].data, dtype=np.float32)  # big-endian -> native
        f.close()
        t1 = time.perf_counter()
        x = np.ascontiguousarray(xyz.transpose(1, 2, 0))
        t2 = time.perf_counter()
        assert np.array_equal(x.view(np.int32), coords.cpu().numpy().view(np.int32))
        host = dict(what="scipy.io.netcdf_file read of the coordinates (to native float32) and the (F, N, 3) -> "
                         "(N, 3, F) transposition, one core",
                    read_s=t1 - t0, transpose_s=t2 - t1, total_s=t2 - t0)
        del xyz, x
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()

    def share(ms):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="AMBER NetCDF read / write (K23)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, float32_bytes=12 * af, file_bytes=file_bytes),
        reps=a.reps, bytes_per_atom_frame=dict(read=12, written=12),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_netcdf_s=stats(write_s), read_netcdf_device_s=stats(read_s),
        read_note="read_netcdf_device right after write_netcdf: the file sits in the page cache",
        host_baseline=host if host is not None else "not measured",
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
