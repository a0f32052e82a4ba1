"""K32 benchmark: LAMMPS dump trajectories of 50 000 atoms x 1 000 frames (``id type x y z``, ids shuffled per frame
and the same data sorted, plus an ``id type xs ys zs ix iy iz`` file read with unwrap=True).  Prints one JSON line:
the file sizes, the index, head, decode and encode kernel times (torch.profiler, each step in a run of its own) with
their share of the H100's 3.35 TB/s over the bytes the step must move, ``read_lammpstrj_device`` and
``write_lammpstrj`` end to end, and the oracle reader on one core over 10 frames, scaled to the file.  Files go to a
temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from moleculekit_b200 import lammpstrj  # noqa: E402
from oracle import lammpstrj_format as lf  # noqa: E402

HBM = 3.35e12


def _gpu():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name()


def _make(path, x, box, shuffle, scaled, rng):
    """one frame at a time through the writer: ids permuted per frame, or xs ys zs ix iy iz written as x y z and
    velocities with the ATOMS header renamed"""
    N, _, F = x.shape
    ids = np.arange(1, N + 1)
    with open(path, "wb") as fh:
        for f in range(F):
            p = rng.permutation(N) if shuffle else np.arange(N)
            xf = x[p, :, f:f + 1]
            img = None
            if scaled:
                img = np.floor(xf / 40.0).astype(np.float32)
                xf = (xf / np.float32(40.0) - img).astype(np.float32)
            raw = lammpstrj.lammpstrj_bytes(np.ascontiguousarray(xf), box, step=[f], ids=ids[p],
                                            velocities=None if img is None else np.ascontiguousarray(img))
            if scaled:
                raw = raw.replace(b"ITEM: ATOMS id type x y z vx vy vz", b"ITEM: ATOMS id type xs ys zs ix iy iz")
            fh.write(raw)


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out[e.key] = out.get(e.key, 0.0) + e.device_time_total * 1e-6
    return out


def _sum(k, *names):
    return sum(t for key, t in k.items() if any(n in key for n in names))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--atoms", type=int, default=50000)
    ap.add_argument("--frames", type=int, default=1000)
    args = ap.parse_args()
    N, F = args.atoms, args.frames
    rng = np.random.default_rng(0)
    x = rng.uniform(0, 40, (N, 3, F)).astype(np.float32)
    box = np.zeros((3, 3, 1), np.float32)
    box[0, 0] = box[1, 1] = box[2, 2] = 40.0
    res = dict(bench="lammpstrj", atoms=N, frames=F, gpu=_gpu())
    with tempfile.TemporaryDirectory() as tmp:
        files = {k: os.path.join(tmp, k + ".lammpstrj") for k in ("shuffled", "sorted", "scaled")}
        _make(files["shuffled"], x, box, True, False, rng)
        _make(files["sorted"], x, box, False, False, rng)
        _make(files["scaled"], x, box, True, True, rng)
        for name, fn in files.items():
            E = os.path.getsize(fn)
            unwrap = name == "scaled"
            idx = lammpstrj.index_lammpstrj(fn)  # warm-up: module load, page cache
            lammpstrj.read_lammpstrj_device(fn, index=idx, unwrap=unwrap)
            torch.cuda.synchronize()
            ki = _kernels(lambda: lammpstrj.index_lammpstrj(fn))
            kd = _kernels(lambda: lammpstrj.read_lammpstrj_device(fn, index=idx, unwrap=unwrap))
            t_index = _sum(ki, "xyz_count", "xyz_scan", "xyz_emit", "lt_check")
            t_head = _sum(ki, "lt_head")
            t_dec = _sum(kd, "xyz_count", "xyz_scan", "xyz_emit", "lt_parse")
            t0 = time.perf_counter()
            out, _, _ = lammpstrj.read_lammpstrj_device(fn, unwrap=unwrap)
            torch.cuda.synchronize()
            t_read = time.perf_counter() - t0
            with open(fn, "rb") as fh:
                head = fh.read(int(idx["offsets"][min(10, F)]))
            t0 = time.perf_counter()
            lf.read(head, unwrap=unwrap)
            t_oracle = (time.perf_counter() - t0) * F / min(10, F)
            res[name] = dict(bytes=E, index_ms=1e3 * t_index, index_hbm=E / t_index / HBM, head_ms=1e3 * t_head,
                             decode_ms=1e3 * t_dec, decode_hbm=(E + 12 * N * F) / t_dec / HBM,
                             read_device_s=t_read, oracle_1core_s=t_oracle)
            del out
        xd = torch.from_numpy(x).cuda()
        boxes = np.repeat(box, F, axis=2)
        enc = lammpstrj.encode_lammpstrj_device(xd[:, :, :10], boxes[:, :, :10])  # warm-up
        chunk = F // 4 or 1
        ke = _kernels(lambda: lammpstrj.encode_lammpstrj_device(xd[:, :, :chunk], boxes[:, :, :chunk]))
        nbytes = int(lammpstrj.encode_lammpstrj_device(xd[:, :, :chunk], boxes[:, :, :chunk]).numel())
        t_enc = _sum(ke, "lt_len", "lt_emit", "Scan")
        out_fn = os.path.join(tmp, "w.lammpstrj")
        t0 = time.perf_counter()
        lammpstrj.write_lammpstrj(out_fn, xd, boxes)
        torch.cuda.synchronize()
        t_write = time.perf_counter() - t0
        res["encode"] = dict(frames=chunk, bytes=nbytes, encode_ms=1e3 * t_enc,
                             encode_hbm=(nbytes + 12 * N * chunk) / t_enc / HBM, write_s=t_write,
                             written_bytes=os.path.getsize(out_fn))
        del enc
    print(json.dumps(res))


if __name__ == "__main__":
    main()
