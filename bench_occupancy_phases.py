"""Where the time of one 8-channel occupancy step goes, on one GPU.  Prints one JSON line.

Workloads: C3 (256 protein pockets x ~3000 atoms, 64^3 @ 1 A, bench.py's headline), C2 (1024 ligand poses x 50 atoms,
24^3 @ 1 A) and C5 (4 fine grids at 0.5 A), the sizes bench.py times, inputs resident on the device, through
VoxelBatch.run.

Reported per workload: the step time, the median over windows of back-to-back steps that each last at least 200 ms
(CUDA events, profiler off); and from torch.profiler with CUDA activities, in a pass of its own, the mean device time
per step of every kernel, memset and copy, grouped into phases:
  upload     descriptor copy
  memset     tile counts and block bits, band bitmap, queue and fix-list header
  band       occ_band_kernel (gate-band pre-pass, on a side stream beside the list build for large batches)
  prep       occ_prep_kernel (records + per-tile counts and block bits)
  scan       cub ExclusiveSum of the counts
  list_fill  occ_blk_fill_kernel (candidate lists)
  fill       occ_fill_runs_kernel
  fix        occ_fix_list_kernel / occ_fix_scan_kernel
list_build = prep + scan + list_fill.  The phases of the band pre-pass and the list build overlap, so their sum can
exceed the step.  The GPU's name and power limit are read in the same run.

    python bench_occupancy_phases.py [--reps 5] [--window-ms 200] [--profile-steps 10] [--workloads c3,c2,c5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_align import gpu_info  # noqa: E402

PHASES = (("occ_band_kernel", "band"), ("occ_prep_kernel", "prep"), ("occ_blk_fill_kernel", "list_fill"),
          ("occ_fill_runs_kernel", "fill"), ("occ_fix_", "fix"), ("Scan", "scan"), ("emset", "memset"),
          ("Memcpy", "upload"))


def phase_of(name: str) -> str:
    for key, ph in PHASES:
        if key in name:
            return ph
    return "other"


def make(kind: str):
    from moleculekit_b200 import workloads

    if kind == "c3":
        return workloads.protein_pockets(B=256, seed=1000)
    if kind == "c2":
        return workloads.ligand_poses(B=1024)
    return workloads.fine_grids(B=4)


def run(kind: str, a, dev):
    from torch.profiler import ProfilerActivity, profile

    from moleculekit_b200.tools import voxeldescriptors as vd

    w = make(kind)
    vb = vd.VoxelBatch(w["coords"], w["sigmas"], boxsize=w["boxsize"], centers=w["centers"], voxelsize=w["voxelsize"])
    d_c, d_s = vb.to_device(dev)
    out = torch.empty((vb.total_voxels, vb.C), dtype=torch.float32, device=dev)
    step = lambda: vb.run(d_c, d_s, out)  # noqa: E731
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    step()
    e1.record()
    e1.synchronize()
    steps = max(1, int(np.ceil(a.window_ms / max(e0.elapsed_time(e1), 1e-3))))
    ts = []
    for _ in range(a.reps):
        e0.record()
        for _ in range(steps):
            step()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / steps)
    n = a.profile_steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    kernels, phases = {}, {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA" or ev.count == 0:
            continue
        ms = ev.device_time_total / 1e3 / n
        kernels[ev.key[:120]] = dict(ms_per_step=ms, calls_per_step=ev.count / n)
        ph = phase_of(ev.key)
        phases[ph] = phases.get(ph, 0.0) + ms
    lb = sum(phases.get(p, 0.0) for p in ("prep", "scan", "list_fill"))
    step_ms = float(np.median(ts))
    return dict(workload=w["name"], items=vb.B, atoms=int(vb.coords.shape[0]), voxel_channels=int(vb.total_voxels * vb.C),
                step_ms=step_ms, step_ms_min=float(np.min(ts)), step_ms_max=float(np.max(ts)), steps_per_window=steps,
                phase_ms=phases, list_build_ms=lb, outside_fill_ms=step_ms - phases.get("fill", 0.0), kernels=kernels)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=5, help="timed windows per workload")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--profile-steps", type=int, default=10)
    ap.add_argument("--workloads", default="c3,c2,c5")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_occupancy_phases.py needs a CUDA device: nothing is measured without one")
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = gpu_info(0)
    res = [run(k, a, dev) for k in a.workloads.split(",")]
    print(json.dumps(dict(bench="occupancy step phases (K1 + K2')", gpu=card, workloads=res)), flush=True)


if __name__ == "__main__":
    main()
