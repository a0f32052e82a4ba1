"""C12: aligned coordinate features, frame sums and fluctuations (K15) on one GPU.  Prints one JSON line.

Workload: bench_align.py's C12 -- 59 000 atoms (a 5 000-atom rigid solute under a per-frame random rotation,
translation and 0.5 A noise, plus 18 000 three-atom waters over five box lengths) over 2 000 frames, generated on the
device from a seed.  The fit uses 1 000 solute atoms; coordinates, frame sums and fluctuations cover all 5 000.

Reported: the coordinate, frame-sum and fluctuation kernel times from the library's CUDA events (with the fit records
applied on the fly), their algorithmic bytes (coordinates: 12 B read + 12 B written per selected atom-frame; sums: 12 B
read; fluctuation: 12 B read + 4 B written per output atom-frame) and the share of the H100 SXM data sheet's 3.35 TB/s;
MetricCoordinate.project (with a reference) and MetricFluctuation.project (mean structure) end to end from host arrays;
and the reference's float32 numpy path on one CPU core (per frame fit + superpose all atoms + gather for the
coordinates; mean + squared deviations for the fluctuations; no wrapping), timed on a subset of frames and scaled to the
whole trajectory.  The GPU's name and power limit are read in the same run.

    python bench_coords.py [--frames 2000] [--reps 10] [--cpu-frames 20] [--seed 12]
"""
from __future__ import annotations

import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):  # the CPU reference runs on one core
    os.environ.setdefault(_v, "1")

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_align import PEAK_BYTES_S, c12, gpu_info  # noqa: E402


def reference_coordinates(X, ref, aln, sel, frames):
    """moleculekit's float32 sequence per frame: fit (_pp_measure_fit), superpose all atoms (_pp_align), then the
    selection's coordinates as one row (MetricCoordinate's gather and transpose)."""
    out = np.empty((len(frames), 3 * len(sel)), np.float32)
    Q = ref[aln, :, 0]
    for i, f in enumerate(frames):
        P = X[aln, :, f]
        pc, qc = P.mean(0), Q.mean(0)
        V, _, W = np.linalg.svd(np.dot((P - pc).T, Q - qc))
        if np.linalg.det(V) * np.linalg.det(W) < 0:
            V[:, -1] = -V[:, -1]
        moved = np.dot(X[:, :, f] - pc, np.dot(V, W)) + qc
        out[i] = moved[sel].T.reshape(-1)
    return out


def reference_fluctuation(X, sel, frames):
    """the mean structure and squared deviations in float32 numpy (MetricFluctuation without a reference, no wrap)"""
    C = X[sel][:, :, frames]
    m = C.mean(axis=2)
    return np.sum((C - m[:, :, None]) ** 2, axis=1).T


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-frames", type=int, default=20)
    ap.add_argument("--seed", type=int, default=12)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_coords.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200.align import superpose_device
    from moleculekit_b200.coords import coord_sums_device, coordinates_device, fluctuation_device
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    F, n_sol = a.frames, 5000
    X, ref, bonds, box = c12(dev, a.seed, F)
    N = X.shape[0]
    aln_idx = np.arange(0, n_sol, 5, dtype=np.int32)
    sel_idx = np.arange(n_sol, dtype=np.int32)
    d_aln, d_sel = torch.from_numpy(aln_idx).to(dev), torch.from_numpy(sel_idx).to(dev)
    d_ref = torch.cat([ref, torch.zeros((N - n_sol, 3, 1), device=dev)]).contiguous()
    rec, st = superpose_device(X, d_aln, d_ref, d_aln)
    assert int(st.sum().item()) == 0
    k = len(sel_idx)
    out = torch.empty((F, 3 * k), device=dev)
    fl = torch.empty((F, k), device=dev)

    _lib.set_timing(True, 0)
    t_co, t_sum, t_fl = [], [], []
    for it in range(a.reps + 2):
        coordinates_device(X, d_sel, rec, out=out)
        _, co_ms = _lib.get_timing(0)
        sums = coord_sums_device(X, d_sel, rec)
        _, sum_ms = _lib.get_timing(0)
        fluctuation_device(X, d_sel, sums / F, rec, out=fl)
        _, fl_ms = _lib.get_timing(0)
        if it >= 2:
            t_co.append(co_ms); t_sum.append(sum_ms); t_fl.append(fl_ms)
    _lib.set_timing(False, 0)

    def kern(ms_list, nbytes):
        ms = float(np.median(ms_list))
        return dict(ms=ms, ms_min=float(np.min(ms_list)), ms_max=float(np.max(ms_list)), algorithmic_bytes=nbytes,
                    gbs=nbytes / (ms * 1e-3) / 1e9, frac_of_peak=nbytes / (ms * 1e-3) / PEAK_BYTES_S)

    coords_k = kern(t_co, 24 * k * F)
    sums_k = kern(t_sum, 12 * k * F)
    fluct_k = kern(t_fl, 16 * k * F)

    # end to end from host arrays: upload, wrap around the solute, (fit,) K15, result back
    host = X.cpu().numpy()
    solute = np.arange(N) < n_sol
    aln_mask = np.zeros(N, bool)
    aln_mask[aln_idx] = True
    mol = MolLite(host, box=box.cpu().numpy(), bonds=bonds, named_selections={"solute": solute, "aln": aln_mask})
    refmol = MolLite(d_ref.cpu().numpy(), named_selections={"solute": solute, "aln": aln_mask})
    e2e = {}
    for name, m in (("metriccoordinate_project_e2e", MetricCoordinate("solute", refmol=refmol, trajalnsel="aln",
                                                                        centersel="solute")),
                    ("metricfluctuation_project_e2e", MetricFluctuation("solute", centerstr="solute"))):
        res = m.project(mol)
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = m.project(mol)
            times.append(time.perf_counter() - t0)
        s = float(np.median(times))
        e2e[name] = dict(s=s, s_min=float(np.min(times)), s_max=float(np.max(times)), frames_per_s=F / s,
                         host_bytes_up=host.nbytes, host_bytes_down=res.nbytes)

    # the reference's float32 numpy path on one core, on a subset of frames, scaled
    sub = np.linspace(0, F - 1, a.cpu_frames).astype(int)
    ref_h = d_ref.cpu().numpy()
    t0 = time.perf_counter()
    cpu_co = reference_coordinates(host, ref_h, aln_idx, sel_idx, sub)
    cpu_co_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    reference_fluctuation(host, sel_idx, sub)
    cpu_fl_s = time.perf_counter() - t0
    gpu_co = out[torch.from_numpy(sub).to(dev)].cpu().numpy()

    line = dict(
        bench="C12 aligned coordinates and fluctuations (K15)", gpu=card,
        workload=dict(atoms=N, frames=F, solute=n_sol, waters=18000, fit_atoms=len(aln_idx), selected_atoms=k,
                      seed=a.seed),
        peak_bytes_per_s=PEAK_BYTES_S, reps=a.reps,
        coordinates=coords_k, frame_sums=sums_k, fluctuation=fluct_k, **e2e,
        reference_cpu_float32=dict(
            kind="scaled", frames_timed=len(sub), threads=1,
            coordinates_s_scaled=cpu_co_s / len(sub) * F, fluctuation_s_scaled=cpu_fl_s / len(sub) * F,
            speedup_coordinates_e2e=cpu_co_s / len(sub) * F / e2e["metriccoordinate_project_e2e"]["s"]),
        coordinates_vs_reference_max_abs=float(np.max(np.abs(gpu_co - cpu_co))),
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
