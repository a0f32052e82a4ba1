"""C12: per-frame group moments (K20) for MetricGyration and MetricSphericalCoordinate on one GPU.  Prints one JSON line.

Workload: bench_align.py's C12 -- 59 000 atoms (a 5 000-atom rigid solute under a per-frame random rotation,
translation and 0.5 A noise, plus 18 000 three-atom waters over five box lengths) over 2 000 frames, generated on the
device from a seed.  The fit uses 1 000 solute atoms.  Two K20 calls, both with the fit records applied on the fly:
the mass-weighted radius of gyration of the 5 000 solute atoms (one group), and the spherical coordinate of a 50-atom
solute subset against the whole solute (two plain groups, 5 050 positions).

Reported: the K20 kernel times (partial + finish) from the library's CUDA events, medians of 10 after warm-up, their
algorithmic bytes (12 B read per selected atom-frame) and the share of the H100 SXM data sheet's 3.35 TB/s;
MetricGyration.project and MetricSphericalCoordinate.project end to end from host arrays (upload, wrap around the
solute, fit, K20, result back); and the reference's float32 numpy path on one CPU core (per frame fit, superpose all
atoms, then the weighted centre and spread of the selection; no wrapping), timed on a subset of frames and scaled to the
whole trajectory.  The GPU's name and power limit are read in the same run.

    python bench_moments.py [--frames 2000] [--reps 10] [--cpu-frames 20] [--seed 12]
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
from bench_coords import reference_coordinates  # noqa: E402


def reference_gyration(rows, masses):
    """the float32 numpy sequence on the reference's aligned rows (n, 3k): mass-weighted centre, then the per-axis
    spread around it and its square roots"""
    k = masses.size
    P = rows.reshape(rows.shape[0], 3, k)
    M = masses.sum()
    com = (P * masses).sum(axis=2) / M
    v = ((P - com[:, :, None]) ** 2 * masses).sum(axis=2) / M
    return np.column_stack([np.sqrt(v.sum(axis=1)), np.sqrt(v)])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-frames", type=int, default=20)
    ap.add_argument("--seed", type=int, default=12)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_moments.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200.align import superpose_device
    from moleculekit_b200.coords import frame_moments_device
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricgyration import MetricGyration, gyration_features
    from moleculekit_b200.projections.metricsphericalcoordinate import MetricSphericalCoordinate

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    F, n_sol, n_sub = a.frames, 5000, 50
    X, ref, bonds, box = c12(dev, a.seed, F)
    N = X.shape[0]
    aln_idx = np.arange(0, n_sol, 5, dtype=np.int32)
    sol_idx = np.arange(n_sol, dtype=np.int32)
    sub_idx = np.arange(0, n_sol, n_sol // n_sub, dtype=np.int32)[:n_sub]
    masses = np.tile(np.float32([14.0067, 12.0107, 12.0107, 15.9994, 1.00794]), N // 5 + 1)[:N]
    d_aln = torch.from_numpy(aln_idx).to(dev)
    d_ref = torch.cat([ref, torch.zeros((N - n_sol, 3, 1), device=dev)]).contiguous()
    rec, st = superpose_device(X, d_aln, d_ref, d_aln)
    assert int(st.sum().item()) == 0
    d_sol = torch.from_numpy(sol_idx).to(dev)
    w_sol = masses[sol_idx].astype(np.float64)
    d_sph = torch.from_numpy(np.concatenate([sol_idx, sub_idx])).to(dev)
    g_sph = np.array([0, n_sol, n_sol + n_sub], np.int64)

    _lib.set_timing(True, 0)
    t_rg, t_sph = [], []
    for it in range(a.reps + 2):
        rg_m = frame_moments_device(X, d_sol, rec, weights=w_sol)
        _, rg_ms = _lib.get_timing(0)
        frame_moments_device(X, d_sph, rec, groups=g_sph)
        _, sph_ms = _lib.get_timing(0)
        if it >= 2:
            t_rg.append(rg_ms); t_sph.append(sph_ms)
    _lib.set_timing(False, 0)

    def kern(ms_list, nbytes):
        ms = float(np.median(ms_list))
        return dict(ms=ms, ms_min=float(np.min(ms_list)), ms_max=float(np.max(ms_list)), algorithmic_bytes=nbytes,
                    gbs=nbytes / (ms * 1e-3) / 1e9, frac_of_peak=nbytes / (ms * 1e-3) / PEAK_BYTES_S)

    rg_k = kern(t_rg, 12 * n_sol * F)
    sph_k = kern(t_sph, 12 * (n_sol + n_sub) * F)

    # end to end from host arrays: upload, wrap around the solute, fit, K20, result back
    host = X.cpu().numpy()
    solute = np.arange(N) < n_sol
    aln_mask = np.zeros(N, bool)
    aln_mask[aln_idx] = True
    sub_mask = np.zeros(N, bool)
    sub_mask[sub_idx] = True
    names = {"solute": solute, "aln": aln_mask, "sub": sub_mask}
    mol = MolLite(host, box=box.cpu().numpy(), bonds=bonds, named_selections=names)
    mol.masses = masses
    refmol = MolLite(d_ref.cpu().numpy(), named_selections=names)
    e2e = {}
    for name, m in (("metricgyration_project_e2e", MetricGyration("solute", refmol=refmol, trajalnstr="aln",
                                                                   centerstr="solute")),
                    ("metricsphericalcoordinate_project_e2e",
                     MetricSphericalCoordinate(refmol, "sub", "solute", trajalnstr="aln", centerstr="solute"))):
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
    cpu_rg = reference_gyration(reference_coordinates(host, ref_h, aln_idx, sol_idx, sub), masses[sol_idx])
    cpu_rg_s = time.perf_counter() - t0
    gpu_rg = gyration_features(rg_m[:, 0].cpu().numpy())[sub].astype(np.float64)

    line = dict(
        bench="C12 per-frame group moments (K20)", gpu=card,
        workload=dict(atoms=N, frames=F, solute=n_sol, waters=18000, fit_atoms=len(aln_idx), gyration_atoms=n_sol,
                      spherical_groups=[n_sol, n_sub], seed=a.seed),
        peak_bytes_per_s=PEAK_BYTES_S, reps=a.reps,
        gyration_moments=rg_k, spherical_moments=sph_k, **e2e,
        reference_cpu_float32=dict(
            kind="scaled", frames_timed=len(sub), threads=1, gyration_s_scaled=cpu_rg_s / len(sub) * F,
            speedup_gyration_e2e=cpu_rg_s / len(sub) * F / e2e["metricgyration_project_e2e"]["s"]),
        gyration_vs_reference_max_rel=float(np.max(np.abs(gpu_rg - cpu_rg) / np.abs(cpu_rg))),
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
