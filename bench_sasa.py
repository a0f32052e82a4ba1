"""Shrake-Rupley SASA (K17) on one GPU.  Prints one JSON line.

Workload 1: the traj20 system (4 507 atoms with hydrogens: a 4 480-atom protein, a ligand and Cl- ions), sel = protein,
filtersel = all, 960 sphere points, probe 1.4 A.  Its 20 real frames are tiled to 2 000: frames are independent, so
the work per frame is that of a real protein.
Workload 2: a large solute -- workloads._sphere_lattice at 60 000 atoms (a jittered 2.2 A lattice, protein-like
density) with the traj20 element mix, 4 frames of independent jitter, every atom queried.

Reported per workload: the time of one mkb_sasa call, the median over windows of back-to-back calls that each last at
least 200 ms (CUDA events around the window); the time of each phase (gather, cell-list scan and scatter, surface)
from torch.profiler in a separate pass; point-neighbour tests per second against the upper bound counted on the host
from the exact neighbour lists (points x neighbours, no early exit); MetricSasa.project end to end from host arrays
(workload 1); and the C restatement of mdtraj's loop on one CPU core, timed on a few frames and scaled (mdtraj itself
may use more threads).  The kernel is bound by FP32 issue, not HBM: a test is 8 float32 operations (3 subtractions, 3
multiplications, 2 additions) and a compare, so the roofline is the data sheet's FP32 rate, 67 TFLOP/s counting an FMA
as two operations, i.e. 33.5e12 non-fused operations/s, 4.2e12 tests/s.  The GPU's name and power limit are read in the
same run.

    python bench_sasa.py [--frames 2000] [--reps 5] [--window-ms 200] [--cpu-frames 2]
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
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_align import gpu_info  # noqa: E402

OPS_PER_TEST = 8
FP32_OPS_S = 33.5e12  # H100 SXM data sheet: 67 TFLOP/s FP32 with an FMA counted as two operations
PEAK_TESTS_S = FP32_OPS_S / OPS_PER_TEST


def neighbour_counts(X_nm, radii, query):
    """exact float32 neighbour count of every query atom of one frame (the kernel's and the reference's test)"""
    from scipy.spatial import cKDTree

    tree = cKDTree(X_nm.astype(np.float64))
    rmax = float(radii.max())
    out = np.zeros(len(query), np.int64)
    for n, i in enumerate(query):
        cand = np.array(tree.query_ball_point(X_nm[i].astype(np.float64), float(radii[i]) + rmax + 1e-4), np.int64)
        cand = cand[cand != i]
        d = X_nm[i] - X_nm[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        rc = radii[i] + radii[cand]
        out[n] = int(np.count_nonzero(d2 < rc * rc))
    return out


def run(name, X, radii, query, sphere, a, distinct):
    """time sasa_device on X (host (N, 3, F)); ``distinct`` = how many leading frames are distinct (the rest repeat
    them), over which the neighbour lists are counted"""
    import sasa_oracle
    from moleculekit_b200.sasa import sasa_device

    dev = torch.device("cuda:0")
    t = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v, dtype=dt)).to(dev)  # noqa: E731
    d, env, r, q, s = t(X, np.float32), t(np.arange(X.shape[0]), np.int32), t(radii, np.float32), t(query, np.int32), \
        t(sphere, np.float32)
    out = torch.empty((X.shape[2], len(query)), device=dev)
    call = lambda: sasa_device(d, env, r, q, s, out=out)  # noqa: E731
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    call()
    one = time.perf_counter() - t0
    launches = max(1, int(np.ceil(a.window_ms / 1e3 / one)))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(a.reps):
        start.record()
        for _ in range(launches):
            call()
        end.record()
        end.synchronize()
        ts.append(start.elapsed_time(end) / launches)
    ms = float(np.median(ts))
    # phases from the profiler, in a pass of their own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            call()
        torch.cuda.synchronize()
    phases = {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA" or ev.count == 0:
            continue
        k = ev.key
        ph = "gather" if "sasa_gather" in k else "surface" if "sasa_surface" in k else \
            "cell_list" if ("sasa_scatter" in k or "Scan" in k or "scan" in k or "emset" in k) else \
            "other" if "sasa" in k else None
        if ph:
            phases[ph] = phases.get(ph, 0.0) + ev.device_time_total / 1e3 / 3  # ms per call
    # upper bound of the point-neighbour tests from the exact neighbour lists of the distinct frames
    F = X.shape[2]
    nb = sum(int(neighbour_counts(X[:, :, f] / np.float32(10), radii, query).sum()) for f in range(distinct))
    tests = nb * (F / distinct) * len(sphere)
    # the C restatement of the reference loop, one core, a few frames, scaled
    cf = list(range(min(a.cpu_frames, distinct)))
    t0 = time.perf_counter()
    want = sasa_oracle.sasa(X, radii, query, sphere, frames=cf)
    cpu_s = (time.perf_counter() - t0) / len(cf) * F
    same = bool(np.array_equal(out[cf].cpu().numpy().view(np.int32), want.view(np.int32)))
    return dict(workload=name, atoms=int(X.shape[0]), query_atoms=int(len(query)), frames=int(F),
                sphere_points=int(len(sphere)), call_ms=ms, call_ms_min=float(np.min(ts)), call_ms_max=float(np.max(ts)),
                launches_per_window=launches, phase_ms=phases, mean_neighbours=nb / distinct / len(query),
                upper_bound_tests=float(tests), upper_bound_tests_per_s=tests / (ms * 1e-3),
                share_of_fp32_bound_at_upper_bound=tests / (ms * 1e-3) / PEAK_TESTS_S,
                reference_cpu=dict(kind="scaled", frames_timed=len(cf), threads=1, s_scaled=cpu_s,
                                   speedup_vs_call=cpu_s / (ms * 1e-3)),
                bit_identical_on_timed_frames=same)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5, help="timed windows per workload")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--cpu-frames", type=int, default=2)
    ap.add_argument("--seed", type=int, default=17)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sasa.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import workloads
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricsasa import MetricSasa
    from moleculekit_b200.sasa import sasa_radii, sphere_points

    torch.cuda.set_device(0)
    card = gpu_info(0)
    with np.load(os.path.join(ROOT, "tests", "golden", "traj20.npz")) as z:
        g = {k: z[k] for k in ("coords", "element", "name", "resname", "resid", "chain", "segid", "sel_masks")}
    X20 = g["coords"]
    F = a.frames
    X = np.ascontiguousarray(np.tile(X20, (1, 1, F // X20.shape[2] + 1))[:, :, :F])
    prot = g["sel_masks"][5]
    radii = sasa_radii(g["element"], 1.4)
    S = sphere_points(960)
    w1 = run("traj20 system tiled", X, radii, np.where(prot)[0], S, a, X20.shape[2])

    mol = MolLite(X, element=g["element"], name=g["name"], resname=g["resname"], resid=g["resid"], chain=g["chain"],
                  segid=g["segid"], named_selections={"protein": prot})
    m = MetricSasa(sel="protein")
    m.project(mol)
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.project(mol)
        times.append(time.perf_counter() - t0)
    w1["metricsasa_project_e2e_s"] = dict(s=float(np.median(times)), s_min=float(np.min(times)),
                                          s_max=float(np.max(times)))

    rng = np.random.default_rng(a.seed)
    n2 = 60000
    base = workloads._sphere_lattice(rng, n2, 55.0, np.zeros(3))
    X2 = np.ascontiguousarray(np.stack([base + rng.normal(0, 0.3, base.shape).astype(np.float32) for _ in range(4)], 2))
    el = rng.choice(g["element"][prot], n2)
    w2 = run("sphere lattice 60k", X2, sasa_radii(el, 1.4), np.arange(n2), S, a, 4)

    print(json.dumps(dict(bench="SASA (K17)", gpu=card, peak_tests_per_s=PEAK_TESTS_S, ops_per_test=OPS_PER_TEST,
                          workloads=[w1, w2])), flush=True)


if __name__ == "__main__":
    main()
