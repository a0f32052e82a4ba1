"""DSSP secondary structure (K18) on one GPU.  Prints one JSON line.

Workload 1: the traj20 protein (277 residues with N, CA, C and O), its 20 real frames tiled to 2 000: frames are
independent, so the work per frame is that of a real protein.
Workload 2: 16 copies of that protein translated 100 A apart as separate chains (4 432 residues) x 200 frames.

Reported per workload: the time of one mkb_dssp call, the median over windows of back-to-back calls that each last at
least 200 ms (CUDA events around the window); the time of each phase (gather, hydrogen bonds, assignment = flags, ladders
and codes) from torch.profiler in a separate pass; the CA pairs screened (n (n - 1) / 2 per frame, from shapes) and the
energies evaluated (from the C restatement's own counts); MetricSecondaryStructure.project end to end from host arrays;
and the C restatement of the reference on one CPU core, timed on a few frames and scaled.  mdtraj is not available here,
so its own time is not measured.  The GPU's name and power limit are read in the same run.

    python bench_dssp.py [--frames 2000] [--reps 5] [--window-ms 200] [--cpu-frames 4]
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


def run(name, X, bb, flags, a, distinct):
    """time dssp_device on X (host (N, 3, F)); ``distinct`` = how many leading frames are distinct (the rest repeat
    them), over which the oracle counts the energies evaluated"""
    import dssp_oracle
    from moleculekit_b200.dssp import dssp_device

    dev = torch.device("cuda:0")
    t = lambda v, dt: torch.from_numpy(np.ascontiguousarray(v, dtype=dt)).to(dev)  # noqa: E731
    d, b, f = t(X, np.float32), t(bb, np.int32), t(flags, np.uint8)
    n, F = bb.shape[0], X.shape[2]
    out = torch.empty((F, n), dtype=torch.uint8, device=dev)
    call = lambda: dssp_device(d, b, f, out=out)  # noqa: E731
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    call()
    torch.cuda.synchronize()
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
        ph = "gather" if "dssp_gather" in k else "hbond" if "dssp_hbond" in k else \
            "assign_flags" if "dssp_flags" in k else "assign_ladders" if "dssp_ladder" in k else \
            "assign_codes" if "dssp_codes" in k else None
        if ph:
            phases[ph] = phases.get(ph, 0.0) + ev.device_time_total / 1e3 / 3  # ms per call
    # counts: CA pairs from shapes, energies from the oracle's loop on the distinct frames
    cf = list(range(min(a.cpu_frames, distinct)))
    evaluated = 0
    t0 = time.perf_counter()
    for fr in cf:
        codes, _, _, (screened, ev_) = dssp_oracle.frame(X[bb, :, fr], flags)
        evaluated += ev_
    cpu_s = (time.perf_counter() - t0) / len(cf) * F
    want = dssp_oracle.dssp(X, bb, flags, frames=cf)[0]
    same = bool(np.array_equal(out[cf].cpu().numpy(), want))
    pairs = n * (n - 1) // 2 * F
    energies = evaluated / len(cf) * F
    return dict(workload=name, residues=int(n), frames=int(F), call_ms=ms, call_ms_min=float(np.min(ts)),
                call_ms_max=float(np.max(ts)), launches_per_window=launches, phase_ms=phases,
                ca_pairs_screened=int(pairs), energies_evaluated=float(energies),
                ca_pairs_per_s=pairs / (ms * 1e-3), energies_per_s=energies / (ms * 1e-3),
                reference_cpu=dict(kind="C restatement, scaled", frames_timed=len(cf), threads=1, s_scaled=cpu_s,
                                   speedup_vs_call=cpu_s / (ms * 1e-3), mdtraj="not available, not measured"),
                codes_equal_on_timed_frames=same)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--frames2", type=int, default=200)
    ap.add_argument("--copies", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="timed windows per workload")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--cpu-frames", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dssp.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricsecondarystructure import MetricSecondaryStructure, dssp_residues

    torch.cuda.set_device(0)
    card = gpu_info(0)
    with np.load(os.path.join(ROOT, "tests", "golden", "traj20.npz")) as z:
        g = {k: z[k] for k in ("coords", "name", "resname", "resid", "chain", "segid", "sel_masks")}
    prot = g["sel_masks"][5]
    mol20 = MolLite(g["coords"], name=g["name"], resname=g["resname"], resid=g["resid"], chain=g["chain"],
                    segid=g["segid"], named_selections={"protein": prot})
    bb, fl, _, _ = dssp_residues(mol20, prot)
    atoms = np.unique(bb)
    rows = np.searchsorted(atoms, bb)
    X20 = g["coords"][atoms]
    F = a.frames
    X = np.ascontiguousarray(np.tile(X20, (1, 1, F // 20 + 1))[:, :, :F])
    w1 = run("traj20 protein tiled", X, rows, fl, a, 20)

    mol = MolLite(np.ascontiguousarray(np.tile(g["coords"], (1, 1, F // 20 + 1))[:, :, :F]), name=g["name"],
                  resname=g["resname"], resid=g["resid"], chain=g["chain"], segid=g["segid"],
                  named_selections={"protein": prot})
    m = MetricSecondaryStructure(sel="protein")
    m.project(mol)
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.project(mol)
        times.append(time.perf_counter() - t0)
    w1["metric_project_e2e_s"] = dict(s=float(np.median(times)), s_min=float(np.min(times)), s_max=float(np.max(times)))

    c, F2 = a.copies, a.frames2
    X2 = np.ascontiguousarray(np.concatenate([X20 + np.float32(100 * k) for k in range(c)])[:, :, :20])
    X2 = np.ascontiguousarray(np.tile(X2, (1, 1, F2 // 20 + 1))[:, :, :F2])
    BB = np.concatenate([rows + k * atoms.size for k in range(c)])
    FL = np.tile(fl, c)
    FL[::bb.shape[0]] |= 2
    w2 = run(f"{c} chains", X2, BB, FL, a, 20)

    print(json.dumps(dict(bench="DSSP (K18)", gpu=card, workloads=[w1, w2])), flush=True)


if __name__ == "__main__":
    main()
