"""TM-score search (K19) on one GPU.  Prints one JSON line.

Workload 1: the 277 CA atoms of traj20, its 20 real frames tiled to 2 000, against frame 0: frames are independent, so
the work per frame is that of a real protein.
Workload 2: 16 copies of that protein translated 100 A apart as one selection of 4 432 pairs, x 20 frames, against
frame 0: the search is O(L^2) per frame (every seed passes over all L pairs), so this is the large-L case.

Reported per workload: the mkb_tmscore call time, the median over windows of back-to-back calls that each last at least
200 ms (CUDA events around the window); seeds, fits and pair evaluations per frame from the C restatement's counters (a
pair evaluation is one pair of one score pass, L per fit); pair evaluations per second; the share of the FP64 bound, from
FP64_OPS_PER_PAIR_EVAL operations per pair evaluation against the H100 SXM data sheet's 34 TFLOP/s non-tensor FP64 (a
lower bound on the work: the fit passes add 30 operations per fitted pair, which the counters do not see);
MetricTMscore.project end to end from host arrays (workload 1); and the C restatement on one CPU core, timed on a few
frames and scaled, with its TM-scores checked equal to the GPU's bits.  The GPU's name and power limit are read in the
same run.

    python bench_tmscore.py [--frames 2000] [--reps 5] [--window-ms 200] [--cpu-frames 20] [--cpu-frames2 2]
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

# one score-pass pair: x - p (3), R (x - p) (9 mul, 6 add), + q (3), - y (3), squared distance (3 mul, 2 add), sqrt,
# / d0, t t, 1 +, 1 /, the score sum and the squared-distance sum (sqrt and divisions counted as one operation each)
FP64_OPS_PER_PAIR_EVAL = 37
FP64_PEAK = 34e12  # H100 SXM data sheet, non-tensor FP64


def run(name, X, Y, a, distinct, cpu_frames):
    """time tmscore_device on model rows X (host (L, 3, F)) against reference rows Y (L, 3); the first ``distinct``
    frames are distinct (the rest repeat them); the oracle counts and is timed on the last ``cpu_frames`` of them"""
    import tmscore_oracle
    from moleculekit_b200.tmscore import tmscore_device

    dev = torch.device("cuda:0")
    L, F = X.shape[0], X.shape[2]
    d = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
    r = torch.from_numpy(np.ascontiguousarray(Y[:, :, None], dtype=np.float32)).to(dev)
    sel = torch.arange(L, dtype=torch.int32, device=dev)
    call = lambda: tmscore_device(d, sel, r, sel)  # noqa: E731
    for _ in range(2):
        tm, _ = call()
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
    gpu_tm = tm.cpu().numpy()
    cf = list(range(distinct))[-cpu_frames:]
    counts = np.zeros(3)
    cpu_tm = np.zeros(len(cf))
    t0 = time.perf_counter()
    for k, fr in enumerate(cf):
        cpu_tm[k], _, c = tmscore_oracle.frame(X[:, :, fr], Y)
        counts += c
    cpu_s = (time.perf_counter() - t0) / len(cf) * F
    seeds, fits, evals = counts / len(cf)
    pair_evals = evals * F
    return dict(workload=name, pairs=int(L), frames=int(F), call_ms=ms, call_ms_min=float(np.min(ts)),
                call_ms_max=float(np.max(ts)), launches_per_window=launches,
                per_frame=dict(seeds=seeds, fits=fits, pair_evaluations=evals, counted_on_frames=len(cf)),
                pair_evaluations_per_s=pair_evals / (ms * 1e-3),
                fp64_share=dict(value=pair_evals * FP64_OPS_PER_PAIR_EVAL / FP64_PEAK / (ms * 1e-3),
                                ops_per_pair_evaluation=FP64_OPS_PER_PAIR_EVAL,
                                bound="H100 SXM data sheet, 34 TFLOP/s non-tensor FP64"),
                reference_cpu=dict(kind="C restatement, scaled", frames_timed=len(cf), threads=1, s_scaled=cpu_s,
                                   speedup_vs_call=cpu_s / (ms * 1e-3)),
                tm_equal_on_timed_frames=bool(np.array_equal(gpu_tm[cf].view(np.int64), cpu_tm.view(np.int64))))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--frames2", type=int, default=20)
    ap.add_argument("--copies", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="timed windows per workload")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--cpu-frames", type=int, default=20, help="oracle frames of workload 1")
    ap.add_argument("--cpu-frames2", type=int, default=2, help="oracle frames of workload 2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tmscore.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metrictmscore import MetricTMscore

    torch.cuda.set_device(0)
    card = gpu_info(0)
    with np.load(os.path.join(ROOT, "tests", "golden", "traj20.npz")) as z:
        g = {k: z[k] for k in ("coords", "name")}
    ca = np.where(g["name"] == "CA")[0]
    X20 = g["coords"][ca]
    F = a.frames
    X = np.ascontiguousarray(np.tile(X20, (1, 1, F // 20 + 1))[:, :, :F])
    w1 = run("traj20 CA tiled", X, X20[:, :, 0], a, 20, a.cpu_frames)

    mol = MolLite(np.ascontiguousarray(np.tile(g["coords"], (1, 1, F // 20 + 1))[:, :, :F]), name=g["name"])
    m = MetricTMscore(MolLite(g["coords"][:, :, 0], name=g["name"]), "all", pbc=False)
    m.project(mol)
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.project(mol)
        times.append(time.perf_counter() - t0)
    w1["metric_project_e2e_s"] = dict(s=float(np.median(times)), s_min=float(np.min(times)), s_max=float(np.max(times)))

    c = a.copies
    X2 = np.ascontiguousarray(np.concatenate([X20 + np.float32(100 * k) for k in range(c)]))
    X2 = np.ascontiguousarray(np.tile(X2, (1, 1, a.frames2 // 20 + 1))[:, :, :a.frames2])
    w2 = run(f"{c} copies as one selection", X2, X2[:, :, 0], a, 20, a.cpu_frames2)

    print(json.dumps(dict(bench="TM-score (K19)", gpu=card, workloads=[w1, w2])), flush=True)


if __name__ == "__main__":
    main()
