"""TM-align (K27) on one GPU.  Prints one JSON line.

Workload 1: the 277 CA atoms of traj20 x 2 000 frames onto the 223 protein CA atoms of 3PTB: the 20 real frames, each
repeated with its own seeded Gaussian noise of 0.1 to 1 A per frame, so every frame differs.
Workload 2: traj20's 20 frames onto its own frame 0.
Workload 3: traj20's frame 1 alone onto its frame 0 (the one-structure call).
Workload 4: one item at the residue cap on both sides, a seeded random walk of 3.8 A steps onto a noisy copy of itself
(the longest single item a call accepts).

Reported per workload: the mkb_tmalign call time, the median over windows of back-to-back calls that each last at least
200 ms (CUDA events around the window, the call warmed up first); frames per second; DP cells, fits and pair
evaluations per frame from the C restatement's counters; and the C restatement on one core of the same host, in the same
run, timed on a few frames and scaled to the workload, with its results checked equal to the GPU's bits on those frames.
The GPU's name and power limit are read in the same run.

    python bench_tmalign.py [--frames 2000] [--reps 5] [--window-ms 200] [--cpu-frames 4]
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


def run(name, X, Y, a, reps=None):
    """time tmalign_device of x rows X (host (xlen, 3, F)) onto y rows Y (ylen, 3); the oracle counts and is timed on
    the first a.cpu_frames frames"""
    import tmalign_oracle
    from moleculekit_b200.tmalign import tmalign_device

    dev = torch.device("cuda:0")
    F = X.shape[2]
    d = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
    r = torch.from_numpy(np.ascontiguousarray(Y[:, :, None], dtype=np.float32)).to(dev)
    sel = torch.arange(X.shape[0], dtype=torch.int32, device=dev)
    rsel = torch.arange(Y.shape[0], dtype=torch.int32, device=dev)
    call = lambda: tmalign_device(d, sel, r, rsel)  # noqa: E731
    out = call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = call()
    torch.cuda.synchronize()
    one = time.perf_counter() - t0
    launches = max(1, int(np.ceil(a.window_ms / 1e3 / one)))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps or a.reps):
        start.record()
        for _ in range(launches):
            call()
        end.record()
        end.synchronize()
        ts.append(start.elapsed_time(end) / launches)
    ms = float(np.median(ts))
    got = [o.cpu().numpy() for o in out]
    cf = list(range(min(a.cpu_frames, F)))
    t0 = time.perf_counter()
    want = tmalign_oracle.tmalign(X, Y, cf)
    cpu_s = (time.perf_counter() - t0) / len(cf) * F
    counts = np.mean([tmalign_oracle.frame(X[:, :, f], Y)["counts"] for f in cf], axis=0)
    equal = all(np.array_equal(np.ascontiguousarray(g[cf]).view(np.uint8), np.ascontiguousarray(w).view(np.uint8))
                for g, w in zip(got, want))
    return dict(workload=name, xlen=int(X.shape[0]), ylen=int(Y.shape[0]), frames=int(F), call_ms=ms,
                call_ms_min=float(np.min(ts)), call_ms_max=float(np.max(ts)), launches_per_window=launches,
                frames_per_s=F / (ms * 1e-3),
                per_frame=dict(dp_cells=float(counts[0]), fits=float(counts[1]), pair_evaluations=float(counts[2]),
                               counted_on_frames=len(cf)),
                mean_tm_ref=float(np.nanmean(got[0][:, 0])),
                reference_cpu=dict(kind="C restatement, scaled", frames_timed=len(cf), threads=1, s_scaled=cpu_s,
                                   speedup_vs_call=cpu_s / (ms * 1e-3)),
                bits_equal_on_timed_frames=bool(equal))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5, help="timed windows per workload")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--cpu-frames", type=int, default=4, help="oracle frames per workload")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tmalign.py needs a CUDA device: nothing is measured without one")
    torch.cuda.set_device(0)
    card = gpu_info(0)
    with np.load(os.path.join(ROOT, "tests", "golden", "traj20.npz")) as z:
        X20 = z["coords"][z["name"] == "CA"]
    with np.load(os.path.join(ROOT, "tests", "golden", "pdb_3ptb.npz")) as z:
        P = z["coords"][(z["name"] == "CA") & z["sel_protein"], :, 0]
    F = a.frames
    rng = np.random.default_rng(2027)
    sigma = rng.uniform(0.1, 1.0, size=F)
    X = X20[:, :, np.arange(F) % 20] + (rng.normal(size=(X20.shape[0], 3, F)) * sigma).astype(np.float32)
    w1 = run("traj20 CA x noisy frames onto 3PTB CA", np.ascontiguousarray(X, np.float32), P, a)
    w2 = run("traj20 CA onto its frame 0", np.ascontiguousarray(X20), X20[:, :, 0], a)
    w3 = run("traj20 CA frame 1 onto its frame 0", np.ascontiguousarray(X20[:, :, 1:2]), X20[:, :, 0], a)
    from moleculekit_b200.tmalign import max_residues

    cap = max_residues()
    steps = rng.normal(size=(cap, 3))
    Yc = np.cumsum(3.8 * steps / np.linalg.norm(steps, axis=1, keepdims=True), axis=0).astype(np.float32)
    Xc = (Yc + rng.normal(0, 0.5, size=Yc.shape)).astype(np.float32)[:, :, None]
    w4 = run("one item at the cap", Xc, Yc, a, reps=3)
    print(json.dumps(dict(bench="TM-align (K27)", gpu=card, workloads=[w1, w2, w3, w4])), flush=True)


if __name__ == "__main__":
    main()
