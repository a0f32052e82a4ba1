"""C12 dihedrals (K16) on one GPU.  Prints one JSON line.

Workload: bench_align.py's C12 trajectory -- 59 000 atoms (a 5 000-atom solute under a per-frame random rigid motion
and 0.5 A noise, plus 18 000 waters) over 2 000 frames, generated on the device from a seed.  The solute is given a
protein topology: the 20 standard residues in turn, heavy atoms only, until 5 000 atoms are used.  MetricDihedral
takes every phi, psi and chi1-chi5 of it.  The coordinates are random, so the angles are meaningless but the memory
traffic and the arithmetic are those of a real protein.  A second run repeats the referenced atoms' 2 000 frames 50
times: 100 000 frames.

Reported: per-launch kernel time for sin / cos and for angles, the median over 10 windows of back-to-back launches
that each last at least 200 ms (CUDA events around the window), with the library's per-launch kernel event beside it;
algorithmic bytes (12 B read per referenced atom-frame, 8 B or 4 B written per dihedral-frame) and their share of the
H100 SXM data sheet's 3.35 TB/s;
MetricDihedral.project end to end from host arrays (gather of the referenced atoms, upload, kernel, result back); and
a float32 numpy restatement of the reference's per-dihedral loop on one CPU core, timed on a subset of frames and
scaled to the whole trajectory.  The GPU's name and power limit are read in the same run.

    python bench_dihedral.py [--frames 2000] [--reps 10] [--window-ms 200] [--cpu-frames 200] [--seed 12]
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

HEAVY = {
    "ALA": "CB", "ARG": "CB CG CD NE CZ NH1 NH2", "ASN": "CB CG OD1 ND2", "ASP": "CB CG OD1 OD2", "CYS": "CB SG",
    "GLN": "CB CG CD OE1 NE2", "GLU": "CB CG CD OE1 OE2", "GLY": "", "HIS": "CB CG ND1 CD2 CE1 NE2",
    "ILE": "CB CG1 CG2 CD1", "LEU": "CB CG CD1 CD2", "LYS": "CB CG CD CE NZ", "MET": "CB CG SD CE",
    "PHE": "CB CG CD1 CD2 CE1 CE2 CZ", "PRO": "CB CG CD", "SER": "CB OG", "THR": "CB OG1 CG2",
    "TRP": "CB CG CD1 CD2 NE1 CE2 CE3 CZ2 CZ3 CH2", "TYR": "CB CG CD1 CD2 CE1 CE2 CZ OH", "VAL": "CB CG1 CG2",
}
ALL = ("phi", "psi", "chi1", "chi2", "chi3", "chi4", "chi5")


def topology(N, n_sol):
    """(name, resname, resid, protein mask) of N atoms: the first residues fill up to n_sol atoms, the rest is water"""
    name, resname, resid = [], [], []
    types = sorted(HEAVY)
    r = 0
    while True:
        rn = types[r % len(types)]
        atoms = ["N", "CA", "C", "O"] + HEAVY[rn].split()
        if len(name) + len(atoms) > n_sol:
            break
        name += atoms
        resname += [rn] * len(atoms)
        resid += [r + 1] * len(atoms)
        r += 1
    n_prot = len(name)
    name += ["X"] * (N - n_prot)
    resname += ["WAT"] * (N - n_prot)
    resid += list(range(r + 1, r + 1 + N - n_prot))
    return np.array(name), np.array(resname), np.array(resid), np.arange(N) < n_prot


def reference_project(X, quads, frames):
    """float32 numpy, one dihedral at a time over the listed frames (the reference's loop over dihedralAngle), then
    sin and cos interleaved"""
    out = np.empty((len(frames), 2 * len(quads)), np.float32)
    for j, q in enumerate(quads):
        P = X[q][:, :, frames]
        b0, b1, b2 = P[1] - P[0], P[2] - P[1], P[3] - P[2]
        n1, n2 = np.cross(b0, b1, axis=0), np.cross(b1, b2, axis=0)
        a = np.arctan2(np.sqrt((b1 * b1).sum(0)) * (b0 * n2).sum(0), (n1 * n2).sum(0))
        out[:, 2 * j] = np.sin(a)
        out[:, 2 * j + 1] = np.cos(a)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=10, help="timed windows per kernel")
    ap.add_argument("--window-ms", type=float, default=200.0, help="least length of one timed window")
    ap.add_argument("--cpu-frames", type=int, default=200)
    ap.add_argument("--seed", type=int, default=12)
    ap.add_argument("--repeat", type=int, default=50, help="frame repeats of the long run")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dihedral.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200.dihedral import dihedrals_device
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricdihedral import MetricDihedral

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    F, n_sol = a.frames, 5000
    X, _, _, box = c12(dev, a.seed, F)
    N = X.shape[0]
    name, resname, resid, prot = topology(N, n_sol)
    host = X.cpu().numpy()
    mol = MolLite(host, box=box.cpu().numpy(), name=name, resname=resname, resid=resid,
                  named_selections={"protein": prot})
    m = MetricDihedral(dih=ALL, sincos=True)
    quads, labels = m._getMolProp(mol, "dihedrals")
    atoms, rows = np.unique(quads, return_inverse=True)
    nq, na = len(quads), len(atoms)
    compact = X[torch.from_numpy(atoms).to(dev)].contiguous()
    d_quads = torch.from_numpy(rows.reshape(nq, 4).astype(np.int32)).to(dev)

    def timed(traj, sincos, out):
        """a.reps windows of back-to-back launches, each window at least a.window_ms long (CUDA events around the
        window, time per launch = window / launches); the library's own per-launch kernel event is reported beside"""
        ev = []
        _lib.set_timing(True, 0)
        for _ in range(5):
            dihedrals_device(traj, d_quads, sincos, out=out)
            ev.append(_lib.get_timing(0)[1])
        _lib.set_timing(False, 0)
        launches = max(1, int(np.ceil(a.window_ms / min(ev[2:]))))
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(a.reps):
            start.record()
            for _ in range(launches):
                dihedrals_device(traj, d_quads, sincos, out=out)
            end.record()
            end.synchronize()
            ts.append(start.elapsed_time(end) / launches)
        n = traj.shape[2]
        nbytes = 12 * na * n + (8 if sincos else 4) * nq * n
        ms = float(np.median(ts))
        return dict(ms=ms, ms_min=float(np.min(ts)), ms_max=float(np.max(ts)), launches_per_window=launches,
                    kernel_event_ms=float(np.median(ev[2:])), algorithmic_bytes=nbytes,
                    gbs=nbytes / (ms * 1e-3) / 1e9, frac_of_peak=nbytes / (ms * 1e-3) / PEAK_BYTES_S)

    sc_out = torch.empty((F, 2 * nq), device=dev)
    kern = dict(sincos=timed(compact, True, sc_out), angle=timed(compact, False, torch.empty((F, nq), device=dev)))
    long_traj = compact.repeat(1, 1, a.repeat).contiguous()
    FL = long_traj.shape[2]
    kern_long = dict(sincos=timed(long_traj, True, torch.empty((FL, 2 * nq), device=dev)))
    del long_traj
    torch.cuda.empty_cache()
    kern_long["angle"] = timed(compact.repeat(1, 1, a.repeat).contiguous(), False,
                               torch.empty((FL, nq), device=dev))

    # end to end from host arrays
    res = m.project(mol)
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = m.project(mol)
        times.append(time.perf_counter() - t0)
    e2e = dict(s=float(np.median(times)), s_min=float(np.min(times)), s_max=float(np.max(times)),
               frames_per_s=F / float(np.median(times)), host_bytes_up=int(na * 3 * F * 4), host_bytes_down=res.nbytes)

    # the reference's float32 numpy path on one core, on a subset of frames, scaled
    sub = np.linspace(0, F - 1, min(a.cpu_frames, F)).astype(int)
    t0 = time.perf_counter()
    cpu = reference_project(host, quads, sub)
    cpu_s = time.perf_counter() - t0

    kinds = [d for d, _ in labels]
    line = dict(
        bench="C12 dihedrals (K16)", gpu=card,
        workload=dict(atoms=N, frames=F, solute=n_sol, residues=int(len(np.unique(resid[prot]))), dihedrals=nq,
                      per_type={d: kinds.count(d) for d in ALL}, referenced_atoms=na, long_frames=FL, seed=a.seed),
        peak_bytes_per_s=PEAK_BYTES_S, reps=a.reps, kernel=kern, kernel_100k=kern_long,
        metricdihedral_project_e2e=e2e,
        reference_cpu_float32=dict(kind="scaled", frames_timed=len(sub), threads=1, s_scaled=cpu_s / len(sub) * F,
                                   speedup_e2e=cpu_s / len(sub) * F / e2e["s"]),
        sincos_vs_reference_max_abs=float(np.max(np.abs(res[sub] - cpu))),
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
