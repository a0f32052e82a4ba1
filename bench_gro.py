"""Multi-frame GRO reading and writing on one GPU (K29).  Prints one JSON line.

Workloads: seeded random-walk motion built on the device (bench_dcd.random_walk, so the formats' kernels compare
directly) with a box that breathes from frame to frame, formatted by mkb_gro_encode with " t= " / " step= " titles:
50 000 atoms x 1 000 frames with positions only (about 2.25 GB of text), and 30 000 atoms x 1 000 frames with
positions and velocities (about 2.1 GB), the two layouts `gmx trjconv` writes.

Reported per workload: from the library's CUDA events (median and min-max of --reps calls after 2 warm-up calls) the
index passes over the whole text, the decode (line index and parse; the text of every frame as one staged span) and
the encode kernel, with the bytes they move (the text, and 12 bytes of float32 per atom-frame and block for decode and
encode) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet); the title and box pass (mkb_gro_head) from CUDA
events around it; write_gro and read_gro_device end to end over 3 runs, each file having just been written to a
temporary directory, so it sits in the page cache; and the host baseline: oracle/gro_format.py's reader (column slices
and float()) on one core over the first 10 frames, scaled x100 and labelled as scaled.  The card's name and power limit
are read in the same run.

    python bench_gro.py [--reps 10] [--seed 29] [--out DIR] [--no-host] [--small]
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
from bench_dcd import HBM_BYTES_PER_S, random_walk, stats  # noqa: E402
from bench_pdb import kernel_ms  # noqa: E402


def run(dev, N: int, F: int, vel: bool, a) -> dict:
    from moleculekit_b200 import _lib
    from moleculekit_b200 import gro
    from oracle import gro_format as og

    x, lengths = random_walk(dev, N, F, a.seed)
    x = x / 10  # Angstrom -> nm
    lo, hi = (float(v) for v in torch.aminmax(x))
    assert -999.0 < lo and hi < 9999.0, "the walk left the writable range"
    g = torch.Generator(device=dev).manual_seed(a.seed)
    v = (torch.randn((N, 3, F), generator=g, device=dev) * 0.5).clamp_(-99.0, 99.0) if vel else None
    box = torch.zeros((3, 3, F), dtype=torch.float32, device=dev)
    lb = torch.from_numpy(lengths).to(dev) / 10
    for i in range(3):
        box[i, i] = lb[i]
    top = og.random_topology(N, a.seed)
    times, steps = np.arange(F) * 2.0, np.arange(F) * 1000
    xd, vd, bd, _, _, heads, prefix, box9 = gro._prepare(x, top, box, times, steps, "Protein in water", v, None, 1)
    head_d, prefix_d = torch.from_numpy(heads).to(dev), torch.from_numpy(prefix).to(dev)
    S = gro.frame_bytes(N, heads.shape[1], vel, box9)
    nb = 2 if vel else 1
    af = N * F

    buf = torch.zeros(F * S + 16, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: gro._encode(xd, vd, bd, N, F, head_d, prefix_d, box9, out=buf[:F * S]), a.reps)
    n_text = F * S

    cap = F + 16
    state = torch.empty(3, dtype=torch.int64, device=dev)
    frame_off = torch.empty(cap + 1, dtype=torch.int64, device=dev)
    status = torch.empty(cap, dtype=torch.uint8, device=dev)

    def index():
        state.copy_(torch.tensor([0, gro.INT64_MAX, 0]))
        _lib.call(dev, "mkb_gro_index", _lib.ptr(buf), n_text, n_text, 0, N, _lib.ptr(state), _lib.ptr(frame_off),
                  _lib.ptr(status), cap)

    idx_ms = kernel_ms(index, a.reps)
    lines, lone_cr, past = (int(q) for q in state.cpu())
    assert lines == F * (N + 3) and lone_cr == gro.INT64_MAX and past == 0 and not status[:F].any()

    dx = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    dv = torch.empty_like(dx) if vel else None
    flags = torch.zeros(1 + gro.FLAG_CAP, dtype=torch.int64, device=dev)
    frame_of = np.arange(F, dtype=np.int32)
    dec_ms = kernel_ms(lambda: gro.decode_gro_device(buf[:n_text], F, frame_of, N, 8, vel, out=dx, vout=dv,
                                                     flags=flags), a.reps)
    want = (torch.round(xd.double() * 1000) / 1000).float()  # '%8.3f' then float()
    assert torch.equal(dx.view(torch.int32), want.view(torch.int32)) and int(flags[0].item()) == 0
    if vel:
        wv = (torch.round(vd.double() * 10000) / 10000).float()
        assert torch.equal(dv.view(torch.int32), wv.view(torch.int32))
    del dx, dv

    at = np.arange(F + 1, dtype=np.int64) * S
    head_ms = []
    for it in range(a.reps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        hb, ht, hs, hst = gro._head_device(buf, at, dev)
        e1.record()
        torch.cuda.synchronize()
        if it >= 2:
            head_ms.append(e0.elapsed_time(e1))
    assert not hst.any() and torch.equal(hs.cpu(), torch.from_numpy(steps))

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench.gro")
    write_s, read_s = [], []
    fields = ("x", "v") if vel else ("x",)
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gro.write_gro(fn, xd, top, bd, times, steps, "Protein in water", vd)
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, _, info = gro.read_gro_device(fn, fields=fields)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back["x"].view(torch.int32), want.view(torch.int32)) and info["host_lines"] == 0
        del back
    with open(fn, "rb") as fh:
        assert fh.read(4096) == bytes(buf[:4096].cpu().numpy())
    del buf
    host = "not measured"
    if not a.no_host:
        n_host = min(10, F)
        with open(fn, "rb") as fh:
            head = fh.read(n_host * S)
        t0 = time.perf_counter()
        o = og.read(head)
        t1 = time.perf_counter()
        assert o["coords"].shape[0] == n_host
        host = dict(what=f"oracle/gro_format.py read (column slices, float() per field) of the first {n_host} frames, "
                         "one core, scaled x%g to the whole file" % (F / n_host), frames_timed=n_host,
                    read_s=t1 - t0, scaled_total_s=(t1 - t0) * F / n_host, scaled=True)
        del o
    file_bytes = os.path.getsize(fn)
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()
        a.out = None

    def share(ms, moved):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    return dict(
        workload=dict(atoms=N, frames=F, velocities=vel, seed=a.seed, text_bytes=n_text, file_bytes=file_bytes,
                      float32_bytes=12 * af * nb),
        bytes_moved=dict(index=n_text, decode=n_text + 12 * af * nb, encode=n_text + 12 * af * nb),
        index_kernel_ms=stats(idx_ms), index_hbm_share=share(idx_ms, n_text),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms, n_text + 12 * af * nb),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms, n_text + 12 * af * nb),
        head_kernel_ms=stats(head_ms),
        write_gro_s=stats(write_s), read_gro_device_s=stats(read_s),
        read_note="read_gro_device right after the file was written: it sits in the page cache",
        host_baseline=host,
    )


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=29)
    ap.add_argument("--out", default=None, help="directory for the files (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    ap.add_argument("--small", action="store_true", help="1/100 of the atoms, to check the script itself")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gro.py needs a CUDA device: nothing is measured without one")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    k = 100 if a.small else 1
    runs = [run(dev, 50000 // k, 1000, False, a), run(dev, 30000 // k, 1000, True, a)]
    print(json.dumps(dict(bench="multi-frame GRO read / write (K29)", gpu=card, reps=a.reps,
                          hbm_peak_bytes_per_s=HBM_BYTES_PER_S, runs=runs)), flush=True)


if __name__ == "__main__":
    main()
