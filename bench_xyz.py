"""Multi-frame XYZ reading and writing on one GPU (K26).  Prints one JSON line.

Workload: 50 000 atoms x 1 000 frames of seeded random-walk motion built on the device (bench_dcd.random_walk, so the
formats' kernels compare directly), elements C / H / N / O, written as '%-1s %15.8f %15.8f %15.8f': about 2.5 GB of
text.

Reported: the card's name and power limit; from the library's CUDA events (median and min-max of --reps calls after 2
warm-up calls) the index pass over the whole file staged on the device (one call), the decode kernel with the line
pass it runs first (the file's frames staged as read_xyz_device stages them; the parse kernel alone is reported too)
and the encode kernel, each with the text bytes it reads or writes and their share of 3.35 TB/s (H100 SXM HBM3, data
sheet); write_xyz and read_xyz_device end to end over 3 runs, each file having just been written to a temporary
directory, so it sits in the page cache (read_xyz_device runs the index pass first, which reads the file once more);
and the host baseline: oracle/xyz_format.py's reader (split() and float() per line) on one core over the first 10
frames, scaled to the whole file and labelled as scaled.

    python bench_xyz.py [--atoms 50000] [--frames 1000] [--reps 10] [--seed 26] [--out DIR] [--no-host]
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


def kernel_ms(fn, reps: int, which: int):
    """library CUDA event times of ``reps`` calls after 2 warm-up calls: which 1 = main kernel, 0 + 1 = the whole call"""
    from moleculekit_b200 import _lib

    _lib.set_timing(True, 0)
    ms = []
    for it in range(reps + 2):
        fn()
        torch.cuda.synchronize()
        if it >= 2:
            prep, main = _lib.get_timing(0)
            ms.append(main if which == 1 else prep + main)
    _lib.set_timing(False, 0)
    return ms


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=50000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=26)
    ap.add_argument("--out", default=None, help="directory for the file write_xyz writes (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_xyz.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200 import xyz as pxyz

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, _ = random_walk(dev, N, F, a.seed)
    element = [("C", "H", "N", "O")[i % 4] for i in range(N)]
    comment = "bench_xyz"
    head = f"{N}\n{comment}\n".encode()
    S = pxyz.frame_bytes(N, head, 1)
    text = F * S
    af = N * F
    head_d, column_d = pxyz._device_text(head, np.frombuffer("".join(element).encode(), np.uint8), dev)

    # encode the whole trajectory into one device buffer: it is also the staged file for the index and decode passes
    enc = torch.empty(text + 64, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pxyz._encode(coords, N, F, head_d, column_d, 1, out=enc), a.reps, 1)
    state = torch.zeros(3, dtype=torch.int64, device=dev)
    cap = F + 2
    frame_off = torch.zeros(cap + 1, dtype=torch.int64, device=dev)
    status = torch.zeros(cap, dtype=torch.uint8, device=dev)

    def index():
        state.copy_(torch.tensor([0, pxyz.INT64_MAX, 0]))
        _lib.call(dev, "mkb_xyz_index", _lib.ptr(enc), text - 1, text - 1, 0, N, _lib.ptr(state), _lib.ptr(frame_off),
                  _lib.ptr(status), cap)

    idx_ms = kernel_ms(index, a.reps, 1)
    assert int(state[0]) + 1 == F * (N + 2) and int(status[1:F].sum()) == 0
    assert np.array_equal(frame_off[1:F].cpu().numpy(), np.arange(1, F) * S)
    out = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    flags = torch.zeros(1 + 2 * 1024, dtype=torch.int64, device=dev)
    frame_of = np.arange(F, dtype=np.int32)
    dec = lambda: pxyz.decode_xyz_device(enc[:text], F, frame_of, N, out=out, flags=flags, flag_cap=1024)  # noqa: E731
    dec_ms = kernel_ms(dec, a.reps, 0)
    parse_ms = kernel_ms(dec, a.reps, 1)
    assert int(flags[0]) == 0
    want = (torch.round(coords.double() * 1e8) / 1e8).float()
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))
    del enc, out

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench.xyz")
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pxyz.write_xyz(fn, coords, element, comment=comment)
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, info = pxyz.read_xyz_device(fn)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), want.view(torch.int32)) and info["host_lines"] == 0
        del back
    file_bytes = os.path.getsize(fn)
    host = "not measured"
    if not a.no_host:
        from oracle import xyz_format as of

        n_host = min(10, F)
        with open(fn, "rb") as fh:
            part = fh.read(n_host * S)
        t0 = time.perf_counter()
        o = of.read(part)
        t1 = time.perf_counter()
        x = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
        t2 = time.perf_counter()
        host = dict(what=f"oracle/xyz_format.py read (split() and float() per line) of the first {n_host} frames and "
                         "their (F, N, 3) -> (N, 3, F) transposition, one core, scaled x%g to the whole file"
                         % (F / n_host),
                    frames_timed=n_host, read_s=t1 - t0, transpose_s=t2 - t1,
                    scaled_total_s=(t2 - t0) * F / n_host, scaled=True)
        del o, x
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()

    def share(ms, moved):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="multi-frame XYZ read / write (K26)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, frame_bytes=S, text_bytes=text, file_bytes=file_bytes,
                      float32_bytes=12 * af),
        reps=a.reps,
        index_kernel_ms=stats(idx_ms), index_text_gb_s=text / (float(np.median(idx_ms)) * 1e6),
        index_hbm_share=share(idx_ms, 2 * text),
        index_note="count, scan and emit passes: the text is read twice",
        decode_ms=stats(dec_ms), decode_text_gb_s=text / (float(np.median(dec_ms)) * 1e6),
        decode_hbm_share=share(dec_ms, 3 * text + 12 * af),
        decode_note="the line pass (text read twice, 8-byte line starts) and the parse kernel; shares count 3 text "
                    "reads (two line passes, one parse) and the float32 written, not the line starts",
        parse_kernel_ms=stats(parse_ms), parse_hbm_share=share(parse_ms, text + 12 * af),
        encode_kernel_ms=stats(enc_ms), encode_text_gb_s=text / (float(np.median(enc_ms)) * 1e6),
        encode_hbm_share=share(enc_ms, text + 12 * af),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_xyz_s=stats(write_s), read_xyz_device_s=stats(read_s),
        read_note="read_xyz_device right after write_xyz (the file sits in the page cache); it runs the index pass "
                  "first, which reads the file once more",
        host_baseline=host,
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
