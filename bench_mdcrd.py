"""AMBER ASCII trajectory (mdcrd) reading and writing on one GPU (K25).  Prints one JSON line.

Workload: 100 000 atoms x 1 000 frames of seeded random-walk motion with a box that breathes from frame to frame, built
on the device (bench_dcd.random_walk, so the formats' kernels compare directly; every value lies inside the writable
range of F8.3), with a box line per frame: about 2.4 GB of text.

Reported: the card's name and power limit; from the library's CUDA events (median and min-max of --reps calls after 2
warm-up calls) the decode kernel (the encoder's frames restaged at 16-byte-aligned rows, as the reader stages them) and
the encode kernel, with the bytes they move per atom-frame (text and float32, from the shape) and their share of 3.35
TB/s (H100 SXM HBM3, data sheet); write_mdcrd and read_mdcrd_device end to end over 3 runs, each file having just been
written to a temporary directory, so it sits in the page cache; and the host baseline: oracle/mdcrd_format.py's reader
(float() per field) on one core over the first 10 frames, scaled x100 and labelled as scaled.

    python bench_mdcrd.py [--atoms 100000] [--frames 1000] [--reps 10] [--seed 25] [--out DIR] [--no-host]
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
from bench_dcd import HBM_BYTES_PER_S, kernel_ms, random_walk, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=100000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=25)
    ap.add_argument("--out", default=None, help="directory for the file write_mdcrd writes (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mdcrd.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import mdcrd as pm

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, lengths = random_walk(dev, N, F, a.seed)
    lo, hi = (float(v) for v in torch.aminmax(coords))
    assert -999.0 < lo and hi < 9999.0, "the walk left the writable range"
    box = torch.from_numpy(lengths).to(dev)
    S = pm.frame_bytes(N, True)
    af = N * F
    text_per_af = S / N  # about 24.3 bytes of text per atom-frame, box line included

    # encode the whole trajectory into one device buffer, then restage it at 16-byte-aligned rows for the decoder
    enc = torch.empty(F * S, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pm._encode(coords, box, N, F, out=enc), a.reps)
    row = (S + 15) & ~15
    staged = torch.zeros((F, row), dtype=torch.uint8, device=dev)
    staged[:, :S] = enc.view(F, S)
    staged = staged.view(-1)
    del enc
    offsets = np.arange(F, dtype=np.int64) * row
    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    dbox = torch.empty((3, F), dtype=torch.float32, device=dev)
    bad = torch.full((1,), pm.INT64_MAX, dtype=torch.int64, device=dev)
    dec_ms = kernel_ms(lambda: pm.decode_mdcrd_device(staged, offsets, N, True, out=dec, box_out=dbox, bad=bad), a.reps)
    assert int(bad.item()) == pm.INT64_MAX
    # what the text holds: fl32(rint(x * 1000) / 1000) in float64, '%8.3f' then float()
    want = (torch.round(coords.double() * 1000) / 1000).float()
    want_box = (torch.round(box.double() * 1000) / 1000).float().cpu().numpy()
    assert torch.equal(dec.view(torch.int32), want.view(torch.int32))
    assert np.array_equal(dbox.cpu().numpy().view(np.int32), want_box.view(np.int32))
    del staged, dec

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn = os.path.join(a.out, "bench.mdcrd")
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pm.write_mdcrd(fn, coords, box, title="bench_mdcrd")
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, bbox, _ = pm.read_mdcrd_device(fn, N)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), want.view(torch.int32))
        assert np.array_equal(bbox.view(np.int32), want_box.view(np.int32))
        del back
    file_bytes = os.path.getsize(fn)
    host = "not measured"
    if not a.no_host:
        from oracle import mdcrd_format as of

        n_host = min(10, F)
        with open(fn, "rb") as fh:
            head = fh.read(81 + n_host * S)
        t0 = time.perf_counter()
        o = of.read(head, N, True)
        t1 = time.perf_counter()
        x = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
        t2 = time.perf_counter()
        host = dict(what=f"oracle/mdcrd_format.py read (float() per field) of the first {n_host} frames and their "
                         "(F, N, 3) -> (N, 3, F) transposition, one core, scaled x%g to the whole file" % (F / n_host),
                    frames_timed=n_host, read_s=t1 - t0, transpose_s=t2 - t1,
                    scaled_total_s=(t2 - t0) * F / n_host, scaled=True)
        del o, x
    os.remove(fn)
    if tmp is not None:
        tmp.cleanup()

    def share(ms, moved):
        return moved * af / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    moved = text_per_af + 12  # text one way, float32 the other, per atom-frame
    line = dict(
        bench="AMBER ASCII mdcrd read / write (K25)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, box=True, frame_bytes=S, text_bytes=F * S, file_bytes=file_bytes,
                      float32_bytes=12 * af),
        reps=a.reps, bytes_per_atom_frame=dict(text=text_per_af, float32=12, moved=moved),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms, moved),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms, moved),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_mdcrd_s=stats(write_s), read_mdcrd_device_s=stats(read_s),
        read_note="read_mdcrd_device right after write_mdcrd: the file sits in the page cache",
        host_baseline=host,
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
