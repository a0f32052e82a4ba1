"""Multi-model PDB reading and writing on one GPU (K28).  Prints one JSON line.

Workload: 30 000 atoms x 1 000 frames of seeded random-walk motion with a box that breathes from frame to frame, built
on the device (bench_dcd.random_walk, so the formats' kernels compare directly), formatted by mkb_pdb_encode with a
CRYST1 record per model, and a TER record inserted after each chain of 1 000 atoms: about 2.4 GB of text.

Reported: the card's name and power limit; from the library's CUDA events (median and min-max of --reps calls after 2
warm-up calls) the index passes over the whole text, the decode (atom-record ranking and parse; the text of every frame
as one staged span) and the encode kernel, with the bytes they move (the text, and 12 bytes of float32 per atom-frame
for decode and encode) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet); write_pdb and read_pdb_device end to
end over 3 runs, each file having just been written to a temporary directory, so it sits in the page cache; and the
host baseline: oracle/pdb_format.py's reader (column slices and float()) on one core over the first 10 frames, scaled
x100 and labelled as scaled.

    python bench_pdb.py [--atoms 30000] [--frames 1000] [--chain 1000] [--reps 10] [--seed 28] [--out DIR] [--no-host]
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

TER = b"TER                                                                             \n"  # 80 columns


def kernel_ms(fn, reps: int):
    """library CUDA-event time of every pass of ``reps`` calls after 2 warm-up calls"""
    from moleculekit_b200 import _lib

    _lib.set_timing(True, 0)
    ms = []
    for it in range(reps + 2):
        fn()
        torch.cuda.synchronize()
        if it >= 2:
            ms.append(sum(_lib.get_timing(0)))
    _lib.set_timing(False, 0)
    return ms


def with_ter(enc: torch.Tensor, F: int, S: int, N: int, chain: int) -> torch.Tensor:
    """the encoder's F frames of S bytes with a TER line after every ``chain`` atoms of each frame"""
    rows = enc.view(F, S)
    H = S - 81 * N - 7
    ter = torch.frombuffer(bytearray(TER), dtype=torch.uint8).to(enc.device).expand(F, len(TER))
    parts = [rows[:, :H]]
    for a0 in range(0, N, chain):
        parts += [rows[:, H + 81 * a0:H + 81 * min(N, a0 + chain)], ter]
    parts.append(rows[:, S - 7:])
    body = torch.cat(parts, dim=1).reshape(-1)
    return torch.cat([body, torch.frombuffer(bytearray(b"END\n"), dtype=torch.uint8).to(enc.device)])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=30000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--chain", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=28)
    ap.add_argument("--out", default=None, help="directory for the files (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pdb.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200 import pdb as pp
    from oracle import pdb_format as of

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, lengths = random_walk(dev, N, F, a.seed)
    lo, hi = (float(v) for v in torch.aminmax(coords))
    assert -999.0 < lo and hi < 9999.0, "the walk left the writable range"
    box = torch.from_numpy(lengths).to(dev)
    angles = torch.full_like(box, 90.0)
    top = of.random_topology(N, a.seed)
    tmpl = torch.from_numpy(pp._template(pp._fields(top, N), N)).to(dev)
    S = pp.frame_bytes(N, True)
    af = N * F

    enc = torch.empty(F * S, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pp._encode(coords, box, angles, N, F, tmpl, out=enc), a.reps)
    text = with_ter(enc, F, S, N, a.chain)
    del enc
    n_text = int(text.numel())
    buf = torch.zeros(n_text + 16, dtype=torch.uint8, device=dev)
    buf[:n_text] = text
    del text

    cap = 8 * F + 16
    state = torch.empty(3, dtype=torch.int64, device=dev)
    marks = torch.empty(2 * cap, dtype=torch.int64, device=dev)

    def index():
        state.copy_(torch.tensor([0, pp.INT64_MAX, 0]))
        _lib.call(dev, "mkb_pdb_index", _lib.ptr(buf), n_text, n_text, 0, _lib.ptr(state), _lib.ptr(marks), cap)

    idx_ms = kernel_ms(index, a.reps)
    total, lone_cr, n_marks = (int(v) for v in state.cpu())
    assert total == af and lone_cr == pp.INT64_MAX and n_marks == 3 * F + 1, (total, lone_cr, n_marks)

    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    flags = torch.zeros(1 + pp.FLAG_CAP, dtype=torch.int64, device=dev)
    frame_of = np.arange(F, dtype=np.int32)
    dec_ms = kernel_ms(lambda: pp.decode_pdb_device(buf[:n_text], F, frame_of, N, out=dec, flags=flags), a.reps)
    want = (torch.round(coords.double() * 1000) / 1000).float()  # '%8.3f' then float()
    assert torch.equal(dec.view(torch.int32), want.view(torch.int32)) and int(flags[0].item()) == 0
    del dec

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn_ter = os.path.join(a.out, "bench_ter.pdb")
    with open(fn_ter, "wb") as fh:
        fh.write(memoryview(buf[:n_text].cpu().numpy()))
    del buf
    fn_w = os.path.join(a.out, "bench_write.pdb")
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pp.write_pdb(fn_w, coords, top, box, angles)
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, info = pp.read_pdb_device(fn_ter)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), want.view(torch.int32)) and info["host_lines"] == 0
        del back
    host = "not measured"
    if not a.no_host:
        n_host = min(10, F)
        with open(fn_ter, "rb") as fh:
            head = fh.read(n_host * (S + (-(-N // a.chain)) * len(TER)))
        t0 = time.perf_counter()
        o = of.read(head)
        t1 = time.perf_counter()
        x = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
        t2 = time.perf_counter()
        assert o["coords"].shape[0] == n_host
        host = dict(what=f"oracle/pdb_format.py read (column slices, float() per field) of the first {n_host} frames "
                         "and their (F, N, 3) -> (N, 3, F) transposition, one core, scaled x%g to the whole file"
                         % (F / n_host), frames_timed=n_host, read_s=t1 - t0, transpose_s=t2 - t1,
                    scaled_total_s=(t2 - t0) * F / n_host, scaled=True)
        del o, x
    file_bytes = os.path.getsize(fn_ter)
    written_bytes = os.path.getsize(fn_w)
    os.remove(fn_ter)
    os.remove(fn_w)
    if tmp is not None:
        tmp.cleanup()

    def share(ms, moved):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="multi-model PDB read / write (K28)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, chain=a.chain, cryst1_per_model=True, text_bytes=n_text,
                      file_bytes=file_bytes, written_file_bytes=written_bytes, float32_bytes=12 * af),
        reps=a.reps, bytes_moved=dict(index=n_text, decode=n_text + 12 * af, encode=F * S + 12 * af),
        index_kernel_ms=stats(idx_ms), index_hbm_share=share(idx_ms, n_text),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms, n_text + 12 * af),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms, F * S + 12 * af),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_pdb_s=stats(write_s), read_pdb_device_s=stats(read_s),
        read_note="read_pdb_device right after the file was written: it sits in the page cache",
        host_baseline=host,
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
