"""Multi-model BinaryCIF reading and writing on one GPU (K31).  Prints one JSON line.

Workload: bench_cif.py's, 30 000 atoms x 1 000 models of seeded random-walk motion (bench_dcd.random_walk) with
bench_pdb.py's topology under one _cell, written by write_bcif, so the file compares directly with mmCIF's 3.81 GB.

Reported: the card's name and power limit; the file size; from the library's CUDA events (median and min-max of --reps
calls after 2 warm-up calls) each device step of one Cartn_x column -- decode (mkb_bcif_decode: every step of the chain
and the frame-minor store), quantize, sizes and emit -- with the bytes the step must read and write (decode: the
payload and 4 bytes of float32 per value; quantize: 4 + 4 per value; sizes: 4 per value; emit: 4 per value and the
payload) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet); a torch.profiler breakdown of one decode and one
encode of that column by kernel; read_bcif_device and write_bcif end to end over 3 runs; and the host baseline:
oracle/bcif_format.py's sequential reader on one core over the first 10 models, scaled x100 and labelled as scaled.

    python bench_bcif.py [--atoms 30000] [--frames 1000] [--reps 10] [--seed 30] [--no-host]
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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--atoms", type=int, default=30000)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=30)
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bcif.py needs a CUDA device: nothing is measured without one")
    import ctypes as C

    from moleculekit_b200 import _lib
    from moleculekit_b200 import bcif as pb
    from oracle import bcif_format as of
    from oracle import pdb_format

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    n = N * F
    coords, lengths = random_walk(dev, N, F, a.seed)
    box = np.repeat(lengths[:, :1], F, axis=1)
    top = pdb_format.random_topology(N, a.seed)
    out = dict(workload=f"{N} atoms x {F} models", card=card)
    with tempfile.TemporaryDirectory() as tmp:
        fn = os.path.join(tmp, "bench.bcif")
        wall = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pb.write_bcif(fn, coords, top, box)
            wall.append(time.perf_counter() - t0)
        out["write_bcif_s"] = stats(wall)
        size = os.path.getsize(fn)
        out["file_bytes"] = size
        out["mmcif_bytes_same_workload"] = 3.81e9
        idx = pb.index_bcif(fn)
        wall = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got, _ = pb.read_bcif_device(fn)
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
        out["read_bcif_device_s"] = stats(wall)
        want = np.float32(np.rint(coords.cpu().numpy().astype(np.float64) * 1000) / 1000)
        out["round_trip_exact"] = bool(np.array_equal(got.cpu().numpy(), want))

        # one Cartn_x column, step by step
        col = idx["columns"]["cartn_x"]["data"]
        payload, steps, m, _ = pb._chain(fn, "Cartn_x", col["data"], col["encoding"])
        P = len(payload)
        buf = torch.zeros((P + 15) & ~15, dtype=torch.uint8)
        buf[:P] = torch.frombuffer(bytearray(payload), dtype=torch.uint8)
        buf = buf.to(dev)
        status = torch.zeros(2, dtype=torch.int64, device=dev)
        sel = np.arange(F, dtype=np.int64)
        dst = torch.empty((N, 3, F), dtype=torch.float32, device=dev)[:, 0, :]
        q = torch.empty(n, dtype=torch.int32, device=dev)
        xs = coords[:, 0, :]
        sizes = (C.c_int64 * 25)()

        def decode():
            _lib.call(dev, "mkb_bcif_decode", _lib.ptr(buf), P, steps.ctypes.data_as(C.c_void_p), len(steps), 1,
                      _lib.ptr(dst), F, sel.ctypes.data_as(C.c_void_p), N, dst.stride(0), _lib.ptr(status))

        def quantize():
            _lib.call(dev, "mkb_bcif_quantize", _lib.ptr(xs), xs.stride(0), xs.stride(1), N, F, 1000.0, _lib.ptr(q))

        def size_pass():
            _lib.call(dev, "mkb_bcif_sizes", _lib.ptr(q), n, 0, n, sizes)

        quantize()
        data, enc = pb._encode_ints(q, n)
        chain = {("IntegerPacking",): 0, ("RunLength",): 1, ("Delta",): 2, ("Delta", "RunLength"): 3}
        kinds = tuple(e["kind"] for e in enc if e["kind"] in ("Delta", "RunLength")) or ("IntegerPacking",)
        w = next((e["byteCount"] for e in enc if e["kind"] == "IntegerPacking"), 4)
        uns = int(next((e["isUnsigned"] for e in enc if e["kind"] == "IntegerPacking"), False))
        n_packed = next((e["srcSize"] for e in enc if e["kind"] == "IntegerPacking"), len(data) // 4)
        emit_out = torch.empty(max(4, (len(data) + 3) & ~3), dtype=torch.uint8, device=dev)

        def emit():
            _lib.call(dev, "mkb_bcif_emit", _lib.ptr(q), n, 0, n, chain[kinds], w, uns, n_packed,
                      _lib.ptr(emit_out), len(data))

        out["cartn_x_encoding"] = [e["kind"] + (f"({e['byteCount']}{'u' if e['isUnsigned'] else 's'})"
                                                if e["kind"] == "IntegerPacking" else "") for e in enc]
        out["cartn_x_payload_bytes"] = P
        steps_out = {}
        for name, fn_, nbytes in (("decode", decode, P + 4 * n), ("quantize", quantize, 8 * n),
                                  ("sizes", size_pass, 4 * n), ("emit", emit, 4 * n + P)):
            ms = kernel_ms(fn_, a.reps)
            med = float(np.median(ms))
            steps_out[name] = dict(ms=stats(ms), bytes=nbytes, hbm_share=nbytes / (med * 1e-3) / HBM_BYTES_PER_S)
        out["cartn_x_steps"] = steps_out
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            decode()
            quantize()
            size_pass()
            emit()
            torch.cuda.synchronize()
        ker = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t:
                ker[ev.key[:80]] = round(t / 1e3, 4)
        out["profiler_kernel_ms"] = ker
        if not a.no_host:
            hf = os.path.join(tmp, "host.bcif")
            pb.write_bcif(hf, coords[:, :, :10], top, box[:, :10])
            raw = open(hf, "rb").read()
            t0 = time.perf_counter()
            of.read(raw)
            out["oracle_reader_1core_s_scaled_x100"] = (time.perf_counter() - t0) * F / 10
    print(json.dumps(out))


if __name__ == "__main__":
    main()
