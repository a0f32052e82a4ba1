"""Multi-model PDBx/mmCIF reading and writing on one GPU (K30).  Prints one JSON line.

Workload: 30 000 atoms x 1 000 models of seeded random-walk motion (bench_dcd.random_walk, so the formats' kernels
compare directly with bench_pdb.py and bench_gro.py), formatted by mkb_cif_encode in RCSB's row layout (21 columns of
_atom_site, id and pdbx_PDB_model_num unique across the file) with bench_pdb.py's topology under one _cell: about
3.8 GB of text.

Reported: the card's name and power limit; from the library's CUDA events (median and min-max of --reps calls after 2
warm-up calls) the index passes over the whole loop body, the decode (row ranking, tokenizing and parse; the text of
every model as one staged span) and the encode kernel, with the bytes they move (the text, and 12 bytes of float32 per
atom-model for decode and encode) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet); write_cif and
read_cif_device end to end over 3 runs, each file having just been written to a temporary directory, so it sits in the
page cache; and the host baseline: oracle/cif_format.py's reader (split(), the quote rule and float()) on one core over
the first 10 models, scaled x100 and labelled as scaled.

    python bench_cif.py [--atoms 30000] [--frames 1000] [--reps 10] [--seed 30] [--out DIR] [--no-host]
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
    ap.add_argument("--out", default=None, help="directory for the files (default: a temporary one)")
    ap.add_argument("--no-host", action="store_true", help="skip the single-core host baseline")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cif.py needs a CUDA device: nothing is measured without one")
    from moleculekit_b200 import _lib
    from moleculekit_b200 import cif as pc
    from oracle import cif_format as of
    from oracle import pdb_format

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    N, F = a.atoms, a.frames
    coords, lengths = random_walk(dev, N, F, a.seed)
    box = np.repeat(lengths[:, :1], F, axis=1)  # an mmCIF data block holds one cell
    top = pdb_format.random_topology(N, a.seed)  # bench_pdb.py's topology: primed names are quoted, none holds a blank
    layout = pc._layout(pc._fields(top, N), N, F)
    tmpl = torch.from_numpy(layout[0]).to(dev)
    R = layout[1]
    S = pc.frame_bytes(N, R)
    af = N * F
    n_text = F * S

    buf = torch.zeros(n_text + 16, dtype=torch.uint8, device=dev)
    enc_ms = kernel_ms(lambda: pc._encode(coords, N, F, tmpl, layout, out=buf[:n_text]), a.reps)
    head = pc._header("bench", box[:, 0], np.full(3, 90.0, np.float32))
    tags = [t.lower() for t in pc.TAGS]

    cap = 4 * F + 16
    state = torch.empty(7, dtype=torch.int64, device=dev)
    marks = torch.empty(3 * cap, dtype=torch.int64, device=dev)

    def index():
        state.copy_(torch.tensor([0, pc.INT64_MAX, 0, pc.INT64_MAX, pc.INT64_MAX, pc.INT64_MIN, -1]))
        _lib.call(dev, "mkb_cif_index", _lib.ptr(buf), n_text, n_text, len(head), 1, len(tags),
                  tags.index("pdbx_pdb_model_num"), _lib.ptr(state), _lib.ptr(marks), cap)

    idx_ms = kernel_ms(index, a.reps)
    st = [int(v) for v in state.cpu()]
    assert st[0] == af and st[1] == pc.INT64_MAX and st[2] == F and st[3] == pc.INT64_MAX, st

    dec = torch.empty((N, 3, F), dtype=torch.float32, device=dev)
    flags = torch.zeros(1 + pc.FLAG_CAP, dtype=torch.int64, device=dev)
    frame_of = np.arange(F, dtype=np.int32)
    dec_ms = kernel_ms(lambda: pc.decode_cif_device(buf[:n_text], F, frame_of, N, pc._cartn(tags), out=dec,
                                                    flags=flags), a.reps)
    want = (torch.round(coords.double() * 1000) / 1000).float()  # '%10.3f' then float()
    assert torch.equal(dec.view(torch.int32), want.view(torch.int32)) and int(flags[0].item()) == 0
    del dec

    tmp = None
    if a.out is None:
        tmp = tempfile.TemporaryDirectory()
        a.out = tmp.name
    os.makedirs(a.out, exist_ok=True)
    fn_w = os.path.join(a.out, "bench_write.cif")
    del buf
    write_s, read_s = [], []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pc.write_cif(fn_w, coords, top, box, title="bench")
        write_s.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        back, info = pc.read_cif_device(fn_w)
        torch.cuda.synchronize()
        read_s.append(time.perf_counter() - t0)
        assert torch.equal(back.view(torch.int32), want.view(torch.int32)) and info["host_lines"] == 0
        del back
    host = "not measured"
    if not a.no_host:
        n_host = min(10, F)
        with open(fn_w, "rb") as fh:
            part = fh.read(len(head) + n_host * S)
        t0 = time.perf_counter()
        o = of.read(part)
        t1 = time.perf_counter()
        x = np.ascontiguousarray(o["coords"].transpose(1, 2, 0))
        t2 = time.perf_counter()
        assert o["coords"].shape[0] == n_host
        host = dict(what=f"oracle/cif_format.py read (split(), quote rule, float() per token) of the first {n_host} "
                         "models and their (F, N, 3) -> (N, 3, F) transposition, one core, scaled x%g to the whole file"
                         % (F / n_host), frames_timed=n_host, read_s=t1 - t0, transpose_s=t2 - t1,
                    scaled_total_s=(t2 - t0) * F / n_host, scaled=True)
        del o, x
    file_bytes = os.path.getsize(fn_w)
    os.remove(fn_w)
    if tmp is not None:
        tmp.cleanup()

    def share(ms, moved):
        return moved / (float(np.median(ms)) * 1e-3) / HBM_BYTES_PER_S

    line = dict(
        bench="multi-model PDBx/mmCIF read / write (K30)", gpu=card,
        workload=dict(atoms=N, frames=F, seed=a.seed, row_bytes=R, text_bytes=n_text, file_bytes=file_bytes,
                      float32_bytes=12 * af),
        reps=a.reps, bytes_moved=dict(index=n_text, decode=n_text + 12 * af, encode=n_text + 12 * af),
        index_kernel_ms=stats(idx_ms), index_hbm_share=share(idx_ms, n_text),
        decode_kernel_ms=stats(dec_ms), decode_hbm_share=share(dec_ms, n_text + 12 * af),
        encode_kernel_ms=stats(enc_ms), encode_hbm_share=share(enc_ms, n_text + 12 * af),
        hbm_peak_bytes_per_s=HBM_BYTES_PER_S,
        write_cif_s=stats(write_s), read_cif_device_s=stats(read_s),
        read_note="read_cif_device right after the file was written: it sits in the page cache",
        host_baseline=host,
    )
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
