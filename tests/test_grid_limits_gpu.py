"""GPU tests of the metric and codec kernels past the 65 535 blocks of one launch's grid y.

Grid y of a launch holds at most 65 535 blocks, so every kernel below either walks its grid rows in a loop
(``for (b = blockIdx.y; b < n; b += gridDim.y)``) or splits the work into chunks of at most 65 535 frames.  Ordinary
inputs reach the second trip: a selection with repeated atoms, a long trajectory of a small system read in one chunk,
SASA or DSSP of a ligand or a short peptide over a long trajectory.  A wrong stride, tile offset or chunk offset there
leaves outputs unwritten or misplaced while every smaller input stays right.

1. K15 coordinates, frame sums and fluctuations (tiles of 64 selection entries) on 65 535 * 64 + 197 entries.
2. K16 dihedrals (tiles of 64 quadruples) on 65 535 * 64 + 197 quadruples, in both output modes.
3. The NetCDF / TRR / DCD codecs (tiles of 32 frames) on 65 535 * 32 + 37 frames: decode, encode, and the public
   readers on files their writers wrote.
4. SASA and DSSP over 2 * 65 535 + 11 frames of a 20-atom molecule and an 8-residue peptide: three chunks, the
   last one partial.

Every output starts out filled with a sentinel that no kernel writes and is checked whole, bit for bit, against numpy,
the oracles, or the same kernel on an input that fits one grid trip.  A failure names the first bad index and the state
at the tile or chunk edges.
"""
import numpy as np
import pytest

import dssp_oracle as dso
import sasa_oracle as so
from oracle import dihedral_oracle as dho
from test_dihedral_gpu import _check_angles, _check_sincos
from test_trr_gpu import _f32, _special32, _special64

pytestmark = pytest.mark.gpu

GRID_Y = 65535
TILE = 64                      # K15 selection entries, K16 quadruples per tile
K_BIG = GRID_Y * TILE + 197    # 4 194 437: the last tile of the second trip is partial
EDGES_K = (GRID_Y * TILE - 1, GRID_Y * TILE, K_BIG - 1)
FT = 32                        # codec frames per tile
F_CODEC = GRID_Y * FT + 37     # 2 097 157
EDGES_CODEC = (GRID_Y * FT - 1, GRID_Y * FT, F_CODEC - 1)
F_CHUNK = 2 * GRID_Y + 11      # 131 081 frames: SASA / DSSP chunks of 65 535, 65 535 and 11
EDGES_CHUNK = (GRID_Y - 1, GRID_Y, GRID_Y + 1, 2 * GRID_Y - 1, 2 * GRID_Y, F_CHUNK - 1)
N_BASE = 97                    # distinct frames of the SASA / DSSP trajectories; 97 does not divide 65 535
SENT32 = 0x7FA5A5A5            # a signalling NaN no kernel here writes: a value left unwritten keeps it
SLICE = 1 << 19                # selection entries compared on the host at a time


def _edges(bad, edges, what):
    """failure text: how many differ, the first one, and the state at the named edges"""
    bad = np.asarray(bad)
    idx = np.flatnonzero(bad)
    state = ", ".join(f"{e} {'BAD' if bad[e] else 'ok'}" for e in edges)
    first = idx[0] if idx.size else None
    return f"{idx.size} of {bad.size} {what}s differ, first {what} {first}; at the edges: {state}"


def _check(bad, edges, what):
    assert not bad.any(), _edges(bad, edges, what)


def _sentinel(shape, dev):
    import torch

    return torch.full(shape, SENT32, dtype=torch.int32, device=dev).view(torch.float32)


def _prime(nbytes, dev):
    """Fill a block of ``nbytes`` with a sentinel and free it, with no other free block cached: the caching allocator
    hands it to the next request of that size, so an output the library allocates itself does not start out holding
    an earlier call's bits."""
    import torch

    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    t = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize(dev)
    del t


def _i32(t):
    import torch

    return t.view(torch.int32)


def _bad_last(got, want):
    """per index of the last dimension: does any element differ?  Bit patterns, compared on the device."""
    d = got != want
    return d.reshape(-1, d.shape[-1]).any(0).cpu().numpy()


def _bad_frames(got, want):
    """(natoms, 3, F) uint32 host arrays -> per frame: does any word differ?"""
    assert got.shape == want.shape
    return (got != want).any(axis=(0, 1))


# ---------------------------------------------------------------------------------------------------- 1. K15 tiles
N15, F15 = 1000, 34     # one full 32-frame tile and a partial one


@pytest.fixture(scope="module")
def k15():
    import torch

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(15)
    X = (rng.normal(0, 20, size=(N15, 3, 1)) + rng.normal(0, 2, size=(N15, 3, F15))).astype(np.float32)
    assert (X < 0).any() and (X > 0).any()
    sel = rng.integers(0, N15, K_BIG).astype(np.int32)
    return dict(dev=dev, rng=rng, X=X, d=torch.from_numpy(X).to(dev), sel=sel, d_sel=torch.from_numpy(sel).to(dev))


def _records(p):
    """fit records of every frame onto a rotated copy of frame 7, through the library's align path on 50 atoms"""
    import torch
    from scipy.spatial.transform import Rotation

    from moleculekit_b200.align import superpose_device

    X, dev = p["X"], p["dev"]
    ref = (X[:, :, 7].astype(np.float64) @ Rotation.random(random_state=3).as_matrix() + [4.5, -12.0, 30.25])
    aln = torch.from_numpy(np.arange(0, N15, 20, dtype=np.int32)).to(dev)
    rec, st = superpose_device(p["d"], aln, torch.from_numpy(ref.astype(np.float32)[:, :, None]).to(dev), aln)
    assert int(st.sum()) == 0
    return rec


def test_coordinates_more_than_65535_tiles(k15):
    """no records against the numpy gather; fit records, an explicit frame list with repeats and a column slice of a
    wider matrix against the call on the distinct atoms (each value depends only on atom, frame and record)"""
    import torch
    from moleculekit_b200.coords import coordinates_device

    p = k15
    dev, X, sel, d, d_sel = p["dev"], p["X"], p["sel"], p["d"], p["d_sel"]
    K = K_BIG
    assert K > GRID_Y * TILE and K % TILE != 0
    out = _sentinel((F15, 3 * K), dev)
    coordinates_device(d, d_sel, out=out)
    bad = np.zeros(K, bool)
    for i0 in range(0, K, SLICE):
        i1 = min(K, i0 + SLICE)
        got = torch.stack([out[:, a * K + i0:a * K + i1] for a in range(3)], 1).cpu().numpy()
        want = np.ascontiguousarray(X[sel[i0:i1]].transpose(2, 1, 0))
        bad[i0:i1] = (got.view(np.uint32) != want.view(np.uint32)).any(axis=(0, 1))
    _check(bad, EDGES_K, "selection entry")
    del out

    rec = _records(p)
    uniq, inv = np.unique(sel, return_inverse=True)
    small = coordinates_device(d, torch.from_numpy(uniq.astype(np.int32)).to(dev), rec)  # 16 tiles: one grid trip
    U, d_inv = uniq.size, torch.from_numpy(inv.reshape(-1)).to(dev)
    out = _sentinel((F15, 3 * K), dev)
    coordinates_device(d, d_sel, rec, out=out)
    want = small.view(F15, 3, U)[:, :, d_inv]
    _check(_bad_last(_i32(out).view(F15, 3, K), _i32(want)), EDGES_K, "selection entry")
    del out, want

    fl = np.array([33, 0, 0, 17, 33, 5] + list(range(31, 0, -1)), np.int32)  # 37 listed frames: two frame tiles
    n, lead = fl.size, 21
    wide = _sentinel((n, 3 * K + 40), dev)
    d_fl = torch.from_numpy(fl).to(dev)
    coordinates_device(d, d_sel, rec[d_fl.long()], d_fl, out=wide[:, lead:lead + 3 * K])
    assert wide.stride(0) > 3 * K
    want = small[d_fl.long()].view(n, 3, U)[:, :, d_inv]
    _check(_bad_last(_i32(wide[:, lead:lead + 3 * K]).unflatten(1, (3, K)), _i32(want)), EDGES_K, "selection entry")
    assert bool((_i32(wide[:, :lead]) == SENT32).all()) and bool((_i32(wide[:, lead + 3 * K:]) == SENT32).all()), \
        "a margin of the wider matrix was written"


def test_frame_sums_more_than_65535_tiles(k15):
    """130 frames (64-frame chunks 64, 64 and 2): float64 sums of each chunk in list order, the chunks added in order"""
    import torch
    from moleculekit_b200.coords import coord_sums_device

    p = k15
    dev, sel, d_sel = p["dev"], p["sel"], p["d_sel"]
    F = 130
    assert F // 64 == 2 and F % 64 != 0
    X = (p["rng"].normal(0, 20, size=(N15, 3, 1)) + p["rng"].normal(0, 2, size=(N15, 3, F))).astype(np.float32)
    total = np.zeros((N15, 3))
    for c0 in range(0, F, 64):
        s = np.zeros((N15, 3))
        for f in range(c0, min(F, c0 + 64)):
            s = s + X[:, :, f].astype(np.float64)
        total = total + s
    _prime(K_BIG * 3 * 8, dev)
    got = coord_sums_device(torch.from_numpy(X).to(dev), d_sel)
    want = torch.from_numpy(total[sel]).to(dev)
    _check(_bad_last(got.view(torch.int64).T, want.view(torch.int64).T), EDGES_K, "selection entry")


def test_fluctuation_more_than_65535_tiles(k15):
    """per atom, and averaged over more than 65 535 * 64 groups of 1 to 3 positions: the kernel's formula
    ((e0 e0 + e1 e1) + e2 e2) in float64 (as tests/test_coords_gpu.py::_same_formula), group sums in selection order,
    one rounding to float32"""
    import torch
    from moleculekit_b200.coords import fluctuation_device

    p = k15
    dev, X, sel, d, d_sel, rng = p["dev"], p["X"], p["sel"], p["d"], p["d_sel"], p["rng"]

    def sqdev(rows, centre):  # (c,) atom rows, (c, 3) float64 centres -> (c, F) float64
        e = X[rows].astype(np.float64) - centre[:, :, None]
        return (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]

    K = K_BIG
    centre = rng.normal(0, 20, size=(K, 3))
    out = _sentinel((F15, K), dev)
    fluctuation_device(d, d_sel, torch.from_numpy(centre).to(dev), out=out)
    bad = np.zeros(K, bool)
    for i0 in range(0, K, SLICE):
        i1 = min(K, i0 + SLICE)
        want = sqdev(sel[i0:i1], centre[i0:i1]).astype(np.float32).T
        bad[i0:i1] = (out[:, i0:i1].cpu().numpy().view(np.uint32) != want.view(np.uint32)).any(axis=0)
    _check(bad, EDGES_K, "selection entry")
    del out

    G = K_BIG
    assert G > GRID_Y * TILE
    size = rng.integers(1, 4, G)
    off = np.concatenate([[0], np.cumsum(size)]).astype(np.int64)
    k2 = int(off[-1])
    sel2 = rng.integers(0, N15, k2).astype(np.int32)
    centre2 = rng.normal(0, 20, size=(k2, 3))
    out = _sentinel((F15, G), dev)
    fluctuation_device(d, torch.from_numpy(sel2).to(dev), torch.from_numpy(centre2).to(dev),
                       groups=torch.from_numpy(off).to(dev), out=out)
    bad = np.zeros(G, bool)
    for g0 in range(0, G, SLICE // 2):
        g1 = min(G, g0 + SLICE // 2)
        a0, a1 = int(off[g0]), int(off[g1])
        v = sqdev(sel2[a0:a1], centre2[a0:a1])
        first, sz = off[g0:g1] - a0, size[g0:g1]
        s = v[first]
        for j in (1, 2):
            m = sz > j
            s[m] = s[m] + v[first[m] + j]
        want = (s / sz[:, None]).astype(np.float32).T
        bad[g0:g1] = (out[:, g0:g1].cpu().numpy().view(np.uint32) != want.view(np.uint32)).any(axis=0)
    _check(bad, EDGES_K, "group")


# ------------------------------------------------------------------------------------------------------ 2. K16 tiles
@pytest.mark.parametrize("sincos", [False, True])
def test_dihedrals_more_than_65535_tiles(sincos):
    """4 194 437 quadruples drawn from 3 000 distinct ones: bit-equal to the call on the distinct quadruples, gathered;
    a sample including the last 64 against the float64 oracle"""
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(16)
    N, F, D, K = 300, 34, 3000, K_BIG
    assert K > GRID_Y * TILE
    X = (rng.normal(0, 8, size=(N, 3, 1)) + rng.normal(0, 1.5, size=(N, 3, F))).astype(np.float32)
    distinct = np.unique(np.argsort(rng.random((D, N)), axis=1)[:, :4], axis=0).astype(np.int32)
    D = distinct.shape[0]
    pick = rng.integers(0, D, K)
    quads = np.ascontiguousarray(distinct[pick])
    d, q = torch.from_numpy(X).to(dev), torch.from_numpy(quads).to(dev)
    assert q.data_ptr() % 16 == 0
    nv = 2 if sincos else 1
    out = _sentinel((F, nv * K), dev)
    dihedrals_device(d, q, sincos, out=out)
    small = dihedrals_device(d, torch.from_numpy(distinct).to(dev), sincos)   # 47 tiles: one grid trip
    want = small.view(F, D, nv)[:, torch.from_numpy(pick).to(dev), :]
    _check(_bad_last(_i32(out).view(F, K, nv).transpose(1, 2), _i32(want).transpose(1, 2)), EDGES_K, "quadruple")
    del want
    sample = np.concatenate([np.sort(rng.choice(K - 64, 200, replace=False)), np.arange(K - 64, K)])
    got = out.view(F, K, nv)[:, torch.from_numpy(sample).to(dev), :].reshape(F, nv * sample.size).cpu().numpy()
    (_check_sincos if sincos else _check_angles)(got, dho.project(X, quads[sample].astype(np.int64), sincos))


# ----------------------------------------------------------------------------------------------------- 3. codec tiles
def _values32(rng, F, natoms):
    """(F, natoms, 3) float32 of varied bit patterns: -0.0, NaN payloads, signalling NaNs and subnormals included"""
    return _special32(rng.normal(0, 30, size=(F, natoms, 3)).astype(np.float32))


def _frame_minor(V):
    """(F, natoms, 3) -> (natoms, 3, F) uint32 words"""
    return np.ascontiguousarray(V.transpose(1, 2, 0)).view(np.uint32)


def _into_slice(dev, natoms, F, lead=6, tail=7):
    """(the sentinel-filled (natoms, 3, F + lead + tail) tensor, its frame slice [lead, lead + F))"""
    big = _sentinel((natoms, 3, F + lead + tail), dev)
    return big, big[:, :, lead:lead + F]


DECODE_CASES = [("netcdf", 3), ("trr4", 3), ("trr4", 35), ("trr8", 3), ("dcd", 3), ("dcd_swapped", 3)]


@pytest.mark.parametrize("fmt,natoms", DECODE_CASES, ids=[f"{f}-{n}" for f, n in DECODE_CASES])
def test_decode_more_than_65535_frame_tiles(fmt, natoms):
    """records built with numpy, decoded into a frame slice of a sentinel-filled tensor: every frame is the numpy
    transpose (float64 rounded as numpy's astype(np.float32) rounds it), the margins keep the sentinel"""
    import torch
    from moleculekit_b200 import dcd
    from moleculekit_b200.netcdf import decode_netcdf_device
    from moleculekit_b200.trr import decode_trr_device

    dev = torch.device("cuda", 0)
    F = F_CODEC
    assert -(-F // FT) > GRID_Y
    rng = np.random.default_rng(23 + natoms)
    nv = 3 * natoms
    if fmt == "trr8":
        V64 = _special64(rng.normal(0, 30, size=(F, natoms, 3)))
        want = _frame_minor(_f32(V64))
        rec = np.zeros(F, [("pad", "u1", (8,)), ("x", ">u8", (nv,))])
        rec["x"] = V64.reshape(F, nv).view(np.uint64)
    else:
        V = _values32(rng, F, natoms)
        want = _frame_minor(V)
        if fmt.startswith("dcd"):
            rec = np.zeros(F, [("r", "<u4" if fmt == "dcd" else ">u4", (3, natoms + 2))])
            rec["r"][:, :, 0] = rec["r"][:, :, -1] = 4 * natoms
            rec["r"][:, :, 1:-1] = V.transpose(0, 2, 1).view(np.uint32)
        else:
            rec = np.zeros(F, [("pad", "u1", (4 if fmt == "netcdf" else 8,)), ("x", ">u4", (nv,))])
            rec["x"] = V.reshape(F, nv).view(np.uint32)
    rb = rec.dtype.itemsize
    buf = torch.from_numpy(rec.view(np.uint8)).to(dev)
    big, out = _into_slice(dev, natoms, F)
    if fmt == "netcdf":
        decode_netcdf_device(buf, np.arange(F, dtype=np.int64) * rb + 4, natoms, out=out)
    elif fmt.startswith("trr"):
        decode_trr_device(buf, np.arange(F, dtype=np.int64) * rb + 8, natoms, 8 if fmt == "trr8" else 4, out=out)
    else:
        desc = np.zeros(F, dcd.FRAME_DESC)
        desc["offset"] = np.arange(F, dtype=np.int64)[:, None] * rb + np.arange(3) * (8 + 4 * natoms) + 4
        desc["count"] = natoms
        dcd.decode_dcd_device(buf, desc, natoms, swap=fmt == "dcd_swapped", out=out)
    got = big.cpu().numpy().view(np.uint32)
    _check(_bad_frames(got[:, :, 6:6 + F], want), EDGES_CODEC, "frame")
    assert (got[:, :, :6] == SENT32).all() and (got[:, :, 6 + F:] == SENT32).all(), "a margin frame was written"


ENCODE_CASES = ["netcdf", "trr_x", "trr_xv", "trr_xvf", "dcd"]


@pytest.mark.parametrize("fmt", ENCODE_CASES)
def test_encode_more_than_65535_frame_tiles(fmt):
    """frame-slice inputs encoded into records; the expected records are assembled with numpy, vectorised over frames:
    the head / extra words and the byte-swapped (NetCDF, TRR) or native (DCD) slabs"""
    import torch
    from moleculekit_b200 import dcd, trr
    from moleculekit_b200.netcdf import encode_netcdf_device

    dev = torch.device("cuda", 0)
    F, natoms = F_CODEC, 3
    assert -(-F // FT) > GRID_Y
    rng = np.random.default_rng(29)
    nsrc = len(fmt) - 4 if fmt.startswith("trr") else 1
    V = [_values32(rng, F, natoms) for _ in range(nsrc)]
    lead, Fb = 4, F + 9
    views = []
    for v in V:
        t = _sentinel((natoms, 3, Fb), dev)
        t[:, :, lead:lead + F] = torch.from_numpy(np.ascontiguousarray(v.transpose(1, 2, 0))).to(dev)
        views.append(t[:, :, lead:lead + F])
        assert views[-1].stride() == (3 * Fb, Fb, 1)
    words = [v.reshape(F, 3 * natoms).view(np.uint32) for v in V]
    if fmt == "netcdf":
        box = rng.uniform(20, 90, size=(3, F)).astype(np.float32)
        angles = rng.uniform(60, 120, size=(3, F)).astype(np.float32)
        time = rng.uniform(0, 1e5, size=F).astype(np.float32)
        want = np.zeros(F, [("time", ">f4"), ("x", ">u4", (3 * natoms,)), ("lengths", ">f8", (3,)),
                            ("angles", ">f8", (3,))])
        want["time"], want["x"], want["lengths"], want["angles"] = time, words[0], box.T, angles.T
        _prime(F * want.dtype.itemsize, dev)
        got = encode_netcdf_device(views[0], box=box, boxangles=angles, time=time)
    elif fmt.startswith("trr"):
        box = rng.uniform(-5, 9, size=(3, 3, F)).astype(np.float32)
        time = rng.uniform(0, 1e5, size=F).astype(np.float32)
        step = np.arange(F, dtype=np.int64) * 250
        fields = [("head", "u1", (trr.HEAD.itemsize,))] + [(c, ">u4", (3 * natoms,)) for c in "xvf"[:nsrc]]
        want = np.zeros(F, fields)
        want["head"] = trr._heads(natoms, F, box, time, step, None, nsrc > 1, nsrc > 2)
        for c, w in zip("xvf", words):
            want[c] = w
        _prime(F * want.dtype.itemsize, dev)
        got = trr.encode_trr_device(views[0], box, time, step, velocities=views[1] if nsrc > 1 else None,
                                    forces=views[2] if nsrc > 2 else None)
    else:
        box = np.tile(rng.uniform(20, 90, size=(3, 5)).astype(np.float32), (1, F // 5 + 1))[:, :F]
        angles = np.tile(rng.uniform(60, 120, size=(3, 5)).astype(np.float32), (1, F // 5 + 1))[:, :F]
        want = np.zeros(F, [("m0", "<u4"), ("cell", "<f8", (6,)), ("m1", "<u4"), ("r", "<u4", (3, natoms + 2))])
        want["m0"] = want["m1"] = 48
        want["cell"] = dcd.box_to_unitcell(box, angles)
        want["r"][:, :, 0] = want["r"][:, :, -1] = 4 * natoms
        want["r"][:, :, 1:-1] = V[0].transpose(0, 2, 1).view(np.uint32)
        _prime(F * want.dtype.itemsize, dev)
        got = dcd.encode_dcd_device(views[0], box, angles)
    rb = want.dtype.itemsize
    assert tuple(got.shape) == (F * rb,)
    g = got.cpu().numpy().reshape(F, rb)
    _check((g != want.view(np.uint8).reshape(F, rb)).any(axis=1), EDGES_CODEC, "frame")


@pytest.mark.parametrize("fmt", ["netcdf", "trr", "dcd"])
def test_reader_round_trip_more_than_65535_frame_tiles(fmt, tmp_path):
    """one atom over 2 097 157 frames, written by the library's writer (its records are the encode test's) and read
    back whole: the default chunk size keeps the file in one chunk, so one decode call gets every frame"""
    import torch
    from moleculekit_b200 import dcd, netcdf, trr

    dev = torch.device("cuda", 0)
    F, natoms = F_CODEC, 1
    rng = np.random.default_rng(["netcdf", "trr", "dcd"].index(fmt) + 31)
    V = _values32(rng, F, natoms)
    # written from a device copy that stays alive, so the reader's output cannot reuse its block and bits
    X = torch.from_numpy(np.ascontiguousarray(V.transpose(1, 2, 0))).to(dev)
    path = str(tmp_path / f"long.{fmt}")
    if fmt == "netcdf":
        slab, chunk_bytes = 12 * natoms, netcdf.CHUNK_BYTES
        netcdf.write_netcdf(path, X)
        _prime(X.numel() * 4, dev)
        got = netcdf.read_netcdf_device(path)[0]
    elif fmt == "trr":
        slab, chunk_bytes = 12 * natoms, trr.CHUNK_BYTES
        trr.write_trr(path, X, np.zeros((3, 3, F), np.float32), np.zeros(F, np.float32), np.arange(F))
        _prime(X.numel() * 4, dev)
        got = trr.read_trr_device(path)[0]["x"]
    else:
        slab, chunk_bytes = 3 * (8 + 4 * natoms), dcd.CHUNK_BYTES
        dcd.write_dcd(path, X)
        _prime(X.numel() * 4, dev)
        got = dcd.read_dcd_device(path)[0]
    # the readers cut the listed frames into chunks of at most chunk_bytes of staged slabs: this file is one chunk,
    # hence one decode call
    assert F * slab <= chunk_bytes
    assert tuple(got.shape) == (natoms, 3, F)
    _check(_bad_frames(got.cpu().numpy().view(np.uint32), _frame_minor(V)), EDGES_CODEC, "frame")


# ----------------------------------------------------------------------------------------------- 4. SASA / DSSP chunks
def _tiled(base):
    """frame k = base frame k mod 97, over F_CHUNK frames"""
    return np.ascontiguousarray(base[:, :, np.arange(F_CHUNK) % N_BASE])


def _rows_bad(got, base_rows, order):
    """per output row r: does it differ from base row order[r] mod 97?  Bit patterns."""
    want = base_rows[np.asarray(order) % N_BASE]
    g = np.ascontiguousarray(got)
    return (g.view(np.uint8).reshape(g.shape[0], -1) != want.view(np.uint8).reshape(g.shape[0], -1)).any(axis=1)


@pytest.fixture(scope="module")
def sasa_mol():
    from moleculekit_b200.sasa import sasa_radii, sphere_points

    rng = np.random.default_rng(17)
    n = 20
    centre = rng.normal(0, 3.0, size=(n, 3, 1))
    base = (centre + rng.normal(0, 0.4, size=(n, 3, N_BASE))).astype(np.float32)
    radii = sasa_radii(rng.choice(["C", "N", "O", "S", "H"], n), 1.4)
    return dict(base=base, radii=radii, sphere=sphere_points(240), groups=np.array([0, 4, 9, 9, 15, 20], np.int64))


@pytest.mark.parametrize("grouped", [False, True])
def test_sasa_three_chunks(sasa_mol, grouped):
    """131 081 frames of a 20-atom molecule: every row equals its base frame's row, for the whole trajectory into a
    wider matrix and for the reversed frame list; the base rows match the oracle"""
    import torch
    from moleculekit_b200.sasa import chunk_frames, sasa_device

    dev = torch.device("cuda", 0)
    m = sasa_mol
    base, radii, sphere = m["base"], m["radii"], m["sphere"]
    n = base.shape[0]
    groups = m["groups"] if grouped else None
    assert chunk_frames(n, n, 0 if groups is None else len(groups) - 1) == GRID_Y
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    env, q, r, s = t(np.arange(n), np.int32), t(np.arange(n), np.int32), t(radii, np.float32), t(sphere, np.float32)
    g = None if groups is None else t(groups, np.int64)
    base_rows = sasa_device(t(base, np.float32), env, r, q, s, g).cpu().numpy()
    want = so.sasa(base, radii, np.arange(n), sphere, groups)
    assert np.array_equal(base_rows.view(np.int32), want.view(np.int32)), "the base frames differ from the oracle"
    assert len({row.tobytes() for row in base_rows}) == N_BASE  # a misplaced row cannot match by chance
    cols = base_rows.shape[1]
    d = t(_tiled(base), np.float32)
    wide = _sentinel((F_CHUNK, cols + 7), dev)
    sasa_device(d, env, r, q, s, g, out=wide[:, 3:3 + cols])
    w = wide.cpu().numpy()
    _check(_rows_bad(w[:, 3:3 + cols], base_rows, np.arange(F_CHUNK)), EDGES_CHUNK, "row")
    assert (w[:, :3].view(np.uint32) == SENT32).all() and (w[:, 3 + cols:].view(np.uint32) == SENT32).all()
    rev = np.arange(F_CHUNK - 1, -1, -1)
    out = _sentinel((F_CHUNK, cols), dev)
    sasa_device(d, env, r, q, s, g, frames=t(rev, np.int32), out=out)
    _check(_rows_bad(out.cpu().numpy(), base_rows, rev), EDGES_CHUNK, "row")


def test_sasa_coincident_atoms_in_the_second_chunk(sasa_mol):
    """atoms 0 and 1 coincide in frame 65 540 only: the error names that frame of the trajectory, not frame 5 of its
    chunk"""
    import torch
    from moleculekit_b200.sasa import CoincidentAtomsError, sasa_device

    dev = torch.device("cuda", 0)
    m = sasa_mol
    n = m["base"].shape[0]
    X = _tiled(m["base"])
    X[1, :, GRID_Y + 5] = X[0, :, GRID_Y + 5]
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    idx = t(np.arange(n), np.int32)
    with pytest.raises(CoincidentAtomsError, match=f"frame {GRID_Y + 5}") as e:
        sasa_device(t(X, np.float32), idx, t(m["radii"], np.float32), idx, t(m["sphere"], np.float32))
    assert e.value.frame == GRID_Y + 5 and e.value.atoms == (0, 1)


@pytest.mark.parametrize("with_hbonds", [False, True])
def test_dssp_three_chunks(with_hbonds):
    """131 081 frames of an 8-residue peptide (the longest whose chunk holds 65 535 frames): the codes (and both
    hydrogen-bond slots of every donor) of every row equal their base frame's, for the whole trajectory into a wider
    matrix and for the reversed frame list; the base frames match the oracle"""
    import torch
    from moleculekit_b200.dssp import chunk_frames, dssp_device

    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(18)
    nres = 8
    assert chunk_frames(nres) == GRID_Y
    frames = []
    for _ in range(N_BASE):
        helix = rng.random(nres) < 0.7
        phi = np.where(helix, -57.0, -120.0) + rng.normal(0, 12, nres)
        psi = np.where(helix, -47.0, 130.0) + rng.normal(0, 12, nres)
        frames.append(dso.chain(phi, psi).reshape(4 * nres, 3) + rng.normal(0, 0.05, size=(4 * nres, 3)))
    base = np.ascontiguousarray(np.stack(frames, axis=2).astype(np.float32))
    bb = np.arange(4 * nres).reshape(nres, 4)
    flags = np.zeros(nres, np.uint8)
    flags[6] = 1
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    d_bb, d_fl = t(bb, np.int32), t(flags, np.uint8)

    def run(coords, n, frames=None, out=None):
        hb = None
        if with_hbonds:
            hb = (torch.full((n, nres, 2), 0x7EADBEEF, dtype=torch.int32, device=dev),
                  torch.full((n, nres, 2), 0x7FF4A5A5A5A5A5A5, dtype=torch.int64, device=dev).view(torch.float64))
        codes = dssp_device(coords, d_bb, d_fl, frames=frames, out=out, hbonds=hb)
        return codes, hb

    codes, hb = run(t(base, np.float32), N_BASE)
    base_rows = [codes.cpu().numpy()]
    want = dso.dssp(base, bb, flags)
    assert np.array_equal(base_rows[0], want[0]), "the base frames' codes differ from the oracle"
    if with_hbonds:
        base_rows += [hb[0].cpu().numpy(), hb[1].cpu().numpy()]
        assert np.array_equal(base_rows[1], want[1])
        assert np.array_equal(base_rows[2].view(np.int64), want[2].view(np.int64))
        assert len({e.tobytes() for e in base_rows[2]}) == N_BASE  # a misplaced row cannot match by chance
    assert len({c.tobytes() for c in base_rows[0]}) > 20

    d = t(_tiled(base), np.float32)
    wide = torch.full((F_CHUNK, nres + 9), 0xEE, dtype=torch.uint8, device=dev)
    _, hb = run(d, F_CHUNK, out=wide[:, 4:4 + nres])
    w = wide.cpu().numpy()
    assert (w[:, :4] == 0xEE).all() and (w[:, 4 + nres:] == 0xEE).all(), "a margin of the wider matrix was written"
    got = [w[:, 4:4 + nres]] + ([x.cpu().numpy() for x in hb] if with_hbonds else [])
    for name, gv, bv in zip(("code", "partner", "energy"), got, base_rows):
        _check(_rows_bad(gv, bv, np.arange(F_CHUNK)), EDGES_CHUNK, f"{name} row")
    rev = np.arange(F_CHUNK - 1, -1, -1)
    out = torch.full((F_CHUNK, nres), 0xEE, dtype=torch.uint8, device=dev)
    _, hb = run(d, F_CHUNK, frames=t(rev, np.int32), out=out)
    got = [out.cpu().numpy()] + ([x.cpu().numpy() for x in hb] if with_hbonds else [])
    for name, gv, bv in zip(("code", "partner", "energy"), got, base_rows):
        _check(_rows_bad(gv, bv, rev), EDGES_CHUNK, f"{name} row")
