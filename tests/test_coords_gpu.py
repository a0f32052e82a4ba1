"""GPU parity of K15 (aligned coordinates, frame sums, fluctuations): coordinates bit-identical to the K14 apply followed
by a gather (hence within one float32 ulp of the float64 oracle), frame sums whose bits depend only on the selection and
the ordered frame list, fluctuations bit-identical to the same formula on the device's own coordinates and within
1e-6 relative of the float64 oracle (oracle/coords_oracle.py), and the MetricCoordinate / MetricFluctuation drop-ins."""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import coords_oracle as co

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _within_ulp(got, want64):
    """every coordinate within one float32 ulp of the float64 result rounded to float32 (never below 1e-12 A)"""
    w32 = want64.astype(np.float32)
    assert got.dtype == np.float32 and got.shape == w32.shape
    err = np.abs(got.astype(np.float64) - w32.astype(np.float64))
    ok = err <= np.maximum(np.spacing(np.abs(w32)).astype(np.float64), 1e-12)
    assert ok.all(), f"{np.count_nonzero(~ok)} coordinates off by up to {err[~ok].max():.3e} A"


def _f32(rows64):
    """the float64 superposition rounded to float32, as the device rounds it"""
    return rows64.astype(np.float32).astype(np.float64)


def _rotated(frame, seed):
    G = Rotation.random(random_state=seed).as_matrix()
    return (frame.astype(np.float64) @ G + [12.5, -30.0, 7.25]).astype(np.float32)


def _t(a, dev, dtype=None):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).to(dev)


def _gathered(applied, sel):
    """(N, 3, F) tensor -> (F, 3k) rows of the ``sel`` atoms, X block | Y block | Z block"""
    S = applied[sel.long()]
    return S.permute(2, 1, 0).reshape(S.shape[2], 3 * S.shape[0])


def _bits(t):
    import torch

    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def _setup(g_traj):
    import torch
    from moleculekit_b200.align import superpose_device

    dev = torch.device("cuda:0")
    X = g_traj["coords"]
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    d = _t(X, dev)
    ref = _rotated(X[:, :, 7], 2)[:, :, None]
    d_ca = _t(np.where(ca)[0], dev, np.int32)
    rec, st = superpose_device(d, d_ca, _t(ref, dev), d_ca)
    assert int(st.sum()) == 0
    return dev, X, ca, noh, d, ref, d_ca, rec


def test_coordinates_equal_apply_then_gather(g_traj):
    import torch
    from moleculekit_b200.align import apply_device, superpose_device
    from moleculekit_b200.coords import coordinates_device

    dev, X, ca, noh, d, ref, d_ca, rec = _setup(g_traj)
    sel = _t(np.where(noh)[0][::-1].copy(), dev, np.int32)  # any order: columns follow the selection
    k, F = int(sel.numel()), X.shape[2]
    whole = coordinates_device(d, sel, rec)
    assert whole.shape == (F, 3 * k) and torch.equal(_bits(whole), _bits(_gathered(apply_device(d.clone(), rec), sel)))
    assert torch.equal(_bits(coordinates_device(d, sel)), _bits(_gathered(d, sel)))
    assert np.array_equal(d.cpu().numpy(), X)  # the trajectory is not modified
    fl = _t(np.array([17, 2, 9, 0]), dev, np.int32)
    rec_fl, _ = superpose_device(d, d_ca, _t(ref, dev), d_ca, fl)
    assert torch.equal(_bits(coordinates_device(d, sel, rec_fl, fl)), _bits(whole[fl.long()]))
    # frame shards written through the row stride into column slices of a wider matrix
    wide = torch.full((F, 3 * k + 37), -1.0, device=dev)
    for f0, f1 in ((0, 7), (7, 8), (8, 20)):
        coordinates_device(d[:, :, f0:f1], sel, rec[f0:f1], out=wide[f0:f1, 5:5 + 3 * k])
    assert torch.equal(_bits(wide[:, 5:5 + 3 * k]), _bits(whole))
    assert bool((wide[:, :5] == -1).all()) and bool((wide[:, 5 + 3 * k:] == -1).all())
    want = co.coordinates(X, sel.cpu().numpy(), ref, ca, ca)
    _within_ulp(whole.cpu().numpy(), want)


def test_frame_sums_fixed_order(g_traj):
    import torch
    from moleculekit_b200.align import superpose_device
    from moleculekit_b200.coords import coord_sums_device, coordinates_device

    dev = torch.device("cuda:0")
    X = g_traj["coords"]
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    rng = np.random.default_rng(3)
    Y = np.concatenate([X] * 30, axis=2) + rng.normal(0, 0.4, size=(X.shape[0], 3, 600)).astype(np.float32)
    d = _t(Y, dev)
    d_ca, sel = _t(np.where(ca)[0], dev, np.int32), _t(np.where(noh)[0], dev, np.int32)
    rec, _ = superpose_device(d, d_ca, d[:, :, :1], d_ca)
    s1 = coord_sums_device(d, sel, rec)
    assert s1.shape == (int(sel.numel()), 3) and s1.dtype == torch.float64
    assert torch.equal(_bits(s1), _bits(coord_sums_device(d, sel, rec)))
    # a frame-slice view gives the bits of the same explicit frame list (several 64-frame chunks)
    f0, f1 = 37, 581
    fl = _t(np.arange(f0, f1), dev, np.int32)
    sv = coord_sums_device(d[:, :, f0:f1], sel, rec[f0:f1])
    assert torch.equal(_bits(sv), _bits(coord_sums_device(d, sel, rec[f0:f1], fl)))
    rows = coordinates_device(d, sel, rec).cpu().numpy().astype(np.float64)
    want = co.as_points(rows).sum(axis=0)
    assert np.allclose(s1.cpu().numpy(), want, rtol=1e-12, atol=0)
    assert np.allclose(sv.cpu().numpy(), co.as_points(rows[f0:f1]).sum(axis=0), rtol=1e-12, atol=0)
    assert torch.equal(coord_sums_device(d, sel, rec[:0], _t(np.zeros(0), dev, np.int32)), torch.zeros_like(s1))
    assert coordinates_device(d, sel, rec[:0], _t(np.zeros(0), dev, np.int32)).shape == (0, 3 * int(sel.numel()))


def _same_formula(rows32, centre, offsets):
    """the kernel's formula in numpy on the device's own coordinates: ((e0*e0 + e1*e1) + e2*e2) per atom in float64,
    group sums added in selection order, one rounding to float32"""
    e = co.as_points(rows32.astype(np.float64)) - centre[None]
    v = e[:, :, 0] * e[:, :, 0] + e[:, :, 1] * e[:, :, 1] + e[:, :, 2] * e[:, :, 2]
    if offsets is None:
        return v.astype(np.float32)
    out = np.empty((v.shape[0], offsets.size - 1))
    for g, (a, b) in enumerate(zip(offsets[:-1], offsets[1:])):
        s = np.zeros(v.shape[0])
        for j in range(a, b):
            s = s + v[:, j]
        out[:, g] = s / (b - a)
    return out.astype(np.float32)


@pytest.mark.parametrize("mode", ["atom", "residue"])
@pytest.mark.parametrize("with_ref", [False, True])
def test_fluctuation_bitwise_and_oracle(g_traj, mode, with_ref):
    import torch
    from moleculekit_b200.coords import coord_sums_device, coordinates_device, fluctuation_device

    dev, X, ca, noh, d, ref, d_ca, rec = _setup(g_traj)
    idx = np.where(noh)[0]
    offsets = None
    if mode == "residue":
        order, offsets = co.residue_groups(g_traj["resid"][idx])
        idx = idx[order]
    sel = _t(idx, dev, np.int32)
    d_off = None if offsets is None else _t(offsets, dev)
    records = rec if with_ref else None
    F = X.shape[2]
    if with_ref:
        centre = _t(ref[idx, :, 0], dev, np.float64)
    else:
        centre = coord_sums_device(d, sel, records) / F
    got = fluctuation_device(d, sel, centre, records, groups=d_off)
    rows32 = coordinates_device(d, sel, records).cpu().numpy()
    c = centre.cpu().numpy()
    assert got.shape == (F, idx.size if offsets is None else offsets.size - 1)
    assert np.array_equal(got.cpu().numpy().view(np.uint32), _same_formula(rows32, c, offsets).view(np.uint32))
    rows = _f32(co.coordinates(X, idx, ref if with_ref else None, ca, ca))
    want = co.fluctuation(rows, ref[idx, :, 0] if with_ref else co.mean(rows), offsets)
    assert np.allclose(got.cpu().numpy(), want, rtol=1e-6, atol=1e-9)
    # frame shards through the row stride equal the whole call
    out = torch.empty_like(got)
    for f0, f1 in ((0, 13), (13, 20)):
        fluctuation_device(d[:, :, f0:f1], sel, centre, None if records is None else records[f0:f1], groups=d_off,
                           out=out[f0:f1])
    assert torch.equal(_bits(out), _bits(got))


def _names(g_traj):
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    return {"protein and name CA": ca, "protein and noh": noh, "protein": noh}


def _lite(coords, g=None, **kw):
    from moleculekit_b200.molecule_lite import MolLite

    if g is not None:
        kw.update(resid=g["resid"], resname=g["resname"], name=g["name"], named_selections=_names(g))
    return MolLite(coords, **kw)


def test_projections_traj20(g_traj):
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation

    X = g_traj["coords"]
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    idx = np.where(noh)[0]
    ref = _lite(np.stack([X[:, :, 0], _rotated(X[:, :, 7], 2)], axis=2), g_traj, frame=1)
    mol = _lite(X.copy(), g_traj)
    got = MetricCoordinate("protein and noh", refmol=ref, pbc=False).project(mol)
    R = ref.coords[:, :, 1:2]
    want = co.coordinates(X, idx, R, ca, ca)
    assert got.dtype == np.float32 and got.shape == (20, 3 * idx.size)
    _within_ulp(got, want)
    plain = MetricCoordinate("protein and noh", pbc=False).project(mol)
    assert np.array_equal(plain, co.coordinates(X, idx).astype(np.float32))
    for mode in ("atom", "residue"):
        offsets, order = None, np.arange(idx.size)
        if mode == "residue":
            order, offsets = co.residue_groups(g_traj["resid"][idx])
        rows = _f32(want)
        pts = co.as_points(rows)[:, order]
        rows_o = np.ascontiguousarray(np.transpose(pts, (0, 2, 1)).reshape(20, -1))
        f = MetricFluctuation("protein and noh", refmol=ref, pbc=False, mode=mode).project(mol)
        assert f.dtype == np.float32
        assert np.allclose(f, co.fluctuation(rows_o, R[idx[order], :, 0], offsets), rtol=1e-6, atol=1e-9)
        f = MetricFluctuation("protein and noh", pbc=False, mode=mode).project(mol)
        rows_p = co.coordinates(X, idx[order])
        assert np.allclose(f, co.fluctuation(rows_p, co.mean(rows_p), offsets), rtol=1e-6, atol=1e-9)
        if mode == "residue":
            assert f.shape == (20, np.unique(g_traj["resid"][idx]).size)
    assert np.array_equal(mol.coords, X)  # project does not modify the molecule


@pytest.mark.parametrize("cell", ["orthorhombic", "triclinic"])
def test_projections_pbc_wrap(cell, request):
    """pbc=True wraps on the device exactly as Molecule.wrap around `centerstr` (the MetricRmsd pattern): the expected
    values are the oracle applied to the reference's own wrapped coordinates; the selection holds solvent atoms that
    the wrap moves, so a missing or different wrap changes the result."""
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation

    if cell == "orthorhombic":
        g = request.getfixturevalue("g_wrap")
        W, bonds, angles = g["ref_wrapped"], g["bonds"], None
    else:
        g = request.getfixturevalue("g_tric")
        W, angles = g["ref_rectangular"], g["boxangles"]
        gr = g["groups"].astype(np.int64)
        bonds = np.concatenate([np.stack([np.arange(a, b - 1), np.arange(a + 1, b)], 1)
                                for a, b in zip(gr[:-1], gr[1:]) if b - a > 1]).astype(np.uint32)
    X = g["coords"]
    N = X.shape[0]
    protein = np.zeros(N, bool)
    protein[g["centersel"]] = True
    aln = protein & (np.arange(N) % 4 == 0)
    moved_solvent = np.where(np.any(X != W, axis=(1, 2)) & ~protein)[0][:400]
    assert moved_solvent.size == 400
    sel = protein & (np.arange(N) % 3 == 0)
    sel[moved_solvent] = True
    idx = np.where(sel)[0]
    names = {"protein": protein, "aln": aln, "sel": sel}
    ref = _lite(X[:, :, 0], named_selections=names)
    mol = _lite(X.copy(), box=g["box"], bonds=bonds, boxangles=angles, named_selections=names)
    got = MetricCoordinate("sel", refmol=ref, trajalnsel="aln", centersel="protein").project(mol)
    want = co.coordinates(W, idx, ref.coords, aln, aln)
    _within_ulp(got, want)
    unwrapped = MetricCoordinate("sel", refmol=ref, trajalnsel="aln", pbc=False).project(mol)
    _within_ulp(unwrapped, co.coordinates(X, idx, ref.coords, aln, aln))
    f = MetricFluctuation("sel", refmol=ref, trajalnstr="aln", centerstr="protein").project(mol)
    assert np.allclose(f, co.fluctuation(_f32(want), ref.coords[idx, :, 0]), rtol=1e-6, atol=1e-9)
    f = MetricFluctuation("sel", centerstr="protein").project(mol)
    rows_w = co.coordinates(W, idx)
    assert np.allclose(f, co.fluctuation(rows_w, co.mean(rows_w)), rtol=1e-6, atol=1e-9)
    rows_x = co.coordinates(X, idx)
    assert not np.allclose(f, co.fluctuation(rows_x, co.mean(rows_x)), rtol=1e-3)  # the wrap matters
    assert np.array_equal(mol.coords, X)  # project does not modify the molecule


def test_nonfinite_coordinates(g_traj):
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation

    X = g_traj["coords"][:, :, :8].copy()
    ca, noh = g_traj["sel_masks"][0], g_traj["sel_masks"][2]
    ref = _lite(_rotated(X[:, :, 3], 5), g_traj)
    Xn = X.copy()
    Xn[int(np.where(ca)[0][3]), 1, 5] = np.nan
    for m in (MetricCoordinate("protein and noh", refmol=ref, pbc=False),
              MetricFluctuation("protein and noh", refmol=ref, pbc=False)):
        with pytest.raises(np.linalg.LinAlgError):
            m.project(_lite(Xn.copy(), g_traj))

    idx = np.where(noh)[0]
    free = np.where(noh & ~ca)[0][10]
    col = int(np.where(idx == free)[0][0])
    Xn = X.copy()
    Xn[free, 0, 5] = np.nan
    mol = _lite(Xn, g_traj)
    got = MetricCoordinate("protein and noh", refmol=ref, pbc=False).project(mol)
    nan = np.isnan(got)
    k = idx.size
    assert nan[5, [col, k + col, 2 * k + col]].all() and nan.sum() == 3
    keep = np.ones(k, bool)
    keep[col] = False
    want = co.coordinates(X, idx, ref.coords, ca, ca)
    kk = np.concatenate([keep] * 3)
    _within_ulp(got[:, kk], want[:, kk])
    f = MetricFluctuation("protein and noh", refmol=ref, pbc=False).project(mol)
    assert np.isnan(f[5, col]) and np.isnan(f).sum() == 1
    wf = co.fluctuation(_f32(want), ref.coords[idx, :, 0])
    ok = ~np.isnan(f)
    assert np.allclose(f[ok], wf[ok], rtol=1e-6, atol=1e-9)


def test_full_size_shards_and_oracle():
    """10 000 frames x 5 000 selected atoms: frame shards equal the whole call, sampled frames match the oracle"""
    import torch
    from moleculekit_b200.align import superpose_device
    from moleculekit_b200.coords import coord_sums_device, coordinates_device, fluctuation_device

    dev = torch.device("cuda:0")
    N, F = 6000, 10000
    g = torch.Generator(device=dev).manual_seed(7)
    base = torch.randn((N, 3, 1), generator=g, device=dev) * 15 + 80
    X = (base + torch.randn((N, 3, F), generator=g, device=dev) * 0.7).contiguous()
    aln = torch.from_numpy(np.arange(0, N, 6, dtype=np.int32)).to(dev)
    idx = np.arange(500, 5500, dtype=np.int32)
    sel = torch.from_numpy(idx).to(dev)
    ref = X[:, :, 123:124]
    rec, st = superpose_device(X, aln, ref, aln)
    assert int(st.sum()) == 0
    whole = coordinates_device(X, sel, rec)
    shards = torch.empty_like(whole)
    for f0, f1 in ((0, 2500), (2500, 7001), (7001, 10000)):
        coordinates_device(X[:, :, f0:f1], sel, rec[f0:f1], out=shards[f0:f1])
    assert torch.equal(_bits(shards), _bits(whole))
    sample = np.random.default_rng(1).choice(F, 10, replace=False)
    Xs = X[:, :, sample].cpu().numpy()
    a = aln.cpu().numpy()
    want = co.coordinates(Xs, idx, ref.cpu().numpy(), a, a)
    _within_ulp(whole[sample].cpu().numpy(), want)
    sums = coord_sums_device(X, sel, rec)
    assert torch.equal(_bits(sums), _bits(coord_sums_device(X, sel, rec)))
    want_sums = whole.double().sum(0).reshape(3, -1).T
    assert torch.allclose(sums, want_sums, rtol=1e-12, atol=0)
    del whole, shards
    centre = sums / F
    fl = fluctuation_device(X, sel, centre, rec)
    part = torch.empty_like(fl)
    for f0, f1 in ((0, 4096), (4096, 10000)):
        fluctuation_device(X[:, :, f0:f1], sel, centre, rec[f0:f1], out=part[f0:f1])
    assert torch.equal(_bits(part), _bits(fl))
    wf = co.fluctuation(_f32(want), centre.cpu().numpy())
    assert np.allclose(fl[sample].cpu().numpy(), wf, rtol=1e-6, atol=1e-9)


WORKER = r'''
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["MKB_ROOT"])
rank = int(os.environ["RANK"]); local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from moleculekit_b200.molecule_lite import MolLite
from moleculekit_b200.projections.metricfluctuation import MetricFluctuation
from moleculekit_b200.sharding import fluctuation_sharded
g = np.random.default_rng(4)
N, F = 300, 41
X = (g.normal(size=(N, 1, 1)) * 10 + g.normal(size=(N, 3, F))).astype(np.float32)
sel = np.arange(N) % 2 == 0
mol = MolLite(X, resid=np.arange(N) // 7, named_selections={"sel": sel})
for mode in ("atom", "residue"):
    m = MetricFluctuation("sel", pbc=False, mode=mode)
    one = m.project(mol)
    two = fluctuation_sharded(m, mol)
    assert two.shape == one.shape and np.allclose(two, one, rtol=1e-6, atol=0), mode
dist.barrier(); dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_fluctuation_sharded_two_gpus(tmp_path):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, MKB_ROOT=ROOT)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537", str(script)],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "rank 0 ok" in r.stdout and "rank 1 ok" in r.stdout
