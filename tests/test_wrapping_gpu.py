"""GPU parity of K9 (orthorhombic wrap_box, SURVEY 8f row 4): bit-exact against the reference's compiled kernel outputs
(tests/golden/wrap.npz), the reference's stored golden trajectory, and the oracle on seeded systems."""
import logging

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _fbits(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


def test_reference_golden(g_wrap):
    """tests/test_wrapping.py:9-16 on the committed cut of the reference's system: bit-identical to the reference kernel,
    within the reference test's atol of its stored golden; plus the fixed-centre variant (test_wrapping.py:18-24)."""
    from moleculekit_b200.wrapping import wrap_box

    g = g_wrap
    out = g["coords"].copy()
    assert wrap_box(g["groups"], out, g["box"], g["centersel"], np.zeros(3, np.float32)) is None
    assert np.array_equal(_fbits(out), _fbits(g["ref_wrapped"]))
    assert np.allclose(out, g["gold_wrapped_xtc"], atol=1e-2)
    out = g["coords"].copy()
    wrap_box(g["groups"], out, g["box"], np.zeros(0, np.uint32), g["center_fixed"])
    assert np.array_equal(_fbits(out), _fbits(g["ref_wrapped_fixed"]))


def test_seeded_reference_cases(g_wrap):
    """empty groups (repeated offsets), single-atom groups, a zero box component (NaN translation as in the reference)."""
    from moleculekit_b200.wrapping import wrap_box

    g = g_wrap
    for c in range(int(g["ncase"])):
        out = g[f"r{c}_coords"].copy()
        wrap_box(g[f"r{c}_groups"], out, g[f"r{c}_box"], g[f"r{c}_centersel"], g[f"r{c}_center"])
        assert np.array_equal(_fbits(out), _fbits(g[f"r{c}_ref"])), c


def _solvated(rng, n_protein, n_water, F, box_edge=40.0):
    """unwrapped-looking system: one big group + 3-atom groups that diffused several boxes away"""
    N = n_protein + 3 * n_water
    groups = np.concatenate([[0], n_protein + 3 * np.arange(n_water + 1)]).astype(np.uint32)
    base = rng.normal(0, 8, size=(n_protein, 3, 1)).astype(np.float32) + rng.normal(0, 30, size=(1, 3, F)).astype(np.float32)
    wat_c = rng.uniform(-3 * box_edge, 3 * box_edge, size=(n_water, 1, 3, F)).astype(np.float32)
    wat = (wat_c + rng.normal(0, 0.6, size=(n_water, 3, 3, 1)).astype(np.float32)).reshape(3 * n_water, 3, F)
    coords = np.ascontiguousarray(np.concatenate([base + rng.normal(0, 0.3, size=(n_protein, 3, F)).astype(np.float32), wat]))
    box = (box_edge + rng.uniform(-1, 1, size=(3, F))).astype(np.float32)
    assert coords.shape == (N, 3, F)
    return groups, coords, box


def test_large_vs_oracle_and_device_api(oracle):
    """a solvated system over 64 frames vs the oracle; the device entry wraps the resident tensor in place; a frame shard
    (slice of a resident trajectory, frame_stride > n_frames) wraps only its frames."""
    import torch
    from moleculekit_b200.wrapping import wrap_box, wrap_box_device

    rng = np.random.default_rng(17)
    groups, coords, box = _solvated(rng, 700, 2500, 64)
    centersel = np.arange(0, 700, 3, dtype=np.uint32)
    want = coords.copy()
    oracle.wrap_box(groups, want, box, centersel, np.zeros(3, np.float32))
    got = coords.copy()
    wrap_box(groups, got, box, centersel, np.zeros(3, np.float32))
    assert np.array_equal(_fbits(got), _fbits(want))
    assert (got != coords).mean() > 0.3  # most waters really moved
    # idempotence (size-independent property): wrapping a wrapped trajectory around the same centre moves nothing
    again = got.copy()
    wrap_box(groups, again, box, centersel, np.zeros(3, np.float32))
    assert np.array_equal(_fbits(again), _fbits(got))

    dev = torch.device("cuda:0")
    d_coords = torch.from_numpy(coords).to(dev)
    d_box = torch.from_numpy(box).to(dev)
    d_groups = torch.from_numpy(groups.view(np.int32)).to(dev)
    d_cs = torch.from_numpy(centersel.view(np.int32)).to(dev)
    ret = wrap_box_device(d_coords[:, :, 16:48], d_box[:, 16:48], d_groups, d_cs)
    assert ret.data_ptr() == d_coords[:, :, 16:48].data_ptr()
    shard = d_coords.cpu().numpy()
    assert np.array_equal(_fbits(shard[:, :, 16:48]), _fbits(want[:, :, 16:48]))
    assert np.array_equal(shard[:, :, :16], coords[:, :, :16]) and np.array_equal(shard[:, :, 48:], coords[:, :, 48:])
    # fixed centre on the device path
    cen = np.array([3.5, -2.25, 10.0], np.float32)
    d2 = torch.from_numpy(coords).to(dev)
    wrap_box_device(d2, d_box, d_groups, None, cen)
    want2 = coords.copy()
    oracle.wrap_box(groups, want2, box, np.zeros(0, np.uint32), cen)
    assert np.array_equal(_fbits(d2.cpu().numpy()), _fbits(want2))


def test_single_frame_and_big_group(oracle):
    """F = 1 (a structure) with a 20k-atom group: the sequential running mean of one long group, bit-exact."""
    from moleculekit_b200.wrapping import wrap_box

    rng = np.random.default_rng(23)
    groups, coords, box = _solvated(rng, 20000, 300, 1, box_edge=25.0)
    coords[:20000] += np.float32(60.0)                           # the big group sits several boxes away ...
    centersel = np.arange(20000, 20000 + 90, dtype=np.uint32)    # ... from the centre, taken on some waters
    want = coords.copy()
    oracle.wrap_box(groups, want, box, centersel, np.zeros(3, np.float32))
    got = coords.copy()
    wrap_box(groups, got, box, centersel, np.zeros(3, np.float32))
    assert np.array_equal(_fbits(got), _fbits(want))
    assert not np.array_equal(got[:20000], coords[:20000])


def test_molecule_wrap_mirror(g_wrap, oracle, caplog):
    """Molecule.wrap mirror (molecule.py:1987-2090): bonds -> groups -> wrap_box; zero box is a logged no-op
    (tests/test_wrapping.py:48-75); triclinic cells and bad unitcell names raise."""
    from moleculekit_b200 import wrapping as wr
    from moleculekit_b200.molecule_lite import MolLite

    g = g_wrap
    mask = np.zeros(g["coords"].shape[0], dtype=bool)
    mask[g["centersel"]] = True
    mol = MolLite(g["coords"].copy(), box=g["box"], bonds=g["bonds"], named_selections={"protein or resname ACE NME": mask})
    wr.wrap(mol, "protein or resname ACE NME")
    assert np.array_equal(_fbits(mol.coords), _fbits(g["ref_wrapped"]))
    mol = MolLite(g["coords"].copy(), box=g["box"], bonds=g["bonds"])
    wr.wrap(mol, wrapcenter=g["center_fixed"])
    assert np.array_equal(_fbits(mol.coords), _fbits(g["ref_wrapped_fixed"]))
    mol = MolLite(g["coords"].copy(), box=g["box"], bonds=g["bonds"])
    wr.wrap(mol, wrapsel=mask)                                     # boolean mask selection
    assert np.array_equal(_fbits(mol.coords), _fbits(g["ref_wrapped"]))

    mol = MolLite(g["coords"].copy(), box=np.zeros_like(g["box"]), bonds=g["bonds"])
    with caplog.at_level(logging.WARNING, logger="moleculekit_b200.wrapping"):
        wr.wrap(mol, wrapsel=mask)
    assert np.array_equal(mol.coords, g["coords"])
    assert any("Zero box size" in r.getMessage() for r in caplog.records)

    with pytest.raises(ValueError, match="Invalid unit cell type"):
        wr.wrap(mol, unitcell="cubic")
    mol = MolLite(g["coords"].copy(), box=g["box"][:, :2], bonds=g["bonds"])
    with pytest.raises(RuntimeError, match="different number of simulation frames"):
        wr.wrap(mol, wrapsel=mask)
    # a cell with angles != 90 goes to the triclinic kernels (molecule.py:2078-2090); 60/60/90 = rhombic dodecahedron
    ang = np.repeat(np.array([[60.0], [60.0], [90.0]], np.float32), g["box"].shape[1], axis=1)
    bx = np.repeat(g["box"][:1], 3, axis=0)
    tri = MolLite(g["coords"].copy(), box=bx, bonds=g["bonds"], boxangles=ang)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        wr.wrap(tri, wrapsel=mask, unitcell="compact")
        bv = wr.box_vectors(bx, ang)
    want = g["coords"].copy()
    oracle.wrap_compact_unitcell(g["groups"], want, bv, g["centersel"], np.zeros(3, np.float32), 1)
    assert np.array_equal(_fbits(tri.coords), _fbits(want))


def test_argument_checks():
    from moleculekit_b200.wrapping import wrap_box

    c = np.zeros((4, 3, 2), np.float32)
    b = np.ones((3, 2), np.float32)
    g = np.array([0, 2, 4], np.uint32)
    z = np.zeros(3, np.float32)
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        wrap_box(g.astype(np.int64), c, b, np.zeros(0, np.uint32), z)
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        wrap_box(g, c.astype(np.float64), b, np.zeros(0, np.uint32), z)
    with pytest.raises(IndexError):
        wrap_box(np.array([0, 9], np.uint32), c, b, np.zeros(0, np.uint32), z)
    with pytest.raises(IndexError):
        wrap_box(g, c, b, np.array([4], np.uint32), z)
    # nothing to do: no groups / no atoms / no frames
    wrap_box(np.array([0], np.uint32), c, b, np.zeros(0, np.uint32), z)
    wrap_box(g, np.zeros((0, 3, 2), np.float32), b, np.zeros(0, np.uint32), z)
    wrap_box(g, np.zeros((4, 3, 0), np.float32), np.zeros((3, 0), np.float32), np.zeros(0, np.uint32), z)


def test_exact_division_sequence(tmp_path):
    """csrc/exact_div.cuh (the reciprocal hoisted off the running-mean chain) against __fdiv_rn on ~1.2e9 operand pairs:
    every divisor 1..2^17 plus large ones, numerators over the whole float range and at rounding boundaries."""
    import os
    import shutil
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "divcheck")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-I" + os.path.join(root, "moleculekit_b200", "csrc"),
                    os.path.join(root, "tests", "cuda", "divcheck.cu"), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "mismatches=0" in r.stdout


# ------------------------------------------------------------------------- K9b: triclinic / compact wrapping
TRIC_MODES = (("triclinic", None), ("compact", 1), ("rectangular", 0))


def _gpu_tric(mode, groups, coords, bv, cs, cen):
    from moleculekit_b200.wrapping import wrap_compact_unitcell, wrap_triclinic_unitcell

    if mode is None:
        assert wrap_triclinic_unitcell(groups, coords, bv, cs, cen) is None
    else:
        assert wrap_compact_unitcell(groups, coords, bv, cs, cen, mode) is None


def _oracle_tric(oracle, mode, groups, coords, bv, cs, cen):
    if mode is None:
        oracle.wrap_triclinic_unitcell(groups, coords, bv, cs, cen)
    else:
        oracle.wrap_compact_unitcell(groups, coords, bv, cs, cen, mode)


def test_triclinic_reference_golden(g_tric):
    """tests/test_wrapping.py:26-44 on the committed cut of the reference's dodecahedral system, all three unit cells:
    bit-identical to the reference kernels, within the reference test's tolerance of its stored goldens; the fixed-centre
    variant; seeded reference cases incl. empty groups and atoms outside every group."""
    g = g_tric
    zero = np.zeros(3, np.float32)
    for name, mode in TRIC_MODES:
        out = g["coords"].copy()
        _gpu_tric(mode, g["groups"], out, g["boxvectors"], g["centersel"], zero)
        assert np.array_equal(_fbits(out), _fbits(g[f"ref_{name}"])), name
        assert np.max(np.abs(out - g[f"gold_{name}_xtc"])) < 1e-2, name
        out = g["coords"].copy()
        _gpu_tric(mode, g["groups"], out, g["boxvectors"], np.zeros(0, np.uint32), g["center_fixed"])
        assert np.array_equal(_fbits(out), _fbits(g[f"ref_{name}_fixed"])), name
        for c in range(int(g["ncase"])):
            out = g[f"r{c}_coords"].copy()
            _gpu_tric(mode, g[f"r{c}_groups"], out, g[f"r{c}_boxvectors"], g[f"r{c}_centersel"], g[f"r{c}_center"])
            assert np.array_equal(_fbits(out), _fbits(g[f"r{c}_ref_{name}"])), (name, c)


def _dodecahedron(rng, F, L=62.0):
    vec = np.array([[L, 0, 0], [0, L, 0], [L / 2, L / 2, L * np.sqrt(2) / 2]])
    return np.repeat(vec[:, :, None], F, axis=2) * (1 + 0.002 * rng.normal(size=(1, 1, F)))


def test_triclinic_large_vs_oracle_and_device_api(oracle):
    """a solvated system (one 700-atom group, 2500 waters that diffused several cells away) over 70 frames in a rhombic
    dodecahedron vs the oracle, all three unit cells; the device entry on a resident tensor and on a frame shard."""
    import torch
    from moleculekit_b200.wrapping import wrap_triclinic_device

    rng = np.random.default_rng(23)
    groups, coords, _ = _solvated(rng, 700, 2500, 70, box_edge=60.0)
    bv = _dodecahedron(rng, 70)
    centersel = np.arange(0, 700, 3, dtype=np.uint32)
    zero = np.zeros(3, np.float32)
    for name, mode in TRIC_MODES:
        want = coords.copy()
        _oracle_tric(oracle, mode, groups, want, bv, centersel, zero)
        got = coords.copy()
        _gpu_tric(mode, groups, got, bv, centersel, zero)
        assert np.array_equal(_fbits(got), _fbits(want)), name
        # wrapped groups sit in the cell: wrapping the result again moves (almost) nothing
        if name != "triclinic":
            again = got.copy()
            _gpu_tric(mode, groups, again, bv, centersel, zero)
            assert np.max(np.abs(again - got)) < 1e-2
    # device API, frames 16..48 of a resident trajectory (frame_stride 70 > 32 frames)
    dev = torch.device("cuda:0")
    d = torch.from_numpy(coords).to(dev)
    dbv = torch.from_numpy(bv).to(dev)
    dg = torch.from_numpy(groups.view(np.int32)).to(dev)
    dcs = torch.from_numpy(centersel.view(np.int32)).to(dev)
    out = wrap_triclinic_device(d[:, :, 16:48], dbv[:, :, 16:48], dg, dcs, None, "compact")
    assert out.data_ptr() == d[:, :, 16:48].data_ptr()
    want = coords.copy()
    sub = np.ascontiguousarray(coords[:, :, 16:48])
    oracle.wrap_compact_unitcell(groups, sub, np.ascontiguousarray(bv[:, :, 16:48]), centersel, zero, 1)
    want[:, :, 16:48] = sub
    assert np.array_equal(_fbits(d.cpu().numpy()), _fbits(want))


def test_triclinic_long_groups_and_edge_cases(oracle):
    """a 20 000-atom group (many pipeline stages), odd frame counts, groups of every small size, a fixed centre far from
    the cell, and the reference's ValueError for a cell with more than 12 correction vectors."""
    from moleculekit_b200.wrapping import wrap_compact_unitcell

    rng = np.random.default_rng(31)
    for F in (1, 33):
        sizes = [20000, 1, 2, 3, 4, 5, 37, 1, 260]
        groups = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
        N = int(groups[-1])
        coords = (rng.normal(0, 5, size=(N, 3, F)) + rng.uniform(-200, 200, size=(1, 3, F))).astype(np.float32)
        for k in range(1, len(sizes)):
            coords[groups[k]:groups[k + 1]] += rng.uniform(-150, 150, size=(1, 3, F)).astype(np.float32)
        L = 48.0
        vec = np.array([[L, 0, 0], [L / 3, 2 * np.sqrt(2) * L / 3, 0], [-L / 3, np.sqrt(2) * L / 3, np.sqrt(6) * L / 3]])
        bv = np.repeat(vec[:, :, None], F, axis=2) * (1 + 0.002 * rng.normal(size=(1, 1, F)))
        cen = np.array([300.0, -120.0, 55.5], np.float32)
        for name, mode in TRIC_MODES:
            for cs in (np.zeros(0, np.uint32), np.arange(10, 19000, 7, dtype=np.uint32)):
                want, got = coords.copy(), coords.copy()
                _oracle_tric(oracle, mode, groups, want, bv, cs, cen)
                _gpu_tric(mode, groups, got, bv, cs, cen)
                assert np.array_equal(_fbits(got), _fbits(want)), (F, name, len(cs))
    # heavily skewed, unreduced cell: get_pbc finds more than 12 vectors (wrapping.pyx:439-441)
    bad = np.array([[30.0, 0, 0], [11.9, 27.0, 0], [-11.8, 11.9, 33.0]])[:, :, None].copy()
    xyz = rng.normal(0, 30, size=(10, 3, 1)).astype(np.float32)
    g2 = np.array([0, 5, 10], np.uint32)
    try:
        oracle.wrap_compact_unitcell(g2, xyz.copy(), bad, np.zeros(0, np.uint32), np.zeros(3, np.float32), 1)
        raised = False
    except ValueError:
        raised = True
    if raised:
        with pytest.raises(ValueError, match="Too many triclinic vectors"):
            wrap_compact_unitcell(g2, xyz.copy(), bad, np.zeros(0, np.uint32), np.zeros(3, np.float32), 1)


def test_wrap_mirror_dispatches_on_boxangles(g_tric):
    """wrapping.wrap (Molecule.wrap mirror, molecule.py:2075-2090) takes the triclinic kernels when a box angle != 90 and
    builds the box vectors from lengths / angles when the container has no boxvectors attribute."""
    import warnings

    from moleculekit_b200.wrapping import wrap

    g = g_tric

    class Mol:
        pass

    for unitcell in ("triclinic", "compact", "rectangular"):
        m = Mol()
        m.coords = g["coords"].copy()
        m.box, m.boxangles = g["box"], g["boxangles"]
        m.numAtoms = m.coords.shape[0]
        # one "bond" chain per group so that getBondedGroups reproduces the fixture's groups
        gr = g["groups"].astype(np.int64)
        m.bonds = np.concatenate([np.stack([np.arange(a, b - 1), np.arange(a + 1, b)], 1) for a, b in zip(gr[:-1], gr[1:])
                                  if b - a > 1]).astype(np.uint32)
        sel = np.zeros(m.numAtoms, bool)
        sel[g["centersel"]] = True
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            wrap(m, wrapsel=sel, unitcell=unitcell)
        assert np.array_equal(_fbits(m.coords), _fbits(g[f"ref_{unitcell}"])), unitcell


def test_triclinic_edge_cases(oracle):
    """no groups (every atom is only centred), a single closing offset, zero frames, one atom"""
    from moleculekit_b200.wrapping import wrap_compact_unitcell, wrap_triclinic_unitcell

    rng = np.random.default_rng(9)
    L = 15.0
    xyz = rng.normal(0, 40, size=(11, 3, 4)).astype(np.float32)
    bv = np.repeat(np.array([[L, 0, 0], [0, L, 0], [L / 2, L / 2, L * 2 ** 0.5 / 2]])[:, :, None], 4, axis=2)
    cen = np.array([1.0, -2.0, 3.0], np.float32)
    for groups in (np.zeros(0, np.uint32), np.array([11], np.uint32), np.array([0, 11], np.uint32), np.array([3, 7], np.uint32)):
        for mode in (None, 0, 1):
            want, got = xyz.copy(), xyz.copy()
            _oracle_tric(oracle, mode, groups, want, bv, np.zeros(0, np.uint32), cen)
            _gpu_tric(mode, groups, got, bv, np.zeros(0, np.uint32), cen)
            assert np.array_equal(_fbits(got), _fbits(want)), (groups.tolist(), mode)
    empty = xyz[:, :, :0].copy()
    wrap_triclinic_unitcell(np.array([0, 11], np.uint32), empty, bv[:, :, :0].copy(), np.zeros(0, np.uint32), cen)
    wrap_compact_unitcell(np.array([0, 1], np.uint32), xyz[:1].copy(), bv, np.zeros(0, np.uint32), cen, 1)
