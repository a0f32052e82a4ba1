"""GPU parity of K18 (DSSP) against the C restatement of the reference (tests/dssp_oracle.c): the codes are equal and
both hydrogen-bond slots of every donor are bit-identical (partners, and energies as float64 bits), so a wrong energy
that happens not to flip a decision is still caught."""
import numpy as np
import pytest

import dssp_oracle as do

pytestmark = pytest.mark.gpu


def _t(a, dtype):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to("cuda:0")


def _device(X, bb, flags, frames=None):
    """(codes, partner, energy) of dssp_device on host arrays"""
    import torch
    from moleculekit_b200.dssp import dssp_device

    n = X.shape[2] if frames is None else len(frames)
    hp = torch.empty((n, bb.shape[0], 2), dtype=torch.int32, device="cuda:0")
    he = torch.empty((n, bb.shape[0], 2), dtype=torch.float64, device="cuda:0")
    codes = dssp_device(_t(X, np.float32), _t(bb, np.int32), _t(flags, np.uint8),
                        None if frames is None else _t(frames, np.int32), hbonds=(hp, he))
    return codes.cpu().numpy(), hp.cpu().numpy(), he.cpu().numpy()


def _same(got, want):
    (gc, gp, ge), (wc, wp, we) = got, want
    assert gc.shape == wc.shape and gp.shape == wp.shape and ge.shape == we.shape
    bad = np.argwhere(gp != wp)
    assert bad.size == 0, f"{len(bad)} partners differ, first at {bad[0].tolist()}"
    bad = np.argwhere(ge.view(np.int64) != we.view(np.int64))
    assert bad.size == 0, f"{len(bad)} energies differ, first at {bad[0].tolist()}: {ge[tuple(bad[0])]} vs {we[tuple(bad[0])]}"
    bad = np.argwhere(gc != wc)
    assert bad.size == 0, f"{len(bad)} codes differ, first (frame, residue) {bad[0].tolist()}"


def _check(X, bb, flags, frames=None):
    got = _device(X, bb, flags, frames)
    _same(got, do.dssp(X, bb, flags, frames))
    return got


def _table(g, prot):
    from moleculekit_b200.molecule_lite import MolLite
    from moleculekit_b200.projections.metricsecondarystructure import dssp_residues

    mol = MolLite(g["coords"], name=g["name"], resname=g["resname"], resid=g["resid"], chain=g["chain"],
                  segid=g["segid"], named_selections={"protein": prot})
    bb, fl, _, _ = dssp_residues(mol, prot)
    return mol, bb, fl


def test_3ptb(g_3ptb):
    _, bb, fl = _table(g_3ptb, g_3ptb["sel_protein"])
    codes, _, _ = _check(g_3ptb["coords"], bb, fl)
    assert bb.shape[0] == 220 and (fl & 1).sum() == 8
    assert (codes == 3).sum() > 50 and (codes == 1).sum() > 10


def test_traj20_all_frames(g_traj):
    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    assert bb.shape[0] == 277
    _check(g_traj["coords"], bb, fl)


def test_traj20_noisy_frames(g_traj):
    """200 frames with 0.1-0.5 A Gaussian noise: bonds cross -0.5 and bends cross 70 degrees"""
    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    rng = np.random.default_rng(7)
    atoms = np.unique(bb)
    X = np.ascontiguousarray(np.tile(g_traj["coords"][atoms], (1, 1, 10)))
    sigma = rng.uniform(0.1, 0.5, size=X.shape[2]).astype(np.float32)
    X += (rng.normal(size=X.shape) * sigma).astype(np.float32)
    rows = np.searchsorted(atoms, bb)
    codes, _, _ = _check(X, rows, fl)
    assert len({c.tobytes() for c in codes}) > 150  # the noise changes the assignment from frame to frame


def _constructions():
    out = [("helix", do.chain([-57] * 20, [-47] * 20).astype(np.float32), np.zeros(20, np.uint8)),
           ("310", do.chain([-49] * 20, [-26] * 20).astype(np.float32), np.zeros(20, np.uint8))]
    out.append(("anti",) + do.strand_pair(10, True))
    out.append(("par",) + do.strand_pair(10, False))
    bb, fl = do.strand_pair(10, True)
    f = np.zeros(13, np.uint8)
    f[10] = 2
    out.append(("iso", np.concatenate([bb[:10], bb[13:16]]), f))
    phi, psi = [180.0] * 12, [180.0] * 12
    phi[6], psi[6] = 60.0, 60.0
    out.append(("bend", do.chain(phi, psi).astype(np.float32), np.zeros(12, np.uint8)))
    bb = do.chain([-57] * 20, [-47] * 20)
    d = bb[10, 0] - bb[9, 2]
    bb[10:] += 2.0 * d / np.linalg.norm(d)
    out.append(("split", bb.astype(np.float32), np.zeros(20, np.uint8)))
    return out


@pytest.mark.parametrize("case", range(7))
def test_constructions(case):
    name, bb, fl = _constructions()[case]
    n = bb.shape[0]
    X = np.ascontiguousarray(bb.reshape(n * 4, 3)[:, :, None])
    codes, _, _ = _check(X, np.arange(4 * n).reshape(n, 4), fl)
    assert codes.any()


@pytest.mark.parametrize("second", [3, 34])
def test_mirror_tie(second):
    """donor 1 sees acceptors 2 and ``second`` at mirror-image positions (y -> -y with the donor's N, H and CA on y = 0),
    so their energies tie bit for bit; the lower index takes slot 0.  34 shares lane 2's stride in the warp, 3 does
    not."""
    n = second + 1
    bb = np.zeros((n, 4, 3), np.float32)
    for r in range(n):  # fillers far apart, each its own chain
        bb[r] = np.array([[0, 0, 0], [1.4, 0, 0], [2.0, 1.2, 0], [1.6, 2.3, 0]]) + np.array([0, 0, 60.0 * r])
    bb[0] = [[-2.5, 0, 0.5], [-2.4, 0, 1.9], [-1.3, 0, 0], [-1.3, 0, 1.25]]
    bb[1] = [[0, 0, 0], [0.5, 0, 1.4], [1.9, 0, 1.6], [2.4, 0, 2.7]]
    acc = np.array([[2.2, 2.4, -3.6], [1.0, 2.5, -4.5], [0, 1.4, -4.0], [0, 1.0, -2.9]], np.float32)
    bb[2] = acc
    bb[second] = acc * np.array([1, -1, 1], np.float32)
    fl = np.full(n, 2, np.uint8)
    fl[1] = 0  # residue 1 continues residue 0, so its H follows C0 = O0
    X = np.ascontiguousarray(bb.reshape(n * 4, 3)[:, :, None])
    _, partner, energy = _check(X, np.arange(4 * n).reshape(n, 4), fl)
    assert partner[0, 1].tolist() == [2, second] and energy[0, 1, 0] == energy[0, 1, 1] < 0


def test_proline_donors(g_traj):
    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    fl = fl.copy()
    fl[np.random.default_rng(3).choice(bb.shape[0], 40, replace=False)] |= 1
    _, partner, energy = _check(g_traj["coords"][:, :, :4], bb, fl)
    pro = (fl & 1) == 1
    assert (partner[:, pro] == -1).all() and (energy[:, pro] == 0).all()


def test_nan_coordinates(g_traj):
    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    X = np.ascontiguousarray(g_traj["coords"][:, :, :4]).copy()
    X[bb[10, 1], 0, 1] = np.nan       # a CA: no pair screened with it
    X[bb[50, 3], :, 2] = np.nan       # an O
    X[bb[51, 0], 2, 2] = np.nan       # an N: C-N distance NaN, not a break
    X[bb[120:125, 2], 1, 3] = np.inf  # C atoms
    _check(X, bb, fl)


def test_tiled_5000_residues(g_traj):
    """19 translated copies of the protein as separate chains: 5 263 residues"""
    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    atoms = np.unique(bb)
    rows = np.searchsorted(atoms, bb)
    X0 = g_traj["coords"][atoms][:, :, :2]
    copies = 19
    X = np.ascontiguousarray(np.concatenate([X0 + np.float32(100 * c) for c in range(copies)]))
    BB = np.concatenate([rows + c * atoms.size for c in range(copies)])
    FL = np.tile(fl, copies)
    FL[::bb.shape[0]] |= 2
    codes, _, _ = _check(X, BB, FL)
    assert BB.shape[0] >= 5000
    assert (codes[:, :277] == codes[:, -277:]).all()


def test_chunk_boundary(g_traj):
    """enough frames that the call crosses a frame-chunk boundary; the tiled frames repeat every 20"""
    from moleculekit_b200.dssp import chunk_frames

    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    atoms = np.unique(bb)
    rows = np.searchsorted(atoms, bb)
    fc = chunk_frames(bb.shape[0])
    F = fc + 25
    X = np.ascontiguousarray(np.tile(g_traj["coords"][atoms], (1, 1, F // 20 + 1))[:, :, :F])
    codes, partner, energy = _device(X, rows, fl)
    want = do.dssp(X, rows, fl, frames=list(range(20)))
    k = np.arange(F) % 20
    _same((codes, partner, energy), (want[0][k], want[1][k], want[2][k]))


def test_frames_slices_and_shards(g_traj):
    import torch
    from moleculekit_b200.dssp import dssp_device

    _, bb, fl = _table(g_traj, g_traj["sel_masks"][5])
    n = bb.shape[0]
    d, b, f = _t(g_traj["coords"], np.float32), _t(bb, np.int32), _t(fl, np.uint8)
    whole = dssp_device(d, b, f)
    wide = torch.full((20, n + 9), 99, dtype=torch.uint8, device="cuda:0")
    for f0, f1 in ((0, 6), (6, 7), (7, 20)):
        dssp_device(d[:, :, f0:f1], b, f, out=wide[f0:f1, 4:4 + n])
    assert torch.equal(wide[:, 4:4 + n], whole)
    assert bool((wide[:, :4] == 99).all()) and bool((wide[:, 4 + n:] == 99).all())
    fr = _t([19, 3, 3, 0, 11], np.int32)
    assert torch.equal(dssp_device(d, b, f, frames=fr), whole[fr.long()])
    assert dssp_device(d, b, f, frames=_t([], np.int32)).shape == (0, n)
    got = _device(g_traj["coords"], bb, fl, frames=[19, 3, 3, 0, 11])
    _same(got, do.dssp(g_traj["coords"], bb, fl, frames=[19, 3, 3, 0, 11]))


@pytest.mark.parametrize("simplified", [True, False])
@pytest.mark.parametrize("integer", [True, False])
def test_metric_project(g_traj, simplified, integer):
    from moleculekit_b200.dssp import FULL_INT, LETTERS, SIMPLE_INT, SIMPLE_LETTERS
    from moleculekit_b200.projections.metricsecondarystructure import MetricSecondaryStructure
    from moleculekit_b200.sharding import _frame_view, project_sharded

    prot = g_traj["sel_masks"][5].copy()
    mol, bb, fl = _table(g_traj, prot)
    mol.name = mol.name.copy()
    mol.name[bb[30, 3]] = "OXT"  # residue 30 loses its O: an NA column, and the sequence closes over it
    m = MetricSecondaryStructure(sel="protein", simplified=simplified, integer=integer)
    got = m.project(mol)
    bb2, fl2, pos, _ = m._getMolProp(mol, "dssp")
    assert bb2.shape[0] == 276 and pos[30] == -1 and got.shape == (20, 277)
    codes = do.dssp(mol.coords, bb2, fl2)[0]
    table = (SIMPLE_INT if simplified else FULL_INT) if integer else (SIMPLE_LETTERS if simplified else LETTERS)
    want = np.full((20, 277), -1 if integer else "NA", np.int64 if integer else "<U2")
    want[:, pos >= 0] = table[codes]
    assert got.dtype == want.dtype and np.array_equal(got, want)
    parts = [m.project(_frame_view(mol, a, b)) for a, b in ((0, 7), (7, 8), (8, 20))]
    assert np.array_equal(np.concatenate(parts), got)
    assert np.array_equal(project_sharded(m, mol), got)
    assert np.array_equal(mol.coords, g_traj["coords"])
