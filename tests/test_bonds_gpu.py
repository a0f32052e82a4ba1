"""GPU parity of K7 (bond perception, SURVEY row a13) against the reference's csv goldens and the oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _canonical(b):
    b = np.sort(np.asarray(b, dtype=np.uint32).reshape(-1, 2), axis=1)
    return np.unique(b, axis=0)


def test_reference_goldens(g_bonds):
    """tests/test_bondguesser.py:27-44 for all 15 structures: guess_bonds == csv (bit-exact as a set, canonical order)."""
    from moleculekit_b200.bondguesser import guess_bonds
    from moleculekit_b200.molecule_lite import MolLite

    g = g_bonds
    for pid in g["pdbids"].tolist():
        mol = MolLite(g[f"{pid}_coords"], element=g[f"{pid}_element"], name=g[f"{pid}_name"])
        bonds = guess_bonds(mol)
        assert bonds.dtype == np.uint32 and bonds.shape[1] == 2
        assert np.array_equal(bonds, g[f"{pid}_bonds"]), pid


def test_random_vs_oracle_and_box_enlargement(oracle):
    """Random clouds incl. a sparse unwrapped-like system that triggers the max_boxes enlargement loop, H-H pairs,
    coincident atoms (d2 < 0.001) -- compared with the oracle as canonical sets."""
    from moleculekit_b200.bondguesser import bond_grid_search

    rng = np.random.default_rng(8)
    for n, span, max_boxes in ((400, 12.0, 4e6), (3000, 40.0, 4e6), (500, 900.0, 2e4), (64, 3.0, 4e6)):
        c = (rng.random((n, 3)) * span - span / 3).astype(np.float32)
        c[5] = c[4]                                  # identical coordinates: never bonded
        c[7] = c[6] + np.float32(0.02)               # d2 = 0.0012 > 0.001: bonded if radii allow
        radii = rng.choice([1.0, 1.5, 1.7, 1.9, 2.0], n).astype(np.float32)
        ish = (radii == 1.0).astype(np.uint32)
        want = _canonical(oracle.bond_grid_search(c, np.max(radii) * 1.2, ish, radii, max_boxes=max_boxes))
        got = bond_grid_search(c, np.max(radii) * 1.2, ish, radii, max_boxes=max_boxes)
        assert np.array_equal(got, want), (n, span)
        assert not ((ish[got[:, 0]] == 1) & (ish[got[:, 1]] == 1)).any()


def test_edge_cases_and_errors():
    from moleculekit_b200.bondguesser import bond_grid_search, guess_bonds
    from moleculekit_b200.molecule_lite import MolLite

    assert guess_bonds(MolLite(np.zeros((0, 3, 1), np.float32))).shape == (0, 2)
    one = guess_bonds(MolLite(np.zeros((1, 3, 1), np.float32), element=["C"], name=["C1"]))
    assert one.shape == (0, 2) and one.dtype == np.uint32
    two = MolLite(np.array([[0, 0, 0], [1.5, 0, 0]], np.float32), element=["C", "C"], name=["C1", "C2"])
    assert guess_bonds(two).tolist() == [[0, 1]]
    two.frame = 3
    with pytest.raises(RuntimeError, match="out of range"):
        guess_bonds(two)
    c = np.zeros((3, 3), np.float32); c[1, 0] = np.nan
    with pytest.raises(ValueError, match="non-finite coordinates"):
        bond_grid_search(c, 2.0, np.zeros(3, np.uint32), np.ones(3, np.float32))
    with pytest.raises(ValueError, match="positive, finite grid_cutoff"):
        bond_grid_search(np.zeros((3, 3), np.float32), -1.0, np.zeros(3, np.uint32), np.ones(3, np.float32))


# ------------------------------------------------------------------------------------------------------------------
# the reference's rule at its edges (oracle/bond_grid.py): the float32 `_is_close` predicate AND reference boxes
# floor(fl32(fl32(x - xyzmin) / pairdist)) at most one apart.  Every comparison is an exact set equality with the oracle on
# uncanonicalised output: bond_grid_search returns its rows sorted, so equality with the oracle's unique canonical rows
# also proves that no row repeats.
# ------------------------------------------------------------------------------------------------------------------
from oracle import bond_grid as bg  # noqa: E402

F32 = np.float32


def _same_as_oracle(oracle, c, grid_cutoff, is_h, radii, **kw):
    from moleculekit_b200.bondguesser import bond_grid_search

    got = bond_grid_search(c, grid_cutoff, is_h, radii, **kw)
    want = _canonical(oracle.bond_grid_search(c, grid_cutoff, is_h, radii, **kw))
    assert got.dtype == np.uint32 and got.shape[1:] == (2,)
    assert np.array_equal(got, want), (len(got), len(want))
    return got


def test_named_box_edge_case(oracle):
    """x = -3.7, 3.5, 5.9 and a far atom, radii 2.0: (1, 2) passes _is_close with d2 == cut * cut, but the reference boxes
    3.5 and 5.9 as 2 and 4 and never compares them -- through bond_grid_search and through guess_bonds (Fe)."""
    from moleculekit_b200.bondguesser import guess_bonds
    from moleculekit_b200.molecule_lite import MolLite

    c = bg.NAMED_CASE
    got = _same_as_oracle(oracle, c, bg.PD_FE, np.zeros(4, np.uint32), np.full(4, 2.0, F32))
    assert got.shape == (0, 2)
    mol = MolLite(c, element=["Fe"] * 4, name=["FE"] * 4)
    bonds = guess_bonds(mol)
    assert bonds.dtype == np.uint32 and bonds.shape == (0, 2)
    # one ulp closer the pair is binned 2 and 3 and is a bond for both
    c2 = c.copy()
    c2[2, 0] = np.nextafter(c2[2, 0], F32(0))
    assert guess_bonds(MolLite(c2, element=["Fe"] * 4, name=["FE"] * 4)).tolist() == [[1, 2]]


def test_box_edge_straddles(oracle):
    """Pairs pairdist +- a few ulps apart along x (dy, dz of 0..3 ulps) at the reference's box edges 2^k, k = 1..17, for
    xyzmin from -1e6 to 1e6 (the far ones put the atoms 1e4..1e6 A from the origin): same box, adjacent boxes, two boxes
    apart.  At least 100 of the pairs pass _is_close two boxes apart, which the reference does not report."""
    n_miss, n_diff = 0, np.zeros(3, int)
    for s in bg.straddle_systems(bg.STRADDLE_MINS + bg.FAR_MINS):
        got = _same_as_oracle(oracle, s["coords"], s["pairdist"], s["is_h"], s["radii"])
        diff, close, miss = bg.classify_pairs(s)
        p = s["pairs"]
        found = {tuple(r) for r in got.tolist()}
        assert all((tuple(r) in found) == (c and not m) for r, c, m in zip(p.tolist(), close, miss)), float(s["xyzmin"])
        n_miss += miss.sum()
        n_diff += np.bincount(np.minimum(diff, 2), minlength=3)
    assert n_miss >= 100, n_miss
    assert (n_diff > 100).all(), n_diff


def _radius_pairs():
    from moleculekit_b200.bondguesser import vdw_radii

    r = sorted(set(vdw_radii.values()))
    rp = [(a, b) for i, a in enumerate(r) for b in r[i:]]
    hp = [(a == 1.0, b == 1.0) for a, b in rp]  # radius 1.0 is H in the table: H-H excluded, H-X kept
    return rp + [(1.0, 1.0)], hp + [(False, False)]  # ... and two non-H atoms of radius 1.0 at the same distances


@pytest.mark.parametrize("offset", [0.0, 1e4, 1e5, 1e6])
def test_thresholds(oracle, offset):
    """d2 at fl(cut * cut) and 1..3 ulps either side for every radius pair of vdw_radii (cut = fl32(0.6 (double)(ri + rj))
    rounds differently per pair), H-H and H-X pairs at the same distances, and d2 either side of the double literal 0.001
    -- at the origin, where every float32 d2 is reachable, and shifted by 1e4..1e6 A, where the nearest reachable d2
    either side stand in for them."""
    rp, hp = _radius_pairs()
    s, d2 = bg.threshold_system(rp, hp, offset=offset)
    T = s["T"]
    if offset == 0.0:
        steps = d2.view(np.int32).astype(np.int64) - T.view(np.int32)
        assert np.array_equal(np.sort(steps.reshape(-1, 7), axis=1), np.tile(np.arange(-3, 4), (len(rp), 1)))
    else:
        assert (d2 <= T).sum() >= 4 * len(rp) and (d2 > T).sum() >= 3 * len(rp)
    parts = [s]
    if offset <= 1e5:  # d2 near 0.001 needs coordinate steps finer than 0.03 A
        t, _ = bg.threshold_system([(1.7, 1.7), (1.0, 1.52), (1.0, 1.0)], [(0, 0), (1, 0), (1, 1)], offset=offset,
                                   T=F32(0.001))
        t["coords"][:, 2] += F32(s["coords"][:, 2].max() + 10.0)
        parts.append(t)
    c = np.concatenate([q["coords"] for q in parts])
    radii = np.concatenate([q["radii"] for q in parts])
    ish = np.concatenate([q["is_h"] for q in parts])
    got = _same_as_oracle(oracle, c, np.max(radii) * 1.2, ish, radii)
    pairs = np.arange(len(c)).reshape(-1, 2)
    found = {tuple(r) for r in got.tolist()}
    bonded = np.array([tuple(r) in found for r in pairs.tolist()])
    hh = (ish[pairs[:, 0]] == 1) & (ish[pairs[:, 1]] == 1)
    hx = (ish[pairs[:, 0]] + ish[pairs[:, 1]]) == 1
    assert not bonded[hh].any() and bonded[hx].any() and bonded[~hh & ~hx].any()
    if offset == 0.0:  # the non-H radius-1.0 pairs are bonded exactly where the predicate allows: d2 <= fl(1.2 * 1.2)
        one = (radii[pairs[:, 0]] == 1.0) & (radii[pairs[:, 1]] == 1.0) & ~hh
        assert bonded[one].sum() == 4 * int(one.sum() // 7)


def test_threshold_after_enlargement(oracle):
    """A 1000 A system (the reference widens its boxes 1.26x until at most 4e6 fit): pairs with d2 at the widened
    fl(pairdist^2) and 1..3 ulps either side are never bonds (pairdist > every cut now), pairs at fl(cut^2) still are."""
    corners = np.array([[0, 0, 0], [1000, 1000, 1000]], F32)
    pd = bg.pairdist_after_enlargement(corners, F32(2.0) * 1.2)
    assert pd > F32(2.0) * 1.2 * 2
    far, _ = bg.threshold_system([(2.0, 2.0)] * 4, [(0, 0)] * 4, offset=20.0, T=pd * pd, spacing=2 * float(pd))
    near, _ = bg.threshold_system([(2.0, 2.0), (1.0, 2.0)], [(0, 0), (1, 0)], offset=500.0)
    c = np.concatenate([far["coords"], near["coords"], corners])
    radii = np.concatenate([far["radii"], near["radii"], [2.0, 2.0]]).astype(F32)
    ish = np.concatenate([far["is_h"], near["is_h"], [0, 0]]).astype(np.uint32)
    assert bg.pairdist_after_enlargement(c, F32(2.0) * 1.2) == pd
    got = _same_as_oracle(oracle, c, F32(2.0) * 1.2, ish, radii)
    nf = len(far["coords"])
    assert (got >= nf).all() and len(got) >= 8  # nothing from the pairdist^2 pairs; the cut pairs at or below fl(cut^2)


@pytest.mark.parametrize("offset", [1e4, 1e5, 1e6])
def test_far_unwrapped_cloud(oracle, offset):
    """A sparse 2000 A cloud 1e4..1e6 A from the origin with bonded clusters (boxes widened by the enlargement loop), plus
    pairs pairdist +- a few ulps apart at the widened box edges: after enlargement pairdist > cut, so none is a bond."""
    rng = np.random.default_rng(int(offset))
    cloud = (offset + rng.uniform(0, 2000, size=(3000, 3))).astype(F32)
    cloud[1::3] = cloud[0::3] + rng.normal(0, 0.9, size=(1000, 3)).astype(F32)
    cloud[2::3] = cloud[0::3] + rng.normal(0, 0.9, size=(1000, 3)).astype(F32)
    cloud = np.concatenate([cloud, [[offset] * 3, [offset + 2000.0] * 3]]).astype(F32)
    radii = np.concatenate([rng.choice([1.0, 1.52, 1.7, 2.0], 3000), [2.0, 2.0]]).astype(F32)
    gc = F32(2.0) * 1.2
    pd = bg.pairdist_after_enlargement(cloud, gc)
    assert pd > gc * 4
    s = bg.straddle_system(offset, pd=pd, ks=range(1, 7))
    c = np.concatenate([s["coords"], cloud])
    assert bg.pairdist_after_enlargement(c, gc) == pd
    r = np.concatenate([s["radii"], radii])
    ish = np.concatenate([s["is_h"], (radii == 1.0).astype(np.uint32)])
    got = _same_as_oracle(oracle, c, gc, ish, r)
    ns = len(s["coords"])
    assert (got >= ns).all() and len(got) > 500


def test_hash_collisions(oracle):
    """K7 hashes cells into 1024 buckets (n <= 512).  (a) Atoms two of whose 27 neighbour cells share a bucket, with a
    bonded partner in each: the bucket is visited twice and the member filter must keep each pair once.  (b) A
    neighbour cell sharing its bucket with a cell outside the 27, whose atoms (bonded among themselves) are walked and
    must be skipped."""
    pd = bg.PD_FE
    w = float(pd) * 1.00001
    hmask = bg.k7_buckets(512) - 1
    assert hmask == 1023
    g = np.stack(np.meshgrid(*[np.arange(0, 60, 4)] * 3, indexing="ij"), -1).reshape(-1, 3)  # cells 4 apart
    nb = g[:, None, :] + bg.NEIGH[None, :, :]
    h = bg.k7_hash(nb[..., 0], nb[..., 1], nb[..., 2], hmask)  # (cells, 27)
    rows, cases_a, cases_b = [], 0, 0

    def put(cell, frac):
        x = ((np.asarray(cell, np.float64) + 0.5 + np.asarray(frac)) * w).astype(F32)
        assert (bg.k7_cell(x, pd) == cell).all()
        rows.append(x)

    for ci, hh in enumerate(h):
        same = [(a, b) for a in range(27) for b in range(a + 1, 27) if hh[a] == hh[b]]
        if same and cases_a < 6:
            a, b = same[0]
            put(g[ci], (0, 0, 0))
            for k in (a, b):
                o = bg.NEIGH[k]
                put(g[ci] + o, (0.3, 0, 0) if not o.any() else -0.45 * o)  # 0.55 w * o from the atom
            cases_a += 1
        elif not same and cases_b < 6 and ci % 7 == 0:
            # a cell far away (not a neighbour) with the bucket of neighbour k of this cell
            k = 13 + 1 + (ci % 13)
            tgt = hh[k]
            far = np.stack(np.meshgrid(*[np.arange(-80, -10)] * 3, indexing="ij"), -1).reshape(-1, 3)
            fh = bg.k7_hash(far[:, 0], far[:, 1], far[:, 2], hmask)
            f = far[np.flatnonzero(fh == tgt)[0]]
            o = bg.NEIGH[k]
            put(g[ci], (0, 0, 0))
            put(g[ci] + o, -0.45 * o)
            put(f, (0, 0, 0))
            put(f, (0.3, 0, 0))
            cases_b += 1
    assert cases_a == 6 and cases_b == 6
    c = np.stack(rows).astype(F32)
    assert len(c) <= 512 and bg.k7_buckets(len(c)) == 1024 and bg.pairdist_after_enlargement(c, pd) == pd
    r, ish = np.full(len(c), 2.0, F32), np.zeros(len(c), np.uint32)
    got = _same_as_oracle(oracle, c, pd, ish, r)
    assert len(got) >= 2 * cases_a + 2 * cases_b


def test_three_million_atom_water_lattice(oracle):
    """1 M waters (3 M atoms, > 2^21): K7's bucket count stops at 2^22, so buckets hold several occupied cells."""
    rng = np.random.default_rng(3)
    s = 100
    o = (np.stack(np.meshgrid(*[np.arange(s)] * 3, indexing="ij"), -1).reshape(-1, 3) * 3.1
         + rng.normal(0, 0.1, size=(s ** 3, 3)))
    u = rng.normal(size=(2, s ** 3, 3))
    u /= np.linalg.norm(u, axis=2)[..., None]
    c = np.stack([o, o + 0.9572 * u[0], o + 0.9572 * u[1]], 1).reshape(-1, 3).astype(F32)
    radii = np.tile(np.array([1.52, 1.0, 1.0], F32), s ** 3)
    ish = (radii == 1.0).astype(np.uint32)
    gc = np.max(radii) * 1.2
    n = len(c)
    assert n > 2 ** 21 and bg.k7_buckets(n) == 2 ** 22
    cells = np.unique(bg.k7_cell(c, gc), axis=0)
    per_bucket = np.bincount(bg.k7_hash(cells[:, 0], cells[:, 1], cells[:, 2], 2 ** 22 - 1))
    assert len(cells) > 2 ** 20 and (per_bucket >= 2).sum() > 10_000
    got = _same_as_oracle(oracle, c, gc, ish, radii, max_boxes=1e7)
    assert len(got) >= 2 * s ** 3
