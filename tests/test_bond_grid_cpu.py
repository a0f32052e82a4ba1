"""The reference's bond rule, pinned on the CPU (no GPU): an independent numpy restatement (oracle/bond_grid.py) -- the
float32 `_is_close` predicate AND reference boxes floor(fl32(fl32(x - xyzmin) / fl32(pairdist))) at most one apart on every
axis -- equals the C oracle's grid traversal as a set.  The predicate alone does not: atoms pairdist apart can be binned
two boxes apart, and the reference never compares them."""
import numpy as np
import pytest

from oracle import bond_grid as bg

f32 = np.float32


def _check(oracle, c, grid_cutoff, is_h, radii, **kw):
    rule, pred = bg.reference_pairs(c, grid_cutoff, is_h, radii, **kw)
    got = oracle.bond_grid_search(c, grid_cutoff, is_h, radii, **kw)
    assert len(np.unique(bg.canonical(got), axis=0)) == len(got), "the oracle repeats a pair"
    assert np.array_equal(bg.canonical(got), bg.canonical(rule))
    return rule, pred


def test_named_case(oracle):
    """x = 3.5 and 5.9 (xyzmin -3.7): d2 == cut * cut, but the reference boxes them as 2 and 4."""
    c = bg.NAMED_CASE
    r, h = np.full(4, 2.0, f32), np.zeros(4, np.uint32)
    assert bg.ref_boxes(c, bg.PD_FE)[1:3, 0].tolist() == [2, 4]
    assert bg.d2_f32(c[1], c[2]) == bg.cut_f32(2.0, 2.0) ** 2
    rule, pred = _check(oracle, c, bg.PD_FE, h, r)
    assert rule.tolist() == [] and pred.tolist() == [[1, 2]]


def test_straddles(oracle):
    """Pairs pairdist +- a few ulps apart at the reference's box edges 2^k (k = 1..17), for xyzmin near and far from the
    origin: same box, adjacent boxes and two boxes apart, bonded or not."""
    n_miss, n_diff = 0, np.zeros(3, int)
    for s in bg.straddle_systems(bg.STRADDLE_MINS + bg.FAR_MINS):
        rule, pred = _check(oracle, s["coords"], s["pairdist"], s["is_h"], s["radii"])
        diff, close, miss = bg.classify_pairs(s)
        assert len(pred) - len(rule) == miss.sum()  # the anchor and the slots add no straddle of their own
        n_miss += miss.sum()
        n_diff += np.bincount(np.minimum(diff, 2), minlength=3)
    assert n_miss >= 100, n_miss
    assert (n_diff > 100).all(), n_diff


@pytest.mark.parametrize("n, span, max_boxes", [(400, 12.0, 4e6), (2000, 40.0, 4e6), (600, 900.0, 2e4), (64, 3.0, 4e6)])
def test_random_clouds(oracle, n, span, max_boxes):
    """Random clouds with H atoms and coincident atoms; (600, 900 A, 2e4) goes through the max_boxes enlargement."""
    rng = np.random.default_rng(n)
    c = (rng.random((n, 3)) * span - span / 3).astype(f32)
    c[5] = c[4]
    c[7] = c[6] + f32(0.02)
    radii = rng.choice([1.0, 1.5, 1.7, 1.9, 2.0], n).astype(f32)
    ish = (radii == 1.0).astype(np.uint32)
    gc = np.max(radii) * 1.2
    pd = bg.pairdist_after_enlargement(c, gc, max_boxes)
    assert (pd > f32(gc)) == (max_boxes < 1e5)
    rule, pred = _check(oracle, c, gc, ish, radii, max_boxes=max_boxes)
    assert len(rule) > 0


def test_random_pairs_near_an_edge(oracle):
    """1500 pairs pairdist (1 +- 2e-7) apart, within 1e-3 rad of the x axis, across the edge of box 4 (xyzmin -3.7): random
    pairs that do produce straddles the predicate alone would report."""
    rng = np.random.default_rng(5)
    pd = bg.PD_FE
    u = np.concatenate([np.ones((1500, 1)), rng.normal(0, 1e-3, size=(1500, 2))], 1)
    u /= np.linalg.norm(u, axis=1)[:, None]
    mid = np.array([-3.7 + 3.5 * float(pd), 0.0, 0.0]) + rng.normal(0, 1e-6, size=(1500, 3))
    sep = float(pd) * (1 + rng.uniform(-2e-7, 2e-7, size=(1500, 1)))
    a, b = mid - u * sep / 2, mid + u * sep / 2
    # pairs spread along y, z so that different pairs stay more than pairdist apart
    spot = np.stack([np.zeros(1500), 3.0 * (np.arange(1500) % 40), 3.0 * (np.arange(1500) // 40)], 1)
    c = np.concatenate([a + spot, b + spot, [[-3.7, -3.7, -3.7]]]).astype(f32)
    r, h = np.full(len(c), 2.0, f32), np.zeros(len(c), np.uint32)
    rule, pred = _check(oracle, c, pd, h, r)
    assert len(pred) > len(rule)
