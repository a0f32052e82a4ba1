"""numpy restatement of the reference's bond rule (bondguesser.py:259-392 + bondguesser_utils.pyx:30-163) and generators of
the geometries where a grid-based bond search can disagree with it: pairs straddling the reference's box edges, distances
at the `_is_close` thresholds, and hash collisions of the K7 cell grid (csrc/bonds.cu).

TEST INFRASTRUCTURE ONLY.  The reference reports a pair when BOTH hold:
  * `_is_close`: not H-H, and with d2 = fl(fl(fl(dx dx) + fl(dy dy)) + fl(dz dz)) (float32, each operation rounded),
    0.001 <= d2 (double literal), d2 <= fl(pairdist pairdist) and d2 <= fl(cut cut), cut = fl32(0.6 (double) fl(ri + rj));
  * its box grid compares them: boxes floor(fl(fl(x - xyzmin) / pairdist)) (float32, xyzmin the per-axis minimum over
    all atoms) differ by at most 1 on every axis -- the 14-entry half-shell table visits nothing further.
Two such rounded quotients can put atoms that are pairdist apart two boxes apart; the reference never compares those.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
f64 = np.float64


def pairdist_after_enlargement(coords, grid_cutoff, max_boxes=4e6, cutoff_incr=1.26):
    """bondguesser.py: widen the box edge by cutoff_incr until the float32 box count fits max_boxes; float32 edge."""
    c = np.asarray(coords, f32)
    rng = c.max(axis=0) - c.min(axis=0)
    pd = float(grid_cutoff)
    while np.prod([int(v) + 1 for v in np.floor(rng / f32(pd))]) > max_boxes:
        pd *= cutoff_incr
    return f32(pd)


def d2_f32(a, b):
    """((dx dx) + dy dy) + dz dz in float32, every operation rounded; a, b (..., 3)."""
    d = np.asarray(a, f32) - np.asarray(b, f32)
    s = d[..., 0] * d[..., 0]
    s = s + d[..., 1] * d[..., 1]
    return s + d[..., 2] * d[..., 2]


def cut_f32(ri, rj):
    return (0.6 * (np.asarray(ri, f32) + np.asarray(rj, f32)).astype(f64)).astype(f32)


def is_close(c, radii, is_h, pd, i, j):
    """bondguesser_utils.pyx `_is_close` for the index arrays i, j."""
    pd = f32(pd)
    d2 = d2_f32(c[i], c[j])
    cut = cut_f32(radii[i], radii[j])
    return ~((is_h[i] != 0) & (is_h[j] != 0)) & ~(d2 > pd * pd) & ~(d2.astype(f64) < 0.001) & ~(d2 > cut * cut)


def ref_boxes(c, pd):
    """The reference's float32 box index of every atom along every axis (never clamped: rounding is monotone)."""
    c = np.asarray(c, f32)
    return np.floor((c - c.min(axis=0)) / f32(pd)).astype(np.int64)


def reference_pairs(coords, grid_cutoff, is_h, radii, max_boxes=4e6, cutoff_incr=1.26):
    """(rule, predicate): the reference's bonds as a canonical (n, 2) uint32 array, and every pair that passes `_is_close`
    whatever its boxes.  O(n^2) memory: for a few thousand atoms."""
    c = np.asarray(coords, f32)
    radii, is_h = np.asarray(radii, f32), np.asarray(is_h)
    pd = pairdist_after_enlargement(c, grid_cutoff, max_boxes, cutoff_incr)
    i, j = np.triu_indices(len(c), 1)
    close = is_close(c, radii, is_h, pd, i, j)
    i, j = i[close], j[close]
    box = ref_boxes(c, pd)
    adj = (np.abs(box[i] - box[j]) <= 1).all(axis=1)
    pred = np.stack([i, j], 1).astype(np.uint32)
    return pred[adj], pred


def canonical(b):
    b = np.sort(np.asarray(b, dtype=np.uint32).reshape(-1, 2), axis=1)
    return np.unique(b, axis=0)


def ulps(v, k):
    """v moved by k float32 ulps (k an int array), for v away from zero."""
    v = np.asarray(v, f32)
    return (v.view(np.int32) + np.sign(v).astype(np.int32) * np.asarray(k, np.int32)).view(f32)


# ------------------------------------------------------------------------------------------------------------------
# box-edge straddles
# ------------------------------------------------------------------------------------------------------------------
PD_FE = f32(2.0) * 1.2  # guess_bonds' box edge when the largest radius is 2.0 (Fe, or an element the table lacks)
# xyzmin values: round ones near and far from the origin, and seeded ones of every magnitude (whether fl(x - xyzmin)
# rounds, and which way, decides how many straddles an edge has)
_RNG = np.random.default_rng(20261017)
STRADDLE_MINS = (0.0, -3.7, -1234.567, -5e4, -1e5, -1e6) + tuple(
    float(f32(s * 10 ** e)) for s, e in zip(_RNG.choice([-1.0, 1.0], 12), _RNG.uniform(-1, 6, 12)))
FAR_MINS = (1e4, 1e5, 1e6)
# (x box difference, bonded) wanted in the 16 slots of one edge; a bonded pair two boxes apart first, as many as exist
WANT = ((2, True),) * 11 + ((2, False), (1, True), (1, False), (0, None), (1, None))


def straddle_system(m, pd=PD_FE, ks=range(1, 18), window=24):
    """One system with xyzmin = (m, m, m) (an anchor atom there) and, for every k in ks, 16 pairs of radius-2.0 atoms
    along x whose separation is pd within +-window float32 ulps of the coordinates, placed where the farther atom's
    reference box index along x is 2^k (the quotient crosses a binade there, so its ulp doubles).  The pairs sit on a
    4 x 4 grid of (y, z) slots 3 A apart; slot s has dy = s % 4 and dz = (s // 4) % 4 ulps.  Slots take the
    (x box difference, bonded) classes of WANT while the edge has candidates of that class left, else a pair in adjacent
    boxes, bonded if possible.  Returns coords, radii, is_h, pairdist and the (p, 2) atom indices of the generated pairs."""
    m, pd = f32(m), f32(pd)
    rows, pairs = [np.array([m, m, m], f32)], []
    off = np.arange(-window, window + 1)
    q = lambda x: np.floor((x - m) / pd).astype(np.int64)
    for k in ks:
        x2 = ulps(f32(float(m) + 2 ** k * float(pd)), off)                       # around the edge of box 2^k
        x1 = ulps((x2.astype(f64) - float(pd)).astype(f32)[:, None], off[None, :])  # around the edge of box 2^k - 1
        x2 = np.broadcast_to(x2[:, None], x1.shape).ravel()
        x1 = x1.ravel()
        diff = q(x2) - q(x1)
        used = set()
        for s, (want_diff, want_bond) in enumerate(WANT):
            y = f32(float(m) + 3.0 * (s % 4))
            z = f32(float(m) + 3.0 * (s // 4))
            y2, z2 = ulps(y, s % 4), ulps(z, (s // 4) % 4)  # no move at 0 (m = 0): dy = dz = 0 there
            a = np.stack([x1, np.full_like(x1, y), np.full_like(x1, z)], 1)
            b = np.stack([x2, np.full_like(x2, y2), np.full_like(x2, z2)], 1)
            d2 = d2_f32(a, b)
            bond = ~(d2 > pd * pd) & ~(d2 > cut_f32(2.0, 2.0) ** 2)
            cand = []
            for wd, wb in ((want_diff, want_bond), (1, True), (1, None)):
                ok = (diff == wd) & ((bond == wb) if wb is not None else True)
                cand = [c for c in np.flatnonzero(ok).tolist() if c not in used]
                if cand:
                    break
            pick = cand[(s * 7919 + k * 104729) % len(cand)]  # spread the choices over the candidates
            used.add(pick)
            pairs.append((len(rows), len(rows) + 1))
            rows += [a[pick], b[pick]]
    c = np.stack(rows).astype(f32)
    n = len(c)
    return dict(coords=c, radii=np.full(n, 2.0, f32), is_h=np.zeros(n, np.uint32), pairdist=pd, xyzmin=m,
                pairs=np.array(pairs, np.int64))


def straddle_systems(mins=STRADDLE_MINS, pd=PD_FE):
    """Every edge 2^k (k = 1..17) for each xyzmin in `mins`, then each edge alone with xyzmin = -2^k pd (1 +- 1/16): the
    edge's atoms then sit near x = 0, where the float32 coordinates are far finer than fl(x - xyzmin), so the
    subtraction's rounding takes every value and bonded pairs two boxes apart are plentiful."""
    for m in mins:
        yield straddle_system(m, pd)
    for k in range(1, 18):
        for d in (1 / 16, -1 / 16):
            yield straddle_system(-(2 ** k) * float(pd) * (1 + d), pd, ks=(k,))


def classify_pairs(sys_, pairs=None):
    """(x box difference, passes _is_close, two boxes apart on some axis and passes) for the given pairs."""
    c, pd = sys_["coords"], sys_["pairdist"]
    p = sys_["pairs"] if pairs is None else pairs
    box = ref_boxes(c, pd)
    close = is_close(c, sys_["radii"], sys_["is_h"], pd, p[:, 0], p[:, 1])
    far = (np.abs(box[p[:, 0]] - box[p[:, 1]]) > 1).any(axis=1)
    return np.abs(box[p[:, 0], 0] - box[p[:, 1], 0]), close, close & far


NAMED_CASE = np.array([[-3.7, 0, 0], [3.5, 0, 0], [5.9, 0, 0], [20, 20, 20]], f32)  # radii 2.0: (1, 2) passes
# _is_close with d2 == cut * cut, but the reference boxes x = 3.5 and x = 5.9 as 2 and 4


# ------------------------------------------------------------------------------------------------------------------
# thresholds
# ------------------------------------------------------------------------------------------------------------------
def threshold_offsets(a, T, n_below=4, n_above=3):
    """Partner positions b near a (float32 (P, 3), y and z free) with d2(a, b) the n_below largest values <= T and the
    n_above smallest values > T that the search reaches (T, T - 1..3 ulps and T + 1..3 ulps wherever the float32
    coordinates are fine enough).  Search: x2 within 4 ulps of a_x + sqrt(T), then y2 = a_y + sqrt(t - fl(dx dx)) and its
    neighbours for every target t.  Returns (P, n_below + n_above, 3) positions and their d2."""
    a = np.asarray(a, f32)
    T = np.asarray(T, f32)
    P = len(a)
    x2 = ulps((a[:, 0].astype(f64) + np.sqrt(T.astype(f64))).astype(f32)[:, None], np.arange(-4, 5)[None, :])  # (P, 9)
    dx = x2 - a[:, :1]
    s = (dx * dx).astype(f64)
    tk = np.arange(-n_below + 1, n_above + 1)
    targets = (T.view(np.int32)[:, None] + tk[None, :]).view(f32).astype(f64)  # (P, 7)
    r = np.maximum(targets[:, None, :] - s[:, :, None], 0.0)                    # (P, 9, 7)
    y2 = (a[:, 1].astype(f64)[:, None, None] + np.sqrt(r)).astype(f32)
    y2 = np.stack([np.nextafter(y2, f32(-np.inf)), y2, np.nextafter(y2, f32(np.inf))], -1)  # (P, 9, 7, 3)
    X2 = np.broadcast_to(x2[:, :, None, None], y2.shape)
    cand = np.stack([X2, y2, np.broadcast_to(a[:, 2, None, None, None], y2.shape)], -1).reshape(P, -1, 3)
    d2 = d2_f32(a[:, None, :], cand)
    out = np.empty((P, n_below + n_above, 3), f32)
    out_d2 = np.empty((P, n_below + n_above), f32)
    for p in range(P):
        vals, first = np.unique(d2[p], return_index=True)
        lo, hi = first[vals <= T[p]][-n_below:], first[vals > T[p]][:n_above]
        sel = np.concatenate([lo, hi])
        assert len(sel) == n_below + n_above, "threshold search found too few distinct distances"
        out[p], out_d2[p] = cand[p, sel], d2[p, sel]
    return out, out_d2


def threshold_system(radius_pairs, is_h_pairs, offset=0.0, T=None, spacing=8.0):
    """Pairs of atoms (radius ri with flag hi, radius rj with flag hj) at distances around fl(cut cut) (or around T when
    given: one float32 d2 value, e.g. fl32(0.001)), on a square (x, z) lattice `spacing` apart with the first atom at
    y = 0 -- where every float32 d2 is reachable -- shifted by `offset` on every axis.  Returns the system and the d2
    of every pair."""
    rp = np.asarray(radius_pairs, f32).reshape(-1, 2)
    hp = np.asarray(is_h_pairs, np.uint32).reshape(-1, 2)
    Tp = (cut_f32(rp[:, 0], rp[:, 1]) ** 2) if T is None else np.full(len(rp), f32(T), f32)
    side = int(np.ceil(np.sqrt(len(rp) * 7)))
    k = np.arange(len(rp) * 7)
    first = (np.stack([(k % side) * spacing, np.zeros(len(k)), (k // side) * spacing], 1) + offset).astype(f32)
    T7 = np.repeat(Tp, 7)
    b, d2 = threshold_offsets(first, T7)  # 7 sites per radius pair; site t keeps the t-th distance found from it
    second, d2 = b[k, k % 7], d2[k, k % 7]
    c = np.stack([first, second], 1).reshape(-1, 3)
    radii = np.repeat(rp, 7, axis=0).reshape(-1)
    is_h = np.repeat(hp, 7, axis=0).reshape(-1)
    n = len(c)
    return dict(coords=c, radii=radii.astype(f32), is_h=is_h.astype(np.uint32),
                pairs=np.arange(n).reshape(-1, 2), T=T7), d2


# ------------------------------------------------------------------------------------------------------------------
# K7's cell hash (csrc/bonds.cu `bond_hash`, `cell_of`, `bond_build`)
# ------------------------------------------------------------------------------------------------------------------
def k7_buckets(n):
    nb = 1024
    while nb < 2 * n and nb < (1 << 22):
        nb <<= 1
    return nb


def k7_cell(x, pairdist):
    """floor((double)x * (1 / ((double)pairdist * 1.00001))), per coordinate."""
    inv_w = 1.0 / (float(f32(pairdist)) * 1.00001)
    return np.floor(np.asarray(x, f32).astype(f64) * inv_w).astype(np.int64)


def k7_hash(cx, cy, cz, hmask):
    """bond_hash with unsigned 64-bit wraparound."""
    u = lambda v: np.asarray(v, np.int64).astype(np.uint64)
    h = (u(cx) * np.uint64(73856093)) ^ (u(cy) * np.uint64(19349663)) ^ (u(cz) * np.uint64(83492791))
    return ((h ^ (h >> np.uint64(23))) & np.uint64(hmask)).astype(np.int64)


NEIGH = np.array([(k // 9 - 1, (k // 3) % 3 - 1, k % 3 - 1) for k in range(27)], np.int64)
