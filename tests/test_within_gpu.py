"""GPU parity of K10 (`within` / `exwithin` selections, SURVEY 8f row 3): identical masks to the reference's goldens and
to the oracle, including pairs a few ulps either side of the cutoff."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_reference_goldens(g_within):
    from moleculekit_b200.atomselect_utils import within
    from moleculekit_b200.molecule_lite import MolLite

    n_stored = 0
    for pid, op, cutoff, src, origin, key in g_within["cases"].tolist():
        mol = MolLite(g_within[f"{pid}_coords"])
        mask = within(mol, float(cutoff), g_within[key + "_source"], exclude_source=(op == "exwithin"))
        assert mask.dtype == bool and np.array_equal(mask, g_within[key + "_expected"]), (pid, op, cutoff, src)
        n_stored += origin == "stored"
    assert n_stored == 8
    # an index array as the source, an empty source
    mol = MolLite(g_within["3ptb_coords"])
    src = np.where(g_within["3ptb_2_source"])[0]
    assert np.array_equal(within(mol, 8.3, src), g_within["3ptb_2_expected"])
    assert not within(mol, 5.0, np.zeros(mol.numAtoms, bool)).any()


def test_drop_in_signature_vs_oracle(oracle):
    """within_distance(coords, cutoff, sel1, sel2, min, max, results) in place: threshold ties, query subsets, pre-set
    results, huge / tiny / negative cutoffs, NaN coordinates, a sparse system spanning many cells."""
    from moleculekit_b200.atomselect_utils import within_distance

    rng = np.random.default_rng(31)
    for t in range(14):
        N = int(rng.integers(2, 3000))
        span = [8.0, 60.0, 2000.0][t % 3]
        coords = (rng.normal(0, span, size=(N, 3))).astype(np.float32)
        cutoff = float(np.float32(rng.uniform(1, 9)))
        if t % 4 == 0:
            dirs = rng.normal(size=(N - 1, 3))
            dirs /= np.linalg.norm(dirs, axis=1)[:, None]
            coords[1:] = (coords[0] + dirs * (cutoff * (1 + rng.normal(0, 2e-7, size=(N - 1, 1))))).astype(np.float32)
            sel2 = np.array([0], np.uint32)
        else:
            sel2 = np.sort(rng.choice(N, int(rng.integers(1, min(N, 400) + 1)), replace=False)).astype(np.uint32)
        if t == 5:
            cutoff = 1e30
        if t == 6:
            cutoff = 1e-20
            coords[7] = coords[sel2[0]]  # identical coordinates: d2 = 0 < tiny^2 is false in float32 (underflow to 0)
        if t == 7:
            cutoff = -cutoff              # the reference squares it
        if t == 8:
            coords[3, 1] = np.nan
            coords[sel2[-1], 0] = np.nan
        sel1 = np.sort(rng.choice(N, int(rng.integers(1, N + 1)), replace=False)).astype(np.uint32)
        want, got = np.zeros(len(sel1), bool), np.zeros(len(sel1), bool)
        want[-1] = got[-1] = True
        with np.errstate(all="ignore"):
            mn, mx = coords[sel2].min(axis=0), coords[sel2].max(axis=0)
            oracle.within_distance(coords, cutoff, sel1, sel2, mn, mx, want)
        within_distance(coords, cutoff, sel1, sel2, mn, mx, got)
        assert np.array_equal(got, want), (t, int(got.sum()), int(want.sum()))
    c = np.zeros((4, 3), np.float32)
    with pytest.raises(ValueError, match="Buffer dtype mismatch"):
        within_distance(c.astype(np.float64), 1.0, np.arange(4, dtype=np.uint32), np.arange(2, dtype=np.uint32), c[0], c[0],
                        np.zeros(4, bool))
    with pytest.raises(IndexError):
        within_distance(c, 1.0, np.arange(4, dtype=np.uint32), np.array([9], np.uint32), c[0], c[0], np.zeros(4, bool))


def test_device_api_large_system(oracle):
    """100k atoms, 5k source atoms, 5 A: the device entry on resident tensors (query = all atoms) vs the oracle."""
    import torch
    from moleculekit_b200.atomselect_utils import within_distance_device

    rng = np.random.default_rng(41)
    N, n2 = 100_000, 5_000
    coords = rng.uniform(0, 100, size=(N, 3)).astype(np.float32)
    sel2 = np.sort(rng.choice(N, n2, replace=False)).astype(np.uint32)
    dev = torch.device("cuda:0")
    got = within_distance_device(torch.from_numpy(coords).to(dev), 5.0, torch.from_numpy(sel2.view(np.int32)).to(dev))
    want = np.zeros(N, bool)
    oracle.within_distance(coords, 5.0, np.arange(N, dtype=np.uint32), sel2, coords[sel2].min(0), coords[sel2].max(0), want)
    assert got.dtype == torch.bool and np.array_equal(got.cpu().numpy(), want) and 0.05 < want.mean() < 0.95


def test_box_edge_straddles_stay_within(oracle):
    """K10 shares K7's cell grid but its reference tests every pair: pairs pairdist apart that the bond reference's float32
    boxes put two boxes apart (oracle/bond_grid.py) must still be found, with the cutoff just above their separation
    (`within` compares d2 < cutoff * cutoff)."""
    from moleculekit_b200.atomselect_utils import within_distance

    from oracle import bond_grid as bg

    n_miss = 0
    for s in bg.straddle_systems(bg.STRADDLE_MINS + bg.FAR_MINS):
        c, p = s["coords"], s["pairs"]
        miss = bg.classify_pairs(s)[2]
        d2 = bg.d2_f32(c[p[:, 0]], c[p[:, 1]])
        cutoff = np.float32(np.sqrt(float(d2[miss].max() if miss.any() else d2.max())))
        while not cutoff * cutoff > d2[miss].max(initial=0):
            cutoff = np.nextafter(cutoff, np.float32(np.inf))
        sel1, sel2 = p[:, 0].astype(np.uint32), p[:, 1].astype(np.uint32)
        want, got = np.zeros(len(sel1), bool), np.zeros(len(sel1), bool)
        mn, mx = c[sel2].min(axis=0), c[sel2].max(axis=0)
        oracle.within_distance(c, float(cutoff), sel1, sel2, mn, mx, want)
        within_distance(c, float(cutoff), sel1, sel2, mn, mx, got)
        assert want[miss].all() and np.array_equal(got, want), float(s["xyzmin"])
        n_miss += miss.sum()
    assert n_miss >= 100
