"""The host prologues of the drop-in projections against the reference's own outputs, CPU only.

tests/golden/traj20.npz holds the reference's test system (tests/test_projections/trajectory: 4507 atoms, every 10th
frame) with the reference's selection masks and the float32 outputs of the reference's own ``MetricDistance`` /
``MetricSelfDistance.project`` and ``calculate_contacts`` on it (tests/golden/make_golden.py).  Here the GPU kernel behind
our wrappers is replaced by the C oracle (oracle/mkb_oracle.c, pinned bit for bit to the reference's compiled kernels
by tests/test_oracle_golden.py), so what is compared is what the host prologue hands to the kernel -- selections, chain ids,
self-distance / periodic flags, groups, masses, reductions, the truncate / threshold post-ops -- and the outputs must be
the reference's bit for bit.
"""
import numpy as np
import pytest


def _bits(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000
    return b


@pytest.fixture
def refmol(g_traj, oracle, monkeypatch):
    """A MolLite of the reference's test system whose distance kernels are the C oracle."""
    from moleculekit_b200 import distance_utils as du
    from moleculekit_b200.molecule_lite import MolLite

    def post(results, metric, truncate, threshold):  # projections/util.py:74-84,212-223 of the reference
        if truncate is not None:
            results[results > truncate] = truncate
        return results <= threshold if metric == "contacts" else results

    def dist_trajectory(coords, box, sel1, sel2, chains, selfdist, pbc, results, device=None, metric="distances",
                        truncate=None, threshold=8.0, exact=True):
        oracle.dist_trajectory(coords, box, sel1, sel2, chains, selfdist, pbc, results)
        return post(results, metric, truncate, threshold)

    def dist_trajectory_reduction(coords, box, groups1, groups2, ch1, ch2, selfdist, pbc, masses, r1, r2, results,
                                  device=None, metric="distances", truncate=None, threshold=8.0):
        oracle.dist_trajectory_reduction(coords, box, groups1, groups2, ch1, ch2, selfdist, pbc, masses, r1, r2, results)
        return post(results, metric, truncate, threshold)

    def contacts_trajectory_arrays(coords, box, sel1, sel2, chains, selfdist, pbc, threshold, device=None):
        per_frame = oracle.contacts_trajectory(coords, box, sel1, sel2, chains, selfdist, pbc, threshold)
        off = np.concatenate([[0], np.cumsum([len(x) // 2 for x in per_frame])]).astype(np.int64)
        pairs = np.array([v for x in per_frame for v in x], dtype=np.uint32).reshape(-1, 2)
        return off, pairs

    monkeypatch.setattr(du, "dist_trajectory", dist_trajectory)
    monkeypatch.setattr(du, "dist_trajectory_reduction", dist_trajectory_reduction)
    monkeypatch.setattr(du, "contacts_trajectory_arrays", contacts_trajectory_arrays)
    g = g_traj
    return MolLite(g["coords"], g["box"], element=g["element"], name=g["name"], resname=g["resname"], resid=g["resid"],
                   chain=g["chain"], segid=g["segid"],
                   named_selections={s: m for s, m in zip(g["sel_strings"].tolist(), g["sel_masks"])})


@pytest.mark.parametrize("periodic", [None, "chains", "selections"])
def test_metricdistance_prologue_with_reference_molecule(refmol, g_traj, periodic):
    """MetricDistance / calculate_contacts with string selections: selection indices, chain ids and the selfdist / pbc
    flags reach the kernel as the reference's do (metricdistance.py:132-179, util.py:12-85, distance.py)."""
    from moleculekit_b200.distance import calculate_contacts
    from moleculekit_b200.projections.metricdistance import MetricDistance

    g = g_traj
    masks = dict(zip(g["sel_strings"].tolist(), g["sel_masks"]))
    ca, lig, noh = masks["protein and name CA"], masks["resname MOL and noh"], masks["protein and noh"]
    if periodic == "selections":
        d = MetricDistance("protein and name CA", "resname MOL and noh", metric="distances", periodic=periodic).project(refmol)
        assert d.dtype == np.float32 and np.array_equal(_bits(d), _bits(g["ref_distances"]))
        c = MetricDistance("protein and name CA", "resname MOL and noh", metric="contacts", threshold=8,
                           periodic=periodic).project(refmol)
        assert c.dtype == bool and np.array_equal(c, g["ref_distances"] <= np.float32(8))
        cnt, pairs, got = g["ct_ca_lig_sel8_cnt"], g["ct_ca_lig_sel8_pairs"], calculate_contacts(refmol, ca, lig, periodic, 8)
    elif periodic == "chains":
        d = MetricDistance("protein and resid 1 to 20 and noh", "resname MOL and noh", periodic=periodic).project(refmol)
        assert np.array_equal(_bits(d), _bits(g["ref_chains_distances"]))
        cnt, pairs, got = g["ct_noh_lig_chains5_cnt"], g["ct_noh_lig_chains5_pairs"], calculate_contacts(refmol, noh, lig, periodic, 5)
    else:
        cnt, pairs, got = g["ct_ca_ca_none6_cnt"], g["ct_ca_ca_none6_pairs"], calculate_contacts(refmol, ca, ca, periodic, 6)
    assert [len(x) for x in got] == cnt.tolist()
    assert np.array_equal(np.concatenate(got).astype(np.uint32), pairs)


def test_selfdistance_and_mapping_with_reference_molecule(refmol, g_traj):
    """MetricSelfDistance + groupsel="residue" (metricdistance.py:244-364): the residue groups and the self-distance
    column order give the reference's output, and the mapping has one row per column."""
    from moleculekit_b200.projections.metricdistance import MetricDistance, MetricSelfDistance

    sel = "protein and resid 1 to 50 and noh"
    auto = MetricSelfDistance(sel, groupsel="residue").project(refmol)
    assert auto.shape == (20, 1225) and np.array_equal(_bits(auto), _bits(g_traj["ref_selfmindistance"]))
    manual = MetricDistance(sel, sel, periodic=None, groupsel1="residue", groupsel2="residue").project(refmol)
    assert np.array_equal(_bits(manual), _bits(auto))
    mp = MetricSelfDistance(sel, groupsel="residue").getMapping(refmol)
    assert len(mp) == auto.shape[1]
    resid = np.asarray(g_traj["resid"])
    a, b = (np.atleast_1d(x) for x in mp["atomIndexes"].iloc[0])  # first column: the selection's first two residues
    assert len(set(resid[a])) == 1 and len(set(resid[b])) == 1 and resid[a][0] < resid[b][0]


def test_reduction_prologue_with_reference_molecule(refmol, g_traj):
    """Residue groups against a ligand (get_reduced_distances, util.py:88-223): groups, group chain ids, masses and the
    closest / com reductions give the reference's outputs."""
    from moleculekit_b200.projections.metricdistance import MetricDistance

    g = g_traj
    kw = dict(groupsel1="residue", groupsel2="all")
    d = MetricDistance("protein and noh", "resname MOL and noh", periodic="selections", **kw).project(refmol)
    assert d.shape == (20, 277) and np.array_equal(_bits(d), _bits(g["ref_mindistances"]))
    c = MetricDistance("protein and noh", "resname MOL and noh", periodic="selections", metric="contacts", threshold=6,
                       **kw).project(refmol)
    assert np.array_equal(c, g["ref_mindistances"] <= np.float32(6))
    b = "protein and resid 1 to 50 and noh"
    cc = MetricDistance(b, "resname MOL and noh", "selections", groupreduce1="com", groupreduce2="com", **kw).project(refmol)
    assert np.array_equal(_bits(cc), _bits(g["ref_com_com"]))
    cl = MetricDistance(b, "resname MOL and noh", "selections", groupreduce1="com", groupreduce2="closest", **kw).project(refmol)
    assert np.array_equal(_bits(cl), _bits(g["ref_com_closest"]))
