"""The hydrogen-bond (K12) and ring (K13) detectors decide at their cut-offs through host-computed bounds on the float
cosine.  These CPU tests build the independent reference for those bounds (an exhaustive walk over every float of [-1, 1]
with the host libm), and check that every probe of tests/cutoff_probes.py lands where it is meant to: its designed cosine,
dot product or squared distance is what the kernels' float operations give, and the oracle's decision flips exactly at the
transition float.  tests/test_interaction_cutoffs_gpu.py runs the same probes through the kernels."""
import numpy as np
import pytest

import cutoff_probes as cp


@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    s = cp.run_scan(tmp_path_factory.mktemp("acosf_scan"))
    if s is None:
        pytest.skip("no host C compiler")
    return s


@pytest.fixture(scope="module")
def probe_sets(scan):
    return cp.angle_sets(scan) + cp.distance_sets()


def test_acosf_non_increasing(scan):
    """both kernels' host bounds assume libm's acosf never increases over [-1, 1]; checked on every float"""
    assert scan.mono_bad == 0, f"acosf increases at {cp.funkey(scan.mono_first)!r}"


def test_k12_bounds(scan):
    """c* from the exhaustive walk: acosf(c*) exceeds the threshold and acosf of the next float does not"""
    found = 0
    for angle in cp.K12_ANGLES:
        thr = float(cp.f32(float(cp.f32(angle)) / cp.ANGLE_SCALE))
        k = scan.cstar[angle]
        if k is None:
            assert not cp.acosf(-1.0) > thr and angle >= 180.0
            continue
        assert cp.acosf(cp.funkey(k)) > thr
        if k < cp.KMAX:
            assert not cp.acosf(cp.funkey(k + 1)) > thr
            found += 1
    assert found >= 8
    assert scan.cstar[120.0] is not None and scan.cstar[120.0] != scan.cstar[119.99999]


def test_k13_transition_sets(scan):
    """each transition float and its lower neighbour give different predicate values through ctypes acosf, the value at -1
    is the reported one, and random floats agree with the set the transitions describe"""
    rng = np.random.default_rng(2)
    xs = np.concatenate([rng.uniform(-1, 1, 300), [-1.0, 1.0, 0.0]]).astype(np.float32)
    n_tr = 0
    for (angle, pred), (v0, trs) in scan.sets.items():
        assert cp.k13_pred(angle, pred, -1.0) == v0
        for kt in trs:
            assert cp.k13_pred(angle, pred, cp.funkey(kt)) != cp.k13_pred(angle, pred, cp.funkey(kt - 1))
        n_tr += len(trs)
        for x in xs[:: 3 if pred else 1]:
            assert scan.member(angle, pred, cp.fkey(x)) == cp.k13_pred(angle, pred, x), (angle, pred, x)
    assert n_tr >= 60
    # the fold makes every non-trivial pi-pi predicate hold on two intervals: two transitions each
    assert len(scan.sets[(30.0, cp.LE)][1]) == 2 and len(scan.sets[(60.0, cp.PLANE)][1]) == 2


def _flip_at_edge(ps, hits):
    """inside every boundary group equal values decide alike, the decision changes exactly once along the values, and it
    changes next to the transition float"""
    for name, frames in ps.groups().items():
        by_value = {}
        for f in frames:
            by_value.setdefault(float(ps.value[f]) if ps.what[f] else f, set()).add(bool(hits[f]))
        assert all(len(v) == 1 for v in by_value.values()), (ps.name, name)
        if ps.what[frames[0]] is None:
            continue
        vals = sorted(by_value)
        seq = [by_value[v].pop() for v in vals]
        changes = [i for i in range(1, len(seq)) if seq[i] != seq[i - 1]]
        assert len(changes) == 1, (ps.name, name, seq)
        edge = {float(ps.value[f]) for f in frames if ps.edge[f]}
        assert len(edge) == 1, (ps.name, name)
        e = vals.index(edge.pop())
        assert changes[0] in (e, e + 1), (ps.name, name, seq, e)


def test_probes_land_on_their_targets(oracle, scan, probe_sets):
    """every probe's designed value is the kernels' float result; the oracle agrees with the reference predicate evaluated
    on it (and, for the angle probes, with the exhaustive sets), and flips exactly at each transition float"""
    total = 0
    for ps in probe_sets:
        cp.check_construction(ps)
        want = cp.reference_hits(ps)
        got = cp.hits_of(ps, cp.call(ps, oracle))
        assert np.array_equal(got, want), (ps.name, np.flatnonzero(got != want)[:10])
        if ps.what[0] in ("c", "dot"):
            assert np.array_equal(got, cp.scan_hits(scan, ps)), ps.name
        for name, frames in ps.groups().items():
            assert got[frames].any() and not got[frames].all(), (ps.name, name)
            assert any(ps.edge[f] for f in frames), (ps.name, name)
        _flip_at_edge(ps, got)
        total += len(ps)
    assert total > 2000


def test_short_rings_rejected():
    """a ring of fewer than 3 atoms has no normal of its own (the reference reads the next ring's atoms): the wrappers raise
    ValueError naming the ring, before any device work"""
    from moleculekit_b200 import interactions, ringpairs

    xyz = np.zeros((12, 3, 1), np.float32)
    box = np.zeros((3, 1), np.float32)
    ra = np.arange(12, dtype=np.uint32)
    good, short = np.array([0, 6, 12], np.uint32), np.array([0, 6, 8, 12], np.uint32)
    with pytest.raises(ValueError, match="ring 1 of rings1_start_indexes has 2 atoms"):
        ringpairs.pipi_calculate(ra, short, good, xyz, box)
    with pytest.raises(ValueError, match="ring 1 of rings2_start_indexes has 2 atoms"):
        ringpairs.pipi_calculate(ra, good, short, xyz, box)
    with pytest.raises(ValueError, match="ring 0 of rings_start_indexes has 0 atoms"):
        ringpairs.cationpi_calculate(ra, np.array([0, 0, 6], np.uint32), np.array([7], np.uint32), xyz, box)
    with pytest.raises(ValueError, match="ring 1 of rings_start_indexes has 1 atoms"):
        ringpairs.sigmahole_calculate(ra, np.array([0, 6, 7], np.uint32), np.array([[8, 9]], np.uint32), xyz, box)

    class Mol:
        numAtoms, numFrames = 12, 1

    Mol.coords, Mol.box = xyz, box
    rings = [np.arange(6), np.arange(6, 12)]
    with pytest.raises(ValueError, match=r"rings2\[1\] has 2 atoms"):
        interactions.pipi_calculate(Mol, rings, [np.arange(6), np.array([6, 7])])
    with pytest.raises(ValueError, match=r"rings1\[0\] has 0 atoms"):
        interactions.pipi_calculate(Mol, [np.array([], int)], rings)
    with pytest.raises(ValueError, match=r"rings\[1\] has 1 atoms"):
        interactions.cationpi_calculate(Mol, [np.arange(6), np.array([7])], [8])
    with pytest.raises(ValueError, match=r"rings\[0\] has 2 atoms"):
        interactions.sigmahole_calculate(Mol, [np.array([0, 1])], [[8, 9]])
