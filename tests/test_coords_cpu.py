"""Coordinate and fluctuation projections without a GPU: the float64 oracle (oracle/coords_oracle.py) on analytic cases,
the constructor defaults, mappings and error messages of MetricCoordinate / MetricFluctuation (all checked before any
device work), residue grouping, and the frame-sharded fluctuation on world_size-2 gloo with a CPU stand-in compute."""
import os
import socket
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import coords_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_rigid_motion_gives_zero_fluctuation():
    rng = np.random.default_rng(0)
    S = rng.normal(0, 10, size=(30, 3))
    F = 6
    X = np.stack([S @ Rotation.random(random_state=f).as_matrix() + rng.normal(0, 20, 3) for f in range(F)], axis=2)
    sel = np.arange(0, 30, 2)
    aln = np.ones(30, bool)
    rows = co.coordinates(X, sel, refcoords=S[:, :, None], alnsel=aln, refalnsel=aln)
    assert rows.shape == (F, 3 * sel.size)
    assert np.abs(rows - co.coordinates(np.repeat(S[:, :, None], F, 2), sel)).max() < 1e-10
    assert np.abs(co.fluctuation(rows, S[sel])).max() < 1e-20
    assert np.abs(co.fluctuation(rows, co.mean(rows))).max() < 1e-20


def test_oracle_column_order_and_residue_means():
    X = np.arange(2 * 3 * 4, dtype=np.float64).reshape(2, 3, 4)  # 2 atoms, 4 frames
    rows = co.coordinates(X, [1, 0])
    assert rows[2].tolist() == [X[1, 0, 2], X[0, 0, 2], X[1, 1, 2], X[0, 1, 2], X[1, 2, 2], X[0, 2, 2]]
    # three atoms in one frame, deviations 1, 4 and 9 from the origin; groups {0, 1} and {2}
    rows = np.array([[1.0, 0.0, 0.0, 0.0, 2.0, 0.0, 0.0, 0.0, 3.0]])
    dev = co.fluctuation(rows, np.zeros((3, 3)))
    assert dev.tolist() == [[1.0, 4.0, 9.0]]
    assert co.fluctuation(rows, np.zeros((3, 3)), np.array([0, 2, 3])).tolist() == [[2.5, 9.0]]
    assert np.allclose(co.mean(np.array([[0.0] * 3, [2.0] * 3])), [[1.0, 1.0, 1.0]])


def test_residue_groups_non_contiguous():
    from moleculekit_b200.projections.metricfluctuation import residue_groups

    resid = np.array([7, 3, 7, 12, 3, 3, 7])
    order, offsets, residues = residue_groups(resid)
    assert residues.tolist() == [3, 7, 12] and offsets.tolist() == [0, 3, 6, 7]
    assert order.tolist() == [1, 4, 5, 0, 2, 6, 3]  # stable: selection order inside a residue
    o2, off2 = co.residue_groups(resid)
    assert np.array_equal(o2, order) and np.array_equal(off2, offsets)


def _mol(F=4, n=12, seed=0, resid=None):
    from moleculekit_b200.molecule_lite import MolLite

    rng = np.random.default_rng(seed)
    names = {"protein": np.arange(n) < n - 2, "protein and name CA": np.arange(n) % 3 == 0,
             "sel": np.isin(np.arange(n), [1, 2, 5, 9])}
    return MolLite(rng.normal(0, 5, size=(n, 3, F)).astype(np.float32), named_selections=names,
                   resname=[f"R{i % 4}" for i in range(n)], name=[f"A{i}" for i in range(n)],
                   resid=np.arange(n) // 3 if resid is None else resid)


def test_metriccoordinate_defaults_and_mapping():
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate

    ref = _mol(F=3, seed=1)
    ref.frame = 2
    m = MetricCoordinate("sel", refmol=ref)
    assert m._trajalnsel == "protein and name CA" and m._centersel == "protein" and m._pbc
    assert np.array_equal(m._refalnsel, ref.atomselect("protein and name CA"))
    assert np.array_equal(m._refcoords[:, :, 0], ref.coords[:, :, 2])
    m2 = MetricCoordinate("sel", refmol=ref, trajalnsel="protein")
    assert np.array_equal(m2._refalnsel, ref.atomselect("protein"))  # refalnsel defaults to trajalnsel
    m3 = MetricCoordinate("sel")
    assert m3._refmol is None and m3._trajalnsel is None  # nothing is superposed
    mol = _mol()
    mp = m.getMapping(mol)
    assert len(mp) == 12 and set(mp["type"]) == {"coordinate"}
    assert mp["atomIndexes"].tolist() == [1, 2, 5, 9] * 3
    assert mp["description"].tolist()[:2] == ["X coordinate of R1 0 A1", "X coordinate of R2 0 A2"]
    assert mp["description"].tolist()[4] == "Y coordinate of R1 0 A1"
    assert mp["description"].tolist()[11] == "Z coordinate of R1 3 A9"
    empty = _mol(F=0)
    assert MetricCoordinate("sel", pbc=False).project(empty).shape == (0, 12)


def test_metriccoordinate_errors():
    from moleculekit_b200.projections.metriccoordinate import MetricCoordinate

    mol, ref = _mol(), _mol(seed=1)
    with pytest.raises(RuntimeError, match="Reference alignment selection resulted in 0 atoms"):
        MetricCoordinate("sel", refmol=ref, trajalnsel=np.zeros(12, bool))
    with pytest.raises(RuntimeError, match="Atom selection resulted in 0 atoms"):
        MetricCoordinate(np.zeros(12, bool), pbc=False).project(mol)
    with pytest.raises(RuntimeError, match="Alignment selection resulted in 0 atoms"):
        MetricCoordinate("sel", refmol=ref, trajalnsel=np.zeros(12, bool), refalnsel="protein").project(mol)
    with pytest.raises(RuntimeError, match="Centering selection resulted in 0 atoms"):
        MetricCoordinate("sel", centersel=np.zeros(12, bool)).project(mol)
    with pytest.raises(RuntimeError, match=r"alignment selections .* differ in size: 4 and 10"):
        MetricCoordinate("sel", refmol=ref, refalnsel="protein", pbc=False).project(mol)


def test_metricfluctuation_defaults_mapping_and_errors():
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation

    resid = np.array([5, 5, 2, 2, 9, 2, 5, 9, 9, 2, 1, 1])
    mol = _mol(resid=resid)
    ref = _mol(seed=1, resid=resid)
    ref.frame = 3
    m = MetricFluctuation("sel", refmol=ref)
    assert m._trajalnsel == "protein and name CA" and m._centersel == "protein" and m._mode == "atom" and m._pbc
    assert np.array_equal(m._refalnsel, ref.atomselect("protein and name CA"))  # refalnstr defaults to trajalnstr
    assert np.array_equal(m._refcoords[:, :, 0], ref.coords[:, :, 3])
    mp = m.getMapping(mol)
    assert mp["type"].tolist() == ["fluctuation"] * 4 and mp["atomIndexes"].tolist() == [1, 2, 5, 9]
    assert mp["description"].tolist() == ["Fluctuation of R1 5 A1", "Fluctuation of R2 2 A2",
                                          "Fluctuation of R1 2 A5", "Fluctuation of R1 2 A9"]
    assert np.array_equal(m.reference_centre(mol), ref.coords[[1, 2, 5, 9], :, 3].astype(np.float64))

    r = MetricFluctuation("sel", refmol=ref, mode="residue")
    mp = r.getMapping(mol)  # selection 1, 2, 5, 9 has resids 5, 2, 2, 2: residue 2 first
    assert mp["description"].tolist() == ["Fluctuation of residue R2 2", "Fluctuation of residue R1 5"]
    assert [a.tolist() for a in mp["atomIndexes"]] == [[2, 5, 9], [1]]
    sel, offsets = r._layout(mol)
    assert sel.tolist() == [2, 5, 9, 1] and offsets.tolist() == [0, 3, 4]
    assert np.array_equal(r.reference_centre(mol), ref.coords[[2, 5, 9, 1], :, 3].astype(np.float64))
    assert MetricFluctuation("sel", mode="residue", pbc=False).project(_mol(F=0, resid=resid)).shape == (0, 2)

    with pytest.raises(ValueError, match="mode"):
        MetricFluctuation("sel", mode="chain")
    with pytest.raises(RuntimeError, match="Reference atom selection resulted in 0 atoms"):
        MetricFluctuation(np.zeros(12, bool), refmol=ref)
    with pytest.raises(RuntimeError, match="Atom selection resulted in 0 atoms"):
        MetricFluctuation(np.zeros(12, bool), pbc=False).project(mol)
    with pytest.raises(RuntimeError, match="Centering selection resulted in 0 atoms"):
        MetricFluctuation("sel", centerstr=np.zeros(12, bool)).project(mol)
    small = _mol(n=12, seed=2, resid=resid)
    small.named_selections["sel"] = np.isin(np.arange(12), [1, 2])
    with pytest.raises(RuntimeError, match=r"atom selections .* differ in size: 4 and 2"):
        MetricFluctuation("sel", refmol=small, pbc=False).project(mol)
    with pytest.raises(RuntimeError, match=r"alignment selections .* differ in size: 4 and 10"):
        MetricFluctuation("sel", refmol=ref, refalnstr="protein", pbc=False).project(mol)


def test_project_sharded_refuses_referenceless_fluctuation():
    from moleculekit_b200.projections.metricfluctuation import MetricFluctuation
    from moleculekit_b200.sharding import project_sharded

    with pytest.raises(ValueError, match="fluctuation_sharded"):
        project_sharded(MetricFluctuation("sel", pbc=False), _mol())


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _oracle_compute(metric, view, centre):
    """CPU stand-in for the K15 kernels (no superposition, no wrap): frame sums or deviations in the metric's layout"""
    sel, offsets = metric._layout(view)
    rows = co.coordinates(view.coords, sel)
    if centre is None:
        return co.as_points(rows).sum(axis=0)
    return co.fluctuation(rows, centre, offsets).astype(np.float32)


def _gloo_worker(rank, world, port, tmpdir):
    import torch.distributed as dist

    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from moleculekit_b200.projections.metricfluctuation import MetricFluctuation
        from moleculekit_b200.sharding import fluctuation_sharded

        resid = np.array([5, 5, 2, 2, 9, 2, 5, 9, 9, 2, 1, 1])
        mol = _mol(F=7, resid=resid)
        for mode in ("atom", "residue"):
            m = MetricFluctuation("protein", pbc=False, mode=mode)
            # single rank: the mean of all frames
            centre = _oracle_compute(m, mol, None) / 7
            want = _oracle_compute(m, mol, centre)
            got = fluctuation_sharded(m, mol, compute_fn=_oracle_compute)
            # float64 sums of float32 coordinates over 7 frames are exact, whatever the order of the ranks
            assert got.shape == want.shape and np.array_equal(got, want), mode
            part, (f0, f1) = fluctuation_sharded(m, mol, gather=False, compute_fn=_oracle_compute)
            assert (f0, f1) == ((0, 4) if rank == 0 else (4, 7)) and np.array_equal(part, want[f0:f1])
        open(os.path.join(tmpdir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_fluctuation_sharded_gloo_world2(tmp_path):
    import torch.multiprocessing as mp

    mp.spawn(_gloo_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()
