"""DSSP without a GPU: known answers of the C restatement (tests/dssp_oracle.c) on ideal constructions, the bend
threshold, and MetricSecondaryStructure's residue table, output maps, mapping and errors."""
import math

import numpy as np
import pytest

import dssp_oracle as do


def _letters(codes):
    from moleculekit_b200.dssp import LETTERS

    return "".join(LETTERS[codes]).replace(" ", "-")


def _run(bb, flags=None):
    flags = np.zeros(bb.shape[0], np.uint8) if flags is None else flags
    return _letters(do.frame(np.asarray(bb, np.float32), flags)[0])


def test_alpha_helix():
    """phi -57, psi -47: every NH(i+4) -> O(i) bond holds, so there is a 4-turn at i = 0..15; H needs 4-turns at i and
    i - 1 (i = 1..15) and covers i..i+3, i.e. residues 1..18.  Residues 0 and 19 stay loop (T and S skip the ends)."""
    bb = do.chain([-57] * 20, [-47] * 20)
    assert _run(bb) == "-" + "H" * 18 + "-"
    _, partner, energy, _ = do.frame(bb.astype(np.float32), np.zeros(20, np.uint8))
    for d in range(4, 20):
        assert d - 4 in partner[d] and energy[d][list(partner[d]).index(d - 4)] < -0.5


def test_310_helix():
    """phi -49, psi -26: 3-turns at i = 0..16 and no two consecutive 4-turns, so G covers residues 1..18"""
    assert _run(do.chain([-49] * 20, [-26] * 20)) == "-" + "G" * 18 + "-"


def test_antiparallel_and_parallel_pairs():
    bb, fl = do.strand_pair(10, True)
    assert _run(bb, fl) == "-EEEEEEE---EEEEEEE--"
    bb, fl = do.strand_pair(10, False)
    assert _run(bb, fl) == "-EEEEEEEE--EEEEEEEE-"
    # moved apart, no bond survives
    bb, fl = do.strand_pair(10, True, dist=9.0)
    assert _run(bb, fl) == "-" * 20


def test_isolated_bridge():
    """a three-residue partner: one bridge of size one, B on both sides"""
    bb, fl = do.strand_pair(10, True)
    short = np.concatenate([bb[:10], bb[13:16]])
    f = np.zeros(13, np.uint8)
    f[10] = 2
    assert _run(short, f) == "----B------B-"


def test_bend():
    """an extended chain with one residue at phi 60, psi 60: the CA(i-2), CA(i), CA(i+2) angle exceeds 70 degrees and no
    turn covers it"""
    phi, psi = [180.0] * 12, [180.0] * 12
    phi[6], psi[6] = 60.0, 60.0
    assert _run(do.chain(phi, psi)) == "------S-----"


def test_chain_split():
    """the helix cut by moving residues 10.. 2 A along C9 -> N10 (C-N 3.3 A): no turn spans the break, so H stops at
    residue 8 and restarts at 11, and residues 9, 10 have neither a turn nor a kappa"""
    bb = do.chain([-57] * 20, [-47] * 20)
    d = bb[10, 0] - bb[9, 2]
    bb[10:] += 2.0 * d / np.linalg.norm(d)
    assert _run(bb) == "-" + "H" * 8 + "--" + "H" * 8 + "-"
    # the same cut by a chain flag alone
    fl = np.zeros(20, np.uint8)
    fl[10] = 2
    assert _run(do.chain([-57] * 20, [-47] * 20), fl) == "-" + "H" * 8 + "--" + "H" * 8 + "-"


def test_proline_donor():
    """a proline donates no hydrogen bond: its slots stay empty and the 4-turn at 8 is lost.  One lost turn does not
    open an alpha helix (the starts at 7 and 10 still cover 7..13); three lost turns in a row do."""
    bb = do.chain([-57] * 20, [-47] * 20).astype(np.float32)
    fl = np.zeros(20, np.uint8)
    fl[12] = 1
    codes, partner, energy, _ = do.frame(bb, fl)
    assert list(partner[12]) == [-1, -1] and list(energy[12]) == [0.0, 0.0]
    assert _letters(codes) == "-" + "H" * 18 + "-"
    fl[13] = fl[14] = 1  # no 4-turn at 8, 9, 10: the starts at 7 (7..10) and 12 (12..15) leave residue 11 out
    got = _letters(do.frame(bb, fl)[0])
    assert got[11] != "H" and got[1:11] == "H" * 10 and got[12:19] == "H" * 7


def test_bend_threshold():
    from moleculekit_b200.dssp import bend_threshold

    c = bend_threshold()
    below = np.nextafter(c, -1.0)
    assert (math.acos(c) * 180) / 3.14159265358979323846 <= 70
    assert (math.acos(below) * 180) / 3.14159265358979323846 > 70
    assert abs(c - math.cos(math.radians(70))) < 1e-15


def _mol(names, resnames, resid, chain):
    from moleculekit_b200.molecule_lite import MolLite

    n = len(names)
    return MolLite(np.zeros((n, 3, 2), np.float32), name=names, resname=resnames, resid=resid, chain=chain,
                   named_selections={"protein": np.ones(n, bool)})


def test_residue_table():
    from moleculekit_b200.projections.metricsecondarystructure import dssp_residues

    names = ["N", "CA", "C", "O", "N", "CA", "C", "N", "CA", "CA", "C", "O", "N", "CA", "C", "O"]
    resn = ["ALA"] * 4 + ["GLY"] * 3 + ["PRO"] * 5 + ["SER"] * 4
    resid = [1] * 4 + [2] * 3 + [3] * 5 + [4] * 4
    chain = ["A"] * 12 + ["B"] * 4
    mol = _mol(names, resn, resid, chain)
    bb, fl, pos, res = dssp_residues(mol, np.ones(16, bool))
    assert len(res) == 4 and pos.tolist() == [0, -1, 1, 2]  # residue 2 has no O
    assert bb.tolist() == [[0, 1, 2, 3], [7, 8, 10, 11], [12, 13, 14, 15]]  # the first CA of residue 3
    assert fl.tolist() == [0, 1, 2]  # PRO; a new chain


def test_output_maps_and_mapping(monkeypatch):
    from moleculekit_b200.dssp import FULL_INT, LETTERS, SIMPLE_INT, SIMPLE_LETTERS
    from moleculekit_b200.projections.metricsecondarystructure import MetricSecondaryStructure

    assert "".join(LETTERS) == " HBEGIT S".replace("T S", "TS")
    assert FULL_INT.tolist() == [7, 0, 1, 2, 3, 4, 5, 6] and SIMPLE_INT.tolist() == [2, 0, 1, 1, 0, 0, 2, 2]
    assert "".join(SIMPLE_LETTERS) == "CHEEHHCC"
    codes = np.arange(8, dtype=np.uint8)[None, :]
    pos = np.array([0, -1, 1, 2, 3, 4, 5, 6, 7])
    m = MetricSecondaryStructure()
    assert m._encode(codes, pos).tolist() == [[2, -1, 0, 1, 1, 0, 0, 2, 2]]
    m = MetricSecondaryStructure(simplified=False)
    assert m._encode(codes, pos).tolist() == [[7, -1, 0, 1, 2, 3, 4, 5, 6]]
    m = MetricSecondaryStructure(integer=False)
    out = m._encode(codes, pos)
    assert out.dtype == np.dtype("<U2") and out.tolist() == [["C", "NA", "H", "E", "E", "H", "H", "C", "C"]]
    m = MetricSecondaryStructure(simplified=False, integer=False)
    assert m._encode(codes, pos).tolist() == [[" ", "NA", "H", "B", "E", "G", "I", "T", "S"]]

    mol = _mol(["N", "CA", "C", "O", "N", "CA"], ["ALA"] * 4 + ["GLY"] * 2, [5] * 4 + [6] * 2, ["A"] * 6)
    mp = MetricSecondaryStructure(sel="protein").getMapping(mol)
    assert mp["type"].tolist() == ["secondary structure"] * 2
    assert mp["description"].tolist() == ["Secondary structure of residue ALA 5", "Secondary structure of residue GLY 6"]
    assert mp["atomIndexes"][1].tolist() == [4, 5]
    # no residue has a full backbone: every column is NA and nothing reaches the device
    only = MetricSecondaryStructure(sel=np.array([0, 0, 0, 0, 1, 1], bool), integer=False)
    assert only.project(mol).tolist() == [["NA"], ["NA"]]
    with pytest.raises(RuntimeError, match="0 atoms"):
        MetricSecondaryStructure(sel=np.zeros(6, bool)).getMapping(mol)


def test_string_mode_refuses_gather(monkeypatch):
    from moleculekit_b200 import sharding
    from moleculekit_b200.projections.metricsecondarystructure import MetricSecondaryStructure

    mol = _mol(["N", "CA", "C", "O"], ["ALA"] * 4, [1] * 4, ["A"] * 4)
    monkeypatch.setattr(sharding, "world_info", lambda group=None: (2, 0))
    with pytest.raises(ValueError, match="integer=True"):
        sharding.project_sharded(MetricSecondaryStructure(integer=False), mol)


def test_no_cpu_fallback():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from moleculekit_b200 import _lib
    from moleculekit_b200.dssp import dssp_device
    from moleculekit_b200.projections.metricsecondarystructure import MetricSecondaryStructure

    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        dssp_device(torch.zeros((4, 3, 2)), torch.zeros((1, 4), dtype=torch.int32), torch.zeros(1, dtype=torch.uint8))
    mol = _mol(["N", "CA", "C", "O"], ["ALA"] * 4, [1] * 4, ["A"] * 4)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        MetricSecondaryStructure().project(mol)
