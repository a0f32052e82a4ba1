"""Interaction detectors on top of the GPU contact kernel (K4) and the hydrogen-bond kernel (K12) -- SURVEY 8f row 2.

Mirrors of the detectors in the reference that are thin consumers of ``calculate_contacts`` or ``hbonds.calculate``
(moleculekit/interactions/interactions.py):

  hbonds_calculate                :365-467     donor-H ... acceptor distance + angle test per frame (K12)
  waterbridge_calculate           :470-618     chains of hydrogen bonds through waters (host graph search over K12 shells)
  pipi_calculate / cationpi_calculate / sigmahole_calculate   :621-946   ring centroid / normal tests per frame (K13)
  saltbridge_calculate            :724-788     charged atoms within `threshold`, one positive + one negative per pair
  hydrophobic_calculate           :949-992     carbon - carbon contacts
  metal_coordination_calculate    :995-1056    metal - (N, O, S, halogen) contacts, both directions
  get_protein_charged / get_metal_charged      :292-306  (pure table look-ups on resname / name / element)

Selections are boolean masks / index arrays, or strings resolved by ``mol.atomselect``; the pair search itself is
``mkb_contacts_count`` + ``mkb_contacts_fill`` (bit-exact index output, reference order); hydrogen bonds run in
``mkb_hbonds_count`` + ``mkb_hbonds_fill``, the ring detectors in ``mkb_ring_pairs_count`` + ``mkb_ring_pairs_fill``.  The
perception helpers that need rdkit or residue templates (get_ligand_rings, get_protein_rings, ...) stay with moleculekit:
rings, cations and halogen bonds are inputs here, as they are for the reference's Cython kernels.
"""
from __future__ import annotations

import numpy as np

from .distance import calculate_contacts

# the element set moleculekit.periodictable.METAL_ELEMENTS (periodictable.py:317-407)
METAL_ELEMENTS = frozenset(
    "Ac Ag Al Am Au Ba Be Bi Bk Ca Cd Ce Cf Cm Co Cr Cs Cu Db Dy Er Es Eu Fe Fm Fr Ga Gd Ge Hf Hg Ho In Ir K La Li Lr Lu "
    "Md Mg Mn Mo Na Nb Nd Ni No Np Os Pa Pb Pd Pm Po Pr Pt Pu Ra Rb Re Rf Rh Ru Sb Sc Sg Sm Sn Sr Ta Tb Tc Th Ti Tl Tm U V "
    "W Y Yb Zn Zr".split())
COORDINATING_ELEMENTS = ["N", "O", "Cl", "F", "Br", "I", "CL", "BR", "S"]  # interactions.py:1034


def _mask(mol, sel) -> np.ndarray:
    """str -> mol.atomselect; bool mask as is; integer index array -> mask (what Molecule.atomselect accepts)."""
    if isinstance(sel, str):
        return np.asarray(mol.atomselect(sel), dtype=bool)
    sel = np.asarray(sel)
    if sel.dtype == bool:
        return sel.copy()
    m = np.zeros(int(mol.numAtoms), dtype=bool)
    m[sel] = True
    return m


def _periodic(mol):
    return "selections" if not np.all(mol.box == 0) else None


def get_protein_charged(mol):
    """interactions.py:296-306: (positive, negative) uint32 index arrays from residue / atom names."""
    resname, name = np.asarray(mol.resname), np.asarray(mol.name)
    pos = ((resname == "LYS") & (name == "NZ")) | ((resname == "ARG") & (name == "CZ")) | \
          ((resname == "HIP") & (name == "CE1"))
    neg = ((resname == "ASP") & (name == "CG")) | ((resname == "GLU") & (name == "CD"))
    return np.where(pos)[0].astype(np.uint32), np.where(neg)[0].astype(np.uint32)


def saltbridge_calculate(mol, pos, neg, sel1="all", sel2=None, threshold: float = 4, device=None):
    """interactions.py:724-788: per frame the (n, 2) pairs of charged atoms within ``threshold`` holding exactly one
    positive atom."""
    if len(pos) == 0 or len(neg) == 0:
        return [[] for _ in range(mol.numFrames)]
    m1 = _mask(mol, sel1)
    m2 = m1.copy() if sel2 is None else _mask(mol, sel2)
    charged = np.zeros(m1.shape, dtype=bool)
    charged[pos] = True
    charged[neg] = True
    inter = calculate_contacts(mol, m1 & charged, m2 & charged, _periodic(mol), threshold, device=device)
    return [fr[np.sum(np.isin(fr, pos), axis=1) == 1] for fr in inter]


def hydrophobic_calculate(mol, sel1, sel2, dist_threshold: float = 4.0, device=None):
    """interactions.py:949-992: carbon - carbon contacts between the two selections."""
    carbons = np.asarray(mol.element) == "C"
    return calculate_contacts(mol, _mask(mol, sel1) & carbons, _mask(mol, sel2) & carbons, _periodic(mol), dist_threshold,
                              device=device)


def metal_coordination_calculate(mol, sel1, sel2, dist_threshold: float = 3.5, device=None):
    """interactions.py:995-1056: metals of sel1 against coordinating atoms of sel2, then the other way round, stacked."""
    metals = sorted(METAL_ELEMENTS)
    m1, m2 = _mask(mol, sel1), _mask(mol, sel2)
    element = np.asarray(mol.element)
    is_metal, is_coord = np.isin(element, metals), np.isin(element, COORDINATING_ELEMENTS)
    periodic = _periodic(mol)
    inter1 = calculate_contacts(mol, m1 & is_metal, m2 & is_coord, periodic, dist_threshold, device=device)
    inter2 = calculate_contacts(mol, m1 & is_coord, m2 & is_metal, periodic, dist_threshold, device=device)
    return [np.vstack((inter1[f], inter2[f])) for f in range(mol.numFrames)]


def hbonds_calculate(mol, donors, acceptors, sel1="all", sel2=None, dist_threshold: float = 2.5,
                     angle_threshold: float = 120, ignore_hs: bool = False, device=None):
    """interactions.py:365-467: per frame the (n, 3) int64 array of (donor heavy atom, donor hydrogen | -1, acceptor)."""
    from . import hbonds

    if mol.box.shape[1] != mol.coords.shape[2]:
        raise RuntimeError("mol.box should have same number of frames as mol.coords")
    donors, acceptors = np.asarray(donors), np.asarray(acceptors)
    if len(donors) == 0 or len(acceptors) == 0:
        return [np.empty((0, 3), dtype=np.int64) for _ in range(mol.numFrames)]
    s1 = _mask(mol, sel1).astype(np.uint32)
    if sel2 is None:
        s2 = s1.copy()
        intra = True
    else:
        s2 = _mask(mol, sel2).astype(np.uint32)
        intra = False
    if len(s1) != mol.numAtoms or len(s2) != mol.numAtoms:
        raise RuntimeError("Selections must be boolean of size equal to number of atoms in the molecule")
    # donors / acceptors outside both selections can never pass (interactions.py:439-442)
    sel_idx = np.where(s1 | s2)[0]
    donors = donors[np.all(np.isin(donors, sel_idx), axis=1)]
    acceptors = acceptors[np.isin(acceptors, sel_idx)]
    if ignore_hs:
        donors = np.unique(donors[:, 0])[:, None]
    off, tri = hbonds.calculate_arrays(
        np.ascontiguousarray(donors.astype(np.uint32)), np.ascontiguousarray(acceptors.astype(np.uint32)),
        np.ascontiguousarray(mol.coords.astype(np.float32)), np.ascontiguousarray(mol.box.astype(np.float32)), s1, s2,
        dist_threshold=float(dist_threshold), angle_threshold=float(angle_threshold), intra=bool(intra),
        ignore_hs=bool(ignore_hs), device=device)
    return [tri[off[f]:off[f + 1]].astype(np.int64).reshape(-1, 3) for f in range(mol.numFrames)]


def waterbridge_calculate(mol, donors, acceptors, sel1, sel2, order: int = 1, dist_threshold: float = 2.5,
                          angle_threshold: float = 120, ignore_hs: bool = False, water="water", device=None):
    """interactions.py:470-618: per frame the list of atom-index paths from a sel1 atom to a sel2 atom whose intermediate
    atoms are all water; the hydrogen-bond shells run on K12, the path search is the reference's networkx walk.  ``water``:
    selection of the water atoms (string for ``mol.atomselect``, mask or indices; the reference hard-codes "water")."""
    import networkx as nx

    if len(donors) == 0 or len(acceptors) == 0:
        return [[] for _ in range(mol.numFrames)]
    sel1_b, sel2_b, water_b = _mask(mol, sel1), _mask(mol, sel2), _mask(mol, water)
    args = dict(mol=mol, donors=donors, acceptors=acceptors, dist_threshold=dist_threshold,
                angle_threshold=angle_threshold, ignore_hs=ignore_hs, device=device)
    water_goal = water_b | sel2_b
    water_goal_idx = np.where(water_goal)[0]
    water_idx = np.where(water_b)[0]
    order += 1  # an order-1 bridge needs two shells to reach the target (interactions.py:556-557)
    edges = [[] for _ in range(mol.numFrames)]
    sel1_b_curr = sel1_b.copy()
    for _ in range(order):
        curr_shell = hbonds_calculate(sel1=sel1_b_curr, sel2=water_goal, **args)
        for f in range(mol.numFrames):
            curr_shell[f] = np.array(curr_shell[f])
            if len(curr_shell[f]) == 0:
                continue
            has_water = np.any(np.isin(curr_shell[f], water_idx), axis=1)  # keep interactions with at least one water
            curr_shell[f] = curr_shell[f][has_water, :]
            if ignore_hs:
                edges[f].append(curr_shell[f][:, [0, 2]])
            else:
                edges[f].append(curr_shell[f][:, :2])
                edges[f].append(curr_shell[f][:, 1:])
        curr_shell = [cs for cs in curr_shell if len(cs) > 0]
        if len(curr_shell) == 0:
            break
        shell = np.vstack(curr_shell)[:, [0, 2]]
        sel1_b_curr = np.zeros(mol.numAtoms, dtype=bool)
        interacted = np.unique(shell[np.isin(shell, water_goal_idx)])
        if len(interacted) == 0:
            break
        sel1_b_curr[interacted] = True
    sel1_idx, sel2_idx = np.where(sel1_b)[0], np.where(sel2_b)[0]
    water_bridges = []
    for f in range(mol.numFrames):
        water_bridges.append([])
        if len(edges[f]) == 0:
            continue
        ee = np.vstack(edges[f])
        starts = np.unique(ee[np.isin(ee, sel1_idx)])
        ends = np.unique(ee[np.isin(ee, sel2_idx)])
        if not (np.any(starts) and np.any(ends)):  # (the reference's test: also skips when the only index is 0)
            continue
        network = nx.Graph()
        network.add_edges_from(ee)
        for st in starts:
            for en in ends:
                for pp in nx.all_simple_paths(network, source=st, target=en):
                    if len(pp) < 3:
                        continue
                    if not np.all(np.isin(pp[1:-1], water_idx)):
                        continue
                    water_bridges[f].append(pp)
    return water_bridges


def _check_rings(name, rings):
    """rings of fewer than 3 atoms have no normal (the reference reads the next ring's atoms for one): rejected"""
    for i, rr in enumerate(rings):
        if len(rr) < 3:
            raise ValueError(f"{name}[{i}] has {len(rr)} atoms; rings need at least 3")


def _ring_lists(mol, rings, off, pairs, da, return_rings, second_rings=None):
    index_list, dist_ang_list = [], []
    for f in range(mol.numFrames):
        pp = pairs[off[f]:off[f + 1]].tolist()
        if return_rings:
            index_list.append([[rings[a], second_rings[b] if second_rings is not None else b] for a, b in pp])
        else:
            index_list.append(pp)
        dist_ang_list.append(da[off[f]:off[f + 1]].tolist())
    return index_list, dist_ang_list


def pipi_calculate(mol, rings1, rings2, dist_threshold1: float = 4.4, angle_threshold1_max: float = 30,
                   dist_threshold2: float = 5.5, angle_threshold2_min: float = 60, return_rings: bool = False, device=None):
    """interactions.py:621-721: per frame the [ring1 index, ring2 index] pairs (or the rings themselves) and their
    [centroid distance, angle between the planes]."""
    from . import ringpairs

    if angle_threshold1_max < 0 or angle_threshold1_max > 90 or angle_threshold2_min < 0 or angle_threshold2_min > 90:
        raise RuntimeError("Values for angles should be [0, 90] degrees")
    _check_rings("rings1", rings1)
    _check_rings("rings2", rings2)
    if len(rings1) == 0 or len(rings2) == 0:
        return [[] for _ in range(mol.numFrames)], [[] for _ in range(mol.numFrames)]
    ring_atoms = np.hstack((np.hstack(rings1), np.hstack(rings2)))
    ring_starts1 = np.insert(np.cumsum([len(rr) for rr in rings1]), 0, 0)
    ring_starts2 = np.insert(np.cumsum([len(rr) for rr in rings2]), 0, 0)
    ring_starts2 += ring_starts1.max()
    off, pairs, da = ringpairs.calculate_arrays(
        ringpairs.PIPI, ring_atoms.astype(np.uint32), ring_starts1.astype(np.uint32), ring_starts2.astype(np.uint32),
        np.ascontiguousarray(mol.coords, dtype=np.float32), np.ascontiguousarray(mol.box, dtype=np.float32),
        dist_threshold1, angle_threshold1_max, dist_threshold2, angle_threshold2_min, device=device)
    return _ring_lists(mol, rings1, off, pairs, da, return_rings, second_rings=rings2)


def cationpi_calculate(mol, rings, cations, dist_threshold: float = 5, angle_threshold_min: float = 60,
                       return_rings: bool = False, device=None):
    """interactions.py:791-868: per frame [ring index, cation atom] and [centroid-cation distance, angle to the ring plane]."""
    from . import ringpairs

    if angle_threshold_min < 0 or angle_threshold_min > 90:
        raise RuntimeError("Values for angles should be [0, 90] degrees")
    _check_rings("rings", rings)
    if len(rings) == 0 or len(cations) == 0:
        return [[] for _ in range(mol.numFrames)], [[] for _ in range(mol.numFrames)]
    ring_atoms = np.hstack(rings)
    ring_starts = np.insert(np.cumsum([len(rr) for rr in rings]), 0, 0)
    off, pairs, da = ringpairs.calculate_arrays(
        ringpairs.CATIONPI, ring_atoms.astype(np.uint32), ring_starts.astype(np.uint32), np.array(cations, dtype=np.uint32),
        np.ascontiguousarray(mol.coords, dtype=np.float32), np.ascontiguousarray(mol.box, dtype=np.float32), dist_threshold,
        angle_threshold_min, device=device)
    return _ring_lists(mol, rings, off, pairs, da, return_rings)


def sigmahole_calculate(mol, rings, halides, dist_threshold: float = 4.5, angle_threshold_min: float = 60,
                        return_rings: bool = False, device=None):
    """interactions.py:871-946: per frame [ring index, halogen atom] and [centroid-halogen distance, angle of the halogen's
    bond to the ring plane]; ``halides``: (halogen, bonded atom) index pairs."""
    from . import ringpairs

    if angle_threshold_min < 0 or angle_threshold_min > 90:
        raise RuntimeError("Values for angles should be [0, 90] degrees")
    _check_rings("rings", rings)
    if len(rings) == 0 or len(halides) == 0:
        return [[] for _ in range(mol.numFrames)], [[] for _ in range(mol.numFrames)]
    ring_atoms = np.hstack(rings)
    ring_starts = np.insert(np.cumsum([len(rr) for rr in rings]), 0, 0)
    off, pairs, da = ringpairs.calculate_arrays(
        ringpairs.SIGMAHOLE, ring_atoms.astype(np.uint32), ring_starts.astype(np.uint32),
        np.array(halides, dtype=np.uint32).reshape(-1, 2), np.ascontiguousarray(mol.coords, dtype=np.float32),
        np.ascontiguousarray(mol.box, dtype=np.float32), dist_threshold, angle_threshold_min, device=device)
    return _ring_lists(mol, rings, off, pairs, da, return_rings)
