"""Host code shared by the trajectory projections: selection masks, the reference frame, the selections a metric
resolves per molecule, residues, and the device prologue of the superposing metrics (one upload of the trajectory,
the wrap of Molecule.wrap, the fit).  Plain functions: a metric module keeps only what is specific to that metric."""
from __future__ import annotations

import numpy as np

from ..atomselect_utils import as_mask


def nonempty(mol, sel, what):
    """Boolean mask of ``sel`` on ``mol``; RuntimeError ("{what} selection resulted in 0 atoms.") when it is empty."""
    mask = as_mask(mol.atomselect(sel), mol.numAtoms)
    if not mask.any():
        raise RuntimeError(f"{what} selection resulted in 0 atoms.")
    return mask


def check_sizes(what, a, b):
    """RuntimeError when the trajectory mask ``a`` and the reference mask ``b`` select different numbers of atoms."""
    if int(a.sum()) != int(b.sum()):
        raise RuntimeError(f"The {what} selections of the trajectory and the reference differ in size: "
                           f"{int(a.sum())} and {int(b.sum())} atoms.")


def reference(refmol, logger=None, name=None):
    """(a copy of ``refmol``, its coordinates at ``refmol.frame`` as (N, 3, 1) float32).  With ``logger``, a reference
    of more than one frame logs a warning that the metric ``name`` uses that frame."""
    ref = refmol.copy()
    frame = int(getattr(refmol, "frame", 0))
    if logger is not None and ref.coords.shape[2] > 1:
        logger.warning(f"Reference molecule contains multiple frames. {name} will use frame {frame} as reference.")
    return ref, np.ascontiguousarray(refmol.coords[:, :, frame:frame + 1], dtype=np.float32)


def selections(mol, props, entries):
    """``_calculateMolProp`` of a metric whose properties are selection masks.  ``entries`` lists (name, selection,
    what, used) in the order the selections are resolved, which decides the error raised when several are empty; the
    requested names (``props`` "all" or a list of names) get their :func:`nonempty` mask, and an entry that is not
    ``used`` (an alignment without a reference, a centre without ``pbc``) is skipped."""
    return {name: nonempty(mol, sel, what) for name, sel, what, used in entries
            if used and (props == "all" or name in props)}


def column(mol, field, default):
    """The per-atom array ``mol.<field>``, or ``default`` for every atom when the container has no such field."""
    v = getattr(mol, field, None)
    return np.full(mol.numAtoms, default, dtype=object) if v is None else np.asarray(v)


def residues(mol, sel):
    """The residues of the ``sel`` atoms in atom order: a new residue starts wherever resid, insertion, chain or segid
    changes from one selected atom to the next.  Returns a list of atom index arrays."""
    idx = np.where(sel)[0]
    if idx.size == 0:
        return []
    keys = [np.asarray(column(mol, f, d))[idx] for f, d in (("resid", 0), ("insertion", ""), ("chain", ""),
                                                           ("segid", ""))]
    change = np.zeros(idx.size, dtype=bool)
    change[0] = True
    for k in keys:
        change[1:] |= k[1:] != k[:-1]
    starts = np.append(np.where(change)[0], idx.size)
    return [idx[a:b] for a, b in zip(starts[:-1], starts[1:])]


def device_indices(mask, dev):
    """The atoms of ``mask`` as an int32 tensor on ``dev``."""
    import torch

    return torch.from_numpy(np.where(mask)[0].astype(np.int32)).to(dev)


def upload_wrapped(mol, centersel, device):
    """``mol.coords`` uploaded once as an (N, 3, F) float32 CUDA tensor on ``device`` (None: the current device) and,
    unless ``centersel`` is None, wrapped in place around that mask as Molecule.wrap does."""
    import torch

    from .. import _lib
    from ..wrapping import wrap_plan

    dev = _lib.device(device)
    d = torch.from_numpy(np.ascontiguousarray(mol.coords, dtype=np.float32)).to(dev)
    if centersel is not None:
        plan = wrap_plan(mol, centersel)
        if plan is not None:
            plan.run_device(d, torch.from_numpy(np.ascontiguousarray(mol.box, dtype=np.float32)).to(dev))
    return d


def fit(d, trajalnsel, ref, refalnsel):
    """The fit records of every frame of ``d`` superposed onto ``ref`` (the (M, 3, 1) float32 reference, a numpy array
    or a tensor on d's device): the ``trajalnsel`` atoms onto the ``refalnsel`` atoms (masks).  A non-finite fit raises
    ``numpy.linalg.LinAlgError`` before anything else runs."""
    import torch

    from ..align import raise_if_nonfinite, superpose_device

    records, status = superpose_device(d, device_indices(trajalnsel, d.device), torch.as_tensor(ref, device=d.device),
                                       device_indices(refalnsel, d.device))
    raise_if_nonfinite(status, np.arange(d.shape[2]))
    return records
