"""Float64 restatement of the reference's coordinate and fluctuation projections -- TEST INFRASTRUCTURE ONLY.

  moleculekit/projections/metriccoordinate.py     align, then the selection's coordinates, one row per frame
  moleculekit/projections/metricfluctuation.py    squared deviation from the mean or a reference, per atom or residue

Coordinates come from :func:`oracle.align_oracle.align` (the reference's SVD fit in float64).  The device rounds every
aligned coordinate to float32 before it measures a deviation, so :func:`fluctuation` takes the coordinate rows it is
given (the tests pass the float64 superposition rounded to float32) and does the rest in float64.
"""
from __future__ import annotations

import numpy as np

from oracle import align_oracle


def coordinates(coords, sel, refcoords=None, alnsel=None, refalnsel=None, refframe=0):
    """(F, 3k) float64: the ``sel`` atoms of ``coords`` (N, 3, F), superposed frame by frame onto ``refcoords`` at
    ``refframe`` on ``alnsel`` / ``refalnsel`` (no superposition without ``refcoords``); columns X block | Y | Z."""
    X = np.asarray(coords, dtype=np.float64)
    if refcoords is not None:
        X = align_oracle.align(coords, refcoords, alnsel, refalnsel, refframe=refframe)
    S = X[np.asarray(sel)]                       # (k, 3, F)
    return np.ascontiguousarray(np.transpose(S, (2, 1, 0)).reshape(S.shape[2], 3 * S.shape[0]))


def as_points(rows):
    """(F, 3k) rows -> (F, k, 3)"""
    F, k3 = rows.shape
    return np.transpose(np.asarray(rows, dtype=np.float64).reshape(F, 3, k3 // 3), (0, 2, 1))


def mean(rows):
    """(k, 3) float64 mean structure over the frames of (F, 3k) coordinate rows"""
    return as_points(rows).mean(axis=0)


def fluctuation(rows, centre, offsets=None):
    """(F, k) float64 squared deviations of (F, 3k) coordinate rows from ``centre`` (k, 3), or with group ``offsets``
    (G + 1,) over the columns' atoms, (F, G) per-group means."""
    dev = np.sum((as_points(rows) - np.asarray(centre, dtype=np.float64)[None]) ** 2, axis=2)
    if offsets is None:
        return dev
    return np.stack([dev[:, a:b].mean(axis=1) for a, b in zip(offsets[:-1], offsets[1:])], axis=1)


def residue_groups(resid):
    """(order, offsets): the stable sort of a selection by resid and the group boundaries of its distinct resids"""
    resid = np.asarray(resid)
    order = np.argsort(resid, kind="stable")
    bounds = np.flatnonzero(np.diff(resid[order])) + 1
    return order, np.concatenate([[0], bounds, [resid.size]]).astype(np.int64)
