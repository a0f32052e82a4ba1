"""Float64 restatement of the per-frame group moments and the two projections built on them -- TEST INFRASTRUCTURE ONLY.

  moleculekit/projections/metricgyration.py             mass-weighted radius of gyration and its x, y, z components
  moleculekit/projections/metricsphericalcoordinate.py  r, theta, phi of one selection's centre relative to another's

Like ``oracle/coords_oracle.fluctuation`` these take (F, 3k) coordinate rows (X block | Y block | Z block, as
``coords_oracle.coordinates`` returns them; the tests pass the float64 superposition rounded to float32, or the device's
own coordinates) and do the rest in float64 numpy, two passes (mean, then the spread around it).
"""
from __future__ import annotations

import numpy as np

from oracle.coords_oracle import as_points


def moments(rows, weights=None, offsets=None):
    """(F, G, 6) float64: per frame and group of columns' atoms [offsets[g], offsets[g+1]) the weighted mean (0-2) and
    the weighted per-axis variance around it (3-5); weights None = 1, offsets None = one group"""
    P = as_points(rows)
    k = P.shape[1]
    w = np.ones(k) if weights is None else np.asarray(weights, dtype=np.float64)
    offsets = np.array([0, k]) if offsets is None else np.asarray(offsets)
    out = np.empty((P.shape[0], offsets.size - 1, 6))
    for g, (a, b) in enumerate(zip(offsets[:-1], offsets[1:])):
        wg, Pg = w[a:b], P[:, a:b]
        mu = np.einsum("k,fkd->fd", wg, Pg) / wg.sum()
        out[:, g, :3] = mu
        out[:, g, 3:] = np.einsum("k,fkd->fd", wg, (Pg - mu[:, None]) ** 2) / wg.sum()
    return out


def gyration(rows, masses):
    """(F, 4) float64 [rg, rg_x, rg_y, rg_z] of (F, 3k) rows weighted by ``masses`` (k,)"""
    v = moments(rows, masses)[:, 0, 3:]
    return np.column_stack([np.sqrt(v.sum(axis=1)), np.sqrt(v)])


def spherical(rows, ref_idx, tgt_idx):
    """(F, 3) float64 [r, theta, phi] of the plain centre of the columns' atoms ``tgt_idx`` relative to that of
    ``ref_idx``"""
    P = as_points(rows)
    x = P[:, np.asarray(tgt_idx)].mean(axis=1) - P[:, np.asarray(ref_idx)].mean(axis=1)
    r = np.linalg.norm(x, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        theta = np.arccos(x[:, 2] / r)
    return np.column_stack([r, theta, np.arctan2(x[:, 1], x[:, 0])])
