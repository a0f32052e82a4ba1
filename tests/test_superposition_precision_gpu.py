"""The float64 reductions of K14 (fit, apply, RMSD), K15 (frame sums), K20 (group moments) and K19 (the all-pairs fit
of the TM-score search) against the exact reference of oracle/exact_superposition.py, on the inputs where such
reductions lose precision: near-planar, near-collinear and mirror-image selections, 180 degree rotations, two- to
four-atom and repeated selections, coincident atoms, coordinates 1e4-1e5 A from the origin, structures 1e-3 A across, a
first selected atom far from the rest, and selections of 511 to 2^20 atoms.

The fit objective and the fitted RMSD are second order in the rotation error, so they cannot see most fit defects:
wherever Horn's eigenvalue gap makes the optimal rotation R* well defined, the records are compared with R* itself.
Every case runs with one reference frame and with matching frames, and through an explicit frame list."""
import functools
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import exact_superposition as ex

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


def _rigid(P, R, t):
    """q = R p + t for every row p, rounded to float32"""
    return (P.astype(np.float64) @ np.asarray(R, dtype=np.float64).T + t).astype(np.float32)


def _rot(seed):
    return Rotation.random(random_state=seed).as_matrix()


def _turn(axis):
    """the 180 degree rotation about ``axis``"""
    n = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return 2 * np.outer(n, n) - np.eye(3)


SIGNED_PERMUTATIONS = [np.eye(3), np.diag([1, -1, -1]), np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]]),
                       np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]]), np.array([[0, 0, -1], [0, -1, 0], [-1, 0, 0]])]


def _stack(frames):
    return np.ascontiguousarray(np.stack(frames, axis=2))


def _copies(B, seed, F=3, noise=0.0, offset=0.0, ref=None):
    """trajectory of F rigid copies of the (k, 3) base B (plus noise) and F reference frames (rigid copies of B, or
    ``ref`` (k, 3) in every frame), all placed around ``offset``"""
    rng = np.random.default_rng(seed)
    off = np.array([offset, -offset, 0.5 * offset])
    X, Y = [], []
    for f in range(F):
        t = off + rng.uniform(-20, 20, 3)
        x = _rigid(B, _rot(seed * 31 + f), t)
        if noise:
            x = (x + rng.normal(0, noise, x.shape)).astype(np.float32)
        X.append(x)
        Y.append(_rigid(B, _rot(seed * 37 + f + 1000), off + rng.uniform(-20, 20, 3)) if ref is None else ref)
    return _stack(X), _stack(Y)


def _turned(B, axes, seed):
    """frame f = B turned 180 degrees about axes[f] and moved; the reference is B"""
    rng = np.random.default_rng(seed)
    X = [_rigid(B, _turn(a), rng.uniform(-20, 20, 3)) for a in axes]
    return _stack(X), _stack([B] * len(axes))


def _case_data(name):
    """(trajectory (N, 3, F), reference frames (N, 3, F), selection) float32, float32, int32"""
    rng = np.random.default_rng(sum(map(ord, name)))
    cloud = lambda k, s=10.0: rng.normal(0, s, (k, 3)).astype(np.float32)  # noqa: E731
    sel = None
    if name == "rigid":
        X, Y = _copies(cloud(60), 1)
    elif name == "noisy":
        X, Y = _copies(cloud(60), 2, noise=1.0)
    elif name in ("mirror", "near-planar mirror"):
        B = cloud(60)
        if name != "mirror":
            B[:, 2] = rng.normal(0, 1e-4, 60)
        X, Y = _copies(B, 3, ref=(B * np.float32([1, 1, -1])).astype(np.float32))
    elif name == "near-planar":
        B = cloud(60)
        B[:, 2] = rng.normal(0, 1e-4, 60)
        X, Y = _copies(B, 4, noise=1e-5)
    elif name == "near-collinear":
        B = np.column_stack([np.linspace(-30, 30, 60), rng.normal(0, 1e-4, 60), rng.normal(0, 1e-4, 60)])
        X, Y = _copies(B.astype(np.float32), 5)
    elif name == "collinear":
        line = (np.arange(-20, 21, dtype=np.float32)[:, None] * np.float32([1, 2, -2])).astype(np.float32)
        X = _stack([(line @ M.T.astype(np.float32) + np.float32([3, -4, 5]) * f).astype(np.float32)
                    for f, M in enumerate(SIGNED_PERMUTATIONS[1:4])])
        Y = _stack([line] * 3)
    elif name == "turn xyz":
        X, Y = _turned(cloud(60), [[1, 0, 0], [0, 1, 0], [0, 0, 1]], 6)
    elif name == "turn diagonal":
        X, Y = _turned(cloud(60), [[1, 1, 1], [1, -1, 0], [0, 1, -1]], 7)
    elif name == "integer 90":
        B = rng.integers(-50, 50, (48, 3)).astype(np.float32)
        X = _stack([(B @ M.T.astype(np.float32) + rng.integers(-9, 9, 3)).astype(np.float32)
                    for M in SIGNED_PERMUTATIONS[1:]])
        Y = _stack([(B @ M.T.astype(np.float32) + rng.integers(-9, 9, 3)).astype(np.float32)
                    for M in SIGNED_PERMUTATIONS[:4]])
    elif name.startswith("atoms "):
        X, Y = _copies(cloud(int(name[6:])), 8, noise=0.5)
    elif name == "repeated":
        X, Y = _copies(cloud(20), 9, noise=0.5)
        sel = np.array([0, 1, 2, 0, 1, 2, 5, 5, 5, 5, 19, 7, 7, 0])
    elif name == "coincident":
        p = np.float32([[12.5, -3.25, 7.0]])
        X, Y = _stack([np.repeat(p + f, 9, axis=0) for f in range(3)]), _stack([np.repeat(p - 100, 9, axis=0)] * 3)
    elif name.startswith("offset "):
        X, Y = _copies(cloud(60), 10, offset=float(name[7:]))
    elif name.startswith("offset-noisy "):
        X, Y = _copies(cloud(60), 11, noise=0.5, offset=float(name[13:]))
    elif name == "tiny":
        X, Y = _copies(cloud(60, 2.5e-4), 12)
    elif name == "far first atom":
        B = cloud(60)
        B[0] = [500.0, 0.0, 0.0]
        X, Y = _copies(B, 13, noise=0.5)
    elif name.startswith("size "):
        k = int(name[5:])
        X, Y = _copies(cloud(k, 30.0), 14, F=2 if k > 10 ** 5 else 3, noise=1.0)
    else:
        raise KeyError(name)
    if sel is None:
        k = X.shape[0]
        sel = np.arange(k)
        if k < 10 ** 5:  # two atoms outside the selection: apply moves every atom
            X = np.concatenate([X, X[:2] + np.float32(1.5)])
            Y = np.concatenate([Y, Y[:2]])
    return X, Y, sel.astype(np.int32)


CASES = ["rigid", "noisy", "mirror", "near-planar mirror", "near-planar", "near-collinear", "collinear", "turn xyz",
         "turn diagonal", "integer 90", "atoms 1", "atoms 2", "atoms 3", "atoms 4", "repeated", "coincident",
         "offset 1e4", "offset 1e5", "offset-noisy 1e5", "tiny", "far first atom", "size 511", "size 512", "size 513",
         "size 8193", "size 1048576"]
MODES = ["single", "matching"]


@functools.lru_cache(maxsize=None)
def _data(name):
    return _case_data(name)


@functools.lru_cache(maxsize=None)
def _exact(name, f, rf):
    X, Y, sel = _data(name)
    return ex.ExactFit(X[sel, :, f], Y[sel, :, rf])


def _ref(name, mode):
    X, Y, sel = _data(name)
    return Y if mode == "matching" else np.ascontiguousarray(Y[:, :, :1])


_DEVICE = {}


def _fit(name, mode):
    """(trajectory, reference, selection on the device, records and status on the host) of the call over every
    frame"""
    import torch
    from moleculekit_b200.align import superpose_device

    if (name, mode) not in _DEVICE:
        _DEVICE.clear()  # one case at a time on the device
        X, Y, sel = _data(name)
        dev = torch.device("cuda:0")
        d, r = torch.from_numpy(X).to(dev), torch.from_numpy(_ref(name, mode)).to(dev)
        s = torch.from_numpy(sel).to(dev)
        rec, st = superpose_device(d, s, r, s)
        _DEVICE[(name, mode)] = (d, r, s, rec.cpu().numpy(), st.cpu().numpy())
    return _DEVICE[(name, mode)]


def _frame_list(F):
    return np.array([F - 1, 0] if F > 1 else [0], dtype=np.int32)


def _signed_permutation(R):
    """the exact R* as a float64 matrix when it is a signed permutation (else None)"""
    if R is None:
        return None
    M = np.array([[float(x) for x in row] for row in R])
    P = np.round(M)
    ok = all(abs(x - p) < mp.mpf(10) ** -40 for row, prow in zip(R, P) for x, p in zip(row, prow))
    return P if ok and np.array_equal(np.abs(P).sum(0), np.ones(3)) else None


def _ulps(a, b):
    """|a - b| in float32 ulps of b (elementwise, float32 arrays)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.abs(b)).astype(np.float64)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_fit_records(name, mode):
    """det R = +1 and R orthogonal to 8 eps; centroids within 4 eps max|x|; R within 64 eps lam1 / gap of R* where the
    gap is at least 1e-6 lam1, else the objective within 16 eps G of the optimum; H = 0 gives the identity bit for bit;
    exact signed permutations within 8 eps; an explicit frame list gives the bits of the whole call"""
    import torch
    from moleculekit_b200.align import superpose_device

    X, Y, sel = _data(name)
    d, r, s, rec, st = _fit(name, mode)
    F = X.shape[2]
    assert not st.any()
    for f in range(F):
        fit = _exact(name, f, f if mode == "matching" else 0)
        R, pb, qb = rec[f, :9].reshape(3, 3), rec[f, 9:12], rec[f, 12:15]
        P, Q = X[sel, :, f], Y[sel, :, f if mode == "matching" else 0]
        assert np.abs(R @ R.T - np.eye(3)).max() <= 8 * EPS, f
        assert abs(np.linalg.det(R) - 1) <= 8 * EPS, f
        for got, want, scale in ((pb, fit.p_bar, np.abs(P).max()), (qb, fit.q_bar, np.abs(Q).max())):
            err = max(abs(ex.to_mpf(Fraction(float(g)) - w)) for g, w in zip(got, want))
            assert err <= 4 * EPS * scale, (f, float(err))
        if all(x == 0 for row in fit.H for x in row):
            assert np.array_equal(R, np.eye(3)), f
            continue
        if fit.gap > 0 and fit.gap >= mp.mpf("1e-6") * fit.lam1:
            Rs = np.array([[float(x) for x in row] for row in fit.R])
            bound = 64 * EPS * float(fit.lam1 / fit.gap)
            assert np.abs(R - Rs).max() <= bound, (f, np.abs(R - Rs).max() / bound)
        else:
            assert ex.to_mpf(fit.objective(R)) <= fit.E + 16 * EPS * ex.to_mpf(fit.G), f
        M = _signed_permutation(fit.R)
        if M is not None:
            assert np.abs(R - M).max() <= 8 * EPS, f
    fl = _frame_list(F)
    rec2, st2 = superpose_device(d, s, r, s, torch.from_numpy(fl).to(d.device))
    assert np.array_equal(rec2.cpu().numpy().view(np.int64), rec[fl].view(np.int64))
    assert not st2.cpu().numpy().any()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_apply(name, mode):
    """every coordinate of every atom within 1 float32 ulp of fl32 of the exact R (x - p_bar) + q_bar under the device's
    own record, plus the float64 evaluation's own error (a few eps of |R| |x - p_bar| + |q_bar|: it decides only where the
    terms cancel to near 0), nearly all of the others equal to it; integer cases give the exact integers (0 within that float64
    error); an explicit frame list moves only
    its frames, with the same bits; the gathered coordinates have the applied bits"""
    import torch
    from moleculekit_b200.align import apply_device, superpose_device
    from moleculekit_b200.coords import coordinates_device

    X, Y, sel = _data(name)
    d, r, s, rec, st = _fit(name, mode)
    F = X.shape[2]
    out = apply_device(d.clone(), torch.from_numpy(rec).to(d.device)).cpu().numpy()
    exact = total = 0
    for f in range(F):
        R, pb, qb = rec[f, :9].reshape(3, 3), rec[f, 9:12], rec[f, 12:15]
        want = ex.transform_f32(R, pb, qb, X[:, :, f])
        f64 = 4 * EPS * (np.abs(X[:, :, f] - pb) @ np.abs(R).T + np.abs(qb))
        err = np.abs(out[:, :, f].astype(np.float64) - want)
        assert (err <= np.spacing(np.abs(want)).astype(np.float64) + f64).all(), (f, _ulps(out[:, :, f], want).max())
        clean = f64 < 0.5 * np.spacing(np.abs(want)).astype(np.float64)  # no cancellation to near 0
        exact += int((out[:, :, f] == want)[clean].sum())
        total += int(clean.sum())
        fit = _exact(name, f, f if mode == "matching" else 0)
        M = _signed_permutation(fit.R)
        if M is not None and fit.objective(M) == 0 and np.array_equal(X[sel], np.round(X[sel])):
            # the integers themselves; an exact 0 keeps what R's last-bit departure from M times x leaves
            ints, got = Y[sel, :, f if mode == "matching" else 0], out[sel, :, f]
            assert np.array_equal(got[ints != 0], ints[ints != 0]), f
            assert (np.abs(got[ints == 0]) <= f64[sel][ints == 0]).all(), f
    assert exact >= 0.99 * total, (exact, total)
    rows = coordinates_device(d, s, torch.from_numpy(rec).to(d.device)).cpu().numpy()
    k = sel.size
    for f in range(F):
        assert np.array_equal(rows[f].reshape(3, k).T.view(np.uint32), out[sel, :, f].view(np.uint32))
    fl = _frame_list(F)
    dfl = torch.from_numpy(fl).to(d.device)
    rec2, _ = superpose_device(d, s, r, s, dfl)
    part = apply_device(d.clone(), rec2, dfl).cpu().numpy()
    assert np.array_equal(part[:, :, fl].view(np.uint32), out[:, :, fl].view(np.uint32))
    rest = np.setdiff1d(np.arange(F), fl)
    assert np.array_equal(part[:, :, rest].view(np.uint32), X[:, :, rest].view(np.uint32))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", CASES)
def test_rmsd(name, mode):
    """with the records: within 1 float32 ulp of the exact RMSD under those records, plus the float64 evaluation of a
    deviation (a few eps of the coordinate scale: it decides only where the RMSD is near 0); without records: within 1
    ulp of the exact molRMSD; an explicit frame list gives the same values"""
    import torch
    from moleculekit_b200.align import rmsd_device

    X, Y, sel = _data(name)
    d, r, s, rec, st = _fit(name, mode)
    F = X.shape[2]
    drec = torch.from_numpy(rec).to(d.device)
    fitted = rmsd_device(d, s, r, s, drec).cpu().numpy()
    plain = rmsd_device(d, s, r, s).cpu().numpy()
    for f in range(F):
        fit = _exact(name, f, f if mode == "matching" else 0)
        want = fit.rmsd(rec[f, :9], rec[f, 9:12], rec[f, 12:15])
        scale = np.abs(X[sel, :, f]).max() + np.abs(Y[sel]).max()
        tol = float(np.spacing(np.float32(float(want)))) + 8 * EPS * scale
        assert abs(float(fitted[f]) - want) <= tol, (f, float(fitted[f]), float(want))
        want = fit.rmsd()
        assert abs(float(plain[f]) - want) <= float(np.spacing(np.float32(float(want)))), (f, float(plain[f]), float(want))
    fl = _frame_list(F)
    dfl = torch.from_numpy(fl).to(d.device)
    got = rmsd_device(d, s, r, s, drec[torch.from_numpy(fl.astype(np.int64)).to(d.device)].contiguous(), dfl)
    assert np.array_equal(got.cpu().numpy(), fitted[fl])


def _alternating_rows(F, k, cancel, seed):
    """(N, 3, F) raw coordinates near the origin and records that turn frame f and move it by +-1e4 A: the offsets
    alternate in sign (cancel) or are all +1e4"""
    rng = np.random.default_rng(seed)
    X = rng.normal(0, 3.0, (k, 3, F)).astype(np.float32)
    rec = np.zeros((F, 16))
    for f in range(F):
        rec[f, :9] = _rot(seed + f).ravel()
        rec[f, 9:12] = rng.normal(0, 1, 3)
        rec[f, 12:15] = (1e4 if (f % 2 == 0 or not cancel) else -1e4) + rng.normal(0, 1, 3)
    return X, rec


@pytest.mark.parametrize("cancel", [True, False])
@pytest.mark.parametrize("F", [63, 65, 127, 129])
def test_frame_sums(F, cancel):
    """K15 sums over 64 k +- 1 frames of the device's own aligned rows: within n eps sum |c| of the exact sum (the
    offsets cancel: sum |c| >> |s*|), and within 1e-12 relative where they do not; an explicit frame list over the same
    frames in the same order gives the same bits"""
    import torch
    from moleculekit_b200.coords import coord_sums_device, coordinates_device

    k = 70
    X, rec = _alternating_rows(F, k, cancel, F)
    dev = torch.device("cuda:0")
    d, s, drec = torch.from_numpy(X).to(dev), torch.arange(k, dtype=torch.int32, device=dev), torch.from_numpy(rec).to(dev)
    rows = coordinates_device(d, s, drec).cpu().numpy().reshape(F, 3, k).transpose(0, 2, 1)
    got = coord_sums_device(d, s, drec).cpu().numpy()
    want = ex.frame_sums(rows)
    absum = np.abs(rows.astype(np.float64)).sum(0)
    err = np.array([[float(abs(Fraction(float(got[i, a])) - want[i, a])) for a in range(3)] for i in range(k)])
    assert (err <= F * EPS * absum).all(), (err / (F * EPS * absum)).max()
    if not cancel:
        wf = np.array([[float(w) for w in row] for row in want])
        assert (err <= 1e-12 * np.abs(wf)).all()
    fl = torch.arange(F, dtype=torch.int32, device=dev)
    assert np.array_equal(coord_sums_device(d, s, drec, fl).cpu().numpy().view(np.int64), got.view(np.int64))


MOMENT_CASES = ["tiny spread far out", "far first position", "wide weights", "small groups"]


def _moment_case(name):
    """(coordinates (N, 3, F), weights, group offsets, records (F, 16)) of a K20 case"""
    rng = np.random.default_rng(sum(map(ord, name)))
    F, m = 5, 1200
    off = np.array([1e4, -1e4, 0.5e4])
    X = (rng.normal(0, 1e-3, (m, 3, F)) + off[None, :, None]).astype(np.float32)
    w = None
    groups = [0, 600, m]  # one group of 2 segments, one of 2 segments
    if name == "far first position":
        X = rng.normal(0, 5.0, (m, 3, F)).astype(np.float32)
        X[0] += np.float32([500, 0, 0])[:, None]
        X[600] -= np.float32([0, 500, 0])[:, None]
    elif name == "wide weights":
        X = (rng.normal(0, 2.0, (m, 3, F)) + off[None, :, None]).astype(np.float32)
        w = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), m))
        w[0] = w[600] = 1e-3
        groups = [0, 513, m]
    elif name == "small groups":
        X = (rng.normal(0, 1.0, (m, 3, F)) + off[None, :, None]).astype(np.float32)
        w = rng.uniform(0.5, 16, m)
        groups = [0, 1, 3, 4, 6, m]
    rec = np.zeros((F, 16))
    for f in range(F):
        rec[f, :9] = _rot(f + 50).ravel()
        rec[f, 9:12] = X[:, :, f].astype(np.float64).mean(0)
        rec[f, 12:15] = off + rng.normal(0, 1, 3)
    return X, w, np.asarray(groups, np.int64), rec


@pytest.mark.parametrize("name", MOMENT_CASES)
def test_group_moments(name):
    """K20 on the device's own aligned rows against the exact two-pass moments:
    |mu - mu*| <= 4 eps |mu*| + gamma sum w |c - s| / W and |v - v*| <= 16 eps (v* + (mu* - s)^2) + gamma sum w (c - s)^2 / W,
    gamma = (m / 512 + 512) eps for a group of m positions and s the group's first position"""
    import torch
    from moleculekit_b200.coords import coordinates_device, frame_moments_device

    X, w, groups, rec = _moment_case(name)
    F, k = X.shape[2], X.shape[0]
    dev = torch.device("cuda:0")
    d, s, drec = torch.from_numpy(X).to(dev), torch.arange(k, dtype=torch.int32, device=dev), torch.from_numpy(rec).to(dev)
    rows = coordinates_device(d, s, drec).cpu().numpy().reshape(F, 3, k).transpose(0, 2, 1)
    got = frame_moments_device(d, s, drec, weights=w, groups=groups).cpu().numpy()
    want = ex.moments(rows, w, groups)
    wt = np.ones(k) if w is None else w
    for g, (a, b) in enumerate(zip(groups[:-1], groups[1:])):
        gamma = ((b - a) / 512 + 512) * EPS
        W = wt[a:b].sum()
        for f in range(F):
            c = rows[f, a:b].astype(np.float64)
            e = c - c[0]
            for ax in range(3):
                mu, v = want[f, g, ax], want[f, g, 3 + ax]
                s0 = Fraction(float(c[0, ax]))
                err = abs(Fraction(float(got[f, g, ax])) - mu)
                bound = 4 * EPS * abs(float(mu)) + gamma * float((wt[a:b] * np.abs(e[:, ax])).sum() / W)
                assert float(err) <= bound, (g, f, ax, float(err) / bound)
                err = abs(Fraction(float(got[f, g, 3 + ax])) - v)
                bound = 16 * EPS * float(v + (mu - s0) ** 2) + gamma * float((wt[a:b] * e[:, ax] ** 2).sum() / W)
                assert float(err) <= bound, (g, f, ax, float(err) / bound)


TM_CASES = ["integer 90", "noisy", "offset-noisy 1e5", "far first atom", "size 513"]


@pytest.mark.parametrize("name", TM_CASES)
def test_tmscore_first_fit(name):
    """K19's rmsd (the all-pairs first fit) within 1e-12 relative plus 1e-13 of the coordinate scale of the exact Kabsch
    RMSD; rigid integer copies score exactly 1"""
    import torch
    from moleculekit_b200.tmscore import tmscore_device

    X, Y, sel = _data(name)
    F = X.shape[2]
    dev = torch.device("cuda:0")
    d, r = torch.from_numpy(X).to(dev), torch.from_numpy(np.ascontiguousarray(Y[:, :, :1])).to(dev)
    s = torch.from_numpy(sel).to(dev)
    tm, rmsd = (t.cpu().numpy() for t in tmscore_device(d, s, r, s))
    for f in range(F):
        fit = _exact(name, f, 0)
        want = float(fit.min_rmsd())
        scale = max(np.abs(X[sel, :, f]).max(), np.abs(Y[sel, :, 0]).max())
        assert abs(rmsd[f] - want) <= 1e-12 * want + 1e-13 * scale, (f, rmsd[f], want)
        M = _signed_permutation(fit.R)
        if M is not None and fit.objective(M) == 0:
            assert tm[f] == 1.0, (f, tm[f])


@pytest.mark.parametrize("k", [513, 4097])
def test_rmsd_dominated_sum(k):
    """one deviation of 4096 A among deviations of 0.5 A: in float32 every later square (0.25) would vanish against the
    first (2^24), so the RMSD is within 1 ulp of the exact one only if its sums run in float64 (with an identity record
    and without a record)"""
    import torch
    from moleculekit_b200.align import rmsd_device

    rng = np.random.default_rng(k)
    F = 3
    Y = (rng.integers(-400, 400, (k, 3, F)) / 8).astype(np.float32)
    dev_ = np.zeros((k, 3, F), np.float32)
    axis = rng.integers(0, 3, (k, F))
    for f in range(F):
        dev_[np.arange(k), axis[:, f], f] = np.where(rng.random(k) < 0.5, -0.5, 0.5)
    dev_[0, :, :] = 0
    dev_[0, 0, :] = 4096
    X = (Y + dev_).astype(np.float32)
    dev = torch.device("cuda:0")
    d, r = torch.from_numpy(X).to(dev), torch.from_numpy(Y).to(dev)
    s = torch.arange(k, dtype=torch.int32, device=dev)
    rec = np.zeros((F, 16))
    rec[:, [0, 4, 8]] = 1.0
    for records in (None, torch.from_numpy(rec).to(dev)):
        got = rmsd_device(d, s, r, s, records).cpu().numpy()
        for f in range(F):
            want = ex.ExactFit(X[:, :, f], Y[:, :, f]).rmsd()
            assert abs(float(got[f]) - want) <= float(np.spacing(np.float32(float(want)))), (f, float(got[f]), float(want))
