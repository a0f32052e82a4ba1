"""Probes of the hydrogen-bond (K12, csrc/hbonds.cu) and ring (K13, csrc/rings.cu) detectors at their cut-offs.

Both kernels decide the reference's `acosf(c) > thr` / `fold((double)acosf(dot) * 57.29578) <op> thr` without a device
acos: the host turns each decision into a bound (K12) or into intervals (K13) of the float cosine.  This module gives the
tests an independent reference for those decisions and geometries that land exactly on them:

* `run_scan` builds a small C program that walks every float of [-1, 1] with the host libm: it checks that acosf never
  increases, finds each K12 bound c* by exhaustion, and lists the floats at which each K13 predicate changes value.
* the `*_set` builders make one frame per probe, placed so that the decided quantity (cosine, dot product, squared
  distance) equals a chosen float exactly.  `simulate` recomputes those quantities from the coordinates with numpy float32
  operations in the kernels' order, so a construction that misses its target is caught before any detector runs.
* `reference_hits` evaluates the reference's predicate on the simulated quantities with ctypes libm acosf.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
import os
import shutil
import subprocess

import numpy as np

f32 = np.float32
ANGLE_SCALE = 57.29578
LE, GE, PLANE = 0, 1, 2  # K13 predicates: pi-pi angle <= a1max, pi-pi angle >= a2min, cation-pi / sigma-hole 90 - angle >= amin
PRED_NAMES = ("le", "ge", "plane")
K12_ANGLES = (0.0, 1e-3, 37.5, 90.0, 119.99999, 120.0, 150.0, 179.9, 180.0, 180.0001, 400.0)
K13_ANGLES = (0.0, 1e-5, 30.0, 45.0, 60.0, 89.99999, 90.0, 0.3183, 12.345, 57.2957, 71.03, 88.8888)
OFFSETS = (-3, -2, -1, 0, 1, 2, 3)  # floats either side of a transition


def fkey(x) -> int:
    """Order-preserving integer image of a float32 (-0 and +0 share key 0), as rings.cu's fkey."""
    b = int(np.array(x, np.float32).view(np.int32))
    return b if b >= 0 else -(b & 0x7FFFFFFF)


def funkey(k: int):
    b = k if k >= 0 else (0x80000000 | (-k))
    return np.array(b, np.uint32).view(np.float32)[()]


KMIN, KMAX = fkey(-1.0), fkey(1.0)

# ---------------------------------------------------------------------------------------------------------------------
# the exhaustive scan

SCAN_SRC = r"""
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* Every float x of [-1, 1] in key order: acosf(x) must not increase; per K12 threshold the bit acosf(x) > thr
 * (hbonds.pyx:50, 129), per K13 threshold the bits of the three predicates on the folded double angle (pipi.pyx:176-177,
 * cationpi.pyx:165).  Each thread reports the bit words at its first float and every key where a word changes. */
#define MAXH 64
#define MAXR 21
#define MAXCHG 4096
static int nh, nr;
static float hthr[MAXH];   /* (float)((double)angle_threshold / 57.29578) */
static double rthr[MAXR];  /* the float threshold, compared in double */
static const int64_t KMIN = -0x3f800000LL, KMAX = 0x3f800000LL;

static float unkey(int64_t k)
{
    int32_t b = k >= 0 ? (int32_t)k : (int32_t)(0x80000000u | (uint32_t)(-k));
    float x;
    memcpy(&x, &b, 4);
    return x;
}

typedef struct {
    int64_t k0, k1, mono_bad, mono_first, nchg;
    uint64_t h0, r0;
    int64_t chg_k[MAXCHG];
    uint64_t chg_h[MAXCHG], chg_r[MAXCHG];
} Part;

static void words(float a, uint64_t *h, uint64_t *r)
{
    uint64_t wh = 0, wr = 0;
    for (int j = 0; j < nh; ++j) wh |= (uint64_t)(a > hthr[j]) << j;
    double ang = (double)a * 57.29578;
    if (ang > 90) ang = 180 - ang;
    for (int j = 0; j < nr; ++j)
        wr |= ((uint64_t)(ang <= rthr[j]) | (uint64_t)(ang >= rthr[j]) << 1 | (uint64_t)(90 - ang >= rthr[j]) << 2) << (3 * j);
    *h = wh; *r = wr;
}

static void *run(void *arg)
{
    Part *p = (Part *)arg;
    uint64_t ph = 0, pr = 0, h, r;
    float aprev = 0.f;
    int have = 0;
    if (p->k0 > KMIN) { aprev = acosf(unkey(p->k0 - 1)); words(aprev, &ph, &pr); have = 1; }
    for (int64_t k = p->k0; k < p->k1; ++k) {
        const float a = acosf(unkey(k));
        if (have && !(a <= aprev)) { if (!p->mono_bad) p->mono_first = k; ++p->mono_bad; }
        words(a, &h, &r);
        if (k == p->k0) { p->h0 = h; p->r0 = r; }
        if (have && (h != ph || r != pr)) {
            if (p->nchg < MAXCHG) { p->chg_k[p->nchg] = k; p->chg_h[p->nchg] = h; p->chg_r[p->nchg] = r; }
            ++p->nchg;
        }
        ph = h; pr = r; aprev = a; have = 1;
    }
    return NULL;
}

static float from_hex(const char *s)
{
    uint32_t b = (uint32_t)strtoul(s, NULL, 16);
    float x;
    memcpy(&x, &b, 4);
    return x;
}

/* argv: nthreads nh <nh float bits in hex> nr <nr float bits in hex> */
int main(int argc, char **argv)
{
    int a = 1;
    if (argc < 4) return 2;
    int nt = atoi(argv[a++]);
    nh = atoi(argv[a++]);
    if (nh > MAXH) return 2;
    for (int j = 0; j < nh; ++j) hthr[j] = (float)((double)from_hex(argv[a++]) / 57.29578);
    nr = atoi(argv[a++]);
    if (nr > MAXR) return 2;
    for (int j = 0; j < nr; ++j) rthr[j] = (double)from_hex(argv[a++]);
    if (nt < 1) nt = 1;
    if (nt > 256) nt = 256;
    Part *parts = (Part *)calloc(nt, sizeof(Part));
    pthread_t th[256];
    const int64_t n = KMAX - KMIN + 1;
    for (int t = 0; t < nt; ++t) {
        parts[t].k0 = KMIN + n * t / nt;
        parts[t].k1 = KMIN + n * (t + 1) / nt;
        pthread_create(&th[t], NULL, run, &parts[t]);
    }
    int64_t bad = 0, first = 0;
    for (int t = 0; t < nt; ++t) {
        pthread_join(th[t], NULL);
        if (parts[t].mono_bad && !bad) first = parts[t].mono_first;
        bad += parts[t].mono_bad;
    }
    printf("mono %lld %lld\n", (long long)bad, (long long)first);
    printf("start %llx %llx\n", (unsigned long long)parts[0].h0, (unsigned long long)parts[0].r0);
    for (int t = 0; t < nt; ++t) {
        if (parts[t].nchg > MAXCHG) { printf("overflow\n"); return 1; }
        for (int64_t q = 0; q < parts[t].nchg; ++q)
            printf("chg %lld %llx %llx\n", (long long)parts[t].chg_k[q], (unsigned long long)parts[t].chg_h[q],
                   (unsigned long long)parts[t].chg_r[q]);
    }
    return 0;
}
"""


class Scan:
    """Result of the exhaustive walk over the floats of [-1, 1]: `mono_bad` floats where acosf increased, `cstar[angle]`
    the largest key with acosf > the K12 threshold (None when there is none), `sets[(angle, pred)]` the K13 predicate's
    value at -1 and the keys where it changes."""

    def __init__(self, text: str, k12_angles, k13_angles):
        chg = []
        for line in text.split("\n"):
            w = line.split()
            if not w:
                continue
            assert w[0] != "overflow", "more changes than the scan records"
            if w[0] == "mono":
                self.mono_bad, self.mono_first = int(w[1]), int(w[2])
            elif w[0] == "start":
                h0, r0 = int(w[1], 16), int(w[2], 16)
            elif w[0] == "chg":
                chg.append((int(w[1]), int(w[2], 16), int(w[3], 16)))
        self.cstar, self.sets = {}, {}
        for j, angle in enumerate(k12_angles):
            v, last = (h0 >> j) & 1, None
            for k, h, _ in chg:
                nv = (h >> j) & 1
                if nv != v:
                    if v:
                        last = k - 1
                    v = nv
            self.cstar[angle] = KMAX if v else last
        for j, angle in enumerate(k13_angles):
            for i in range(3):
                b = 3 * j + i
                v0 = bool((r0 >> b) & 1)
                v, trs = v0, []
                for k, _, r in chg:
                    nv = bool((r >> b) & 1)
                    if nv != v:
                        trs.append(k)
                        v = nv
                self.sets[(angle, i)] = (v0, trs)

    def member(self, angle, pred, key: int) -> bool:
        """Is the float of `key` in the set where K13 predicate `pred` at threshold `angle` holds?"""
        v, trs = self.sets[(angle, pred)]
        for t in trs:
            if key >= t:
                v = not v
        return v


def run_scan(workdir, k12_angles=K12_ANGLES, k13_angles=K13_ANGLES, nthreads=None):
    """Build and run the scan in `workdir`; None when the host has no C compiler."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        return None
    src = os.path.join(str(workdir), "acosf_scan.c")
    exe = os.path.join(str(workdir), "acosf_scan")
    with open(src, "w") as fh:
        fh.write(SCAN_SRC)
    subprocess.run([cc, "-O2", "-ffp-contract=off", "-fno-fast-math", "-pthread", src, "-o", exe, "-lm"], check=True,
                   capture_output=True)
    hexes = lambda xs: [format(int(np.array(x, np.float32).view(np.uint32)), "08x") for x in xs]
    nt = nthreads or max(1, min(64, os.cpu_count() or 1))
    args = [exe, str(nt), str(len(k12_angles)), *hexes(k12_angles), str(len(k13_angles)), *hexes(k13_angles)]
    out = subprocess.run(args, check=True, capture_output=True, text=True).stdout
    return Scan(out, k12_angles, k13_angles)


_libm = None


def acosf(x) -> float:
    """The host libm's acosf through ctypes (the library the reference and the kernels' host code call)."""
    global _libm
    if _libm is None:
        _libm = ctypes.CDLL(ctypes.util.find_library("m"))
        _libm.acosf.restype = ctypes.c_float
        _libm.acosf.argtypes = [ctypes.c_float]
    return float(f32(_libm.acosf(float(f32(x)))))


def folded(dot) -> float:
    a = acosf(dot) * ANGLE_SCALE
    return 180.0 - a if a > 90.0 else a


def k13_pred(angle, pred, dot) -> bool:
    a, t = folded(dot), float(f32(angle))
    return a <= t if pred == LE else (a >= t if pred == GE else 90.0 - a >= t)


# ---------------------------------------------------------------------------------------------------------------------
# float32 helpers in the kernels' order of operations

def roundf(q):
    """C roundf (half away from zero) on float32 values."""
    q = np.asarray(q, np.float32)
    t = np.trunc(q)
    return np.where(np.abs(q - t) >= f32(0.5), t + np.sign(q), t).astype(np.float32)


def wrap(v, b):
    """val - fl(b * roundf(fl(val / b))) when |val| > b / 2 and b != 0 (the interactions rule, every op in float32)."""
    v, b = np.asarray(v, np.float32), np.asarray(b, np.float32)
    with np.errstate(all="ignore"):
        w = v - b * roundf(v / b)
        return np.where((np.abs(v) > b / f32(2)) & (b != 0), w, v).astype(np.float32)


def sq3(x, y, z):
    x, y, z = (np.asarray(a, np.float32) for a in (x, y, z))
    return (x * x + y * y) + z * z


def ratio(p, q):
    """fl(p / sqrtf(fl(fl(q*q) + fl(p*p)))): the normalised component every angle probe is built on."""
    p, q = np.asarray(p, np.float32), np.asarray(q, np.float32)
    with np.errstate(all="ignore"):
        return p / np.sqrt(q * q + p * p)


def solve_ratio(T, R=2.0):
    """(p, q) float32 with ratio(p, q) == T exactly and hypot(p, q) ~ R."""
    T = f32(T)
    if T == 1 or T == -1:
        return f32(T) * f32(R), f32(0)
    s, t = (f32(1) if T > 0 else f32(-1)), abs(float(T))
    if t < 2.0 ** -12:  # q = 2: fl(4 + p*p) == 4, so the ratio is p / 2
        p = f32(2 * t)
        if ratio(p, f32(2)) == f32(t):
            return s * p, f32(2)
    rng = np.random.default_rng(fkey(T) & 0x7FFFFFFF)
    p0, q0 = t * R, math.sqrt(max(1.0 - t * t, 0.0)) * R
    for scale in (1e-7, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 0.3):
        p = (p0 * (1 + scale * rng.uniform(-1, 1, 40000))).astype(np.float32)
        q = (q0 * (1 + scale * rng.uniform(-1, 1, 40000))).astype(np.float32)
        ok = np.flatnonzero(ratio(p, q) == f32(t))
        if ok.size:
            return s * p[ok[0]], q[ok[0]]
    raise AssertionError(f"no (p, q) gives ratio {T!r}")


def solve_sumsq(T, grid, lo=0.35, hi=0.93):
    """(x, y) on multiples of `grid` (a power of two) with fl(fl(x*x) + fl(y*y)) == T exactly, x / sqrt(T) in [lo, hi]."""
    T = f32(T)
    r = math.sqrt(float(T))
    xs = (np.arange(math.ceil(lo * r / grid), math.floor(hi * r / grid) + 1, dtype=np.float64) * grid).astype(np.float32)
    x2 = xs * xs
    y0 = np.round(np.sqrt(np.maximum(float(T) - x2.astype(np.float64), 0)) / grid)
    for dy in (0, -1, 1, -2, 2):
        y = ((y0 + dy) * grid).astype(np.float32)
        ok = np.flatnonzero(x2 + y * y == T)
        if ok.size:
            i = ok[len(ok) // 2]
            return xs[i], y[i]
    raise AssertionError(f"no grid point gives squared norm {T!r}")


def neighbours(x, offsets=OFFSETS, lo=None, hi=None):
    """[(offset, float)] of the floats `offset` keys from x, inside [lo, hi] when given."""
    k = fkey(x)
    out = []
    for d in offsets:
        v = funkey(k + d)
        if (lo is not None and v < lo) or (hi is not None and v > hi) or not np.isfinite(v):
            continue
        out.append((d, v))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# probe sets: every frame one probe of a tiny system

class ProbeSet:
    """Frames of one detector call.  kind: 'hb', 'pipi', 'cationpi' or 'sigmahole'; `args` the detector's arguments besides
    coords and box.  Per frame: `value` (the designed cosine / dot / squared distance, float32), `what` ('c', 'dot', 'd2',
    'd2a', 'first'), `group` (frames of one boundary, None for free probes) and `edge` (the frame sits on the transition
    float itself)."""

    def __init__(self, name, kind, n_atoms, args):
        self.name, self.kind, self.n_atoms, self.args = name, kind, n_atoms, dict(args)
        self._xyz, self._box, self.value, self.what, self.group, self.edge = [], [], [], [], [], []

    def add(self, xyz, box, value=np.nan, what=None, group=None, edge=False):
        xyz = np.asarray(xyz, np.float32)
        assert xyz.shape == (self.n_atoms, 3)
        self._xyz.append(xyz)
        self._box.append(np.broadcast_to(np.asarray(box, np.float32), (3,)))
        self.value.append(f32(value)); self.what.append(what); self.group.append(group); self.edge.append(bool(edge))

    @property
    def coords(self):
        return np.ascontiguousarray(np.stack(self._xyz, axis=2))

    @property
    def box(self):
        return np.ascontiguousarray(np.stack(self._box, axis=1))

    def __len__(self):
        return len(self._xyz)

    def groups(self):
        g = {}
        for f, name in enumerate(self.group):
            if name is not None:
                g.setdefault(name, []).append(f)
        return g


SHIFTS = ((1, 0, 0), (0, -2, 0), (0, 0, 3), (-1, 2, -3), (3, -1, 1))


def _shifted(p, shift, L):
    return np.asarray(p, np.float32) + np.asarray(shift, np.float32) * f32(L)


# ---- K12 ------------------------------------------------------------------------------------------------------------
# atoms: 0 = H, 1 = donor heavy atom D, 2 = acceptor A; donors [[1, 0]], acceptors [2]

def _hb_args(dist, angle, ignore_hs=False):
    return dict(donors=np.array([[1, 0]], np.uint32), acceptors=np.array([2], np.uint32),
                sel1=np.ones(3, np.uint32), sel2=np.ones(3, np.uint32), dist_threshold=dist, angle_threshold=angle,
                intra=True, ignore_hs=ignore_hs)


def hb_angle_set(scan, angle, dist=2.5):
    """H at the origin, D at (1, 0, 0), A at (p, q, 0) with c == c* and its neighbours (c* found by the scan)."""
    ps = ProbeSet(f"hb_angle_{angle}", "hb", 3, _hb_args(dist, angle))
    ck = scan.cstar[angle]
    centre = funkey(KMIN) if ck is None else funkey(ck)
    grp = f"c*@{angle}" if ck is not None and KMIN <= ck < KMAX else None
    for d, c in neighbours(centre, lo=f32(-1), hi=f32(1)):
        p, q = solve_ratio(c)
        ps.add([[0, 0, 0], [1, 0, 0], [p, q, 0]], 0.0, c, "c", grp, edge=d == 0)
    return ps


def hb_distance_set(dist, angle=60.0, L=8.0, ignore_hs=False):
    """A at squared distance fl(t*t) and 1-3 floats either side from H (from D with ignore_hs), along one axis and two,
    then shifted by whole boxes on every axis; D on the far side so the angle passes."""
    ps = ProbeSet(f"hb_dist_{dist}_{int(ignore_hs)}", "hb", 3, _hb_args(dist, angle, ignore_hs))
    T2 = f32(dist) * f32(dist)
    grid = 2.0 ** -16
    for d, t in neighbours(T2):
        x, y = solve_sumsq(t, grid)
        base = [(x, y, 0), (0, x, y), (y, 0, x)]
        if d == 0:
            base.append((f32(dist), 0, 0))
        for a in base:
            a = np.asarray(a, np.float32)
            far = -np.sign(a) * (a == a.max()) * f32(1)  # one unit behind the tested atom along A's largest axis
            on_grid = np.all(np.round(a.astype(np.float64) / grid) * grid == a)  # exact after a shift by whole boxes
            for s in ((0, 0, 0),) + (SHIFTS if on_grid else ()):
                xyz = [far, [0, 0, 0], _shifted(a, s, L)] if ignore_hs else [[0, 0, 0], far, _shifted(a, s, L)]
                ps.add(xyz, L, t, "d2a", f"d2@{dist}", edge=d == 0)
    return ps


def hb_fastwrap_set(L=5.0, dist=float(np.nextafter(f32(2.5), f32(0)))):
    """Quotients v / L a few ulps from k + 0.5: wrap_fast_if flags them and hb_rewrap redoes the exact step.  The wrapped
    |v| is L / 2 exactly (too far: the threshold is the float below L / 2) at the half-integers and a few ulps less next
    to them, so both outcomes occur."""
    ps = ProbeSet("hb_fastwrap", "hb", 3, _hb_args(dist, 30.0))
    for k in range(-4, 4):
        v0 = f32((k + 0.5) * L)
        for d, v in neighbours(v0, offsets=range(-4, 5)):
            for axis in range(3):
                a = np.zeros(3, np.float32); a[axis] = v
                dd = np.zeros(3, np.float32); dd[(axis + 1) % 3] = 1
                ps.add([[0, 0, 0], dd, a], L, group="half-box", edge=d == 0)
    return ps


def hb_clamp_pairs(n=4):
    """Near-collinear D-H-A with H at the origin whose unclamped cosine rounds past 1 (A beside D) or past -1 (A opposite)."""
    rng = np.random.default_rng(7)
    A = rng.uniform(0.5, 1.4, size=(200000, 3)).astype(np.float32)
    m = rng.uniform(0.3, 0.9, size=(200000, 1)).astype(np.float32)
    out = {1: [], -1: []}
    for sgn in (1, -1):
        D = (A * m * f32(sgn)).astype(np.float32)
        c = hb_cos(A, D)
        sel = np.flatnonzero(c > 1 if sgn == 1 else c < -1)
        out[sgn] = [(A[i], D[i]) for i in sel[:n]]
    return out


def hb_cos(A, D):
    """the kernel's unclamped cosine for H at the origin (the vectors are A and D themselves)"""
    A, D = np.asarray(A, np.float32), np.asarray(D, np.float32)
    dot = ((f32(0) + A[..., 0] * D[..., 0]) + A[..., 1] * D[..., 1]) + A[..., 2] * D[..., 2]
    den = np.sqrt(sq3(A[..., 0], A[..., 1], A[..., 2])) * np.sqrt(sq3(D[..., 0], D[..., 1], D[..., 2]))
    with np.errstate(all="ignore"):
        return (dot.astype(np.float64) / den.astype(np.float64)).astype(np.float32)


def hb_special_sets():
    """cosines clamped at +-1, H on A or on D (a zero squared distance), NaN and infinite coordinates; and ignore_hs with a
    failing angle (emitted: the angle is not tested)"""
    ps = ProbeSet("hb_special", "hb", 3, _hb_args(2.5, 120.0))
    cl = hb_clamp_pairs()
    assert len(cl[1]) and len(cl[-1])
    for sgn in (1, -1):
        for A, D in cl[sgn]:
            ps.add([[0, 0, 0], D, A], 0.0, what=None)
    ps.add([[0, 0, 0], [1, 0, 0], [0, 0, 0]], 0.0)           # H on A
    ps.add([[0, 0, 0], [0, 0, 0], [-2, 0, 0]], 0.0)          # H on D
    ps.add([[0, 0, 0], [1, 0, 0], [-1, 0, 0]], 10.0)         # D-H-A straight
    for bad in (np.nan, np.inf, -np.inf):
        for atom in range(3):
            xyz = np.array([[0, 0, 0], [1, 0, 0], [-2, 0.5, 0]], np.float32)
            xyz[atom, atom % 3] = bad
            ps.add(xyz, 10.0)
    ign = ProbeSet("hb_ignore_hs", "hb", 3, _hb_args(2.5, 120.0, ignore_hs=True))
    ign.add([[0, 0, 0], [0, 0, 0], [2, 0, 0]], 0.0)          # D on A's side: the angle would fail, distance from D 2
    ign.add([[0, 0, 0], [1, 0, 0], [2, 0, 0]], 0.0)          # A 1 from D, angle 0
    ign.add([[0, 0, 0], [1, 0, 0], [4, 0, 0]], 0.0)          # too far from D
    ign.add([[0, 0, 0], [1, 0, 0], [np.nan, 0, 0]], 0.0)     # NaN distance: passes, as the reference
    return [ps, ign]


# ---- K13 ------------------------------------------------------------------------------------------------------------
# ring 1: a hexagon in z = 0 around the origin whose float sums are exact; its normal is +z, or -z with y mirrored

HEX = np.array([[2, 0, 0], [1, 2, 0], [-1, 2, 0], [-2, 0, 0], [-1, -2, 0], [1, -2, 0]], np.float32)


def hexagon(sign):
    h = HEX.copy()
    h[:, 1] *= f32(sign)
    return h


def ring_layout(kind, n2_atoms=3):
    """(n_atoms, rings_atoms, starts1, second) of the one-ring-pair probe systems: the hexagon is atoms 0..5; then pi-pi's
    second ring (n2_atoms), the cation, or the halogen and its bonded partner"""
    if kind == "pipi":
        n = 6 + n2_atoms
        return n, np.arange(n, dtype=np.uint32), np.array([0, 6], np.uint32), np.array([6, n], np.uint32)
    if kind == "cationpi":
        return 7, np.arange(6, dtype=np.uint32), np.array([0, 6], np.uint32), np.array([6], np.uint32)
    return 8, np.arange(6, dtype=np.uint32), np.array([0, 6], np.uint32), np.array([[6, 7]], np.uint32)


def ring_set(kind, name, p, n2_atoms=3):
    n, ra, st, sec = ring_layout(kind, n2_atoms)
    ps = ProbeSet(name, kind, n, dict(rings_atoms=ra, starts=st, second=sec, p=tuple(float(f32(x)) for x in p)))
    return ps


def _dot_partner(kind, sign, T):
    """atoms after the hexagon (normal `sign` z) that make the kernel's dot product exactly T"""
    p, q = solve_ratio(f32(sign) * T)
    if kind == "pipi":    # ring 2: p0 - p2 = (p, 0, q) ... normal (-q, 0, p): dot = sign * ratio(p, q)
        return [[p, 0, q], [0, 1, 0], [0, 0, 0]]
    if kind == "cationpi":  # centroid at the origin -> cation (q, 0, p)
        return [[q, 0, p]]
    return [[0, 1, 0], [-q, 1, -p]]  # halogen - partner = (q, 0, p)


def ring_angle_set(scan, kind, angle, pred):
    """probes whose dot product is each transition float of the predicate and 1-3 floats either side, both normal signs;
    the other pi-pi predicate is made empty (threshold 1000 or -1) and every distance passes"""
    if kind == "pipi":
        p = (4.4, angle, 5.5, 1000.0) if pred == LE else (4.4, -1.0, 5.5, angle)
    else:
        p = (5.0, angle)
    ps = ring_set(kind, f"{kind}_{PRED_NAMES[pred]}_{angle}", p)
    _, trs = scan.sets[(angle, pred)]
    for kt in trs:
        for d, T in neighbours(funkey(kt), lo=f32(-1), hi=f32(1)):
            for sign in (1, -1):
                xyz = np.concatenate([hexagon(sign), np.asarray(_dot_partner(kind, sign, T), np.float32)])
                ps.add(xyz, 0.0, T, "dot", f"{PRED_NAMES[pred]}@{angle}:{kt}:{sign}", edge=d == 0)
    return ps


def ring_distance_sets(L=16.0):
    """squared centroid distances fl(t*t) and 1-3 floats either side (pi-pi: around d1, around d2, and around d2 with
    d1 > d2, where `!(dist2 > d2)` passes and only `dist2 < d1` decides), two axes, shifted by whole boxes"""
    grid = 2.0 ** -14
    sets = []
    specs = [("cationpi", "cationpi_d", (4.0, 0.0), 4.0), ("sigmahole", "sigmahole_d", (3.3, 0.0), 3.3),
             ("pipi", "pipi_d1", (4.4, 90.0, 5.5, 1000.0), 4.4), ("pipi", "pipi_d2", (4.4, -1.0, 5.5, -1.0), 5.5),
             ("pipi", "pipi_d2_inner", (6.5, 90.0, 5.5, 1000.0), 5.5)]
    for kind, name, p, t in specs:
        ps = ring_set(kind, name, p, n2_atoms=6)
        T2 = f32(t) * f32(t)
        for d, target in neighbours(T2):
            x, y = solve_sumsq(target, grid)
            for off in ((x, y, 0), (0, x, y), (-y, 0, -x)):
                off = np.asarray(off, np.float32)
                for s in ((0, 0, 0),) + SHIFTS:
                    o = _shifted(off, s, L)
                    if kind == "pipi":
                        xyz = np.concatenate([hexagon(1), hexagon(1) + o])
                    elif kind == "cationpi":
                        xyz = np.concatenate([hexagon(1), o[None]])
                    else:
                        xyz = np.concatenate([hexagon(1), o[None], (o + np.float32([0.25, 0.5, 1.0]))[None]])
                    ps.add(xyz, L, target, "d2", f"{name}@{t}", edge=d == 0)
        sets.append(ps)
    return sets


def pipi_first_atom_set(L=40.0):
    """the first atoms of the two rings at squared distance 225 and 1-3 floats either side (the early exit), the centroids
    within both thresholds and every angle accepted; shifted by whole boxes"""
    ps = ring_set("pipi", "pipi_first", (10.0, 90.0, 10.0, 1000.0), n2_atoms=3)
    grid = 2.0 ** -14
    for d, target in neighbours(f32(225.0)):
        sols = [solve_sumsq(target, grid)]
        if d == 0:
            sols.append((f32(15), f32(0)))
        for x, y in sols:
            for s in ((0, 0, 0),) + SHIFTS[:3]:
                r2 = np.array([[2 + x, y, 0], [0, 0, 0], [0, 1, 0]], np.float32)
                xyz = np.concatenate([hexagon(1), _shifted(r2, s, L)])
                ps.add(xyz, L, target, "first", "first@225", edge=d == 0)
    return ps


# ---------------------------------------------------------------------------------------------------------------------
# the quantities the kernels decide on, recomputed in float32 in their order of operations

def _ring_geom(xyz, atoms):
    """centroid (float sum in atom order / count), normal from the first three atoms, first atom; xyz (N, 3, F)"""
    m = np.zeros((3, xyz.shape[2]), np.float32)
    for a in atoms:
        m = m + xyz[a]
    m = m / f32(len(atoms))
    p0, p1, p2 = xyz[atoms[0]], xyz[atoms[1]], xyz[atoms[2]]
    t1, t2 = p0 - p2, p1 - p2
    n = np.stack([t1[1] * t2[2] - t1[2] * t2[1], t1[2] * t2[0] - t1[0] * t2[2], t1[0] * t2[1] - t1[1] * t2[0]])
    with np.errstate(all="ignore"):
        n = n / np.sqrt(sq3(*n))
    return m, n, p0


def _wdist(a, b, box):
    v = a - b
    return sq3(*(wrap(v[i], box[i]) for i in range(3)))


def _dot3(a, b):
    return ((f32(0) + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]


def simulate(ps):
    """dict of per-frame float32 arrays: hb -> d2a, d2b, c (clamped); rings -> dist2, dot (+ first for pi-pi)"""
    xyz, box = ps.coords, ps.box
    if ps.kind == "hb":
        H, D, A = xyz[0], xyz[1], xyz[2]
        src = D if ps.args["ignore_hs"] else H
        with np.errstate(all="ignore"):
            a = np.stack([wrap(A[i] - src[i], box[i]) for i in range(3)])
            b = np.stack([wrap(D[i] - H[i], box[i]) for i in range(3)])
            d2a, d2b = sq3(*a), sq3(*b)
            dot = _dot3(a, b)
            c = (dot.astype(np.float64) / (np.sqrt(d2a) * np.sqrt(d2b)).astype(np.float64)).astype(np.float32)
        return dict(d2a=d2a, d2b=d2b, c=np.clip(c, -1, 1))
    ra, st, sec = ps.args["rings_atoms"], ps.args["starts"], ps.args["second"]
    m1, n1, a1 = _ring_geom(xyz, ra[st[0]:st[1]])
    with np.errstate(all="ignore"):
        if ps.kind == "pipi":
            m2, n2, a2 = _ring_geom(xyz, ra[sec[0]:sec[1]])
            return dict(first=_wdist(a1, a2, box), dist2=_wdist(m1, m2, box), dot=_dot3(n1, n2))
        pa = xyz[int(np.ravel(sec)[0])]
        t = pa - m1 if ps.kind == "cationpi" else pa - xyz[int(np.ravel(sec)[1])]
        t = t / np.sqrt(sq3(*t))
        return dict(dist2=_wdist(m1, pa, box), dot=_dot3(n1, t))


def check_construction(ps):
    """every designed value equals the simulated one, bit for bit"""
    sim = simulate(ps)
    key = {"c": "c", "dot": "dot", "d2": "dist2", "d2a": "d2a", "first": "first"}
    for f, (w, v) in enumerate(zip(ps.what, ps.value)):
        if w is not None:
            got = sim[key[w]][f]
            assert np.array_equal(np.float32(got).view(np.uint32), np.float32(v).view(np.uint32)), (ps.name, f, w, got, v)


def reference_hits(ps):
    """the reference's predicate on the simulated quantities, with libm's acosf through ctypes"""
    sim = simulate(ps)
    F = len(ps)
    out = np.zeros(F, bool)
    if ps.kind == "hb":
        a = ps.args
        thr2 = f32(a["dist_threshold"]) * f32(a["dist_threshold"])
        athr = f32(float(f32(a["angle_threshold"])) / ANGLE_SCALE)
        for f in range(F):
            d2a, d2b, c = sim["d2a"][f], sim["d2b"][f], sim["c"][f]
            if d2a > thr2:
                continue
            if a["ignore_hs"]:
                out[f] = True
            elif not (d2a == 0 or d2b == 0):
                out[f] = acosf(c) > athr  # NaN compares false
        return out
    p = [float(f32(x)) for x in ps.args["p"]]
    d1 = f32(p[0]) * f32(p[0])
    for f in range(F):
        dist2, dot = sim["dist2"][f], sim["dot"][f]
        if ps.kind == "pipi":
            d2 = f32(p[2]) * f32(p[2])
            if sim["first"][f] > f32(225) or dist2 > d2:
                continue
            ang = folded(dot)
            out[f] = bool((dist2 < d1 and ang <= p[1]) or (dist2 < d2 and ang >= p[3]))
        else:
            if dist2 > d1:
                continue
            out[f] = 90.0 - folded(dot) >= p[1]
    return out


def scan_hits(scan, ps):
    """for the angle sets: the decision read off the exhaustive sets (c <= c*, or membership of the transition set)"""
    out = np.zeros(len(ps), bool)
    if ps.kind == "hb":
        ck = scan.cstar[ps.args["angle_threshold"]]
        for f, c in enumerate(ps.value):
            out[f] = ck is not None and fkey(c) <= ck
        return out
    p = ps.args["p"]
    for f, dot in enumerate(ps.value):
        k = fkey(dot)
        if ps.kind == "pipi":
            out[f] = any(float(f32(a)) == float(f32(p[1])) and scan.member(a, LE, k) for a in K13_ANGLES) or \
                any(float(f32(a)) == float(f32(p[3])) and scan.member(a, GE, k) for a in K13_ANGLES)
        else:
            out[f] = any(float(f32(a)) == float(f32(p[1])) and scan.member(a, PLANE, k) for a in K13_ANGLES)
    return out


def angle_sets(scan):
    sets = [hb_angle_set(scan, a) for a in K12_ANGLES]
    for angle in K13_ANGLES:
        for kind, pred in (("pipi", LE), ("pipi", GE), ("cationpi", PLANE), ("sigmahole", PLANE)):
            ps = ring_angle_set(scan, kind, angle, pred)
            if len(ps):
                sets.append(ps)
    return sets


def distance_sets():
    return ([hb_distance_set(2.5), hb_distance_set(3.1, ignore_hs=True), hb_fastwrap_set()] + ring_distance_sets()
            + [pipi_first_atom_set()] + hb_special_sets())


# ---------------------------------------------------------------------------------------------------------------------
# running a probe set

def call(ps, mod):
    """run `ps` through `mod` (the oracle module, or None for the device): hb -> per-frame flat triples;
    rings -> (per-frame flat pairs, per-frame flat (distance, angle))"""
    xyz, box = ps.coords, ps.box
    a = ps.args
    if ps.kind == "hb":
        if mod is None:
            from moleculekit_b200 import hbonds
            return hbonds.calculate(a["donors"], a["acceptors"], xyz, box, a["sel1"], a["sel2"],
                                    dist_threshold=a["dist_threshold"], angle_threshold=a["angle_threshold"],
                                    intra=a["intra"], ignore_hs=a["ignore_hs"])
        return mod.hbonds_calculate(a["donors"], a["acceptors"], xyz, box, a["sel1"], a["sel2"], a["dist_threshold"],
                                    a["angle_threshold"], a["intra"], a["ignore_hs"])
    mode = {"pipi": 0, "cationpi": 1, "sigmahole": 2}[ps.kind]
    args = (a["rings_atoms"], a["starts"], a["second"], xyz, box, *a["p"])
    if mod is None:
        from moleculekit_b200 import ringpairs
        return (ringpairs.pipi_calculate, ringpairs.cationpi_calculate, ringpairs.sigmahole_calculate)[mode](*args)
    return mod.ring_interactions(mode, *args)


def hits_of(ps, res):
    return np.array([len(x) > 0 for x in (res if ps.kind == "hb" else res[0])])
