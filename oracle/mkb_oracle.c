/*
 * mkb_oracle.c -- CPU restatement of the moleculekit voxel/distance hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and the cpu_baseline /
 * --impl reference legs of bench.py may load this library.  The product path
 * (moleculekit_b200/) never links, imports or calls it and has no CPU fallback.
 *
 * Parity is PINNED: tests/test_oracle_golden.py checks every function below bit-for-bit against the
 * reference's own Cython kernels compiled from /root/reference (oracle/_ref, see
 * oracle/build_ref.py) and against the reference's golden vectors (tests/golden/).
 *
 * Each function cites the reference file:line it restates (paths relative to
 * /root/reference/moleculekit/).  Arithmetic notes that matter for bit parity:
 *   - occupancy is all-double (coords are float, promoted), strict "< 25" gate, "value > old"
 *     update (NaN never stored), sigma == 0 skipped.
 *   - distances are all-float with every operation individually rounded (x86-64 baseline has
 *     no FMA; compile this file with -ffp-contract=off), roundf = half away from zero.
 * Build: gcc -O3 -ffp-contract=off -fno-fast-math -shared -fPIC mkb_oracle.c -o libmkb_oracle.so -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EXPORT __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * occupancy_utils/occupancy_utils.pyx:34-61  calculate_occupancy
 * centers (M,3) f64, coords (N,3) f32, sigmas (N,C) f64, results (M,C) f64 accumulated in place.
 * ------------------------------------------------------------------------------------------ */
EXPORT void oracle_calculate_occupancy(const double *centers, const float *coords,
                                       const double *sigmas, double *results,
                                       int64_t n_centers, int64_t n_atoms, int64_t n_channels)
{
    for (int64_t a = 0; a < n_atoms; ++a) {
        const double ax = (double)coords[3 * a + 0];
        const double ay = (double)coords[3 * a + 1];
        const double az = (double)coords[3 * a + 2];
        const double *sig = sigmas + a * n_channels;
        for (int64_t c = 0; c < n_centers; ++c) {
            const double dx = ax - centers[3 * c + 0];
            const double dy = ay - centers[3 * c + 1];
            const double dz = az - centers[3 * c + 2];
            const double d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < 25.0) {
                double *res = results + c * n_channels;
                for (int64_t h = 0; h < n_channels; ++h) {
                    if (sig[h] == 0.0) continue;
                    const double x = sig[h] / sqrt(d2);
                    const double x3 = (x * x) * x;
                    const double x12 = ((x3 * x3) * x3) * x3;
                    const double v = 1.0 - exp(-x12);
                    if (v > res[h]) res[h] = v;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * distance_utils/distance_utils.pyx:34-54  _dist  (frame-minor coords (N,3,F), box (3,F))
 * ------------------------------------------------------------------------------------------ */
static inline float wrap1(float d, float b)
{
    /* d - b * roundf(d / b), each op rounded to float (pyx:50-52) */
    float q = d / b;
    float n = roundf(q);
    float p = b * n;
    return d - p;
}

static inline float pair_d2(const float *coords, const float *box, const uint32_t *chains,
                            int64_t F, int64_t i, int64_t j, int64_t f, int pbc)
{
    float dx = coords[(i * 3 + 0) * F + f] - coords[(j * 3 + 0) * F + f];
    float dy = coords[(i * 3 + 1) * F + f] - coords[(j * 3 + 1) * F + f];
    float dz = coords[(i * 3 + 2) * F + f] - coords[(j * 3 + 2) * F + f];
    if (pbc && chains[i] != chains[j]) {
        dx = wrap1(dx, box[0 * F + f]);
        dy = wrap1(dy, box[1 * F + f]);
        dz = wrap1(dz, box[2 * F + f]);
    }
    float s = dx * dx;
    s = s + dy * dy;
    s = s + dz * dz;
    return s;
}

/* distance_utils.pyx:126-155  dist_trajectory: results (F, P) f32, i-major / j-minor columns,
 * selfdist starts j at i+1 (positions, not atom ids). */
EXPORT void oracle_dist_trajectory(const float *coords, const float *box,
                                   const uint32_t *sel1, int64_t n1,
                                   const uint32_t *sel2, int64_t n2,
                                   const uint32_t *chains, int selfdist, int pbc,
                                   float *results, int64_t n_frames, int64_t n_cols)
{
    for (int64_t f = 0; f < n_frames; ++f) {
        int64_t idx = 0;
        for (int64_t i = 0; i < n1; ++i) {
            const int64_t a = sel1[i];
            for (int64_t j = selfdist ? i + 1 : 0; j < n2; ++j) {
                const float d2 = pair_d2(coords, box, chains, n_frames, a, sel2[j], f, pbc);
                results[f * n_cols + idx] = sqrtf(d2);
                ++idx;
            }
        }
    }
}

/* distance_utils.pyx:59-93  contacts_trajectory.  Two-call protocol: pairs == NULL -> only
 * counts[f] (number of PAIRS of frame f) is written; else pairs receives (a, b) uint32 couples,
 * frames concatenated, in (i asc, j asc) order.  thr2 = thr * thr in float (pyx:77). */
EXPORT int64_t oracle_contacts_trajectory(const float *coords, const float *box,
                                          const uint32_t *sel1, int64_t n1,
                                          const uint32_t *sel2, int64_t n2,
                                          const uint32_t *chains, int selfdist, int pbc,
                                          float threshold, int64_t n_frames,
                                          int64_t *counts, uint32_t *pairs)
{
    const float thr2 = threshold * threshold;
    int64_t total = 0;
    for (int64_t f = 0; f < n_frames; ++f) {
        int64_t cnt = 0;
        for (int64_t i = 0; i < n1; ++i) {
            const uint32_t a = sel1[i];
            for (int64_t j = selfdist ? i + 1 : 0; j < n2; ++j) {
                const uint32_t b = sel2[j];
                const float d2 = pair_d2(coords, box, chains, n_frames, a, b, f, pbc);
                if (d2 <= thr2) {
                    if (pairs) {
                        pairs[2 * (total + cnt) + 0] = a;
                        pairs[2 * (total + cnt) + 1] = b;
                    }
                    ++cnt;
                }
            }
        }
        if (counts) counts[f] = cnt;
        total += cnt;
    }
    return total;
}

/* distance_utils.pyx:98-121  get_collisions: single frame, no pbc, LOCAL (i, j) indices. */
EXPORT int64_t oracle_get_collisions(const float *c1, int64_t n1, const float *c2, int64_t n2,
                                     float threshold, uint32_t *pairs)
{
    const float thr2 = threshold * threshold;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n1; ++i)
        for (int64_t j = 0; j < n2; ++j) {
            const float dx = c1[3 * i + 0] - c2[3 * j + 0];
            const float dy = c1[3 * i + 1] - c2[3 * j + 1];
            const float dz = c1[3 * i + 2] - c2[3 * j + 2];
            float s = dx * dx;
            s = s + dy * dy;
            s = s + dz * dz;
            if (s <= thr2) {
                if (pairs) {
                    pairs[2 * cnt + 0] = (uint32_t)i;
                    pairs[2 * cnt + 1] = (uint32_t)j;
                }
                ++cnt;
            }
        }
    return cnt;
}

/* distance_utils.pyx:160-183  _calc_com: float accumulation in atom order, mul then add. */
static void calc_com(const float *coords, int64_t F, int64_t f, const int32_t *atoms, int64_t n,
                     const float *masses, float *com)
{
    float tm = 0.f, cx = 0.f, cy = 0.f, cz = 0.f;
    for (int64_t k = 0; k < n; ++k) {
        const int64_t a = atoms[k];
        const float m = masses[a];
        float t;
        t = coords[(a * 3 + 0) * F + f] * m; cx = cx + t;
        t = coords[(a * 3 + 1) * F + f] * m; cy = cy + t;
        t = coords[(a * 3 + 2) * F + f] * m; cz = cz + t;
        tm = tm + m;
    }
    com[0] = cx / tm;
    com[1] = cy / tm;
    com[2] = cz / tm;
}

/* distance_utils.pyx:188-206  _dist2 on two explicit points */
static inline float point_d2(const float *p, const float *q, const float *box, int wrap)
{
    float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
    if (wrap) {
        dx = wrap1(dx, box[0]);
        dy = wrap1(dy, box[1]);
        dz = wrap1(dz, box[2]);
    }
    float s = dx * dx;
    s = s + dy * dy;
    s = s + dz * dz;
    return s;
}

static float group_pair(const float *coords, int64_t F, int64_t f, const float *bx,
                        const int32_t *g1, int64_t m1, const int32_t *g2, int64_t m2,
                        const float *masses, int red1, int red2, int wrap)
{
    /* pyx:240-279 inner body: COM side collapses to one pseudo atom; mindist=-1 sentinel. */
    float com1[3], com2[3];
    if (red1 == 1) calc_com(coords, F, f, g1, m1, masses, com1);
    if (red2 == 1) calc_com(coords, F, f, g2, m2, masses, com2);
    const int64_t l1 = (red1 == 1) ? 1 : m1;
    const int64_t l2 = (red2 == 1) ? 1 : m2;
    float mind = -1.f;
    for (int64_t a = 0; a < l1; ++a) {
        float p[3];
        if (red1 == 1) { p[0] = com1[0]; p[1] = com1[1]; p[2] = com1[2]; }
        else { const int64_t x = g1[a]; p[0] = coords[(x*3+0)*F+f]; p[1] = coords[(x*3+1)*F+f]; p[2] = coords[(x*3+2)*F+f]; }
        for (int64_t b = 0; b < l2; ++b) {
            float q[3];
            if (red2 == 1) { q[0] = com2[0]; q[1] = com2[1]; q[2] = com2[2]; }
            else { const int64_t y = g2[b]; q[0] = coords[(y*3+0)*F+f]; q[1] = coords[(y*3+1)*F+f]; q[2] = coords[(y*3+2)*F+f]; }
            const float d2 = point_d2(p, q, bx, wrap);
            if (d2 < mind || mind < 0.f) mind = d2;
        }
    }
    return sqrtf(mind);
}

/* distance_utils.pyx:211-281  dist_trajectory_reduction.  Groups are CSR: off (G+1), atoms. */
EXPORT void oracle_dist_trajectory_reduction(const float *coords, const float *box,
                                             const int64_t *off1, const int32_t *atoms1, int64_t G1,
                                             const int64_t *off2, const int32_t *atoms2, int64_t G2,
                                             const uint32_t *chains1, const uint32_t *chains2,
                                             int selfdist, int pbc, const float *masses,
                                             int red1, int red2, float *results,
                                             int64_t n_frames, int64_t n_cols)
{
    for (int64_t f = 0; f < n_frames; ++f) {
        const float bx[3] = { box[0 * n_frames + f], box[1 * n_frames + f], box[2 * n_frames + f] };
        int64_t idx = 0;
        for (int64_t a = 0; a < G1; ++a)
            for (int64_t b = selfdist ? a + 1 : 0; b < G2; ++b) {
                const int wrap = pbc && (chains1[a] != chains2[b]);
                results[f * n_cols + idx] = group_pair(coords, n_frames, f, bx,
                        atoms1 + off1[a], off1[a + 1] - off1[a],
                        atoms2 + off2[b], off2[b + 1] - off2[b], masses, red1, red2, wrap);
                ++idx;
            }
    }
}

/* distance_utils.pyx:286-350  dist_trajectory_reduction_pairs (group g of set 1 vs group g of set 2) */
EXPORT void oracle_dist_trajectory_reduction_pairs(const float *coords, const float *box,
                                                   const int64_t *off1, const int32_t *atoms1,
                                                   const int64_t *off2, const int32_t *atoms2, int64_t G,
                                                   const uint32_t *chains1, const uint32_t *chains2,
                                                   int pbc, const float *masses,
                                                   int red1, int red2, float *results,
                                                   int64_t n_frames, int64_t n_cols)
{
    for (int64_t f = 0; f < n_frames; ++f) {
        const float bx[3] = { box[0 * n_frames + f], box[1 * n_frames + f], box[2 * n_frames + f] };
        for (int64_t g = 0; g < G; ++g) {
            const int wrap = pbc && (chains1[g] != chains2[g]);
            results[f * n_cols + g] = group_pair(coords, n_frames, f, bx,
                    atoms1 + off1[g], off1[g + 1] - off1[g],
                    atoms2 + off2[g], off2[g + 1] - off2[g], masses, red1, red2, wrap);
        }
    }
}

/* distance_utils.pyx:355-383  cdist: float accumulate over D in index order, sqrtf */
EXPORT void oracle_cdist(const float *c1, int64_t n1, const float *c2, int64_t n2, int64_t D, float *out)
{
    for (int64_t i = 0; i < n1; ++i)
        for (int64_t j = 0; j < n2; ++j) {
            float s = 0.f;
            for (int64_t k = 0; k < D; ++k) {
                const float d = c1[i * D + k] - c2[j * D + k];
                s = s + d * d;
            }
            out[i * n2 + j] = sqrtf(s);
        }
}

/* distance_utils.pyx:388-416  pdist: condensed i<j */
EXPORT void oracle_pdist(const float *c, int64_t n, int64_t D, float *out)
{
    int64_t t = 0;
    for (int64_t i = 0; i < n; ++i)
        for (int64_t j = i + 1; j < n; ++j) {
            float s = 0.f;
            for (int64_t k = 0; k < D; ++k) {
                const float d = c[i * D + k] - c[j * D + k];
                s = s + d * d;
            }
            out[t++] = sqrtf(s);
        }
}

/* distance_utils.pyx:421-435  squareform: n' = int((sqrt(8n+1)+1)/2), symmetric fill */
EXPORT int64_t oracle_squareform_dim(int64_t n)
{
    return (int64_t)((sqrt((double)(8 * n + 1)) + 1.0) / 2.0);
}

EXPORT void oracle_squareform(const float *d, int64_t n, float *out)
{
    const int64_t m = oracle_squareform_dim(n);
    memset(out, 0, sizeof(float) * (size_t)(m * m));
    int64_t k = 0;
    for (int64_t i = 0; i < m; ++i)
        for (int64_t j = i + 1; j < m; ++j) {
            out[i * m + j] = d[k];
            out[j * m + i] = d[k];
            ++k;
        }
}

/* ------------------------------------------------------------------------------------------
 * Row a13 (stretch): bond guessing on a uniform non-periodic grid.
 * bondguesser.py:259-392 (bond_grid_search: binning, traversal) +
 * bondguesser_utils/bondguesser_utils.pyx:30-85 (14-entry half-shell neighbour table),
 * :89-115 (_is_close), :119-163 (grid_bonds).
 * coords (N,3) f32, radii (N) f32, is_hydrogen (N) u32, pairdist = final grid box edge (after the max_boxes
 * enlargement loop, done by the caller).  pairs == NULL -> count only.  Output order = the reference's:
 * boxes in order of first appearance (dict insertion order, :357-388), atoms of a box in index order,
 * neighbour boxes in table order, (i, j) as emitted (not canonicalised).
 * ------------------------------------------------------------------------------------------ */
static int is_close(const float *c, const float *radii, const uint32_t *is_h, int64_t i, int64_t j, float cutoff2)
{
    if (is_h[i] && is_h[j]) return 0;
    const float dx = c[3 * i + 0] - c[3 * j + 0];
    const float dy = c[3 * i + 1] - c[3 * j + 1];
    const float dz = c[3 * i + 2] - c[3 * j + 2];
    float d2 = dx * dx;
    d2 = d2 + dy * dy;
    d2 = d2 + dz * dz;
    if (d2 > cutoff2 || (double)d2 < 0.001) return 0;      /* pyx:106: float vs double literal */
    const float cut = (float)(0.6 * (double)(radii[i] + radii[j]));   /* pyx:109: 0.6 is a double literal */
    if (d2 > cut * cut) return 0;
    return 1;
}

EXPORT int64_t oracle_bond_grid_search(const float *coords, const float *radii, const uint32_t *is_h,
                                       int64_t n, double pairdist, uint32_t *pairs)
{
    if (n <= 0) return 0;
    float mn[3], mx[3];
    for (int d = 0; d < 3; ++d) { mn[d] = coords[d]; mx[d] = coords[d]; }
    for (int64_t a = 1; a < n; ++a)
        for (int d = 0; d < 3; ++d) {
            const float v = coords[3 * a + d];
            if (v < mn[d]) mn[d] = v;
            if (v > mx[d]) mx[d] = v;
        }
    /* numpy: xyzrange f32; xyzrange / pairdist with a python float keeps f32 (weak scalar), floor, +1 */
    const float pdf = (float)pairdist;
    int64_t nb[3];
    for (int d = 0; d < 3; ++d) nb[d] = (int64_t)floorf((mx[d] - mn[d]) / pdf) + 1;
    const int64_t nboxes = nb[0] * nb[1] * nb[2], xy = nb[0] * nb[1];
    int64_t *box = (int64_t *)malloc(sizeof(int64_t) * (size_t)n);
    int64_t *cnt = (int64_t *)calloc((size_t)nboxes + 1, sizeof(int64_t));
    int64_t *first = (int64_t *)malloc(sizeof(int64_t) * (size_t)nboxes);   /* first atom of each box */
    for (int64_t b = 0; b < nboxes; ++b) first[b] = -1;
    for (int64_t a = 0; a < n; ++a) {
        int64_t bi[3];
        for (int d = 0; d < 3; ++d) {
            int64_t v = (int64_t)floorf((coords[3 * a + d] - mn[d]) / pdf);
            if (v < 0) v = 0;
            if (v > nb[d] - 1) v = nb[d] - 1;
            bi[d] = v;
        }
        box[a] = bi[2] * xy + bi[1] * nb[0] + bi[0];
        if (first[box[a]] < 0) first[box[a]] = a;
        cnt[box[a] + 1]++;
    }
    for (int64_t b = 0; b < nboxes; ++b) cnt[b + 1] += cnt[b];          /* cnt = start offsets */
    int64_t *members = (int64_t *)malloc(sizeof(int64_t) * (size_t)n);
    int64_t *cur = (int64_t *)malloc(sizeof(int64_t) * (size_t)nboxes);
    memcpy(cur, cnt, sizeof(int64_t) * (size_t)nboxes);
    for (int64_t a = 0; a < n; ++a) members[cur[box[a]]++] = a;           /* index order inside a box */
    const float cutoff2 = pdf * pdf;                                       /* pyx:136: float product */
    int64_t total = 0;
    /* boxes in order of first appearance == order of their first atom */
    for (int64_t a0 = 0; a0 < n; ++a0) {
        const int64_t b = box[a0];
        if (first[b] != a0) continue;
        const int64_t zi = b / xy, yi = (b % xy) / nb[0], xi = b % nb[0];
        int64_t neigh[14];
        int m = 0;
        const int xr = xi < nb[0] - 1, yr = yi < nb[1] - 1, zr = zi < nb[2] - 1, xl = xi > 0, yl = yi > 0;
        neigh[m++] = b;                                                   /* pyx:44-84, same order */
        if (xr) neigh[m++] = b + 1;
        if (yr) neigh[m++] = b + nb[0];
        if (zr) neigh[m++] = b + xy;
        if (xr && yr) neigh[m++] = b + nb[0] + 1;
        if (xr && zr) neigh[m++] = b + xy + 1;
        if (yr && zr) neigh[m++] = b + xy + nb[0];
        if (xr && yl) neigh[m++] = b - nb[0] + 1;
        if (xl && zr) neigh[m++] = b + xy - 1;
        if (yl && zr) neigh[m++] = b + xy - nb[0];
        if (xr && yr && zr) neigh[m++] = b + xy + nb[0] + 1;
        if (xl && yr && zr) neigh[m++] = b + xy + nb[0] - 1;
        if (xr && yl && zr) neigh[m++] = b + xy - nb[0] + 1;
        if (xl && yl && zr) neigh[m++] = b + xy - nb[0] - 1;
        for (int64_t ii = cnt[b]; ii < cnt[b + 1]; ++ii) {
            const int64_t i = members[ii];
            for (int k = 0; k < m; ++k) {
                const int64_t nbx = neigh[k];
                for (int64_t jj = (nbx == b) ? ii + 1 : cnt[nbx]; jj < cnt[nbx + 1]; ++jj) {
                    const int64_t j = members[jj];
                    if (is_close(coords, radii, is_h, i, j, cutoff2)) {
                        if (pairs) { pairs[2 * total] = (uint32_t)i; pairs[2 * total + 1] = (uint32_t)j; }
                        ++total;
                    }
                }
            }
        }
    }
    free(box); free(cnt); free(first); free(members); free(cur);
    return total;
}

/* ------------------------------------------------------------------------------------------------
 * wrap_box -- moleculekit/wrapping/wrapping.pyx:91-144 (orthorhombic wrapping, SURVEY 8f row 4).
 * coords (n_atoms, 3, F) frame-minor float32, modified in place; box (3, F); groups [n_groups] are the
 * first-atom offsets of consecutive bonded groups (group g = atoms [groups[g], groups[g+1])), the last
 * entry closes the last group (pyx:123-125).  Centre of the box: running mean over centersel
 * (pyx:113-118) or `center` when centersel is empty (pyx:106-108).  A group is translated along an
 * axis by box*round(diff/box) when its running-mean centre is more than half a box from the box
 * centre (pyx:137-142).  All arithmetic float32, one rounding per operation.
 * ------------------------------------------------------------------------------------------------ */
EXPORT void oracle_wrap_box(const uint32_t *groups, int64_t n_groups, float *coords, const float *box,
                            int64_t F, const uint32_t *centersel, int64_t n_centersel, const float *center)
{
    float box_center[3] = {0.f, 0.f, 0.f}, half_box[3], grp_center[3];
    if (n_centersel == 0)
        for (int i = 0; i < 3; ++i) box_center[i] = center[i];
    for (int64_t f = 0; f < F; ++f) {
        if (n_centersel > 0) {
            for (int i = 0; i < 3; ++i) box_center[i] = 0.f;
            for (int64_t n = 0; n < n_centersel; ++n)
                for (int i = 0; i < 3; ++i) {
                    const float x = coords[((int64_t)centersel[n] * 3 + i) * F + f];
                    box_center[i] = box_center[i] + (x - box_center[i]) / (float)(n + 1);
                }
        }
        for (int i = 0; i < 3; ++i) half_box[i] = box[i * F + f] / 2.f;
        for (int64_t g = 0; g + 1 < n_groups; ++g) {
            const int64_t s = groups[g], e = groups[g + 1];
            for (int i = 0; i < 3; ++i) grp_center[i] = 0.f;
            int64_t n = 0;
            for (int64_t k = s; k < e; ++k, ++n)
                for (int i = 0; i < 3; ++i)
                    grp_center[i] = grp_center[i] + (coords[(k * 3 + i) * F + f] - grp_center[i]) / (float)(n + 1);
            for (int i = 0; i < 3; ++i) {
                const float diff = grp_center[i] - box_center[i];
                if (fabsf(diff) > half_box[i]) {
                    const float b = box[i * F + f];
                    const float translation = b * roundf(diff / b);
                    for (int64_t a = s; a < e; ++a) coords[(a * 3 + i) * F + f] = coords[(a * 3 + i) * F + f] - translation;
                }
            }
        }
    }
}

/* ------------------------------------------------------------------------------------------------
 * within_distance -- moleculekit/atomselect_utils/atomselect_utils.pyx:612-653 (the kernel of the
 * `within` / `exwithin` atom selections, atomselect/atomselect.py:231-254; SURVEY 8f row 3).
 * results[ii] is SET (never cleared) when some sel2 atom j has
 *   ((0 + dx*dx) + dy*dy) + dz*dz < cutoff*cutoff      -- all float32, strict '<'
 * (the generated C calls powf(d, 2.0), which the compiler folds to d*d; pinned against the binary).
 * The reference's bounding-box pre-check (pyx:632-643) passes for every finite coordinate and a NaN
 * coordinate can never satisfy the distance test either, so it does not influence the result.
 * ------------------------------------------------------------------------------------------------ */
EXPORT void oracle_within_distance(const float *coords, float cutoff, const uint32_t *sel1, int64_t n1,
                                   const uint32_t *sel2, int64_t n2, uint8_t *results)
{
    const float sq = cutoff * cutoff;
    for (int64_t ii = 0; ii < n1; ++ii) {
        const float *a = coords + 3 * (int64_t)sel1[ii];
        for (int64_t jj = 0; jj < n2; ++jj) {
            const float *b = coords + 3 * (int64_t)sel2[jj];
            float diff = 0.f;
            for (int k = 0; k < 3; ++k) {
                const float d = a[k] - b[k];
                diff = diff + d * d;
            }
            if (diff < sq) { results[ii] = 1; break; }
        }
    }
}

/* ------------------------------------------------------------------------------------------------
 * XTC compressed-coordinate decoding (SURVEY 8f row 4, second half) -- the algorithm of
 * xdrfile_decompress_coord_float, moleculekit/fileformats/xtc/src/xdrfile.cpp:750-982 (the xdrfile / GROMACS "xdr3dfcoord"
 * format), restated on a big-integer type instead of the reference's byte arrays:
 *   bit stream, most significant bit first (decodebits, :637-670);
 *   a group of 3 small integers is one mixed-radix number stored in 8-bit chunks, least significant chunk first
 *   (decodeints, :681-729): value = sum_j chunk_j * 256^j, nums[2] = value % sizes[2], nums[1] = (value / sizes[2]) % sizes[1],
 *   nums[0] = value / (sizes[1] sizes[2]);
 *   per atom: full-range triple (+ minint), 1 flag bit, optional 5-bit run/adapt code, then run/3 atoms coded relative to the
 *   previous one with the current small size magicints[smallidx]; the first atom of a run is swapped with its predecessor
 *   (:906-925: water oxygen/hydrogen order); output = (float)int * inv_precision with inv_precision = (float)(1.0 / precision).
 * One frame's coordinate block (after the `lsize` word) is decoded; returns 0 or a negative error.
 * ------------------------------------------------------------------------------------------------ */
static const int xtc_magic[] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 8, 10, 12, 16, 20, 25, 32, 40, 50, 64, 80, 101, 128, 161, 203, 256, 322,
    406, 512, 645, 812, 1024, 1290, 1625, 2048, 2580, 3250, 4096, 5060, 6501, 8192, 10321, 13003, 16384, 20642, 26007, 32768, 41285,
    52015, 65536, 82570, 104031, 131072, 165140, 208063, 262144, 330280, 416127, 524287, 660561, 832255, 1048576, 1321122, 1664510,
    2097152, 2642245, 3329021, 4194304, 5284491, 6658042, 8388607, 10568983, 13316085, 16777216};
#define XTC_FIRSTIDX 9
#define XTC_LASTIDX ((int)(sizeof(xtc_magic) / sizeof(xtc_magic[0])))

typedef struct { const uint8_t *p; int64_t nbytes; int64_t pos; /* bit position */ } xtc_bits;

static uint32_t xtc_take(xtc_bits *b, int n)  /* n <= 32 bits, MSB first; bits past the end read as 0 */
{
    uint64_t v = 0;
    for (int k = 0; k < n; ++k) {
        const int64_t byte = b->pos >> 3;
        const int bit = byte < b->nbytes ? (b->p[byte] >> (7 - (b->pos & 7))) & 1 : 0;
        v = (v << 1) | (uint64_t)bit;
        ++b->pos;
    }
    return (uint32_t)v;
}

static void xtc_take3(xtc_bits *b, int nbits, const uint32_t sizes[3], int32_t nums[3])
{
    unsigned __int128 v = 0;
    int shift = 0;
    while (nbits > 8) { v |= (unsigned __int128)xtc_take(b, 8) << shift; shift += 8; nbits -= 8; }
    if (nbits > 0) v |= (unsigned __int128)xtc_take(b, nbits) << shift;
    nums[2] = (int32_t)(v % sizes[2]); v /= sizes[2];
    nums[1] = (int32_t)(v % sizes[1]); v /= sizes[1];
    nums[0] = (int32_t)(uint32_t)v;
}

static int xtc_bits_of(uint32_t size)  /* xdrfile.cpp:455-465 */
{
    int n = 0;
    uint64_t num = 1;
    while (size >= num && n < 32) { ++n; num <<= 1; }
    return n;
}

static int xtc_bits_of3(const uint32_t sizes[3])  /* xdrfile.cpp:480-510: bits of sizes[0]*sizes[1]*sizes[2] */
{
    unsigned __int128 prod = (unsigned __int128)sizes[0] * sizes[1] * sizes[2];
    /* the reference counts whole low bytes plus the bits of the top byte (value >= num loop, so an exact power of two
       gets one extra bit) */
    int nbytes = 0;
    unsigned __int128 t = prod;
    while (t > 0xff) { t >>= 8; ++nbytes; }
    int nb = 0;
    unsigned num = 1;
    while ((unsigned)t >= num) { ++nb; num *= 2; }
    return nb + nbytes * 8;
}

EXPORT int oracle_xtc_decode_block(const uint8_t *data, int64_t nbytes, int64_t natoms, float precision, const int32_t minint[3],
                                   const int32_t maxint[3], int32_t smallidx, float *out /* [natoms*3] */)
{
    uint32_t sizeint[3], bitsizeint[3] = {0, 0, 0};
    for (int d = 0; d < 3; ++d) {
        sizeint[d] = (uint32_t)maxint[d] - (uint32_t)minint[d] + 1u;  /* modulo 2^32: ranges >= 2^31 overflow int */
        if (!sizeint[d]) return -2;
    }
    int bitsize;
    if ((sizeint[0] | sizeint[1] | sizeint[2]) > 0xffffff) {
        for (int d = 0; d < 3; ++d) bitsizeint[d] = (uint32_t)xtc_bits_of(sizeint[d]);
        bitsize = 0;
    } else {
        bitsize = xtc_bits_of3(sizeint);
    }
    if (smallidx < XTC_FIRSTIDX || smallidx >= XTC_LASTIDX) return -3;
    int tmp = smallidx - 1;
    if (tmp < XTC_FIRSTIDX) tmp = XTC_FIRSTIDX;
    int smaller = xtc_magic[tmp] / 2, smallnum = xtc_magic[smallidx] / 2;
    uint32_t sizesmall[3] = {(uint32_t)xtc_magic[smallidx], (uint32_t)xtc_magic[smallidx], (uint32_t)xtc_magic[smallidx]};
    const float inv_precision = (float)(1.0 / precision);
    xtc_bits b = {data, nbytes, 0};
    int64_t i = 0, w = 0;
    int run = 0;
    while (i < natoms) {
        int32_t cur[3], prev[3];
        if (bitsize == 0) {
            for (int d = 0; d < 3; ++d) cur[d] = (int32_t)xtc_take(&b, (int)bitsizeint[d]);
        } else {
            xtc_take3(&b, bitsize, sizeint, cur);
        }
        ++i;
        for (int d = 0; d < 3; ++d) { cur[d] = (int32_t)((uint32_t)cur[d] + (uint32_t)minint[d]); prev[d] = cur[d]; }
        int is_smaller = 0;
        if (xtc_take(&b, 1)) {
            run = (int)xtc_take(&b, 5);
            is_smaller = run % 3;
            run -= is_smaller;
            --is_smaller;
        }
        if (run > 0) {
            for (int k = 0; k < run; k += 3) {
                int32_t s[3];
                xtc_take3(&b, smallidx, sizesmall, s);
                ++i;
                for (int d = 0; d < 3; ++d) s[d] = (int32_t)((uint32_t)s[d] + (uint32_t)prev[d] - (uint32_t)smallnum);
                if (k == 0) {  /* the first atom of the run goes BEFORE the atom it was coded against */
                    if (w + 3 > natoms * 3) return -4;
                    for (int d = 0; d < 3; ++d) { out[w++] = (float)s[d] * inv_precision; prev[d] = s[d]; }
                    for (int d = 0; d < 3; ++d) s[d] = cur[d];
                } else {
                    for (int d = 0; d < 3; ++d) prev[d] = s[d];
                }
                if (w + 3 > natoms * 3) return -4;
                for (int d = 0; d < 3; ++d) out[w++] = (float)s[d] * inv_precision;
            }
        } else {
            if (w + 3 > natoms * 3) return -4;
            for (int d = 0; d < 3; ++d) out[w++] = (float)cur[d] * inv_precision;
        }
        smallidx += is_smaller;
        if (is_smaller < 0) {
            smallnum = smaller;
            smaller = smallidx > XTC_FIRSTIDX ? xtc_magic[smallidx - 1] / 2 : 0;
        } else if (is_smaller > 0) {
            smaller = smallnum;
            smallnum = xtc_magic[smallidx] / 2;
        }
        if (smallidx < 0 || smallidx >= XTC_LASTIDX || !xtc_magic[smallidx]) return -3;
        sizesmall[0] = sizesmall[1] = sizesmall[2] = (uint32_t)xtc_magic[smallidx];
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------
 * Triclinic / compact wrapping -- moleculekit/wrapping/wrapping.pyx:147-344 (Molecule.wrap for cells
 * with a box angle != 90, moleculekit/molecule.py:2078-2090).  coords (n_atoms, 3, F) float32 frame
 * minor, in place; boxvectors (3, 3, F) float64, row i = box vector i.  The reference mixes float32
 * state (wrap_center, box_middle, grp_center) with float64 box arithmetic; every assignment below keeps
 * the C type the generated code has (float op float -> float, float op double -> double, rounded to
 * float on store).  The running means are as in wrap_box.
 * ------------------------------------------------------------------------------------------------ */
static void tric_frame_setup(const double *bv, int64_t F, int64_t f, float *coords, int64_t n_atoms,
                             const uint32_t *centersel, int64_t n_centersel, float wrap_center[3],
                             double box[3][3], float box_middle[3])
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) box[i][j] = bv[(i * 3 + j) * F + f];
    if (n_centersel > 0) {                                                    /* pyx:180-185 / 271-276 */
        for (int i = 0; i < 3; ++i) wrap_center[i] = 0.f;
        for (int64_t n = 0; n < n_centersel; ++n)
            for (int i = 0; i < 3; ++i) {
                const float x = coords[((int64_t)centersel[n] * 3 + i) * F + f];
                wrap_center[i] = wrap_center[i] + (x - wrap_center[i]) / (float)(n + 1);
            }
    }
    for (int i = 0; i < 3; ++i) box_middle[i] = 0.f;                          /* pyx:187-191 / 278-282 */
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) box_middle[j] = (float)((double)box_middle[j] + 0.5 * box[i][j]);
    (void)n_atoms;
}

/* pyx:147-250 wrap_triclinic_unitcell.  The while loops of the reference never end for a box whose
 * diagonal element is <= 0 while the centre is outside; `max_iter` bounds them here (the GPU kernel
 * uses the same bound) -- inputs that reach it have no reference result. */
EXPORT void oracle_wrap_triclinic(const uint32_t *groups, int64_t n_groups, float *coords, int64_t n_atoms,
                                  const double *boxvectors, int64_t F, const uint32_t *centersel,
                                  int64_t n_centersel, const float *center, int64_t max_iter)
{
    float wrap_center[3] = {0.f, 0.f, 0.f}, box_middle[3], grp_center[3], grp_center_init[3] = {0.f, 0.f, 0.f};
    double box[3][3], shift_center[3];
    if (n_centersel == 0)
        for (int i = 0; i < 3; ++i) wrap_center[i] = center[i];
    for (int64_t f = 0; f < F; ++f) {
        tric_frame_setup(boxvectors, F, f, coords, n_atoms, centersel, n_centersel, wrap_center, box, box_middle);
        const double shm01 = box[1][0] / box[1][1];                           /* pyx:198-200 */
        const double shm02 = (box[1][1] * box[2][0] - box[2][1] * box[1][0]) / (box[1][1] * box[2][2]);
        const double shm12 = box[2][1] / box[2][2];
        for (int i = 0; i < 3; ++i) shift_center[i] = 0.0;                    /* pyx:203-213 */
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) shift_center[j] = shift_center[j] + box[i][j];
        for (int i = 0; i < 3; ++i) shift_center[i] = shift_center[i] * 0.5;
        for (int i = 0; i < 3; ++i) shift_center[i] = (double)box_middle[i] - shift_center[i];
        shift_center[0] = shm01 * shift_center[1] + shm02 * shift_center[2];  /* pyx:216-218 */
        shift_center[1] = shm12 * shift_center[2];
        shift_center[2] = 0.0;
        for (int64_t a = 0; a < n_atoms; ++a)                                 /* pyx:221-223 */
            for (int i = 0; i < 3; ++i) {
                float *x = &coords[(a * 3 + i) * F + f];
                *x = (*x - wrap_center[i]) + box_middle[i];
            }
        for (int64_t g = 0; g + 1 < n_groups; ++g) {
            const int64_t s = groups[g], e = groups[g + 1];
            for (int i = 0; i < 3; ++i) grp_center[i] = 0.f;
            int64_t n = 0;
            for (int64_t k = s; k < e; ++k, ++n)                              /* pyx:230-237 */
                for (int i = 0; i < 3; ++i) {
                    grp_center[i] = grp_center[i] + (coords[(k * 3 + i) * F + f] - grp_center[i]) / (float)(n + 1);
                    grp_center_init[i] = grp_center[i];   /* (keeps the previous group's value for an empty group) */
                }
            for (int m = 2; m >= 0; --m) {                                    /* pyx:239-259 */
                double shift = shift_center[m];
                if (m == 0) shift += shm01 * (double)grp_center[1] + shm02 * (double)grp_center[2];
                else if (m == 1) shift += shm12 * (double)grp_center[2];
                int64_t it = 0;
                while ((double)grp_center[m] - shift < 0 && it++ < max_iter)
                    for (int d = 0; d <= m; ++d) grp_center[d] = (float)((double)grp_center[d] + box[m][d]);
                it = 0;
                while ((double)grp_center[m] - shift >= box[m][m] && it++ < max_iter)
                    for (int d = 0; d <= m; ++d) grp_center[d] = (float)((double)grp_center[d] - box[m][d]);
                for (int64_t a = s; a < e; ++a) {
                    float *x = &coords[(a * 3 + m) * F + f];
                    *x = *x - (grp_center_init[m] - grp_center[m]);
                }
            }
        }
    }
}

static double tric_norm2(const double *v) { return v[0] * v[0] + v[1] * v[1] + v[2] * v[2]; }
static double tric_min(double a, double b) { return a < b ? a : b; }
static double tric_max(double a, double b) { return a > b ? a : b; }

/* pyx:357-451 get_pbc (GROMACS low_set_pbc): up to 12 correction vectors; returns ntric_vec or -1 for the
 * reference's ValueError("Too many triclinic vectors!!"). */
static int tric_get_pbc(double box[3][3], double tric_vec[12][3], double *max_cutoff2_out)
{
    static const int order[3] = {0, -1, 1};
    const double skew = 1.001;
    double hbox[3], trial[3], pos[3];
    int ntric = 0;
    for (int i = 0; i < 3; ++i) hbox[i] = box[i][i] * 0.5;
    double min_hv2 = 0.25 * tric_min(tric_norm2(box[0]), tric_norm2(box[1]));
    min_hv2 = tric_min(min_hv2, 0.25 * tric_norm2(box[2]));
    const double min_ss = tric_min(box[0][0], tric_min(box[1][1] - fabs(box[2][1]), box[2][2]));
    *max_cutoff2_out = tric_min(min_hv2, min_ss * min_ss);
    for (int kk = 0; kk < 3; ++kk) {
        const int k = order[kk];
        for (int jj = 0; jj < 3; ++jj) {
            const int j = order[jj];
            for (int ii = 0; ii < 3; ++ii) {
                const int i = order[ii];
                if (!(j != 0 || k != 0)) continue;
                double d2old = 0, d2new = 0;
                for (int d = 0; d < 3; ++d) {
                    trial[d] = i * box[0][d] + j * box[1][d] + k * box[2][d];
                    if (trial[d] < 0) pos[d] = tric_min(hbox[d], -trial[d]);
                    else pos[d] = tric_max(-hbox[d], -trial[d]);
                    d2old += pos[d] * pos[d];
                    d2new += (pos[d] + trial[d]) * (pos[d] + trial[d]);
                }
                if (skew * d2new < d2old) {
                    int use = 1;
                    for (int dd = 0; dd < 3; ++dd) {
                        const int shift = dd == 0 ? i : (dd == 1 ? j : k);
                        if (shift) {
                            double d2c = 0;
                            for (int e = 0; e < 3; ++e) {
                                const double t = pos[e] + trial[e] - shift * box[dd][e];
                                d2c += t * t;
                            }
                            if (d2c <= skew * d2new) { use = 0; break; }
                        }
                    }
                    if (use) {
                        if (ntric >= 12) return -1;
                        for (int e = 0; e < 3; ++e) tric_vec[ntric][e] = trial[e];
                        ++ntric;
                    }
                }
            }
        }
    }
    return ntric;
}

/* pyx:454-505 pbc_dx (note: in mode 1 the correction-vector search sits INSIDE the loop over the axes) */
static void tric_pbc_dx(const float *x1, const float *x2, double box[3][3], const double *hbox,
                        double tric_vec[12][3], double max_cutoff2, int ntric, int mode, double *dx, int64_t max_iter)
{
    double dx_start[3], trial[3];
    for (int i = 0; i < 3; ++i) dx[i] = (double)(x1[i] - x2[i]);
    if (mode == 0) {
        for (int i = 0; i < 3; ++i) {
            int64_t it = 0;
            while (dx[i] > hbox[i] && it++ < max_iter) dx[i] -= box[i][i];
            it = 0;
            while (dx[i] <= -hbox[i] && it++ < max_iter) dx[i] += box[i][i];
        }
    } else if (mode == 1) {
        for (int i = 2; i >= 0; --i) {
            int64_t it = 0;
            while (dx[i] > hbox[i] && it++ < max_iter)
                for (int j = i; j >= 0; --j) dx[j] -= box[i][j];
            it = 0;
            while (dx[i] <= -hbox[i] && it++ < max_iter)
                for (int j = i; j >= 0; --j) dx[j] += box[i][j];
            double d2min = tric_norm2(dx);
            if (d2min > max_cutoff2) {
                for (int j = 0; j < 3; ++j) dx_start[j] = dx[j];
                int k = 0;
                while (d2min > max_cutoff2 && k < ntric) {
                    for (int j = 0; j < 3; ++j) trial[j] = dx_start[j] + tric_vec[k][j];
                    const double d2trial = tric_norm2(trial);
                    if (d2trial < d2min) {
                        for (int j = 0; j < 3; ++j) dx[j] = trial[j];
                        d2min = d2trial;
                    }
                    ++k;
                }
            }
        }
    }
}

/* pyx:255-344 wrap_compact_unitcell; mode 0 = "rectangular" cell of a triclinic box, 1 = "compact".
 * Returns 0, or -1 - f for the frame whose box yields more than 12 correction vectors. */
EXPORT int64_t oracle_wrap_compact(const uint32_t *groups, int64_t n_groups, float *coords, int64_t n_atoms,
                                   const double *boxvectors, int64_t F, const uint32_t *centersel,
                                   int64_t n_centersel, const float *center, int mode, int64_t max_iter)
{
    float wrap_center[3] = {0.f, 0.f, 0.f}, box_middle[3], grp_center[3];
    double box[3][3], tric_vec[12][3], hbox[3], dx[3], max_cutoff2;
    if (n_centersel == 0)
        for (int i = 0; i < 3; ++i) wrap_center[i] = center[i];
    for (int64_t f = 0; f < F; ++f) {
        tric_frame_setup(boxvectors, F, f, coords, n_atoms, centersel, n_centersel, wrap_center, box, box_middle);
        for (int i = 0; i < 3; ++i) hbox[i] = box[i][i] * 0.5;
        for (int64_t a = 0; a < n_atoms; ++a)
            for (int i = 0; i < 3; ++i) {
                float *x = &coords[(a * 3 + i) * F + f];
                *x = (*x - wrap_center[i]) + box_middle[i];
            }
        memset(tric_vec, 0, sizeof tric_vec);
        const int ntric = tric_get_pbc(box, tric_vec, &max_cutoff2);
        if (ntric < 0) return -1 - f;
        for (int64_t g = 0; g + 1 < n_groups; ++g) {
            const int64_t s = groups[g], e = groups[g + 1];
            for (int i = 0; i < 3; ++i) grp_center[i] = 0.f;
            int64_t n = 0;
            for (int64_t a = s; a < e; ++a, ++n)
                for (int i = 0; i < 3; ++i)
                    grp_center[i] = grp_center[i] + (coords[(a * 3 + i) * F + f] - grp_center[i]) / (float)(n + 1);
            tric_pbc_dx(grp_center, box_middle, box, hbox, tric_vec, max_cutoff2, ntric, mode, dx, max_iter);
            for (int64_t a = s; a < e; ++a)
                for (int i = 0; i < 3; ++i) {
                    float *x = &coords[(a * 3 + i) * F + f];
                    *x = (float)((double)((*x - grp_center[i]) + box_middle[i]) + dx[i]);
                }
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------------
 * Hydrogen bonds -- moleculekit/interactions/hbonds/hbonds.pyx:25-134 (called by hbonds_calculate,
 * moleculekit/interactions/interactions.py:365-467).  donors (n_donors, 2) = (heavy, hydrogen),
 * acceptors (n_acceptors), sel1 / sel2 0/1 flags per atom, coords (N, 3, F) f32, box (3, F) f32.
 * Per frame, donor-major / acceptor-minor, a triple (heavy, hydrogen | -1, acceptor) is emitted when the
 * hydrogen (heavy atom with ignore_hs) is within dist_threshold of the acceptor and the
 * heavy-hydrogen-acceptor angle exceeds angle_threshold.  Types as generated: `val`, the squared
 * distances, the dot product and `angle` are float; see the note on the C++ float overloads below.
 * counts[f] receives the number of triples of frame f; up to `capacity` triples are written; the total
 * is returned.
 * ------------------------------------------------------------------------------------------------ */
/* The reference is compiled as C++ (setup.py: language="c++"), where the unqualified round / sqrt / acos the generated
 * code calls on float arguments resolve to the float overloads of <cmath>: the wrap is val - fl(box * roundf(fl(val / box)))
 * with every operation rounded to float (as distance_utils._dist), the norms are sqrtf with a float product, and the angle is
 * acosf.  (A first restatement went through double as the .pyx reads in C; index outputs rarely tell the two apart --
 * tests/test_oracle_golden.py::test_hbonds_float_overloads pins the difference on ~1e9 pair tests.)  hb_model_double = 1
 * selects that discarded model, for that test only. */
static int hb_model_double = 0;
EXPORT void oracle_hbonds_set_model(int use_double) { hb_model_double = use_double; }
static float hb_wrap_val(float val, float b)
{
    if (hb_model_double) return (float)((double)val - (double)b * round((double)(val / b)));
    return val - b * roundf(val / b);
}

EXPORT int64_t oracle_hbonds(const uint32_t *donors, int64_t n_donors, const uint32_t *acceptors, int64_t n_acceptors,
                             const float *coords, const float *box, int64_t F, const uint32_t *sel1,
                             const uint32_t *sel2, float dist_threshold, float angle_threshold, int intra,
                             int ignore_hs, int64_t *counts, int32_t *out, int64_t capacity)
{
    float dist_vec_a[3], dist_vec_b[3], half_box[3];
    int64_t total = 0;
    dist_threshold = dist_threshold * dist_threshold;                          /* pyx:49 */
    angle_threshold = (float)((double)angle_threshold / 57.29578);            /* pyx:50 */
    for (int64_t f = 0; f < F; ++f) {
        int64_t nf = 0;
        for (int i = 0; i < 3; ++i) half_box[i] = box[i * F + f] / 2;
        for (int64_t d = 0; d < n_donors; ++d)
            for (int64_t a = 0; a < n_acceptors; ++a) {
                const uint32_t a_idx = acceptors[a], d_idx_d = donors[2 * d];
                uint32_t d_idx = d_idx_d, d_idx_h = 0;
                if (!ignore_hs) { d_idx_h = donors[2 * d + 1]; d_idx = d_idx_h; }
                if (a_idx == d_idx_d) continue;
                if (intra) {
                    if (sel1[a_idx] == 0 || sel1[d_idx_d] == 0) continue;
                } else if (!((sel1[a_idx] == 1 && sel2[d_idx_d] == 1) || (sel2[a_idx] == 1 && sel1[d_idx_d] == 1)))
                    continue;
                float dist2_a = 0, dist2_b = 0;
                for (int i = 0; i < 3; ++i) {
                    const float b = box[i * F + f];
                    float val = coords[((int64_t)a_idx * 3 + i) * F + f] - coords[((int64_t)d_idx * 3 + i) * F + f];
                    if (fabsf(val) > half_box[i] && b != 0) val = hb_wrap_val(val, b);
                    dist_vec_a[i] = val;
                    dist2_a = dist2_a + (val * val);
                }
                if (dist2_a > dist_threshold) continue;
                if (ignore_hs) {
                    if (total < capacity) { out[3 * total] = (int32_t)d_idx_d; out[3 * total + 1] = -1; out[3 * total + 2] = (int32_t)a_idx; }
                    ++total; ++nf;
                    continue;
                }
                for (int i = 0; i < 3; ++i) {
                    const float b = box[i * F + f];
                    float val = coords[((int64_t)d_idx_d * 3 + i) * F + f] - coords[((int64_t)d_idx_h * 3 + i) * F + f];
                    if (fabsf(val) > half_box[i] && b != 0) val = hb_wrap_val(val, b);
                    dist_vec_b[i] = val;
                    dist2_b = dist2_b + (val * val);
                }
                if (dist2_a == 0 || dist2_b == 0) continue;
                float dotprod = 0;
                for (int i = 0; i < 3; ++i) dotprod = dotprod + dist_vec_a[i] * dist_vec_b[i];
                float angle = hb_model_double ? (float)((double)dotprod / (sqrt((double)dist2_a) * sqrt((double)dist2_b)))
                                              : (float)((double)dotprod / (double)(sqrtf(dist2_a) * sqrtf(dist2_b)));
                if (angle > 1) angle = 1;
                if (angle < -1) angle = -1;
                angle = hb_model_double ? (float)acos((double)angle) : acosf(angle);
                if (angle > angle_threshold) {
                    if (total < capacity) { out[3 * total] = (int32_t)d_idx_d; out[3 * total + 1] = (int32_t)d_idx_h; out[3 * total + 2] = (int32_t)a_idx; }
                    ++total; ++nf;
                }
            }
        counts[f] = nf;
    }
    return total;
}

/* ------------------------------------------------------------------------------------------------
 * Ring interactions -- moleculekit/interactions/pipi/pipi.pyx:86-185 (mode 0), cationpi/cationpi.pyx:91-173
 * (mode 1), sigmahole/sigmahole.pyx:91-174 (mode 2); callers pipi_calculate / cationpi_calculate /
 * sigmahole_calculate, moleculekit/interactions/interactions.py:621-946.
 * rings_atoms + starts1 [n1 + 1]: the rings of the first set.  `second`: mode 0 ring start indexes
 * [n2 + 1] into the same rings_atoms; mode 1 cation atom indexes [n2]; mode 2 (halogen, bonded
 * partner) pairs [n2][2].  Helpers shared by the three files: ring centroid = float sum in atom order /
 * (float)count (pyx:23-41); wrapped distance (pyx:46-62), cross product and normalisation (pyx:67-83) in
 * float -- the modules are C++, so round / sqrt / acos on float arguments are the float overloads (see
 * oracle_hbonds).  `angle` is an untyped (double) variable: (double)acosf(dot) * 57.29578, folded to
 * [0, 90], for modes 1 / 2 turned into the angle to the plane.
 * Emits per frame, ring-major: (r1, r2 | cation atom | halogen atom) and (sqrt(dist2), angle) as floats.
 * ------------------------------------------------------------------------------------------------ */
static void ring_mean(const float *coords, int64_t F, int64_t f, const uint32_t *atoms, int64_t s, int64_t e, float *m)
{
    for (int i = 0; i < 3; ++i) m[i] = 0.f;
    for (int64_t r = s; r < e; ++r)
        for (int i = 0; i < 3; ++i) m[i] = m[i] + coords[((int64_t)atoms[r] * 3 + i) * F + f];
    for (int i = 0; i < 3; ++i) m[i] = m[i] / (float)(e - s);
}
static float ring_wrapped_dist(const float *p1, const float *p2, const float *half_box, const float *box, int64_t F, int64_t f)
{
    float dist2 = 0.f;
    for (int i = 0; i < 3; ++i) {
        const float b = box[i * F + f];
        float val = p1[i] - p2[i];
        if (fabsf(val) > half_box[i] && b != 0) val = val - b * roundf(val / b);   /* C++ float overload of round */
        dist2 = dist2 + (val * val);
    }
    return dist2;
}
static void ring_normalize(float *v)
{
    float n = 0.f;
    for (int i = 0; i < 3; ++i) n = n + (v[i] * v[i]);
    n = sqrtf(n);
    for (int i = 0; i < 3; ++i) v[i] = v[i] / n;
}
static void ring_normal(const float *coords, int64_t F, int64_t f, const uint32_t *atoms, int64_t s, float *res)
{
    float a[3], b[3];
    for (int i = 0; i < 3; ++i) {
        a[i] = coords[((int64_t)atoms[s] * 3 + i) * F + f] - coords[((int64_t)atoms[s + 2] * 3 + i) * F + f];
        b[i] = coords[((int64_t)atoms[s + 1] * 3 + i) * F + f] - coords[((int64_t)atoms[s + 2] * 3 + i) * F + f];
    }
    res[0] = a[1] * b[2] - a[2] * b[1];
    res[1] = a[2] * b[0] - a[0] * b[2];
    res[2] = a[0] * b[1] - a[1] * b[0];
    ring_normalize(res);
}

EXPORT int64_t oracle_ring_interactions(int mode, const uint32_t *rings_atoms, const uint32_t *starts1, int64_t n1,
                                        const uint32_t *second, int64_t n2, const float *coords, const float *box,
                                        int64_t F, float p0, float p1, float p2, float p3, int64_t *counts,
                                        int32_t *pairs, float *distangles, int64_t capacity)
{
    float half_box[3], m1[3], m2[3], nrm1[3], nrm2[3], t1[3], t2[3];
    int64_t total = 0;
    const float d1 = p0 * p0;                       /* pipi: dist_threshold1^2; others: dist_threshold^2 */
    const float d2 = mode == 0 ? p2 * p2 : 0.f;     /* pipi: dist_threshold2^2 */
    for (int64_t f = 0; f < F; ++f) {
        int64_t nf = 0;
        for (int i = 0; i < 3; ++i) half_box[i] = box[i * F + f] / 2;
        for (int64_t r1 = 0; r1 < n1; ++r1)
            for (int64_t r2 = 0; r2 < n2; ++r2) {
                const int64_t s1 = starts1[r1], e1 = starts1[r1 + 1];
                float dist2;
                double angle;
                int32_t second_id;
                if (mode == 0) {
                    const int64_t s2 = second[r2], e2 = second[r2 + 1];
                    if (s1 == s2 && e1 == e2) continue;                       /* identical rings */
                    for (int i = 0; i < 3; ++i) {
                        t1[i] = coords[((int64_t)rings_atoms[s1] * 3 + i) * F + f];
                        t2[i] = coords[((int64_t)rings_atoms[s2] * 3 + i) * F + f];
                    }
                    if (ring_wrapped_dist(t1, t2, half_box, box, F, f) > 225) continue;
                    ring_mean(coords, F, f, rings_atoms, s1, e1, m1);
                    ring_mean(coords, F, f, rings_atoms, s2, e2, m2);
                    dist2 = ring_wrapped_dist(m1, m2, half_box, box, F, f);
                    if (dist2 > d2) continue;
                    ring_normal(coords, F, f, rings_atoms, s1, nrm1);
                    ring_normal(coords, F, f, rings_atoms, s2, nrm2);
                    float dot = 0.f;
                    for (int i = 0; i < 3; ++i) dot = dot + nrm1[i] * nrm2[i];
                    angle = (double)acosf(dot) * 57.29578;
                    if (angle > 90) angle = 180 - angle;
                    if (!((dist2 < d1 && angle <= (double)p1) || (dist2 < d2 && angle >= (double)p3))) continue;
                    second_id = (int32_t)r2;
                } else {
                    const uint32_t atom = mode == 1 ? second[r2] : second[2 * r2];
                    ring_mean(coords, F, f, rings_atoms, s1, e1, m1);
                    for (int i = 0; i < 3; ++i) m2[i] = coords[((int64_t)atom * 3 + i) * F + f];
                    dist2 = ring_wrapped_dist(m1, m2, half_box, box, F, f);
                    if (dist2 > d1) continue;
                    ring_normal(coords, F, f, rings_atoms, s1, nrm1);
                    if (mode == 1) {
                        for (int i = 0; i < 3; ++i) t1[i] = m2[i] - m1[i];                     /* ring -> cation */
                    } else {
                        const uint32_t partner = second[2 * r2 + 1];
                        for (int i = 0; i < 3; ++i) t1[i] = m2[i] - coords[((int64_t)partner * 3 + i) * F + f];
                    }
                    ring_normalize(t1);
                    float dot = 0.f;
                    for (int i = 0; i < 3; ++i) dot = dot + nrm1[i] * t1[i];
                    angle = (double)acosf(dot) * 57.29578;
                    if (angle > 90) angle = 180 - angle;
                    angle = 90 - angle;
                    if (!(angle >= (double)p1)) continue;
                    second_id = (int32_t)atom;
                }
                if (total < capacity) {
                    pairs[2 * total] = (int32_t)r1; pairs[2 * total + 1] = second_id;
                    distangles[2 * total] = sqrtf(dist2); distangles[2 * total + 1] = (float)angle;
                }
                ++total; ++nf;
            }
        counts[f] = nf;
    }
    return total;
}
