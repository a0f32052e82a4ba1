// rings.cu -- K13: ring-based interaction detectors over a trajectory for sm_90a (H100).
//
// Replaces pipi.calculate (moleculekit/interactions/pipi/pipi.pyx:86-185, mode 0), cationpi.calculate
// (interactions/cationpi/cationpi.pyx:91-173, mode 1) and sigmahole.calculate (interactions/sigmahole/sigmahole.pyx:91-174,
// mode 2), the kernels under pipi_calculate / cationpi_calculate / sigmahole_calculate
// (moleculekit/interactions/interactions.py:621-946).  Per frame the reference walks rings x partners (ring major) and emits
// (ring, partner) with (distance, angle) when the ring centroid is close enough to the partner (a second ring's centroid, a
// cation, a halogen) and the angle between the ring normal and a second direction (the other ring's normal, the
// centroid -> cation vector, the halogen's bond) passes a threshold.  As in K4 / K12 only the ORDER is sequential: one
// thread per (frame, ring) prepares centroid, normal and first atom once (the reference recomputes them per pair, with
// the same values), then one warp per (frame, ring) row counts / fills its partners in order.
//
// Bit parity.  The modules are C++: round / sqrt / acos on float arguments are the float overloads (see hbonds.cu).  All
// geometry is float with one rounding per operation (centroid = float sum in atom order / (float)count; wrapped distance
// val - fl(box * roundf(fl(val / box))); cross product, norms by sqrtf): bit-identical on the device.  The decisions
// compare the DOUBLE `angle = fold((double)acosf(dot) * 57.29578)` with the thresholds; fold and every comparison are
// monotone on each side of the fold, so the host turns each decision into at most two closed intervals of the float `dot`
// (bisection with the libm the reference calls) and the device tests interval membership: the reference's booleans
// without a device acosf.  Emitted distances are sqrtf(dist2), bit-identical; emitted angles come from the device's acos
// and can differ from glibc's acosf-based value in the last bits (not correctly rounded there).
#include <cmath>
#include <cstring>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace mkb {

enum { RING_PIPI = 0, RING_CATIONPI = 1, RING_SIGMAHOLE = 2 };

struct RingSet {    // a decision on the float dot product: x in [lo[0], hi[0]] or x in [lo[1], hi[1]]
    float lo[2], hi[2];
};

struct RingArgs {
    int mode;
    long long F, fsb, n1, n2, nrings;  // nrings: rings prepared per frame (set 1 first, then set 2 for pipi)
    const float *box;
    const unsigned *starts1, *starts2;  // ring start indexes (pipi: identical-ring test)
    const unsigned *second;             // cationpi: cation atoms [n2]; sigmahole: (halogen, partner) [n2][2]
    const float4 *R;                    // [F][nrings][3]: centroid, normal, first atom
    const float4 *PA, *PB;              // [F][n2] gathered partner atoms (cationpi: cation; sigmahole: halogen, bonded partner)
    float d1, d2;                       // squared distance thresholds (float products, as the reference)
    RingSet c1, c2;                     // pipi: angle <= a1max, angle >= a2min;  cationpi / sigmahole: c1 = (90 - angle >= amin)
};

__device__ __forceinline__ bool ring_in(const RingSet &s, float x) {
    return (x >= s.lo[0] && x <= s.hi[0]) || (x >= s.lo[1] && x <= s.hi[1]);
}

// pyx:46-62 `_wrapped_dist`: every operation rounded to float
__device__ __forceinline__ float ring_wdist(const float4 a, const float4 b, float bx, float by, float bz, float hx, float hy,
                                            float hz) {
    float v0 = __fsub_rn(a.x, b.x), v1 = __fsub_rn(a.y, b.y), v2 = __fsub_rn(a.z, b.z);
    if (fabsf(v0) > hx && bx != 0.f) v0 = __fsub_rn(v0, __fmul_rn(bx, roundf(__fdiv_rn(v0, bx))));
    if (fabsf(v1) > hy && by != 0.f) v1 = __fsub_rn(v1, __fmul_rn(by, roundf(__fdiv_rn(v1, by))));
    if (fabsf(v2) > hz && bz != 0.f) v2 = __fsub_rn(v2, __fmul_rn(bz, roundf(__fdiv_rn(v2, bz))));
    return __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(v0, v0)), __fmul_rn(v1, v1)), __fmul_rn(v2, v2));
}

// pyx:67-83: vec / sqrtf(sum of squares), float
__device__ __forceinline__ void ring_normalize(float &x, float &y, float &z) {
    float n = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(x, x)), __fmul_rn(y, y)), __fmul_rn(z, z));
    n = __fsqrt_rn(n);
    x = __fdiv_rn(x, n); y = __fdiv_rn(y, n); z = __fdiv_rn(z, n);
}

// one thread per (ring, frame), frame fastest: centroid (pyx:23-41), normal from the first three atoms, first atom
__global__ void ring_prep_kernel(const float *__restrict__ coords, long long fs, long long F,
                                 const unsigned *__restrict__ atoms, const unsigned *__restrict__ starts1, long long n1,
                                 const unsigned *__restrict__ starts2, long long n2r, float4 *__restrict__ R) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long nr = n1 + n2r;
    if (tid >= nr * F) return;
    const long long r = tid / F, f = tid - r * F;
    const long long s = r < n1 ? starts1[r] : starts2[r - n1], e = r < n1 ? starts1[r + 1] : starts2[r - n1 + 1];
    float m[3] = {0.f, 0.f, 0.f};
    for (long long k = s; k < e; ++k) {
        const float *p = coords + (long long)atoms[k] * 3 * fs + f;
#pragma unroll
        for (int i = 0; i < 3; ++i) m[i] = __fadd_rn(m[i], p[i * fs]);
    }
    const float cnt = (float)(int)(e - s);
#pragma unroll
    for (int i = 0; i < 3; ++i) m[i] = __fdiv_rn(m[i], cnt);
    float a[3] = {0.f, 0.f, 0.f}, nrm[3] = {0.f, 0.f, 0.f};
    if (e - s >= 3) {  // the reference reads atoms s, s + 1, s + 2 whatever the ring size; rings have >= 3 atoms
        const float *p0 = coords + (long long)atoms[s] * 3 * fs + f, *p1 = coords + (long long)atoms[s + 1] * 3 * fs + f,
                    *p2 = coords + (long long)atoms[s + 2] * 3 * fs + f;
        float t1[3], t2[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            a[i] = p0[i * fs];
            t1[i] = __fsub_rn(a[i], p2[i * fs]);
            t2[i] = __fsub_rn(p1[i * fs], p2[i * fs]);
        }
        nrm[0] = __fsub_rn(__fmul_rn(t1[1], t2[2]), __fmul_rn(t1[2], t2[1]));
        nrm[1] = __fsub_rn(__fmul_rn(t1[2], t2[0]), __fmul_rn(t1[0], t2[2]));
        nrm[2] = __fsub_rn(__fmul_rn(t1[0], t2[1]), __fmul_rn(t1[1], t2[0]));
        ring_normalize(nrm[0], nrm[1], nrm[2]);
    } else if (e > s) {
        const float *p0 = coords + (long long)atoms[s] * 3 * fs + f;
#pragma unroll
        for (int i = 0; i < 3; ++i) a[i] = p0[i * fs];
    }
    float4 *o = R + (f * nr + r) * 3;
    o[0] = make_float4(m[0], m[1], m[2], 0.f);
    o[1] = make_float4(nrm[0], nrm[1], nrm[2], 0.f);
    o[2] = make_float4(a[0], a[1], a[2], 0.f);
}

// G[f][k] = coords[idx[k * stride_idx + off], 0..2, f]
__global__ void ring_gather_kernel(const float *__restrict__ coords, long long fs, long long F,
                                   const unsigned *__restrict__ idx, int stride_idx, int off, long long n,
                                   float4 *__restrict__ G) {
    const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (tid >= n * F) return;
    const long long k = tid / F, f = tid - k * F;
    const float *p = coords + (long long)idx[k * stride_idx + off] * 3 * fs + f;
    G[f * n + k] = make_float4(p[0], p[fs], p[2 * fs], 0.f);
}

template <bool FILL>
__global__ void __launch_bounds__(256) ring_pair_kernel(const RingArgs A, long long *__restrict__ counts,
                                                        const long long *__restrict__ row_offsets,
                                                        int *__restrict__ pairs, float *__restrict__ distangles) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= A.F * A.n1) return;
    const long long f = row / A.n1, r1 = row - f * A.n1;
    long long base = FILL ? row_offsets[row] : 0;
    const long long row_end = FILL ? row_offsets[row + 1] : 0;
    if (FILL && base == row_end) return;
    const float4 *R1 = A.R + (f * A.nrings + r1) * 3;
    const float4 m1 = R1[0], n1v = R1[1], a1 = R1[2];
    const float bx = A.box[f], by = A.box[A.fsb + f], bz = A.box[2 * A.fsb + f];
    const float hx = __fdiv_rn(bx, 2.f), hy = __fdiv_rn(by, 2.f), hz = __fdiv_rn(bz, 2.f);
    const unsigned s1 = A.mode == RING_PIPI ? A.starts1[r1] : 0u, e1 = A.mode == RING_PIPI ? A.starts1[r1 + 1] : 0u;
    long long total = 0;
    const int n2 = (int)A.n2;
    for (int k0 = 0; k0 < n2; k0 += 32) {
        const int k = k0 + lane;
        bool hit = false;
        float dist2 = 0.f, dot = 0.f;
        int second_id = 0;
        if (k < n2) {
            if (A.mode == RING_PIPI) {
                const unsigned s2 = A.starts2[k], e2 = A.starts2[k + 1];
                if (!(s1 == s2 && e1 == e2)) {                                               // pyx:129-131 identical rings
                    const float4 *R2 = A.R + (f * A.nrings + A.n1 + k) * 3;
                    const float4 a2 = R2[2];
                    if (!(ring_wdist(a1, a2, bx, by, bz, hx, hy, hz) > 225.f)) {             // pyx:134-140 early exit
                        const float4 m2 = R2[0], n2v = R2[1];
                        dist2 = ring_wdist(m1, m2, bx, by, bz, hx, hy, hz);
                        if (!(dist2 > A.d2)) {                                               // pyx:150-152
                            dot = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(n1v.x, n2v.x)), __fmul_rn(n1v.y, n2v.y)),
                                            __fmul_rn(n1v.z, n2v.z));
                            hit = (dist2 < A.d1 && ring_in(A.c1, dot)) || (dist2 < A.d2 && ring_in(A.c2, dot));  // pyx:176-177
                            second_id = k;
                        }
                    }
                }
            } else {
                const float4 pa = A.PA[f * A.n2 + k];
                dist2 = ring_wdist(m1, pa, bx, by, bz, hx, hy, hz);
                if (!(dist2 > A.d1)) {                                                       // cationpi.pyx:139-141
                    float t0, t1, t2;
                    if (A.mode == RING_CATIONPI) {
                        t0 = __fsub_rn(pa.x, m1.x); t1 = __fsub_rn(pa.y, m1.y); t2 = __fsub_rn(pa.z, m1.z);
                    } else {
                        const float4 pb = A.PB[f * A.n2 + k];
                        t0 = __fsub_rn(pa.x, pb.x); t1 = __fsub_rn(pa.y, pb.y); t2 = __fsub_rn(pa.z, pb.z);
                    }
                    ring_normalize(t0, t1, t2);
                    dot = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(n1v.x, t0)), __fmul_rn(n1v.y, t1)), __fmul_rn(n1v.z, t2));
                    hit = ring_in(A.c1, dot);
                    second_id = (int)(A.mode == RING_CATIONPI ? A.second[k] : A.second[2 * k]);
                }
            }
        }
        const unsigned mball = __ballot_sync(0xffffffffu, hit);
        if (FILL) {
            if (hit) {
                const long long o = base + __popc(mball & ((1u << lane) - 1u));
                pairs[2 * o] = (int)r1;
                pairs[2 * o + 1] = second_id;
                // the reported angle: (double)acosf(dot) * 57.29578 folded to [0, 90] (and 90 - that for modes 1 / 2)
                double ang = (double)__double2float_rn(acos((double)dot)) * 57.29578;
                if (ang > 90.0) ang = 180.0 - ang;
                if (A.mode != RING_PIPI) ang = 90.0 - ang;
                distangles[2 * o] = __fsqrt_rn(dist2);
                distangles[2 * o + 1] = (float)ang;
            }
            base += __popc(mball);
            if (base == row_end) break;
        } else {
            total += __popc(mball);
        }
    }
    if (!FILL && lane == 0) counts[row] = total;
}

__global__ void ring_set_last_zero(long long *p, long long n) {
    if (threadIdx.x == 0 && blockIdx.x == 0) p[n] = 0;
}

// ---- host: decisions on the double angle as intervals of the float dot product
static long long fkey(float x) {
    int32_t b;
    memcpy(&b, &x, 4);
    return b >= 0 ? (long long)b : -(long long)(b & 0x7fffffff);
}
static float funkey(long long k) {
    int32_t b = k >= 0 ? (int32_t)k : (int32_t)(0x80000000u | (uint32_t)(-k));
    float x;
    memcpy(&x, &b, 4);
    return x;
}
// largest key in [ka, kb] whose float satisfies pred, pred being true on a prefix of the range; ka - 1 when none
template <class P>
static long long last_true(long long ka, long long kb, P pred) {
    if (ka > kb || !pred(funkey(ka))) return ka - 1;
    if (pred(funkey(kb))) return kb;
    long long lo = ka, hi = kb;  // lo true, hi false
    while (hi - lo > 1) {
        const long long mid = lo + (hi - lo) / 2;
        if (pred(funkey(mid))) lo = mid; else hi = mid;
    }
    return lo;
}
// `decide(angle)` is the reference's test on the folded double angle (monotone in the angle); `to_plane`: modes 1 / 2
// (90 - angle).  Returns the floats x in [-1, 1] for which decide(folded(x)) holds, as two closed intervals.
template <class D>
static RingSet ring_decision_set(D decide, bool to_plane) {
    auto raw = [](float x) { return (double)acosf(x) * 57.29578; };  // the C++ float overload the reference calls
    auto folded = [&](float x) {
        double a = raw(x);
        if (a > 90.0) a = 180.0 - a;
        if (to_plane) a = 90.0 - a;
        return a;
    };
    const long long kmin = fkey(-1.f), kmax = fkey(1.f);
    // lower branch: the floats whose raw angle exceeds 90 (a prefix of [-1, 1]: acosf is non-increasing)
    const long long kb = last_true(kmin, kmax, [&](float x) { return raw(x) > 90.0; });
    RingSet s;
    s.lo[0] = s.lo[1] = 1.f; s.hi[0] = s.hi[1] = -1.f;  // empty
    // On the lower branch the folded angle (before 90 - .) grows with x, on the upper branch it falls; with to_plane the
    // directions swap.  In each branch the decision is monotone in x: find where it flips.
    auto P = [&](float x) { return decide(folded(x)); };
    if (kb >= kmin) {  // lower branch [kmin, kb]
        const bool at_lo = P(funkey(kmin)), at_hi = P(funkey(kb));
        if (at_lo && at_hi) { s.lo[0] = -1.f; s.hi[0] = funkey(kb); }
        else if (at_lo) { s.lo[0] = -1.f; s.hi[0] = funkey(last_true(kmin, kb, P)); }
        else if (at_hi) { s.lo[0] = funkey(last_true(kmin, kb, [&](float x) { return !P(x); }) + 1); s.hi[0] = funkey(kb); }
    }
    if (kb < kmax) {   // upper branch [kb + 1, kmax]
        const long long ka = kb + 1;
        const bool at_lo = P(funkey(ka)), at_hi = P(funkey(kmax));
        if (at_lo && at_hi) { s.lo[1] = funkey(ka); s.hi[1] = 1.f; }
        else if (at_lo) { s.lo[1] = funkey(ka); s.hi[1] = funkey(last_true(ka, kmax, P)); }
        else if (at_hi) { s.lo[1] = funkey(last_true(ka, kmax, [&](float x) { return !P(x); }) + 1); s.hi[1] = 1.f; }
    }
    return s;
}

static int ring_setup(mkb_ctx *h, cudaStream_t st, int32_t mode, const mkb_traj *t, const uint32_t *rings_atoms,
                      const uint32_t *starts1, int64_t n1, const uint32_t *second, int64_t n2, float p0, float p1,
                      float p2, float p3, RingArgs *A) {
    if (mode < 0 || mode > 2) return fail(h, MKB_ERR_BAD_ARG, "mode must be 0 (pi-pi), 1 (cation-pi) or 2 (sigma hole)");
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory view");
    if (t->n_atoms < 0 || t->n_frames < 0 || n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (t->n_frames > 0 && (!t->coords || !t->box)) return fail(h, MKB_ERR_BAD_ARG, "null coords/box");
    if (t->frame_stride < t->n_frames || t->frame_stride_box < t->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame_stride smaller than n_frames");
    const long long F = t->n_frames, rows = F * n1;
    if (rows >= (1ll << 31) / 32 || n2 >= (1ll << 31) || F * (n1 + n2) >= (1ll << 40))
        return fail(h, MKB_ERR_BAD_ARG, "frames x rings too large for one call");
    memset(A, 0, sizeof(*A));
    A->mode = mode; A->F = F; A->fsb = t->frame_stride_box; A->n1 = n1; A->n2 = n2; A->box = t->box;
    A->nrings = n1 + (mode == RING_PIPI ? n2 : 0);
    A->starts1 = starts1; A->starts2 = mode == RING_PIPI ? second : nullptr; A->second = second;
    A->d1 = p0 * p0;                                   // pyx: dist_threshold * dist_threshold (float)
    A->d2 = mode == RING_PIPI ? p2 * p2 : 0.f;
    if (mode == RING_PIPI) {
        const double t1 = (double)p1, t2 = (double)p3;
        A->c1 = ring_decision_set([=](double a) { return a <= t1; }, false);  // pyx:176
        A->c2 = ring_decision_set([=](double a) { return a >= t2; }, false);  // pyx:177
    } else {
        const double tmin = (double)p1;
        A->c1 = ring_decision_set([=](double a) { return a >= tmin; }, true);  // cationpi.pyx:165 on 90 - angle
        A->c2 = A->c1;
    }
    if (rows == 0 || n2 == 0) return MKB_OK;
    if (!rings_atoms || !starts1 || !second) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    float4 *buf;
    int rc;
    const size_t nR = (size_t)(F * A->nrings * 3), nP = mode == RING_PIPI ? 0 : (size_t)(F * n2) * (mode == RING_SIGMAHOLE ? 2 : 1);
    if ((rc = scratch_get(h, S_SORT_PX, nR + nP + 1, &buf))) return rc;
    A->R = buf;
    ring_prep_kernel<<<(unsigned)cdiv(A->nrings * F, 128), 128, 0, st>>>(t->coords, t->frame_stride, F, rings_atoms, starts1, n1,
                                                                       mode == RING_PIPI ? second : nullptr,
                                                                       mode == RING_PIPI ? n2 : 0, buf);
    MKB_LAUNCHED(h);
    if (mode != RING_PIPI) {
        float4 *pa = buf + nR;
        A->PA = pa;
        const int stride = mode == RING_SIGMAHOLE ? 2 : 1;
        ring_gather_kernel<<<(unsigned)cdiv(n2 * F, 256), 256, 0, st>>>(t->coords, t->frame_stride, F, second, stride, 0, n2, pa);
        MKB_LAUNCHED(h);
        if (mode == RING_SIGMAHOLE) {
            A->PB = pa + F * n2;
            ring_gather_kernel<<<(unsigned)cdiv(n2 * F, 256), 256, 0, st>>>(t->coords, t->frame_stride, F, second, 2, 1, n2,
                                                                           pa + F * n2);
            MKB_LAUNCHED(h);
        }
    }
    return MKB_OK;
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_ring_pairs_count(mkb_handle_t h, void *stream, int32_t mode, const mkb_traj *t,
                                    const uint32_t *rings_atoms, const uint32_t *starts1, int64_t n_rings1,
                                    const uint32_t *second, int64_t n_second, float p0, float p1, float p2, float p3,
                                    int64_t *row_offsets, int64_t *total_pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets || !total_pairs) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/total_pairs");
    RingArgs A;
    int rc = ring_setup(h, st, mode, t, rings_atoms, starts1, n_rings1, second, n_second, p0, p1, p2, p3, &A);
    if (rc) return rc;
    const long long rows = A.F * A.n1;
    long long *counts;
    if ((rc = scratch_get(h, S_ROWCNT, (size_t)rows + 1, &counts))) return rc;
    if (rows > 0) {
        if (A.n2 > 0) {
            ring_pair_kernel<false><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(A, counts, nullptr, nullptr, nullptr);
            MKB_LAUNCHED(h);
        } else {
            MKB_CUDA(h, cudaMemsetAsync(counts, 0, (size_t)rows * sizeof(long long), st));
        }
    }
    ring_set_last_zero<<<1, 32, 0, st>>>(counts, rows);
    MKB_LAUNCHED(h);
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, (long long *)row_offsets, (int)(rows + 1), st));
    void *tmp = nullptr;
    if ((rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp))) return rc;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, (long long *)row_offsets, (int)(rows + 1), st));
    h->launches++;
    long long total = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&total, row_offsets + rows, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    *total_pairs = total;
    h->last_kernel = "ring_pair_kernel";
    return MKB_OK;
}

extern "C" int mkb_ring_pairs_fill(mkb_handle_t h, void *stream, int32_t mode, const mkb_traj *t,
                                   const uint32_t *rings_atoms, const uint32_t *starts1, int64_t n_rings1,
                                   const uint32_t *second, int64_t n_second, float p0, float p1, float p2, float p3,
                                   const int64_t *row_offsets, int32_t *pairs, float *distangles) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets");
    RingArgs A;
    int rc = ring_setup(h, st, mode, t, rings_atoms, starts1, n_rings1, second, n_second, p0, p1, p2, p3, &A);
    if (rc) return rc;
    const long long rows = A.F * A.n1;
    if (rows == 0 || A.n2 == 0) return MKB_OK;
    if (!pairs || !distangles) return fail(h, MKB_ERR_BAD_ARG, "null output");
    ring_pair_kernel<true><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(A, nullptr, (const long long *)row_offsets, pairs,
                                                                          distangles);
    MKB_LAUNCHED(h);
    return MKB_OK;
}
