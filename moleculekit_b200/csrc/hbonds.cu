// hbonds.cu -- K12: hydrogen-bond detection over a trajectory for sm_90a (H100).
//
// Replaces hbonds.calculate (moleculekit/interactions/hbonds/hbonds.pyx:25-134), the kernel under hbonds_calculate
// (moleculekit/interactions/interactions.py:365-467).  Per frame the reference walks donors x acceptors (donor major) and
// emits (heavy, hydrogen | -1, acceptor) when the hydrogen (the heavy atom with ignore_hs) is within dist_threshold of the
// acceptor and the heavy-hydrogen-acceptor angle exceeds angle_threshold.  Frames and pairs are independent; only the
// ORDER of the output is sequential, so this is the count -> scan -> ordered-fill scheme of K4 (one warp per
// (frame, donor) row, ballot + popc ranks inside the row).
//
// Bit parity.  The reference is compiled as C++ (setup.py: language="c++"): the unqualified round / sqrt / acos of the generated
// code, called on float arguments, resolve to the FLOAT overloads of <cmath>.  So
//   val  = a - d;  if |val| > box/2 and box != 0:  val = val - fl(box * roundf(fl(val / box)))      (every op rounded to float,
//                                                                                                   the _dist of distance_utils)
//   d2   = (v0*v0 + v1*v1) + v2*v2 (float);  skip when d2 > thr*thr  (a NaN d2 is NOT skipped)
//   cosv = (float)((double)dot / (double)fl(sqrtf(d2a) * sqrtf(d2b))), clamped to [-1, 1]
//   hit  = acosf(cosv) > (float)(angle_threshold / 57.29578)
// (a restatement that went through double, as the .pyx reads in C, differs from the reference binary in ~2 bonds per
// 10 million; tests/test_oracle_golden.py::test_hbonds_float_overloads).  Every operation has an IEEE counterpart on the
// device (__f*_rn, __ddiv_rn) except acosf.  acosf is a non-increasing function of its float argument, so the host finds,
// with the same libm the reference calls, the largest float c* whose arc cosine still exceeds the threshold; the device
// tests c <= c* -- the same booleans without a device acos (the trick K3 uses for sqrt).  The wrap is pairs.cuh's
// minimum-image step under the interactions rule (wrap_fast_if, with wrap_axis_if for flagged pairs).
#include <cmath>
#include <cstring>

#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "pairs.cuh"

namespace mkb {

// the record word of a gathered donor / acceptor: bit0: sel1 != 0, bit1: sel1 == 1, bit2: sel2 == 1, bits 3..31: the atom
// index itself (n_atoms < 2^29), so the pair loop needs no second load
struct HbTag {
    const unsigned *sel1, *sel2;
    __device__ unsigned operator()(long long a) const {
        const unsigned s1 = sel1[a], s2 = sel2[a];
        return (s1 != 0u ? 1u : 0u) | (s1 == 1u ? 2u : 0u) | (s2 == 1u ? 4u : 0u) | ((unsigned)a << 3);
    }
};

// pyx:88-94, kept out of line: the exact step is the rare path of the pair loop
__device__ __noinline__ float hb_rewrap(float val, float b, float hb) { return wrap_axis_if(val, b, hb); }

struct HbArgs {
    const float4 *GA;        // [F][na] acceptors
    const float4 *GD;        // [F][nd][2] donor heavy atom, donor hydrogen
    const unsigned *donors;  // [nd][2]
    const unsigned *acceptors;
    const float *box;
    long long F, fsb, nd, na;
    float thr2, cstar;
    int intra, ignore_hs;
};

template <bool FILL>
__global__ void __launch_bounds__(256) hbond_kernel(const HbArgs A, long long *__restrict__ counts,
                                                    const long long *__restrict__ row_offsets,
                                                    int *__restrict__ triples) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= A.F * A.nd) return;
    const long long f = row / A.nd, d = row - f * A.nd;
    const float4 ph = A.GD[row * 2], pH = A.GD[row * 2 + 1];
    const unsigned d_heavy = A.donors[2 * d], d_hyd = A.donors[2 * d + 1];
    const unsigned dbits = __float_as_uint(ph.w);
    // read by hand rather than through load_box, which made this kernel about 1 % slower on an H100 (C10)
    const float bx = A.box[f], by = A.box[A.fsb + f], bz = A.box[2 * A.fsb + f];
    const float hx = __fdiv_rn(bx, 2.f), hy = __fdiv_rn(by, 2.f), hz = __fdiv_rn(bz, 2.f);
    const float rbx = __frcp_rn(bx), rby = __frcp_rn(by), rbz = __frcp_rn(bz);
    const float4 pd = A.ignore_hs ? ph : pH;  // the atom whose distance to the acceptor is tested (pyx:60-64)
    // heavy -> hydrogen vector: the same for every acceptor of the row (pyx:107-114)
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, d2b = 0.f;
    if (!A.ignore_hs) {
        b0 = hb_rewrap(__fsub_rn(ph.x, pH.x), bx, hx);
        b1 = hb_rewrap(__fsub_rn(ph.y, pH.y), by, hy);
        b2 = hb_rewrap(__fsub_rn(ph.z, pH.z), bz, hz);
        d2b = sq3(b0, b1, b2);
    }
    long long base = FILL ? row_offsets[row] : 0;
    const long long row_end = FILL ? row_offsets[row + 1] : 0;
    if (FILL && base == row_end) return;  // most (frame, donor) rows have no bond: the count pass already knows
    long long total = 0;
    const float4 *ga = A.GA + f * A.na;
    const int na = (int)A.na;
    for (int a0 = 0; a0 < na; a0 += 32) {
        const int a = a0 + lane;
        bool hit = false;
        unsigned a_idx = 0;
        if (a < na) {
            const float4 pa = ga[a];
            const unsigned abits = __float_as_uint(pa.w);
            a_idx = abits >> 3;
            bool ok = a_idx != d_heavy;                                            // pyx:67-68
            if (A.intra) ok = ok && (abits & 1u) && (dbits & 1u);                  // pyx:70-73
            else ok = ok && (((abits & 2u) && (dbits & 4u)) || ((abits & 4u) && (dbits & 2u)));  // pyx:74-77
            if (ok) {
                const float v0 = __fsub_rn(pa.x, pd.x), v1 = __fsub_rn(pa.y, pd.y), v2 = __fsub_rn(pa.z, pd.z);
                bool risky = false;
                float a0v = wrap_fast_if(v0, bx, rbx, hx, risky);
                float a1v = wrap_fast_if(v1, by, rby, hy, risky);
                float a2v = wrap_fast_if(v2, bz, rbz, hz, risky);
                if (risky) {  // quotient next to a half-integer, or huge: the exactly rounded division
                    a0v = hb_rewrap(v0, bx, hx); a1v = hb_rewrap(v1, by, hy); a2v = hb_rewrap(v2, bz, hz);
                }
                const float d2a = sq3(a0v, a1v, a2v);
                if (!(d2a > A.thr2)) {                                             // pyx:97-98 (NaN passes, as there)
                    if (A.ignore_hs) {
                        hit = true;                                                // pyx:101-105
                    } else if (!(d2a == 0.f || d2b == 0.f)) {                      // pyx:117-118
                        float dot = __fadd_rn(0.f, __fmul_rn(a0v, b0));
                        dot = __fadd_rn(dot, __fmul_rn(a1v, b1));
                        dot = __fadd_rn(dot, __fmul_rn(a2v, b2));
                        float c = __double2float_rn(
                            __ddiv_rn((double)dot, (double)__fmul_rn(__fsqrt_rn(d2a), __fsqrt_rn(d2b))));  // sqrtf * sqrtf in float
                        if (c > 1.f) c = 1.f;
                        if (c < -1.f) c = -1.f;
                        hit = c <= A.cstar;                                        // acosf(c) > angle threshold
                    }
                }
            }
        }
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (FILL) {
            if (hit) {
                int *o = triples + 3 * (base + __popc(m & ((1u << lane) - 1u)));
                o[0] = (int)d_heavy;
                o[1] = A.ignore_hs ? -1 : (int)d_hyd;
                o[2] = (int)a_idx;
            }
            base += __popc(m);
            if (base == row_end) break;  // every bond of the row is out (warp-uniform)
        } else {
            total += __popc(m);
        }
    }
    if (!FILL && lane == 0) counts[row] = total;
}

__global__ void hb_set_last_zero(long long *p, long long n) {
    if (threadIdx.x == 0 && blockIdx.x == 0) p[n] = 0;
}

// largest float c in [-1, 1] with acosf(c) > athr (host libm = the reference's); -inf when none.  glibc's acosf is
// non-increasing over all 2.13e9 floats of [-1, 1] (tests/test_interaction_cutoffs_cpu.py walks them all with the host
// libm), so one bound is exact.
static float hb_cos_threshold(float athr) {
    auto passes = [&](float c) { return acosf(c) > athr; };
    if (!passes(-1.f)) return -INFINITY;
    if (passes(1.f)) return 1.f;
    auto key = [](float x) {  // order-preserving integer image of a float
        int32_t b;
        memcpy(&b, &x, 4);
        return b >= 0 ? (long long)b : -(long long)(b & 0x7fffffff);
    };
    auto unkey = [](long long k) {
        int32_t b = k >= 0 ? (int32_t)k : (int32_t)(0x80000000u | (uint32_t)(-k));
        float x;
        memcpy(&x, &b, 4);
        return x;
    };
    long long lo = key(-1.f), hi = key(1.f);  // lo passes, hi fails
    while (hi - lo > 1) {
        const long long mid = lo + (hi - lo) / 2;
        if (passes(unkey(mid))) lo = mid; else hi = mid;
    }
    return unkey(lo);
}

static int hb_setup(mkb_ctx *h, cudaStream_t st, const mkb_traj *t, const uint32_t *donors, int64_t n_donors,
                    const uint32_t *acceptors, int64_t n_acceptors, const uint32_t *sel1, const uint32_t *sel2,
                    float dist_threshold, float angle_threshold, int32_t intra, int32_t ignore_hs, HbArgs *A) {
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory view");
    if (t->n_atoms < 0 || t->n_frames < 0 || n_donors < 0 || n_acceptors < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (t->n_frames > 0 && (!t->coords || !t->box)) return fail(h, MKB_ERR_BAD_ARG, "null coords/box");
    if (t->frame_stride < t->n_frames || t->frame_stride_box < t->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame_stride smaller than n_frames");
    const long long F = t->n_frames, rows = F * n_donors;
    if (rows >= (1ll << 31) / 32) return fail(h, MKB_ERR_BAD_ARG, "frames x donors too large for one call (%lld)", rows);
    if (t->n_atoms >= (1ll << 29) || n_acceptors >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_atoms must be < 2^29");
    A->F = F; A->fsb = t->frame_stride_box; A->nd = n_donors; A->na = n_acceptors;
    A->box = t->box; A->donors = donors; A->acceptors = acceptors;
    A->thr2 = dist_threshold * dist_threshold;                                            // pyx:49 (float product)
    A->cstar = hb_cos_threshold((float)((double)angle_threshold / 57.29578));             // pyx:50
    A->intra = intra ? 1 : 0; A->ignore_hs = ignore_hs ? 1 : 0;
    A->GA = A->GD = nullptr;
    if (rows == 0 || n_acceptors == 0) return MKB_OK;
    if (!donors || !acceptors || !sel1 || !sel2) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    float4 *G;
    int rc;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)(F * (n_acceptors + 2 * n_donors)), &G))) return rc;
    A->GA = G;
    A->GD = G + F * n_acceptors;
    const unsigned gx = (unsigned)cdiv(F, 32);
    const long long gya = cdiv(n_acceptors, 32), gyd = cdiv(2 * n_donors, 32);
    if (gya > 65535 || gyd > 65535) return fail(h, MKB_ERR_BAD_ARG, "too many donors / acceptors for one call");
    gather_kernel<unsigned, HbTag><<<dim3(gx, (unsigned)gya), dim3(32, 8), 0, st>>>(t->coords, t->frame_stride, F, acceptors,
                                                                                    n_acceptors, HbTag{sel1, sel2}, G);
    MKB_LAUNCHED(h);
    gather_kernel<unsigned, HbTag><<<dim3(gx, (unsigned)gyd), dim3(32, 8), 0, st>>>(t->coords, t->frame_stride, F, donors,
                                                                                    2 * n_donors, HbTag{sel1, sel2},
                                                                                    G + F * n_acceptors);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_hbonds_count(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *donors,
                                int64_t n_donors, const uint32_t *acceptors, int64_t n_acceptors, const uint32_t *sel1,
                                const uint32_t *sel2, float dist_threshold, float angle_threshold, int32_t intra,
                                int32_t ignore_hs, int64_t *row_offsets, int64_t *total_triples) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets || !total_triples) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/total_triples");
    HbArgs A;
    int rc = hb_setup(h, st, t, donors, n_donors, acceptors, n_acceptors, sel1, sel2, dist_threshold, angle_threshold,
                      intra, ignore_hs, &A);
    if (rc) return rc;
    const long long rows = A.F * A.nd;
    long long *counts;
    if ((rc = scratch_get(h, S_ROWCNT, (size_t)rows + 1, &counts))) return rc;
    if (rows > 0) {
        if (A.na > 0) {
            hbond_kernel<false><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(A, counts, nullptr, nullptr);
            MKB_LAUNCHED(h);
        } else {
            MKB_CUDA(h, cudaMemsetAsync(counts, 0, (size_t)rows * sizeof(long long), st));
        }
    }
    hb_set_last_zero<<<1, 32, 0, st>>>(counts, rows);
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
    *total_triples = total;
    h->last_kernel = "hbond_kernel";
    return MKB_OK;
}

extern "C" int mkb_hbonds_fill(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *donors,
                               int64_t n_donors, const uint32_t *acceptors, int64_t n_acceptors, const uint32_t *sel1,
                               const uint32_t *sel2, float dist_threshold, float angle_threshold, int32_t intra,
                               int32_t ignore_hs, const int64_t *row_offsets, int32_t *triples) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets");
    HbArgs A;
    int rc = hb_setup(h, st, t, donors, n_donors, acceptors, n_acceptors, sel1, sel2, dist_threshold, angle_threshold,
                      intra, ignore_hs, &A);
    if (rc) return rc;
    const long long rows = A.F * A.nd;
    if (rows == 0 || A.na == 0) return MKB_OK;
    if (!triples) return fail(h, MKB_ERR_BAD_ARG, "null triples");
    hbond_kernel<true><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(A, nullptr, (const long long *)row_offsets, triples);
    MKB_LAUNCHED(h);
    return MKB_OK;
}
