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
// tests c <= c* -- the same booleans without a device acos (the trick K3 uses for sqrt).
#include <cmath>
#include <cstring>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace mkb {

// G[f][k] = (coords[idx[k], 0..2, f], tag of idx[k]); tag bit0: sel1 != 0, bit1: sel1 == 1, bit2: sel2 == 1, bits 3..31: the
// atom index itself (n_atoms < 2^29), so the pair loop needs no second load
__global__ void hb_gather_kernel(const float *__restrict__ coords, long long stride, long long n_frames,
                                 const unsigned *__restrict__ idx, long long n, const unsigned *__restrict__ sel1,
                                 const unsigned *__restrict__ sel2, float4 *__restrict__ G) {
    __shared__ float tile[3][32][33];
    const long long f0 = (long long)blockIdx.x * 32, k0 = (long long)blockIdx.y * 32;
    const int lane = threadIdx.x, row = threadIdx.y;  // blockDim = (32, 8)
    for (int kk = row; kk < 32; kk += 8) {
        const long long k = k0 + kk, f = f0 + lane;
        if (k < n && f < n_frames) {
            const long long a = (long long)idx[k];
#pragma unroll
            for (int d = 0; d < 3; ++d) tile[d][kk][lane] = coords[(a * 3 + d) * stride + f];
        }
    }
    __syncthreads();
    for (int ff = row; ff < 32; ff += 8) {
        const long long f = f0 + ff, k = k0 + lane;
        if (k < n && f < n_frames) {
            const long long a = (long long)idx[k];
            const unsigned s1 = sel1[a], s2 = sel2[a];
            const unsigned t = (s1 != 0u ? 1u : 0u) | (s1 == 1u ? 2u : 0u) | (s2 == 1u ? 4u : 0u) | ((unsigned)a << 3);
            G[f * n + k] = make_float4(tile[0][lane][ff], tile[1][lane][ff], tile[2][lane][ff], __uint_as_float(t));
        }
    }
}

// pyx:88-94: one component of a minimum-image vector, every operation rounded to float (general path)
__device__ __noinline__ float hb_wrap_exact(float val, float b, float hb) {
    if (fabsf(val) > hb && b != 0.f) val = __fsub_rn(val, __fmul_rn(b, roundf(__fdiv_rn(val, b))));
    return val;
}

// Branch-free form of the same step for the pair loop: K3's wrap_fast (csrc/distance.cu).  n = rint(val * fl(1/b)) by the
// magic-number trick, r = val - fl(b n) as the reference rounds it, and ONE test that n is the reference's
// roundf(fl(val / b)):  |r| < b/2 - 1e-6 |val|.  Were the integers different, val / b would lie within 2e-7 of a half-integer
// and |r| >= b/2 - 3e-7 |val|.  Exact ties, |val / b| >= 2^22, NaN and non-positive boxes fail the test; such pairs set
// `risky` and are redone with hb_wrap_exact.  No wrap (|val| <= b/2 or b == 0) leaves val untouched, as there.
__device__ __forceinline__ float hb_wrap_fast(float val, float b, float rb, float hb, bool &risky) {
    const bool w = fabsf(val) > hb && b != 0.f;
    const float MAGIC = 12582912.f;  // 1.5 * 2^23
    const float n = __fsub_rn(__fadd_rn(__fmul_rn(val, rb), MAGIC), MAGIC);
    const float r = __fsub_rn(val, __fmul_rn(b, n));
    risky = risky || (w && !(fabsf(r) < __fmaf_rn(-1e-6f, fabsf(val), hb)));
    return w ? r : val;
}

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
    const float bx = A.box[f], by = A.box[A.fsb + f], bz = A.box[2 * A.fsb + f];
    const float hx = __fdiv_rn(bx, 2.f), hy = __fdiv_rn(by, 2.f), hz = __fdiv_rn(bz, 2.f);
    const float rbx = __frcp_rn(bx), rby = __frcp_rn(by), rbz = __frcp_rn(bz);
    const float4 pd = A.ignore_hs ? ph : pH;  // the atom whose distance to the acceptor is tested (pyx:60-64)
    // heavy -> hydrogen vector: the same for every acceptor of the row (pyx:107-114)
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, d2b = 0.f;
    if (!A.ignore_hs) {
        b0 = hb_wrap_exact(__fsub_rn(ph.x, pH.x), bx, hx);
        b1 = hb_wrap_exact(__fsub_rn(ph.y, pH.y), by, hy);
        b2 = hb_wrap_exact(__fsub_rn(ph.z, pH.z), bz, hz);
        d2b = __fadd_rn(__fadd_rn(__fmul_rn(b0, b0), __fmul_rn(b1, b1)), __fmul_rn(b2, b2));
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
                float a0v = hb_wrap_fast(v0, bx, rbx, hx, risky);
                float a1v = hb_wrap_fast(v1, by, rby, hy, risky);
                float a2v = hb_wrap_fast(v2, bz, rbz, hz, risky);
                if (risky) {  // quotient next to a half-integer, or huge: the exactly rounded division
                    a0v = hb_wrap_exact(v0, bx, hx); a1v = hb_wrap_exact(v1, by, hy); a2v = hb_wrap_exact(v2, bz, hz);
                }
                const float d2a = __fadd_rn(__fadd_rn(__fmul_rn(a0v, a0v), __fmul_rn(a1v, a1v)), __fmul_rn(a2v, a2v));
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
// non-increasing over all 2.13e9 floats of [-1, 1] (checked exhaustively on glibc 2.39), so one bound is exact.
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
    hb_gather_kernel<<<dim3(gx, (unsigned)gya), dim3(32, 8), 0, st>>>(t->coords, t->frame_stride, F, acceptors, n_acceptors,
                                                                      sel1, sel2, G);
    MKB_LAUNCHED(h);
    hb_gather_kernel<<<dim3(gx, (unsigned)gyd), dim3(32, 8), 0, st>>>(t->coords, t->frame_stride, F, donors, 2 * n_donors,
                                                                      sel1, sel2, G + F * n_acceptors);
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
