// distance.cu -- K3/K4/K5/K6: trajectory distances, ordered contacts, group reductions, cdist/pdist for sm_90a (H100).
//
// Replaces moleculekit/distance_utils/distance_utils.pyx (all functions) with the post-ops of
// moleculekit/projections/util.py:74-84,212-223 fused into the stores.
//
// Data flow (not the reference's frame/i/j triple loop):
//   gather   the selected atoms of the frame-minor trajectory (N,3,F) are transposed once, through shared memory,
//            into frame-major float4 rows G[f][k] = (x, y, z, chain-id bits): reads are coalesced along frames, writes
//            along atoms.  This is ~3 % extra traffic for the dense kernels and makes every later access coalesced.
//   K3       CTA = (frame, 16 rows of sel1, 256 columns of sel2); a thread keeps its sel2 atom in registers, sel1 atoms
//            arrive by L1 broadcast, stores are 128-byte coalesced rows of the (F, P) matrix; truncate / `<= threshold`
//            are applied in the store (float32 or uint8 output).
//   K4       one warp per (frame, i) row: ballot + popc gives the row count (pass 1) and, after a cub scan, the
//            ORDERED position of every hit (pass 2) -> output order identical to the reference's nested loops.
//   K5       COM pre-pass (one thread per (frame, group), sequential float sums in atom order = reference bits),
//            then one warp per (frame, group pair) min-reduction.
// Bit parity: the reference binary has no FMA and rounds every float op; so do we (__fmul_rn/__fadd_rn/..., roundf
// half-away via an exactly-rounded quotient on the rare near-half cases, __fsqrt_rn).
#include <cub/device/device_scan.cuh>

#include <cmath>
#include <cstring>

#include "common.cuh"

namespace mkb {

// d - b * roundf(d / b) with every op rounded to float (distance_utils.pyx:50-52).
// Fast path: q~ = d * (1/b) differs from fl(d/b) by <= 2 ulp, and round-to-nearest-integer of q~ (magic-number add)
// equals roundf(fl(d/b)) unless a half-integer lies within that error; those cases (and huge / non-finite quotients)
// take the exact division + roundf.
__device__ __forceinline__ float wrap_axis(float d, float b, float rb) {
    const float q = __fmul_rn(d, rb);
    float n = __fsub_rn(__fadd_rn(q, 12582912.0f), 12582912.0f);
    const float fr = fabsf(__fsub_rn(q, n));
    const float lim = fmaf(-6e-7f, fabsf(q), 0.5f);  // negative for |q| > 8e5 -> always exact path; NaN -> exact path
    if (!(fr < lim)) n = roundf(__fdiv_rn(d, b));
    return __fsub_rn(d, __fmul_rn(b, n));
}

__device__ __forceinline__ float sq3(float dx, float dy, float dz) {
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

struct BoxF {
    float bx, by, bz, rx, ry, rz;
    float hx, hy, hz;  // b / 2
};

__device__ __forceinline__ BoxF load_box(const float *box, long long stride, long long f) {
    BoxF b;
    b.bx = box[f];
    b.by = box[stride + f];
    b.bz = box[2 * stride + f];
    b.rx = __frcp_rn(b.bx);
    b.ry = __frcp_rn(b.by);
    b.rz = __frcp_rn(b.bz);
    b.hx = __fmul_rn(b.bx, 0.5f); b.hy = __fmul_rn(b.by, 0.5f); b.hz = __fmul_rn(b.bz, 0.5f);
    asm volatile("" : "+f"(b.hx), "+f"(b.hy), "+f"(b.hz));  // keep the halves in registers (else recomputed per pair)
    return b;
}

// squared distance of two gathered atoms, distance_utils.pyx:34-54 (_dist) / :188-206 (_dist2)
__device__ __forceinline__ float pair_d2(const float4 a, const float4 b, const BoxF &bx, bool wrap) {
    float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
    if (wrap) {
        dx = wrap_axis(dx, bx.bx, bx.rx);
        dy = wrap_axis(dy, bx.by, bx.ry);
        dz = wrap_axis(dz, bx.bz, bx.rz);
    }
    return sq3(dx, dy, dz);
}

// store with the fused host post-ops of projections/util.py:74-84: results[results > truncate] = truncate, then
// (contacts) results <= threshold.  NaN distances stay NaN / compare false exactly like numpy.
constexpr int DIST_CONTACTS_D2 = 2;  // internal: contacts without truncate, decided on d2 <= T (no sqrt), see contact_d2_threshold

template <int MODE>
__device__ __forceinline__ void store_dist(void *out, long long idx, float d, float truncate, float threshold) {
    if (d > truncate) d = truncate;  // truncate = NaN disables (comparison false)
    if (MODE == MKB_DIST_CONTACTS) reinterpret_cast<unsigned char *>(out)[idx] = (d <= threshold) ? 1 : 0;
    else reinterpret_cast<float *>(out)[idx] = d;
}

// ---------------------------------------------------------------------------------------------------------
// gather + transpose: G[f][k] = (coords[idx[k], 0..2, f], chain bits) ; 32 frames x 32 atoms per CTA
// ---------------------------------------------------------------------------------------------------------
template <typename IdxT>
__global__ void gather_kernel(const float *__restrict__ coords, long long stride, long long n_frames,
                              const IdxT *__restrict__ idx, long long n, const unsigned *__restrict__ tag,
                              float4 *__restrict__ G) {
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
            const unsigned t = tag ? tag[(long long)idx[k]] : 0u;
            G[f * n + k] = make_float4(tile[0][lane][ff], tile[1][lane][ff], tile[2][lane][ff], __uint_as_float(t));
        }
    }
}

template <typename IdxT>
static int launch_gather(mkb_ctx *h, cudaStream_t st, const mkb_traj *t, const IdxT *idx, int64_t n,
                         const unsigned *tag, float4 *G) {
    if (n == 0 || t->n_frames == 0) return MKB_OK;
    dim3 grid((unsigned)cdiv(t->n_frames, 32), (unsigned)cdiv(n, 32));
    if (grid.y > 65535) return fail(h, MKB_ERR_BAD_ARG, "selection too large (%lld atoms)", (long long)n);
    gather_kernel<IdxT><<<grid, dim3(32, 8), 0, st>>>(t->coords, t->frame_stride, t->n_frames, idx, n, tag, G);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// K3: dense distances.  grid = (col tiles, row tiles, frames)
// ---------------------------------------------------------------------------------------------------------
constexpr int K3_ROWS = 16;
constexpr int K3_COLS = 256;

// Minimum-image step of the dense kernels: n = rint(d * fl(1/b)) by the magic-number trick, w = d - fl(b n) exactly as
// the reference rounds it (pyx:41-49), and ONE test that n is the reference's roundf(fl(d / b)):  |w| < b/2 - 1e-6 |d|.
// If the two integers differed, d/b would lie within 2e-7 |d/b| of a half-integer, hence |w| >= b/2 - 3e-7 |d| and the
// test fails; exact ties (|w| == b/2: half-away vs half-even), |d/b| >= 2^22 (magic rounding invalid), NaN and boxes
// that are zero / negative / non-finite fail it as well.  One rare branch per PAIR then redoes the flagged pair with the
// general wrap_axis (exact division).  7 instructions per axis instead of 9 for the former quotient-distance test.
__device__ __forceinline__ float wrap_fast(float d, float b, float rb, float hb, bool &risky) {
    const float q = __fmul_rn(d, rb);
    const float n = __fsub_rn(__fadd_rn(q, 12582912.0f), 12582912.0f);
    const float w = __fsub_rn(d, __fmul_rn(b, n));
    risky = risky | !(fabsf(w) < fmaf(-1e-6f, fabsf(d), hb));
    return w;
}

__device__ __forceinline__ float pair_d2_fastwrap(const float4 a, const float4 b, unsigned cb, const BoxF &bx, int pbc) {
    float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
    if (pbc && (__float_as_uint(a.w) != cb)) {
        bool risky = false;
        const float wx = wrap_fast(dx, bx.bx, bx.rx, bx.hx, risky), wy = wrap_fast(dy, bx.by, bx.ry, bx.hy, risky),
                    wz = wrap_fast(dz, bx.bz, bx.rz, bx.hz, risky);
        if (risky) {
            dx = wrap_axis(dx, bx.bx, bx.rx);
            dy = wrap_axis(dy, bx.by, bx.ry);
            dz = wrap_axis(dz, bx.bz, bx.rz);
        } else {
            dx = wx; dy = wy; dz = wz;
        }
    }
    return sq3(dx, dy, dz);
}

// K3 hot loop variant: the rare exact re-wrap is an out-of-line call (the inlined form merged its registers back with a
// dozen MOV / BSSY / BSYNC per pair), the half boxes live in registers, and the threshold folds |d| in with one FFMA:
//   risky  <=>  |w| + 1e-6 |d| >= b/2  on some axis   (the same test as wrap_fast, rearranged)
__device__ __noinline__ float pair_d2_rewrap(float dx, float dy, float dz, float bxx, float bxy, float bxz, float rx, float ry, float rz) {
    return sq3(wrap_axis(dx, bxx, rx), wrap_axis(dy, bxy, ry), wrap_axis(dz, bxz, rz));
}
__device__ __forceinline__ float pair_d2_lean(const float4 a, const float4 b, unsigned cb, const BoxF &bx, int pbc) {
    const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
    if (!(pbc && (__float_as_uint(a.w) != cb))) return sq3(dx, dy, dz);
    const float nx = __fsub_rn(__fadd_rn(__fmul_rn(dx, bx.rx), 12582912.0f), 12582912.0f);
    const float ny = __fsub_rn(__fadd_rn(__fmul_rn(dy, bx.ry), 12582912.0f), 12582912.0f);
    const float nz = __fsub_rn(__fadd_rn(__fmul_rn(dz, bx.rz), 12582912.0f), 12582912.0f);
    const float wx = __fsub_rn(dx, __fmul_rn(bx.bx, nx)), wy = __fsub_rn(dy, __fmul_rn(bx.by, ny)), wz = __fsub_rn(dz, __fmul_rn(bx.bz, nz));
    const bool safe = (fmaf(1e-6f, fabsf(dx), fabsf(wx)) < bx.hx) & (fmaf(1e-6f, fabsf(dy), fabsf(wy)) < bx.hy) &
                      (fmaf(1e-6f, fabsf(dz), fabsf(wz)) < bx.hz);
    if (!safe) return pair_d2_rewrap(dx, dy, dz, bx.bx, bx.by, bx.bz, bx.rx, bx.ry, bx.rz);
    return sq3(wx, wy, wz);
}

// same with the wrap decision made by the caller (group chains, K5)
__device__ __forceinline__ float pair_d2_fastwrap_flag(const float4 a, const float4 b, const BoxF &bx, bool wrap) {
    float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
    if (wrap) {
        bool risky = false;
        const float wx = wrap_fast(dx, bx.bx, bx.rx, bx.hx, risky), wy = wrap_fast(dy, bx.by, bx.ry, bx.hy, risky),
                    wz = wrap_fast(dz, bx.bz, bx.rz, bx.hz, risky);
        if (risky) {
            dx = wrap_axis(dx, bx.bx, bx.rx);
            dy = wrap_axis(dy, bx.by, bx.ry);
            dz = wrap_axis(dz, bx.bz, bx.rz);
        } else {
            dx = wx; dy = wy; dz = wz;
        }
    }
    return sq3(dx, dy, dz);
}

// Contact maps only need the BOOLEAN d2 <= T of the reference's float32 sequence, not its bits.  A fused estimate of d2
// (3 instead of 8 instructions per axis) decides every pair whose estimate lies outside a 4e-6 band around T; pairs inside
// the band, pairs with NaN / out-of-range quotients, and whole frames whose box is too small for the shortcut take the exact
// sequence.  Why this is the reference's answer: (a) when the estimate's image integer n equals the reference's
// roundf(fl(d/b)), the two d2 differ by < 1e-6 relative (a handful of float roundings); (b) when the integers differ, d/b
// is within 1e-6 of a half-integer, so |w| >= b/2 (1 - 1e-5) in BOTH computations and both d2 exceed T as long as
// (b/2)^2 (1 - 1e-4) > T -- checked once per frame (`shortcut`), else the exact sequence is used throughout.
__device__ __forceinline__ bool contact_shortcut_ok(const BoxF &bx, float T) {
    const float m = fminf(fminf(bx.hx, bx.hy), bx.hz);
    return m * m * (1.0f - 1e-4f) > T;  // false for NaN / zero / negative boxes as well
}
__device__ __forceinline__ bool pair_contact(const float4 a, const float4 b, unsigned cb, const BoxF &bx, int pbc, float T,
                                             bool shortcut) {
    if (shortcut) {
        float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
        float qm = 0.0f;
        if (pbc && (__float_as_uint(a.w) != cb)) {
            const float qx = dx * bx.rx, qy = dy * bx.ry, qz = dz * bx.rz;
            dx = fmaf(-bx.bx, (qx + 12582912.0f) - 12582912.0f, dx);
            dy = fmaf(-bx.by, (qy + 12582912.0f) - 12582912.0f, dy);
            dz = fmaf(-bx.bz, (qz + 12582912.0f) - 12582912.0f, dz);
            qm = fmaxf(fmaxf(fabsf(qx), fabsf(qy)), fabsf(qz));
        }
        const float d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz));
        // decided unless the estimate is within the band, not a number, or the magic rounding left its range
        if (fabsf(d2 - T) > 4e-6f * T && qm < 2097152.0f) return d2 <= T;
    }
    return pair_d2_fastwrap(a, b, cb, bx, pbc) <= T;
}

// MKB_DIST_DISTANCES_FAST: float32 distances within 4 ulp of the reference's sequence instead of its exact bits.
// The minimum-image step keeps the reference's own roundings, w = fl(d - fl(b n)) with n = rint(d * fl(1/b)) -- so w is
// bit-identical whenever n is the reference's roundf(fl(d/b)), and when the two integers differ (d/b within 2e-7 of a
// half-integer) both |w| are b/2 (1 -+ 4e-7).  What is dropped: the test for that case, the unfused sum of squares
// (two FFMA instead of four roundings) and the correctly rounded square root (MUFU.SQRT, <= 1 ulp + flush of subnormal
// d2 to 0).  Same NaN behaviour (zero / non-finite boxes); quotients |d/b| >= 2^22 are outside the magic rounding's range.
// 21 instead of 48 instructions per pair: the kernel becomes HBM-store bound.
__device__ __forceinline__ float pair_d2_quick(const float4 a, const float4 b, unsigned cb, const BoxF &bx, int pbc) {
    float dx = a.x - b.x, dy = a.y - b.y, dz = a.z - b.z;
    if (pbc && (__float_as_uint(a.w) != cb)) {
        const float nx = __fsub_rn(fmaf(dx, bx.rx, 12582912.0f), 12582912.0f);
        const float ny = __fsub_rn(fmaf(dy, bx.ry, 12582912.0f), 12582912.0f);
        const float nz = __fsub_rn(fmaf(dz, bx.rz, 12582912.0f), 12582912.0f);
        dx = __fsub_rn(dx, __fmul_rn(bx.bx, nx));
        dy = __fsub_rn(dy, __fmul_rn(bx.by, ny));
        dz = __fsub_rn(dz, __fmul_rn(bx.bz, nz));
    }
    return fmaf(dx, dx, fmaf(dy, dy, dz * dz));
}
__device__ __forceinline__ float sqrt_quick(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
constexpr int DIST_QUICK = MKB_DIST_DISTANCES_FAST;

template <int MODE>
__device__ __forceinline__ float pair_d2_of(const float4 a, const float4 b, unsigned cb, const BoxF &bx, int pbc) {
    return MODE == DIST_QUICK ? pair_d2_quick(a, b, cb, bx, pbc) : pair_d2_fastwrap(a, b, cb, bx, pbc);
}

template <int MODE, bool TRUNC = true>
__device__ __forceinline__ void emit_dist(void *out, long long idx, float d2, float truncate, float threshold) {
    if (MODE == DIST_QUICK) {
        float d = sqrt_quick(d2);
        if (TRUNC && d > truncate) d = truncate;
        reinterpret_cast<float *>(out)[idx] = d;
    } else if (MODE == DIST_CONTACTS_D2) reinterpret_cast<unsigned char *>(out)[idx] = (d2 <= threshold) ? 1 : 0;
    else if (MODE == MKB_DIST_DISTANCES && !TRUNC) reinterpret_cast<float *>(out)[idx] = __fsqrt_rn(d2);  // no truncate given
    else store_dist<MODE>(out, idx, __fsqrt_rn(d2), truncate, threshold);
}

// Each thread owns TWO sel2 columns (j and j + K3_COLS) so one broadcast load of the sel1 atom, the loop control and the
// index arithmetic are shared by two pairs.  SELF / PBC are compile-time: the rectangular non-periodic-free inner loop
// carries no per-row diagonal tests.
#ifdef MKB_K3_MIN_CTAS
#define MKB_K3_BOUNDS __launch_bounds__(K3_COLS, MKB_K3_MIN_CTAS)
#else
#define MKB_K3_BOUNDS __launch_bounds__(K3_COLS)
#endif
template <int MODE, bool SELF, bool TRUNC = true>
__global__ void MKB_K3_BOUNDS dist_kernel(const float4 *__restrict__ G1, const float4 *__restrict__ G2,
                                                        long long n1, long long n2, const float *__restrict__ box,
                                                        long long box_stride, int pbc, float truncate,
                                                        float threshold, long long P, void *__restrict__ out,
                                                        long long frame0) {
    const long long f = frame0 + blockIdx.z;
    const long long j0 = (long long)blockIdx.x * (2 * K3_COLS) + threadIdx.x, j1 = j0 + K3_COLS;
    const long long i0 = (long long)blockIdx.y * K3_ROWS;
    if (SELF && (long long)(blockIdx.x + 1) * (2 * K3_COLS) <= i0 + 1) return;  // tile entirely below the diagonal
    if (j0 >= n2) return;
    const bool has1 = j1 < n2;
    const float4 b0 = G2[f * n2 + j0];
    const float4 b1 = has1 ? G2[f * n2 + j1] : b0;
    const unsigned cb0 = __float_as_uint(b0.w), cb1 = __float_as_uint(b1.w);
    const BoxF bx = load_box(box, box_stride, f);
    const int rows = (int)(min(i0 + K3_ROWS, n1) - i0);
    const float4 *__restrict__ arow = G1 + f * n1 + i0;
    if (MODE == DIST_CONTACTS_D2) {  // boolean map: fused estimate + exact re-check in the band (pair_contact)
        const bool shortcut = contact_shortcut_ok(bx, threshold);
        unsigned char *const o8 = reinterpret_cast<unsigned char *>(out);
        long long idx = f * P + (SELF ? (i0 * n2 - (i0 * (i0 + 1)) / 2 + (j0 - i0 - 1)) : (i0 * n2 + j0));
        long long step = SELF ? n2 - i0 - 2 : n2;
#pragma unroll 2
        for (int r = 0; r < rows; ++r) {
            const float4 a = __ldg(arow + r);
            if (!SELF || j0 > i0 + r) o8[idx] = pair_contact(a, b0, cb0, bx, pbc, threshold, shortcut) ? 1 : 0;
            if (has1 && (!SELF || j1 > i0 + r)) o8[idx + K3_COLS] = pair_contact(a, b1, cb1, bx, pbc, threshold, shortcut) ? 1 : 0;
            idx += step;
            if (SELF) --step;
        }
        return;
    }
    // running output index: non-self (i, j) -> i*n2 + j ; self -> i*n2 - i(i+1)/2 + (j - i - 1), step n2 - i - 2
    long long idx = f * P + (SELF ? (i0 * n2 - (i0 * (i0 + 1)) / 2 + (j0 - i0 - 1)) : (i0 * n2 + j0));
    if (SELF) {
        long long step = n2 - i0 - 2;
#pragma unroll 2
        for (int r = 0; r < rows; ++r) {
            const float4 a = __ldg(arow + r);
            if (j0 > i0 + r) emit_dist<MODE>(out, idx, pair_d2_of<MODE>(a, b0, cb0, bx, pbc), truncate, threshold);
            if (has1 && j1 > i0 + r)
                emit_dist<MODE>(out, idx + K3_COLS, pair_d2_of<MODE>(a, b1, cb1, bx, pbc), truncate, threshold);
            idx += step;
            --step;
        }
    } else if (has1) {
#pragma unroll 2
        for (int r = 0; r < rows; ++r) {
            const float4 a = __ldg(arow + r);
            emit_dist<MODE, TRUNC>(out, idx, MODE == DIST_QUICK ? pair_d2_quick(a, b0, cb0, bx, pbc) : pair_d2_lean(a, b0, cb0, bx, pbc), truncate, threshold);
            emit_dist<MODE, TRUNC>(out, idx + K3_COLS, MODE == DIST_QUICK ? pair_d2_quick(a, b1, cb1, bx, pbc) : pair_d2_lean(a, b1, cb1, bx, pbc), truncate, threshold);
            idx += n2;
        }
    } else {
        for (int r = 0; r < rows; ++r) {
            emit_dist<MODE>(out, idx, pair_d2_of<MODE>(__ldg(arow + r), b0, cb0, bx, pbc), truncate, threshold);
            idx += n2;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// K4: ordered contacts.  One warp per (frame, i) row.  FILL = false: counts; FILL = true: ordered write.
// ---------------------------------------------------------------------------------------------------------
// BAL: 0 = no ballot buffer; 1 = count pass that also SAVES one ballot word per (row, 32-column chunk); 2 = fill pass that
// READS those words instead of evaluating the distances again.
template <bool FILL, int BAL>
__global__ void __launch_bounds__(256) contacts_kernel(const float4 *__restrict__ G1, const float4 *__restrict__ G2,
                                                       long long n1, long long n2, long long n_frames,
                                                       const float *__restrict__ box, long long box_stride,
                                                       int selfdist, int pbc, float thr2,
                                                       const unsigned *__restrict__ sel1,
                                                       const unsigned *__restrict__ sel2,
                                                       long long *__restrict__ row_counts,
                                                       const long long *__restrict__ row_offsets,
                                                       unsigned *__restrict__ pairs, unsigned *__restrict__ ballots) {
    const int lane = threadIdx.x & 31;
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_frames * n1) return;
    const long long f = row / n1, i = row - f * n1;
    const long long chunks = (n2 + 31) >> 5;
    const unsigned s1 = FILL ? sel1[i] : 0u;
    long long pos = FILL ? row_offsets[row] : 0;
    long long cnt = 0;
    const long long jstart = selfdist ? i + 1 : 0;
    if (BAL == 2) {
        const unsigned *rb = ballots + row * chunks;
        for (long long c0 = jstart >> 5; c0 < chunks; c0 += 32) {  // 32 chunk words per coalesced load
            const unsigned mine = c0 + lane < chunks ? rb[c0 + lane] : 0u;
            unsigned nz = __ballot_sync(0xffffffffu, mine != 0u);
            while (nz) {
                const int k = __ffs(nz) - 1;
                nz &= nz - 1;
                const unsigned bal = __shfl_sync(0xffffffffu, mine, k);
                if ((bal >> lane) & 1u) {
                    const long long p = pos + __popc(bal & ((1u << lane) - 1u));
                    pairs[2 * p + 0] = s1;
                    pairs[2 * p + 1] = sel2[((c0 + k) << 5) + lane];
                }
                pos += __popc(bal);
            }
        }
        return;
    }
    const float4 a = G1[f * n1 + i];
    const BoxF bx = load_box(box, box_stride, f);
    for (long long jb = jstart - (jstart & 31); jb < n2; jb += 32) {  // aligned chunks keep loads coalesced
        const long long j = jb + lane;
        bool hit = false;
        if (j >= jstart && j < n2) {
            const float4 b = G2[f * n2 + j];
            hit = pair_d2_fastwrap(a, b, __float_as_uint(b.w), bx, pbc) <= thr2;  // distance_utils.pyx:90
        }
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (BAL == 1 && lane == 0) ballots[row * chunks + (jb >> 5)] = bal;
        if (FILL) {
            if (hit) {
                const long long p = pos + __popc(bal & ((1u << lane) - 1u));
                pairs[2 * p + 0] = s1;
                pairs[2 * p + 1] = sel2[j];
            }
            pos += __popc(bal);
        } else {
            cnt += __popc(bal);
        }
    }
    if (!FILL && lane == 0) row_counts[row] = cnt;
}

// get_collisions (distance_utils.pyx:98-121): single frame, row-major (n,3) inputs, local indices
template <bool FILL>
__global__ void __launch_bounds__(256) collisions_kernel(const float *__restrict__ c1, long long n1,
                                                         const float *__restrict__ c2, long long n2, float thr2,
                                                         long long *__restrict__ row_counts,
                                                         const long long *__restrict__ row_offsets,
                                                         unsigned *__restrict__ pairs) {
    const int lane = threadIdx.x & 31;
    const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n1) return;
    const float ax = c1[3 * i], ay = c1[3 * i + 1], az = c1[3 * i + 2];
    long long pos = FILL ? row_offsets[i] : 0, cnt = 0;
    for (long long jb = 0; jb < n2; jb += 32) {
        const long long j = jb + lane;
        bool hit = false;
        if (j < n2)
            hit = sq3(__fsub_rn(ax, c2[3 * j]), __fsub_rn(ay, c2[3 * j + 1]), __fsub_rn(az, c2[3 * j + 2])) <= thr2;
        const unsigned bal = __ballot_sync(0xffffffffu, hit);
        if (FILL) {
            if (hit) {
                const long long p = pos + __popc(bal & ((1u << lane) - 1u));
                pairs[2 * p + 0] = (unsigned)i;
                pairs[2 * p + 1] = (unsigned)j;
            }
            pos += __popc(bal);
        } else {
            cnt += __popc(bal);
        }
    }
    if (!FILL && lane == 0) row_counts[i] = cnt;
}

// ---------------------------------------------------------------------------------------------------------
// K8 (SURVEY 8f row 2): MetricShell -- radial shell histogram fused onto the distance evaluation.
// Replaces the O(F*P) numpy post-pass of moleculekit/projections/metricshell.py:183-202 (_shells) AND the (F, P)
// distance matrix it needed: counts[f][c][e] = #partners j with edges[e] < d(c, j) <= edges[e+1], d = the reference's
// truncated float32 distance compared in float64 like numpy does (float32 array vs float64 edges).
// One warp per (frame, centre); lane e keeps the count of shell e (numshells <= 32).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) shell_kernel(const float4 *__restrict__ G1, const float4 *__restrict__ G2,
                                                    long long n1, long long n2, long long n_frames,
                                                    const float *__restrict__ box, long long box_stride, int selfdist,
                                                    int pbc, float truncate, const double *__restrict__ edges,
                                                    int numshells, unsigned *__restrict__ counts) {
    const int lane = threadIdx.x & 31;
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= n_frames * n1) return;
    const long long f = row / n1, c = row - f * n1;
    const float4 a = G1[f * n1 + c];
    const BoxF bx = load_box(box, box_stride, f);
    const double lo_mine = lane < numshells ? edges[lane] : 0.0, hi_mine = lane < numshells ? edges[lane + 1] : 0.0;
    unsigned mine = 0;
    for (long long jb = 0; jb < n2; jb += 32) {
        const long long j = jb + lane;
        const bool valid = j < n2 && !(selfdist && j == c);
        double d = 0.0;
        if (valid) {
            const float4 b = G2[f * n2 + j];
            float df = __fsqrt_rn(pair_d2_fastwrap(a, b, __float_as_uint(b.w), bx, pbc));
            if (df > truncate) df = truncate;  // projections/util.py:74-75 before the histogram
            d = (double)df;
        }
        for (int e = 0; e < numshells; ++e) {
            const double lo = __shfl_sync(0xffffffffu, lo_mine, e), hi = __shfl_sync(0xffffffffu, hi_mine, e);
            const unsigned bal = __ballot_sync(0xffffffffu, valid && d > lo && d <= hi);  // NaN: both false
            if (lane == e) mine += __popc(bal);
        }
    }
    if (lane < numshells) counts[row * numshells + lane] = mine;
}

__global__ void set_last_zero(long long *p, long long n) {
    if (threadIdx.x == 0 && blockIdx.x == 0) p[n] = 0;
}

static int scan_i64(mkb_ctx *h, cudaStream_t st, long long *in, long long *out, long long n) {
    if (n >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many rows for one call (%lld)", n);
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, in, out, (int)n, st));
    void *tmp = nullptr;
    int rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp);
    if (rc) return rc;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, in, out, (int)n, st));
    h->launches++;
    return MKB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// K5: group reductions
// ---------------------------------------------------------------------------------------------------------
// _calc_com (distance_utils.pyx:160-183): sequential float sums in atom order, product rounded before the add.
__global__ void com_kernel(const float4 *__restrict__ G, long long nflat, long long n_frames,
                           const long long *__restrict__ off, long long ngroups, const int *__restrict__ atoms,
                           const float *__restrict__ masses, float4 *__restrict__ com) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_frames * ngroups) return;
    const long long f = t / ngroups, g = t - f * ngroups;
    float tm = 0.f, cx = 0.f, cy = 0.f, cz = 0.f;
    for (long long k = off[g]; k < off[g + 1]; ++k) {
        const float4 p = G[f * nflat + k];
        const float m = masses[atoms[k]];
        cx = __fadd_rn(cx, __fmul_rn(p.x, m));
        cy = __fadd_rn(cy, __fmul_rn(p.y, m));
        cz = __fadd_rn(cz, __fmul_rn(p.z, m));
        tm = __fadd_rn(tm, m);
    }
    com[t] = make_float4(__fdiv_rn(cx, tm), __fdiv_rn(cy, tm), __fdiv_rn(cz, tm), 0.f);
}

template <int MODE>
__global__ void __launch_bounds__(256) reduction_kernel(const float4 *__restrict__ G1, long long nflat1,
                                                        const float4 *__restrict__ G2, long long nflat2,
                                                        const float4 *__restrict__ com1,
                                                        const float4 *__restrict__ com2,
                                                        const long long *__restrict__ off1, long long NG1,
                                                        const long long *__restrict__ off2, long long NG2,
                                                        const unsigned *__restrict__ gch1,
                                                        const unsigned *__restrict__ gch2, long long n_frames,
                                                        const float *__restrict__ box, long long box_stride,
                                                        int selfdist, int pbc, int red1, int red2, int pairs,
                                                        float truncate, float threshold, long long P,
                                                        void *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long per_frame = pairs ? NG1 : NG1 * NG2;
    if (w >= n_frames * per_frame) return;
    const long long f = w / per_frame, r = w - f * per_frame;
    long long a, b, col;
    if (pairs) { a = r; b = r; col = r; }
    else {
        a = r / NG2; b = r - a * NG2;
        if (selfdist) { if (b <= a) return; col = a * NG2 - (a * (a + 1)) / 2 + (b - a - 1); }
        else col = r;
    }
    const bool wrap = pbc && (gch1[a] != gch2[b]);
    const BoxF bx = load_box(box, box_stride, f);
    const long long s1 = off1[a], m1 = red1 ? 1 : off1[a + 1] - s1;
    const long long s2 = off2[b], m2 = red2 ? 1 : off2[b + 1] - s2;
    const long long total = m1 * m2;
    float best = INFINITY;  // min over non-NaN candidates
    float first = 0.f;      // d2 of the first pair: the reference always takes it (mindist = -1 sentinel, pyx:260-275)
    for (long long p = lane; p < total; p += 32) {
        const long long ia = p / m2, ib = p - ia * m2;
        const float4 pa = red1 ? com1[f * NG1 + a] : G1[f * nflat1 + s1 + ia];
        const float4 pb = red2 ? com2[f * NG2 + b] : G2[f * nflat2 + s2 + ib];
        const float d2 = pair_d2(pa, pb, bx, wrap);
        if (p == 0) first = d2;
        if (d2 < best) best = d2;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) best = fminf(best, __shfl_xor_sync(0xffffffffu, best, o));
    first = __shfl_sync(0xffffffffu, first, 0);
    if (lane == 0) {
        float m;
        if (total <= 0) m = -1.f;             // empty group: sqrt(-1) = NaN like the reference
        else if (first != first) m = first;   // a NaN first element sticks (all later `<` comparisons are false)
        else m = best;
        store_dist<MODE>(out, f * P + col, __fsqrt_rn(m), truncate, threshold);
    }
}

// Small groups (residue - residue minimum distances: ~100 atom pairs per group pair): ONE THREAD per (frame, group pair)
// walks the m1 x m2 atom pairs itself -- every lane busy, no shuffle reduction, no index divisions in the loop.  Threads of
// a warp share group a (broadcast loads) and take consecutive groups b.  Same semantics as reduction_kernel.
template <int MODE>
__global__ void __launch_bounds__(128) reduction_thread_kernel(const float4 *__restrict__ G1, long long nflat1,
                                                                const float4 *__restrict__ G2, long long nflat2,
                                                                const float4 *__restrict__ com1,
                                                                const float4 *__restrict__ com2,
                                                                const long long *__restrict__ off1, long long NG1,
                                                                const long long *__restrict__ off2, long long NG2,
                                                                const unsigned *__restrict__ gch1,
                                                                const unsigned *__restrict__ gch2, long long n_frames,
                                                                const float *__restrict__ box, long long box_stride,
                                                                int selfdist, int pbc, int red1, int red2, int pairs,
                                                                float truncate, float threshold, long long P,
                                                                void *__restrict__ out) {
    const long long per_frame = pairs ? NG1 : NG1 * NG2;
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long f = blockIdx.y;
    if (r >= per_frame) return;
    long long a, b, col;
    if (pairs) { a = r; b = r; col = r; }
    else {
        a = r / NG2; b = r - a * NG2;
        if (selfdist) { if (b <= a) return; col = a * NG2 - (a * (a + 1)) / 2 + (b - a - 1); }
        else col = r;
    }
    const bool wrap = pbc && (gch1[a] != gch2[b]);
    const BoxF bx = load_box(box, box_stride, f);
    const long long s1 = off1[a], s2 = off2[b];
    const int m1 = red1 ? 1 : (int)(off1[a + 1] - s1), m2 = red2 ? 1 : (int)(off2[b + 1] - s2);
    const float4 *pa0 = red1 ? com1 + f * NG1 + a : G1 + f * nflat1 + s1;
    const float4 *pb0 = red2 ? com2 + f * NG2 + b : G2 + f * nflat2 + s2;
    float best = INFINITY, first = 0.f;
    for (int ia = 0; ia < m1; ++ia) {
        const float4 pa = __ldg(pa0 + ia);
        for (int ib = 0; ib < m2; ++ib) {
            const float d2 = pair_d2_fastwrap_flag(pa, __ldg(pb0 + ib), bx, wrap);
            if ((ia | ib) == 0) first = d2;
            if (d2 < best) best = d2;
        }
    }
    float m;
    if (m1 <= 0 || m2 <= 0) m = -1.f;     // empty group: sqrt(-1) = NaN like the reference
    else if (first != first) m = first;   // a NaN first element sticks (all later `<` comparisons are false)
    else m = best;
    store_dist<MODE>(out, f * P + col, __fsqrt_rn(m), truncate, threshold);
}

// ---------------------------------------------------------------------------------------------------------
// K6: cdist / pdist / squareform
// ---------------------------------------------------------------------------------------------------------
__global__ void cdist_kernel(const float *__restrict__ a, long long n1, const float *__restrict__ b, long long n2, int D,
                             float *__restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (j >= n2 || i >= n1) return;
    float s = 0.f;
    for (int k = 0; k < D; ++k) {
        const float d = __fsub_rn(a[i * D + k], b[j * D + k]);
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    out[i * n2 + j] = __fsqrt_rn(s);
}

__global__ void pdist_kernel(const float *__restrict__ a, long long n, int D, float *__restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (j >= n || j <= i) return;
    float s = 0.f;
    for (int k = 0; k < D; ++k) {
        const float d = __fsub_rn(a[i * D + k], a[j * D + k]);
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    out[i * n - (i * (i + 1)) / 2 + (j - i - 1)] = __fsqrt_rn(s);
}

__global__ void squareform_kernel(const float *__restrict__ d, long long dim, float *__restrict__ out) {
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long i = blockIdx.y;
    if (j >= dim || i >= dim) return;
    float v = 0.f;
    if (i != j) {
        const long long lo = min(i, j), hi = max(i, j);
        v = d[lo * dim - (lo * (lo + 1)) / 2 + (hi - lo - 1)];
    }
    out[i * dim + j] = v;
}

static int check_traj(mkb_ctx *h, const mkb_traj *t) {
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory view");
    if (t->n_atoms < 0 || t->n_frames < 0) return fail(h, MKB_ERR_BAD_ARG, "negative trajectory size");
    if (t->n_frames > 0 && (!t->coords || !t->box)) return fail(h, MKB_ERR_BAD_ARG, "null coords/box");
    if (t->frame_stride < t->n_frames || t->frame_stride_box < t->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame_stride smaller than n_frames");
    return MKB_OK;
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_dist_trajectory(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                                   const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist,
                                   int32_t pbc, int32_t mode, float truncate, float threshold, void *out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    int rc = check_traj(h, t);
    if (rc) return rc;
    if (n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative selection size");
    if (mode != MKB_DIST_DISTANCES && mode != MKB_DIST_CONTACTS && mode != MKB_DIST_DISTANCES_FAST)
        return fail(h, MKB_ERR_BAD_ARG, "bad mode %d", mode);
    if (selfdist && n1 != n2) return fail(h, MKB_ERR_BAD_ARG, "selfdist needs sel1 == sel2");
    const long long P = selfdist ? (n1 * (n2 - 1)) / 2 : n1 * n2;
    if (t->n_frames == 0 || P <= 0) return MKB_OK;
    if (!sel1 || !sel2 || !chains || !out) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    float4 *G;
    const long long F = t->n_frames;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)(F * (n1 + n2)), &G))) return rc;
    float4 *G1 = G, *G2 = G + F * n1;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    if ((rc = launch_gather<uint32_t>(h, st, t, sel1, n1, chains, G1))) return rc;
    if ((rc = launch_gather<uint32_t>(h, st, t, sel2, n2, chains, G2))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const unsigned gx = (unsigned)cdiv(n2, 2 * K3_COLS), gy = (unsigned)cdiv(n1, K3_ROWS);
    if (gy > 65535) return fail(h, MKB_ERR_BAD_ARG, "sel1 too large for one call (%lld)", (long long)n1);
    // contacts without truncate: sqrtf(d2) <= thr  <=>  d2 <= T with T the largest float whose correctly rounded square
    // root is <= thr -- the comparison moves to d2 and the square root disappears (NaN compares false either way)
    int kmode = mode;
    float kthr = threshold;
    if (mode == MKB_DIST_CONTACTS && std::isnan(truncate) && threshold >= 0.0f && std::isfinite(threshold)) {
        float T = threshold * threshold;
        while (sqrtf(T) > threshold) T = nextafterf(T, -INFINITY);
        while (sqrtf(nextafterf(T, INFINITY)) <= threshold) T = nextafterf(T, INFINITY);
        kmode = DIST_CONTACTS_D2;
        kthr = T;
    }
    for (long long f0 = 0; f0 < F; f0 += 65535) {
        const unsigned gz = (unsigned)std::min<long long>(65535, F - f0);
        dim3 grid(gx, gy, gz);
#define MKB_K3_LAUNCH(M, S)                                                                                       \
    dist_kernel<M, S><<<grid, K3_COLS, 0, st>>>(G1, G2, n1, n2, t->box, t->frame_stride_box, pbc, truncate, kthr, P, out, f0)
        if (kmode == MKB_DIST_DISTANCES) {
            if (selfdist) MKB_K3_LAUNCH(MKB_DIST_DISTANCES, true);
            else if (truncate != truncate)  // NaN = no truncate: the rectangular kernel without the compare / select per pair
                dist_kernel<MKB_DIST_DISTANCES, false, false><<<grid, K3_COLS, 0, st>>>(G1, G2, n1, n2, t->box, t->frame_stride_box, pbc, truncate, kthr, P, out, f0);
            else MKB_K3_LAUNCH(MKB_DIST_DISTANCES, false);
        } else if (kmode == MKB_DIST_CONTACTS) {
            if (selfdist) MKB_K3_LAUNCH(MKB_DIST_CONTACTS, true); else MKB_K3_LAUNCH(MKB_DIST_CONTACTS, false);
        } else if (kmode == DIST_QUICK) {
            if (selfdist) MKB_K3_LAUNCH(DIST_QUICK, true);
            else if (truncate != truncate)
                dist_kernel<DIST_QUICK, false, false><<<grid, K3_COLS, 0, st>>>(G1, G2, n1, n2, t->box, t->frame_stride_box, pbc, truncate, kthr, P, out, f0);
            else MKB_K3_LAUNCH(DIST_QUICK, false);
        } else {
            if (selfdist) MKB_K3_LAUNCH(DIST_CONTACTS_D2, true); else MKB_K3_LAUNCH(DIST_CONTACTS_D2, false);
        }
#undef MKB_K3_LAUNCH
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

static int contacts_common(mkb_ctx *h, cudaStream_t st, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                           const uint32_t *sel2, int64_t n2, const uint32_t *chains, float4 **G1, float4 **G2) {
    int rc = check_traj(h, t);
    if (rc) return rc;
    if (n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative selection size");
    if (t->n_frames * n1 > 0 && (!sel1 || !sel2 || !chains)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    float4 *G;
    const long long F = t->n_frames;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)std::max<long long>(F * (n1 + n2), 1), &G))) return rc;
    *G1 = G;
    *G2 = G + F * n1;
    if ((rc = launch_gather<uint32_t>(h, st, t, sel1, n1, chains, *G1))) return rc;
    if ((rc = launch_gather<uint32_t>(h, st, t, sel2, n2, chains, *G2))) return rc;
    return MKB_OK;
}

extern "C" int mkb_contacts_count(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                                  const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist,
                                  int32_t pbc, float threshold, int64_t *row_offsets, int64_t *total_pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets || !total_pairs) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/total_pairs");
    float4 *G1, *G2;
    int rc = contacts_common(h, st, t, sel1, n1, sel2, n2, chains, &G1, &G2);
    if (rc) return rc;
    const long long rows = t->n_frames * n1;
    long long *counts;
    if ((rc = scratch_get(h, S_ROWCNT, (size_t)rows + 1, &counts))) return rc;
    const float thr2 = threshold * threshold;  // float product, distance_utils.pyx:77
    h->k4_key.valid = false;
    if (rows > 0) {
        // one ballot word per (row, 32 columns) for the fill call that follows -- unless that would be excessive
        const long long chunks = (n2 + 31) / 32;
        const long long words = rows * chunks;
        unsigned *ballots = nullptr;
        if (words > 0 && words <= (1ll << 29) && !getenv("MKB_K4_NO_BALLOTS")) {
            if ((rc = scratch_get(h, S_K4_BALLOTS, (size_t)words, &ballots))) return rc;
        }
        if (ballots) {
            contacts_kernel<false, 1><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(
                G1, G2, n1, n2, t->n_frames, t->box, t->frame_stride_box, selfdist, pbc, thr2, sel1, sel2, counts,
                nullptr, nullptr, ballots);
            mkb_ctx::K4Key &k = h->k4_key;
            k.coords = t->coords; k.box = t->box; k.sel1 = sel1; k.sel2 = sel2; k.chains = chains;
            k.F = t->n_frames; k.n1 = n1; k.n2 = n2; k.fs = t->frame_stride; k.fsb = t->frame_stride_box;
            k.selfdist = selfdist; k.pbc = pbc;
            memcpy(&k.thr_bits, &threshold, sizeof(float));
            k.valid = true;
        } else {
            contacts_kernel<false, 0><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(
                G1, G2, n1, n2, t->n_frames, t->box, t->frame_stride_box, selfdist, pbc, thr2, sel1, sel2, counts,
                nullptr, nullptr, nullptr);
        }
        MKB_LAUNCHED(h);
    }
    set_last_zero<<<1, 32, 0, st>>>(counts, rows);
    MKB_LAUNCHED(h);
    if ((rc = scan_i64(h, st, counts, (long long *)row_offsets, rows + 1))) return rc;
    long long total = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&total, row_offsets + rows, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    *total_pairs = total;
    return MKB_OK;
}

extern "C" int mkb_contacts_fill(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                                 const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist,
                                 int32_t pbc, float threshold, const int64_t *row_offsets, uint32_t *pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!row_offsets) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets");
    int rc = check_traj(h, t);
    if (rc) return rc;
    if (n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative selection size");
    const long long rows = t->n_frames * n1;
    if (rows == 0) return MKB_OK;
    if (!pairs) return fail(h, MKB_ERR_BAD_ARG, "null pairs");
    const float thr2 = threshold * threshold;
    // the count call with exactly these arguments left its hit masks behind: emit the pairs from them (row_offsets were
    // computed from the same masks, so the two stay consistent whatever happened to the coordinates in between)
    mkb_ctx::K4Key now;
    now.coords = t->coords; now.box = t->box; now.sel1 = sel1; now.sel2 = sel2; now.chains = chains;
    now.F = t->n_frames; now.n1 = n1; now.n2 = n2; now.fs = t->frame_stride; now.fsb = t->frame_stride_box;
    now.selfdist = selfdist; now.pbc = pbc;
    memcpy(&now.thr_bits, &threshold, sizeof(float));
    now.valid = true;
    if (h->k4_key.same(now) && h->scratch[S_K4_BALLOTS].ptr) {
        if (!sel1 || !sel2) return fail(h, MKB_ERR_BAD_ARG, "null argument");
        contacts_kernel<true, 2><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(
            nullptr, nullptr, n1, n2, t->n_frames, nullptr, 0, selfdist, pbc, thr2, sel1, sel2, nullptr,
            (const long long *)row_offsets, pairs, static_cast<unsigned *>(h->scratch[S_K4_BALLOTS].ptr));
        MKB_LAUNCHED(h);
        h->k4_key.valid = false;  // one fill per count
        return MKB_OK;
    }
    float4 *G1, *G2;
    if ((rc = contacts_common(h, st, t, sel1, n1, sel2, n2, chains, &G1, &G2))) return rc;
    contacts_kernel<true, 0><<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(
        G1, G2, n1, n2, t->n_frames, t->box, t->frame_stride_box, selfdist, pbc, thr2, sel1, sel2, nullptr,
        (const long long *)row_offsets, pairs, nullptr);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_dist_reduction(mkb_handle_t h, void *stream, const mkb_traj *t, const int64_t *g1_off,
                                  const int32_t *g1_atoms, int64_t NG1, const int64_t *g2_off,
                                  const int32_t *g2_atoms, int64_t NG2, const uint32_t *gchains1,
                                  const uint32_t *gchains2, int32_t selfdist, int32_t pbc, const float *masses,
                                  int32_t red1, int32_t red2, int32_t pairs, int32_t mode, float truncate,
                                  float threshold, void *out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    int rc = check_traj(h, t);
    if (rc) return rc;
    if (NG1 < 0 || NG2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative group count");
    if (mode != MKB_DIST_DISTANCES && mode != MKB_DIST_CONTACTS) return fail(h, MKB_ERR_BAD_ARG, "bad mode %d", mode);
    if (pairs && NG1 != NG2) return fail(h, MKB_ERR_BAD_ARG, "pairs mode needs as many groups in both sets");
    if (selfdist && NG1 != NG2) return fail(h, MKB_ERR_BAD_ARG, "selfdist needs identical group sets");
    const long long P = pairs ? NG1 : (selfdist ? (NG1 * (NG2 - 1)) / 2 : NG1 * NG2);
    const long long F = t->n_frames;
    if (F == 0 || P <= 0) return MKB_OK;
    if (!g1_off || !g2_off || !g1_atoms || !g2_atoms || !gchains1 || !gchains2 || !masses || !out)
        return fail(h, MKB_ERR_BAD_ARG, "null argument");
    // group sizes live on the device; the flat lengths are the last offsets (tiny D2H, synchronising)
    long long nf1 = 0, nf2 = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&nf1, g1_off + NG1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaMemcpyAsync(&nf2, g2_off + NG2, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    if (nf1 < 0 || nf2 < 0) return fail(h, MKB_ERR_BAD_ARG, "bad group offsets");
    float4 *G, *com;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)std::max<long long>(F * (nf1 + nf2), 1), &G))) return rc;
    if ((rc = scratch_get(h, S_COM, (size_t)(F * (NG1 + NG2)), &com))) return rc;
    float4 *G1 = G, *G2 = G + F * nf1, *com1 = com, *com2 = com + F * NG1;
    if ((rc = launch_gather<int32_t>(h, st, t, g1_atoms, nf1, nullptr, G1))) return rc;
    if ((rc = launch_gather<int32_t>(h, st, t, g2_atoms, nf2, nullptr, G2))) return rc;
    if (red1) {
        com_kernel<<<(unsigned)cdiv(F * NG1, 128), 128, 0, st>>>(G1, nf1, F, (const long long *)g1_off, NG1, g1_atoms,
                                                                masses, com1);
        MKB_LAUNCHED(h);
    }
    if (red2) {
        com_kernel<<<(unsigned)cdiv(F * NG2, 128), 128, 0, st>>>(G2, nf2, F, (const long long *)g2_off, NG2, g2_atoms,
                                                                masses, com2);
        MKB_LAUNCHED(h);
    }
    const long long per_frame = pairs ? NG1 : NG1 * NG2;
    const long long warps = F * per_frame;
    // average atom pairs per group pair decides the work decomposition: small groups -> one thread per group pair
    const double avg_pairs = (double)(red1 ? NG1 : nf1) / (double)std::max<long long>(NG1, 1) *
                             (double)(red2 ? NG2 : nf2) / (double)std::max<long long>(NG2, 1);
    const bool thread_per_pair = avg_pairs <= 512.0 && per_frame >= 4096 && F <= 65535 && !getenv("MKB_K5_WARP");
    if (thread_per_pair) {
        const dim3 grid((unsigned)cdiv(per_frame, 128), (unsigned)F);
        if (mode == MKB_DIST_DISTANCES)
            reduction_thread_kernel<MKB_DIST_DISTANCES><<<grid, 128, 0, st>>>(
                G1, nf1, G2, nf2, com1, com2, (const long long *)g1_off, NG1, (const long long *)g2_off, NG2, gchains1,
                gchains2, F, t->box, t->frame_stride_box, selfdist, pbc, red1, red2, pairs, truncate, threshold, P, out);
        else
            reduction_thread_kernel<MKB_DIST_CONTACTS><<<grid, 128, 0, st>>>(
                G1, nf1, G2, nf2, com1, com2, (const long long *)g1_off, NG1, (const long long *)g2_off, NG2, gchains1,
                gchains2, F, t->box, t->frame_stride_box, selfdist, pbc, red1, red2, pairs, truncate, threshold, P, out);
        MKB_LAUNCHED(h);
        return MKB_OK;
    }
    if (warps * 32 / 256 >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many group pairs for one call");
    const unsigned nb = (unsigned)cdiv(warps * 32, 256);
    if (mode == MKB_DIST_DISTANCES)
        reduction_kernel<MKB_DIST_DISTANCES><<<nb, 256, 0, st>>>(
            G1, nf1, G2, nf2, com1, com2, (const long long *)g1_off, NG1, (const long long *)g2_off, NG2, gchains1,
            gchains2, F, t->box, t->frame_stride_box, selfdist, pbc, red1, red2, pairs, truncate, threshold, P, out);
    else
        reduction_kernel<MKB_DIST_CONTACTS><<<nb, 256, 0, st>>>(
            G1, nf1, G2, nf2, com1, com2, (const long long *)g1_off, NG1, (const long long *)g2_off, NG2, gchains1,
            gchains2, F, t->box, t->frame_stride_box, selfdist, pbc, red1, red2, pairs, truncate, threshold, P, out);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_cdist(mkb_handle_t h, void *stream, const float *a, int64_t n1, const float *b, int64_t n2,
                         int32_t D, float *out) {
    MKB_ENTER(h);
    if (n1 < 0 || n2 < 0 || D < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n1 == 0 || n2 == 0) return MKB_OK;
    if (!a || !b || !out) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (n1 > 65535) return fail(h, MKB_ERR_BAD_ARG, "cdist: at most 65535 rows per call");
    cdist_kernel<<<dim3((unsigned)cdiv(n2, 128), (unsigned)n1), 128, 0, (cudaStream_t)stream>>>(a, n1, b, n2, D, out);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_pdist(mkb_handle_t h, void *stream, const float *a, int64_t n, int32_t D, float *out) {
    MKB_ENTER(h);
    if (n < 0 || D < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n < 2) return MKB_OK;
    if (!a || !out) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (n > 65535) return fail(h, MKB_ERR_BAD_ARG, "pdist: at most 65535 points per call");
    pdist_kernel<<<dim3((unsigned)cdiv(n, 128), (unsigned)n), 128, 0, (cudaStream_t)stream>>>(a, n, D, out);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_squareform(mkb_handle_t h, void *stream, const float *d, int64_t n, int64_t dim, float *out) {
    MKB_ENTER(h);
    if (n < 0 || dim < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (dim == 0) return MKB_OK;
    if (!out || (n > 0 && !d)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (dim * (dim - 1) / 2 > n) return fail(h, MKB_ERR_BAD_ARG, "condensed vector too short for dim %lld", (long long)dim);
    if (dim > 65535) return fail(h, MKB_ERR_BAD_ARG, "squareform: dim too large");
    squareform_kernel<<<dim3((unsigned)cdiv(dim, 128), (unsigned)dim), 128, 0, (cudaStream_t)stream>>>(d, dim, out);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_collisions_count(mkb_handle_t h, void *stream, const float *c1, int64_t n1, const float *c2,
                                    int64_t n2, float threshold, int64_t *row_offsets, int64_t *total_pairs) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (!row_offsets || !total_pairs) return fail(h, MKB_ERR_BAD_ARG, "null row_offsets/total_pairs");
    if (n1 > 0 && n2 > 0 && (!c1 || !c2)) return fail(h, MKB_ERR_BAD_ARG, "null coordinates");
    long long *counts;
    int rc;
    if ((rc = scratch_get(h, S_ROWCNT, (size_t)n1 + 1, &counts))) return rc;
    const float thr2 = threshold * threshold;
    if (n1 > 0) {
        collisions_kernel<false><<<(unsigned)cdiv(n1 * 32, 256), 256, 0, st>>>(c1, n1, c2, n2, thr2, counts, nullptr,
                                                                               nullptr);
        MKB_LAUNCHED(h);
    }
    set_last_zero<<<1, 32, 0, st>>>(counts, n1);
    MKB_LAUNCHED(h);
    if ((rc = scan_i64(h, st, counts, (long long *)row_offsets, n1 + 1))) return rc;
    long long total = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&total, row_offsets + n1, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    *total_pairs = total;
    return MKB_OK;
}

extern "C" int mkb_collisions_fill(mkb_handle_t h, void *stream, const float *c1, int64_t n1, const float *c2,
                                   int64_t n2, float threshold, const int64_t *row_offsets, uint32_t *pairs) {
    MKB_ENTER(h);
    if (n1 < 0 || n2 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n1 == 0 || n2 == 0) return MKB_OK;
    if (!c1 || !c2 || !row_offsets || !pairs) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    const float thr2 = threshold * threshold;
    collisions_kernel<true><<<(unsigned)cdiv(n1 * 32, 256), 256, 0, (cudaStream_t)stream>>>(
        c1, n1, c2, n2, thr2, nullptr, (const long long *)row_offsets, pairs);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_shell_counts(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel1, int64_t n1,
                                const uint32_t *sel2, int64_t n2, const uint32_t *chains, int32_t selfdist,
                                int32_t pbc, float truncate, const double *edges, int32_t numshells,
                                uint32_t *counts) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (numshells < 1 || numshells > 32) return fail(h, MKB_ERR_BAD_ARG, "numshells=%d: 1..32 supported", numshells);
    if (selfdist && n1 != n2) return fail(h, MKB_ERR_BAD_ARG, "selfdist needs sel1 == sel2");
    float4 *G1, *G2;
    int rc = contacts_common(h, st, t, sel1, n1, sel2, n2, chains, &G1, &G2);
    if (rc) return rc;
    const long long rows = t->n_frames * n1;
    if (rows == 0) return MKB_OK;
    if (!edges || !counts) return fail(h, MKB_ERR_BAD_ARG, "null edges/counts");
    shell_kernel<<<(unsigned)cdiv(rows * 32, 256), 256, 0, st>>>(G1, G2, n1, n2, t->n_frames, t->box,
                                                                 t->frame_stride_box, selfdist, pbc, truncate, edges,
                                                                 numshells, counts);
    MKB_LAUNCHED(h);
    return MKB_OK;
}
