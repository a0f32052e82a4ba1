// pairs.cuh -- what the periodic pair kernels of distance.cu (K3 / K4 / K5 / K8), hbonds.cu (K12) and rings.cu (K13)
// share: the reference's float32 minimum-image step d - fl(b * roundf(fl(d / b))), its fast form with the test that proves
// the two agree, and the tiled gather of selected atoms.  distance_utils wraps every axis of a wrapped pair (wrap_axis,
// wrap_fast); the interactions modules only axes with |d| > b/2 and b != 0 (wrap_axis_if, wrap_fast_if).
// The device code has internal linkage, as in frame_tile.cuh.
#pragma once
#include "common.cuh"

namespace mkb {
namespace {

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

// Branch-free minimum-image step: n = rint(d * fl(1/b)) by the magic-number trick, w = d - fl(b n) exactly as the
// reference rounds it (pyx:41-49), and ONE test that n is the reference's roundf(fl(d / b)):  |w| < b/2 - 1e-6 |d|.
// If the two integers differed, d/b would lie within 2e-7 |d/b| of a half-integer, hence |w| >= b/2 - 3e-7 |d| and the
// test fails; exact ties (|w| == b/2: half-away vs half-even), |d/b| >= 2^22 (magic rounding invalid), NaN and boxes
// that are zero / negative / non-finite fail it as well.  A failed test sets `risky`, and the caller redoes the pair with
// the exact step.  7 instructions per axis.
__device__ __forceinline__ float wrap_fast(float d, float b, float rb, float hb, bool &risky) {
    const float q = __fmul_rn(d, rb);
    const float n = __fsub_rn(__fadd_rn(q, 12582912.0f), 12582912.0f);
    const float w = __fsub_rn(d, __fmul_rn(b, n));
    risky = risky | !(fabsf(w) < fmaf(-1e-6f, fabsf(d), hb));
    return w;
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

// pair_d2's value through wrap_fast, the pair redone with wrap_axis when any axis is flagged; wrapped when pbc is set and
// the chain words of the two atoms differ
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

// the same with the wrap decision made by the caller (group chains, K5); handing the decision to pair_d2_fastwrap instead
// moves the chain test away from the differences and changes the code generated for K3 / K4 / K8
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

// the exact re-wrap of a flagged pair out of line: inlined into a hot loop, it merges its registers back with a dozen
// MOV / BSSY / BSYNC per pair
__device__ __noinline__ float pair_d2_rewrap(float dx, float dy, float dz, float bxx, float bxy, float bxz, float rx, float ry, float rz) {
    return sq3(wrap_axis(dx, bxx, rx), wrap_axis(dy, bxy, ry), wrap_axis(dz, bxz, rz));
}

// The interactions rule: wrap_axis's step through the exactly rounded division, taken only when |v| > b/2 and b != 0.
__device__ __forceinline__ float wrap_axis_if(float v, float b, float hb) {
    if (fabsf(v) > hb && b != 0.f) v = __fsub_rn(v, __fmul_rn(b, roundf(__fdiv_rn(v, b))));
    return v;
}

// wrap_fast's step and test under the interactions rule: v untouched, and never flagged, when it is not wrapped
__device__ __forceinline__ float wrap_fast_if(float v, float b, float rb, float hb, bool &risky) {
    const bool w = fabsf(v) > hb && b != 0.f;
    const float n = __fsub_rn(__fadd_rn(__fmul_rn(v, rb), 12582912.0f), 12582912.0f);
    const float r = __fsub_rn(v, __fmul_rn(b, n));
    risky = risky || (w && !(fabsf(r) < fmaf(-1e-6f, fabsf(v), hb)));
    return w ? r : v;
}

// G[f][k] = (coords[idx[k], 0..2, f], tag(idx[k])): the selected atoms of the frame-minor trajectory (N, 3, F) transposed
// through shared memory into frame-major float4 rows, reads coalesced along frames and writes along atoms.  A CTA of
// (32, 8) threads owns 32 frames x 32 atoms.  Tag maps an atom index to the word stored in .w.
template <typename IdxT, typename Tag>
__global__ void gather_kernel(const float *__restrict__ coords, long long stride, long long n_frames,
                              const IdxT *__restrict__ idx, long long n, const Tag tag, float4 *__restrict__ G) {
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
            const unsigned t = tag((long long)idx[k]);
            G[f * n + k] = make_float4(tile[0][lane][ff], tile[1][lane][ff], tile[2][lane][ff], __uint_as_float(t));
        }
    }
}

}  // namespace
}  // namespace mkb
