// dihedral.cu -- K16: torsion angles of atom quadruples over a trajectory for sm_90a (H100).
//
// Replaces the per-dihedral numpy loop of MetricDihedral (moleculekit/projections/metricdihedral.py, which calls
// moleculekit.dihedral.dihedralAngle on mol.coords[quad] for every quadruple).  The kernel reads the (N, 3, F)
// frame-minor trajectory with lane = frame (one 128-byte line per (atom, axis) row when the frames are consecutive),
// evaluates every (frame, quadruple) independently in float64 and writes frame-major rows through a shared-memory
// transpose, the layout of the K15 kernels.  No minimum image: the coordinates are used as given.
//
//   geometry    b0 = p0 - p1, b1 = p2 - p1, b2 = p3 - p2, u = b1 / |b1|,
//               v = b0 - (b0.u) u, w = b2 - (b2.u) u, x = v.w, y = (u x v).w, angle = atan2(y, x).
//   convention  IUPAC: looking along p1 -> p2, the angle is positive when the p1-p0 bond turns clockwise (by less than
//               180 degrees) onto the p2-p3 bond; cis = 0, trans = +-pi.  Range [-pi, pi] before the float32 rounding.
//   sin / cos   (y, x) / hypot(x, y), not sin(atan2(..)).
//   degenerate  b0 x b1 = 0 or b1 x b2 = 0, evaluated unfused in float64 (p0, p1, p2 or p1, p2, p3 collinear, or
//               p1 == p2): angle 0 and (sin, cos) = (0, 1), decided before the projected form, which would return
//               rounding noise there.  A non-finite coordinate gives NaN.
//
// A CTA owns 32 listed frames x a block of 64 quadruples.  Consecutive quadruples (phi / psi / chi of neighbouring
// residues) share atoms, so the lines a CTA reads are re-read from L1 rather than from memory.
#include <algorithm>

#include "common.cuh"

namespace mkb {

constexpr int DH_THREADS = 256;
constexpr int DH_WARPS = DH_THREADS / 32;
constexpr int DH_TILE = 64;                    // quadruples per tile
constexpr int DH_PER_WARP = DH_TILE / DH_WARPS;
constexpr int DH_BATCH = 2;                    // quadruples whose 12 coordinates are loaded before any is evaluated

struct DihArgs {
    const float *coords;
    long long fs;
    const int4 *quads;
    long long m;              // quadruples
    const unsigned *frames;
    long long n;              // listed frames
};

// a[i] b[j] - a[j] b[i] in float64 without a fused multiply-add: zero exactly when the two products are equal
__device__ __forceinline__ double dh_cross(const double (&a)[3], const double (&b)[3], int i, int j) {
    return __dsub_rn(__dmul_rn(a[i], b[j]), __dmul_rn(a[j], b[i]));
}

// true when b0 x b1 or b1 x b2 is the zero vector: the bonds are exact float64 differences of the float32 points, and
// equal real products round to equal doubles, so collinear points give exact zeros in any orientation (the projected
// form below leaves rounding noise there, whose atan2 would be an arbitrary angle)
__device__ __forceinline__ bool dh_degenerate(const double (&b0)[3], const double (&b1)[3], const double (&b2)[3]) {
    const bool z1 = dh_cross(b0, b1, 1, 2) == 0.0 && dh_cross(b0, b1, 2, 0) == 0.0 && dh_cross(b0, b1, 0, 1) == 0.0;
    const bool z2 = dh_cross(b1, b2, 1, 2) == 0.0 && dh_cross(b1, b2, 2, 0) == 0.0 && dh_cross(b1, b2, 0, 1) == 0.0;
    return z1 || z2;
}

// fl32 angle, or fl32 (sin, cos), of one quadruple from its four float32 points
template <bool SINCOS>
__device__ __forceinline__ void dh_eval(const float (&p)[4][3], float (&o)[SINCOS ? 2 : 1]) {
    double b0[3], b1[3], b2[3];
    bool finite = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        b0[d] = (double)p[0][d] - (double)p[1][d];
        b1[d] = (double)p[2][d] - (double)p[1][d];
        b2[d] = (double)p[3][d] - (double)p[2][d];
        finite = finite && isfinite(b0[d]) && isfinite(b1[d]) && isfinite(b2[d]);
    }
    double x = 0.0, y = 0.0;
    if (!dh_degenerate(b0, b1, b2)) {  // b1 != 0 here: b1 = 0 makes both cross products zero
        const double s = 1.0 / sqrt(b1[0] * b1[0] + b1[1] * b1[1] + b1[2] * b1[2]);
        const double u[3] = {b1[0] * s, b1[1] * s, b1[2] * s};
        const double a0 = b0[0] * u[0] + b0[1] * u[1] + b0[2] * u[2];
        const double a2 = b2[0] * u[0] + b2[1] * u[1] + b2[2] * u[2];
        const double v[3] = {b0[0] - a0 * u[0], b0[1] - a0 * u[1], b0[2] - a0 * u[2]};
        const double w[3] = {b2[0] - a2 * u[0], b2[1] - a2 * u[1], b2[2] - a2 * u[2]};
        x = v[0] * w[0] + v[1] * w[1] + v[2] * w[2];
        y = (u[1] * v[2] - u[2] * v[1]) * w[0] + (u[2] * v[0] - u[0] * v[2]) * w[1] + (u[0] * v[1] - u[1] * v[0]) * w[2];
    }
    const float nan = __int_as_float(0x7fffffff);
    if constexpr (SINCOS) {
        const double r = hypot(x, y);
        o[0] = !finite ? nan : r > 0.0 ? __double2float_rn(y / r) : 0.f;
        o[1] = !finite ? nan : r > 0.0 ? __double2float_rn(x / r) : 1.f;
    } else {
        o[0] = !finite ? nan : x == 0.0 && y == 0.0 ? 0.f : __double2float_rn(atan2(y, x));  // not atan2(+0, -0) = pi
    }
}

// out[k * ld + NV * j + c] = value c of quadruple j in listed frame k (NV = 1: angle; NV = 2: sin, cos)
template <bool SINCOS>
__global__ void __launch_bounds__(DH_THREADS) dihedral_kernel(const DihArgs A, float *__restrict__ out, long long ld) {
    constexpr int NV = SINCOS ? 2 : 1;
    __shared__ float tile[NV * DH_TILE][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item0 = 32ll * blockIdx.x, item = item0 + lane;
    const bool valid = item < A.n;
    const int rows = A.n - item0 < 32 ? (int)(A.n - item0) : 32;
    const long long f = valid ? (A.frames ? (long long)A.frames[item] : item) : 0;
    const long long nblk = (A.m + DH_TILE - 1) / DH_TILE;
    for (long long b = blockIdx.y; b < nblk; b += gridDim.y) {
        const long long j0 = b * DH_TILE;
        for (int u0 = 0; u0 < DH_PER_WARP; u0 += DH_BATCH) {
            float p[DH_BATCH][4][3];
#pragma unroll
            for (int q = 0; q < DH_BATCH; ++q) {
                const long long j = j0 + w + DH_WARPS * (u0 + q);
                if (valid && j < A.m) {
                    const int4 r = __ldg(A.quads + j);
                    const int row[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
                    for (int a = 0; a < 4; ++a) {
                        const float *src = A.coords + (long long)row[a] * 3 * A.fs + f;
#pragma unroll
                        for (int d = 0; d < 3; ++d) p[q][a][d] = __ldg(src + d * A.fs);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < DH_BATCH; ++q) {
                const int t = w + DH_WARPS * (u0 + q);
                float o[NV];
                if (valid && j0 + t < A.m) {
                    dh_eval<SINCOS>(p[q], o);
                } else {
#pragma unroll
                    for (int c = 0; c < NV; ++c) o[c] = 0.f;
                }
#pragma unroll
                for (int c = 0; c < NV; ++c) tile[NV * t + c][lane] = o[c];
            }
        }
        __syncthreads();
        const long long cols = NV * A.m, c0 = NV * j0;
        for (int kk = w; kk < rows; kk += DH_WARPS) {
            float *o = out + (item0 + kk) * ld + c0;
#pragma unroll
            for (int h = 0; h < NV * DH_TILE / 32; ++h) {
                const int j = 32 * h + lane;
                if (c0 + j < cols) o[j] = tile[j][kk];
            }
        }
        __syncthreads();
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_dihedrals(mkb_handle_t h, void *stream, const mkb_traj *t, const int32_t *quads, int64_t n_quads,
                             const uint32_t *frames, int64_t n_frames, int32_t sincos, float *out, int64_t ld_out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_quads <= 0) return fail(h, MKB_ERR_BAD_ARG, "n_quads must be >= 1");
    if (t->n_frames < 0 || (frames && n_frames < 0)) return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !quads) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (((uintptr_t)quads & 15) != 0) return fail(h, MKB_ERR_BAD_ARG, "quads must be 16-byte aligned");
    if (t->frame_stride < t->n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (sincos != 0 && sincos != 1) return fail(h, MKB_ERR_BAD_ARG, "sincos must be 0 or 1");
    const long long cols = (sincos ? 2 : 1) * n_quads;
    if (ld_out < cols) return fail(h, MKB_ERR_BAD_ARG, "ld_out %lld < %lld output columns", (long long)ld_out, cols);
    DihArgs A;
    A.coords = t->coords; A.fs = t->frame_stride;
    A.quads = reinterpret_cast<const int4 *>(quads); A.m = n_quads;
    A.frames = frames; A.n = frames ? n_frames : t->n_frames;
    if (cdiv(A.n, 32) >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one launch");
    if (A.n == 0) return MKB_OK;
    if (!out) return fail(h, MKB_ERR_BAD_ARG, "null out");
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(A.n, 32), (unsigned)std::min<long long>(cdiv(A.m, DH_TILE), 65535));
    if (sincos) dihedral_kernel<true><<<grid, DH_THREADS, 0, st>>>(A, out, ld_out);
    else dihedral_kernel<false><<<grid, DH_THREADS, 0, st>>>(A, out, ld_out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = sincos ? "dihedral_kernel<sincos>" : "dihedral_kernel<angle>";
    return MKB_OK;
}
