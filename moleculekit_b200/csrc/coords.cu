// coords.cu -- K15: aligned coordinate features, frame sums and per-atom fluctuations for sm_90a (H100).
//
// Replaces the host gather of MetricCoordinate (moleculekit/projections/metriccoordinate.py: align, then
// mol.coords[atomsel] transposed to one row per frame) and the squared deviations of MetricFluctuation
// (moleculekit/projections/metricfluctuation.py).  All three kernels read the (N, 3, F) frame-minor trajectory with
// lane = frame (one 128-byte line per (atom, axis) row when the frames are consecutive) and apply the K14 fit record of
// the lane's frame on the fly with fit_transform (common.cuh), the expression align_apply_kernel writes in place: an
// aligned coordinate here has the bits the apply kernel would have written.
//
//   coordinates  coords_kernel: a CTA owns 32 listed frames x a block of 64 selected atoms, transposes through shared
//                memory and writes out[k][d * n + i] with lane = atom (frame-major rows, X block | Y block | Z block).
//   frame sums   coord_sums_partial_kernel + coord_sums_finish_kernel: the same tile over a fixed chunk of 64 listed
//                frames; one thread per (atom, axis) adds the chunk's frames in list order, the finish kernel adds the
//                chunks in order.  The bits depend only on the selection and the ordered frame list.
//   fluctuation  fluct_kernel<GROUPED>: fl32(sum_d (c_d - m_d)^2) per (frame, atom) in float64, or the float64 mean of
//                that over each group of selection positions, rounded once; the same transpose, one value per atom.
//
// K20 (same file, same read): weighted per-frame moments of groups of selection positions, for MetricGyration and
// MetricSphericalCoordinate.
//   moments      moments_partial_kernel + moments_finish_kernel: a CTA owns 32 listed frames and one segment of at most
//                512 positions of one group (segments never straddle groups); its 8 warps split the segment in a fixed
//                interleave and combine in shared memory in warp order; the finish kernel (one thread per (frame,
//                group)) adds the group's segments in order.  Sums of w e and w e^2 run in float64 with e = c - s, s the
//                aligned coordinate of the group's first position in the same frame, so the spread is not lost to the
//                magnitude of the coordinates.  The bits depend only on the selection, groups and weights.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include <math_constants.h>

#include "common.cuh"

namespace mkb {

constexpr int CO_THREADS = 256;
constexpr int CO_WARPS = CO_THREADS / 32;
constexpr int CO_TILE = 64;                   // selected atoms (or groups) per tile
constexpr int CO_PER_WARP = CO_TILE / CO_WARPS;
constexpr int CO_CHUNK = 64;                  // listed frames per frame-sum chunk: fixes the summation order
constexpr int CO_REC = 16;                    // doubles per K14 fit record
constexpr int CO_GROUP_BATCH = 4;             // grouped fluctuation: atoms of a group loaded per round

struct CoordArgs {
    const float *coords;
    long long fs;
    const unsigned *sel;
    long long k;              // selected atoms
    const unsigned *frames;
    long long n;              // listed frames
    const double *rec;        // per listed frame fit records, NULL = no transform
};

// lane's transform: the fit record of listed frame `item` (K14 layout)
struct LaneFit {
    double R[9], pb[3], qb[3];
};

// the lane's frame and (when there are records) its fit record
__device__ __forceinline__ long long co_frame(const CoordArgs &A, long long item, LaneFit &T) {
    if (A.rec) fit_record_load(A.rec + item * CO_REC, T.R, T.pb, T.qb);
    return A.frames ? (long long)A.frames[item] : item;
}

// aligned float32 coordinates of selected atom i in frame f
__device__ __forceinline__ void co_point(const CoordArgs &A, const LaneFit &T, float x0, float x1, float x2,
                                         float (&c)[3]) {
    if (A.rec) {
        fit_transform(T.R, T.pb, T.qb, x0, x1, x2, c);
    } else {
        c[0] = x0; c[1] = x1; c[2] = x2;
    }
}

// aligned coordinates of the tile atoms i0 + w + CO_WARPS * u of frame f; zero past the selection or on an idle lane
__device__ __forceinline__ void co_tile_read(const CoordArgs &A, const LaneFit &T, long long i0, long long f, bool valid,
                                             int w, float (&c)[CO_PER_WARP][3]) {
    float x[CO_PER_WARP][3];
#pragma unroll
    for (int u = 0; u < CO_PER_WARP; ++u) {
        const long long i = i0 + w + CO_WARPS * u;
        if (valid && i < A.k) {
            const float *p = A.coords + (long long)__ldg(A.sel + i) * 3 * A.fs + f;
#pragma unroll
            for (int d = 0; d < 3; ++d) x[u][d] = __ldg(p + d * A.fs);
        }
    }
#pragma unroll
    for (int u = 0; u < CO_PER_WARP; ++u) {
        const long long i = i0 + w + CO_WARPS * u;
        if (valid && i < A.k) {
            co_point(A, T, x[u][0], x[u][1], x[u][2], c[u]);
        } else {
            c[u][0] = c[u][1] = c[u][2] = 0.f;
        }
    }
}

// out[k * ld + d * n_sel + i] = aligned coordinate d of selected atom i in listed frame k
__global__ void __launch_bounds__(CO_THREADS) coords_kernel(const CoordArgs A, float *__restrict__ out, long long ld) {
    __shared__ float tile[3][CO_TILE][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item0 = 32ll * blockIdx.x, item = item0 + lane;
    const bool valid = item < A.n;
    const int rows = A.n - item0 < 32 ? (int)(A.n - item0) : 32;
    LaneFit T;
    const long long f = valid ? co_frame(A, item, T) : 0;
    const long long nblk = (A.k + CO_TILE - 1) / CO_TILE;
    for (long long b = blockIdx.y; b < nblk; b += gridDim.y) {
        const long long i0 = b * CO_TILE;
        float c[CO_PER_WARP][3];
        co_tile_read(A, T, i0, f, valid, w, c);
#pragma unroll
        for (int u = 0; u < CO_PER_WARP; ++u)
#pragma unroll
            for (int d = 0; d < 3; ++d) tile[d][w + CO_WARPS * u][lane] = c[u][d];
        __syncthreads();
        for (int r = w; r < 3 * rows; r += CO_WARPS) {
            const int kk = r / 3, d = r - 3 * kk;
            float *o = out + (item0 + kk) * ld + d * A.k + i0;
#pragma unroll
            for (int h = 0; h < CO_TILE / 32; ++h) {
                const int j = 32 * h + lane;
                if (i0 + j < A.k) o[j] = tile[d][j][kk];
            }
        }
        __syncthreads();
    }
}

// partial[(chunk * n_sel + i) * 3 + d] = sum over the chunk's listed frames, in list order, of aligned coordinate d
__global__ void __launch_bounds__(CO_THREADS) coord_sums_partial_kernel(const CoordArgs A, double *__restrict__ partial) {
    __shared__ float tile[3][CO_TILE][33];
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const int sd = t / CO_TILE, sj = t - CO_TILE * sd;  // the (axis, atom) this thread sums when t < 3 * CO_TILE
    const long long chunk0 = (long long)blockIdx.x * CO_CHUNK;
    const long long nblk = (A.k + CO_TILE - 1) / CO_TILE;
    for (long long b = blockIdx.y; b < nblk; b += gridDim.y) {
        const long long i0 = b * CO_TILE;
        double s = 0.0;
        for (int sub = 0; sub < CO_CHUNK / 32; ++sub) {
            const long long item0 = chunk0 + 32 * sub, item = item0 + lane;
            if (item0 >= A.n) break;
            const bool valid = item < A.n;
            const int rows = A.n - item0 < 32 ? (int)(A.n - item0) : 32;
            LaneFit T;
            const long long f = valid ? co_frame(A, item, T) : 0;
            float c[CO_PER_WARP][3];
            co_tile_read(A, T, i0, f, valid, w, c);
#pragma unroll
            for (int u = 0; u < CO_PER_WARP; ++u)
#pragma unroll
                for (int d = 0; d < 3; ++d) tile[d][w + CO_WARPS * u][lane] = c[u][d];
            __syncthreads();
            if (sd < 3)
                for (int kk = 0; kk < rows; ++kk) s += (double)tile[sd][sj][kk];
            __syncthreads();
        }
        if (sd < 3 && i0 + sj < A.k) partial[((long long)blockIdx.x * A.k + i0 + sj) * 3 + sd] = s;
    }
}

// sums[j] = the chunk partials of entry j added in chunk order (zero without frames)
__global__ void coord_sums_finish_kernel(const double *__restrict__ partial, long long nchunk, long long k3,
                                         double *__restrict__ sums) {
    const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (j >= k3) return;
    double s = 0.0;
    for (long long c = 0; c < nchunk; ++c) s += partial[c * k3 + j];
    sums[j] = s;
}

// sum_d (c_d - m_d)^2 in float64, unfused, in axis order: the same bits as numpy's ((e0*e0 + e1*e1) + e2*e2)
__device__ __forceinline__ double co_sqdev(const float (&c)[3], const double *__restrict__ m) {
    const double e0 = (double)c[0] - __ldg(m), e1 = (double)c[1] - __ldg(m + 1), e2 = (double)c[2] - __ldg(m + 2);
    return __dadd_rn(__dadd_rn(__dmul_rn(e0, e0), __dmul_rn(e1, e1)), __dmul_rn(e2, e2));
}

// out[k * ld + g] = fl32(squared deviation of selected atom g in listed frame k) or, GROUPED, fl32(the float64 mean of
// the squared deviations of selection positions [goff[g], goff[g+1]))
template <bool GROUPED>
__global__ void __launch_bounds__(CO_THREADS) fluct_kernel(const CoordArgs A, const double *__restrict__ centre,
                                                           const long long *__restrict__ goff, long long G,
                                                           float *__restrict__ out, long long ld) {
    __shared__ float tile[CO_TILE][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item0 = 32ll * blockIdx.x, item = item0 + lane;
    const bool valid = item < A.n;
    const int rows = A.n - item0 < 32 ? (int)(A.n - item0) : 32;
    LaneFit T;
    const long long f = valid ? co_frame(A, item, T) : 0;
    const long long nblk = (G + CO_TILE - 1) / CO_TILE;
    for (long long b = blockIdx.y; b < nblk; b += gridDim.y) {
        const long long g0 = b * CO_TILE;
        if (!GROUPED) {
            float c[CO_PER_WARP][3];
            co_tile_read(A, T, g0, f, valid, w, c);
#pragma unroll
            for (int u = 0; u < CO_PER_WARP; ++u) {
                const long long i = g0 + w + CO_WARPS * u;
                tile[w + CO_WARPS * u][lane] = valid && i < A.k ? __double2float_rn(co_sqdev(c[u], centre + 3 * i)) : 0.f;
            }
        } else {
            for (int u = 0; u < CO_PER_WARP; ++u) {
                const long long g = g0 + w + CO_WARPS * u;
                float v = 0.f;
                if (valid && g < G) {
                    const long long a0 = __ldg(goff + g), a1 = __ldg(goff + g + 1);
                    double s = 0.0;
                    for (long long a = a0; a < a1; a += CO_GROUP_BATCH) {
                        float x[CO_GROUP_BATCH][3];
#pragma unroll
                        for (int q = 0; q < CO_GROUP_BATCH; ++q) {
                            if (a + q < a1) {
                                const float *p = A.coords + (long long)__ldg(A.sel + a + q) * 3 * A.fs + f;
#pragma unroll
                                for (int d = 0; d < 3; ++d) x[q][d] = __ldg(p + d * A.fs);
                            }
                        }
#pragma unroll
                        for (int q = 0; q < CO_GROUP_BATCH; ++q) {
                            if (a + q < a1) {
                                float c[3];
                                co_point(A, T, x[q][0], x[q][1], x[q][2], c);
                                s += co_sqdev(c, centre + 3 * (a + q));
                            }
                        }
                    }
                    v = __double2float_rn(s / (double)(a1 - a0));
                }
                tile[w + CO_WARPS * u][lane] = v;
            }
        }
        __syncthreads();
        for (int kk = w; kk < rows; kk += CO_WARPS) {
            float *o = out + (item0 + kk) * ld + g0;
#pragma unroll
            for (int h = 0; h < CO_TILE / 32; ++h) {
                const int j = 32 * h + lane;
                if (g0 + j < G) o[j] = tile[j][kk];
            }
        }
        __syncthreads();
    }
}

constexpr int MO_SEG = 512;   // selection positions per segment, at most
constexpr int MO_BATCH = 4;   // positions per warp per round: 12 independent loads in flight per thread
constexpr int MO_ACC = 6;     // sum w e_d, then sum w e_d^2, per (segment, listed frame)

// the per-call table the host builds and uploads: segment s = positions [seg_pos[s], seg_pos[s+1]) of group seg_grp[s];
// group g = positions [goff[g], goff[g+1]), segments [gseg[g], gseg[g+1]), weight total wsum[g]; w[n_sel] or NULL
struct MomentArgs {
    const long long *seg_pos, *seg_grp, *goff, *gseg;
    const double *wsum, *w;
    long long nseg, G;
};

// aligned coordinates of selection position i in the lane's frame f (zeros on an idle lane)
__device__ __forceinline__ void mo_point(const CoordArgs &A, const LaneFit &T, long long i, long long f, bool valid,
                                         float (&c)[3]) {
    float x[3] = {0.f, 0.f, 0.f};
    if (valid) {
        const float *p = A.coords + (long long)__ldg(A.sel + i) * 3 * A.fs + f;
#pragma unroll
        for (int d = 0; d < 3; ++d) x[d] = __ldg(p + d * A.fs);
    }
    co_point(A, T, x[0], x[1], x[2], c);
}

// partial[(s * MO_ACC + j) * n + item] = over the positions i of segment s: sum w_i e_d (j = d) and sum w_i e_d^2
// (j = 3 + d), e = c_i - c_first in float64.  Warp w takes positions seg0 + w + 8 m, the warps are added in order.
__global__ void __launch_bounds__(CO_THREADS) moments_partial_kernel(const CoordArgs A, const MomentArgs M,
                                                                     double *__restrict__ partial) {
    __shared__ double red[CO_WARPS][MO_ACC][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item = 32ll * blockIdx.x + lane;
    const bool valid = item < A.n;
    LaneFit T;
    const long long f = valid ? co_frame(A, item, T) : 0;
    for (long long s = blockIdx.y; s < M.nseg; s += gridDim.y) {
        const long long a0 = __ldg(M.seg_pos + s), a1 = __ldg(M.seg_pos + s + 1);
        float sh[3];
        mo_point(A, T, __ldg(M.goff + __ldg(M.seg_grp + s)), f, valid, sh);
        double acc[MO_ACC];
#pragma unroll
        for (int j = 0; j < MO_ACC; ++j) acc[j] = 0.0;
        for (long long i0 = a0 + w; i0 < a1; i0 += CO_WARPS * MO_BATCH) {
            float x[MO_BATCH][3];
#pragma unroll
            for (int u = 0; u < MO_BATCH; ++u) {
                const long long i = i0 + CO_WARPS * u;
                x[u][0] = x[u][1] = x[u][2] = 0.f;
                if (valid && i < a1) {
                    const float *p = A.coords + (long long)__ldg(A.sel + i) * 3 * A.fs + f;
#pragma unroll
                    for (int d = 0; d < 3; ++d) x[u][d] = __ldg(p + d * A.fs);
                }
            }
#pragma unroll
            for (int u = 0; u < MO_BATCH; ++u) {
                const long long i = i0 + CO_WARPS * u;
                if (i >= a1) break;
                float c[3];
                co_point(A, T, x[u][0], x[u][1], x[u][2], c);
                const double wt = M.w ? __ldg(M.w + i) : 1.0;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    const double e = (double)c[d] - (double)sh[d], we = wt * e;
                    acc[d] += we;
                    acc[3 + d] = fma(we, e, acc[3 + d]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < MO_ACC; ++j) red[w][j][lane] = acc[j];
        __syncthreads();
        if (w < MO_ACC && valid) {
            double t = red[0][w][lane];
#pragma unroll
            for (int ww = 1; ww < CO_WARPS; ++ww) t += red[ww][w][lane];
            partial[(s * MO_ACC + w) * A.n + item] = t;
        }
        __syncthreads();
    }
}

// one thread per (listed frame, group): the group's segments added in order, then
// out[(k G + g) 6 + d] = mu_d = c_first,d + S1_d / W and out[... + 3 + d] = v_d = S2_d / W - (S1_d / W)^2 (>= 0);
// all six NaN when a sum is not finite
__global__ void moments_finish_kernel(const CoordArgs A, const MomentArgs M, const double *__restrict__ partial,
                                      double *__restrict__ out) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= A.n * M.G) return;
    const long long g = t / A.n, item = t - g * A.n;
    LaneFit T;
    const long long f = co_frame(A, item, T);
    float sh[3];
    mo_point(A, T, M.goff[g], f, true, sh);
    double acc[MO_ACC];
#pragma unroll
    for (int j = 0; j < MO_ACC; ++j) acc[j] = 0.0;
    for (long long s = M.gseg[g]; s < M.gseg[g + 1]; ++s)
#pragma unroll
        for (int j = 0; j < MO_ACC; ++j) acc[j] += partial[(s * MO_ACC + j) * A.n + item];
    bool finite = true;
#pragma unroll
    for (int j = 0; j < MO_ACC; ++j) finite = finite && isfinite(acc[j]);
    const double W = M.wsum[g];
    double *o = out + (item * M.G + g) * MO_ACC;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double m = acc[d] / W, v = acc[3 + d] / W - m * m;
        o[d] = finite ? (double)sh[d] + m : CUDART_NAN;
        o[3 + d] = finite ? (v < 0.0 ? 0.0 : v) : CUDART_NAN;
    }
}

// shared argument checks of the K15 entry points (those of align_args without a reference)
static int coord_args(mkb_ctx *h, const mkb_traj *t, const uint32_t *sel, int64_t n_sel, const uint32_t *frames,
                      int64_t n_frames, const double *records, CoordArgs &A) {
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_sel <= 0) return fail(h, MKB_ERR_BAD_ARG, "n_sel must be >= 1");
    if (n_sel >= (1ll << 31) || t->n_atoms >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "n_sel / n_atoms must be < 2^31");
    if (t->n_frames < 0 || (frames && n_frames < 0)) return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !sel) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < t->n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    A.coords = t->coords; A.fs = t->frame_stride;
    A.sel = sel; A.k = n_sel;
    A.frames = frames; A.n = frames ? n_frames : t->n_frames;
    A.rec = records;
    if (cdiv(A.n, 32) >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one launch");
    return MKB_OK;
}

static unsigned co_blocks_y(long long items) { return (unsigned)std::min<long long>(cdiv(items, CO_TILE), 65535); }

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_coordinates(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                               const uint32_t *frames, int64_t n_frames, const double *records, float *out,
                               int64_t ld_out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    CoordArgs A;
    int rc = coord_args(h, t, sel, n_sel, frames, n_frames, records, A);
    if (rc) return rc;
    if (ld_out < 3 * n_sel) return fail(h, MKB_ERR_BAD_ARG, "ld_out %lld < 3 * n_sel", (long long)ld_out);
    if (A.n == 0) return MKB_OK;
    if (!out) return fail(h, MKB_ERR_BAD_ARG, "null out");
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    coords_kernel<<<dim3((unsigned)cdiv(A.n, 32), co_blocks_y(A.k)), CO_THREADS, 0, st>>>(A, out, ld_out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "coords_kernel";
    return MKB_OK;
}

extern "C" int mkb_coord_sums(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                              const uint32_t *frames, int64_t n_frames, const double *records, double *sums) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    CoordArgs A;
    int rc = coord_args(h, t, sel, n_sel, frames, n_frames, records, A);
    if (rc) return rc;
    if (!sums) return fail(h, MKB_ERR_BAD_ARG, "null sums");
    const long long nchunk = cdiv(A.n, CO_CHUNK), k3 = 3 * A.k;
    double *partial = nullptr;
    if (nchunk > 0 && (rc = scratch_get(h, S_COORD_PART, (size_t)(nchunk * k3), &partial))) return rc;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    if (nchunk > 0) {
        coord_sums_partial_kernel<<<dim3((unsigned)nchunk, co_blocks_y(A.k)), CO_THREADS, 0, st>>>(A, partial);
        MKB_LAUNCHED(h);
    }
    coord_sums_finish_kernel<<<(unsigned)cdiv(k3, 256), 256, 0, st>>>(partial, nchunk, k3, sums);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "coord_sums_partial_kernel";
    return MKB_OK;
}

extern "C" int mkb_fluctuation(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                               const uint32_t *frames, int64_t n_frames, const double *records, const double *centre,
                               const int64_t *group_offsets, int64_t n_groups, float *out, int64_t ld_out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    CoordArgs A;
    int rc = coord_args(h, t, sel, n_sel, frames, n_frames, records, A);
    if (rc) return rc;
    if (group_offsets && (n_groups < 1 || n_groups > n_sel))
        return fail(h, MKB_ERR_BAD_ARG, "n_groups must be in [1, n_sel]");
    const long long G = group_offsets ? n_groups : n_sel;
    if (ld_out < G) return fail(h, MKB_ERR_BAD_ARG, "ld_out %lld < %lld output columns", (long long)ld_out, G);
    if (A.n == 0) return MKB_OK;
    if (!out || !centre) return fail(h, MKB_ERR_BAD_ARG, "null out / centre");
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(A.n, 32), co_blocks_y(G));
    const long long *goff = reinterpret_cast<const long long *>(group_offsets);
    if (group_offsets) fluct_kernel<true><<<grid, CO_THREADS, 0, st>>>(A, centre, goff, G, out, ld_out);
    else fluct_kernel<false><<<grid, CO_THREADS, 0, st>>>(A, centre, nullptr, G, out, ld_out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = group_offsets ? "fluct_kernel<grouped>" : "fluct_kernel";
    return MKB_OK;
}

extern "C" int mkb_frame_moments(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t n_sel,
                                 const uint32_t *frames, int64_t n_frames, const double *records,
                                 const double *weights, const int64_t *group_offsets, int64_t n_groups, double *out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    CoordArgs A;
    int rc = coord_args(h, t, sel, n_sel, frames, n_frames, records, A);
    if (rc) return rc;
    if (!group_offsets) return fail(h, MKB_ERR_BAD_ARG, "null group_offsets");
    if (n_groups < 1 || n_groups > n_sel) return fail(h, MKB_ERR_BAD_ARG, "n_groups must be in [1, n_sel]");
    const long long G = n_groups;
    if (group_offsets[0] != 0 || group_offsets[G] != n_sel)
        return fail(h, MKB_ERR_BAD_ARG, "group_offsets must run from 0 to n_sel = %lld", (long long)n_sel);
    for (long long g = 0; g < G; ++g) {
        if (group_offsets[g + 1] < group_offsets[g]) return fail(h, MKB_ERR_BAD_ARG, "group_offsets decrease at group %lld", g);
        if (group_offsets[g + 1] == group_offsets[g]) return fail(h, MKB_ERR_BAD_ARG, "group %lld is empty", g);
    }
    if (A.n > (1ll << 37) / G) return fail(h, MKB_ERR_BAD_ARG, "too many (frame, group) outputs for one launch");
    // the table: segment boundaries, segment groups, group offsets, first segments, weight totals (8-byte words)
    std::vector<long long> seg_pos, seg_grp, gseg((size_t)G + 1);
    std::vector<double> wsum((size_t)G);
    for (long long g = 0; g < G; ++g) {
        const long long a0 = group_offsets[g], a1 = group_offsets[g + 1];
        double W = 0.0;
        for (long long i = a0; i < a1; ++i) W += weights ? weights[i] : 1.0;
        if (!(W > 0.0) || !std::isfinite(W))
            return fail(h, MKB_ERR_BAD_ARG, "the weights of group %lld sum to %g: must be finite and > 0", g, W);
        wsum[(size_t)g] = W;
        // segments depend only on the group's size: as few as hold at most MO_SEG positions, of equal length
        const long long ns = cdiv(a1 - a0, MO_SEG), len = cdiv(a1 - a0, ns);
        gseg[(size_t)g] = (long long)seg_grp.size();
        for (long long j = 0; j < ns; ++j) {
            seg_pos.push_back(a0 + j * len);
            seg_grp.push_back(g);
        }
    }
    const long long nseg = (long long)seg_grp.size();
    gseg[(size_t)G] = nseg;
    seg_pos.push_back(n_sel);
    if (A.n == 0) return MKB_OK;
    if (!out) return fail(h, MKB_ERR_BAD_ARG, "null out");
    const size_t words = (size_t)(2 * nseg + 1) + 2 * ((size_t)G + 1) + (size_t)G + (weights ? (size_t)n_sel : 0);
    long long *tab = nullptr;
    double *partial = nullptr;
    if ((rc = scratch_get(h, S_MOMENT_TAB, words, &tab))) return rc;
    if ((rc = scratch_get(h, S_MOMENT_PART, (size_t)(nseg * MO_ACC * A.n), &partial))) return rc;
    {   // one upload from page-locked staging
        void *stage = nullptr;
        cudaEvent_t *sev = nullptr;
        if ((rc = host_stage_get(h, words * 8, &stage, &sev))) return rc;
        char *p = static_cast<char *>(stage);
        const auto put = [&p](const void *src, size_t n_words) {
            memcpy(p, src, n_words * 8);
            p += n_words * 8;
        };
        put(seg_pos.data(), seg_pos.size());
        put(seg_grp.data(), seg_grp.size());
        put(group_offsets, (size_t)G + 1);
        put(gseg.data(), gseg.size());
        put(wsum.data(), wsum.size());
        if (weights) put(weights, (size_t)n_sel);
        MKB_CUDA(h, cudaMemcpyAsync(tab, stage, words * 8, cudaMemcpyHostToDevice, st));
        MKB_CUDA(h, cudaEventRecord(*sev, st));
    }
    MomentArgs M;
    M.seg_pos = tab;
    M.seg_grp = M.seg_pos + nseg + 1;
    M.goff = M.seg_grp + nseg;
    M.gseg = M.goff + G + 1;
    M.wsum = reinterpret_cast<const double *>(M.gseg + G + 1);
    M.w = weights ? M.wsum + G : nullptr;
    M.nseg = nseg;
    M.G = G;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(A.n, 32), (unsigned)std::min<long long>(nseg, 65535));
    moments_partial_kernel<<<grid, CO_THREADS, 0, st>>>(A, M, partial);
    MKB_LAUNCHED(h);
    moments_finish_kernel<<<(unsigned)cdiv(A.n * G, 128), 128, 0, st>>>(A, M, partial, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "moments_partial_kernel";
    return MKB_OK;
}
