// align.cu -- K14: trajectory superposition (Kabsch fit, in-place apply, RMSD) for sm_90a (H100).
//
// Replaces the frame loop of Molecule.align (moleculekit/align.py, _pp_align / _pp_measure_fit): per frame a float32 3x3
// SVD of the covariance of the selected atoms and a float32 matrix product over all atoms.  Here every frame is fitted in
// float64 and the coordinates are rounded to float32 once.
//
//   fit      align_partial_kernel<FIT_*> + align_solve_kernel.  A CTA owns 32 listed frames (lane = frame, so each load of
//            an (atom, axis) row is one 128-byte line when the frames are consecutive) and one segment of the selection;
//            its 8 warps split the segment's atoms and combine in shared memory, the solve kernel adds the segments in
//            order.  The segment count depends only on the selection size, so a frame's summation order depends only on
//            the selection: a frame slice gives the same bits as the whole call.  One reference frame: the reference is
//            centred once (align_ref_center_kernel) and H = sum (p - p_s) q'^T - S_p (sum q')^T / k, the second term
//            removing what the rounding of the float64 centroid leaves in sum q' (far from the origin it would otherwise
//            tilt H by k (p_bar - p_s) times that error); matching frames: sums relative to the first selected atom of
//            each frame and H = S_pq - S_p S_q^T / k.  The solve kernel (one thread per frame) takes the
//            eigenvector of the largest eigenvalue of Horn's symmetric 4x4 matrix by cyclic Jacobi in float64: det R = +1
//            by construction, ties go to the lowest index (H = 0 gives the identity, as numpy's SVD of a zero matrix).
//   apply    align_apply_kernel: x' = fl32(R (x - p) + q) in float64, one thread per (frame, atom stride), the frame's
//            record loaded once; a pure HBM stream of 12 B in and 12 B out per atom-frame.
//   rmsd     align_partial_kernel<RMSD> + align_rmsd_kernel: same layout as the fit, sum of |T(x) - q|^2 in float64.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace mkb {

constexpr int AL_THREADS = 256;
constexpr int AL_WARPS = AL_THREADS / 32;
constexpr int AL_SEG_ATOMS = 512;  // atoms per selection segment (one CTA row of the partial grid)
constexpr int AL_MAX_SEG = 16;
constexpr int AL_BATCH = 4;        // atoms per warp per round: independent loads in flight
constexpr int AL_REC = 16;         // doubles per frame record: R[9] row-major, p[3], q[3], pad

enum AlignMode { FIT_SINGLE = 0, FIT_MATCH = 1, RMSD = 2 };

template <int MODE>
struct AlignAcc {
    static constexpr int N = MODE == FIT_SINGLE ? 12 : (MODE == FIT_MATCH ? 15 : 1);
};

struct AlignArgs {
    const float *coords;
    long long fs;
    const float *ref;
    long long rfs;
    int ref_match;  // reference frame = the frame itself (else reference frame 0)
    const unsigned *sel, *refsel;
    long long k;
    const unsigned *frames;
    long long n;      // listed frames
    const double *qc; // FIT_SINGLE: centred reference [k][3], q_bar [3], sum q' [3]
    const double *rec;  // RMSD: per-frame fit records, NULL = no transform
    int nseg;
    long long seg_len;
};

__device__ __forceinline__ long long al_frame(const AlignArgs &A, long long item) {
    return A.frames ? (long long)A.frames[item] : item;
}

__device__ __forceinline__ double ldf(const float *p) { return (double)__ldg(p); }

// Partial sums of one (32-frame chunk, selection segment).  FIT_*: acc = [S_p(3) | S_pq(9) | S_q(3, matching only)]
// relative to the first selected atom of the frame (p) and of the reference frame (q, matching) or to the centred
// reference (q', single).  RMSD: acc = sum |T(x) - q|^2.  partial[(seg * NACC + j) * n + item].
template <int MODE>
__global__ void __launch_bounds__(AL_THREADS) align_partial_kernel(const AlignArgs A, double *__restrict__ partial) {
    constexpr int NACC = AlignAcc<MODE>::N;
    __shared__ double red[AL_WARPS][NACC][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item0 = 32ll * blockIdx.x, item = item0 + lane;
    const bool valid = item < A.n;
    const long long f = al_frame(A, valid ? item : item0);  // an idle lane shadows lane 0 (results discarded)
    const long long rf = A.ref_match ? f : 0;
    const long long seg0 = (long long)blockIdx.y * A.seg_len;
    const long long seg1 = seg0 + A.seg_len < A.k ? seg0 + A.seg_len : A.k;
    double acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0.0;
    double ps[3] = {0.0, 0.0, 0.0}, qs[3] = {0.0, 0.0, 0.0};
    double R[9], pb[3], qb[3];
    if (MODE != RMSD) {
        const float *p0 = A.coords + (long long)A.sel[0] * 3 * A.fs + f;
#pragma unroll
        for (int d = 0; d < 3; ++d) ps[d] = ldf(p0 + d * A.fs);
        if (MODE == FIT_MATCH) {
            const float *q0 = A.ref + (long long)A.refsel[0] * 3 * A.rfs + rf;
#pragma unroll
            for (int d = 0; d < 3; ++d) qs[d] = ldf(q0 + d * A.rfs);
        }
    } else if (A.rec) {
        const double *r = A.rec + (valid ? item : item0) * AL_REC;
#pragma unroll
        for (int j = 0; j < 9; ++j) R[j] = r[j];
#pragma unroll
        for (int d = 0; d < 3; ++d) { pb[d] = r[9 + d]; qb[d] = r[12 + d]; }
    }
    for (long long i0 = seg0 + w; i0 < seg1; i0 += AL_WARPS * AL_BATCH) {
        double p[AL_BATCH][3], q[AL_BATCH][3];
#pragma unroll
        for (int u = 0; u < AL_BATCH; ++u) {
            const long long i = i0 + AL_WARPS * u;
            if (i < seg1) {
                const float *pp = A.coords + (long long)__ldg(A.sel + i) * 3 * A.fs + f;
#pragma unroll
                for (int d = 0; d < 3; ++d) p[u][d] = ldf(pp + d * A.fs);
                if (MODE == FIT_SINGLE) {
#pragma unroll
                    for (int d = 0; d < 3; ++d) q[u][d] = __ldg(A.qc + i * 3 + d);
                } else {
                    const float *qq = A.ref + (long long)__ldg(A.refsel + i) * 3 * A.rfs + rf;
#pragma unroll
                    for (int d = 0; d < 3; ++d) q[u][d] = ldf(qq + d * A.rfs);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < AL_BATCH; ++u) {
            if (i0 + AL_WARPS * u >= seg1) break;
            if (MODE == RMSD) {
                double y[3];
                if (A.rec) {
                    const double x0 = p[u][0] - pb[0], x1 = p[u][1] - pb[1], x2 = p[u][2] - pb[2];
#pragma unroll
                    for (int d = 0; d < 3; ++d) y[d] = fma(R[3 * d + 2], x2, fma(R[3 * d + 1], x1, R[3 * d] * x0)) + qb[d];
                } else {
#pragma unroll
                    for (int d = 0; d < 3; ++d) y[d] = p[u][d];
                }
                const double e0 = y[0] - q[u][0], e1 = y[1] - q[u][1], e2 = y[2] - q[u][2];
                acc[0] += fma(e2, e2, fma(e1, e1, e0 * e0));
            } else {
                double a[3], b[3];
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    a[d] = p[u][d] - ps[d];
                    b[d] = q[u][d] - qs[d];
                    acc[d] += a[d];
                }
#pragma unroll
                for (int r = 0; r < 3; ++r)
#pragma unroll
                    for (int c = 0; c < 3; ++c) acc[3 + 3 * r + c] = fma(a[r], b[c], acc[3 + 3 * r + c]);
                if (MODE == FIT_MATCH) {
#pragma unroll
                    for (int d = 0; d < 3; ++d) acc[12 + d] += b[d];
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < NACC; ++j) red[w][j][lane] = acc[j];
    __syncthreads();
    if (w == 0 && valid) {
#pragma unroll
        for (int j = 0; j < NACC; ++j) {
            double s = red[0][j][lane];
#pragma unroll
            for (int ww = 1; ww < AL_WARPS; ++ww) s += red[ww][j][lane];
            partial[((long long)blockIdx.y * NACC + j) * A.n + item] = s;
        }
    }
}

// centroid of the reference selection (fixed-order tree over one CTA) and the centred reference q' = q - q_bar;
// qc[3k .. 3k+2] = q_bar, qc[3k+3 .. 3k+5] = sum q' (the same tree): not zero, as q_bar is rounded
__global__ void __launch_bounds__(AL_THREADS) align_ref_center_kernel(const float *__restrict__ ref, long long rfs,
                                                                      const unsigned *__restrict__ refsel, long long k,
                                                                      double *__restrict__ qc) {
    __shared__ double s[3][AL_THREADS];
    const int t = threadIdx.x;
    double a[3] = {0.0, 0.0, 0.0};
    for (long long i = t; i < k; i += AL_THREADS) {
        const float *q = ref + (long long)refsel[i] * 3 * rfs;
#pragma unroll
        for (int d = 0; d < 3; ++d) a[d] += (double)q[d * rfs];
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) s[d][t] = a[d];
    __syncthreads();
    for (int h = AL_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) {
#pragma unroll
            for (int d = 0; d < 3; ++d) s[d][t] += s[d][t + h];
        }
        __syncthreads();
    }
    const double qb[3] = {s[0][0] / (double)k, s[1][0] / (double)k, s[2][0] / (double)k};
    __syncthreads();  // every thread has read s[.][0]
    double r[3] = {0.0, 0.0, 0.0};
    for (long long i = t; i < k; i += AL_THREADS) {
        const float *q = ref + (long long)refsel[i] * 3 * rfs;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const double c = (double)q[d * rfs] - qb[d];
            qc[i * 3 + d] = c;
            r[d] += c;
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) s[d][t] = r[d];
    __syncthreads();
    for (int h = AL_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) {
#pragma unroll
            for (int d = 0; d < 3; ++d) s[d][t] += s[d][t + h];
        }
        __syncthreads();
    }
    if (t < 3) {
        qc[3 * k + t] = qb[t];
        qc[3 * k + 3 + t] = s[t][0];
    }
}

// one Jacobi rotation of the symmetric 4x4 `a` zeroing a[P][Q]; eigenvectors accumulate in the columns of v
template <int P, int Q>
__device__ __forceinline__ void jacobi_rot(double (&a)[4][4], double (&v)[4][4], bool late) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq);
    if (late && fabs(a[P][P]) + g == fabs(a[P][P]) && fabs(a[Q][Q]) + g == fabs(a[Q][Q])) {
        a[P][Q] = a[Q][P] = 0.0;  // below the precision of both diagonal entries
        return;
    }
    const double h = a[Q][Q] - a[P][P];
    double t;
    if (fabs(h) + g == fabs(h)) {
        t = apq / h;
    } else {
        const double th = 0.5 * h / apq;
        t = 1.0 / (fabs(th) + sqrt(1.0 + th * th));
        if (th < 0.0) t = -t;
    }
    const double c = 1.0 / sqrt(1.0 + t * t), s = t * c, tau = s / (1.0 + c);
    a[P][P] -= t * apq;
    a[Q][Q] += t * apq;
    a[P][Q] = a[Q][P] = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        if (r == P || r == Q) continue;
        const double arp = a[r][P], arq = a[r][Q];
        a[r][P] = a[P][r] = arp - s * (arq + arp * tau);
        a[r][Q] = a[Q][r] = arq + s * (arp - arq * tau);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const double vrp = v[r][P], vrq = v[r][Q];
        v[r][P] = vrp - s * (vrq + vrp * tau);
        v[r][Q] = vrq + s * (vrp - vrq * tau);
    }
}

// optimal proper rotation R (row-major, q ~ R p) for the covariance H[a][b] = sum p_a q_b (Horn's quaternion form)
__device__ __forceinline__ void horn_rotation(const double (&H)[9], double (&R)[9]) {
    const double Sxx = H[0], Sxy = H[1], Sxz = H[2], Syx = H[3], Syy = H[4], Syz = H[5], Szx = H[6], Szy = H[7],
                 Szz = H[8];
    double a[4][4] = {{Sxx + Syy + Szz, Syz - Szy, Szx - Sxz, Sxy - Syx},
                      {Syz - Szy, Sxx - Syy - Szz, Sxy + Syx, Szx + Sxz},
                      {Szx - Sxz, Sxy + Syx, -Sxx + Syy - Szz, Syz + Szy},
                      {Sxy - Syx, Szx + Sxz, Syz + Szy, -Sxx - Syy + Szz}};
    double v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[0][3]) + fabs(a[1][2]) + fabs(a[1][3]) + fabs(a[2][3]);
        if (off == 0.0) break;
        const bool late = sweep > 3;
        jacobi_rot<0, 1>(a, v, late);
        jacobi_rot<0, 2>(a, v, late);
        jacobi_rot<0, 3>(a, v, late);
        jacobi_rot<1, 2>(a, v, late);
        jacobi_rot<1, 3>(a, v, late);
        jacobi_rot<2, 3>(a, v, late);
    }
    double q[4] = {v[0][0], v[1][0], v[2][0], v[3][0]}, best = a[0][0];
#pragma unroll
    for (int j = 1; j < 4; ++j)
        if (a[j][j] > best) {  // strict: ties go to the lowest index
            best = a[j][j];
#pragma unroll
            for (int r = 0; r < 4; ++r) q[r] = v[r][j];
        }
    const double inv = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const double q0 = q[0] * inv, q1 = q[1] * inv, q2 = q[2] * inv, q3 = q[3] * inv;
    R[0] = q0 * q0 + q1 * q1 - q2 * q2 - q3 * q3;
    R[1] = 2.0 * (q1 * q2 - q0 * q3);
    R[2] = 2.0 * (q1 * q3 + q0 * q2);
    R[3] = 2.0 * (q1 * q2 + q0 * q3);
    R[4] = q0 * q0 - q1 * q1 + q2 * q2 - q3 * q3;
    R[5] = 2.0 * (q2 * q3 - q0 * q1);
    R[6] = 2.0 * (q1 * q3 - q0 * q2);
    R[7] = 2.0 * (q2 * q3 + q0 * q1);
    R[8] = q0 * q0 - q1 * q1 - q2 * q2 + q3 * q3;
}

// one thread per listed frame: add the segments in order, build H and the centroids, solve, write the record and status
template <int MODE>
__global__ void align_solve_kernel(const AlignArgs A, const double *__restrict__ partial, double *__restrict__ rec,
                                   int *__restrict__ status) {
    constexpr int NACC = AlignAcc<MODE>::N;
    const long long item = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (item >= A.n) return;
    double acc[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) acc[j] = 0.0;
    for (int s = 0; s < A.nseg; ++s)
#pragma unroll
        for (int j = 0; j < NACC; ++j) acc[j] += partial[((long long)s * NACC + j) * A.n + item];
    const long long f = al_frame(A, item);
    const double k = (double)A.k;
    double pb[3], qb[3], H[9];
    const float *p0 = A.coords + (long long)A.sel[0] * 3 * A.fs + f;
#pragma unroll
    for (int d = 0; d < 3; ++d) pb[d] = (double)p0[d * A.fs] + acc[d] / k;
    if (MODE == FIT_MATCH) {
        const float *q0 = A.ref + (long long)A.refsel[0] * 3 * A.rfs + f;
#pragma unroll
        for (int d = 0; d < 3; ++d) qb[d] = (double)q0[d * A.rfs] + acc[12 + d] / k;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) H[3 * r + c] = acc[3 + 3 * r + c] - acc[r] * acc[12 + c] / k;
    } else {
#pragma unroll
        for (int d = 0; d < 3; ++d) qb[d] = A.qc[3 * A.k + d];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) H[3 * r + c] = acc[3 + 3 * r + c] - acc[r] * A.qc[3 * A.k + 3 + c] / k;
    }
    bool finite = true;
#pragma unroll
    for (int j = 0; j < 9; ++j) finite = finite && isfinite(H[j]);
#pragma unroll
    for (int d = 0; d < 3; ++d) finite = finite && isfinite(pb[d]) && isfinite(qb[d]);
    double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    if (finite) horn_rotation(H, R);
    double *o = rec + item * AL_REC;
#pragma unroll
    for (int j = 0; j < 9; ++j) o[j] = R[j];
#pragma unroll
    for (int d = 0; d < 3; ++d) { o[9 + d] = pb[d]; o[12 + d] = qb[d]; }
    o[15] = 0.0;
    status[item] = finite ? 0 : 1;
}

__global__ void align_rmsd_kernel(const double *__restrict__ partial, long long n, int nseg, long long k,
                                  float *__restrict__ out) {
    const long long item = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (item >= n) return;
    double s = 0.0;
    for (int j = 0; j < nseg; ++j) s += partial[(long long)j * n + item];
    out[item] = (float)sqrt(s / (double)k);
}

// x' = fl32(R (x - p) + q) for every atom of the listed frames whose status is 0.  Lane = frame, warp = atom stride.
__global__ void __launch_bounds__(AL_THREADS) align_apply_kernel(float *__restrict__ coords, long long fs, long long N,
                                                                 const unsigned *__restrict__ frames, long long n,
                                                                 const double *__restrict__ rec,
                                                                 const int *__restrict__ status) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long item = 32ll * blockIdx.x + lane;
    if (item >= n || (status && status[item] != 0)) return;
    const long long f = frames ? (long long)frames[item] : item;
    double R[9], pb[3], qb[3];
    fit_record_load(rec + item * AL_REC, R, pb, qb);
    float *base = coords + f;
    const long long step = (long long)gridDim.y * AL_WARPS;
    for (long long a0 = (long long)blockIdx.y * AL_WARPS + w; a0 < N; a0 += step * AL_BATCH) {
        float x[AL_BATCH][3];
#pragma unroll
        for (int u = 0; u < AL_BATCH; ++u) {
            const long long a = a0 + step * u;
            if (a < N) {
#pragma unroll
                for (int d = 0; d < 3; ++d) x[u][d] = base[(a * 3 + d) * fs];
            }
        }
#pragma unroll
        for (int u = 0; u < AL_BATCH; ++u) {
            const long long a = a0 + step * u;
            if (a < N) {
                float y[3];
                fit_transform(R, pb, qb, x[u][0], x[u][1], x[u][2], y);
#pragma unroll
                for (int d = 0; d < 3; ++d) base[(a * 3 + d) * fs] = y[d];
            }
        }
    }
}

// shared argument checks of the fit and RMSD entry points; fills A (except qc / rec)
static int align_args(mkb_ctx *h, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref, const uint32_t *refsel,
                      int64_t n_sel, const uint32_t *frames, int64_t n_frames, AlignArgs &A) {
    if (!t || !ref) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_sel <= 0) return fail(h, MKB_ERR_BAD_ARG, "n_sel must be >= 1");
    if (n_sel >= (1ll << 31) || t->n_atoms >= (1ll << 31) || ref->n_atoms >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "n_sel / n_atoms must be < 2^31");
    if (t->n_frames < 0 || ref->n_frames < 1 || (frames && n_frames < 0))
        return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (ref->n_frames != 1 && ref->n_frames != t->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "the reference has %lld frames: 1 or the trajectory's %lld",
                    (long long)ref->n_frames, (long long)t->n_frames);
    if (!t->coords || !ref->coords || !sel || !refsel) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < t->n_frames || ref->frame_stride < ref->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    A.coords = t->coords; A.fs = t->frame_stride;
    A.ref = ref->coords; A.rfs = ref->frame_stride;
    A.ref_match = ref->n_frames != 1;
    A.sel = sel; A.refsel = refsel; A.k = n_sel;
    A.frames = frames; A.n = frames ? n_frames : t->n_frames;
    A.qc = nullptr; A.rec = nullptr;
    A.nseg = (int)std::min<long long>(cdiv(n_sel, AL_SEG_ATOMS), AL_MAX_SEG);
    A.seg_len = cdiv(n_sel, A.nseg);
    if (cdiv(A.n, 32) >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one launch");
    return MKB_OK;
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_align_fit(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
                             const uint32_t *refsel, int64_t n_sel, const uint32_t *frames, int64_t n_frames,
                             double *records, int32_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    AlignArgs A;
    int rc = align_args(h, t, sel, ref, refsel, n_sel, frames, n_frames, A);
    if (rc) return rc;
    if (A.n == 0) return MKB_OK;
    if (!records || !status) return fail(h, MKB_ERR_BAD_ARG, "null records / status");
    const int nacc = A.ref_match ? AlignAcc<FIT_MATCH>::N : AlignAcc<FIT_SINGLE>::N;
    double *partial = nullptr, *qc = nullptr;
    if ((rc = scratch_get(h, S_ALIGN_PART, (size_t)(A.nseg * nacc * A.n), &partial))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    if (!A.ref_match) {
        if ((rc = scratch_get(h, S_ALIGN_REF, (size_t)(3 * n_sel + 6), &qc))) return rc;
        align_ref_center_kernel<<<1, AL_THREADS, 0, st>>>(ref->coords, ref->frame_stride, refsel, n_sel, qc);
        MKB_LAUNCHED(h);
        A.qc = qc;
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(A.n, 32), (unsigned)A.nseg);
    const unsigned sblocks = (unsigned)cdiv(A.n, 128);
    if (A.ref_match) {
        align_partial_kernel<FIT_MATCH><<<grid, AL_THREADS, 0, st>>>(A, partial);
        MKB_LAUNCHED(h);
        align_solve_kernel<FIT_MATCH><<<sblocks, 128, 0, st>>>(A, partial, records, status);
    } else {
        align_partial_kernel<FIT_SINGLE><<<grid, AL_THREADS, 0, st>>>(A, partial);
        MKB_LAUNCHED(h);
        align_solve_kernel<FIT_SINGLE><<<sblocks, 128, 0, st>>>(A, partial, records, status);
    }
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "align_partial_kernel";
    return MKB_OK;
}

extern "C" int mkb_align_apply(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *frames,
                               int64_t n_frames, const double *records, const int32_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (t->n_atoms < 0 || t->n_frames < 0 || (frames && n_frames < 0)) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    const long long n = frames ? n_frames : t->n_frames, N = t->n_atoms;
    if (n == 0 || N == 0) return MKB_OK;
    if (!t->coords || !records) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < t->n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const long long gx = cdiv(n, 32);
    if (gx >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one launch");
    // about 8 resident CTAs per SM in total; every CTA walks its atom stride with the frame record in registers
    const long long gy = std::max<long long>(1, std::min<long long>({cdiv(8ll * h->sm_count, gx), cdiv(N, AL_WARPS), 65535}));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    align_apply_kernel<<<dim3((unsigned)gx, (unsigned)gy), AL_THREADS, 0, st>>>(const_cast<float *>(t->coords),
                                                                               t->frame_stride, N, frames, n, records,
                                                                               status);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "align_apply_kernel";
    return MKB_OK;
}

extern "C" int mkb_rmsd(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
                        const uint32_t *refsel, int64_t n_sel, const uint32_t *frames, int64_t n_frames,
                        const double *records, float *out) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    AlignArgs A;
    int rc = align_args(h, t, sel, ref, refsel, n_sel, frames, n_frames, A);
    if (rc) return rc;
    if (A.n == 0) return MKB_OK;
    if (!out) return fail(h, MKB_ERR_BAD_ARG, "null out");
    A.rec = records;
    double *partial = nullptr;
    if ((rc = scratch_get(h, S_ALIGN_PART, (size_t)(A.nseg * A.n), &partial))) return rc;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    align_partial_kernel<RMSD><<<dim3((unsigned)cdiv(A.n, 32), (unsigned)A.nseg), AL_THREADS, 0, st>>>(A, partial);
    MKB_LAUNCHED(h);
    align_rmsd_kernel<<<(unsigned)cdiv(A.n, 128), 128, 0, st>>>(partial, A.n, A.nseg, A.k, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "align_partial_kernel";
    return MKB_OK;
}
