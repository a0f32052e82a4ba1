// tmscore.cu -- K19: the TM-score superposition search over a trajectory for sm_90a (H100).
//
// Replaces moleculekit's molTMscore (the TMscore program's search of Zhang & Skolnick, one frame at a time on the CPU).
// The contract (include/mkb200.h) fixes every float64 operation and its order; each one is rounded on its own
// (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so the scores are bit-identical to a C restatement
// compiled without contraction (tests/tmscore_oracle.c).
//
// The grid is the resident CTAs; each strides over work units of (listed frame, round of TM_THREADS seeds), frame-major,
// so a frame with few seeds per SM (large L, few frames) still fills the GPU.  A unit's pairs live in shared memory as
// float32 structure-of-arrays, the reference's once per CTA.  Each thread runs one seed, the chain of up to 21 fits that
// starts from one fragment, in the sequential order of the contract.  During
// the extension fits every lane of a warp reads the same pair at the same step (a shared-memory broadcast).  A thread's
// cut sets are two bitmasks in global scratch, [word][thread] so a warp's words are one coalesced line: the score pass
// writes the new set word by word while comparing it with the fitted one, so convergence costs no extra pass.  The
// "widen dcut by 0.5 while fewer than 3 pairs" loop is decided on the third smallest distance of the pass, which is
// exactly the literal recount, and re-cuts only when it moved dcut.  A unit's maximum is a warp then CTA max; the units
// of a frame combine with a 64-bit atomicMax on the score's bits (scores are > 0, so the bits order as the values).
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "tm_fit.cuh"

namespace mkb {

constexpr int TM_THREADS = 128;
constexpr int TM_WARPS = TM_THREADS / 32;
constexpr int TM_MAX_PAIRS = 8192;     // 24 B of shared memory per pair: 192 KB
constexpr int TM_MAX_FRAG = 6;
constexpr int TM_EXT = 20;             // extension fits per seed
constexpr int TM_WIDEN_MAX = 1 << 20;  // widening steps of one cut at most

struct TmArgs {
    const float *coords;
    long long fs;
    const float *ref;
    long long rfs;
    const unsigned *sel, *refsel;
    int L, W;                            // pairs, 32-bit words per cut-set mask
    double lnorm, d0, d0s;
    int nfrag;
    int frag[TM_MAX_FRAG];
    int seed0[TM_MAX_FRAG + 1];          // first seed of every fragment length; seed0[nfrag] = seeds per frame
    const unsigned *frames;
    long long n;
    unsigned *mask;                      // [cta][2][W][TM_THREADS]
    double *tm, *rmsd;
};

struct TmFit {
    double R[9], p[3], q[3];
};

struct TmShared {
    const float *x, *y, *z, *rx, *ry, *rz;  // model and reference pairs, structure of arrays
};

// Kabsch fit over the pairs of [k0, k1) that are in the set: all of them (mask == nullptr) or the set bits of the mask
// (words strided by TM_THREADS); c = the set's size.  Centroids first, then H about them.
__device__ __forceinline__ void tm_fit(const TmShared &S, int k0, int k1, const unsigned *mask, int c, TmFit &F) {
    double sx[3] = {0.0, 0.0, 0.0}, sy[3] = {0.0, 0.0, 0.0};
    unsigned word = 0;
    for (int k = k0; k < k1; ++k) {
        if (mask && (k & 31) == 0) word = mask[(k >> 5) * TM_THREADS];
        const double a0 = S.x[k], a1 = S.y[k], a2 = S.z[k], b0 = S.rx[k], b1 = S.ry[k], b2 = S.rz[k];
        if (!mask || (word >> (k & 31)) & 1u) {
            sx[0] = DADD(sx[0], a0); sx[1] = DADD(sx[1], a1); sx[2] = DADD(sx[2], a2);
            sy[0] = DADD(sy[0], b0); sy[1] = DADD(sy[1], b1); sy[2] = DADD(sy[2], b2);
        }
    }
    const double cd = (double)c;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        F.p[d] = DDIV(sx[d], cd);
        F.q[d] = DDIV(sy[d], cd);
    }
    double H[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) H[j] = 0.0;
    for (int k = k0; k < k1; ++k) {
        if (mask && (k & 31) == 0) word = mask[(k >> 5) * TM_THREADS];
        const double a[3] = {DSUB((double)S.x[k], F.p[0]), DSUB((double)S.y[k], F.p[1]), DSUB((double)S.z[k], F.p[2])};
        const double b[3] = {DSUB((double)S.rx[k], F.q[0]), DSUB((double)S.ry[k], F.q[1]),
                             DSUB((double)S.rz[k], F.q[2])};
        if (!mask || (word >> (k & 31)) & 1u) {
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int s = 0; s < 3; ++s) H[3 * r + s] = DADD(H[3 * r + s], DMUL(a[r], b[s]));
        }
    }
    tm_horn_rotation(H, F.R);
}

struct TmPass {
    double score;   // sum over all pairs of 1 / (1 + (dis / d0)^2)
    double sq;      // sum of squared distances
    double third;   // third smallest distance (+inf when L < 3)
    int count;      // pairs with dis < dcut
    bool same;      // the new set equals the compared one
};

// One pass over all L pairs under F: the score, the cut set at dcut written to `out` (and compared with `cmp` when
// given), the third smallest distance.
__device__ __forceinline__ TmPass tm_pass(const TmShared &S, int L, double d0, const TmFit &F, double dcut,
                                          unsigned *out, const unsigned *cmp) {
    TmPass P;
    P.score = 0.0; P.sq = 0.0; P.count = 0; P.same = true;
    double m1 = INFINITY, m2 = INFINITY, m3 = INFINITY;
    unsigned word = 0;
    for (int k = 0; k < L; ++k) {
        const double a0 = DSUB((double)S.x[k], F.p[0]), a1 = DSUB((double)S.y[k], F.p[1]),
                     a2 = DSUB((double)S.z[k], F.p[2]);
        const double y[3] = {S.rx[k], S.ry[k], S.rz[k]};
        double e[3];
#pragma unroll
        for (int d = 0; d < 3; ++d)
            e[d] = DSUB(DADD(DADD(DADD(DMUL(F.R[3 * d], a0), DMUL(F.R[3 * d + 1], a1)), DMUL(F.R[3 * d + 2], a2)),
                             F.q[d]), y[d]);
        const double d2 = DADD(DADD(DMUL(e[0], e[0]), DMUL(e[1], e[1])), DMUL(e[2], e[2]));
        const double dis = __dsqrt_rn(d2);
        const double t = DDIV(dis, d0);
        P.score = DADD(P.score, DDIV(1.0, DADD(1.0, DMUL(t, t))));
        P.sq = DADD(P.sq, d2);
        if (dis < m3) {
            if (dis < m2) {
                m3 = m2;
                if (dis < m1) { m2 = m1; m1 = dis; } else m2 = dis;
            } else {
                m3 = dis;
            }
        }
        const bool in = dis < dcut;
        P.count += in;
        word |= (unsigned)in << (k & 31);
        if ((k & 31) == 31 || k == L - 1) {
            const int w = (k >> 5) * TM_THREADS;
            if (cmp) P.same = P.same && cmp[w] == word;
            out[w] = word;
            word = 0;
        }
    }
    P.third = m3;
    return P;
}

// The chain of fits of seed s; returns its best score.  Writes the frame's RMSD when s is the all-pairs seed 0.
__device__ double tm_seed(const TmArgs &A, const TmShared &S, int s, unsigned *m0, unsigned *m1, double *rmsd_out) {
    int fi = 0;
    while (s >= A.seed0[fi + 1]) ++fi;
    const int Li = A.frag[fi], iL = s - A.seed0[fi], L = A.L;
    TmFit F;
    tm_fit(S, iL, iL + Li, nullptr, Li, F);
    double dcut = DSUB(A.d0s, 1.0);
    TmPass P = tm_pass(S, L, A.d0, F, dcut, m0, nullptr);
    if (s == 0) *rmsd_out = __dsqrt_rn(DDIV(P.sq, (double)L));
    double best = DDIV(P.score, A.lnorm);
    // fewer than 3 pairs below dc is exactly !(third < dc): widen, then cut again into `out`
    auto widen = [&](double dc, unsigned *out, const unsigned *cmp) {
        if (L > 3 && !(P.third < dc)) {
            for (int step = 0; step < TM_WIDEN_MAX && !(P.third < dc); ++step) dc = DADD(dc, 0.5);
            P = tm_pass(S, L, A.d0, F, dc, out, cmp);
        }
    };
    widen(dcut, m0, nullptr);
    unsigned *fitted = m0, *next = m1;
    int nfit = P.count;
    dcut = DADD(A.d0s, 1.0);
    for (int it = 0; it < TM_EXT && nfit > 0; ++it) {
        tm_fit(S, 0, L, fitted, nfit, F);
        P = tm_pass(S, L, A.d0, F, dcut, next, fitted);
        widen(dcut, next, fitted);
        best = fmax(best, DDIV(P.score, A.lnorm));
        if (P.same) break;
        unsigned *tmp = fitted;
        fitted = next;
        next = tmp;
        nfit = P.count;
    }
    return best;
}

// 3 CTAs per SM: without the hint ptxas stops at 128 registers and spills; with it, 138 and no spills
__global__ void __launch_bounds__(TM_THREADS, 3) tmscore_kernel(const TmArgs A) {
    extern __shared__ float sm[];
    __shared__ double wmax[TM_WARPS];
    const int L = A.L, tid = threadIdx.x;
    TmShared S;
    S.x = sm; S.y = sm + L; S.z = sm + 2 * L; S.rx = sm + 3 * L; S.ry = sm + 4 * L; S.rz = sm + 5 * L;
    float *rx = sm + 3 * L;
    bool ref_bad = false;
    for (int k = tid; k < L; k += TM_THREADS) {
        const float *q = A.ref + (long long)A.refsel[k] * 3 * A.rfs;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            rx[d * L + k] = q[d * A.rfs];
            ref_bad = ref_bad || !isfinite(q[d * A.rfs]);
        }
    }
    ref_bad = __syncthreads_or(ref_bad);
    unsigned *m0 = A.mask + (size_t)blockIdx.x * 2 * A.W * TM_THREADS + tid, *m1 = m0 + (size_t)A.W * TM_THREADS;
    const int nseeds = A.seed0[A.nfrag], rounds = (nseeds + TM_THREADS - 1) / TM_THREADS;
    float *mx = sm;
    unsigned long long *tm_bits = reinterpret_cast<unsigned long long *>(A.tm);
    // work unit = (listed frame, round of TM_THREADS seeds), frame-major
    for (long long u = blockIdx.x; u < A.n * rounds; u += gridDim.x) {
        const long long item = u / rounds;
        const int round = (int)(u - item * rounds);
        const long long f = A.frames ? (long long)A.frames[item] : item;
        __syncthreads();  // the previous unit's pairs and warp maxima are no longer read
        bool bad = ref_bad;
        for (int k = tid; k < L; k += TM_THREADS) {
            const float *p = A.coords + (long long)A.sel[k] * 3 * A.fs + f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                mx[d * L + k] = p[d * A.fs];
                bad = bad || !isfinite(p[d * A.fs]);
            }
        }
        if (__syncthreads_or(bad)) {
            if (tid == 0 && round == 0) A.tm[item] = A.rmsd[item] = NAN;
            continue;
        }
        const int s = round * TM_THREADS + tid;
        double best = s < nseeds ? tm_seed(A, S, s, m0, m1, A.rmsd + item) : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, o));
        if ((tid & 31) == 0) wmax[tid >> 5] = best;
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < TM_WARPS; ++w) best = fmax(best, wmax[w]);
            // scores are > 0, so their bit patterns order as the values; the caller zeroed tm
            atomicMax(tm_bits + item, (unsigned long long)__double_as_longlong(best));
        }
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int64_t mkb_tmscore_max_pairs(void) { return TM_MAX_PAIRS; }

extern "C" int mkb_tmscore(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, const mkb_traj *ref,
                           const uint32_t *refsel, int64_t n_pairs, int64_t l_norm, double d0, double d0_search,
                           const int32_t *frag, int32_t n_frag, const uint32_t *frames, int64_t n_frames, double *tm,
                           double *rmsd) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t || !ref) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_pairs < 1 || n_pairs > TM_MAX_PAIRS)
        return fail(h, MKB_ERR_BAD_ARG, "n_pairs %lld outside [1, %d]", (long long)n_pairs, TM_MAX_PAIRS);
    if (l_norm < 1) return fail(h, MKB_ERR_BAD_ARG, "l_norm must be >= 1");
    if (!(d0 > 0.0) || !std::isfinite(d0) || !std::isfinite(d0_search))
        return fail(h, MKB_ERR_BAD_ARG, "d0 must be finite and > 0, d0_search finite");
    if (!frag || n_frag < 1 || n_frag > TM_MAX_FRAG)
        return fail(h, MKB_ERR_BAD_ARG, "n_frag %d outside [1, %d]", (int)n_frag, TM_MAX_FRAG);
    if (t->n_frames < 0 || ref->n_frames < 1 || (frames && n_frames < 0))
        return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !ref->coords || !sel || !refsel) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < t->n_frames || ref->frame_stride < ref->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    TmArgs A;
    A.coords = t->coords; A.fs = t->frame_stride;
    A.ref = ref->coords; A.rfs = ref->frame_stride;
    A.sel = sel; A.refsel = refsel;
    A.L = (int)n_pairs;
    A.W = (int)cdiv(n_pairs, 32);
    A.lnorm = (double)l_norm; A.d0 = d0; A.d0s = d0_search;
    A.nfrag = n_frag;
    A.seed0[0] = 0;
    for (int i = 0; i < n_frag; ++i) {
        if (frag[i] < 1 || frag[i] > n_pairs)
            return fail(h, MKB_ERR_BAD_ARG, "fragment length %d outside [1, n_pairs]", (int)frag[i]);
        A.frag[i] = frag[i];
        A.seed0[i + 1] = A.seed0[i] + (int)(n_pairs - frag[i] + 1);
    }
    A.frames = frames;
    A.n = frames ? n_frames : t->n_frames;
    if (A.n == 0) return MKB_OK;
    if (!tm || !rmsd) return fail(h, MKB_ERR_BAD_ARG, "null tm / rmsd");
    A.tm = tm; A.rmsd = rmsd;

    const size_t smem = (size_t)6 * n_pairs * sizeof(float);
    MKB_CUDA(h, cudaFuncSetAttribute(tmscore_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    MKB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, tmscore_kernel, TM_THREADS, smem));
    if (per_sm < 1) return fail(h, MKB_ERR_CUDA, "tmscore_kernel cannot be resident with %zu B of shared memory", smem);
    const long long units = A.n * cdiv(A.seed0[n_frag], TM_THREADS);
    const long long grid = std::min<long long>(units, (long long)per_sm * h->sm_count);
    int rc;
    if ((rc = scratch_get(h, S_TMSCORE_MASK, (size_t)grid * 2 * A.W * TM_THREADS, &A.mask))) return rc;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    MKB_CUDA(h, cudaMemsetAsync(tm, 0, (size_t)A.n * sizeof(double), st));
    tmscore_kernel<<<(unsigned)grid, TM_THREADS, smem, st>>>(A);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "tmscore_kernel";
    return MKB_OK;
}
