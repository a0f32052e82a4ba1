// wrapping.cu -- K9 (SURVEY 8f row 4): orthorhombic periodic wrapping of bonded groups for sm_90a (H100).
//
// Replaces wrap_box (moleculekit/wrapping/wrapping.pyx:91-144), the loop Molecule.wrap runs for rectangular cells
// (moleculekit/molecule.py:2077).  Per frame the reference (1) takes the box centre as the running mean of the
// `centersel` atoms (pyx:113-118) or a fixed `center` (pyx:106-108), (2) for every bonded group [groups[g],
// groups[g+1]) takes the running mean of its atoms (pyx:127-134) and (3) per axis, when that centre is further than
// half a box from the box centre, subtracts box*round(diff/box) from every atom of the group (pyx:137-142).
//
// Frames, groups and axes are independent (groups are disjoint atom ranges and the box centre is read before any
// group of its frame is moved), so the parallel form is exact.  The running mean itself, c += (x - c)/(n + 1) with one
// float rounding per operation, is a sequential chain by definition and is kept verbatim (bit-identical output).
// The trajectory is frame-minor, so 32 consecutive frames of one (atom, axis) row are one 128-byte line: lanes = frames.
//
//   small groups (<= WRAP_SMALL = 4 atoms: waters, ions)  one thread per (group, frame): the 3*count values are loaded
//       once into registers, the three short chains run on them, moved axes are stored back from the registers.
//       Traffic: one read, one write of what moved -- the HBM-bound bulk of a solvated system.
//   long groups (a solute, lipids) and the centre selection  one CTA per (group, 32 frames): warps 3..7 stream the
//       rows through a 3-stage cp.async ring in shared memory while warps 0..2 (one axis each) walk the chain out of
//       shared memory with the reciprocal of n + 1 precomputed off the chain (exact_div.cuh); the chain (~6 dependent
//       float ops per atom), not DRAM latency, sets the pace.  The translation then goes to all 8 warps, which apply
//       it to the group's rows with 12 independent loads in flight per thread.
//   A classify pre-pass appends the long groups to a device list; the first CTAs of the groups launch are persistent
//   workers over that list, the rest are the small-group threads, so both kinds overlap on the machine.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "exact_div.cuh"

namespace mkb {

constexpr int WRAP_SMALL = 4;     // largest group handled from registers (waters, ions, 4-site water models)
constexpr int WRAP_STAGE = 32;    // atoms per pipeline stage of the long-chain path
constexpr int WRAP_NSTAGE = 3;    // cp.async ring depth
constexpr int WRAP_THREADS = 256;
constexpr int WRAP_WARPS = WRAP_THREADS / 32;
constexpr int WRAP_ROWS = WRAP_STAGE * 3;

struct alignas(16) ChainSmem {
    float v[WRAP_NSTAGE][WRAP_ROWS][32];  // [stage][atom*3 + axis][frame lane]
    float rb[WRAP_NSTAGE][WRAP_STAGE];    // (float)(n + 1)
    float rr[WRAP_NSTAGE][WRAP_STAGE];    // refined reciprocal of it
    float tr[3][32];                      // translation per (axis, frame lane)
    int mv[3][32];                        // the group moves along this axis in this frame
};

__device__ __forceinline__ void cp_async4(float *smem_dst, const float *gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// 16-byte copy of which only the first src_bytes are read (the rest of the destination is zero-filled)
__device__ __forceinline__ void cp_async16(float *smem_dst, const float *gsrc, int src_bytes) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Running mean over `count` atoms for 32 frames [f0, f0 + nf) and the three axes, by the whole CTA.  Atom n of the chain
// is index[n] (INDIRECT: centersel, pyx:113-118) or first_atom + n (a group, pyx:127-134).  Warps 3..7 are the loaders
// (cp.async rows of 32 frames into the ring, plus the (n + 1, reciprocal) tables), warps 0..2 walk the chain of axis =
// warp and return its mean for frame lane (other warps return 0).
// SHIFT (triclinic / compact wrapping, pyx:221-223): the chain runs on (x - sh_sub) + sh_add, the centred coordinate the
// reference has already stored when it averages a group.
template <bool INDIRECT, bool SHIFT = false>
__device__ __forceinline__ float chain_32frames(ChainSmem &sm, const float *coords, long long fs, long long f0, int nf,
                                                const unsigned *__restrict__ index, long long first_atom,
                                                long long count, float sh_sub = 0.f, float sh_add = 0.f) {
    constexpr int LOADERS = WRAP_WARPS - 3;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    const long long nst = (count + WRAP_STAGE - 1) / WRAP_STAGE;
    const float *lane_base = coords + f0 + lane;
    // rows start on 16-byte boundaries: 16-byte cp.async (4-byte copies are issued per element and ~4x slower)
    const bool aligned16 = ((reinterpret_cast<unsigned long long>(coords) | (unsigned long long)(fs * 4)) & 15ull) == 0;
    auto issue = [&](long long s) {
        if (w >= 3 && s < nst) {
            const int buf = (int)(s % WRAP_NSTAGE), lw = w - 3;
            const long long n0 = s * WRAP_STAGE;
            const long long left = count - n0;
            const int rows = left < WRAP_STAGE ? 3 * (int)left : WRAP_ROWS;  // row = atom_in_stage*3 + axis
            if (aligned16) {
                // 16-byte pieces: 8 per row; loader thread lt takes pieces lt, lt + 160, ...
                const int lt = t - 96;
                const float *p = coords + f0 + (INDIRECT ? 0 : (first_atom + n0) * 3 * fs);
#pragma unroll 5
                for (int piece = lt; piece < rows * 8; piece += LOADERS * 32) {
                    const int row = piece >> 3, q = piece & 7;
                    const int vf = nf - 4 * q;  // valid frames in this piece
                    if (vf > 0) {
                        long long off;
                        if (INDIRECT) {
                            const int a = row / 3, i = row - 3 * a;
                            off = ((long long)__ldg(index + n0 + a) * 3 + i) * fs;
                        } else {
                            off = row * fs;
                        }
                        cp_async16(&sm.v[buf][row][4 * q], p + off + 4 * q, vf >= 4 ? 16 : 4 * vf);
                    }
                }
            } else if (lane < nf) {
                if (INDIRECT) {
#pragma unroll 4
                    for (int row = lw; row < rows; row += LOADERS) {
                        const int a = row / 3, i = row - 3 * a;
                        cp_async4(&sm.v[buf][row][lane], lane_base + ((long long)__ldg(index + n0 + a) * 3 + i) * fs);
                    }
                } else {
                    const float *p = lane_base + (first_atom + n0) * 3 * fs;  // row r of the stage is p + r*fs
#pragma unroll 4
                    for (int row = lw; row < rows; row += LOADERS) cp_async4(&sm.v[buf][row][lane], p + row * fs);
                }
            }
            if (lw == 0) {
                const float b = __int2float_rn((int)(n0 + lane) + 1);  // the reference's (n + 1): C int -> float
                sm.rb[buf][lane] = b;
                sm.rr[buf][lane] = refined_rcp(b);
            }
        }
        cp_async_commit();  // one group per stage, empty past the end: keeps the wait distance uniform
    };
#pragma unroll
    for (int s = 0; s < WRAP_NSTAGE - 1; ++s) issue(s);
    float c = 0.f;
    for (long long s = 0; s < nst; ++s) {
        cp_async_wait<WRAP_NSTAGE - 2>();  // this thread's copies of stage s have landed (only stage s + 1 may be pending)
        __syncthreads();                   // ... and everyone's; the chain warps are also done with stage s - 1,
        issue(s + WRAP_NSTAGE - 1);        // whose buffer the loaders refill while the chain walks stage s
        if (w < 3) {
            const int buf = (int)(s % WRAP_NSTAGE);
            const long long left = count - s * WRAP_STAGE;
            const int m = left < WRAP_STAGE ? (int)left : WRAP_STAGE;
            // 8 atoms at a time: operands first (independent shared loads), then the dependent chain on the branch-free
            // fast division.  The range test runs beside the chain (OR of independent terms); when any step of any lane
            // left the fast domain (zero / denormal / huge difference) the batch is redone with __fdiv_rn.
            auto batch = [&](int a0, int nb) {  // nb = 8 (full, branch-free) or the tail length
                float x[8], b[8], r[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {  // a0 + u < WRAP_STAGE always: stale rows are read but never used
                    x[u] = sm.v[buf][(a0 + u) * 3 + w][lane];
                    if (SHIFT) x[u] = __fadd_rn(__fsub_rn(x[u], sh_sub), sh_add);
                    b[u] = sm.rb[buf][a0 + u];
                    r[u] = sm.rr[buf][a0 + u];
                }
                const float c_in = c;
                unsigned bad = 0;
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (u < nb) {
                        const float d = __fsub_rn(x[u], c);
                        bad |= div_fast_ok(d) ? 0u : 1u;
                        c = __fadd_rn(c, div_fast(d, b[u], r[u]));
                    }
                if (bad) {
                    c = c_in;
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        if (u < nb) c = __fadd_rn(c, __fdiv_rn(__fsub_rn(x[u], c), b[u]));
                }
            };
            int a0 = 0;
            for (; a0 + 8 <= m; a0 += 8) batch(a0, 8);
            if (a0 < m) batch(a0, m - a0);
        }
    }
    __syncthreads();  // the last stage is consumed before the caller reuses the ring
    cp_async_wait<0>();
    return c;
}

// box centre per (axis, frame): pyx:113-118.  One CTA per 32 frames.
__global__ void __launch_bounds__(WRAP_THREADS)
wrap_center_kernel(const float *__restrict__ coords, long long F, long long fs, const unsigned *__restrict__ centersel,
                   long long n_centersel, float *__restrict__ centre) {
    __shared__ ChainSmem sm;
    const long long f0 = 32ll * blockIdx.x;
    const int nf = (int)(F - f0 < 32 ? F - f0 : 32);
    const float c = chain_32frames<true>(sm, coords, fs, f0, nf, centersel, 0, n_centersel);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (w < 3 && lane < nf) centre[(long long)w * F + f0 + lane] = c;
}

__global__ void wrap_classify_kernel(const unsigned *__restrict__ groups, long long n_ranges,
                                     unsigned *__restrict__ long_list, unsigned *__restrict__ n_long) {
    const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (g >= n_ranges) return;
    if ((long long)groups[g + 1] - (long long)groups[g] > WRAP_SMALL) long_list[atomicAdd(n_long, 1u)] = (unsigned)g;
}

struct WrapArgs {
    float *coords;
    const float *box;
    long long F, fs, fsb;
    const unsigned *groups;
    long long n_ranges;
    const float *centre;  // [3][F], unused when fixed
    float cx, cy, cz;
    int fixed_centre;
    const unsigned *long_list;
    const unsigned *n_long;
    int n_long_ctas;
};

// pyx:137-139: does the group move along this axis, and by how much
__device__ __forceinline__ bool wrap_decide(const WrapArgs &A, float c, int i, long long f, float *tr) {
    const float bc = A.fixed_centre ? (i == 0 ? A.cx : (i == 1 ? A.cy : A.cz)) : A.centre[(long long)i * A.F + f];
    const float b = A.box[(long long)i * A.fsb + f];
    const float diff = __fsub_rn(c, bc);
    const bool move = fabsf(diff) > __fdiv_rn(b, 2.f);
    *tr = move ? __fmul_rn(b, roundf(__fdiv_rn(diff, b))) : 0.f;
    return move;
}

__device__ __forceinline__ void wrap_small_groups(const WrapArgs &A, long long tid);

// The first n_long_ctas CTAs are persistent workers over (long group, 32-frame chunk) items; the others are the
// small-group threads.  One launch, so the latency-bound long chains run beside the bandwidth-bound small groups.
__global__ void __launch_bounds__(WRAP_THREADS, 4) wrap_groups_kernel(const WrapArgs A) {
    __shared__ ChainSmem sm;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    if ((int)blockIdx.x >= A.n_long_ctas) {
        wrap_small_groups(A, ((long long)blockIdx.x - A.n_long_ctas) * WRAP_THREADS + t);
        return;
    }
    {
        const long long nchunks = (A.F + 31) / 32;
        const long long total = (long long)(*A.n_long) * nchunks;
        for (long long item = blockIdx.x; item < total; item += A.n_long_ctas) {
            const long long slot = item / nchunks, f0 = 32 * (item - slot * nchunks);
            const int nf = (int)(A.F - f0 < 32 ? A.F - f0 : 32);
            const long long g = A.long_list[slot];
            const long long s = A.groups[g], count = (long long)A.groups[g + 1] - s;
            const float c = chain_32frames<false>(sm, A.coords, A.fs, f0, nf, nullptr, s, count);
            if (w < 3) {
                float tr = 0.f;
                const bool move = lane < nf && wrap_decide(A, c, w, f0 + lane, &tr);
                sm.tr[w][lane] = tr;
                sm.mv[w][lane] = move ? 1 : 0;
            }
            __syncthreads();
            const bool m0 = sm.mv[0][lane] != 0, m1 = sm.mv[1][lane] != 0, m2 = sm.mv[2][lane] != 0;
            const float t0 = sm.tr[0][lane], t1 = sm.tr[1][lane], t2 = sm.tr[2][lane];
            if (__syncthreads_or(m0 || m1 || m2)) {
                float *base = A.coords + s * 3 * A.fs + f0 + lane;
                constexpr int BATCH = 4;  // atoms per thread per round: 12 independent loads, then their stores
                for (long long k0 = w; k0 < count; k0 += WRAP_WARPS * BATCH) {
                    float v[BATCH][3];
#pragma unroll
                    for (int u = 0; u < BATCH; ++u) {
                        const long long k = k0 + WRAP_WARPS * u;
                        float *p = base + k * 3 * A.fs;
                        if (k < count) {
                            if (m0) v[u][0] = p[0];
                            if (m1) v[u][1] = p[A.fs];
                            if (m2) v[u][2] = p[2 * A.fs];
                        }
                    }
#pragma unroll
                    for (int u = 0; u < BATCH; ++u) {
                        const long long k = k0 + WRAP_WARPS * u;
                        float *p = base + k * 3 * A.fs;
                        if (k < count) {
                            if (m0) p[0] = __fsub_rn(v[u][0], t0);
                            if (m1) p[A.fs] = __fsub_rn(v[u][1], t1);
                            if (m2) p[2 * A.fs] = __fsub_rn(v[u][2], t2);
                        }
                    }
                }
            }
            __syncthreads();  // sm.tr / sm.mv and the ring are reused by the next item
        }
    }
}

// small groups: one thread per (group, frame), frame fastest
__device__ __forceinline__ void wrap_small_groups(const WrapArgs &A, long long tid) {
    if (tid >= A.n_ranges * A.F) return;
    const long long g = tid / A.F, f = tid - g * A.F;
    const long long s = A.groups[g];
    const int count = (int)max(min((long long)A.groups[g + 1] - s, (long long)(WRAP_SMALL + 1)), -1ll);
    if (count <= 0 || count > WRAP_SMALL) return;  // empty range: nothing to move (pyx:127,141 loop over nothing)
    float *base = A.coords + s * 3 * A.fs + f;
    float v[WRAP_SMALL][3];
#pragma unroll
    for (int k = 0; k < WRAP_SMALL; ++k)
        if (k < count) {
#pragma unroll
            for (int i = 0; i < 3; ++i) v[k][i] = base[(long long)(k * 3 + i) * A.fs];
        }
    float c[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < WRAP_SMALL; ++k)
        if (k < count) {
#pragma unroll
            for (int i = 0; i < 3; ++i) c[i] = __fadd_rn(c[i], __fdiv_rn(__fsub_rn(v[k][i], c[i]), (float)(k + 1)));
        }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float tr;
        if (wrap_decide(A, c[i], i, f, &tr)) {
#pragma unroll
            for (int k = 0; k < WRAP_SMALL; ++k)
                if (k < count) base[(long long)(k * 3 + i) * A.fs] = __fsub_rn(v[k][i], tr);
        }
    }
}


// ---------------------------------------------------------------------------------------------------------------------
// K9b: triclinic cells -- wrap_triclinic_unitcell (pyx:147-250) and wrap_compact_unitcell (pyx:255-344, with get_pbc
// pyx:357-451 and pbc_dx pyx:454-505), the loops Molecule.wrap runs when a box angle differs from 90 (molecule.py:2078-2090).
// Differences from wrap_box that shape the kernels: (1) EVERY coordinate is first centred, x' = (x - wrap_center) +
// box_middle (float), and the group means run on x'; (2) the per-frame cell data (box vectors, shift matrix or correction
// vectors) and the translation are float64 while centres stay float32 -- each assignment keeps the type the generated C
// has; (3) the translation couples the axes (z first, then y, then x).  Per-frame data is computed once by
// tric_frame_kernel into a frame-minor table (lanes = frames read consecutive doubles); the group kernels are the K9
// decompositions (thread per (small group, frame); CTA pipeline per (long group, 32 frames)) with a different decision
// step and an apply step that rewrites all three axes.  The reference's `while` loops do not terminate for a cell whose
// diagonal is <= 0; they are bounded by TRIC_MAX_ITER here (no reference result exists for such input).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TRIC_NINFO = 50;              // doubles per frame in the table
constexpr long long TRIC_MAX_ITER = 1ll << 20;
// table rows: 0..8 box[i][j]; triclinic: 9 shm01, 10 shm02, 11 shm12, 12/13 shift_center[0/1];
//             compact: 9..11 hbox_diag, 12 max_cutoff2, 14 + 3k + j = tric_vec[k][j]
enum { TRIC_RECT = 0, TRIC_COMPACT = 1, TRIC_TRICLINIC = 2 };

struct TricArgs {
    float *coords;
    long long F, fs, n_atoms;
    const unsigned *groups;
    long long n_ranges;
    const double *info;   // [TRIC_NINFO][F]
    const float *bm;      // [3][F] box_middle
    const float *wc;      // [3][F] wrap centre per frame
    const int *ntric;     // [F]
    int mode;
    const unsigned *long_list;
    const unsigned *n_long;
    int n_long_ctas;
};

__device__ __forceinline__ double tric_norm2(const double *v) {
    return __dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2]));
}

// one thread per frame: box_middle, the wrap centre when it is fixed, and the cell data of the mode
__global__ void tric_frame_kernel(const double *__restrict__ bv, long long bvs, long long F, int mode, int fixed_centre,
                                  float cx, float cy, float cz, double *__restrict__ info, float *__restrict__ bm,
                                  float *__restrict__ wc, int *__restrict__ ntric_out, int *__restrict__ err) {
    const long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (f >= F) return;
    double box[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            box[i][j] = bv[(long long)(i * 3 + j) * bvs + f];
            info[(long long)(i * 3 + j) * F + f] = box[i][j];
        }
    float m[3] = {0.f, 0.f, 0.f};  // pyx:187-191: float accumulator, double addend
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) m[j] = __double2float_rn(__dadd_rn((double)m[j], __dmul_rn(0.5, box[i][j])));
#pragma unroll
    for (int j = 0; j < 3; ++j) bm[(long long)j * F + f] = m[j];
    if (fixed_centre) {
        wc[f] = cx; wc[F + f] = cy; wc[2 * F + f] = cz;
    }
    if (mode == TRIC_TRICLINIC) {
        const double shm01 = __ddiv_rn(box[1][0], box[1][1]);  // pyx:198-200
        const double shm02 = __ddiv_rn(__dsub_rn(__dmul_rn(box[1][1], box[2][0]), __dmul_rn(box[2][1], box[1][0])),
                                       __dmul_rn(box[1][1], box[2][2]));
        const double shm12 = __ddiv_rn(box[2][1], box[2][2]);
        double sc[3] = {0.0, 0.0, 0.0};  // pyx:203-213
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) sc[j] = __dadd_rn(sc[j], box[i][j]);
#pragma unroll
        for (int j = 0; j < 3; ++j) sc[j] = __dsub_rn((double)m[j], __dmul_rn(sc[j], 0.5));
        const double s0 = __dadd_rn(__dmul_rn(shm01, sc[1]), __dmul_rn(shm02, sc[2]));  // pyx:216-218
        const double s1 = __dmul_rn(shm12, sc[2]);
        info[9ll * F + f] = shm01; info[10ll * F + f] = shm02; info[11ll * F + f] = shm12;
        info[12ll * F + f] = s0; info[13ll * F + f] = s1;
        ntric_out[f] = 0;
        return;
    }
    // get_pbc, pyx:357-451
    double hbox[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        hbox[i] = __dmul_rn(box[i][i], 0.5);
        info[(long long)(9 + i) * F + f] = hbox[i];
    }
    double min_hv2;
    {
        const double a = tric_norm2(box[0]), b = tric_norm2(box[1]);
        min_hv2 = __dmul_rn(0.25, a < b ? a : b);
        const double c = __dmul_rn(0.25, tric_norm2(box[2]));
        min_hv2 = min_hv2 < c ? min_hv2 : c;
    }
    const double t1 = __dsub_rn(box[1][1], fabs(box[2][1]));
    const double t2 = t1 < box[2][2] ? t1 : box[2][2];
    const double min_ss = box[0][0] < t2 ? box[0][0] : t2;
    const double ss2 = __dmul_rn(min_ss, min_ss);
    info[12ll * F + f] = min_hv2 < ss2 ? min_hv2 : ss2;
    const double skew = 1.001;
    int ntric = 0;
    bool too_many = false;
    for (int kk = 0; kk < 3 && !too_many; ++kk) {
        const int k = kk == 0 ? 0 : (kk == 1 ? -1 : 1);
        for (int jj = 0; jj < 3 && !too_many; ++jj) {
            const int j = jj == 0 ? 0 : (jj == 1 ? -1 : 1);
            for (int ii = 0; ii < 3 && !too_many; ++ii) {
                const int i = ii == 0 ? 0 : (ii == 1 ? -1 : 1);
                if (!(j != 0 || k != 0)) continue;
                double trial[3], pos[3], d2old = 0.0, d2new = 0.0;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    trial[d] = __dadd_rn(__dadd_rn(__dmul_rn((double)i, box[0][d]), __dmul_rn((double)j, box[1][d])),
                                         __dmul_rn((double)k, box[2][d]));
                    const double nt = -trial[d];
                    if (trial[d] < 0) pos[d] = hbox[d] < nt ? hbox[d] : nt;       // cmin(hbox, -trial)
                    else pos[d] = -hbox[d] > nt ? -hbox[d] : nt;                  // cmax(-hbox, -trial)
                    d2old = __dadd_rn(d2old, __dmul_rn(pos[d], pos[d]));
                    const double pt = __dadd_rn(pos[d], trial[d]);
                    d2new = __dadd_rn(d2new, __dmul_rn(pt, pt));
                }
                if (__dmul_rn(skew, d2new) < d2old) {
                    bool use = true;
                    for (int dd = 0; dd < 3; ++dd) {
                        const int shift = dd == 0 ? i : (dd == 1 ? j : k);
                        if (shift) {
                            double d2c = 0.0;
#pragma unroll
                            for (int e = 0; e < 3; ++e) {
                                const double t = __dsub_rn(__dadd_rn(pos[e], trial[e]), __dmul_rn((double)shift, box[dd][e]));
                                d2c = __dadd_rn(d2c, __dmul_rn(t, t));
                            }
                            if (d2c <= __dmul_rn(skew, d2new)) { use = false; break; }
                        }
                    }
                    if (use) {
                        if (ntric >= 12) { too_many = true; break; }
#pragma unroll
                        for (int e = 0; e < 3; ++e) info[(long long)(14 + 3 * ntric + e) * F + f] = trial[e];
                        ++ntric;
                    }
                }
            }
        }
    }
    if (too_many) atomicExch(err, 1);  // the reference raises ValueError("Too many triclinic vectors!!") (pyx:439-441)
    ntric_out[f] = ntric;
}

// decision for one (group, frame): gc = the group's centre on entry.  Triclinic: g[] returns grp_center_init - grp_center
// (pyx:239-262).  Compact: g[] returns the centre itself and dx[] the pbc_dx vector (pyx:338-344).
__device__ __forceinline__ void tric_decide(const TricArgs &A, long long f, const float gc_in[3], const float bmid[3],
                                            float g[3], double dx[3]) {
    const double *I = A.info + f;
    const long long F = A.F;
    if (A.mode == TRIC_TRICLINIC) {
        float gc[3] = {gc_in[0], gc_in[1], gc_in[2]};
        const double shm01 = I[9 * F], shm02 = I[10 * F], shm12 = I[11 * F];
#pragma unroll
        for (int m = 2; m >= 0; --m) {
            double shift = m == 2 ? 0.0 : I[(12 + m) * F];
            if (m == 0) shift = __dadd_rn(shift, __dadd_rn(__dmul_rn(shm01, (double)gc[1]), __dmul_rn(shm02, (double)gc[2])));
            else if (m == 1) shift = __dadd_rn(shift, __dmul_rn(shm12, (double)gc[2]));
            double bmd[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) bmd[d] = d <= m ? I[(3 * m + d) * F] : 0.0;
            long long it = 0;
            while (__dsub_rn((double)gc[m], shift) < 0 && it++ < TRIC_MAX_ITER) {
#pragma unroll
                for (int d = 0; d < 3; ++d)
                    if (d <= m) gc[d] = __double2float_rn(__dadd_rn((double)gc[d], bmd[d]));
            }
            it = 0;
            while (__dsub_rn((double)gc[m], shift) >= bmd[m] && it++ < TRIC_MAX_ITER) {
#pragma unroll
                for (int d = 0; d < 3; ++d)
                    if (d <= m) gc[d] = __double2float_rn(__dsub_rn((double)gc[d], bmd[d]));
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) { g[i] = __fsub_rn(gc_in[i], gc[i]); dx[i] = 0.0; }
        return;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) { g[i] = gc_in[i]; dx[i] = (double)__fsub_rn(gc_in[i], bmid[i]); }
    const double hb[3] = {I[9 * F], I[10 * F], I[11 * F]};
    if (A.mode == TRIC_RECT) {  // pbc_dx mode 0, pyx:473-478
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double b = I[(4 * i) * F];
            long long it = 0;
            while (dx[i] > hb[i] && it++ < TRIC_MAX_ITER) dx[i] = __dsub_rn(dx[i], b);
            it = 0;
            while (dx[i] <= -hb[i] && it++ < TRIC_MAX_ITER) dx[i] = __dadd_rn(dx[i], b);
        }
        return;
    }
    const double max_cutoff2 = I[12 * F];  // pbc_dx mode 1, pyx:479-505: the vector search sits inside the axis loop
    const int ntric = A.ntric[f];
#pragma unroll
    for (int i = 2; i >= 0; --i) {
        double bi[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) bi[j] = j <= i ? I[(3 * i + j) * F] : 0.0;
        long long it = 0;
        while (dx[i] > hb[i] && it++ < TRIC_MAX_ITER) {
#pragma unroll
            for (int j = 2; j >= 0; --j)
                if (j <= i) dx[j] = __dsub_rn(dx[j], bi[j]);
        }
        it = 0;
        while (dx[i] <= -hb[i] && it++ < TRIC_MAX_ITER) {
#pragma unroll
            for (int j = 2; j >= 0; --j)
                if (j <= i) dx[j] = __dadd_rn(dx[j], bi[j]);
        }
        double d2min = tric_norm2(dx);
        if (d2min > max_cutoff2) {
            const double s0 = dx[0], s1 = dx[1], s2 = dx[2];
            int k = 0;
            while (d2min > max_cutoff2 && k < ntric) {
                double trial[3];
                trial[0] = __dadd_rn(s0, I[(14 + 3 * k) * F]);
                trial[1] = __dadd_rn(s1, I[(15 + 3 * k) * F]);
                trial[2] = __dadd_rn(s2, I[(16 + 3 * k) * F]);
                const double d2t = tric_norm2(trial);
                if (d2t < d2min) { dx[0] = trial[0]; dx[1] = trial[1]; dx[2] = trial[2]; d2min = d2t; }
                ++k;
            }
        }
    }
}

// the stored coordinate of one atom / axis: triclinic x' - g (pyx:261-262); compact ((x' - g) + bm) + dx (pyx:343-344)
__device__ __forceinline__ float tric_apply(int mode, float x, float wc, float bm, float g, double dx) {
    const float xp = __fadd_rn(__fsub_rn(x, wc), bm);
    if (mode == TRIC_TRICLINIC) return __fsub_rn(xp, g);
    return __double2float_rn(__dadd_rn((double)__fadd_rn(__fsub_rn(xp, g), bm), dx));
}

// small groups: one thread per (group, frame)
__device__ __forceinline__ void tric_small_groups(const TricArgs &A, long long tid) {
    if (tid >= A.n_ranges * A.F) return;
    const long long g = tid / A.F, f = tid - g * A.F;
    const long long s = A.groups[g];
    const int count = (int)max(min((long long)A.groups[g + 1] - s, (long long)(WRAP_SMALL + 1)), -1ll);
    if (count <= 0 || count > WRAP_SMALL) return;
    float *base = A.coords + s * 3 * A.fs + f;
    float wc[3], bm[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { wc[i] = A.wc[(long long)i * A.F + f]; bm[i] = A.bm[(long long)i * A.F + f]; }
    float v[WRAP_SMALL][3];
#pragma unroll
    for (int k = 0; k < WRAP_SMALL; ++k)
        if (k < count) {
#pragma unroll
            for (int i = 0; i < 3; ++i) v[k][i] = base[(long long)(k * 3 + i) * A.fs];
        }
    float c[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < WRAP_SMALL; ++k)
        if (k < count) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const float xp = __fadd_rn(__fsub_rn(v[k][i], wc[i]), bm[i]);
                c[i] = __fadd_rn(c[i], __fdiv_rn(__fsub_rn(xp, c[i]), (float)(k + 1)));
            }
        }
    float gg[3];
    double dx[3];
    tric_decide(A, f, c, bm, gg, dx);
#pragma unroll
    for (int k = 0; k < WRAP_SMALL; ++k)
        if (k < count) {
#pragma unroll
            for (int i = 0; i < 3; ++i)
                base[(long long)(k * 3 + i) * A.fs] = tric_apply(A.mode, v[k][i], wc[i], bm[i], gg[i], dx[i]);
        }
}

struct TricSmem {
    float g[3][32];
    double dx[3][32];
};

__global__ void __launch_bounds__(WRAP_THREADS, 3) tric_groups_kernel(const TricArgs A) {
    __shared__ ChainSmem sm;
    __shared__ TricSmem ts;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    if ((int)blockIdx.x >= A.n_long_ctas) {
        tric_small_groups(A, ((long long)blockIdx.x - A.n_long_ctas) * WRAP_THREADS + t);
        return;
    }
    const long long nchunks = (A.F + 31) / 32;
    const long long total = (long long)(*A.n_long) * nchunks;
    for (long long item = blockIdx.x; item < total; item += A.n_long_ctas) {
        const long long slot = item / nchunks, f0 = 32 * (item - slot * nchunks);
        const int nf = (int)(A.F - f0 < 32 ? A.F - f0 : 32);
        const long long g = A.long_list[slot];
        const long long s = A.groups[g], count = (long long)A.groups[g + 1] - s;
        const long long f = f0 + (lane < nf ? lane : 0);
        float wcl[3], bml[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) { wcl[i] = A.wc[(long long)i * A.F + f]; bml[i] = A.bm[(long long)i * A.F + f]; }
        const float wsub = w == 0 ? wcl[0] : (w == 1 ? wcl[1] : wcl[2]);
        const float wadd = w == 0 ? bml[0] : (w == 1 ? bml[1] : bml[2]);
        const float c = chain_32frames<false, true>(sm, A.coords, A.fs, f0, nf, nullptr, s, count, wsub, wadd);
        if (w < 3) sm.tr[w][lane] = c;
        __syncthreads();
        if (w == 0 && lane < nf) {
            const float gc[3] = {sm.tr[0][lane], sm.tr[1][lane], sm.tr[2][lane]};
            float gg[3];
            double dx[3];
            tric_decide(A, f, gc, bml, gg, dx);
#pragma unroll
            for (int i = 0; i < 3; ++i) { ts.g[i][lane] = gg[i]; ts.dx[i][lane] = dx[i]; }
        }
        __syncthreads();
        if (lane < nf) {
            const float g0 = ts.g[0][lane], g1 = ts.g[1][lane], g2 = ts.g[2][lane];
            const double d0 = ts.dx[0][lane], d1 = ts.dx[1][lane], d2 = ts.dx[2][lane];
            float *base = A.coords + s * 3 * A.fs + f0 + lane;
            constexpr int BATCH = 4;
            for (long long k0 = w; k0 < count; k0 += WRAP_WARPS * BATCH) {
                float v[BATCH][3];
#pragma unroll
                for (int u = 0; u < BATCH; ++u) {
                    const long long k = k0 + WRAP_WARPS * u;
                    const float *p = base + k * 3 * A.fs;
                    if (k < count) { v[u][0] = p[0]; v[u][1] = p[A.fs]; v[u][2] = p[2 * A.fs]; }
                }
#pragma unroll
                for (int u = 0; u < BATCH; ++u) {
                    const long long k = k0 + WRAP_WARPS * u;
                    float *p = base + k * 3 * A.fs;
                    if (k < count) {
                        p[0] = tric_apply(A.mode, v[u][0], wcl[0], bml[0], g0, d0);
                        p[A.fs] = tric_apply(A.mode, v[u][1], wcl[1], bml[1], g1, d1);
                        p[2 * A.fs] = tric_apply(A.mode, v[u][2], wcl[2], bml[2], g2, d2);
                    }
                }
            }
        }
        __syncthreads();  // sm.tr / ts and the ring are reused by the next item
    }
}

// atoms that belong to no group ([0, groups[0]) and [groups[last], n_atoms)) are only centred (pyx:221-223); normally
// there are none and the fixed-size grid returns after two loads
__global__ void tric_center_only_kernel(float *__restrict__ coords, long long fs, long long F, long long N,
                                        const unsigned *__restrict__ groups, long long n_ranges,
                                        const float *__restrict__ wc, const float *__restrict__ bm) {
    long long lo = N, hi = N;
    if (n_ranges > 0) {
        lo = min((long long)groups[0], N);
        hi = min(max((long long)groups[n_ranges], lo), N);
    }
    const long long rows = (lo + (N - hi)) * 3, total = rows * F;
    for (long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x; tid < total;
         tid += (long long)gridDim.x * blockDim.x) {
        const long long r = tid / F, f = tid - r * F;
        const long long row = r < lo * 3 ? r : r - lo * 3 + hi * 3;  // (atom, axis) row of the trajectory
        const int i = (int)(row % 3);
        float *p = coords + row * fs + f;
        *p = __fadd_rn(__fsub_rn(*p, wc[(long long)i * F + f]), bm[(long long)i * F + f]);
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_wrap_box(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *groups, int64_t n_groups,
                            const uint32_t *centersel, int64_t n_centersel, const float *center) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (t->n_atoms < 0 || t->n_frames < 0 || n_groups < 0 || n_centersel < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (t->n_atoms >= (1ll << 31) || n_centersel >= (1ll << 31) || n_groups >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "n_atoms / n_centersel / n_groups must be < 2^31");
    if (n_centersel == 0 && !center) return fail(h, MKB_ERR_BAD_ARG, "center is required when centersel is empty");
    if (n_centersel > 0 && !centersel) return fail(h, MKB_ERR_BAD_ARG, "null centersel");
    const long long F = t->n_frames, n_ranges = n_groups - 1;
    if (F == 0 || n_ranges <= 0 || t->n_atoms == 0) return MKB_OK;  // pyx:110,123: empty loops
    if (!t->coords || !t->box || !groups) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < F || t->frame_stride_box < F) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const long long nchunks = cdiv(F, 32);
    const long long small_blocks = cdiv(n_ranges * F, WRAP_THREADS);
    if (small_blocks + 4ll * h->sm_count >= (1ll << 31) || nchunks >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "groups x frames too large for one launch");
    float *centre = nullptr;
    unsigned *long_list = nullptr, *n_long = nullptr;
    int rc;
    if ((rc = scratch_get(h, S_COM, (size_t)(3 * F), &centre))) return rc;
    if ((rc = scratch_get(h, S_ITEM_CELL, (size_t)n_ranges, &long_list))) return rc;
    if ((rc = scratch_get(h, S_CELL_COUNT, (size_t)1, &n_long))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemsetAsync(n_long, 0, sizeof(unsigned), st));
    wrap_classify_kernel<<<(unsigned)cdiv(n_ranges, 256), 256, 0, st>>>(groups, n_ranges, long_list, n_long);
    MKB_LAUNCHED(h);
    if (n_centersel > 0) {
        wrap_center_kernel<<<(unsigned)nchunks, WRAP_THREADS, 0, st>>>(t->coords, F, t->frame_stride, centersel,
                                                                      n_centersel, centre);
        MKB_LAUNCHED(h);
    }
    WrapArgs A;
    A.coords = const_cast<float *>(t->coords);
    A.box = t->box;
    A.F = F; A.fs = t->frame_stride; A.fsb = t->frame_stride_box;
    A.groups = groups; A.n_ranges = n_ranges;
    A.centre = centre;
    A.cx = center ? center[0] : 0.f; A.cy = center ? center[1] : 0.f; A.cz = center ? center[2] : 0.f;
    A.fixed_centre = n_centersel == 0 ? 1 : 0;
    A.long_list = long_list; A.n_long = n_long;
    A.n_long_ctas = (int)std::min<long long>(n_ranges * nchunks, 4ll * h->sm_count);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    wrap_groups_kernel<<<(unsigned)(A.n_long_ctas + small_blocks), WRAP_THREADS, 0, st>>>(A);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_wrap_triclinic(mkb_handle_t h, void *stream, const mkb_traj *t, const double *boxvectors,
                                  int64_t bv_frame_stride, const uint32_t *groups, int64_t n_groups,
                                  const uint32_t *centersel, int64_t n_centersel, const float *center, int32_t unitcell) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (unitcell != TRIC_RECT && unitcell != TRIC_COMPACT && unitcell != TRIC_TRICLINIC)
        return fail(h, MKB_ERR_BAD_ARG, "unitcell must be 0 (rectangular), 1 (compact) or 2 (triclinic)");
    if (t->n_atoms < 0 || t->n_frames < 0 || n_groups < 0 || n_centersel < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (t->n_atoms >= (1ll << 31) || n_centersel >= (1ll << 31) || n_groups >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "n_atoms / n_centersel / n_groups must be < 2^31");
    if (n_centersel == 0 && !center) return fail(h, MKB_ERR_BAD_ARG, "center is required when centersel is empty");
    if (n_centersel > 0 && !centersel) return fail(h, MKB_ERR_BAD_ARG, "null centersel");
    const long long F = t->n_frames, n_ranges = n_groups > 0 ? n_groups - 1 : 0, N = t->n_atoms;
    if (F == 0 || N == 0) return MKB_OK;
    if (!t->coords || !boxvectors || (n_groups > 0 && !groups)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < F || bv_frame_stride < F) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const long long nchunks = cdiv(F, 32);
    const long long small_blocks = cdiv(n_ranges * F, WRAP_THREADS);
    if (small_blocks + 4ll * h->sm_count >= (1ll << 31) || nchunks >= (1ll << 31) || cdiv(N * 3 * F, 256) >= (1ll << 31))
        return fail(h, MKB_ERR_BAD_ARG, "atoms x frames too large for one launch");
    // scratch: centre [3][F] | box_middle [3][F] | ntric [F] | err in S_COM; the frame table in S_SORT_PX
    float *fbuf = nullptr;
    double *info = nullptr;
    unsigned *long_list = nullptr, *n_long = nullptr;
    int rc;
    if ((rc = scratch_get(h, S_COM, (size_t)(7 * F + 4), &fbuf))) return rc;
    if ((rc = scratch_get(h, S_SORT_PX, (size_t)(TRIC_NINFO * F), &info))) return rc;
    if ((rc = scratch_get(h, S_ITEM_CELL, (size_t)std::max<long long>(n_ranges, 1), &long_list))) return rc;
    if ((rc = scratch_get(h, S_CELL_COUNT, (size_t)1, &n_long))) return rc;
    float *wc = fbuf, *bm = fbuf + 3 * F;
    int *ntric = reinterpret_cast<int *>(fbuf + 6 * F), *err = ntric + F;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemsetAsync(n_long, 0, sizeof(unsigned), st));
    MKB_CUDA(h, cudaMemsetAsync(err, 0, sizeof(int), st));
    if (n_ranges > 0) {
        wrap_classify_kernel<<<(unsigned)cdiv(n_ranges, 256), 256, 0, st>>>(groups, n_ranges, long_list, n_long);
        MKB_LAUNCHED(h);
    }
    if (n_centersel > 0) {  // pyx:180-185: the wrap centre is the running mean of the selection in the ORIGINAL coordinates
        wrap_center_kernel<<<(unsigned)nchunks, WRAP_THREADS, 0, st>>>(t->coords, F, t->frame_stride, centersel,
                                                                      n_centersel, wc);
        MKB_LAUNCHED(h);
    }
    tric_frame_kernel<<<(unsigned)cdiv(F, 128), 128, 0, st>>>(boxvectors, bv_frame_stride, F, unitcell, n_centersel == 0,
                                                             center ? center[0] : 0.f, center ? center[1] : 0.f,
                                                             center ? center[2] : 0.f, info, bm, wc, ntric, err);
    MKB_LAUNCHED(h);
    if (unitcell != TRIC_TRICLINIC) {
        int herr = 0;
        MKB_CUDA(h, cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, st));
        MKB_CUDA(h, cudaStreamSynchronize(st));
        if (herr) return fail(h, MKB_ERR_BAD_ARG, "Too many triclinic vectors!!");
    }
    TricArgs A;
    A.coords = const_cast<float *>(t->coords);
    A.F = F; A.fs = t->frame_stride; A.n_atoms = N;
    A.groups = groups; A.n_ranges = n_ranges;
    A.info = info; A.bm = bm; A.wc = wc; A.ntric = ntric; A.mode = unitcell;
    A.long_list = long_list; A.n_long = n_long;
    A.n_long_ctas = (int)std::min<long long>(n_ranges * nchunks, 3ll * h->sm_count);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    tric_center_only_kernel<<<(unsigned)(8 * h->sm_count), 256, 0, st>>>(A.coords, A.fs, F, N, groups, n_ranges, wc, bm);
    MKB_LAUNCHED(h);
    if (n_ranges > 0) {
        tric_groups_kernel<<<(unsigned)(A.n_long_ctas + small_blocks), WRAP_THREADS, 0, st>>>(A);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "tric_groups_kernel";
    return MKB_OK;
}
