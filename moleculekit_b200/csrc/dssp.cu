// dssp.cu -- K18: DSSP secondary structure over a trajectory for sm_90a (H100).
//
// Replaces mdtraj's compute_dssp (a single-threaded C++ port of DSSP 2.2.0) that moleculekit's MetricSecondaryStructure
// calls once per frame.  The contract (include/mkb200.h) restates the reference's rules; every float64 operation is
// rounded on its own (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so the energies are bit-identical
// to a C restatement compiled without contraction, and the codes follow from them exactly.
//
// Per chunk of listed frames (bounded scratch, DS_CHUNK_BYTES), every array frame-major [frame][residue]:
//   gather    lane = frame on the read (one 128-byte line per (atom, axis) row of 32 frames); writes the float32 N, CA,
//             C, O, the float64 amide H and the break bit after the residue, plus a compact CA float4 array.
//   hbond     one warp per (frame, donor): the lanes stride over the acceptors, screen the CA distance (a float32
//             pre-screen whose band is decided exactly: d2 > 82 cannot have a float64 distance < 9), evaluate the float64
//             energy, keep a per-lane top-2 with the reference's insertion rule and merge the lanes' lists by (E, index).
//   flags     one thread per (frame, residue): turn bits per stride (IsStart), the bend bit and the bridges of the residue
//             among its <= 8 candidates (the bonded partners of i and i + 1 and those plus one).
//   ladders   one thread per frame: the reference's bridge grouping in its (i, j) order and its ladder erase loop, over
//             the candidates found above.  Only these run sequentially; they touch a few bytes per residue.
//   codes     one CTA per frame: E / B, H, G, I, then T / S, phase by phase with barriers.
#include <algorithm>

#include "common.cuh"

namespace mkb {

constexpr int DS_WARPS = 8;                         // donors per CTA of the hbond kernel
constexpr int DS_THREADS = 32 * DS_WARPS;
constexpr int DS_CAND = 8;                          // bridge candidates per residue
constexpr int DS_ACT = 2 * DS_CAND;                 // bridges that can still grow at one step of the grouping
constexpr size_t DS_CHUNK_BYTES = size_t(256) << 20;
constexpr long long DS_MAX_RES = 1ll << 28;         // j << 2 | type fits an int32
constexpr double DS_K = -27.888, DS_MIN_E = -9.9, DS_BOND_E = -0.5;

enum : unsigned char { F_T3 = 1, F_T4 = 2, F_T5 = 4, F_BENT = 8, F_BRK = 16, F_CAND = 32 };
enum : int { BR_PAR = 1, BR_ANTI = 2 };

struct DsRec {
    float n[3], ca[3], c[3], o[3];
    double h[3];
    int brk;                  // a break lies between this residue and the next
    int pad;
};
static_assert(sizeof(DsRec) == 80, "record layout");

struct DsBridge {
    int type, ib, ie, jb, je, size;
};

struct DsArgs {
    const float *coords;
    long long fs;
    const int *bb;            // [n][4] atom rows of N, CA, C, O
    const unsigned char *flags;
    long long n;
    const unsigned *frames;
    double bend_cos;
};

struct DsChunk {
    DsRec *rec;               // [fc][n]
    float4 *ca;               // [fc][n]
    int2 *bond;               // [fc][n] partners with E < -0.5, else -1
    unsigned char *flg;       // [fc][n] F_* bits
    unsigned char *mark;      // [fc][n] G (bit 0) and I (bit 1) starts
    int *cand;                // [fc][n][DS_CAND] bridges of residue i: j << 2 | type, ascending j, -1 after the last
    int *pre;                 // [fc][n + 1] breaks before each residue (prefix)
    DsBridge *br;             // [fc][DS_CAND n]
    int *nbr;                 // [fc] bridges left after the ladder merge
};

__device__ __forceinline__ double ds_dist(double ax, double ay, double az, double bx, double by, double bz) {
    const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by), dz = __dsub_rn(az, bz);
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

__device__ __forceinline__ double ds_dist(const float *a, const float *b) {
    return ds_dist((double)a[0], (double)a[1], (double)a[2], (double)b[0], (double)b[1], (double)b[2]);
}

// thread t = r * fc + kl (frame fastest: consecutive frames of one atom row are one coalesced read)
__global__ void dssp_gather_kernel(const DsArgs A, long long k0, int fc, DsChunk S) {
    const long long total = (long long)fc * A.n;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / fc, kl = t - r * fc, k = k0 + kl;
        const long long f = A.frames ? (long long)A.frames[k] : k;
        auto ld3 = [&](long long res, int atom, float *p) {
            const float *src = A.coords + (long long)A.bb[4 * res + atom] * 3 * A.fs + f;
            p[0] = __ldg(src); p[1] = __ldg(src + A.fs); p[2] = __ldg(src + 2 * A.fs);
        };
        DsRec R;
        ld3(r, 0, R.n); ld3(r, 1, R.ca); ld3(r, 2, R.c); ld3(r, 3, R.o);
        R.brk = 0;
        R.pad = 0;
        if (r + 1 < A.n) {
            float nn[3];
            ld3(r + 1, 0, nn);
            R.brk = (A.flags[r + 1] & 2) || ds_dist(R.c, nn) > 2.5;
        }
        R.h[0] = R.n[0]; R.h[1] = R.n[1]; R.h[2] = R.n[2];
        if (!(A.flags[r] & 1) && r > 0) {
            float pc[3], po[3];
            ld3(r - 1, 2, pc);
            ld3(r - 1, 3, po);
            const bool brk = (A.flags[r] & 2) || ds_dist(pc, R.n) > 2.5;
            if (!brk) {
                const double vx = __dsub_rn(pc[0], po[0]), vy = __dsub_rn(pc[1], po[1]), vz = __dsub_rn(pc[2], po[2]);
                const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)), __dmul_rn(vz, vz)));
                R.h[0] = __dadd_rn((double)R.n[0], __ddiv_rn(vx, len));
                R.h[1] = __dadd_rn((double)R.n[1], __ddiv_rn(vy, len));
                R.h[2] = __dadd_rn((double)R.n[2], __ddiv_rn(vz, len));
            }
        }
        S.rec[kl * A.n + r] = R;
        S.ca[kl * A.n + r] = make_float4(R.ca[0], R.ca[1], R.ca[2], 0.f);
    }
}

__device__ __forceinline__ double ds_energy(const DsRec &D, const DsRec &Acc) {
    const double dHO = ds_dist(D.h[0], D.h[1], D.h[2], Acc.o[0], Acc.o[1], Acc.o[2]);
    const double dHC = ds_dist(D.h[0], D.h[1], D.h[2], Acc.c[0], Acc.c[1], Acc.c[2]);
    const double dNC = ds_dist(D.n, Acc.c), dNO = ds_dist(D.n, Acc.o);
    double e;
    if (dHO < 0.5 || dHC < 0.5 || dNC < 0.5 || dNO < 0.5)
        e = DS_MIN_E;
    else
        e = __dsub_rn(__dadd_rn(__dsub_rn(__ddiv_rn(DS_K, dHO), __ddiv_rn(DS_K, dHC)), __ddiv_rn(DS_K, dNC)),
                      __ddiv_rn(DS_K, dNO));
    e = __ddiv_rn(round(__dmul_rn(e, 1000.0)), 1000.0);
    if (e < DS_MIN_E) e = DS_MIN_E;
    return e;
}

// (ea, pa) before (eb, pb): energy, then index; an empty slot is (0.0, -1), which sorts after every kept entry (E < 0)
__device__ __forceinline__ bool ds_before(double ea, int pa, double eb, int pb) {
    return ea < eb || (ea == eb && (unsigned)pa < (unsigned)pb);
}

__global__ void __launch_bounds__(DS_THREADS) dssp_hbond_kernel(const DsArgs A, long long k0, DsChunk S,
                                                                int *__restrict__ hb_partner,
                                                                double *__restrict__ hb_energy) {
    const int lane = threadIdx.x & 31;
    const long long d = (long long)blockIdx.x * DS_WARPS + (threadIdx.x >> 5);
    if (d >= A.n) return;  // whole warps only: no block-wide barrier follows
    const long long kl = blockIdx.y, base = kl * A.n;
    double e0 = 0.0, e1 = 0.0;
    int p0 = -1, p1 = -1;
    if (!(A.flags[d] & 1)) {
        const DsRec D = S.rec[base + d];
        const float4 cd = S.ca[base + d];
        for (long long a = lane; a < A.n; a += 32) {
            if (a == d || a == d - 1) continue;
            const float4 ca = S.ca[base + a];
            const float dx = __fsub_rn(ca.x, cd.x), dy = __fsub_rn(ca.y, cd.y), dz = __fsub_rn(ca.z, cd.z);
            const float d2 = sq3(dx, dy, dz);
            if (d2 > 82.f) continue;  // the float64 distance is > 9 there
            if (ds_dist(cd.x, cd.y, cd.z, ca.x, ca.y, ca.z) < 9.0) {
                const double e = ds_energy(D, S.rec[base + a]);
                if (e < e0) {
                    e1 = e0; p1 = p0;
                    e0 = e; p0 = (int)a;
                } else if (e < e1) {
                    e1 = e; p1 = (int)a;
                }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double oe0 = __shfl_xor_sync(0xffffffffu, e0, off), oe1 = __shfl_xor_sync(0xffffffffu, e1, off);
            const int op0 = __shfl_xor_sync(0xffffffffu, p0, off), op1 = __shfl_xor_sync(0xffffffffu, p1, off);
            if (ds_before(oe0, op0, e0, p0)) {
                if (ds_before(oe1, op1, e0, p0)) { e1 = oe1; p1 = op1; }
                else { e1 = e0; p1 = p0; }
                e0 = oe0; p0 = op0;
            } else if (ds_before(oe0, op0, e1, p1)) {
                e1 = oe0; p1 = op0;
            }
        }
    }
    if (lane == 0) {
        S.bond[base + d] = make_int2(e0 < DS_BOND_E ? p0 : -1, e1 < DS_BOND_E ? p1 : -1);
        if (hb_partner) {
            const long long o = 2 * ((k0 + kl) * A.n + d);
            hb_partner[o] = p0; hb_partner[o + 1] = p1;
            hb_energy[o] = e0; hb_energy[o + 1] = e1;
        }
    }
}

__device__ __forceinline__ bool ds_bond(const int2 *bond, long long x, long long y) {
    const int2 b = bond[x];
    return b.x == y || b.y == y;
}

// no break between consecutive residues of [a, b] (short ranges)
__device__ __forceinline__ bool ds_ncb(const DsRec *rec, long long a, long long b) {
    for (long long k = a; k < b; ++k)
        if (rec[k].brk) return false;
    return true;
}

__device__ __forceinline__ int ds_bridge(const DsRec *rec, const int2 *bond, long long i, long long j) {
    const long long a = i - 1, b = i, c = i + 1, d = j - 1, e = j, f = j + 1;
    if (!(ds_ncb(rec, a, c) && ds_ncb(rec, d, f))) return 0;
    if ((ds_bond(bond, c, e) && ds_bond(bond, e, a)) || (ds_bond(bond, f, b) && ds_bond(bond, b, d))) return BR_PAR;
    if ((ds_bond(bond, c, d) && ds_bond(bond, f, a)) || (ds_bond(bond, e, b) && ds_bond(bond, b, e))) return BR_ANTI;
    return 0;
}

// t = kl * n + i
__global__ void dssp_flags_kernel(const DsArgs A, int fc, DsChunk S) {
    const long long n = A.n, total = (long long)fc * n;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long kl = t / n, i = t - kl * n;
        const DsRec *rec = S.rec + kl * n;
        const int2 *bond = S.bond + kl * n;
        unsigned char fl = rec[i].brk ? F_BRK : 0;
        for (int s = 3; s <= 5; ++s)
            if (i + s < n && ds_ncb(rec, i, i + s) && ds_bond(bond, i + s, i)) fl |= (unsigned char)(1 << (s - 3));
        if (i >= 2 && i + 2 < n && ds_ncb(rec, i - 2, i + 2)) {
            const float *p = rec[i - 2].ca, *q = rec[i].ca, *s = rec[i + 2].ca;
            double u[3], w[3];
#pragma unroll
            for (int x = 0; x < 3; ++x) {
                u[x] = __dsub_rn(q[x], p[x]);
                w[x] = __dsub_rn(s[x], q[x]);
            }
            const double uu = __dadd_rn(__dadd_rn(__dmul_rn(u[0], u[0]), __dmul_rn(u[1], u[1])), __dmul_rn(u[2], u[2]));
            const double ww = __dadd_rn(__dadd_rn(__dmul_rn(w[0], w[0]), __dmul_rn(w[1], w[1])), __dmul_rn(w[2], w[2]));
            const double uw = __dadd_rn(__dadd_rn(__dmul_rn(u[0], w[0]), __dmul_rn(u[1], w[1])), __dmul_rn(u[2], w[2]));
            const double x = __dmul_rn(uu, ww);
            double c = 0.0;
            if (x > 0) c = __ddiv_rn(uw, __dsqrt_rn(x));
            if (c < A.bend_cos) fl |= F_BENT;
        }
        int *cand = S.cand + (kl * n + i) * DS_CAND;
        int nc = 0;
        if (i >= 1 && i + 4 < n) {
            // every bridge rule holds a bond whose donor is i or i + 1 and whose acceptor is j or j - 1
            const int2 b0 = bond[i], b1 = bond[i + 1];
            const int src[4] = {b0.x, b0.y, b1.x, b1.y};
            int js[DS_CAND], m = 0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (src[q] < 0) continue;
#pragma unroll
                for (int o = 0; o < 2; ++o) {
                    const int j = src[q] + o;
                    if (j < i + 3 || j + 1 >= n) continue;
                    bool dup = false;
                    for (int z = 0; z < m; ++z) dup |= js[z] == j;
                    if (!dup) js[m++] = j;
                }
            }
            for (int z = 1; z < m; ++z)  // ascending j, the reference's inner loop order
                for (int y = z; y > 0 && js[y - 1] > js[y]; --y) { const int tmp = js[y]; js[y] = js[y - 1]; js[y - 1] = tmp; }
            for (int z = 0; z < m; ++z) {
                const int type = ds_bridge(rec, bond, i, js[z]);
                if (type) cand[nc++] = (js[z] << 2) | type;
            }
        }
        if (nc < DS_CAND) cand[nc] = -1;
        if (nc) fl |= F_CAND;
        S.flg[kl * n + i] = fl;
    }
}

// one thread per frame: the reference's bridge grouping and ladder merge
__global__ void dssp_ladder_kernel(const DsArgs A, int fc, DsChunk S) {
    const long long kl = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (kl >= fc) return;
    const long long n = A.n;
    const unsigned char *flg = S.flg + kl * n;
    int *pre = S.pre + kl * (n + 1);
    DsBridge *br = S.br + kl * DS_CAND * n;
    pre[0] = 0;
    for (long long k = 0; k < n; ++k) pre[k + 1] = pre[k] + ((flg[k] & F_BRK) ? 1 : 0);
    // grouping: bridge (i, j) joins the first bridge in vector order of its type with i == i.back + 1 and
    // j == j.back + 1 (parallel) or j == j.front - 1 (antiparallel).  Only bridges extended or created at step i - 1 can
    // match at step i, at most DS_CAND of them, and `act` keeps them in vector order.
    int act[DS_ACT], na = 0, nb = 0;
    for (long long i = 1; i + 4 < n; ++i) {
        int keep = 0;
        for (int z = 0; z < na; ++z)
            if (br[act[z]].ie == i - 1) act[keep++] = act[z];
        na = keep;
        if (!(flg[i] & F_CAND)) continue;
        const int *cand = S.cand + (kl * n + i) * DS_CAND;
        for (int m = 0; m < DS_CAND && cand[m] >= 0; ++m) {
            const int j = cand[m] >> 2, type = cand[m] & 3;
            bool found = false;
            for (int z = 0; z < na && !found; ++z) {
                DsBridge &B = br[act[z]];
                if (type != B.type || i != B.ie + 1) continue;
                if (type == BR_PAR && B.je + 1 == j) {
                    B.ie = (int)i; B.je = j; ++B.size;
                    found = true;
                } else if (type == BR_ANTI && B.jb - 1 == j) {
                    B.ie = (int)i; B.jb = j; ++B.size;
                    found = true;
                }
            }
            if (!found) {
                br[nb] = DsBridge{type, (int)i, (int)i, j, j, 1};
                act[na++] = nb++;
            }
        }
    }
    // ladders: the bridges are in creation order, which is sorted by i.front; the erase loop with uint32 differences.
    // Later q have ibq >= the current one, so once ibq - iep >= 6 holds as integers nothing after q can merge into p.
    for (int p = 0; p < nb; ++p) {
        if (br[p].type == 0) continue;
        for (int q = p + 1; q < nb; ++q) {
            DsBridge &P = br[p], &Q = br[q];
            if (Q.type == 0) continue;
            if (Q.ib - P.ie >= 6) break;
            const unsigned ibi = P.ib, iei = P.ie, jbi = P.jb, jei = P.je;
            const unsigned ibj = Q.ib, iej = Q.ie, jbj = Q.jb, jej = Q.je;
            const unsigned lo_i = min(ibi, ibj), hi_i = max(iei, iej), lo_j = min(jbi, jbj), hi_j = max(jei, jej);
            if (P.type != Q.type || pre[hi_i] != pre[lo_i] || pre[hi_j] != pre[lo_j] || ibj - iei >= 6u ||
                (iei >= ibj && ibi <= iej))
                continue;
            bool bulge;
            if (P.type == BR_PAR)
                bulge = (jbj - jei < 6u && ibj - iei < 3u) || jbj - jei < 3u;
            else
                bulge = (jbi - jej < 6u && ibj - iei < 3u) || jbi - jej < 3u;
            if (bulge) {
                P.ie = Q.ie;
                if (P.type == BR_PAR) P.je = Q.je;
                else P.jb = Q.jb;
                P.size += Q.size;
                Q.type = 0;  // erased
            }
        }
    }
    int kept = 0;
    for (int b = 0; b < nb; ++b)
        if (br[b].type) br[kept++] = br[b];
    S.nbr[kl] = kept;
}

// one CTA per frame: codes 0 loop, 1 H, 2 B, 3 E, 4 G, 5 I, 6 T, 7 S
__global__ void dssp_codes_kernel(const DsArgs A, long long k0, DsChunk S, unsigned char *__restrict__ codes,
                                  long long ld) {
    const long long kl = blockIdx.x, n = A.n;
    unsigned char *row = codes + (k0 + kl) * ld;
    const unsigned char *flg = S.flg + kl * n;
    unsigned char *mark = S.mark + kl * n;
    const DsBridge *br = S.br + kl * DS_CAND * n;
    const int nb = S.nbr[kl];
    for (long long r = threadIdx.x; r < n; r += blockDim.x) row[r] = 0;
    __syncthreads();
    for (int pass = 0; pass < 2; ++pass) {  // B first, then E over it: E wins wherever a ladder covers a residue
        for (int b = threadIdx.x; b < nb; b += blockDim.x) {
            const DsBridge B = br[b];
            if ((B.size > 1) != (pass == 1)) continue;
            const unsigned char ss = B.size > 1 ? 3 : 2;
            for (int r = B.ib; r <= B.ie; ++r) row[r] = ss;
            for (int r = B.jb; r <= B.je; ++r) row[r] = ss;
        }
        __syncthreads();
    }
    for (long long r = threadIdx.x; r < n; r += blockDim.x) {
        bool h = false;
        for (long long i = max(1ll, r - 3); i <= r; ++i) h |= i + 4 < n && (flg[i] & F_T4) && (flg[i - 1] & F_T4);
        if (h) row[r] = 1;
    }
    __syncthreads();
    // G (stride 3, span 3) and then I (stride 5, span 5): a start counts when every residue of its span is loop before
    // the phase (a G of the same phase is allowed, and the phase writes nothing else)
    for (int ph = 0; ph < 2; ++ph) {
        const int span = ph == 0 ? 3 : 5;
        const unsigned char bit = ph == 0 ? F_T3 : F_T5, code = ph == 0 ? 4 : 5;
        for (long long i = threadIdx.x; i < n; i += blockDim.x) {
            bool ok = i >= 1 && i + span < n && (flg[i] & bit) && (flg[i - 1] & bit);
            for (int k = 0; ok && k < span; ++k) ok = row[i + k] == 0;
            mark[i] = ok;
        }
        __syncthreads();
        for (long long r = threadIdx.x; r < n; r += blockDim.x) {
            bool g = false;
            for (long long i = max(0ll, r - span + 1); i <= r; ++i) g |= mark[i] != 0;
            if (g) row[r] = code;
        }
        __syncthreads();
    }
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        if (i < 1 || i + 1 >= n || row[i] != 0) continue;
        bool turn = false;
        for (int s = 3; s <= 5 && !turn; ++s)
            for (int k = 1; k < s && !turn; ++k) turn = i >= k && (flg[i - k] & (1 << (s - 3)));
        if (turn) row[i] = 6;
        else if (flg[i] & F_BENT) row[i] = 7;
    }
}

inline size_t ds_align(size_t b) { return (b + 255) & ~size_t(255); }

// scratch bytes of fc frames, laid out as the DsChunk arrays
inline size_t ds_bytes(long long fc, long long n) {
    const size_t f = (size_t)fc, m = (size_t)n;
    return ds_align(f * m * sizeof(DsRec)) + ds_align(f * m * sizeof(float4)) + ds_align(f * m * sizeof(int2)) +
           2 * ds_align(f * m) + ds_align(f * m * DS_CAND * sizeof(int)) + ds_align(f * (m + 1) * sizeof(int)) +
           ds_align(f * m * DS_CAND * sizeof(DsBridge)) + ds_align(f * sizeof(int));
}

inline long long ds_chunk_frames(long long n) {
    const long long per = (long long)ds_bytes(1, n);
    long long fc = std::max<long long>(1, (long long)DS_CHUNK_BYTES / per);
    return std::min<long long>(fc, 65535);
}

template <typename T>
inline T *ds_carve(char *&p, size_t count) {
    T *r = reinterpret_cast<T *>(p);
    p += ds_align(count * sizeof(T));
    return r;
}

}  // namespace mkb

using namespace mkb;

extern "C" int64_t mkb_dssp_chunk_frames(int64_t n_res) {
    if (n_res < 1 || n_res > DS_MAX_RES) return 0;
    return ds_chunk_frames(n_res);
}

extern "C" int mkb_dssp(mkb_handle_t h, void *stream, const mkb_traj *t, const int32_t *backbone, const uint8_t *flags,
                        int64_t n_res, double bend_cos, const uint32_t *frames, int64_t n_frames, uint8_t *codes,
                        int64_t ld, int32_t *hb_partner, double *hb_energy) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t) return fail(h, MKB_ERR_BAD_ARG, "null trajectory");
    if (n_res < 1 || n_res > DS_MAX_RES) return fail(h, MKB_ERR_BAD_ARG, "n_res %lld outside [1, 2^28]", (long long)n_res);
    if (t->n_frames < 0 || (frames && n_frames < 0)) return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !backbone || !flags) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((hb_partner == nullptr) != (hb_energy == nullptr))
        return fail(h, MKB_ERR_BAD_ARG, "hb_partner and hb_energy are given together or not at all");
    if (t->frame_stride < t->n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (ld < n_res) return fail(h, MKB_ERR_BAD_ARG, "ld %lld < n_res %lld", (long long)ld, (long long)n_res);
    const long long n = frames ? n_frames : t->n_frames;
    if (n == 0) return MKB_OK;
    if (!codes) return fail(h, MKB_ERR_BAD_ARG, "null codes");
    if (cdiv(n_res, DS_WARPS) >= (1ll << 31)) return fail(h, MKB_ERR_BAD_ARG, "too many residues for one launch");

    DsArgs A;
    A.coords = t->coords; A.fs = t->frame_stride;
    A.bb = backbone; A.flags = flags; A.n = n_res;
    A.frames = frames;
    A.bend_cos = bend_cos;

    const long long fcn = std::min(n, ds_chunk_frames(n_res));
    void *base = nullptr;
    int rc;
    if ((rc = scratch_get(h, S_DSSP, ds_bytes(fcn, n_res), &base)) != MKB_OK) return rc;
    char *p = static_cast<char *>(base);
    const size_t fm = (size_t)(fcn * n_res);
    DsChunk S;
    S.rec = ds_carve<DsRec>(p, fm);
    S.ca = ds_carve<float4>(p, fm);
    S.bond = ds_carve<int2>(p, fm);
    S.flg = ds_carve<unsigned char>(p, fm);
    S.mark = ds_carve<unsigned char>(p, fm);
    S.cand = ds_carve<int>(p, fm * DS_CAND);
    S.pre = ds_carve<int>(p, (size_t)fcn * (size_t)(n_res + 1));
    S.br = ds_carve<DsBridge>(p, fm * DS_CAND);
    S.nbr = ds_carve<int>(p, (size_t)fcn);

    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const int blocks = h->sm_count * 8;
    for (long long k0 = 0; k0 < n; k0 += fcn) {
        const int fc = (int)std::min(fcn, n - k0);
        const long long items = (long long)fc * n_res;
        const int gb = (int)std::min<long long>(cdiv(items, 256), blocks);
        dssp_gather_kernel<<<gb, 256, 0, st>>>(A, k0, fc, S);
        MKB_LAUNCHED(h);
        const dim3 grid((unsigned)cdiv(n_res, DS_WARPS), (unsigned)fc);
        dssp_hbond_kernel<<<grid, DS_THREADS, 0, st>>>(A, k0, S, hb_partner, hb_energy);
        MKB_LAUNCHED(h);
        dssp_flags_kernel<<<gb, 256, 0, st>>>(A, fc, S);
        MKB_LAUNCHED(h);
        dssp_ladder_kernel<<<(unsigned)cdiv(fc, 32), 32, 0, st>>>(A, fc, S);
        MKB_LAUNCHED(h);
        dssp_codes_kernel<<<fc, 256, 0, st>>>(A, k0, S, codes, ld);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "dssp_hbond_kernel";
    return MKB_OK;
}
