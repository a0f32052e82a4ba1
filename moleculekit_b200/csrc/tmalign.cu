// tmalign.cu -- K27: TM-align (Zhang & Skolnick, Nucleic Acids Res. 2005) of every listed frame against a reference,
// for sm_90a (H100).
//
// Replaces moleculekit's molTMalign (the TM-align program, one frame at a time on the CPU).  The contract
// (include/mkb200.h, mkb_tmalign) fixes every float64 operation and its order; products are __dmul_rn, so no multiply
// is fused into an add, and the sums, quotients and square roots are IEEE round-to-nearest as written.  The results are
// bit-identical to the C restatement compiled without contraction (tests/tmalign_oracle.c), which this file follows
// function by function; the fit is K19's (tm_fit.cuh).
//
// One warp runs one item (listed frame).  The searches are a long chain in which every step picks its input from the
// last, so the lanes share the control flow: every lane computes the same scalars (scores, fits, counts), and the work
// over pairs, residues and DP cells is split across the lanes:
//   - per-pair passes (transform, squared distance, score term) one pair per lane; the score is then summed in pair
//     order by every lane from the stored terms, so it keeps the sequential sum's bits;
//   - cut sets and gathered pair lists are compacted in order with a ballot per 32 pairs;
//   - a fit's 6 centroid sums and 9 H sums are 15 lanes' sequential chains, broadcast by shuffles, then K19's
//     Horn rotation (tm_horn_rotation) in every lane;
//   - NWDP_TM is an anti-diagonal wavefront, three diagonals of values and one decision byte per cell (the diagonal,
//     and v >= h), from which lane 0 walks the traceback.
// __syncwarp orders the lanes' stores before other lanes read them.  Each item's traces (float64), lists, codes and DP
// state live in its own slice of global scratch; items run in chunks of mkb_tmalign_chunk_frames(xlen, ylen), so the
// scratch stays bounded.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "common.cuh"
#include "tm_fit.cuh"

namespace mkb {
namespace tma {

constexpr int TA_WARPS = 4;                            // items per CTA
constexpr int TA_THREADS = 32 * TA_WARPS;
constexpr int TA_MAX_RES = 1024;
constexpr size_t TA_SCRATCH_BUDGET = (size_t)1 << 30;  // bytes of per-item scratch per launch at most
constexpr int N_EXT = 20;
constexpr unsigned FULL = 0xffffffffu;

#define MUL __dmul_rn
#define SYNC() __syncwarp()

struct Fit {
    double R[9], p[3], q[3];
};

struct Ctx {
    int xlen, ylen, lane;
    const double (*x)[3], (*y)[3];
    char *secx, *secy;
    double d0, d0_search, score_d8, D0_MIN, Lnorm;
    double (*xt)[3], (*xtm)[3], (*ytm)[3], (*r1)[3], (*r2)[3], *dis, *term;
    int *i_ali, *k_ali, *ifr, *tmpmap;
    double *val;          // three diagonals of xlen + 1
    unsigned char *path;  // (xlen + 1) x (ylen + 1) decision bytes
};

__device__ void identity_fit(Fit *F) {
    for (int k = 0; k < 9; ++k) F->R[k] = 0.0;
    for (int k = 0; k < 3; ++k) F->p[k] = F->q[k] = 0.0;
    F->R[0] = F->R[4] = F->R[8] = 1.0;
}

// K19's fit of the pairs (a[k], b[k]), k < n (n = 0: identity): the centroid sums in lanes 0-5 and the H sums about
// them in lanes 6-14, each a sequential chain in pair order, then the rotation in every lane
__device__ void fit(Ctx *C, const double (*a)[3], const double (*b)[3], int n, Fit *F) {
    SYNC();
    if (n < 1) {
        identity_fit(F);
        return;
    }
    const int lane = C->lane;
    double c = 0;
    if (lane < 6) {
        const double (*s)[3] = lane < 3 ? a : b;
        const int d = lane % 3;
        for (int k = 0; k < n; ++k) c += s[k][d];
        c = c / (double)n;
    }
    for (int d = 0; d < 3; ++d) {
        F->p[d] = __shfl_sync(FULL, c, d);
        F->q[d] = __shfl_sync(FULL, c, 3 + d);
    }
    double hs = 0;
    if (lane >= 6 && lane < 15) {
        const int r = (lane - 6) / 3, s = (lane - 6) % 3;
        const double pr = F->p[r], qs = F->q[s];
        for (int k = 0; k < n; ++k) hs += MUL(a[k][r] - pr, b[k][s] - qs);
    }
    double H[9];
    for (int m = 0; m < 9; ++m) H[m] = __shfl_sync(FULL, hs, 6 + m);
    tm_horn_rotation(H, F->R);
}

__device__ void xform(const Fit *F, const double a[3], double o[3]) {
    const double b0 = a[0] - F->p[0], b1 = a[1] - F->p[1], b2 = a[2] - F->p[2];
    for (int d = 0; d < 3; ++d) o[d] = MUL(F->R[3 * d], b0) + MUL(F->R[3 * d + 1], b1) + MUL(F->R[3 * d + 2], b2) + F->q[d];
}

__device__ double dist2(const double a[3], const double b[3]) {
    const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return MUL(dx, dx) + MUL(dy, dy) + MUL(dz, dz);
}

// the sequential sum of t[0..n), the same in every lane
__device__ double seqsum(const double *t, int n) {
    double s = 0;
    for (int k = 0; k < n; ++k) s += t[k];
    return s;
}

// in-order compaction: emit(pos, k) for every k < n with pred(k), pos counting from 0; returns the count (every lane)
template <class P, class E>
__device__ int compact(const Ctx *C, int n, P pred, E emit) {
    SYNC();
    int out = 0;
    const unsigned below = (1u << C->lane) - 1u;
    for (int base = 0; base < n; base += 32) {
        const int k = base + C->lane;
        const bool p = k < n && pred(k);
        const unsigned m = __ballot_sync(FULL, p);
        if (p) emit(out + __popc(m & below), k);
        out += __popc(m);
    }
    SYNC();
    return out;
}

/* ---------------------------------------------------------------------------------------------- secondary structure */
__device__ char sec_str(double d13, double d14, double d15, double d24, double d25, double d35) {
    double delta = 2.1;
    if (fabs(d15 - 6.37) < delta && fabs(d14 - 5.18) < delta && fabs(d25 - 5.18) < delta && fabs(d13 - 5.45) < delta &&
        fabs(d24 - 5.45) < delta && fabs(d35 - 5.45) < delta)
        return 'H';
    delta = 1.42;
    if (fabs(d15 - 13) < delta && fabs(d14 - 10.4) < delta && fabs(d25 - 10.4) < delta && fabs(d13 - 6.1) < delta &&
        fabs(d24 - 6.1) < delta && fabs(d35 - 6.1) < delta)
        return 'E';
    if (d15 < 8) return 'T';
    return 'C';
}

__device__ void make_sec(const Ctx *C, const double (*x)[3], int len, char *sec) {
    for (int i = C->lane; i < len; i += 32) {
        char c = 'C';
        const int j1 = i - 2, j2 = i - 1, j3 = i, j4 = i + 1, j5 = i + 2;
        if (j1 >= 0 && j5 < len)
            c = sec_str(sqrt(dist2(x[j1], x[j3])), sqrt(dist2(x[j1], x[j4])), sqrt(dist2(x[j1], x[j5])),
                        sqrt(dist2(x[j2], x[j4])), sqrt(dist2(x[j2], x[j5])), sqrt(dist2(x[j3], x[j5])));
        sec[i] = c;
    }
}

/* ---------------------------------------------------------------------------------------------- scoring */
// one pass over the n pairs (xtm[k], ytm[k]) under F: dis[k] = the squared distance, the score term of every pair
// (method 8: 0 for dist > score_d8^2, which leaves the sequential sum's bits as skipping it would), summed in order
__device__ double score_pass(Ctx *C, const Fit *F, int n, int method, double d0) {
    const double d02 = MUL(d0, d0), cut8 = MUL(C->score_d8, C->score_d8);
    SYNC();
    for (int k = C->lane; k < n; k += 32) {
        double xr[3];
        xform(F, C->xtm[k], xr);
        const double di = dist2(xr, C->ytm[k]);
        C->dis[k] = di;
        C->term[k] = method == 8 && !(di <= cut8) ? 0.0 : 1.0 / (1.0 + di / d02);
    }
    SYNC();
    return seqsum(C->term, n);
}

// score_fun8's cut of dis[0..n) at d into i_ali, widened by 0.5 while fewer than 3 pairs and n > 3
__device__ int cut8(Ctx *C, int n, double d) {
    double d_tmp = MUL(d, d);
    int inc = 0;
    for (;;) {
        const double dt = d_tmp;
        int *i_ali = C->i_ali;
        const double *dis = C->dis;
        const int n_cut = compact(C, n, [&](int k) { return dis[k] < dt; }, [&](int pos, int k) { i_ali[pos] = k; });
        if (n_cut < 3 && n > 3) {
            inc++;
            const double dinc = d + MUL((double)inc, 0.5);
            d_tmp = MUL(dinc, dinc);
        } else {
            return n_cut;
        }
    }
}

// TMscore8_search over the n pairs (xtm[k], ytm[k]); `standard` divides by n instead of Lnorm.  F = the fit of the
// best score.  Returns the best score; an empty set scores 0 with the identity.
__device__ double tmscore8_search(Ctx *C, int n, Fit *F, int simplify_step, int method, double local_d0_search,
                                  double Lnorm, double d0, int standard) {
    if (n < 1) {
        identity_fit(F);
        return 0.0;
    }
    const double norm = standard ? (double)n : Lnorm;
    int L_ini[6], n_init = 0;
    const int L_ini_min = n < 4 ? n : 4;
    int i;
    for (i = 0; i < 5; ++i) {
        n_init++;
        L_ini[i] = n >> i;
        if (L_ini[i] <= L_ini_min) {
            L_ini[i] = L_ini_min;
            break;
        }
    }
    if (i == 5) {
        n_init++;
        L_ini[i] = L_ini_min;
    }
    double score_max = -1, score;
    Fit T;
    for (int i_init = 0; i_init < n_init; ++i_init) {
        const int L_frag = L_ini[i_init], iL_max = n - L_frag;
        int s = 0;
        for (;;) {
            fit(C, C->xtm + s, C->ytm + s, L_frag, &T);
            score = score_pass(C, &T, n, method, d0) / norm;
            int n_cut = cut8(C, n, local_d0_search - 1);
            if (score > score_max) {
                score_max = score;
                *F = T;
            }
            for (int it = 0; it < N_EXT && n_cut > 0; ++it) {
                for (int k = C->lane; k < n_cut; k += 32) {
                    const int m = C->i_ali[k];
                    for (int d = 0; d < 3; ++d) {
                        C->r1[k][d] = C->xtm[m][d];
                        C->r2[k][d] = C->ytm[m][d];
                    }
                    C->k_ali[k] = m;
                }
                const int ka = n_cut;
                fit(C, C->r1, C->r2, ka, &T);
                score = score_pass(C, &T, n, method, d0) / norm;
                n_cut = cut8(C, n, local_d0_search + 1);
                if (score > score_max) {
                    score_max = score;
                    *F = T;
                }
                if (n_cut == ka) {
                    bool diff = false;
                    for (int k = C->lane; k < n_cut; k += 32) diff = diff || C->i_ali[k] != C->k_ali[k];
                    if (!__any_sync(FULL, diff)) break;
                }
            }
            if (s < iL_max) {
                s += simplify_step;
                if (s > iL_max) s = iL_max;
            } else {
                break;
            }
        }
    }
    return score_max;
}

// gathers the pairs of map into xtm / ytm; returns their count
__device__ int gather(Ctx *C, const int *map) {
    double(*xtm)[3] = C->xtm, (*ytm)[3] = C->ytm;
    const double(*x)[3] = C->x, (*y)[3] = C->y;
    return compact(C, C->ylen, [&](int j) { return map[j] >= 0; }, [&](int pos, int j) {
        for (int d = 0; d < 3; ++d) {
            xtm[pos][d] = x[map[j]][d];
            ytm[pos][d] = y[j][d];
        }
    });
}

__device__ double detailed_search(Ctx *C, const int *map, Fit *F, int simplify_step, int standard) {
    const int k = gather(C, map);
    return tmscore8_search(C, k, F, simplify_step, 8, C->d0_search, C->Lnorm, C->d0, standard);
}

// the pairs of xtm / ytm with dis <= t into r1 / r2, t widened by 0.5 while fewer than 3 and n > 3
__device__ int cut_fast(Ctx *C, int n, double t) {
    double(*r1)[3] = C->r1, (*r2)[3] = C->r2;
    const double(*xtm)[3] = C->xtm, (*ytm)[3] = C->ytm;
    const double *dis = C->dis;
    for (;;) {
        const double tt = t;
        const int j = compact(C, n, [&](int k) { return dis[k] <= tt; }, [&](int pos, int k) {
            for (int d = 0; d < 3; ++d) {
                r1[pos][d] = xtm[k][d];
                r2[pos][d] = ytm[k][d];
            }
        });
        if (j < 3 && n > 3) t += 0.5;
        else return j;
    }
}

// get_score_fast: three fits, the largest unnormalised score (>=)
__device__ double get_score_fast(Ctx *C, const int *map) {
    const int n = gather(C, map);
    if (n < 1) return 0.0;
    const double d002 = MUL(C->d0_search, C->d0_search);
    Fit F;
    fit(C, C->xtm, C->ytm, n, &F);
    double tm = score_pass(C, &F, n, 0, C->d0), tm1, tm2;
    int j = cut_fast(C, n, d002);
    if (n != j) {
        fit(C, C->r1, C->r2, j, &F);
        tm1 = score_pass(C, &F, n, 0, C->d0);
        j = cut_fast(C, n, d002 + 1);
        fit(C, C->r1, C->r2, j, &F);
        tm2 = score_pass(C, &F, n, 0, C->d0);
    } else {
        tm1 = tm2 = tm;
    }
    if (tm1 >= tm) tm = tm1;
    if (tm2 >= tm) tm = tm2;
    return tm;
}

/* ---------------------------------------------------------------------------------------------- dynamic programming */
enum { DP_TM = 0, DP_SSPLUS = 1, DP_SS = 2 };

// NWDP_TM: mode DP_TM scores 1 / (1 + d^2 / d02) under F; DP_SSPLUS the same plus 0.5 where the codes match; DP_SS 1
// where the codes match.  Cell (i, j) takes the diagonal when d >= h && d >= v, else max(v, h) with v on ties.  The
// cells of one anti-diagonal i + j = D are independent: the lanes share them, three diagonals of values indexed by i.
// Per cell the two decisions (diagonal, v >= h) are kept, from which lane 0 walks the traceback.
__device__ void nwdp(Ctx *C, int mode, const Fit *F, double d02, double gap_open, int *j2i) {
    const int len1 = C->xlen, len2 = C->ylen, W = len2 + 1, lane = C->lane;
    unsigned char *path = C->path;
    double *dm2 = C->val, *dm1 = C->val + (len1 + 1), *cur = C->val + 2 * (len1 + 1);
    SYNC();
    for (int j = lane; j <= len2; j += 32) {
        path[j] = 0;
        if (j < len2) j2i[j] = -1;
    }
    for (int i = lane; i <= len1; i += 32) path[i * W] = 0;
    if (mode != DP_SS)
        for (int i = lane; i < len1; i += 32) xform(F, C->x[i], C->xt[i]);
    SYNC();
    for (int D = 2; D <= len1 + len2; ++D) {
        const int ilo = max(1, D - len2), ihi = min(len1, D - 1);
        for (int i = ilo + lane; i <= ihi; i += 32) {
            const int j = D - i;
            const double diag = i == 1 || j == 1 ? 0.0 : dm2[i - 1];
            double d;
            if (mode == DP_SS) {
                d = C->secx[i - 1] == C->secy[j - 1] ? diag + 1.0 : diag;
            } else {
                double s = 1.0 / (1.0 + dist2(C->xt[i - 1], C->y[j - 1]) / d02);
                if (mode == DP_SSPLUS && C->secx[i - 1] == C->secy[j - 1]) s = s + 0.5;
                d = diag + s;
            }
            double h = i == 1 ? 0.0 : dm1[i - 1];
            if (path[(i - 1) * W + j] & 1) h += gap_open;
            double v = j == 1 ? 0.0 : dm1[i];
            if (path[i * W + j - 1] & 1) v += gap_open;
            const unsigned char vh = v >= h ? 2 : 0;
            unsigned char p;
            if (d >= h && d >= v) {
                p = 1;
                cur[i] = d;
            } else {
                p = 0;
                cur[i] = vh ? v : h;
            }
            path[i * W + j] = p | vh;
        }
        SYNC();
        double *t = dm2;
        dm2 = dm1;
        dm1 = cur;
        cur = t;
    }
    if (lane == 0) {
        int i = len1, j = len2;
        while (i > 0 && j > 0) {
            const unsigned char p = path[i * W + j];
            if (p & 1) {
                j2i[j - 1] = i - 1;
                i--;
                j--;
            } else if (p & 2) {
                j--;
            } else {
                i--;
            }
        }
    }
    SYNC();
}

__device__ void copy_map(const Ctx *C, int *dst, const int *src) {
    SYNC();
    for (int j = C->lane; j < C->ylen; j += 32) dst[j] = src[j];
    SYNC();
}

// DP_iter: F in = the transform of the last search, out = the last search's
__device__ double dp_iter(Ctx *C, Fit *F, int *map0, int g1, int g2, int iteration_max) {
    const double gap_open[2] = {-0.6, 0};
    int *map = C->tmpmap;
    const double d02 = MUL(C->d0, C->d0);
    double tm_max = -1, tm_old = 0;
    for (int g = g1; g < g2; ++g)
        for (int it = 0; it < iteration_max; ++it) {
            nwdp(C, DP_TM, F, d02, gap_open[g], map);
            const double tm = detailed_search(C, map, F, 40, 0);
            if (tm > tm_max) {
                tm_max = tm;
                copy_map(C, map0, map);
            }
            if (it > 0 && fabs(tm_old - tm) < 0.000001) break;
            tm_old = tm;
        }
    return tm_max;
}

/* ---------------------------------------------------------------------------------------------- initial alignments */
__device__ void thread_map(const Ctx *C, int *map, int k) {
    SYNC();
    for (int j = C->lane; j < C->ylen; j += 32) {
        const int i = j + k;
        map[j] = i >= 0 && i < C->xlen ? i : -1;
    }
    SYNC();
}

__device__ void get_initial(Ctx *C, int *y2x) {
    const int xlen = C->xlen, ylen = C->ylen, min_len = xlen < ylen ? xlen : ylen;
    int min_ali = min_len / 2;
    if (min_ali <= 5) min_ali = 5;
    const int n1 = -ylen + min_ali, n2 = xlen - min_ali;
    double tm_max = -1;
    int k_best = n1;
    for (int k = n1; k <= n2; ++k) {
        thread_map(C, y2x, k);
        const double tm = get_score_fast(C, y2x);
        if (tm >= tm_max) {
            tm_max = tm;
            k_best = k;
        }
    }
    thread_map(C, y2x, k_best);
}

__device__ int get_initial5(Ctx *C, int *y2x) {
    const int xlen = C->xlen, ylen = C->ylen, aL = xlen < ylen ? xlen : ylen;
    double d01 = C->d0 + 1.5;
    if (d01 < C->D0_MIN) d01 = C->D0_MIN;
    const double d02 = MUL(d01, d01);
    double GLmax = 0;
    int *map = C->tmpmap, flag = 0;
    int n_jump1 = xlen > 250 ? 45 : xlen > 200 ? 35 : xlen > 150 ? 25 : 15;
    if (n_jump1 > xlen / 3) n_jump1 = xlen / 3;
    int n_jump2 = ylen > 250 ? 45 : ylen > 200 ? 35 : ylen > 150 ? 25 : 15;
    if (n_jump2 > ylen / 3) n_jump2 = ylen / 3;
    int n_frag[2] = {20, 100};
    if (n_frag[0] > aL / 3) n_frag[0] = aL / 3;
    if (n_frag[1] > aL / 2) n_frag[1] = aL / 2;
    Fit F;
    for (int f = 0; f < 2; ++f) {
        const int m1 = xlen - n_frag[f] + 1, m2 = ylen - n_frag[f] + 1;
        for (int i = 0; i < m1; i += n_jump1)
            for (int j = 0; j < m2; j += n_jump2) {
                fit(C, C->x + i, C->y + j, n_frag[f], &F);
                nwdp(C, DP_TM, &F, d02, 0.0, map);
                const double GL = get_score_fast(C, map);
                if (GL > GLmax) {
                    GLmax = GL;
                    copy_map(C, y2x, map);
                    flag = 1;
                }
            }
    }
    return flag;
}

__device__ void get_initial_ssplus(Ctx *C, const int *y2x0, int *y2x) {
    double d01 = C->d0 + 1.5;
    if (d01 < C->D0_MIN) d01 = C->D0_MIN;
    const int k = gather(C, y2x0);
    Fit F;
    fit(C, C->xtm, C->ytm, k, &F);
    nwdp(C, DP_SSPLUS, &F, MUL(d01, d01), -1.0, y2x);
}

/* the longest run of consecutive residues closer than the cutoff, grown by 1.1 per step (a running product) until the
 * run has at least min(4, floor(len / 3)) residues */
__device__ void find_max_frag(const double (*x)[3], int len, int *start_max, int *end_max, double dcu0) {
    int r_min = (int)(MUL((double)len, 1.0) / 3.0);
    if (r_min > 4) r_min = 4;
    int Lfr_max = 0;
    double grow = 1.0, dcu_cut = MUL(dcu0, dcu0);
    while (Lfr_max < r_min) {
        Lfr_max = 0;
        int j = 1, start = 0;
        for (int i = 1; i < len; ++i) {
            if (dist2(x[i - 1], x[i]) < dcu_cut) {
                j++;
                if (i == len - 1) {
                    if (j > Lfr_max) {
                        Lfr_max = j;
                        *start_max = start;
                        *end_max = i;
                    }
                    j = 1;
                }
            } else {
                if (j > Lfr_max) {
                    Lfr_max = j;
                    *start_max = start;
                    *end_max = i - 1;
                }
                j = 1;
                start = i;
            }
        }
        if (Lfr_max < r_min) {
            grow = MUL(grow, 1.1);
            const double dinc = MUL(grow, dcu0);
            dcu_cut = MUL(dinc, dinc);
        }
    }
}

__device__ void get_initial_fgt(Ctx *C, int *y2x, double dcu0) {
    const int xlen = C->xlen, ylen = C->ylen;
    int xstart = 0, ystart = 0, xend = 0, yend = 0;
    find_max_frag(C->x, xlen, &xstart, &xend, dcu0);
    find_max_frag(C->y, ylen, &ystart, &yend, dcu0);
    const int Lx = xend - xstart + 1, Ly = yend - ystart + 1;
    int L_fr = Lx < Ly ? Lx : Ly;
    int *ifr = C->ifr, *map = C->tmpmap;
    const int use_x = Lx < Ly || (Lx == Ly && xlen <= ylen);
    const int L0 = xlen < ylen ? xlen : ylen;
    const int n1t = (int)MUL((double)L0, 0.1), n2t = (int)MUL((double)L0, 0.89);
    SYNC();
    if (C->lane == 0) {
        for (int i = 0; i < L_fr; ++i) ifr[i] = (use_x ? xstart : ystart) + i;
        if (L_fr == L0) {
            int j = 0;
            for (int i = n1t; i <= n2t; ++i) ifr[j++] = ifr[i];
        }
    }
    if (L_fr == L0) L_fr = n2t >= n1t ? n2t - n1t + 1 : 0;
    SYNC();
    double tm_max = -1;
    const int other = use_x ? ylen : xlen, min_len = L_fr < other ? L_fr : other;
    int min_ali = (int)((double)min_len / 2.5);
    if (min_ali <= 3) min_ali = 3;
    const int n1 = -(use_x ? ylen : L_fr) + min_ali, n2 = (use_x ? L_fr : xlen) - min_ali;
    for (int k = n1; k <= n2; ++k) {
        SYNC();
        if (use_x) {
            for (int j = C->lane; j < ylen; j += 32) {
                const int i = j + k;
                map[j] = i >= 0 && i < L_fr ? ifr[i] : -1;
            }
        } else {
            for (int j = C->lane; j < ylen; j += 32) map[j] = -1;
            SYNC();
            for (int j = C->lane; j < L_fr; j += 32) {
                const int i = j + k;
                if (i >= 0 && i < xlen) map[ifr[j]] = i;
            }
        }
        SYNC();
        const double tm = get_score_fast(C, map);
        if (tm >= tm_max) {
            tm_max = tm;
            copy_map(C, y2x, map);
        }
    }
}

__device__ void record_of(const Fit *F, double *rec) {
    for (int k = 0; k < 9; ++k) rec[k] = F->R[k];
    for (int k = 0; k < 3; ++k) {
        rec[9 + k] = F->p[k];
        rec[12 + k] = F->q[k];
    }
    rec[15] = 0.0;
}

struct Args {
    const float *coords;
    long long fs;
    const float *ref;
    long long rfs;
    const unsigned *sel, *refsel;
    int xlen, ylen, ref_per_frame;
    double params[10];
    const unsigned *frames;
    long long item0, n;  // items [item0, item0 + n) of this launch
    char *scratch;
    size_t item_bytes;
    double *tm, *rmsd, *rec;
    int *nali, *invmap;
};

// per-item scratch, carved in this order; every piece starts 16-byte aligned
__host__ __device__ inline size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }
__host__ __device__ inline size_t item_bytes(int xlen, int ylen) {
    const size_t n = (size_t)(xlen > ylen ? xlen : ylen);
    return al16(24 * (size_t)xlen) + al16(24 * (size_t)ylen) + 5 * al16(24 * n) + al16(8 * n) +
           al16(24 * (size_t)(xlen + 1)) + al16(8 * n) + 3 * al16(4 * n) + 3 * al16(4 * (size_t)ylen) + al16(xlen) + al16(ylen) +
           al16((size_t)(xlen + 1) * (size_t)(ylen + 1));
}

__global__ void __launch_bounds__(TA_THREADS) tmalign_kernel(const Args A) {
    const long long local = (long long)blockIdx.x * TA_WARPS + (threadIdx.x >> 5);
    if (local >= A.n) return;  // the whole warp
    const int lane = threadIdx.x & 31;
    const long long item = A.item0 + local;
    const long long f = A.frames ? (long long)A.frames[item] : item;
    const int xlen = A.xlen, ylen = A.ylen, n = max(xlen, ylen);
    char *s = A.scratch + (size_t)local * A.item_bytes;
    auto take = [&](size_t b) {
        char *p = s;
        s += al16(b);
        return p;
    };
    Ctx C;
    C.lane = lane;
    C.xlen = xlen;
    C.ylen = ylen;
    double(*xa)[3] = reinterpret_cast<double(*)[3]>(take(24 * (size_t)xlen));
    double(*ya)[3] = reinterpret_cast<double(*)[3]>(take(24 * (size_t)ylen));
    C.xt = reinterpret_cast<double(*)[3]>(take(24 * (size_t)n));
    C.xtm = reinterpret_cast<double(*)[3]>(take(24 * (size_t)n));
    C.ytm = reinterpret_cast<double(*)[3]>(take(24 * (size_t)n));
    C.r1 = reinterpret_cast<double(*)[3]>(take(24 * (size_t)n));
    C.r2 = reinterpret_cast<double(*)[3]>(take(24 * (size_t)n));
    C.dis = reinterpret_cast<double *>(take(8 * (size_t)n));
    C.val = reinterpret_cast<double *>(take(24 * (size_t)(xlen + 1)));
    C.term = reinterpret_cast<double *>(take(8 * (size_t)n));
    C.i_ali = reinterpret_cast<int *>(take(4 * (size_t)n));
    C.k_ali = reinterpret_cast<int *>(take(4 * (size_t)n));
    C.ifr = reinterpret_cast<int *>(take(4 * (size_t)n));
    C.tmpmap = reinterpret_cast<int *>(take(4 * (size_t)ylen));
    int *map = reinterpret_cast<int *>(take(4 * (size_t)ylen));
    int *map0 = reinterpret_cast<int *>(take(4 * (size_t)ylen));
    C.secx = take(xlen);
    C.secy = take(ylen);
    C.path = reinterpret_cast<unsigned char *>(take((size_t)(xlen + 1) * (size_t)(ylen + 1)));
    C.x = xa;
    C.y = ya;

    double *tm = A.tm + 2 * item, *rec = A.rec + 16 * item;
    int *invmap = A.invmap + (size_t)item * ylen;
    Fit F;
    identity_fit(&F);
    for (int j = lane; j < ylen; j += 32) invmap[j] = -1;
    if (lane == 0) {
        record_of(&F, rec);
        A.nali[item] = 0;
    }
    const long long rf = A.ref_per_frame ? f : 0;
    bool bad = false;
    for (int i = lane; i < xlen; i += 32) {
        const float *p = A.coords + (long long)A.sel[i] * 3 * A.fs + f;
        for (int d = 0; d < 3; ++d) {
            xa[i][d] = p[d * A.fs];
            bad = bad || !isfinite(p[d * A.fs]);
        }
    }
    for (int j = lane; j < ylen; j += 32) {
        const float *p = A.ref + (long long)A.refsel[j] * 3 * A.rfs + rf;
        for (int d = 0; d < 3; ++d) {
            ya[j][d] = p[d * A.rfs];
            bad = bad || !isfinite(p[d * A.rfs]);
        }
    }
    if (__any_sync(FULL, bad)) {
        if (lane == 0) tm[0] = tm[1] = A.rmsd[item] = NAN;
        return;
    }
    SYNC();
    const double *params = A.params;
    C.d0 = params[0];
    C.d0_search = params[1];
    C.score_d8 = params[2];
    C.D0_MIN = params[3];
    C.Lnorm = (double)(xlen < ylen ? xlen : ylen);
    const double ddcc = params[4], dcu0 = params[5];

    make_sec(&C, C.x, xlen, C.secx);
    make_sec(&C, C.y, ylen, C.secy);
    double TMmax = -1, TM;
#define KEEP()                                                 \
    if (TM > TMmax) {                                          \
        TMmax = TM;                                            \
        copy_map(&C, map0, map);                               \
    }
    // 1: gapless threading
    get_initial(&C, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    TM = dp_iter(&C, &F, map, 0, 2, 30);
    KEEP();
    // 2: secondary structure
    nwdp(&C, DP_SS, &F, 1.0, -1.0, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, 0.2)) {
        TM = dp_iter(&C, &F, map, 0, 2, 30);
        KEEP();
    }
    // 3: local superposition
    if (get_initial5(&C, map)) {
        TM = detailed_search(&C, map, &F, 40, 0);
        KEEP();
        if (TM > MUL(TMmax, ddcc)) {
            TM = dp_iter(&C, &F, map, 0, 2, 2);
            KEEP();
        }
    }
    // 4: secondary structure plus the best map so far
    get_initial_ssplus(&C, map0, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, ddcc)) {
        TM = dp_iter(&C, &F, map, 0, 2, 30);
        KEEP();
    }
    // 5: fragment gapless threading
    get_initial_fgt(&C, map, dcu0);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, ddcc)) {
        TM = dp_iter(&C, &F, map, 1, 2, 2);
        KEEP();
    }
#undef KEEP
    // final: the standard search on the best map, the pairs within score_d8 under it, their rmsd and both scores
    detailed_search(&C, map0, &F, 1, 1);
    const double(*x)[3] = C.x, (*y)[3] = C.y;
    double(*xtm)[3] = C.xtm, (*ytm)[3] = C.ytm;
    const double score_d8 = C.score_d8;
    const int k = compact(&C, ylen, [&](int j) {
        const int i = map0[j];
        if (i < 0) return false;
        double xr[3];
        xform(&F, x[i], xr);
        return sqrt(dist2(xr, y[j])) <= score_d8;
    }, [&](int pos, int j) {
        for (int d = 0; d < 3; ++d) {
            xtm[pos][d] = x[map0[j]][d];
            ytm[pos][d] = y[j][d];
        }
        invmap[j] = map0[j];
    });
    if (lane == 0) A.nali[item] = k;
    if (k == 0) {
        if (lane == 0) tm[0] = tm[1] = A.rmsd[item] = 0.0;
        return;
    }
    fit(&C, C.xtm, C.ytm, k, &F);
    score_pass(&C, &F, k, 0, 1.0);  // for dis[], the squared distances under the fit
    const double sq = seqsum(C.dis, k);
    if (lane == 0) A.rmsd[item] = sqrt(sq / (double)k);
    C.d0 = params[6];
    C.d0_search = params[7];
    const double tm_ref = tmscore8_search(&C, k, &F, 1, 0, C.d0_search, (double)ylen, C.d0, 0);
    Fit G;
    C.d0 = params[8];
    C.d0_search = params[9];
    const double tm_mol = tmscore8_search(&C, k, &G, 1, 0, C.d0_search, (double)xlen, C.d0, 0);
    if (lane == 0) {
        tm[0] = tm_ref;
        tm[1] = tm_mol;
        record_of(&F, rec);
    }
}

}  // namespace tma
}  // namespace mkb

using namespace mkb;
using namespace mkb::tma;

extern "C" int64_t mkb_tmalign_max_residues(void) { return TA_MAX_RES; }

extern "C" int64_t mkb_tmalign_chunk_frames(int64_t xlen, int64_t ylen) {
    if (xlen < 1 || ylen < 1 || xlen > TA_MAX_RES || ylen > TA_MAX_RES) return 0;
    const size_t b = item_bytes((int)xlen, (int)ylen);
    return (int64_t)std::max<size_t>(TA_WARPS, TA_SCRATCH_BUDGET / b / TA_WARPS * TA_WARPS);
}

extern "C" int mkb_tmalign(mkb_handle_t h, void *stream, const mkb_traj *t, const uint32_t *sel, int64_t xlen,
                           const mkb_traj *ref, const uint32_t *refsel, int64_t ylen, int32_t ref_per_frame,
                           const double *params, const uint32_t *frames, int64_t n_frames, double *tm, double *rmsd,
                           int32_t *nali, int32_t *invmap, double *records) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!t || !ref || !params) return fail(h, MKB_ERR_BAD_ARG, "null trajectory / params");
    if (xlen < 5 || ylen < 5) return fail(h, MKB_ERR_BAD_ARG, "TM-align needs >= 5 residues each side");
    if (xlen > TA_MAX_RES || ylen > TA_MAX_RES)
        return fail(h, MKB_ERR_BAD_ARG, "residue counts %lld, %lld over %d", (long long)xlen, (long long)ylen,
                    TA_MAX_RES);
    for (int k = 0; k < 10; ++k)
        if (!std::isfinite(params[k])) return fail(h, MKB_ERR_BAD_ARG, "non-finite parameter %d", k);
    if (t->n_frames < 0 || ref->n_frames < 1 || (frames && n_frames < 0))
        return fail(h, MKB_ERR_BAD_ARG, "bad frame counts");
    if (!t->coords || !ref->coords || !sel || !refsel) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (t->frame_stride < t->n_frames || ref->frame_stride < ref->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (ref_per_frame && ref->n_frames < t->n_frames)
        return fail(h, MKB_ERR_BAD_ARG, "a reference frame per frame needs ref n_frames >= t n_frames");
    Args A;
    A.coords = t->coords; A.fs = t->frame_stride;
    A.ref = ref->coords; A.rfs = ref->frame_stride;
    A.sel = sel; A.refsel = refsel;
    A.xlen = (int)xlen; A.ylen = (int)ylen; A.ref_per_frame = ref_per_frame ? 1 : 0;
    for (int k = 0; k < 10; ++k) A.params[k] = params[k];
    A.frames = frames;
    const long long total = frames ? n_frames : t->n_frames;
    if (total == 0) return MKB_OK;
    if (!tm || !rmsd || !nali || !invmap || !records) return fail(h, MKB_ERR_BAD_ARG, "null output");
    A.tm = tm; A.rmsd = rmsd; A.nali = nali; A.invmap = invmap; A.rec = records;
    A.item_bytes = item_bytes(A.xlen, A.ylen);
    const long long chunk = std::min<long long>(total, mkb_tmalign_chunk_frames(xlen, ylen));
    int rc;
    if ((rc = scratch_get(h, S_TMALIGN, (size_t)chunk * A.item_bytes, (void **)&A.scratch))) return rc;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    for (long long i0 = 0; i0 < total; i0 += chunk) {
        A.item0 = i0;
        A.n = std::min(chunk, total - i0);
        tmalign_kernel<<<(unsigned)cdiv(A.n, TA_WARPS), TA_THREADS, 0, st>>>(A);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    h->last_kernel = "tmalign_kernel";
    return MKB_OK;
}
