/* tmalign_oracle.c -- plain-C restatement of TM-align (Zhang & Skolnick, Nucleic Acids Res. 2005), in the shape of the
 * C++ release's TMalign_main, for the K27 parity tests.  TEST INFRASTRUCTURE ONLY: the package never loads it.
 *
 * The contract is also the mkb_tmalign comment of include/mkb200.h.  Compiled with -O3 -ffp-contract=off: every float64
 * operation is rounded on its own, in the order written here; MUL marks each product (the kernel's __dmul_rn).  Every
 * sum runs sequentially in pair order.  This restatement keeps the program's whole DP value matrix and its traceback,
 * which recomputes h and v from the stored values; the kernel keeps three diagonals and two decision bits per cell.
 *
 * Input per item: x [xlen][3] (the mol CA trace) and y [ylen][3] (the reference), float32 Angstrom, widened to
 * float64.  Output: tm[0] = TM_ref (normalised by ylen), tm[1] = TM_mol (by xlen), rmsd, nali, invmap [ylen] (the x
 * residue aligned to y residue j among the nali final pairs, or -1), record [16] (R row-major, p, q, pad:
 * x' = R (x - p) + q), and the counts of DP cells, fits and pair evaluations.  dist is the SQUARED distance.
 *
 * The choices, in program order:
 *   parameters  passed in (tmalign_parameters, host C pow): Lnorm = min(xlen, ylen); d0 = 0.168 (Lnorm <= 19) or
 *               1.24 (Lnorm - 15)^(1/3) - 1.8, then D0_MIN = d0 + 0.8 and d0 = D0_MIN; d0_search = d0 clamped to
 *               [4.5, 8]; score_d8 = 1.5 Lnorm^0.3 + 3.5; dcu0 = 4.25; ddcc = 0.4, or 0.1 when Lnorm <= 40; the final
 *               d0 for length L is 0.5 (L <= 21) or the formula floored at 0.5, d0_search clamped likewise.
 *   fit         K19's: two-pass centroids and H, Horn's quaternion through the cyclic Jacobi (at most 50 sweeps);
 *               x' = ((R0 a0 + R1 a1) + R2 a2) + q per row, a = x - p.  An empty set fits the identity.
 *   sec         the 2019 release's protein rule without smoothing: H within 2.1 of (6.37, 5.18, 5.18, 5.45, 5.45,
 *               5.45) for (d15, d14, d25, d13, d24, d35), else E within 1.42 of (13, 10.4, 10.4, 6.1, 6.1, 6.1), else
 *               T when d15 < 8, else C; C without both neighbours i - 2, i + 2.
 *   score_fun8  cut at dist < (d + 0.5 inc)^2, inc grown while fewer than 3 pairs and n > 3; method 8 sums only the
 *               pairs with dist <= score_d8^2, method 0 all; / Lnorm (the standard form: / n).
 *   search      TMscore8_search: fragment lengths n >> i down to min(4, n), at most 6; starts every simplify_step and
 *               always the last; seed fit, cut at d0_search - 1, up to 20 refits cut at d0_search + 1, stopping on an
 *               empty or repeated cut set; the best (strict >) score and its fit.  An empty pair set scores 0.
 *   get_score_fast  three fits: all pairs, dist <= d0_search^2, dist <= d0_search^2 + 1, each threshold + 0.5 while
 *               fewer than 3 pairs and n > 3; the third only when the second set is not all pairs; the largest (>=).
 *   NWDP_TM     the rotated TM term, the score matrix term (1 / (1 + dist / d01^2), + 0.5 where the codes match) or
 *               the code match (1); the diagonal when d >= h && d >= v, else v when v >= h, else h; the gap applies
 *               when the neighbour took its diagonal; the same rule walks the traceback.
 *   DP_iter     gap opens {-0.6, 0}; per iteration DP under the last fit, detailed_search (simplify_step 40,
 *               method 8); stop when |TM_old - TM| < 1e-6, TM_old carried across the gap opens.
 *   initial     1 gapless threading (min_ali = max(5, min_len / 2), the last of equal scores), DP_iter(0, 2, 30);
 *               2 code DP with gap -1, DP_iter(0, 2, 30) if TM > 0.2 TMmax; 3 get_initial5 (fragments {20, 100}
 *               capped at aL / 3, aL / 2; jumps 45 / 35 / 25 / 15 over 250 / 200 / 150 / else, capped at len / 3;
 *               DP with gap 0 and d01 = max(d0 + 1.5, D0_MIN); the first maximum), DP_iter(0, 2, 2) if TM > ddcc
 *               TMmax; 4 get_initial_ssplus under the best map's fit, gap -1, DP_iter(0, 2, 30) if TM > ddcc TMmax;
 *               5 get_initial_fgt with find_max_frag (cutoff dcu0 times a running product of 1.1, minimum fragment
 *               4; x fragment when Lx < Ly or Lx == Ly and xlen <= ylen; trimmed to [0.1 L0, 0.89 L0] when it spans
 *               L0; min_ali = max(3, min_len / 2.5); the last of equal scores), DP_iter(1, 2, 2) if TM > ddcc TMmax.
 *               Each map goes through detailed_search (40, method 8) first; TMmax and the best map update on >.
 *   final       detailed_search_standard (simplify_step 1, method 8) on the best map; the aligned pairs with
 *               sqrt(dist) <= score_d8 under its fit are the nali pairs; rmsd = sqrt(sum dist / nali) under their
 *               fit; TM_ref and TM_mol = TMscore8_search (1, method 0) over them with the final d0 for ylen and
 *               xlen; the record is TM_ref's best fit.  nali = 0 gives scores and rmsd 0.
 *   rejected    a non-finite x coordinate: NaN scores and rmsd, nali 0, invmap -1, identity record (the caller
 *               rejects a non-finite reference and fewer than 5 residues).
 *
 * Not confirmed against TMalign.cpp or moleculekit (neither source is at hand): the fit (the program has its own
 * Kabsch routine), the running product in place of pow(1.1, inc), the 2019 release's extra tie search for Lx == Ly and
 * xlen == ylen (left out here), the final search's simplify_step, the score_d8 filter on the reported map, and every
 * constant above that was taken from the published description rather than the source. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MUL(a, b) ((a) * (b))
#define N_EXT 20 /* refits per search seed */

typedef struct {
    double R[9], p[3], q[3];
} Fit;

typedef struct {
    int xlen, ylen;
    const double (*x)[3], (*y)[3];
    char *secx, *secy;
    double d0, d0_search, score_d8, D0_MIN, Lnorm;
    /* scratch */
    double (*xt)[3], (*xtm)[3], (*ytm)[3], (*r1)[3], (*r2)[3], *dis;
    int *i_ali, *k_ali, *ifr, *tmpmap;
    double *val;           /* (xlen + 1) x (ylen + 1) */
    unsigned char *path;   /* (xlen + 1) x (ylen + 1) */
    int64_t *counts;       /* DP cells, fits, pair evaluations */
} Ctx;

static void jacobi_rot(double a[4][4], double v[4][4], int P, int Q, int late) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double g = MUL(100.0, fabs(apq));
    if (late && fabs(a[P][P]) + g == fabs(a[P][P]) && fabs(a[Q][Q]) + g == fabs(a[Q][Q])) {
        a[P][Q] = a[Q][P] = 0.0;
        return;
    }
    const double h = a[Q][Q] - a[P][P];
    double t;
    if (fabs(h) + g == fabs(h)) {
        t = apq / h;
    } else {
        const double th = MUL(0.5, h) / apq;
        t = 1.0 / (fabs(th) + sqrt(1.0 + MUL(th, th)));
        if (th < 0.0) t = -t;
    }
    const double c = 1.0 / sqrt(1.0 + MUL(t, t)), s = MUL(t, c), tau = s / (1.0 + c);
    a[P][P] -= MUL(t, apq);
    a[Q][Q] += MUL(t, apq);
    a[P][Q] = a[Q][P] = 0.0;
    for (int r = 0; r < 4; ++r) {
        if (r == P || r == Q) continue;
        const double arp = a[r][P], arq = a[r][Q];
        a[r][P] = a[P][r] = arp - MUL(s, arq + MUL(arp, tau));
        a[r][Q] = a[Q][r] = arq + MUL(s, arp - MUL(arq, tau));
    }
    for (int r = 0; r < 4; ++r) {
        const double vrp = v[r][P], vrq = v[r][Q];
        v[r][P] = vrp - MUL(s, vrq + MUL(vrp, tau));
        v[r][Q] = vrq + MUL(s, vrp - MUL(vrq, tau));
    }
}

/* K19's Horn quaternion: the proper rotation R (row-major, y ~ R x) for H[a][b] = sum x_a y_b */
static void horn_rotation(const double H[9], double R[9]) {
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
        const int late = sweep > 3;
        jacobi_rot(a, v, 0, 1, late);
        jacobi_rot(a, v, 0, 2, late);
        jacobi_rot(a, v, 0, 3, late);
        jacobi_rot(a, v, 1, 2, late);
        jacobi_rot(a, v, 1, 3, late);
        jacobi_rot(a, v, 2, 3, late);
    }
    double q[4] = {v[0][0], v[1][0], v[2][0], v[3][0]}, best = a[0][0];
    for (int j = 1; j < 4; ++j)
        if (a[j][j] > best) {
            best = a[j][j];
            for (int r = 0; r < 4; ++r) q[r] = v[r][j];
        }
    const double inv = 1.0 / sqrt(MUL(q[0], q[0]) + MUL(q[1], q[1]) + MUL(q[2], q[2]) + MUL(q[3], q[3]));
    const double q0 = MUL(q[0], inv), q1 = MUL(q[1], inv), q2 = MUL(q[2], inv), q3 = MUL(q[3], inv);
    const double q00 = MUL(q0, q0), q11 = MUL(q1, q1), q22 = MUL(q2, q2), q33 = MUL(q3, q3);
    R[0] = q00 + q11 - q22 - q33;
    R[1] = MUL(2.0, MUL(q1, q2) - MUL(q0, q3));
    R[2] = MUL(2.0, MUL(q1, q3) + MUL(q0, q2));
    R[3] = MUL(2.0, MUL(q1, q2) + MUL(q0, q3));
    R[4] = q00 - q11 + q22 - q33;
    R[5] = MUL(2.0, MUL(q2, q3) - MUL(q0, q1));
    R[6] = MUL(2.0, MUL(q1, q3) - MUL(q0, q2));
    R[7] = MUL(2.0, MUL(q2, q3) + MUL(q0, q1));
    R[8] = q00 - q11 - q22 + q33;
}

static void identity_fit(Fit *F) {
    memset(F, 0, sizeof(*F));
    F->R[0] = F->R[4] = F->R[8] = 1.0;
}

/* K19's fit of the pairs (a[k], b[k]), k < n: centroids, then H about them in a second pass.  n = 0: identity. */
static void fit(Ctx *C, const double (*a)[3], const double (*b)[3], int n, Fit *F) {
    C->counts[1]++;
    if (n < 1) {
        identity_fit(F);
        return;
    }
    double sx[3] = {0, 0, 0}, sy[3] = {0, 0, 0}, H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < n; ++k)
        for (int d = 0; d < 3; ++d) {
            sx[d] += a[k][d];
            sy[d] += b[k][d];
        }
    for (int d = 0; d < 3; ++d) {
        F->p[d] = sx[d] / (double)n;
        F->q[d] = sy[d] / (double)n;
    }
    for (int k = 0; k < n; ++k) {
        double u[3], v[3];
        for (int d = 0; d < 3; ++d) {
            u[d] = a[k][d] - F->p[d];
            v[d] = b[k][d] - F->q[d];
        }
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 3; ++s) H[3 * r + s] += MUL(u[r], v[s]);
    }
    horn_rotation(H, F->R);
}

static void xform(const Fit *F, const double a[3], double o[3]) {
    const double b0 = a[0] - F->p[0], b1 = a[1] - F->p[1], b2 = a[2] - F->p[2];
    for (int d = 0; d < 3; ++d) o[d] = MUL(F->R[3 * d], b0) + MUL(F->R[3 * d + 1], b1) + MUL(F->R[3 * d + 2], b2) + F->q[d];
}

static double dist2(const double a[3], const double b[3]) {
    const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return MUL(dx, dx) + MUL(dy, dy) + MUL(dz, dz);
}

/* ---------------------------------------------------------------------------------------------- parameters */
/* computed on the host (tmalign_parameters in moleculekit_b200/tmalign.py) and passed in */

/* ---------------------------------------------------------------------------------------------- secondary structure */
static char sec_str(double d13, double d14, double d15, double d24, double d25, double d35) {
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

static void make_sec(const double (*x)[3], int len, char *sec) {
    for (int i = 0; i < len; ++i) {
        sec[i] = 'C';
        const int j1 = i - 2, j2 = i - 1, j3 = i, j4 = i + 1, j5 = i + 2;
        if (j1 >= 0 && j5 < len)
            sec[i] = sec_str(sqrt(dist2(x[j1], x[j3])), sqrt(dist2(x[j1], x[j4])), sqrt(dist2(x[j1], x[j5])),
                             sqrt(dist2(x[j2], x[j4])), sqrt(dist2(x[j2], x[j5])), sqrt(dist2(x[j3], x[j5])));
    }
}

/* ---------------------------------------------------------------------------------------------- scoring */
/* the cut set of the n pairs (xa = transformed x, ya) at d, widened by 0.5 while fewer than 3 pairs and n > 3, into
 * i_ali; *score = the sum (method 8: pairs with d^2 <= score_d8^2; method 0: all) over norm.  Returns the cut size. */
static int score_fun8(Ctx *C, const double (*xa)[3], const double (*ya)[3], int n, double d, int *i_ali, double *score,
                      int method, double norm, double d0) {
    const double d02 = MUL(d0, d0), score_d8_cut = MUL(C->score_d8, C->score_d8);
    double d_tmp = MUL(d, d);
    int inc = 0, n_cut;
    for (;;) {
        n_cut = 0;
        double sum = 0;
        C->counts[2] += n;
        for (int i = 0; i < n; ++i) {
            const double di = dist2(xa[i], ya[i]);
            if (di < d_tmp) i_ali[n_cut++] = i;
            if (method == 8) {
                if (di <= score_d8_cut) sum += 1.0 / (1.0 + di / d02);
            } else {
                sum += 1.0 / (1.0 + di / d02);
            }
        }
        if (n_cut < 3 && n > 3) {
            inc++;
            const double dinc = d + MUL((double)inc, 0.5);
            d_tmp = MUL(dinc, dinc);
        } else {
            *score = sum / norm;
            return n_cut;
        }
    }
}

/* TMscore8_search over the n pairs (xtm[k], ytm[k]); `standard` divides by n instead of Lnorm.  F = the fit of the
 * best score.  Returns the best score; an empty set scores 0 with the identity. */
static double tmscore8_search(Ctx *C, int n, Fit *F, int simplify_step, int method, double local_d0_search,
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
            for (int k = 0; k < n; ++k) xform(&T, C->xtm[k], C->xt[k]);
            int n_cut = score_fun8(C, C->xt, C->ytm, n, local_d0_search - 1, C->i_ali, &score, method, norm, d0);
            if (score > score_max) {
                score_max = score;
                *F = T;
            }
            for (int it = 0; it < N_EXT && n_cut > 0; ++it) {
                for (int k = 0; k < n_cut; ++k) {
                    const int m = C->i_ali[k];
                    memcpy(C->r1[k], C->xtm[m], sizeof(double) * 3);
                    memcpy(C->r2[k], C->ytm[m], sizeof(double) * 3);
                    C->k_ali[k] = m;
                }
                const int ka = n_cut;
                fit(C, C->r1, C->r2, ka, &T);
                for (int k = 0; k < n; ++k) xform(&T, C->xtm[k], C->xt[k]);
                n_cut = score_fun8(C, C->xt, C->ytm, n, local_d0_search + 1, C->i_ali, &score, method, norm, d0);
                if (score > score_max) {
                    score_max = score;
                    *F = T;
                }
                if (n_cut == ka) {
                    int neq = 0;
                    for (int k = 0; k < n_cut; ++k) neq += C->i_ali[k] == C->k_ali[k];
                    if (neq == n_cut) break;
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

/* gathers the pairs of map into xtm / ytm; returns their count */
static int gather(Ctx *C, const int *map) {
    int k = 0;
    for (int j = 0; j < C->ylen; ++j)
        if (map[j] >= 0) {
            memcpy(C->xtm[k], C->x[map[j]], sizeof(double) * 3);
            memcpy(C->ytm[k], C->y[j], sizeof(double) * 3);
            k++;
        }
    return k;
}

static double detailed_search(Ctx *C, const int *map, Fit *F, int simplify_step, int standard) {
    const int k = gather(C, map);
    return tmscore8_search(C, k, F, simplify_step, 8, C->d0_search, C->Lnorm, C->d0, standard);
}

/* three fits: all pairs of map, then the pairs with d^2 <= d0_search^2, then d^2 <= d0_search^2 + 1, each threshold
 * widened by 0.5 while fewer than 3 pairs and more than 3 aligned.  The largest unnormalised score, >= for later. */
static double get_score_fast(Ctx *C, const int *map) {
    const int n = gather(C, map);
    if (n < 1) return 0.0;
    const double d002 = MUL(C->d0_search, C->d0_search), d02 = MUL(C->d0, C->d0);
    Fit F;
    double xr[3];
    fit(C, C->xtm, C->ytm, n, &F);
    double tm = 0, tm1, tm2;
    C->counts[2] += n;
    for (int k = 0; k < n; ++k) {
        xform(&F, C->xtm[k], xr);
        C->dis[k] = dist2(xr, C->ytm[k]);
        tm += 1.0 / (1.0 + C->dis[k] / d02);
    }
    double d002t = d002;
    int j;
    for (;;) {
        j = 0;
        for (int k = 0; k < n; ++k)
            if (C->dis[k] <= d002t) {
                memcpy(C->r1[j], C->xtm[k], sizeof(double) * 3);
                memcpy(C->r2[j], C->ytm[k], sizeof(double) * 3);
                j++;
            }
        if (j < 3 && n > 3) d002t += 0.5;
        else break;
    }
    if (n != j) {
        fit(C, C->r1, C->r2, j, &F);
        tm1 = 0;
        C->counts[2] += n;
        for (int k = 0; k < n; ++k) {
            xform(&F, C->xtm[k], xr);
            C->dis[k] = dist2(xr, C->ytm[k]);
            tm1 += 1.0 / (1.0 + C->dis[k] / d02);
        }
        d002t = d002 + 1;
        for (;;) {
            j = 0;
            for (int k = 0; k < n; ++k)
                if (C->dis[k] <= d002t) {
                    memcpy(C->r1[j], C->xtm[k], sizeof(double) * 3);
                    memcpy(C->r2[j], C->ytm[k], sizeof(double) * 3);
                    j++;
                }
            if (j < 3 && n > 3) d002t += 0.5;
            else break;
        }
        fit(C, C->r1, C->r2, j, &F);
        tm2 = 0;
        C->counts[2] += n;
        for (int k = 0; k < n; ++k) {
            xform(&F, C->xtm[k], xr);
            tm2 += 1.0 / (1.0 + dist2(xr, C->ytm[k]) / d02);
        }
    } else {
        tm1 = tm2 = tm;
    }
    if (tm1 >= tm) tm = tm1;
    if (tm2 >= tm) tm = tm2;
    return tm;
}

/* ---------------------------------------------------------------------------------------------- dynamic programming */
enum { DP_TM = 0, DP_SSPLUS = 1, DP_SS = 2 };

/* NWDP_TM: mode DP_TM scores 1 / (1 + d^2 / d02) under F; DP_SSPLUS the same plus 0.5 where the codes match; DP_SS 1
 * where the codes match.  Cell (i, j) takes the diagonal when d >= h && d >= v, else max(v, h) with v on ties. */
static void nwdp(Ctx *C, int mode, const Fit *F, double d02, double gap_open, int *j2i) {
    const int len1 = C->xlen, len2 = C->ylen, W = len2 + 1;
    double *val = C->val;
    unsigned char *path = C->path;
    double xx[3];
    for (int i = 0; i <= len1; ++i) {
        val[i * W] = 0;
        path[i * W] = 0;
    }
    for (int j = 0; j <= len2; ++j) {
        val[j] = 0;
        path[j] = 0;
        if (j < len2) j2i[j] = -1;
    }
    C->counts[0] += (int64_t)len1 * len2;
    for (int i = 1; i <= len1; ++i) {
        if (mode != DP_SS) xform(F, C->x[i - 1], xx);
        for (int j = 1; j <= len2; ++j) {
            double d;
            if (mode == DP_SS) {
                d = C->secx[i - 1] == C->secy[j - 1] ? val[(i - 1) * W + j - 1] + 1.0 : val[(i - 1) * W + j - 1];
            } else {
                double s = 1.0 / (1.0 + dist2(xx, C->y[j - 1]) / d02);
                if (mode == DP_SSPLUS && C->secx[i - 1] == C->secy[j - 1]) s = s + 0.5;
                d = val[(i - 1) * W + j - 1] + s;
            }
            double h = val[(i - 1) * W + j];
            if (path[(i - 1) * W + j]) h += gap_open;
            double v = val[i * W + j - 1];
            if (path[i * W + j - 1]) v += gap_open;
            if (d >= h && d >= v) {
                path[i * W + j] = 1;
                val[i * W + j] = d;
            } else {
                path[i * W + j] = 0;
                val[i * W + j] = v >= h ? v : h;
            }
        }
    }
    int i = len1, j = len2;
    while (i > 0 && j > 0) {
        if (path[i * W + j]) {
            j2i[j - 1] = i - 1;
            i--;
            j--;
        } else {
            double h = val[(i - 1) * W + j];
            if (path[(i - 1) * W + j]) h += gap_open;
            double v = val[i * W + j - 1];
            if (path[i * W + j - 1]) v += gap_open;
            if (v >= h) j--;
            else i--;
        }
    }
}

/* DP_iter: F in = the transform of the last search, out = the last search's */
static double dp_iter(Ctx *C, Fit *F, int *map0, int g1, int g2, int iteration_max) {
    static const double gap_open[2] = {-0.6, 0};
    int *map = C->tmpmap;
    const double d02 = MUL(C->d0, C->d0);
    double tm_max = -1, tm_old = 0;
    for (int g = g1; g < g2; ++g)
        for (int it = 0; it < iteration_max; ++it) {
            nwdp(C, DP_TM, F, d02, gap_open[g], map);
            const double tm = detailed_search(C, map, F, 40, 0);
            if (tm > tm_max) {
                tm_max = tm;
                memcpy(map0, map, sizeof(int) * (size_t)C->ylen);
            }
            if (it > 0 && fabs(tm_old - tm) < 0.000001) break;
            tm_old = tm;
        }
    return tm_max;
}

/* ---------------------------------------------------------------------------------------------- initial alignments */
static void thread_map(int *map, int ylen, int k, int xlen) {
    for (int j = 0; j < ylen; ++j) {
        const int i = j + k;
        map[j] = i >= 0 && i < xlen ? i : -1;
    }
}

static void get_initial(Ctx *C, int *y2x) {
    const int xlen = C->xlen, ylen = C->ylen, min_len = xlen < ylen ? xlen : ylen;
    int min_ali = min_len / 2;
    if (min_ali <= 5) min_ali = 5;
    const int n1 = -ylen + min_ali, n2 = xlen - min_ali;
    double tm_max = -1;
    int k_best = n1;
    for (int k = n1; k <= n2; ++k) {
        thread_map(y2x, ylen, k, xlen);
        const double tm = get_score_fast(C, y2x);
        if (tm >= tm_max) {
            tm_max = tm;
            k_best = k;
        }
    }
    thread_map(y2x, ylen, k_best, xlen);
}

static int get_initial5(Ctx *C, int *y2x) {
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
                    memcpy(y2x, map, sizeof(int) * (size_t)ylen);
                    flag = 1;
                }
            }
    }
    return flag;
}

static void get_initial_ssplus(Ctx *C, const int *y2x0, int *y2x) {
    double d01 = C->d0 + 1.5;
    if (d01 < C->D0_MIN) d01 = C->D0_MIN;
    const int k = gather(C, y2x0);
    Fit F;
    fit(C, C->xtm, C->ytm, k, &F);
    nwdp(C, DP_SSPLUS, &F, MUL(d01, d01), -1.0, y2x);
}

/* the longest run of consecutive residues closer than the cutoff, grown by 1.1 per step (a running product) until the
 * run has at least min(4, floor(len / 3)) residues */
static void find_max_frag(const double (*x)[3], int len, int *start_max, int *end_max, double dcu0) {
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

static void get_initial_fgt(Ctx *C, int *y2x, double dcu0) {
    const int xlen = C->xlen, ylen = C->ylen;
    int xstart = 0, ystart = 0, xend = 0, yend = 0;
    find_max_frag(C->x, xlen, &xstart, &xend, dcu0);
    find_max_frag(C->y, ylen, &ystart, &yend, dcu0);
    const int Lx = xend - xstart + 1, Ly = yend - ystart + 1;
    int L_fr = Lx < Ly ? Lx : Ly;
    int *ifr = C->ifr, *map = C->tmpmap;
    const int use_x = Lx < Ly || (Lx == Ly && xlen <= ylen);
    for (int i = 0; i < L_fr; ++i) ifr[i] = (use_x ? xstart : ystart) + i;
    const int L0 = xlen < ylen ? xlen : ylen;
    if (L_fr == L0) {
        const int n1 = (int)MUL((double)L0, 0.1), n2 = (int)MUL((double)L0, 0.89);
        int j = 0;
        for (int i = n1; i <= n2; ++i) ifr[j++] = ifr[i];
        L_fr = j;
    }
    double tm_max = -1;
    const int other = use_x ? ylen : xlen, min_len = L_fr < other ? L_fr : other;
    int min_ali = (int)((double)min_len / 2.5);
    if (min_ali <= 3) min_ali = 3;
    const int n1 = -(use_x ? ylen : L_fr) + min_ali, n2 = (use_x ? L_fr : xlen) - min_ali;
    for (int k = n1; k <= n2; ++k) {
        if (use_x) {
            for (int j = 0; j < ylen; ++j) {
                const int i = j + k;
                map[j] = i >= 0 && i < L_fr ? ifr[i] : -1;
            }
        } else {
            for (int j = 0; j < ylen; ++j) map[j] = -1;
            for (int j = 0; j < L_fr; ++j) {
                const int i = j + k;
                if (i >= 0 && i < xlen) map[ifr[j]] = i;
            }
        }
        const double tm = get_score_fast(C, map);
        if (tm >= tm_max) {
            tm_max = tm;
            memcpy(y2x, map, sizeof(int) * (size_t)ylen);
        }
    }
}

static void record_of(const Fit *F, double *rec) {
    memcpy(rec, F->R, sizeof(double) * 9);
    memcpy(rec + 9, F->p, sizeof(double) * 3);
    memcpy(rec + 12, F->q, sizeof(double) * 3);
    rec[15] = 0.0;
}

/* params: [0] d0, [1] d0_search, [2] score_d8, [3] D0_MIN, [4] ddcc, [5] dcu0, [6] d0 and [7] d0_search of the final
 * score for L = ylen, [8] and [9] for L = xlen (tmalign_parameters) */
__attribute__((visibility("default"))) int oracle_tmalign_frame(const float *xf, int32_t xlen, const float *yf,
                                                                int32_t ylen, const double *params, double *tm,
                                                                double *rmsd, int32_t *nali, int32_t *invmap,
                                                                double *rec, int64_t *counts) {
    Fit F;
    identity_fit(&F);
    record_of(&F, rec);
    for (int j = 0; j < ylen; ++j) invmap[j] = -1;
    *nali = 0;
    for (int i = 0; i < 3 * xlen; ++i)
        if (!isfinite(xf[i])) {
            tm[0] = tm[1] = *rmsd = NAN;
            return 0;
        }
    const int n = xlen > ylen ? xlen : ylen;
    Ctx C;
    memset(&C, 0, sizeof(C));
    C.xlen = xlen;
    C.ylen = ylen;
    double(*xa)[3] = malloc(sizeof(double[3]) * (size_t)xlen), (*ya)[3] = malloc(sizeof(double[3]) * (size_t)ylen);
    for (int i = 0; i < 3 * xlen; ++i) xa[i / 3][i % 3] = xf[i];
    for (int i = 0; i < 3 * ylen; ++i) ya[i / 3][i % 3] = yf[i];
    C.x = (const double(*)[3])xa;
    C.y = (const double(*)[3])ya;
    C.secx = malloc((size_t)xlen);
    C.secy = malloc((size_t)ylen);
    C.xt = malloc(sizeof(double[3]) * (size_t)n);
    C.xtm = malloc(sizeof(double[3]) * (size_t)n);
    C.ytm = malloc(sizeof(double[3]) * (size_t)n);
    C.r1 = malloc(sizeof(double[3]) * (size_t)n);
    C.r2 = malloc(sizeof(double[3]) * (size_t)n);
    C.dis = malloc(sizeof(double) * (size_t)n);
    C.i_ali = malloc(sizeof(int) * (size_t)n);
    C.k_ali = malloc(sizeof(int) * (size_t)n);
    C.ifr = malloc(sizeof(int) * (size_t)n);
    C.tmpmap = malloc(sizeof(int) * (size_t)ylen);
    C.val = malloc(sizeof(double) * (size_t)(xlen + 1) * (size_t)(ylen + 1));
    C.path = malloc((size_t)(xlen + 1) * (size_t)(ylen + 1));
    int *map = malloc(sizeof(int) * (size_t)ylen), *map0 = malloc(sizeof(int) * (size_t)ylen);
    C.counts = counts;
    C.d0 = params[0];
    C.d0_search = params[1];
    C.score_d8 = params[2];
    C.D0_MIN = params[3];
    C.Lnorm = (double)(xlen < ylen ? xlen : ylen);
    const double ddcc = params[4], dcu0 = params[5];

    make_sec(C.x, xlen, C.secx);
    make_sec(C.y, ylen, C.secy);
    double TMmax = -1, TM;
#define KEEP()                                                     \
    if (TM > TMmax) {                                              \
        TMmax = TM;                                                \
        memcpy(map0, map, sizeof(int) * (size_t)ylen);             \
    }
    /* 1: gapless threading */
    get_initial(&C, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    TM = dp_iter(&C, &F, map, 0, 2, 30);
    KEEP();
    /* 2: secondary structure */
    nwdp(&C, DP_SS, &F, 1.0, -1.0, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, 0.2)) {
        TM = dp_iter(&C, &F, map, 0, 2, 30);
        KEEP();
    }
    /* 3: local superposition */
    if (get_initial5(&C, map)) {
        TM = detailed_search(&C, map, &F, 40, 0);
        KEEP();
        if (TM > MUL(TMmax, ddcc)) {
            TM = dp_iter(&C, &F, map, 0, 2, 2);
            KEEP();
        }
    }
    /* 4: secondary structure plus the best map so far */
    get_initial_ssplus(&C, map0, map);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, ddcc)) {
        TM = dp_iter(&C, &F, map, 0, 2, 30);
        KEEP();
    }
    /* 5: fragment gapless threading */
    get_initial_fgt(&C, map, dcu0);
    TM = detailed_search(&C, map, &F, 40, 0);
    KEEP();
    if (TM > MUL(TMmax, ddcc)) {
        TM = dp_iter(&C, &F, map, 1, 2, 2);
        KEEP();
    }
#undef KEEP
    /* final: the standard search on the best map, the pairs within score_d8 under it, their rmsd and both scores */
    detailed_search(&C, map0, &F, 1, 1);
    int k = 0;
    double xr[3];
    for (int j = 0; j < ylen; ++j) {
        const int i = map0[j];
        if (i < 0) continue;
        xform(&F, C.x[i], xr);
        if (sqrt(dist2(xr, C.y[j])) <= C.score_d8) {
            memcpy(C.xtm[k], C.x[i], sizeof(double) * 3);
            memcpy(C.ytm[k], C.y[j], sizeof(double) * 3);
            invmap[j] = i;
            k++;
        }
    }
    *nali = k;
    if (k == 0) {
        tm[0] = tm[1] = *rmsd = 0.0;
    } else {
        fit(&C, C.xtm, C.ytm, k, &F);
        double sq = 0;
        for (int m = 0; m < k; ++m) {
            xform(&F, C.xtm[m], xr);
            sq += dist2(xr, C.ytm[m]);
        }
        *rmsd = sqrt(sq / (double)k);
        /* xtm / ytm hold the nali pairs; the searches below gather nothing, they search those pairs */
        C.d0 = params[6];
        C.d0_search = params[7];
        tm[0] = tmscore8_search(&C, k, &F, 1, 0, C.d0_search, (double)ylen, C.d0, 0);
        record_of(&F, rec);
        Fit G;
        C.d0 = params[8];
        C.d0_search = params[9];
        tm[1] = tmscore8_search(&C, k, &G, 1, 0, C.d0_search, (double)xlen, C.d0, 0);
    }
    free(xa); free(ya); free(C.secx); free(C.secy); free(C.xt); free(C.xtm); free(C.ytm); free(C.r1); free(C.r2);
    free(C.dis); free(C.i_ali); free(C.k_ali); free(C.ifr); free(C.tmpmap); free(C.val); free(C.path); free(map);
    free(map0);
    return 0;
}

/* the secondary-structure codes of one trace (for the tests) */
__attribute__((visibility("default"))) void oracle_tmalign_sec(const float *xf, int32_t len, char *sec) {
    double(*x)[3] = malloc(sizeof(double[3]) * (size_t)(len > 0 ? len : 1));
    for (int i = 0; i < 3 * len; ++i) x[i / 3][i % 3] = xf[i];
    make_sec((const double(*)[3])x, len, sec);
    free(x);
}
