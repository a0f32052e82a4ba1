/* tmscore_oracle.c -- plain-C restatement of the TM-score superposition search (Zhang & Skolnick, Proteins 2004, the
 * TMscore program's search as moleculekit's molTMscore uses it), for the K19 parity tests.  TEST INFRASTRUCTURE ONLY:
 * the package never loads it.
 *
 * The contract is the mkb_tmscore comment of include/mkb200.h.  Compiled with -O3 -ffp-contract=off: every float64
 * operation is rounded on its own, in the order written here.  The cut set is found the literal way (count the pairs
 * below dcut, widen by 0.5 and count again), which the kernel replaces by a test on the third smallest distance.
 *
 * Input per frame: x [L][3] model and y [L][3] reference, float32 Angstrom, pair k = (x[k], y[k]).  Output: the
 * TM-score, the RMSD under the all-pairs fit, and the number of seeds, fits and pair evaluations (L per fit). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define N_EXT 20             /* extension fits per seed */
#define WIDEN_MAX (1 << 20)  /* widening steps of one cut at most */

typedef struct {
    double R[9], p[3], q[3];
} Fit;

static void jacobi_rot(double a[4][4], double v[4][4], int P, int Q, int late) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double g = 100.0 * fabs(apq);
    if (late && fabs(a[P][P]) + g == fabs(a[P][P]) && fabs(a[Q][Q]) + g == fabs(a[Q][Q])) {
        a[P][Q] = a[Q][P] = 0.0;
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
    for (int r = 0; r < 4; ++r) {
        if (r == P || r == Q) continue;
        const double arp = a[r][P], arq = a[r][Q];
        a[r][P] = a[P][r] = arp - s * (arq + arp * tau);
        a[r][Q] = a[Q][r] = arq + s * (arp - arq * tau);
    }
    for (int r = 0; r < 4; ++r) {
        const double vrp = v[r][P], vrq = v[r][Q];
        v[r][P] = vrp - s * (vrq + vrp * tau);
        v[r][Q] = vrq + s * (vrp - vrq * tau);
    }
}

/* Horn's quaternion: the proper rotation R (row-major, y ~ R x) for H[a][b] = sum x_a y_b */
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
        if (a[j][j] > best) { /* strict: ties go to the lowest index */
            best = a[j][j];
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

/* Kabsch fit of the pairs idx[0..c) (ascending): centroids, then H about them in a second pass */
static void fit(const float *x, const float *y, const int *idx, int c, Fit *F) {
    double sx[3] = {0, 0, 0}, sy[3] = {0, 0, 0}, H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < c; ++i)
        for (int d = 0; d < 3; ++d) {
            sx[d] += (double)x[3 * idx[i] + d];
            sy[d] += (double)y[3 * idx[i] + d];
        }
    for (int d = 0; d < 3; ++d) {
        F->p[d] = sx[d] / (double)c;
        F->q[d] = sy[d] / (double)c;
    }
    for (int i = 0; i < c; ++i) {
        double a[3], b[3];
        for (int d = 0; d < 3; ++d) {
            a[d] = (double)x[3 * idx[i] + d] - F->p[d];
            b[d] = (double)y[3 * idx[i] + d] - F->q[d];
        }
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 3; ++s) H[3 * r + s] += a[r] * b[s];
    }
    horn_rotation(H, F->R);
}

/* distances of all L pairs under F into dis[]; returns the score sum (before / Lnorm); *sq = sum of squared distances */
static double evaluate(const float *x, const float *y, int64_t L, const Fit *F, double d0, double *dis, double *sq) {
    double s = 0.0, s2 = 0.0;
    for (int64_t k = 0; k < L; ++k) {
        double a[3], e[3];
        for (int d = 0; d < 3; ++d) a[d] = (double)x[3 * k + d] - F->p[d];
        for (int d = 0; d < 3; ++d)
            e[d] = F->R[3 * d] * a[0] + F->R[3 * d + 1] * a[1] + F->R[3 * d + 2] * a[2] + F->q[d] - (double)y[3 * k + d];
        const double d2 = e[0] * e[0] + e[1] * e[1] + e[2] * e[2];
        dis[k] = sqrt(d2);
        const double t = dis[k] / d0;
        s += 1.0 / (1.0 + t * t);
        s2 += d2;
    }
    *sq = s2;
    return s;
}

/* the cut set of dis[] at dcut, widened by 0.5 while it has fewer than 3 pairs and L > 3; returns its size */
static int cut(const double *dis, int64_t L, double dcut, int *out) {
    for (int step = 0;; ++step) {
        int n = 0;
        for (int64_t k = 0; k < L; ++k)
            if (dis[k] < dcut) out[n++] = (int)k;
        if (n < 3 && L > 3 && step < WIDEN_MAX) {
            dcut += 0.5;
            continue;
        }
        return n;
    }
}

__attribute__((visibility("default"))) int oracle_tmscore_frame(const float *x, const float *y, int64_t L, int64_t Lnorm,
                                                                 double d0, double d0_search, const int32_t *frag,
                                                                 int32_t nfrag, double *tm, double *rmsd,
                                                                 int64_t *counts) {
    for (int64_t i = 0; i < 3 * L; ++i)
        if (!isfinite(x[i]) || !isfinite(y[i])) {
            *tm = NAN;
            *rmsd = NAN;
            return 0;
        }
    double *dis = malloc(sizeof(double) * (size_t)L);
    int *fitset = malloc(sizeof(int) * (size_t)L), *cs = malloc(sizeof(int) * (size_t)L);
    if (!dis || !fitset || !cs) return 1;
    double best = -1.0, sq;
    int first = 1;
    for (int fi = 0; fi < nfrag; ++fi) {
        const int Li = frag[fi];
        for (int64_t iL = 0; iL <= L - Li; ++iL) {
            counts[0]++;
            int nfit = Li;
            for (int i = 0; i < Li; ++i) fitset[i] = (int)iL + i;
            Fit F;
            fit(x, y, fitset, nfit, &F);
            double s = evaluate(x, y, L, &F, d0, dis, &sq) / (double)Lnorm;
            counts[1]++;
            counts[2] += L;
            if (first) {
                *rmsd = sqrt(sq / (double)L);
                first = 0;
            }
            if (s > best) best = s;
            int ncut = cut(dis, L, d0_search - 1.0, cs);
            for (int it = 0; it < N_EXT && ncut > 0; ++it) {
                memcpy(fitset, cs, sizeof(int) * (size_t)ncut);
                nfit = ncut;
                fit(x, y, fitset, nfit, &F);
                s = evaluate(x, y, L, &F, d0, dis, &sq) / (double)Lnorm;
                counts[1]++;
                counts[2] += L;
                if (s > best) best = s;
                ncut = cut(dis, L, d0_search + 1.0, cs);
                if (ncut == nfit && memcmp(cs, fitset, sizeof(int) * (size_t)ncut) == 0) break;
            }
        }
    }
    *tm = best;
    free(dis);
    free(fitset);
    free(cs);
    return 0;
}
