/* dssp_oracle.c -- plain-C restatement of the DSSP 2.2.0 secondary-structure assignment that mdtraj's compute_dssp
 * ports, for the K18 parity tests.  TEST INFRASTRUCTURE ONLY: the package never loads it.
 *
 * It keeps the reference's own loop structure: the `for i, for j > i` energy loop that calls both directions, the
 * literal bridge double loop with the first-matching-bridge search, and the std::vector erase loop of the ladder merge
 * with uint32 differences.  Compiled with -O3 -ffp-contract=off: every float64 operation is rounded on its own.
 *
 * Input per frame: bb [n][4][3] float32 (N, CA, C, O of every residue of the DSSP sequence, Angstrom) and flags [n]
 * (bit 0 PRO, bit 1 residue starts a new chain or segid).  Output: codes [n] (0 loop, 1 H, 2 B, 3 E, 4 G, 5 I, 6 T,
 * 7 S), the two (partner, energy) slots of every donor, and the number of CA pairs screened / energies evaluated. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define K_COUPLING (-27.888)
#define K_MIN_E (-9.9)
#define K_MAX_BOND_E (-0.5)

enum { LOOP = 0, HELIX = 1, BRIDGE = 2, STRAND = 3, HELIX3 = 4, HELIX5 = 5, TURN = 6, BEND = 7 };
enum { NO_BRIDGE = 0, PARALLEL = 1, ANTIPARALLEL = 2 };

typedef struct {
    double n[3], ca[3], c[3], o[3], h[3];
    int pro;
} Res;

typedef struct {
    int type;
    int *i, *j;   /* the i and j lists (std::deque in the reference) */
    int ni, nj;
} Bridge;

static double dist(const double *a, const double *b) {
    const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
    return sqrt((dx * dx + dy * dy) + dz * dz);
}

typedef struct {
    int64_t n;
    const Res *r;
    const uint8_t *brk;  /* brk[k]: a break lies between k and k + 1 */
    int32_t *partner;    /* [n][2] */
    double *energy;      /* [n][2] */
} Ctx;

static int no_chain_break(const Ctx *x, int64_t a, int64_t b) {
    for (int64_t k = a; k < b; ++k)
        if (x->brk[k]) return 0;
    return 1;
}

static void hbond(Ctx *x, int64_t d, int64_t a, int64_t *evaluated) {
    const Res *D = &x->r[d], *A = &x->r[a];
    if (D->pro) return;
    ++*evaluated;
    const double dHO = dist(D->h, A->o), dHC = dist(D->h, A->c), dNC = dist(D->n, A->c), dNO = dist(D->n, A->o);
    double e;
    if (dHO < 0.5 || dHC < 0.5 || dNC < 0.5 || dNO < 0.5)
        e = K_MIN_E;
    else
        e = K_COUPLING / dHO - K_COUPLING / dHC + K_COUPLING / dNC - K_COUPLING / dNO;
    e = round(e * 1000) / 1000;
    if (e < K_MIN_E) e = K_MIN_E;
    int32_t *p = x->partner + 2 * d;
    double *E = x->energy + 2 * d;
    if (e < E[0]) {
        p[1] = p[0]; E[1] = E[0];
        p[0] = (int32_t)a; E[0] = e;
    } else if (e < E[1]) {
        p[1] = (int32_t)a; E[1] = e;
    }
}

static int test_bond(const Ctx *x, int64_t d, int64_t a) {
    const int32_t *p = x->partner + 2 * d;
    const double *E = x->energy + 2 * d;
    return (p[0] == a && E[0] < K_MAX_BOND_E) || (p[1] == a && E[1] < K_MAX_BOND_E);
}

static int test_bridge(const Ctx *x, int64_t i, int64_t j) {
    const int64_t a = i - 1, b = i, c = i + 1, d = j - 1, e = j, f = j + 1;
    if (!(no_chain_break(x, a, c) && no_chain_break(x, d, f))) return NO_BRIDGE;
    if ((test_bond(x, c, e) && test_bond(x, e, a)) || (test_bond(x, f, b) && test_bond(x, b, d))) return PARALLEL;
    if ((test_bond(x, c, d) && test_bond(x, f, a)) || (test_bond(x, e, b) && test_bond(x, b, e))) return ANTIPARALLEL;
    return NO_BRIDGE;
}

/* returns 0, or -1 when out of memory */
__attribute__((visibility("default"))) int oracle_dssp_frame(const float *bb, const uint8_t *flags, int64_t n,
                                                             uint8_t *codes, int32_t *partner, double *energy,
                                                             int64_t *counts) {
    Res *r = (Res *)calloc((size_t)(n > 0 ? n : 1), sizeof(Res));
    uint8_t *brk = (uint8_t *)calloc((size_t)(n > 0 ? n : 1), 1);
    uint8_t *start = (uint8_t *)calloc((size_t)(n > 0 ? 3 * n : 1), 1);
    int *bent = (int *)calloc((size_t)(n > 0 ? n : 1), sizeof(int));
    Bridge *br = (Bridge *)calloc((size_t)(n > 0 ? 8 * n : 1), sizeof(Bridge));
    if (!r || !brk || !start || !bent || !br) {
        free(r); free(brk); free(start); free(bent); free(br);
        return -1;
    }
    for (int64_t k = 0; k < n; ++k) {
        for (int d = 0; d < 3; ++d) {
            r[k].n[d] = bb[12 * k + d];
            r[k].ca[d] = bb[12 * k + 3 + d];
            r[k].c[d] = bb[12 * k + 6 + d];
            r[k].o[d] = bb[12 * k + 9 + d];
        }
        r[k].pro = flags[k] & 1;
    }
    for (int64_t k = 0; k + 1 < n; ++k) brk[k] = (flags[k + 1] & 2) || dist(r[k].c, r[k + 1].n) > 2.5;
    for (int64_t k = 0; k < n; ++k) {
        memcpy(r[k].h, r[k].n, sizeof(r[k].h));
        if (!r[k].pro && k > 0 && !brk[k - 1]) {
            const double v[3] = {r[k - 1].c[0] - r[k - 1].o[0], r[k - 1].c[1] - r[k - 1].o[1],
                                 r[k - 1].c[2] - r[k - 1].o[2]};
            const double len = sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
            for (int d = 0; d < 3; ++d) r[k].h[d] = r[k].n[d] + v[d] / len;
        }
    }
    Ctx x = {n, r, brk, partner, energy};
    for (int64_t k = 0; k < 2 * n; ++k) {
        partner[k] = -1;
        energy[k] = 0.0;
    }
    /* energies: the reference's loop over i < j with the CA screen, both directions but donor i + 1 / acceptor i */
    int64_t screened = 0, evaluated = 0;
    for (int64_t i = 0; i < n; ++i)
        for (int64_t j = i + 1; j < n; ++j) {
            ++screened;
            if (dist(r[i].ca, r[j].ca) < 9.0) {
                hbond(&x, i, j, &evaluated);
                if (j != i + 1) hbond(&x, j, i, &evaluated);
            }
        }
    /* bends */
    for (int64_t i = 2; i + 2 < n; ++i) {
        if (!no_chain_break(&x, i - 2, i + 2)) continue;
        double u[3], w[3];
        for (int d = 0; d < 3; ++d) {
            u[d] = r[i].ca[d] - r[i - 2].ca[d];
            w[d] = r[i + 2].ca[d] - r[i].ca[d];
        }
        const double xx = ((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) * ((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]);
        double c = 0;
        if (xx > 0) c = ((u[0] * w[0] + u[1] * w[1]) + u[2] * w[2]) / sqrt(xx);
        bent[i] = (acos(c) * 180) / 3.14159265358979323846 > 70;
    }
    /* helix flags: None 0, Start 1, End 2, StartAndEnd 3, Middle 4 (per stride) */
    uint8_t *hf = start;
    for (int s = 3; s <= 5; ++s) {
        uint8_t *f = hf + (s - 3) * n;
        for (int64_t i = 0; i + s < n; ++i) {
            if (no_chain_break(&x, i, i + s) && test_bond(&x, i + s, i)) {
                f[i + s] = 2;
                for (int64_t k = i + 1; k < i + s; ++k)
                    if (f[k] == 0) f[k] = 4;
                f[i] = f[i] == 2 ? 3 : 1;
            }
        }
    }
#define IS_START(s, k) (hf[((s) - 3) * n + (k)] == 1 || hf[((s) - 3) * n + (k)] == 3)
    /* bridges: the literal double loop, joining the first matching bridge in vector order */
    int64_t nb = 0;
    for (int64_t i = 1; i + 4 < n; ++i)
        for (int64_t j = i + 3; j + 1 < n; ++j) {
            const int type = test_bridge(&x, i, j);
            if (type == NO_BRIDGE) continue;
            int found = 0;
            for (int64_t b = 0; b < nb && !found; ++b) {
                Bridge *B = &br[b];
                if (type != B->type || i != B->i[B->ni - 1] + 1) continue;
                if (type == PARALLEL && B->j[B->nj - 1] + 1 == j) {
                    B->i[B->ni++] = (int)i;
                    B->j[B->nj++] = (int)j;
                    found = 1;
                } else if (type == ANTIPARALLEL && B->j[0] - 1 == j) {
                    B->i[B->ni++] = (int)i;
                    memmove(B->j + 1, B->j, sizeof(int) * (size_t)B->nj);
                    B->j[0] = (int)j;
                    B->nj++;
                    found = 1;
                }
            }
            if (!found) {
                Bridge *B = &br[nb++];
                B->type = type;
                B->i = (int *)malloc(sizeof(int) * (size_t)n);
                B->j = (int *)malloc(sizeof(int) * (size_t)n);
                B->i[0] = (int)i;
                B->j[0] = (int)j;
                B->ni = B->nj = 1;
            }
        }
    /* ladders: stable sort by i.front (creation order already is), then the erase loop with uint32 differences */
    for (int64_t a = 1; a < nb; ++a) {
        Bridge t = br[a];
        int64_t b = a;
        while (b > 0 && br[b - 1].i[0] > t.i[0]) {
            br[b] = br[b - 1];
            --b;
        }
        br[b] = t;
    }
    for (int64_t p = 0; p < nb; ++p)
        for (int64_t q = p + 1; q < nb; ++q) {
            Bridge *P = &br[p], *Q = &br[q];
            const uint32_t ibi = (uint32_t)P->i[0], iei = (uint32_t)P->i[P->ni - 1];
            const uint32_t jbi = (uint32_t)P->j[0], jei = (uint32_t)P->j[P->nj - 1];
            const uint32_t ibj = (uint32_t)Q->i[0], iej = (uint32_t)Q->i[Q->ni - 1];
            const uint32_t jbj = (uint32_t)Q->j[0], jej = (uint32_t)Q->j[Q->nj - 1];
            if (P->type != Q->type || !no_chain_break(&x, ibi < ibj ? ibi : ibj, iei > iej ? iei : iej) ||
                !no_chain_break(&x, jbi < jbj ? jbi : jbj, jei > jej ? jei : jej) || ibj - iei >= 6 ||
                (iei >= ibj && ibi <= iej))
                continue;
            int bulge;
            if (P->type == PARALLEL)
                bulge = (jbj - jei < 6 && ibj - iei < 3) || jbj - jei < 3;
            else
                bulge = (jbi - jej < 6 && ibj - iei < 3) || jbi - jej < 3;
            if (bulge) {
                memcpy(P->i + P->ni, Q->i, sizeof(int) * (size_t)Q->ni);
                P->ni += Q->ni;
                if (P->type == PARALLEL) {
                    memcpy(P->j + P->nj, Q->j, sizeof(int) * (size_t)Q->nj);
                } else {
                    memmove(P->j + Q->nj, P->j, sizeof(int) * (size_t)P->nj);
                    memcpy(P->j, Q->j, sizeof(int) * (size_t)Q->nj);
                }
                P->nj += Q->nj;
                free(Q->i);
                free(Q->j);
                memmove(br + q, br + q + 1, sizeof(Bridge) * (size_t)(nb - q - 1));
                --nb;
                --q;
            }
        }
    /* codes */
    for (int64_t k = 0; k < n; ++k) codes[k] = LOOP;
    for (int64_t b = 0; b < nb; ++b) {
        const Bridge *B = &br[b];
        const uint8_t ss = B->ni > 1 ? STRAND : BRIDGE;
        for (int64_t k = B->i[0]; k <= B->i[B->ni - 1]; ++k)
            if (codes[k] != STRAND) codes[k] = ss;
        for (int64_t k = B->j[0]; k <= B->j[B->nj - 1]; ++k)
            if (codes[k] != STRAND) codes[k] = ss;
    }
    for (int64_t i = 1; i + 4 < n; ++i)
        if (IS_START(4, i) && IS_START(4, i - 1))
            for (int64_t k = i; k <= i + 3; ++k) codes[k] = HELIX;
    for (int64_t i = 1; i + 3 < n; ++i)
        if (IS_START(3, i) && IS_START(3, i - 1)) {
            int empty = 1;
            for (int64_t k = i; empty && k <= i + 2; ++k) empty = codes[k] == LOOP || codes[k] == HELIX3;
            if (empty)
                for (int64_t k = i; k <= i + 2; ++k) codes[k] = HELIX3;
        }
    for (int64_t i = 1; i + 5 < n; ++i)
        if (IS_START(5, i) && IS_START(5, i - 1)) {
            int empty = 1;
            for (int64_t k = i; empty && k <= i + 4; ++k) empty = codes[k] == LOOP || codes[k] == HELIX5;
            if (empty)
                for (int64_t k = i; k <= i + 4; ++k) codes[k] = HELIX5;
        }
    for (int64_t i = 1; i + 1 < n; ++i)
        if (codes[i] == LOOP) {
            int turn = 0;
            for (int s = 3; s <= 5 && !turn; ++s)
                for (int64_t k = 1; k < s && !turn; ++k) turn = i >= k && IS_START(s, i - k);
            if (turn)
                codes[i] = TURN;
            else if (bent[i])
                codes[i] = BEND;
        }
#undef IS_START
    if (counts) {
        counts[0] = screened;
        counts[1] = evaluated;
    }
    for (int64_t b = 0; b < nb; ++b) {
        free(br[b].i);
        free(br[b].j);
    }
    free(r); free(brk); free(start); free(bent); free(br);
    return 0;
}
