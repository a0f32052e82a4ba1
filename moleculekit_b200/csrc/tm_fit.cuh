// tm_fit.cuh -- the float64 Horn / Jacobi rotation of the TM-score search (K19), shared with TM-align (K27).
// Every operation is rounded on its own (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so the rotation is
// bit-identical to a C restatement compiled without contraction.
#pragma once

#include "common.cuh"

namespace mkb {

#define DADD __dadd_rn
#define DSUB __dsub_rn
#define DMUL __dmul_rn
#define DDIV __ddiv_rn

// K14's Jacobi rotation with every operation rounded on its own
template <int P, int Q>
__device__ __forceinline__ void tm_jacobi_rot(double (&a)[4][4], double (&v)[4][4], bool late) {
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double g = DMUL(100.0, fabs(apq));
    if (late && DADD(fabs(a[P][P]), g) == fabs(a[P][P]) && DADD(fabs(a[Q][Q]), g) == fabs(a[Q][Q])) {
        a[P][Q] = a[Q][P] = 0.0;
        return;
    }
    const double h = DSUB(a[Q][Q], a[P][P]);
    double t;
    if (DADD(fabs(h), g) == fabs(h)) {
        t = DDIV(apq, h);
    } else {
        const double th = DDIV(DMUL(0.5, h), apq);
        t = DDIV(1.0, DADD(fabs(th), __dsqrt_rn(DADD(1.0, DMUL(th, th)))));
        if (th < 0.0) t = -t;
    }
    const double c = DDIV(1.0, __dsqrt_rn(DADD(1.0, DMUL(t, t)))), s = DMUL(t, c), tau = DDIV(s, DADD(1.0, c));
    a[P][P] = DSUB(a[P][P], DMUL(t, apq));
    a[Q][Q] = DADD(a[Q][Q], DMUL(t, apq));
    a[P][Q] = a[Q][P] = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        if (r == P || r == Q) continue;
        const double arp = a[r][P], arq = a[r][Q];
        a[r][P] = a[P][r] = DSUB(arp, DMUL(s, DADD(arq, DMUL(arp, tau))));
        a[r][Q] = a[Q][r] = DADD(arq, DMUL(s, DSUB(arp, DMUL(arq, tau))));
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const double vrp = v[r][P], vrq = v[r][Q];
        v[r][P] = DSUB(vrp, DMUL(s, DADD(vrq, DMUL(vrp, tau))));
        v[r][Q] = DADD(vrq, DMUL(s, DSUB(vrp, DMUL(vrq, tau))));
    }
}

// K14's horn_rotation with every operation rounded on its own (K14's own keeps its contracted bits)
__device__ __forceinline__ void tm_horn_rotation(const double (&H)[9], double (&R)[9]) {
    const double Sxx = H[0], Sxy = H[1], Sxz = H[2], Syx = H[3], Syy = H[4], Syz = H[5], Szx = H[6], Szy = H[7],
                 Szz = H[8];
    double a[4][4] = {{DADD(DADD(Sxx, Syy), Szz), DSUB(Syz, Szy), DSUB(Szx, Sxz), DSUB(Sxy, Syx)},
                      {DSUB(Syz, Szy), DSUB(DSUB(Sxx, Syy), Szz), DADD(Sxy, Syx), DADD(Szx, Sxz)},
                      {DSUB(Szx, Sxz), DADD(Sxy, Syx), DSUB(DADD(-Sxx, Syy), Szz), DADD(Syz, Szy)},
                      {DSUB(Sxy, Syx), DADD(Szx, Sxz), DADD(Syz, Szy), DADD(DSUB(-Sxx, Syy), Szz)}};
    double v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[0][3]) + fabs(a[1][2]) + fabs(a[1][3]) + fabs(a[2][3]);
        if (off == 0.0) break;
        const bool late = sweep > 3;
        tm_jacobi_rot<0, 1>(a, v, late);
        tm_jacobi_rot<0, 2>(a, v, late);
        tm_jacobi_rot<0, 3>(a, v, late);
        tm_jacobi_rot<1, 2>(a, v, late);
        tm_jacobi_rot<1, 3>(a, v, late);
        tm_jacobi_rot<2, 3>(a, v, late);
    }
    double q[4] = {v[0][0], v[1][0], v[2][0], v[3][0]}, best = a[0][0];
#pragma unroll
    for (int j = 1; j < 4; ++j)
        if (a[j][j] > best) {  // strict: ties go to the lowest index
            best = a[j][j];
#pragma unroll
            for (int r = 0; r < 4; ++r) q[r] = v[r][j];
        }
    const double inv = DDIV(1.0, __dsqrt_rn(DADD(DADD(DADD(DMUL(q[0], q[0]), DMUL(q[1], q[1])), DMUL(q[2], q[2])),
                                                 DMUL(q[3], q[3]))));
    const double q0 = DMUL(q[0], inv), q1 = DMUL(q[1], inv), q2 = DMUL(q[2], inv), q3 = DMUL(q[3], inv);
    const double q00 = DMUL(q0, q0), q11 = DMUL(q1, q1), q22 = DMUL(q2, q2), q33 = DMUL(q3, q3);
    R[0] = DSUB(DSUB(DADD(q00, q11), q22), q33);
    R[1] = DMUL(2.0, DSUB(DMUL(q1, q2), DMUL(q0, q3)));
    R[2] = DMUL(2.0, DADD(DMUL(q1, q3), DMUL(q0, q2)));
    R[3] = DMUL(2.0, DADD(DMUL(q1, q2), DMUL(q0, q3)));
    R[4] = DSUB(DADD(DSUB(q00, q11), q22), q33);
    R[5] = DMUL(2.0, DSUB(DMUL(q2, q3), DMUL(q0, q1)));
    R[6] = DMUL(2.0, DSUB(DMUL(q1, q3), DMUL(q0, q2)));
    R[7] = DMUL(2.0, DADD(DMUL(q2, q3), DMUL(q0, q1)));
    R[8] = DADD(DSUB(DSUB(q00, q11), q22), q33);
}

}  // namespace mkb
