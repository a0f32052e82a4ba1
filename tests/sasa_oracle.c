/* sasa_oracle.c -- plain-C restatement of mdtraj's Shrake-Rupley frame loop (mdtraj/geometry/src/sasa.cpp, asa_frame)
 * for the K17 parity tests.  TEST INFRASTRUCTURE ONLY: the package never loads it.
 *
 * Compiled with -O3 -ffp-contract=off: every float32 operation is rounded on its own, as in the reference's SSE code.
 * The squared distance is ((dx dx + dy dy) + dz dz), the order of SSE dpps with mask 0x71.  The neighbour search is the
 * reference's O(n^2) scan and the points try the neighbours starting from the one that buried the previous point.
 * Where the reference prints an error and calls exit(1) on two atoms closer than 1e-5 nm, this returns 1 and reports the
 * pair.  Only the atoms listed in `atoms` are computed (each area is independent of the others), and the coincidence
 * check covers the pairs that contain one of them. */
#include <stdint.h>
#include <stdlib.h>

static float dot3(float x, float y, float z) { return (x * x + y * y) + z * z; }

__attribute__((visibility("default"))) int oracle_sasa_frame(const float *xyz, const float *radii, int64_t n,
                                                             const int64_t *atoms, int64_t n_atoms,
                                                             const float *sphere, int32_t n_sphere, float *areas,
                                                             int64_t *bad_pair) {
    const float constant = (float)(4.0 * 3.14159265358979323846 / n_sphere);
    int64_t *nb = (int64_t *)malloc(sizeof(int64_t) * (size_t)(n > 0 ? n : 1));
    if (!nb) return -1;
    for (int64_t a = 0; a < n_atoms; ++a) {
        const int64_t i = atoms[a];
        const float ri = radii[i];
        const float xi = xyz[3 * i], yi = xyz[3 * i + 1], zi = xyz[3 * i + 2];
        int64_t n_nb = 0;
        for (int64_t j = 0; j < n; ++j) {
            if (j == i) continue;
            const float rc = ri + radii[j];
            const float rc2 = rc * rc;
            const float r2 = dot3(xi - xyz[3 * j], yi - xyz[3 * j + 1], zi - xyz[3 * j + 2]);
            if (r2 < rc2) nb[n_nb++] = j;
            if (r2 < 1e-10f) {
                bad_pair[0] = i;
                bad_pair[1] = j;
                free(nb);
                return 1;
            }
        }
        int64_t n_acc = 0, k_closest = 0;
        for (int32_t s = 0; s < n_sphere; ++s) {
            const float px = xi + ri * sphere[3 * s], py = yi + ri * sphere[3 * s + 1], pz = zi + ri * sphere[3 * s + 2];
            int accessible = 1;
            for (int64_t k = k_closest; k < n_nb + k_closest; ++k) {
                const int64_t idx = nb[k % n_nb];
                const float r = radii[idx];
                if (dot3(px - xyz[3 * idx], py - xyz[3 * idx + 1], pz - xyz[3 * idx + 2]) < r * r) {
                    k_closest = k % n_nb;
                    accessible = 0;
                    break;
                }
            }
            n_acc += accessible;
        }
        areas[a] = constant * ri * ri * (float)n_acc;
    }
    free(nb);
    return 0;
}
