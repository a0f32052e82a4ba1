// divcheck.cu -- device check that mkb::div_by(a, b, refined_rcp(b)) == __fdiv_rn(a, b) bit for bit.
// Built and run by tests/test_wrapping_gpu.py on a GPU:  nvcc -arch=sm_90a -I moleculekit_b200/csrc ...
// Divisors: every integer 1..2^17, plus 2^14 larger ones up to 2^31 (the running-mean divisor n + 1).  Numerators per
// divisor: random bit patterns over the whole float range (incl. zeros, denormals, Inf, NaN -> the fallback branch),
// and for random quotients q the neighbours of q*b (rounding-boundary stress).
#include <cstdint>
#include <cstdio>

#include "exact_div.cuh"

__device__ __forceinline__ uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

__global__ void check(unsigned long long *bad, unsigned long long *tested, float *first_a, float *first_b) {
    const uint32_t bi = blockIdx.x;  // divisor index
    float b;
    if (bi < (1u << 17)) b = (float)(int)(bi + 1);
    else b = (float)(int)(((mix(bi) | 0x20000u) & 0x7fffffffu));
    if (b < 1.f) b = 1.f;
    const float r = mkb::refined_rcp(b);
    unsigned long long nbad = 0, n = 0;
    for (uint32_t it = threadIdx.x; it < 8192; it += blockDim.x) {
        const uint32_t h = mix(bi * 8192u + it);
        float a;
        if (it & 1) {
            a = __uint_as_float(h);  // any bit pattern
        } else {
            // q in a moderate range, a = RN(q*b) nudged by -2..2 ulps
            const float q = __uint_as_float((h & 0x007fffffu) | ((100u + (mix(h) % 56u)) << 23) | (h & 0x80000000u));
            const float p = __fmul_rn(q, b);
            a = __uint_as_float(__float_as_uint(p) + (int)(mix(h + 7u) % 5u) - 2);
        }
        const float want = __fdiv_rn(a, b);
        const float got = mkb::div_by(a, b, r);
        const bool same = __float_as_uint(want) == __float_as_uint(got) || (want != want && got != got);
        ++n;
        if (!same) {
            if (nbad == 0 && atomicAdd(bad, 0ull) == 0) { *first_a = a; *first_b = b; }
            ++nbad;
        }
    }
    atomicAdd(bad, nbad);
    atomicAdd(tested, n);
}

int main() {
    unsigned long long *bad, *tested;
    float *fa, *fb;
    cudaMallocManaged(&bad, 8); cudaMallocManaged(&tested, 8);
    cudaMallocManaged(&fa, 4); cudaMallocManaged(&fb, 4);
    *bad = 0; *tested = 0; *fa = 0; *fb = 0;
    check<<<(1u << 17) + (1u << 14), 256>>>(bad, tested, fa, fb);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("CUDA error\n"); return 2; }
    printf("divcheck tested=%llu mismatches=%llu first=(%a / %a)\n", *tested, *bad, *fa, *fb);
    return *bad ? 1 : 0;
}
