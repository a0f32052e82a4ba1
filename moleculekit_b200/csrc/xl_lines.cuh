// xl_lines.cuh -- the pieces of K26's newline index that K28 (pdb.cu) shares with K26 (xyz.cu): the segment shape of
// the count and emit passes, the 16-byte SWAR byte masks, and the one-CTA scan that turns per-segment counts into each
// segment's base and advances a running count kept on the device.
//
// The scan kernel has internal linkage: each .cu that includes this header instantiates its own copy.
#pragma once

#include <cub/block/block_scan.cuh>

namespace mkb {
namespace {

constexpr int XL_THREADS = 256, XL_ITEMS = 8;
constexpr long long XL_SEG = 16LL * XL_THREADS * XL_ITEMS;  // bytes per segment (one CTA of the count and emit passes)
constexpr int XL_SCAN_THREADS = 1024;

// bit b of the result: byte b of the 16 bytes is c
__device__ __forceinline__ unsigned xl_mask(const uint4 &v, unsigned c) {
    const unsigned pat = c * 0x01010101u;
    const unsigned w[4] = {v.x ^ pat, v.y ^ pat, v.z ^ pat, v.w ^ pat};
    unsigned m = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const unsigned z = ~((((w[i] & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w[i])) & 0x80808080u;  // bit 7 of each zero byte
        m |= (((z >> 7) & 1u) | ((z >> 14) & 2u) | ((z >> 21) & 4u) | ((z >> 28) & 8u)) << (4 * i);
    }
    return m;
}

// the bytes of the 16-byte word at p0 that lie below n
__device__ __forceinline__ unsigned xl_valid(long long p0, long long n) {
    const long long r = n - p0;
    return r >= 16 ? 0xffffu : r <= 0 ? 0u : (1u << r) - 1u;
}

// base[s] = state[0] + the counts of segments before s; state[0] += all of them
__global__ void __launch_bounds__(XL_SCAN_THREADS) xyz_scan_kernel(const unsigned *__restrict__ counts, int n_seg,
                                                                   long long *__restrict__ base,
                                                                   long long *__restrict__ state) {
    using Scan = cub::BlockScan<unsigned, XL_SCAN_THREADS>;  // a tile holds at most 1024 * 32 KB items
    __shared__ typename Scan::TempStorage tmp;
    long long carry = state[0];
    for (int s0 = 0; s0 < n_seg; s0 += XL_SCAN_THREADS) {
        const int s = s0 + threadIdx.x;
        unsigned ex, total;
        Scan(tmp).ExclusiveSum(s < n_seg ? counts[s] : 0u, ex, total);
        if (s < n_seg) base[s] = carry + ex;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) state[0] = carry;
}

}  // namespace
}  // namespace mkb
