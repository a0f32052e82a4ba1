// xl_lines.cuh -- K26's newline index, shared by K26 (xyz.cu), K28 (pdb.cu) and K29 (gro.cu): the segment shape of the
// count and emit passes, the 16-byte SWAR byte masks, the one-CTA scan that turns per-segment counts into each
// segment's base and advances a running count kept on the device, the newline count kernel, the count-line check, the
// emit kernel and xyz_lines, which launches the three passes.
//
// The kernels have internal linkage: each .cu that includes this header instantiates its own copies.
#pragma once

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "xyz_number.cuh"

namespace mkb {
namespace {

constexpr int XL_THREADS = 256, XL_ITEMS = 8;
constexpr long long XL_SEG = 16LL * XL_THREADS * XL_ITEMS;  // bytes per segment (one CTA of the count and emit passes)
constexpr int XL_SCAN_THREADS = 1024;
constexpr int XYZ_COUNT_WINDOW = 64;  // bytes of a count line the device reads; a longer one is left to the host

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

__global__ void __launch_bounds__(XL_THREADS) xyz_count_kernel(const uint4 *__restrict__ bytes, long long n,
                                                               unsigned *__restrict__ counts) {
    using Reduce = cub::BlockReduce<unsigned, XL_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    unsigned c = 0;
#pragma unroll
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x;
        if (16 * wi < n) c += __popc(xl_mask(__ldcs(bytes + wi), '\n') & xl_valid(16 * wi, n));
    }
    const unsigned total = Reduce(tmp).Sum(c);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// the count line at b[p]: 0 when its first field is natoms written as [+]digits, else 1 (the host decides)
__device__ unsigned char xyz_count_line(const unsigned char *__restrict__ b, long long p, long long n_read,
                                        long long natoms) {
    const long long e = min(n_read, p + XYZ_COUNT_WINDOW);
    while (p < e && xyz_sep(b[p]) && b[p] != '\n') ++p;
    if (p < e && b[p] == '+') ++p;
    long long v = 0;
    int nd = 0;
    for (; p < e && xyz_digit(b[p]); ++p, ++nd)
        if (v <= INT32_MAX) v = 10 * v + (b[p] - '0');
    return nd > 0 && p < e && xyz_sep(b[p]) && v == natoms ? 0 : 1;
}

// INDEX: lines numbered from state[0]'s value before the scan; a line L that starts a frame (L % P == 0, f = L / P)
// gets frame_off[f] = file_base + its byte and status[f] = its count-line check (f >= frame_cap: state[2] = max f + 1);
// a lone CR atomicMins file_base + its byte into state[1].  Otherwise: starts[L] = its byte for L < starts_cap, and
// starts[0] = 0.
template <bool INDEX>
__global__ void __launch_bounds__(XL_THREADS)
xyz_emit_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, const long long *__restrict__ base,
                long long file_base, long long P, long long natoms, long long *__restrict__ frame_off,
                unsigned char *__restrict__ status, long long frame_cap, long long *__restrict__ state,
                long long *__restrict__ starts, long long starts_cap) {
    using Scan = cub::BlockScan<unsigned, XL_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const unsigned char *b = reinterpret_cast<const unsigned char *>(bytes);
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    long long g0 = base[blockIdx.x];  // number of the first newline of the segment
    if (!INDEX && blockIdx.x == 0 && threadIdx.x == 0 && starts_cap > 0) starts[0] = 0;
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        unsigned nl = 0, cr = 0;
        if (p0 < n) {
            const uint4 v = __ldg(bytes + wi);
            const unsigned ok = xl_valid(p0, n);
            nl = xl_mask(v, '\n') & ok;
            if (INDEX) cr = xl_mask(v, '\r') & ok;
        }
        unsigned ex, total;
        Scan(tmp).ExclusiveSum((unsigned)__popc(nl), ex, total);
        long long g = g0 + ex;
        for (; nl; nl &= nl - 1, ++g) {
            const long long pos = p0 + __ffs(nl) - 1, L = g + 1;
            if (INDEX) {
                if (L % P == 0 && pos + 1 < n_read) {
                    const long long f = L / P;
                    if (f < frame_cap) {
                        frame_off[f] = file_base + pos + 1;
                        status[f] = xyz_count_line(b, pos + 1, n_read, natoms);
                    } else {
                        atomicMax(reinterpret_cast<unsigned long long *>(state + 2), (unsigned long long)(f + 1));
                    }
                }
            } else if (L < starts_cap) {
                starts[L] = pos + 1;
            }
        }
        for (; cr; cr &= cr - 1) {
            const long long pos = p0 + __ffs(cr) - 1;
            if (pos + 1 < n_read && b[pos + 1] != '\n')
                atomicMin(reinterpret_cast<unsigned long long *>(state + 1), (unsigned long long)(file_base + pos));
        }
        g0 += total;
        __syncthreads();  // tmp is reused by the next item's scan
    }
}

// the three newline passes over bytes[0, n); the scan reads and advances state[0]
template <bool INDEX>
int xyz_lines(mkb_ctx *h, cudaStream_t st, const uint8_t *bytes, int64_t n, int64_t n_read, int64_t file_base,
              int64_t P, int64_t natoms, int64_t *frame_off, uint8_t *status, int64_t frame_cap, int64_t *state,
              long long *starts, int64_t starts_cap) {
    const int64_t n_seg = std::max<int64_t>(1, cdiv(n, XL_SEG));
    if (n_seg > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    unsigned *counts;
    long long *base;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_COUNTS, (size_t)n_seg, &counts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_BASE, (size_t)n_seg, &base))) return rc;
    const uint4 *b = reinterpret_cast<const uint4 *>(bytes);
    xyz_count_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, counts);
    MKB_LAUNCHED(h);
    xyz_scan_kernel<<<1, XL_SCAN_THREADS, 0, st>>>(counts, (int)n_seg, base, reinterpret_cast<long long *>(state));
    MKB_LAUNCHED(h);
    xyz_emit_kernel<INDEX><<<(unsigned)n_seg, XL_THREADS, 0, st>>>(
        b, n, n_read, base, file_base, P, natoms, reinterpret_cast<long long *>(frame_off), status, frame_cap,
        reinterpret_cast<long long *>(state), starts, starts_cap);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

}  // namespace
}  // namespace mkb
