// xyz.cu -- K26: multi-frame XYZ trajectories indexed, parsed and formatted on the device.
//
// Replaces the host path of an XYZ reader that splits every line and calls float() on every field.  A frame is N + 2
// lines: the atom count, a comment, and N atom lines "element x y z [anything]" with fields of no fixed width, so a
// frame has no fixed size and every line must be found before it can be parsed.
//
//   lines   a newline index over a span of bytes in three launches (xl_lines.cuh, shared with K29): xyz_count_kernel
//           counts the '\n' of every 32 KB segment (SWAR byte masks over 16-byte loads), xyz_scan_kernel (one CTA)
//           turns the counts into each segment's first line number and advances a running line count kept on the
//           device, and xyz_emit_kernel ranks the newlines inside a segment with block scans.  Line L of the span
//           starts after newline L - 1.
//   index   over the file in chunks (mkb_xyz_index): the emit pass keeps only the lines that start a frame (L a multiple
//           of N + 2), records their file offset and checks the count line there against N; a CR that is not followed
//           by LF (a lone CR line ending) is reported by its file offset.  The running line count makes the chunks
//           independent of each other: no host sync per chunk.
//   decode  over staged whole frames (mkb_xyz_decode): the emit pass stores every line start, then xyz_parse_kernel
//           maps K23's tile (32 frames x 32 atoms per CTA of 256 threads): a thread parses one atom line through a
//           16-byte window (xyz_number.cuh) into a shared-memory tile, and the warps store the tile along frames.  A line
//           the device does not decide is appended to a list for the host.
//   encode  the inverse for fixed-size frames (mkb_xyz_encode): a CTA loads 32 frames x 32 atoms along frames, each
//           warp formats one frame's 32 lines into a shared-memory image, and stores it with aligned 32-bit words.
//
// Encode arithmetic ('%-*s %15.8f %15.8f %15.8f'): k = rint((double)x * 1e8) is exact before the rounding (a float32
// times 10^8 needs 43 bits) and rounds half to even, as a correctly rounded printf does; the sign is printed whenever x
// is negative or -0.0.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "frame_tile.cuh"
#include "xl_lines.cuh"
#include "xyz_number.cuh"

namespace mkb {
namespace {

constexpr int XYZ_FIELD = 16;         // ' ' and a '%15.8f' field
constexpr int XYZ_MAX_WIDTH = 256;    // widest element column the encoder takes

// bytes [p, end) of a 16-byte aligned buffer through a 16-byte window; '\n' at and past end
struct XyzReader {
    const uint4 *base;
    long long end;
    long long wi = -1;
    uint4 w;
    __device__ __forceinline__ unsigned at(long long p) {
        if (p >= end) return '\n';
        if ((p >> 4) != wi) {
            wi = p >> 4;
            w = __ldg(base + wi);
        }
        const unsigned q = (p & 8) ? ((p & 4) ? w.w : w.z) : ((p & 4) ? w.y : w.x);
        return (q >> (8 * (p & 3))) & 0xffu;
    }
};

// coords[(a*3 + d)*frame_stride + k] = field d + 1 of atom line a of listed frame k, staged frame frame_of[k] (lines
// starts[P u + 2 + a] ... of the staged bytes).  An undecided line appends ((frame_base + k) * natoms + a, its byte
// offset from its frame's first byte) to flags[1 ...] (flags[0] counts them; entries past flag_cap are dropped).
__global__ void __launch_bounds__(FT_WARPS * 32)
xyz_parse_kernel(const uint4 *__restrict__ bytes, long long nbytes, const long long *__restrict__ starts,
                 long long n_lines, const int *__restrict__ frame_of, int n_frames, int natoms, long long P,
                 float *__restrict__ coords, long long frame_stride, long long frame_base,
                 unsigned long long *__restrict__ flags, long long flag_cap) {
    __shared__ unsigned tile[FT_W][FT_T + 1];  // [value][frame]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a = blockIdx.x * 32 + lane, v0 = blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile is stored
#pragma unroll
        for (int j = 0; j < FT_T / FT_WARPS; ++j) {
            const int fl = warp + FT_WARPS * j, k = k0 + fl;
            unsigned x = 0u, y = 0u, z = 0u;
            if (k < n_frames && a < natoms) {
                const long long first = P * frame_of[k], li = first + 2 + a;
                const long long s = min(max(starts[li], 0LL), nbytes);
                const long long e = min(max(li + 1 < n_lines ? starts[li + 1] : nbytes, s), nbytes);
                XyzReader rd{bytes, e};
                if (!xyz_atom_line(rd, s, x, y, z)) {
                    const unsigned long long slot = atomicAdd(flags, 1ull);
                    if ((long long)slot < flag_cap) {
                        flags[1 + 2 * slot] = (unsigned long long)((frame_base + k) * natoms + a);
                        flags[2 + 2 * slot] = (unsigned long long)(s - starts[first]);
                    }
                }
            }
            tile[3 * lane][fl] = x;
            tile[3 * lane + 1][fl] = y;
            tile[3 * lane + 2][fl] = z;
        }
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int r = warp + FT_WARPS * i;
            if (v0 + r < 3 * natoms && k < n_frames)
                __stcs(reinterpret_cast<unsigned *>(coords) + (long long)(v0 + r) * frame_stride + k, tile[r][lane]);
        }
    }
}

// ' ' and '%15.8f' of x into d[0 .. 16); the caller has checked the range (|rint(x 1e8)| < 10^14, 10^13 when negative)
__device__ __forceinline__ void xyz_format(float x, unsigned char *d) {
    const bool neg = signbit(x);
    const unsigned long long k = (unsigned long long)fabs(rint((double)x * 1e8));
    unsigned ip = (unsigned)(k / 100000000ull), fp = (unsigned)(k - 100000000ull * ip);
#pragma unroll
    for (int c = 15; c >= 8; --c) {
        d[c] = (unsigned char)('0' + fp % 10u);
        fp /= 10u;
    }
    d[7] = '.';
    int c = 6;
    do {
        d[c--] = (unsigned char)('0' + ip % 10u);
        ip /= 10u;
    } while (ip && c >= 0);
    if (neg && c >= 0) d[c--] = '-';
    for (; c >= 0; --c) d[c] = ' ';
}

// Frame k of out is out[k*S ...], S = head_bytes + natoms*(width + 49): the head (count and comment lines), then per
// atom its width-byte element column from elements[a*width ...] and the three fields of coords[(a*3 + d)*frame_stride
// + k], and '\n'.  out is 4-byte aligned.  Dynamic shared memory: FT_WARPS images of 32 lines + 8 bytes.
__global__ void __launch_bounds__(FT_WARPS * 32)
xyz_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, int natoms,
                  const unsigned char *__restrict__ head, int head_bytes, const unsigned char *__restrict__ elements,
                  int width, long long S, unsigned char *__restrict__ out) {
    __shared__ float tile[FT_W][FT_T + 1];  // [value][frame]
    extern __shared__ __align__(16) unsigned char img_all[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int L = width + 1 + 3 * XYZ_FIELD, row = (32 * L + 8 + 15) & ~15;
    unsigned char *img = img_all + warp * row;
    const int a0 = blockIdx.x * 32, v0 = blockIdx.x * FT_W, na = min(32, natoms - a0);
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile is formatted
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int r = warp + FT_WARPS * i, k = k0 + lane;
            tile[r][lane] = v0 + r < 3 * natoms && k < n_frames
                                ? __ldcs(coords + (long long)(v0 + r) * frame_stride + k) : 0.f;
        }
        __syncthreads();
        for (int j = 0; j < FT_T / FT_WARPS; ++j) {
            const int fl = warp + FT_WARPS * j, k = k0 + fl;
            if (k >= n_frames) break;
            if (blockIdx.x == 0)  // the frame's head
                for (int c = lane; c < head_bytes; c += 32) out[(long long)k * S + c] = head[c];
            const long long g0 = (long long)k * S + head_bytes + (long long)a0 * L;
            const int sh = (int)(g0 & 3), span = na * L;
            if (lane < na) {
                unsigned char *d = img + sh + lane * L;
                const unsigned char *e = elements + (long long)(a0 + lane) * width;
                for (int c = 0; c < width; ++c) d[c] = __ldg(e + c);
#pragma unroll
                for (int x = 0; x < 3; ++x) xyz_format(tile[3 * lane + x][fl], d + width + XYZ_FIELD * x);
                d[L - 1] = '\n';
            }
            __syncwarp();
            unsigned *dst = reinterpret_cast<unsigned *>(out + (g0 - sh));
            const unsigned *src = reinterpret_cast<const unsigned *>(img);
            for (int m = lane; m < (sh + span + 3) >> 2; m += 32) {
                if (4 * m >= sh && 4 * m + 4 <= sh + span) {
                    __stcs(dst + m, src[m]);
                } else {
                    for (int c = max(4 * m, sh); c < min(4 * m + 4, sh + span); ++c) out[g0 - sh + c] = img[c];
                }
            }
            __syncwarp();  // the image is stored before the next frame overwrites it
        }
    }
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_xyz_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                             int64_t file_base, int64_t natoms, int64_t *state, int64_t *frame_off, uint8_t *status,
                             int64_t frame_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n < 0 || n_read < n || file_base < 0 || frame_cap < 0) return fail(h, MKB_ERR_BAD_ARG, "bad size");
    if (natoms < 1 || natoms > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to 2^31 - 1");
    if (!bytes || !state || (frame_cap && (!frame_off || !status))) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(state) & 7) return fail(h, MKB_ERR_BAD_ARG, "state must be 8-byte aligned");
    if (n == 0) return MKB_OK;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    int rc = xyz_lines<true>(h, st, bytes, n, n_read, file_base, natoms + 2, natoms, frame_off, status, frame_cap,
                             state, nullptr, 0);
    if (rc) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_xyz_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                              const int32_t *frame_of, int64_t n_frames, int64_t natoms, float *coords,
                              int64_t frame_stride, int64_t frame_base, int64_t *flags, int64_t flag_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || n_staged < 0 || nbytes < 0 || frame_base < 0 || flag_cap < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!bytes || !frame_of || !coords || !flags) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(coords) & 3) || (reinterpret_cast<uintptr_t>(flags) & 7))
        return fail(h, MKB_ERR_BAD_ARG, "coords must be 4-byte and flags 8-byte aligned");
    for (int64_t k = 0; k < n_frames; ++k)
        if (frame_of[k] < 0 || frame_of[k] >= n_staged)
            return fail(h, MKB_ERR_BAD_ARG, "frame_of[%lld] = %d is not a staged frame (%lld staged)", (long long)k,
                        (int)frame_of[k], (long long)n_staged);
    const int64_t P = natoms + 2, n_lines = n_staged * P;
    long long *starts, *state;
    int *d_map;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_STARTS, (size_t)n_lines + 1, &starts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_STATE, 1, &state))) return rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_map))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_map, frame_of, sizeof(int) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(state, 0, sizeof(long long), st));
    if ((rc = xyz_lines<false>(h, st, bytes, nbytes, nbytes, 0, P, natoms, nullptr, nullptr, 0,
                               reinterpret_cast<int64_t *>(state), starts, n_lines + 1)))
        return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    xyz_parse_kernel<<<grid, FT_WARPS * 32, 0, st>>>(reinterpret_cast<const uint4 *>(bytes), nbytes, starts, n_lines,
                                                     d_map, (int)n_frames, (int)natoms, P, coords, frame_stride,
                                                     frame_base, reinterpret_cast<unsigned long long *>(flags),
                                                     flag_cap);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_xyz_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride,
                              int64_t n_frames, int64_t natoms, const uint8_t *head, int64_t head_bytes,
                              const uint8_t *elements, int64_t width, uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || head_bytes < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (width < 1 || width > XYZ_MAX_WIDTH)
        return fail(h, MKB_ERR_BAD_ARG, "element width must be 1 to %d, got %lld", XYZ_MAX_WIDTH, (long long)width);
    if (head_bytes > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "head too long");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!coords || !elements || !out || (head_bytes && !head)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(out)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords and out must be 4-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const int64_t L = width + 1 + 3 * XYZ_FIELD, S = head_bytes + natoms * L;
    if (n_frames * S > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * S));
    const size_t smem = (size_t)FT_WARPS * ((32 * L + 8 + 15) & ~15);
    MKB_CUDA(h, cudaFuncSetAttribute(xyz_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    xyz_encode_kernel<<<grid, FT_WARPS * 32, smem, st>>>(coords, frame_stride, (int)n_frames, (int)natoms, head,
                                                          (int)head_bytes, elements, (int)width, S, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
