// mdcrd.cu -- K25: AMBER ASCII trajectories (mdcrd / crd / trj, and mdvel) parsed and formatted on the device.
//
// Replaces the host path of an AMBER ASCII trajectory: a reader that turns every 8-character field into a float one by
// one, and the host transposition to the frame-minor (N, 3, F) layout every kernel here consumes.  After a title line,
// a frame holds its 3 N values atom-major (x, y, z of atom 0, then atom 1, ...) as Fortran F8.3 fields, ten to a line;
// value j of a frame starts at byte 8 j + j / 10, a newline follows every value in column 9 (j % 10 == 9) and the
// frame's last value, and a frame with a periodic box ends in one more line of three F8.3 fields (A, B, C) and a
// newline.  Frame bytes: S = 24 N + ceil(3 N / 10) + (box ? 25 : 0).
//
// Mapping: K23's tile (frame_tile.cuh's constants), one CTA of 256 threads per 32 frames x 96 values, the grid's y
// dimension looping over frame tiles.
//   decode  the file side: a warp parses 32 consecutive fields of one frame, each thread a whole field from the three
//           aligned 32-bit words that cover its 8 characters and the byte after them (__byte_perm, SWAR character
//           classes, __dp4a digit sums), then the K23 transposition through shared memory to coalesced stores along
//           frames.  A malformed field or a missing newline atomicMins k * S + its byte into *bad.
//   encode  the array side: a thread loads 12 values along frames (coalesced), formats each into its frame's row of a
//           shared-memory image of the tile's byte span, and the warps store the rows with aligned 32-bit words, byte
//           stores only at the two ragged ends.  A tile owns the bytes of its values, the newline after each of them that
//           ends a line and, for the last value tile, the box line: no two CTAs write the same byte.
//
// Arithmetic (the contract with Python's float() and '%8.3f'; md_parse / md_format in f83.cuh):
//   decode  the digits k of the field (point removed, k < 10^7) give __double2float_rn((double)k / 1000.0), the sign
//           applied afterwards: the double division is correctly rounded like float(), so both round the decimal once
//           to double and once to float32, and '-0.000' gives -0.0.
//   encode  k = rint((double)x * 1000) is exact before the rounding (a float32 times 1000 fits 53 bits) and rounds half
//           to even, which is what printf's correctly rounded '%.3f' does; the sign of x is printed even when k == 0.
#include <algorithm>

#include "common.cuh"
#include "f83.cuh"
#include "frame_tile.cuh"

namespace mkb {
namespace {

constexpr int MD_MAX_SPAN = FT_W * 8 + 10 + 25;  // bytes of one frame in a tile: 96 fields, <= 10 newlines, a box line
constexpr int MD_ROW = 812;                      // image row: the span plus 3 bytes of alignment shift, 203 words (odd)
static_assert(MD_ROW % 4 == 0 && MD_ROW >= MD_MAX_SPAN + 3 && (MD_ROW / 4) % 2 == 1, "image row");

__device__ __forceinline__ long long md_pos(long long j) { return 8 * j + j / 10; }  // byte of value j in its frame

// coords[(a*3 + d)*frame_stride + k] = value a*3 + d of the frame at bytes + offsets[k]; with a box, box[d*box_stride + k]
// = field d of its box line.  Every offset is a multiple of 4.
__global__ void __launch_bounds__(FT_WARPS * 32, 4)
mdcrd_decode_kernel(const unsigned char *__restrict__ bytes, const long long *__restrict__ offsets, int n_frames,
                    int n_vals, int with_box, float *__restrict__ coords, long long frame_stride,
                    float *__restrict__ box, long long box_stride, long long S, unsigned long long *__restrict__ bad) {
    __shared__ unsigned tile[FT_T][FT_W + 1];  // [frame][value]
    __shared__ long long off[FT_T];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int w0 = blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile's reads of `tile` and `off` are done
        if (threadIdx.x < FT_T && k0 + (int)threadIdx.x < n_frames) off[threadIdx.x] = offsets[k0 + threadIdx.x];
        __syncthreads();
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int fl = FT_WARPS * (i / 3) + warp, j = w0 + 32 * (i % 3) + lane;
            unsigned bits = 0;
            if (j < n_vals && k0 + fl < n_frames) {
                const long long p = md_pos(j);
                unsigned lo, hi, next;
                md_field(bytes + off[fl] + p, lo, hi, next);
                bool ok;
                bits = md_parse(lo, hi, ok);
                const long long at = (long long)(k0 + fl) * S + p;
                if (!ok) atomicMin(bad, (unsigned long long)at);
                if ((j % 10 == 9 || j == n_vals - 1) && next != '\n') atomicMin(bad, (unsigned long long)(at + 8));
            }
            tile[fl][j - w0] = bits;
        }
        if (with_box && blockIdx.x == 0 && threadIdx.x < 3 * FT_T) {
            const int d = threadIdx.x >> 5, k = k0 + lane;
            if (k < n_frames) {
                const long long p = md_pos(n_vals - 1) + 9 + 8 * d;
                unsigned lo, hi, next;
                md_field(bytes + off[lane] + p, lo, hi, next);
                bool ok;
                const unsigned bits = md_parse(lo, hi, ok);
                const long long at = (long long)k * S + p;
                if (!ok) atomicMin(bad, (unsigned long long)at);
                if (d == 2 && next != '\n') atomicMin(bad, (unsigned long long)(at + 8));
                reinterpret_cast<unsigned *>(box)[d * box_stride + k] = bits;
            }
        }
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int wl = FT_WARPS * i + warp;
            if (w0 + wl < n_vals && k < n_frames)
                __stcs(reinterpret_cast<unsigned *>(coords) + (long long)(w0 + wl) * frame_stride + k, tile[lane][wl]);
        }
    }
}

// Frame k of out is out[k*S ...]: value a*3 + d from coords[(a*3 + d)*frame_stride + k], with a box the line of
// box[d*box_stride + k].  out is 4-byte aligned.
__global__ void __launch_bounds__(FT_WARPS * 32, 4)
mdcrd_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, int n_vals,
                    const float *__restrict__ box, long long box_stride, long long S, unsigned char *__restrict__ out) {
    __shared__ __align__(16) unsigned char img[FT_T][MD_ROW];  // [frame][the tile's bytes, shifted to out's alignment]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int w0 = blockIdx.x * FT_W, w1 = min(w0 + FT_W, n_vals);
    const bool last = w1 == n_vals;
    const long long b0 = md_pos(w0);
    const int span = (int)(md_pos(w1 - 1) + 8 - b0) + ((w1 - 1) % 10 == 9 || last) + (last && box ? 25 : 0);
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T, k = k0 + lane;
        __syncthreads();  // the previous tile's rows are stored
        float x[FT_ITEMS];
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int j = w0 + FT_WARPS * i + warp;
            x[i] = 0.f;
            if (j < n_vals && k < n_frames) x[i] = __ldcs(coords + (long long)j * frame_stride + k);
        }
        const int shift = (int)(((long long)k * S + b0) & 3);  // out's word alignment of this lane's frame row
        unsigned char *row = img[lane] + shift;                // row[p - b0] = byte p of the frame
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int j = w0 + FT_WARPS * i + warp;
            if (j < n_vals && k < n_frames) {
                unsigned lo, hi;
                md_format(x[i], lo, hi);
                const int p = (int)(md_pos(j) - b0);
                md_put(row + p, lo, hi);
                if (j % 10 == 9 || j == n_vals - 1) row[p + 8] = '\n';
            }
        }
        if (box && last && threadIdx.x < 3 * FT_T && k < n_frames) {
            const int d = threadIdx.x >> 5;
            unsigned lo, hi;
            md_format(__ldcs(box + d * box_stride + k), lo, hi);
            const int p = (int)(md_pos(n_vals - 1) + 9 + 8 * d - b0);
            md_put(row + p, lo, hi);
            if (d == 2) row[p + 8] = '\n';
        }
        __syncthreads();
        for (int r = warp; r < FT_T && k0 + r < n_frames; r += FT_WARPS) {
            const long long g0 = (long long)(k0 + r) * S + b0;
            const int a = (int)(g0 & 3), nw = (a + span + 3) >> 2;
            unsigned *dst = reinterpret_cast<unsigned *>(out + (g0 - a));
            const unsigned *src = reinterpret_cast<const unsigned *>(img[r]);
            for (int m = lane; m < nw; m += 32) {
                if (4 * m >= a && 4 * m + 4 <= a + span) {
                    __stcs(dst + m, src[m]);
                } else {
                    for (int c = max(4 * m, a); c < min(4 * m + 4, a + span); ++c)
                        out[g0 - a + c] = img[r][c];
                }
            }
        }
    }
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_mdcrd_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes,
                                const int64_t *offsets, int64_t n_frames, int64_t natoms, int32_t with_box,
                                float *coords, int64_t frame_stride, float *box, int64_t box_stride, int64_t *bad) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || nbytes < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1) return fail(h, MKB_ERR_BAD_ARG, "natoms must be >= 1, got %lld", (long long)natoms);
    const int64_t S = 24 * natoms + (3 * natoms + 9) / 10 + (with_box ? 25 : 0);
    if (natoms > INT32_MAX / 25 || S > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!bytes || !offsets || !coords || !bad || (with_box && !box)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames || (with_box && box_stride < n_frames))
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(box)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords and box must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(bad) & 7) return fail(h, MKB_ERR_BAD_ARG, "bad must be 8-byte aligned");
    const int64_t words = (S + 3) & ~int64_t(3);  // the kernel reads a frame as whole aligned 32-bit words
    for (int64_t k = 0; k < n_frames; ++k) {
        const int64_t o = offsets[k];
        if (o < 0 || (o & 15) || o > nbytes - words)
            return fail(h, MKB_ERR_BAD_ARG, "offset %lld of frame %lld: the %lld-byte frame must start on a 16-byte "
                        "boundary with its %lld bytes of whole words inside the %lld-byte buffer", (long long)o,
                        (long long)k, (long long)S, (long long)words, (long long)nbytes);
    }
    long long *d_off;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_off))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_off, offsets, sizeof(long long) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(3 * natoms, FT_W), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    mdcrd_decode_kernel<<<grid, FT_WARPS * 32, 0, st>>>(bytes, d_off, (int)n_frames, (int)(3 * natoms), with_box != 0,
                                                        coords, frame_stride, box, box_stride, S,
                                                        reinterpret_cast<unsigned long long *>(bad));
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_mdcrd_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride,
                                int64_t n_frames, int64_t natoms, const float *box, int64_t box_stride, uint8_t *out,
                                int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1) return fail(h, MKB_ERR_BAD_ARG, "natoms must be >= 1, got %lld", (long long)natoms);
    const int64_t S = 24 * natoms + (3 * natoms + 9) / 10 + (box ? 25 : 0);
    if (natoms > INT32_MAX / 25 || S > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!coords || !out) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(box) | reinterpret_cast<uintptr_t>(out)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords, box and out must be 4-byte aligned");
    if (frame_stride < n_frames || (box && box_stride < n_frames))
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (n_frames * S > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * S));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(3 * natoms, FT_W), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    mdcrd_encode_kernel<<<grid, FT_WARPS * 32, 0, st>>>(coords, frame_stride, (int)n_frames, (int)(3 * natoms), box,
                                                        box_stride, S, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
