// netcdf.cu -- K23: AMBER NetCDF trajectory records read and written on the device.
//
// Replaces the host path of an AMBER trajectory: a netCDF-3 reader (moleculekit/fileformats/netcdf.py) that returns the
// big-endian `coordinates` variable as (F, N, 3), and the host transposition to the frame-minor (N, 3, F) layout every
// kernel here consumes.  In the file, frame k's coordinates are 12 * natoms contiguous big-endian bytes (atom-major,
// the three axes of an atom interleaved) inside record k, so the whole job is a byte swap and a transposition of the
// (frame, atom * 3 + axis) plane: the (atom, axis) pairs form one flat dimension of 3 * natoms words.
//
// Mapping: one CTA of 256 threads (8 warps) owns a tile of 32 frames x 96 words (32 atoms x 3 axes), staged in shared
// memory as [frame][word] rows of 97 words: on the file side a warp moves 32 consecutive words of one frame (row writes,
// conflict-free), on the array side a warp moves 32 consecutive frames of one (atom, axis) row (column reads, stride 97,
// odd, conflict-free).  Each thread moves 12 words each way with all 12 loads issued before the first shared-memory
// store.  Values travel as 32-bit words through __byte_perm and never through float arithmetic, so every bit pattern
// (NaN payloads, signalling NaNs, -0.0, subnormals) survives.  12 bytes read and 12 written per atom-frame: the roofline
// is HBM bandwidth.
#include <algorithm>

#include "common.cuh"

namespace mkb {

constexpr int NC_T = 32;                           // frames and atoms per tile
constexpr int NC_W = 3 * NC_T;                     // words of one frame in a tile
constexpr int NC_WARPS = 8;                        // 256 threads
constexpr int NC_ITEMS = NC_T * NC_W / (32 * NC_WARPS);  // 12 words per thread each way
static_assert(NC_ITEMS == 12 && NC_W == 3 * 32, "file side: item i covers frame NC_WARPS * (i / 3) + warp, words 32 * (i % 3) + lane");
constexpr int NC_MAX_GRID_Y = 65535;

__device__ __forceinline__ unsigned nc_swap(unsigned w) { return __byte_perm(w, 0, 0x0123); }

// coords[(a*3 + d)*frame_stride + k] = big-endian word a*3 + d of the coordinate slab at bytes + offsets[k]
__global__ void __launch_bounds__(NC_WARPS * 32, 4)
netcdf_decode_kernel(const unsigned char *__restrict__ bytes, const long long *__restrict__ offsets, int n_frames,
                     long long n_words, float *__restrict__ coords, long long frame_stride) {
    __shared__ unsigned tile[NC_T][NC_W + 1];  // [frame][word]
    __shared__ long long off[NC_T];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long w0 = (long long)blockIdx.x * NC_W;
    const int n_ft = (n_frames + NC_T - 1) / NC_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * NC_T;
        __syncthreads();  // the previous tile's reads of `tile` and `off` are done
        if (threadIdx.x < NC_T && k0 + (int)threadIdx.x < n_frames) off[threadIdx.x] = offsets[k0 + threadIdx.x];
        __syncthreads();
        unsigned w[NC_ITEMS];
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) {
            const int fl = NC_WARPS * (i / 3) + warp, wl = 32 * (i % 3) + lane;
            w[i] = 0;
            if (w0 + wl < n_words && k0 + fl < n_frames)
                w[i] = __ldcs(reinterpret_cast<const unsigned *>(bytes + off[fl]) + w0 + wl);
        }
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) tile[NC_WARPS * (i / 3) + warp][32 * (i % 3) + lane] = nc_swap(w[i]);
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) {
            const int wl = NC_WARPS * i + warp;
            if (w0 + wl < n_words && k < n_frames)
                __stcs(reinterpret_cast<unsigned *>(coords) + (w0 + wl) * frame_stride + k, tile[lane][wl]);
        }
    }
}

// Record k of the output is out[k*record_words ...]: the big-endian coordinates at word coord_word, the frame's
// `extra_words` words of extra (already in file byte order) around them -- those before coord_word first, the rest after
// the coordinates.  The CTAs of the first atom tile copy the extra words of their frames.
__global__ void __launch_bounds__(NC_WARPS * 32, 4)
netcdf_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, long long n_words,
                     const unsigned *__restrict__ extra, int extra_words, int coord_word, unsigned *__restrict__ out,
                     long long record_words) {
    __shared__ unsigned tile[NC_T][NC_W + 1];  // [frame][word]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long w0 = (long long)blockIdx.x * NC_W;
    const int n_ft = (n_frames + NC_T - 1) / NC_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * NC_T;
        __syncthreads();  // the previous tile's reads of `tile` are done
        const int k = k0 + lane;
        unsigned w[NC_ITEMS];
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) {
            const int wl = NC_WARPS * i + warp;
            w[i] = 0;
            if (w0 + wl < n_words && k < n_frames)
                w[i] = __ldcs(reinterpret_cast<const unsigned *>(coords) + (w0 + wl) * frame_stride + k);
        }
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) tile[lane][NC_WARPS * i + warp] = w[i];
        __syncthreads();
#pragma unroll
        for (int i = 0; i < NC_ITEMS; ++i) {
            const int fl = NC_WARPS * (i / 3) + warp, wl = 32 * (i % 3) + lane;
            if (w0 + wl < n_words && k0 + fl < n_frames)
                __stcs(out + (long long)(k0 + fl) * record_words + coord_word + w0 + wl, nc_swap(tile[fl][wl]));
        }
        if (blockIdx.x == 0) {
            const int n_tile = min(NC_T, n_frames - k0);
            for (int t = threadIdx.x; t < n_tile * extra_words; t += NC_WARPS * 32) {
                const int fl = t / extra_words, j = t - fl * extra_words;
                const long long kk = k0 + fl;
                out[kk * record_words + (j < coord_word ? j : j + n_words)] = extra[kk * extra_words + j];
            }
        }
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_netcdf_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes,
                                 const int64_t *offsets, int64_t n_frames, int64_t natoms, float *coords,
                                 int64_t frame_stride) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || nbytes < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0 || natoms == 0) return MKB_OK;
    if (!bytes || !offsets || !coords) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (natoms > INT32_MAX / 12) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - NC_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 3) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(coords) & 3) return fail(h, MKB_ERR_BAD_ARG, "coords must be 4-byte aligned");
    const int64_t slab = 12 * natoms;
    for (int64_t k = 0; k < n_frames; ++k) {
        const int64_t o = offsets[k];
        if (o < 0 || (o & 3) || o > nbytes - slab)
            return fail(h, MKB_ERR_BAD_ARG, "offset %lld of frame %lld: the %lld coordinate bytes must start on a 4-byte "
                        "boundary inside the %lld-byte buffer", (long long)o, (long long)k, (long long)slab,
                        (long long)nbytes);
    }
    long long *d_off;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_off))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_off, offsets, sizeof(long long) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, NC_T), (unsigned)std::min<int64_t>(cdiv(n_frames, NC_T), NC_MAX_GRID_Y));
    netcdf_decode_kernel<<<grid, NC_WARPS * 32, 0, st>>>(bytes, d_off, (int)n_frames, 3 * natoms, coords, frame_stride);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_netcdf_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride,
                                 int64_t n_frames, int64_t natoms, int64_t record_bytes, int64_t coord_offset,
                                 const uint8_t *extra, uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0 || record_bytes < 0 || coord_offset < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (natoms > INT32_MAX / 12) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - NC_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    const int64_t slab = 12 * natoms;
    if ((record_bytes & 3) || (coord_offset & 3) || coord_offset + slab > record_bytes)
        return fail(h, MKB_ERR_BAD_ARG, "record_bytes (%lld) and coord_offset (%lld) must be multiples of 4 with "
                    "coord_offset + %lld coordinate bytes <= record_bytes", (long long)record_bytes,
                    (long long)coord_offset, (long long)slab);
    const int64_t extra_bytes = record_bytes - slab;
    if (extra_bytes / 4 > INT32_MAX / NC_T) return fail(h, MKB_ERR_BAD_ARG, "too many extra bytes per record");
    if (n_frames == 0) return MKB_OK;
    if (!out || (natoms && !coords) || (extra_bytes && !extra)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(out) & 3) return fail(h, MKB_ERR_BAD_ARG, "out must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(extra) & 3) return fail(h, MKB_ERR_BAD_ARG, "extra must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(coords) & 3) return fail(h, MKB_ERR_BAD_ARG, "coords must be 4-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (n_frames * record_bytes > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the records take %lld", (long long)out_capacity,
                    (long long)(n_frames * record_bytes));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    // natoms == 0 still has the extra bytes to copy: one atom tile
    const dim3 grid((unsigned)std::max<int64_t>(cdiv(natoms, NC_T), 1),
                    (unsigned)std::min<int64_t>(cdiv(n_frames, NC_T), NC_MAX_GRID_Y));
    netcdf_encode_kernel<<<grid, NC_WARPS * 32, 0, st>>>(coords, frame_stride, (int)n_frames, 3 * natoms,
                                                           reinterpret_cast<const unsigned *>(extra),
                                                           (int)(extra_bytes / 4), (int)(coord_offset / 4),
                                                           reinterpret_cast<unsigned *>(out), record_bytes / 4);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
