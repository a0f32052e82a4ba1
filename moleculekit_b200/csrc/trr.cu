// trr.cu -- K24: GROMACS TRR trajectory records read and written on the device.
//
// Replaces the host path of a TRR trajectory: xdrfile's read_trr (moleculekit/fileformats/xtc/trr.pyx over the vendored
// xdrfile_trr.c), which returns each frame's x, v and f as (N, 3) reals, and the host transposition to the frame-minor
// (N, 3, F) layout every kernel here consumes.  In the file, a frame's x, v and f blocks are each 3 * natoms contiguous
// big-endian XDR reals (atom-major, the three axes of an atom interleaved), float32 or -- from a double-precision GROMACS
// build -- float64, so decoding is a byte swap and a transposition of the (frame, atom * 3 + axis) plane, plus a rounding
// to float32 for 8-byte reals.  The tile code is frame_tile.cuh's, shared with K23: the 4-byte decode is K23's kernel,
// the 8-byte decode the same tile with one 64-bit load and one cvtsd2ss-exact conversion per value, and the encoder
// K23's with up to three source arrays per record (x, v, f).
#include <algorithm>

#include "common.cuh"
#include "frame_tile.cuh"

using namespace mkb;

extern "C" int mkb_trr_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const int64_t *offsets,
                              int64_t n_frames, int64_t natoms, int32_t value_bytes, float *coords,
                              int64_t frame_stride) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || nbytes < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (value_bytes != 4 && value_bytes != 8)
        return fail(h, MKB_ERR_BAD_ARG, "value_bytes must be 4 or 8, got %d", (int)value_bytes);
    if (n_frames == 0 || natoms == 0) return MKB_OK;
    if (!bytes || !offsets || !coords) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (natoms > INT32_MAX / (3 * value_bytes)) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & (value_bytes - 1))
        return fail(h, MKB_ERR_BAD_ARG, "bytes must be %d-byte aligned", (int)value_bytes);
    if (reinterpret_cast<uintptr_t>(coords) & 3) return fail(h, MKB_ERR_BAD_ARG, "coords must be 4-byte aligned");
    const int64_t slab = 3 * natoms * value_bytes;
    for (int64_t k = 0; k < n_frames; ++k) {
        const int64_t o = offsets[k];
        if (o < 0 || (o & (value_bytes - 1)) || o > nbytes - slab)
            return fail(h, MKB_ERR_BAD_ARG, "offset %lld of frame %lld: the %lld bytes of %d-byte reals must start on a "
                        "%d-byte boundary inside the %lld-byte buffer", (long long)o, (long long)k, (long long)slab,
                        (int)value_bytes, (int)value_bytes, (long long)nbytes);
    }
    long long *d_off;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_off))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_off, offsets, sizeof(long long) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, FT_T), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    if (value_bytes == 4)
        frame_tile_decode_kernel<4><<<grid, FT_WARPS * 32, 0, st>>>(bytes, d_off, (int)n_frames, 3 * natoms, coords,
                                                                    frame_stride);
    else
        frame_tile_decode_kernel<8><<<grid, FT_WARPS * 32, 0, st>>>(bytes, d_off, (int)n_frames, 3 * natoms, coords,
                                                                    frame_stride);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_trr_encode(mkb_handle_t h, void *stream, const float *x, const float *v, const float *f,
                              int64_t frame_stride, int64_t n_frames, int64_t natoms, const uint8_t *head,
                              int64_t head_bytes, uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0 || head_bytes < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (natoms > INT32_MAX / 12) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (head_bytes & 3) return fail(h, MKB_ERR_BAD_ARG, "head_bytes (%lld) must be a multiple of 4", (long long)head_bytes);
    if (head_bytes / 4 > INT32_MAX / FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many head bytes per record");
    const int n_src = 1 + (v != nullptr) + (f != nullptr);
    const int64_t slab = 12 * natoms, record_bytes = head_bytes + n_src * slab;
    if (n_frames == 0) return MKB_OK;
    if (!out || (natoms && !x) || (head_bytes && !head)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    for (const void *p : {(const void *)x, (const void *)v, (const void *)f, (const void *)head, (const void *)out})
        if (reinterpret_cast<uintptr_t>(p) & 3)
            return fail(h, MKB_ERR_BAD_ARG, "x, v, f, head and out must be 4-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (n_frames * record_bytes > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the records take %lld", (long long)out_capacity,
                    (long long)(n_frames * record_bytes));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    // the arrays given, in file order; natoms == 0 still has the head bytes to copy: one atom tile
    const float *src[3] = {x, v ? v : f, v ? f : nullptr};
    const dim3 grid((unsigned)std::max<int64_t>(cdiv(natoms, FT_T), 1),
                    (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    const unsigned *hw = reinterpret_cast<const unsigned *>(head);
    unsigned *ow = reinterpret_cast<unsigned *>(out);
    const int hwords = (int)(head_bytes / 4);
    if (n_src == 1)
        frame_tile_encode_kernel<1><<<grid, FT_WARPS * 32, 0, st>>>(src[0], frame_stride, (int)n_frames, 3 * natoms, hw,
                                                                    hwords, hwords, ow, record_bytes / 4, nullptr, 0,
                                                                    nullptr, 0);
    else if (n_src == 2)
        frame_tile_encode_kernel<2><<<grid, FT_WARPS * 32, 0, st>>>(src[0], frame_stride, (int)n_frames, 3 * natoms, hw,
                                                                    hwords, hwords, ow, record_bytes / 4, src[1],
                                                                    frame_stride, nullptr, 0);
    else
        frame_tile_encode_kernel<3><<<grid, FT_WARPS * 32, 0, st>>>(src[0], frame_stride, (int)n_frames, 3 * natoms, hw,
                                                                    hwords, hwords, ow, record_bytes / 4, src[1],
                                                                    frame_stride, src[2], frame_stride);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
