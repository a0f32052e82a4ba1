// netcdf.cu -- K23: AMBER NetCDF trajectory records read and written on the device.
//
// Replaces the host path of an AMBER trajectory: a netCDF-3 reader (moleculekit/fileformats/netcdf.py) that returns the
// big-endian `coordinates` variable as (F, N, 3), and the host transposition to the frame-minor (N, 3, F) layout every
// kernel here consumes.  In the file, frame k's coordinates are 12 * natoms contiguous big-endian bytes (atom-major,
// the three axes of an atom interleaved) inside record k, so the whole job is a byte swap and a transposition of the
// (frame, atom * 3 + axis) plane: the (atom, axis) pairs form one flat dimension of 3 * natoms words.
//
// The tile transposition is frame_tile.cuh's (shared with K24): 32 frames x 96 words per CTA, values moved as 32-bit
// words through __byte_perm, so every bit pattern (NaN payloads, signalling NaNs, -0.0, subnormals) survives.  12 bytes
// read and 12 written per atom-frame: the roofline is HBM bandwidth.
#include <algorithm>

#include "common.cuh"
#include "frame_tile.cuh"

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
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
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
    const dim3 grid((unsigned)cdiv(natoms, FT_T), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    frame_tile_decode_kernel<4><<<grid, FT_WARPS * 32, 0, st>>>(bytes, d_off, (int)n_frames, 3 * natoms, coords, frame_stride);
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
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    const int64_t slab = 12 * natoms;
    if ((record_bytes & 3) || (coord_offset & 3) || coord_offset + slab > record_bytes)
        return fail(h, MKB_ERR_BAD_ARG, "record_bytes (%lld) and coord_offset (%lld) must be multiples of 4 with "
                    "coord_offset + %lld coordinate bytes <= record_bytes", (long long)record_bytes,
                    (long long)coord_offset, (long long)slab);
    const int64_t extra_bytes = record_bytes - slab;
    if (extra_bytes / 4 > INT32_MAX / FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many extra bytes per record");
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
    const dim3 grid((unsigned)std::max<int64_t>(cdiv(natoms, FT_T), 1),
                    (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    frame_tile_encode_kernel<1><<<grid, FT_WARPS * 32, 0, st>>>(coords, frame_stride, (int)n_frames, 3 * natoms,
                                                                reinterpret_cast<const unsigned *>(extra),
                                                                (int)(extra_bytes / 4), (int)(coord_offset / 4),
                                                                reinterpret_cast<unsigned *>(out), record_bytes / 4,
                                                                nullptr, 0, nullptr, 0);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
