// dcd.cu -- K22: DCD (CHARMM / NAMD / OpenMM) frame records read and written on the device.
//
// Replaces the per-frame fread and X/Y/Z -> xyz interleave of the VMD molfile DCD plugin (read_charmm_timestep /
// write_dcdstep of moleculekit/fileformats/dcd/src/dcdplugin.c) and the host transposition from frame-major (F, N, 3) to
// the frame-minor (N, 3, F) layout every kernel here consumes.  A DCD frame is three records of float32 (X, Y, Z), so
// the file is the trajectory in (F, 3, N) order: the whole job is a transposition of the (frame, atom) plane per axis.
//
// Mapping: one CTA of 256 threads (8 warps) owns a tile of 32 frames x 32 atoms x 3 axes, staged in shared memory as
// 32-bit words (padded rows: conflict-free both ways).  On the file side a warp moves 32 consecutive floats of one
// record of one frame; on the array side a warp moves 32 consecutive frames of one (atom, axis) row.  Each thread moves
// 12 words each way with all 12 loads issued before the first shared-memory store.  Values travel as 32-bit words and
// never pass through float arithmetic, so every bit pattern (NaN payloads, -0.0) survives; the only operation on them
// is the optional byte swap.  12 bytes read and 12 written per atom-frame: the roofline is HBM bandwidth.
#include <algorithm>

#include "common.cuh"

namespace mkb {

struct DcdFrame {
    long long off[3];  // byte offsets of the X, Y, Z float arrays
    long long count;   // floats per record
};
static_assert(sizeof(DcdFrame) == sizeof(mkb_dcd_frame) && sizeof(DcdFrame) == 32, "frame descriptor layout");

constexpr int DCD_T = 32;                         // frames and atoms per tile
constexpr int DCD_WARPS = 8;                      // 256 threads
constexpr int DCD_ITEMS = 3 * DCD_T / DCD_WARPS;  // 12 words per thread each way
static_assert(DCD_ITEMS == 12 && DCD_T == 4 * DCD_WARPS, "item i covers axis i / 4, row DCD_WARPS * (i % 4) + warp");
constexpr int DCD_MAX_GRID_Y = 65535;

inline int64_t dcd_frame_bytes(int64_t natoms, bool with_unitcell) { return (with_unitcell ? 56 : 0) + 3 * (8 + 4 * natoms); }

__device__ __forceinline__ unsigned dcd_swap(unsigned w, bool swap) { return swap ? __byte_perm(w, 0, 0x0123) : w; }

// coords[(a*3 + d)*frame_stride + k] = record d of listed frame k, atom a.  Fixed atoms (slot != NULL): a record of
// `natoms` floats is indexed by atom; a shorter one (the free atoms of a later file frame) by slot[a], and an atom with
// slot[a] < 0 comes from the file's first frame, `first` at `first_bytes`.
__global__ void __launch_bounds__(DCD_WARPS * 32, 4)
dcd_decode_kernel(const unsigned char *__restrict__ bytes, const DcdFrame *__restrict__ frames, int n_frames, int natoms,
                  const int *__restrict__ slot, const unsigned char *__restrict__ first_bytes, DcdFrame first, bool swap,
                  float *__restrict__ coords, long long frame_stride) {
    __shared__ unsigned tile[3][DCD_T][DCD_T + 1];  // [axis][frame][atom]
    __shared__ DcdFrame desc[DCD_T];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a0 = blockIdx.x * DCD_T;
    const int n_ft = (n_frames + DCD_T - 1) / DCD_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * DCD_T;
        __syncthreads();  // the previous tile's reads of `tile` and `desc` are done
        if (threadIdx.x < DCD_T && k0 + (int)threadIdx.x < n_frames) desc[threadIdx.x] = frames[k0 + threadIdx.x];
        __syncthreads();
        const int a = a0 + lane;
        int s = -1;
        if (slot && a < natoms) s = slot[a];
        unsigned w[DCD_ITEMS];
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            const int d = i / 4, fl = DCD_WARPS * (i % 4) + warp;
            w[i] = 0;
            if (a < natoms && k0 + fl < n_frames) {
                const DcdFrame &fr = desc[fl];
                const unsigned *src;
                if (fr.count == natoms) src = reinterpret_cast<const unsigned *>(bytes + fr.off[d]) + a;
                else if (s >= 0) src = reinterpret_cast<const unsigned *>(bytes + fr.off[d]) + s;
                else src = reinterpret_cast<const unsigned *>(first_bytes + first.off[d]) + a;
                w[i] = __ldcs(src);
            }
        }
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            tile[i / 4][DCD_WARPS * (i % 4) + warp][lane] = dcd_swap(w[i], swap);
        }
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            const int d = i / 4, al = DCD_WARPS * (i % 4) + warp, ar = a0 + al;
            if (ar < natoms && k < n_frames)
                __stcs(reinterpret_cast<unsigned *>(coords) + ((long long)ar * 3 + d) * frame_stride + k, tile[d][lane][al]);
        }
    }
}

// Frame k of the output starts at word k*frame_words: [48, unit cell (6 doubles), 48] when `unitcell`, then for each axis
// [4N, N floats, 4N].  The CTAs of the first atom tile also write the markers and the unit cell of their frames.
__global__ void __launch_bounds__(DCD_WARPS * 32, 4)
dcd_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, int natoms,
                  const double *__restrict__ unitcell, unsigned *__restrict__ out, long long frame_words) {
    __shared__ unsigned tile[3][DCD_T][DCD_T + 1];  // [axis][frame][atom]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a0 = blockIdx.x * DCD_T;
    const int n_ft = (n_frames + DCD_T - 1) / DCD_T;
    const int head = unitcell ? 14 : 0;          // words of the unit-cell record
    const long long rec = 2 + (long long)natoms;  // words of one coordinate record with its markers
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * DCD_T;
        __syncthreads();  // the previous tile's reads of `tile` are done
        const int k = k0 + lane;
        unsigned w[DCD_ITEMS];
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            const int d = i / 4, al = DCD_WARPS * (i % 4) + warp, a = a0 + al;
            w[i] = 0;
            if (a < natoms && k < n_frames)
                w[i] = __ldcs(reinterpret_cast<const unsigned *>(coords) + ((long long)a * 3 + d) * frame_stride + k);
        }
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            tile[i / 4][lane][DCD_WARPS * (i % 4) + warp] = w[i];
        }
        __syncthreads();
        const int a = a0 + lane;
#pragma unroll
        for (int i = 0; i < DCD_ITEMS; ++i) {
            const int d = i / 4, fl = DCD_WARPS * (i % 4) + warp;
            if (a < natoms && k0 + fl < n_frames)
                __stcs(out + (long long)(k0 + fl) * frame_words + head + d * rec + 1 + a, tile[d][fl][lane]);
        }
        if (blockIdx.x == 0 && threadIdx.x < DCD_T && k < n_frames) {
            unsigned *f = out + (long long)k * frame_words;
            if (unitcell) {
                const unsigned *uc = reinterpret_cast<const unsigned *>(unitcell + 6 * (long long)k);
                f[0] = f[13] = 48u;
#pragma unroll
                for (int j = 0; j < 12; ++j) f[1 + j] = uc[j];
            }
            const unsigned marker = 4u * (unsigned)natoms;
#pragma unroll
            for (int d = 0; d < 3; ++d) f[head + d * rec] = f[head + d * rec + rec - 1] = marker;
        }
    }
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_dcd_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, const mkb_dcd_frame *frames,
                              int64_t n_frames, int64_t natoms, const int32_t *slot, int64_t n_free,
                              const uint8_t *first_bytes, int64_t first_nbytes, const mkb_dcd_frame *first, int32_t swap,
                              float *coords, int64_t frame_stride) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || nbytes < 0 || n_free < 0 || first_nbytes < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0 || natoms == 0) return MKB_OK;
    if (!bytes || !frames || !coords) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (natoms >= (1ll << 31) / 4) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - DCD_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 3) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 4-byte aligned");
    const bool fixed = slot != nullptr;
    if (fixed) {
        if (!first || !first_bytes) return fail(h, MKB_ERR_BAD_ARG, "fixed atoms need the first frame");
        if (n_free >= natoms) return fail(h, MKB_ERR_BAD_ARG, "n_free must be below natoms when atoms are fixed");
        if (reinterpret_cast<uintptr_t>(first_bytes) & 3) return fail(h, MKB_ERR_BAD_ARG, "first_bytes must be 4-byte aligned");
    }
    // every record must lie inside its buffer, on a 4-byte boundary, and hold natoms floats (or n_free with fixed atoms)
    auto bad_record = [](const mkb_dcd_frame &fr, int64_t size) {
        for (int d = 0; d < 3; ++d)
            if (fr.offset[d] < 0 || (fr.offset[d] & 3) || fr.offset[d] > size - 4 * fr.count) return true;
        return false;
    };
    for (int64_t k = 0; k < n_frames; ++k) {
        const mkb_dcd_frame &fr = frames[k];
        if (!(fr.count == natoms || (fixed && fr.count == n_free)) || bad_record(fr, nbytes))
            return fail(h, MKB_ERR_BAD_ARG, "frame descriptor %lld: bad record count or offset", (long long)k);
    }
    DcdFrame first_d{};
    if (fixed) {
        if (first->count != natoms || bad_record(*first, first_nbytes))
            return fail(h, MKB_ERR_BAD_ARG, "first-frame descriptor: bad record count or offset");
        for (int d = 0; d < 3; ++d) first_d.off[d] = first->offset[d];
        first_d.count = first->count;
    }
    DcdFrame *d_frames;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_frames))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_frames, frames, sizeof(DcdFrame) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, DCD_T), (unsigned)std::min<int64_t>(cdiv(n_frames, DCD_T), DCD_MAX_GRID_Y));
    dcd_decode_kernel<<<grid, DCD_WARPS * 32, 0, st>>>(bytes, d_frames, (int)n_frames, (int)natoms, slot, first_bytes,
                                                        first_d, swap != 0, coords, frame_stride);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_dcd_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                              int64_t natoms, const double *unitcell, uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (natoms > INT32_MAX / 4) return fail(h, MKB_ERR_BAD_ARG, "natoms beyond the int32 record markers");
    if (n_frames >= (1ll << 31) - DCD_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    const int64_t frame_bytes = dcd_frame_bytes(natoms, unitcell != nullptr);
    if (n_frames == 0) return MKB_OK;
    if (!out || (natoms && !coords)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(out) & 3) return fail(h, MKB_ERR_BAD_ARG, "out must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(unitcell) & 7) return fail(h, MKB_ERR_BAD_ARG, "unitcell must be 8-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (n_frames * frame_bytes > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * frame_bytes));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    // natoms == 0 still has its markers (and unit cells) to write: one atom tile
    const dim3 grid((unsigned)std::max<int64_t>(cdiv(natoms, DCD_T), 1),
                    (unsigned)std::min<int64_t>(cdiv(n_frames, DCD_T), DCD_MAX_GRID_Y));
    dcd_encode_kernel<<<grid, DCD_WARPS * 32, 0, st>>>(coords, frame_stride, (int)n_frames, (int)natoms, unitcell,
                                                        reinterpret_cast<unsigned *>(out), frame_bytes / 4);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
