// frame_tile.cuh -- the tile transposition shared by the trajectory codecs whose frame records hold big-endian
// (atom, axis) slabs: AMBER NetCDF (K23, netcdf.cu) and GROMACS TRR (K24, trr.cu).
//
// In a file, frame k's values are 3 * natoms contiguous big-endian reals (atom-major, the three axes of an atom
// interleaved), so decoding is a byte swap and a transposition of the (frame, atom * 3 + axis) plane into the
// frame-minor (natoms, 3, F) layout every kernel here consumes, and encoding is the same the other way round.
//
// Mapping: one CTA of 256 threads (8 warps) owns a tile of 32 frames x 96 values (32 atoms x 3 axes), staged in shared
// memory as [frame][value] rows of 97 32-bit words: on the file side a warp moves 32 consecutive values of one frame
// (row writes, conflict-free), on the array side a warp moves 32 consecutive frames of one (atom, axis) row (column
// reads, stride 97, odd, conflict-free).  Each thread moves 12 values each way with all 12 loads issued before the first
// shared-memory store.
//
// 4-byte reals travel as 32-bit words through __byte_perm and never through float arithmetic, so every bit pattern
// (NaN payloads, signalling NaNs, -0.0, subnormals) survives.  8-byte reals (decode only) are loaded as one 64-bit word
// per value, swapped and rounded to float32 as x86-64's cvtsd2ss does (see ft_f64be_to_f32).
//
// The kernels have internal linkage: each .cu that includes this header instantiates its own copies, so two translation
// units of the library may launch the same instantiation without sharing a registration.
#pragma once

namespace mkb {
namespace {

constexpr int FT_T = 32;                                 // frames and atoms per tile
constexpr int FT_W = 3 * FT_T;                           // values of one frame in a tile
constexpr int FT_WARPS = 8;                              // 256 threads
constexpr int FT_ITEMS = FT_T * FT_W / (32 * FT_WARPS);  // 12 values per thread each way
static_assert(FT_ITEMS == 12 && FT_W == 3 * 32, "file side: item i covers frame FT_WARPS * (i / 3) + warp, values 32 * (i % 3) + lane");
constexpr int FT_MAX_GRID_Y = 65535;

__device__ __forceinline__ unsigned ft_swap(unsigned w) { return __byte_perm(w, 0, 0x0123); }

// A big-endian float64 (its two words as they lie in memory) -> float32 bits, what numpy's astype(np.float32) gives on
// x86-64 (cvtsd2ss, MXCSR at its default): finite values round to nearest, ties to even, with overflow to +-inf and
// gradual underflow into the float32 subnormals (the build has no -ftz, so cvt.rn.f32.f64 keeps them); a NaN keeps its
// sign and the top 23 bits of its mantissa, quietened: sign | 0x7fc00000 | (mantissa >> 29).  The GPU's cvt would give
// its canonical NaN instead, so NaNs are built in integer arithmetic.
__device__ __forceinline__ unsigned ft_f64be_to_f32(uint2 raw) {
    const unsigned hi = ft_swap(raw.x), lo = ft_swap(raw.y);
    // |x| is a NaN exactly when (|hi| | (lo != 0)) > the high word of +inf
    if (((hi & 0x7fffffffu) | (lo != 0u)) > 0x7ff00000u)
        return (hi & 0x80000000u) | 0x7fc00000u | ((hi & 0x000fffffu) << 3) | (lo >> 29);
    return __float_as_uint(__double2float_rn(__hiloint2double((int)hi, (int)lo)));
}

// coords[(a*3 + d)*frame_stride + k] = big-endian real a*3 + d (VB bytes each) of the slab at bytes + offsets[k];
// n_vals = 3 * natoms.  VB == 8 needs every bytes + offsets[k] 8-byte aligned, VB == 4 4-byte aligned.
template <int VB>
__global__ void __launch_bounds__(FT_WARPS * 32, 4)
frame_tile_decode_kernel(const unsigned char *__restrict__ bytes, const long long *__restrict__ offsets, int n_frames,
                         long long n_vals, float *__restrict__ coords, long long frame_stride) {
    static_assert(VB == 4 || VB == 8, "4- or 8-byte reals");
    __shared__ unsigned tile[FT_T][FT_W + 1];  // [frame][value]
    __shared__ long long off[FT_T];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long w0 = (long long)blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile's reads of `tile` and `off` are done
        if (threadIdx.x < FT_T && k0 + (int)threadIdx.x < n_frames) off[threadIdx.x] = offsets[k0 + threadIdx.x];
        __syncthreads();
        unsigned w[FT_ITEMS];
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int fl = FT_WARPS * (i / 3) + warp, wl = 32 * (i % 3) + lane;
            w[i] = 0;
            if (w0 + wl < n_vals && k0 + fl < n_frames) {
                if constexpr (VB == 4)
                    w[i] = __ldcs(reinterpret_cast<const unsigned *>(bytes + off[fl]) + w0 + wl);
                else
                    w[i] = ft_f64be_to_f32(__ldcs(reinterpret_cast<const uint2 *>(bytes + off[fl]) + w0 + wl));
            }
        }
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i)
            tile[FT_WARPS * (i / 3) + warp][32 * (i % 3) + lane] = VB == 4 ? ft_swap(w[i]) : w[i];
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int i = 0; i < FT_ITEMS; ++i) {
            const int wl = FT_WARPS * i + warp;
            if (w0 + wl < n_vals && k < n_frames)
                __stcs(reinterpret_cast<unsigned *>(coords) + (w0 + wl) * frame_stride + k, tile[lane][wl]);
        }
    }
}

// Record k of the output is out[k*record_words ...]: the NSRC float32 (natoms, 3, F) source arrays big-endian one after
// the other from word coord_word (array s at coord_word + s * n_vals), the frame's `extra_words` words of extra (already
// in file byte order) around them -- those before coord_word first, the rest after the last array.  Array 0 is
// (coords0, stride0), arrays 1 and 2 (NSRC > 1) are (coords1, stride1) and (coords2, stride2): element (a, d, k) of
// array s at coords_s[(a*3 + d)*stride_s + k].  A CTA transposes the same tile of every array in turn; the CTAs of the
// first atom tile copy the extra words of their frames.  The arrays are separate parameters, not a struct, and the loop
// over them is unrolled, so no array is chosen at run time: with NSRC == 1 the kernel compiles to K23's encoder
// instruction for instruction, and each array of NSRC > 1 gets the same registers.
template <int NSRC>
__global__ void __launch_bounds__(FT_WARPS * 32, 4)
frame_tile_encode_kernel(const float *__restrict__ coords0, long long stride0, int n_frames, long long n_vals,
                         const unsigned *__restrict__ extra, int extra_words, int coord_word, unsigned *__restrict__ out,
                         long long record_words, const float *__restrict__ coords1, long long stride1,
                         const float *__restrict__ coords2, long long stride2) {
    static_assert(NSRC >= 1 && NSRC <= 3, "one to three source arrays");
    __shared__ unsigned tile[FT_T][FT_W + 1];  // [frame][value]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long w0 = (long long)blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
#pragma unroll
        for (int s = 0; s < NSRC; ++s) {
            const float *__restrict__ coords = s == 0 ? coords0 : (s == 1 ? coords1 : coords2);
            const long long frame_stride = s == 0 ? stride0 : (s == 1 ? stride1 : stride2);
            __syncthreads();  // the previous tile's reads of `tile` are done
            const int k = k0 + lane;
            unsigned w[FT_ITEMS];
#pragma unroll
            for (int i = 0; i < FT_ITEMS; ++i) {
                const int wl = FT_WARPS * i + warp;
                w[i] = 0;
                if (w0 + wl < n_vals && k < n_frames)
                    w[i] = __ldcs(reinterpret_cast<const unsigned *>(coords) + (w0 + wl) * frame_stride + k);
            }
#pragma unroll
            for (int i = 0; i < FT_ITEMS; ++i) tile[lane][FT_WARPS * i + warp] = w[i];
            __syncthreads();
#pragma unroll
            for (int i = 0; i < FT_ITEMS; ++i) {
                const int fl = FT_WARPS * (i / 3) + warp, wl = 32 * (i % 3) + lane;
                if (w0 + wl < n_vals && k0 + fl < n_frames)
                    __stcs(out + (long long)(k0 + fl) * record_words + coord_word + s * n_vals + w0 + wl,
                           ft_swap(tile[fl][wl]));
            }
        }
        if (blockIdx.x == 0) {
            const int n_tile = min(FT_T, n_frames - k0);
            for (int t = threadIdx.x; t < n_tile * extra_words; t += FT_WARPS * 32) {
                const int fl = t / extra_words, j = t - fl * extra_words;
                const long long kk = k0 + fl;
                out[kk * record_words + (j < coord_word ? j : j + NSRC * n_vals)] = extra[kk * extra_words + j];
            }
        }
    }
}

}  // namespace
}  // namespace mkb
