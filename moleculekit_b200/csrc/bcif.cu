// bcif.cu -- K31: BinaryCIF (.bcif) columns decoded and encoded on the device.
//
// A BinaryCIF column is one array of the _atom_site table stored as bytes and a chain of encodings.  Decoding runs the
// chain in reverse, each step a prefix scan or a map over the whole column, so the device work is a handful of scans
// and maps per column, nothing like the text tokenizers of K26 to K30.
//
//   bytes       ByteArray: little-endian Int8/16/32, Uint8/16/32 to 32-bit integers, Float32/64 to float32
//               (bc_bytes_kernel).
//   packing     IntegerPacking: an element equal to a limit (0xFF / 0xFFFF unsigned, 0x7F, -0x80 / 0x7FFF, -0x8000
//               signed) continues a value, any other element ends one.  bc_term_kernel flags the ends, an exclusive scan
//               of the flags gives every value's output index, and bc_unpack_kernel lets each end sum its value's
//               elements back to the previous end (a segmented sum that never crosses more than one value).
//   delta       Delta: out[0] = origin + d[0], out[i] = out[i-1] + d[i]: an exclusive scan of 32-bit words from the
//               origin (so it wraps modulo 2^32), plus d[i] and narrowed to the source type's width (bc_delta_kernel).
//   run-length  RunLength: an exclusive scan of the counts gives each run's first output index; every output value
//               finds its run by binary search over those starts (bc_expand_kernel), so a long run costs no more than
//               a short one.
//   store       the last step maps to the output: a FixedPoint or IntervalQuantization step is applied there, in
//               float64 with each operation rounded on its own, and rounded to float32.  Row order goes to a flat
//               array (bc_rows_kernel); the frames of a coordinate column go to the frame-minor (natoms, 3, F) array
//               through 32 x 32 shared-memory tiles (bc_frames_kernel), K23's tile transposition in one axis; the runs
//               of equal values of a model or mask column go to an O(runs) list (bc_runs_kernel).
//
// Encoding an integer array (a fixed-point coordinate column, an integer column, string indices, offsets, masks):
//   sizes       bc_stats_kernel reads the array once and sums, for the array and its deltas, the elements each value
//               takes at 1 and 2 bytes, signed and unsigned, with their minima; flags the run starts of both; two scans
//               rank the runs, bc_starts_kernel lists their starts and bc_run_stats_kernel sums the same for the
//               (value, count) pairs of both run-length arrays.  25 int64 go back to the host, which picks the chain.
//   emit        the chosen array is built (bc_build_kernel, or the run starts and bc_rle_kernel), then Int32 words are
//               copied as they are, or bc_cost_kernel, an exclusive scan and bc_pack_kernel write the packed bytes.
//   quantize    bc_quantize_kernel reads a coordinate axis of the (natoms, 3, F) input through the same tiles and writes
//               rint(x * factor) in row order.
// An encoded array may be given as one frame's values and a per-frame step (value i = v[i % period] + (i / period) *
// step, modulo 2^32), so the topology columns repeated in every frame, id and pdbx_PDB_model_num are never built whole.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace mkb {
namespace {

constexpr int BC_THREADS = 256;
constexpr int64_t BC_MAX_LEN = INT32_MAX - 1;  // values of one array: its scans of n + 1 values take int counts
constexpr int BC_STEP_WORDS = 6;
enum : int { K_BYTES = 1, K_PACKING = 2, K_DELTA = 3, K_RUN_LENGTH = 4, K_FIXED = 5, K_INTERVAL = 6 };
enum : int { T_I8 = 1, T_I16 = 2, T_I32 = 3, T_U8 = 4, T_U16 = 5, T_U32 = 6, T_F32 = 32, T_F64 = 33 };
enum : int { MODE_ROWS = 0, MODE_FRAMES = 1, MODE_RUNS = 2 };
// status[0] codes
enum : int { BC_MID_VALUE = 1, BC_PACKED_COUNT = 2, BC_RUN_TOTAL = 3, BC_RUN_NEGATIVE = 4 };

unsigned bc_grid(int64_t n) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(cdiv(n, BC_THREADS), 8192)); }
#define BC_FOR(i, n) for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

int type_bytes(int t) {
    switch (t) {
        case T_I8: case T_U8: return 1;
        case T_I16: case T_U16: return 2;
        case T_I32: case T_U32: case T_F32: return 4;
        case T_F64: return 8;
        default: return 0;
    }
}
bool int_type(int t) { return t >= T_I8 && t <= T_U32; }

__device__ __forceinline__ unsigned bc_narrow(unsigned w, int type) {
    return type == T_I8 ? (unsigned)(int)(signed char)w : type == T_U8 ? (w & 0xFFu)
         : type == T_I16 ? (unsigned)(int)(short)w : type == T_U16 ? (w & 0xFFFFu) : w;
}

__device__ __forceinline__ void bc_error(long long *status, int code) {
    atomicCAS(reinterpret_cast<unsigned long long *>(status), 0ull, (unsigned long long)code);
}

__global__ void bc_bytes_kernel(const unsigned char *__restrict__ b, long long n, int type, unsigned *__restrict__ out) {
    BC_FOR(i, n) {
        unsigned w;
        switch (type) {
            case T_I8: w = (unsigned)(int)(signed char)b[i]; break;
            case T_U8: w = b[i]; break;
            case T_I16: w = (unsigned)(int)reinterpret_cast<const short *>(b)[i]; break;
            case T_U16: w = reinterpret_cast<const unsigned short *>(b)[i]; break;
            case T_F64: w = __float_as_uint(__double2float_rn(reinterpret_cast<const double *>(b)[i])); break;
            default: w = reinterpret_cast<const unsigned *>(b)[i];
        }
        out[i] = w;
    }
}

__device__ __forceinline__ bool bc_limit(int x, int w, int u) {
    if (u) return x == (w == 1 ? 0xFF : 0xFFFF);
    return w == 1 ? (x == 0x7F || x == -0x80) : (x == 0x7FFF || x == -0x8000);
}

__global__ void bc_term_kernel(const int *__restrict__ x, long long m, int w, int u, long long *__restrict__ t) {
    BC_FOR(i, m) t[i] = bc_limit(x[i], w, u) ? 0 : 1;
}

// rank = exclusive scan of the end flags; value rank[i] of an end i is the sum of x back to the previous end
__global__ void bc_unpack_kernel(const int *__restrict__ x, long long m, int w, int u, const long long *__restrict__ rank,
                                 long long src_size, unsigned *__restrict__ out, long long *status) {
    BC_FOR(i, m) {
        const bool end = !bc_limit(x[i], w, u);
        if (end) {
            unsigned v = (unsigned)x[i];
            for (long long k = i - 1; k >= 0 && bc_limit(x[k], w, u); --k) v += (unsigned)x[k];
            if (rank[i] < src_size) out[rank[i]] = v;
        }
        if (i == m - 1) {
            if (!end) bc_error(status, BC_MID_VALUE);
            else if (rank[i] + 1 != src_size) bc_error(status, BC_PACKED_COUNT);
        }
    }
}

// out = origin + the deltas before i (an exclusive scan) -> + d[i], narrowed to the source type (modulo 2^32 first)
__global__ void bc_delta_kernel(const unsigned *__restrict__ d, unsigned *__restrict__ out, long long n, int type) {
    BC_FOR(i, n) out[i] = bc_narrow(out[i] + d[i], type);
}

__device__ __forceinline__ long long bc_int(unsigned w, int u32) { return u32 ? (long long)w : (long long)(int)w; }

// start[r] = count of run r, start[R] = 0 (then scanned); a negative count is an error
__global__ void bc_counts_kernel(const unsigned *__restrict__ x, long long R, int u32, long long *__restrict__ start,
                                 long long *status) {
    BC_FOR(r, R + 1) {
        long long c = 0;
        if (r < R) {
            c = bc_int(x[2 * r + 1], u32);
            if (c < 0) { bc_error(status, BC_RUN_NEGATIVE); c = 0; }
        }
        start[r] = c;
    }
}

__global__ void bc_total_kernel(const long long *start, long long R, long long src_size, long long *status) {
    if (start[R] != src_size) bc_error(status, BC_RUN_TOTAL);
}

__global__ void bc_expand_kernel(const unsigned *__restrict__ x, const long long *__restrict__ start, long long R,
                                 long long n, int type, unsigned *__restrict__ out) {
    BC_FOR(i, n) {
        long long lo = 0, hi = R - 1;  // the last run whose start is <= i
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if (start[mid] <= i) lo = mid;
            else hi = mid - 1;
        }
        out[i] = bc_narrow(x[2 * lo], type);
    }
}

// the last step: 0 copies the word, 1 is FixedPoint (a = factor), 2 IntervalQuantization (a = min, b = step)
struct Conv {
    int kind = 0, u32 = 0;
    double a = 0, b = 0;
};

__device__ __forceinline__ unsigned bc_conv(unsigned w, const Conv &c) {
    if (c.kind == 0) return w;
    const double q = (double)bc_int(w, c.u32);
    if (c.kind == 1) return __float_as_uint(__double2float_rn(__ddiv_rn(q, c.a)));
    return __float_as_uint(__double2float_rn(__dadd_rn(c.a, __dmul_rn(c.b, q))));
}

__global__ void bc_rows_kernel(const unsigned *__restrict__ x, long long n, Conv c, unsigned *__restrict__ out) {
    BC_FOR(i, n) out[i] = bc_conv(x[i], c);
}

// out[a*atom_stride + k] = value of row frames[k]*natoms + a; CTA (32, 8) over 32 atoms x 32 frames
__global__ void __launch_bounds__(256) bc_frames_kernel(const unsigned *__restrict__ x, const long long *__restrict__ frames,
                                                        long long n_frames, long long natoms, Conv c,
                                                        unsigned *__restrict__ out, long long atom_stride) {
    __shared__ unsigned tile[32][33];  // [frame][atom]
    const long long a0 = (long long)blockIdx.x * 32;
    const long long n_ft = (n_frames + 31) / 32;
    for (long long ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const long long k0 = ft * 32;
        for (int j = threadIdx.y; j < 32; j += 8) {
            const long long k = k0 + j, a = a0 + threadIdx.x;
            if (k < n_frames && a < natoms) tile[j][threadIdx.x] = bc_conv(x[frames[k] * natoms + a], c);
        }
        __syncthreads();
        for (int j = threadIdx.y; j < 32; j += 8) {
            const long long a = a0 + j, k = k0 + threadIdx.x;
            if (k < n_frames && a < natoms) out[a * atom_stride + k] = tile[threadIdx.x][j];
        }
        __syncthreads();
    }
}

__global__ void bc_runs_kernel(const unsigned *__restrict__ x, long long n, int u32, long long *__restrict__ out,
                               long long cap, long long *status) {
    BC_FOR(i, n) {
        if (i == 0 || x[i] != x[i - 1]) {
            const long long s = (long long)atomicAdd(reinterpret_cast<unsigned long long *>(status + 1), 1ull);
            if (s < cap) {
                out[2 * s] = i;
                out[2 * s + 1] = bc_int(x[i], u32);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------ encode
struct Src {
    const int *v;
    long long period, step;
    __device__ __forceinline__ int at(long long i) const {
        if (i < period) return v[i];
        const long long f = i / period;
        return (int)((unsigned)v[i - f * period] + (unsigned)(f * step));
    }
    __device__ __forceinline__ int delta(long long i) const {
        return i == 0 ? 0 : (int)((unsigned)at(i) - (unsigned)at(i - 1));
    }
};

// per array: min, elements at 1 byte unsigned, 2 bytes unsigned, 1 byte signed, 2 bytes signed
constexpr int BC_STATS = 5;
__device__ __forceinline__ void bc_cost(long long x, long long (&s)[BC_STATS]) {
    s[0] = min(s[0], x);
    s[1] += x >= 0 ? x / 0xFF + 1 : 0;
    s[2] += x >= 0 ? x / 0xFFFF + 1 : 0;
    s[3] += x >= 0 ? x / 0x7F + 1 : (-x) / 0x80 + 1;
    s[4] += x >= 0 ? x / 0x7FFF + 1 : (-x) / 0x8000 + 1;
}

// block sum (min for slot 0) of NV arrays' stats into acc[array * BC_STATS + j]
template <int NV>
__device__ void bc_flush(long long (&s)[NV][BC_STATS], long long *acc) {
    __shared__ long long red[BC_THREADS / 32][NV * BC_STATS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int v = 0; v < NV; ++v)
#pragma unroll
        for (int j = 0; j < BC_STATS; ++j) {
            long long x = s[v][j];
            for (int o = 16; o; o >>= 1) {
                const long long y = __shfl_down_sync(0xffffffffu, x, o);
                x = j == 0 ? min(x, y) : x + y;
            }
            if (lane == 0) red[warp][v * BC_STATS + j] = x;
        }
    __syncthreads();
    if (threadIdx.x < NV * BC_STATS) {
        const int j = threadIdx.x % BC_STATS;
        long long x = red[0][threadIdx.x];
        for (int w = 1; w < BC_THREADS / 32; ++w) x = j == 0 ? min(x, red[w][threadIdx.x]) : x + red[w][threadIdx.x];
        if (j == 0) atomicMin(acc + threadIdx.x, x);
        else atomicAdd(reinterpret_cast<unsigned long long *>(acc + threadIdx.x), (unsigned long long)x);
    }
}

// stats of the array (acc[0..4]) and its deltas (acc[5..9]); rv / rd = run-start flags of both, with rv[n] = rd[n] = 0
__global__ void __launch_bounds__(BC_THREADS) bc_stats_kernel(Src s, long long n, long long *__restrict__ rv,
                                                              long long *__restrict__ rd, long long *acc) {
    long long st[2][BC_STATS];
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        st[v][0] = LLONG_MAX;
        for (int j = 1; j < BC_STATS; ++j) st[v][j] = 0;
    }
    BC_FOR(i, n + 1) {
        if (i == n) {
            rv[n] = rd[n] = 0;
            continue;
        }
        const int x = s.at(i), d = s.delta(i);
        bc_cost(x, st[0]);
        bc_cost(d, st[1]);
        rv[i] = i == 0 || x != s.at(i - 1);
        rd[i] = i == 0 || d != s.delta(i - 1);
    }
    bc_flush<2>(st, acc);
}

// rank = scanned run flags: starts[rank[i]] = i at every run start; rank[n] = R
__global__ void bc_starts_kernel(Src s, long long n, int use_delta, const long long *__restrict__ rank,
                                 long long *__restrict__ starts) {
    BC_FOR(i, n) {
        const bool start = i == 0 || (use_delta ? s.delta(i) != s.delta(i - 1) : s.at(i) != s.at(i - 1));
        if (start) starts[rank[i]] = i;
    }
}

// stats of the (value, count) pairs of both run-length arrays: acc[0..4] of the array's runs, acc[5..9] of the deltas'
__global__ void __launch_bounds__(BC_THREADS) bc_run_stats_kernel(Src s, long long n, const long long *__restrict__ rank_v,
                                                                  const long long *__restrict__ starts_v,
                                                                  const long long *__restrict__ rank_d,
                                                                  const long long *__restrict__ starts_d,
                                                                  long long *acc) {
    long long st[2][BC_STATS];
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        st[v][0] = LLONG_MAX;
        for (int j = 1; j < BC_STATS; ++j) st[v][j] = 0;
    }
    const long long Rv = rank_v[n], Rd = rank_d[n];
    BC_FOR(r, max(Rv, Rd)) {
        if (r < Rv) {
            const long long i = starts_v[r];
            bc_cost(s.at(i), st[0]);
            bc_cost((r + 1 < Rv ? starts_v[r + 1] : n) - i, st[0]);
        }
        if (r < Rd) {
            const long long i = starts_d[r];
            bc_cost(s.delta(i), st[1]);
            bc_cost((r + 1 < Rd ? starts_d[r + 1] : n) - i, st[1]);
        }
    }
    bc_flush<2>(st, acc);
}

// rank[i] = 1 where a run of the array (use_delta 0) or of its deltas starts, rank[n] = 0
__global__ void bc_flags_kernel(Src s, long long n, int use_delta, long long *__restrict__ rank) {
    BC_FOR(i, n + 1) rank[i] = i < n && (i == 0 || (use_delta ? s.delta(i) != s.delta(i - 1) : s.at(i) != s.at(i - 1)));
}

__global__ void bc_init_kernel(long long *acc) {
    if (threadIdx.x < 4 * BC_STATS) acc[threadIdx.x] = threadIdx.x % BC_STATS ? 0 : LLONG_MAX;
}

__global__ void bc_build_kernel(Src s, long long n, int use_delta, int *__restrict__ out) {
    BC_FOR(i, n) out[i] = use_delta ? s.delta(i) : s.at(i);
}

__global__ void bc_rle_kernel(Src s, long long n, int use_delta, const long long *__restrict__ rank,
                              const long long *__restrict__ starts, int *__restrict__ out) {
    const long long R = rank[n];
    BC_FOR(r, R) {
        const long long i = starts[r];
        out[2 * r] = use_delta ? s.delta(i) : s.at(i);
        out[2 * r + 1] = (int)((r + 1 < R ? starts[r + 1] : n) - i);
    }
}

__device__ __forceinline__ long long bc_elems(long long x, int w, int u) {
    if (u) return x / (w == 1 ? 0xFF : 0xFFFF) + 1;
    return x >= 0 ? x / (w == 1 ? 0x7F : 0x7FFF) + 1 : (-x) / (w == 1 ? 0x80 : 0x8000) + 1;
}

__global__ void bc_cost_kernel(const int *__restrict__ x, long long m, int w, int u, long long *__restrict__ off) {
    BC_FOR(i, m + 1) off[i] = i < m ? bc_elems(x[i], w, u) : 0;
}

// the elements of value x from out[o], none at or past out[lim]
template <typename E>
__device__ __forceinline__ void bc_put(long long x, int w, int u, E *out, long long o, long long lim) {
    if (u || x >= 0) {
        const long long L = u ? (w == 1 ? 0xFF : 0xFFFF) : (w == 1 ? 0x7F : 0x7FFF);
        for (; x >= L; x -= L, ++o)
            if (o < lim) out[o] = (E)L;
    } else {
        const long long L = w == 1 ? -0x80 : -0x8000;
        for (; x <= L; x -= L, ++o)
            if (o < lim) out[o] = (E)L;
    }
    if (o < lim) out[o] = (E)x;
}

__global__ void bc_pack_kernel(const int *__restrict__ x, long long m, int w, int u, const long long *__restrict__ off,
                               unsigned char *__restrict__ out, long long lim) {
    BC_FOR(i, m) {
        if (w == 1) bc_put<unsigned char>(x[i], 1, u, out, off[i], lim);
        else bc_put<unsigned short>(x[i], 2, u, reinterpret_cast<unsigned short *>(out), off[i], lim);
    }
}

// q[k*natoms + a] = rint(x[a*atom_stride + k*frame_stride] * factor) in float64 (the caller keeps it inside int32)
__global__ void __launch_bounds__(256) bc_quantize_kernel(const float *__restrict__ x, long long atom_stride,
                                                          long long frame_stride, long long natoms, long long n_frames,
                                                          double factor, int *__restrict__ q) {
    __shared__ int tile[32][33];  // [atom][frame]
    const long long a0 = (long long)blockIdx.x * 32;
    const long long n_ft = (n_frames + 31) / 32;
    for (long long ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const long long k0 = ft * 32;
        for (int j = threadIdx.y; j < 32; j += 8) {
            const long long a = a0 + j, k = k0 + threadIdx.x;
            if (k < n_frames && a < natoms)
                tile[j][threadIdx.x] = (int)rint(__dmul_rn((double)x[a * atom_stride + k * frame_stride], factor));
        }
        __syncthreads();
        for (int j = threadIdx.y; j < 32; j += 8) {
            const long long k = k0 + j, a = a0 + threadIdx.x;
            if (k < n_frames && a < natoms) q[k * natoms + a] = tile[threadIdx.x][j];
        }
        __syncthreads();
    }
}

// cub temp storage for the scans of arrays up to n values
int bc_scan_tmp(mkb_ctx *h, cudaStream_t st, int64_t n, size_t extra, void **tmp, size_t *tmp_bytes) {
    size_t a = 0, b = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, a, (long long *)nullptr, (int)(n + 1), st));
    MKB_CUDA(h, cub::DeviceScan::ExclusiveScan(nullptr, b, (unsigned *)nullptr, (unsigned *)nullptr,
                                               cuda::std::plus<unsigned>{}, 0u, (int)(n), st));
    *tmp_bytes = std::max(a, b);
    unsigned char *p;
    const size_t head = (extra + 255) & ~(size_t)255;
    int rc = scratch_get(h, S_BCIF_TMP, head + *tmp_bytes, &p);
    *tmp = p + head;
    return rc;
}

// the run starts of the array (use_delta 0) or its deltas: flags into rank[0..n], scanned; starts[0..R)
int bc_run_starts(mkb_ctx *h, cudaStream_t st, const Src &s, int64_t n, int use_delta, long long *rank, long long *starts,
                  void *tmp, size_t tmp_bytes) {
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, rank, (int)(n + 1), st));
    bc_starts_kernel<<<bc_grid(n), BC_THREADS, 0, st>>>(s, n, use_delta, rank, starts);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

int bc_src(mkb_ctx *h, const int32_t *v, int64_t period, int64_t n, Src *s) {
    if (!v) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (n < 1 || n > BC_MAX_LEN) return fail(h, MKB_ERR_BAD_ARG, "n must be 1 to 2^31 - 2");
    if (period < 1 || period > n) return fail(h, MKB_ERR_BAD_ARG, "period must be 1 to n");
    if (reinterpret_cast<uintptr_t>(v) & 3) return fail(h, MKB_ERR_BAD_ARG, "values must be 4-byte aligned");
    s->v = v;
    s->period = period;
    return MKB_OK;
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_bcif_decode(mkb_handle_t h, void *stream, const uint8_t *data, int64_t nbytes, const double *steps,
                               int64_t n_steps, int64_t mode, void *out, int64_t n_out, const int64_t *frames,
                               int64_t natoms, int64_t atom_stride, int64_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (!steps || !status || n_steps < 1 || n_steps > 64) return fail(h, MKB_ERR_BAD_ARG, "1 to 64 steps and a status");
    if (nbytes < 0 || n_out < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (nbytes && !data) return fail(h, MKB_ERR_BAD_ARG, "null data");
    if ((reinterpret_cast<uintptr_t>(data) & 15) || (reinterpret_cast<uintptr_t>(out) & (mode == MODE_RUNS ? 7 : 3)) ||
        (reinterpret_cast<uintptr_t>(status) & 7))
        return fail(h, MKB_ERR_BAD_ARG, "data must be 16-byte, out 4-byte (runs: 8-byte) and status 8-byte aligned");
    // walk the chain on the host: every step's length and type, the largest array, and the last step's conversion
    const int type0 = (int)steps[1];
    if ((int)steps[0] != K_BYTES || !type_bytes(type0)) return fail(h, MKB_ERR_BAD_ARG, "the first step must be a ByteArray");
    if (nbytes % type_bytes(type0)) return fail(h, MKB_ERR_BAD_ARG, "nbytes is not a multiple of the type's size");
    int64_t m = nbytes / type_bytes(type0), cap = m;
    bool is_int = int_type(type0), ended = false;
    Conv conv, last;
    for (int64_t s = 1; s < n_steps; ++s) {
        const double *p = steps + s * BC_STEP_WORDS;
        const int kind = (int)p[0];
        if (!is_int || ended) return fail(h, MKB_ERR_BAD_ARG, "step %lld needs integers", (long long)s);
        if (kind == K_PACKING) {
            if ((p[1] != 1 && p[1] != 2) || p[3] < 0 || p[3] > (double)m)
                return fail(h, MKB_ERR_BAD_ARG, "IntegerPacking: byteCount 1 or 2 and srcSize 0 to its elements");
            m = (int64_t)p[3];
        } else if (kind == K_DELTA) {
            if (!int_type((int)p[2])) return fail(h, MKB_ERR_BAD_ARG, "Delta: an integer srcType");
        } else if (kind == K_RUN_LENGTH) {
            if ((m & 1) || !int_type((int)p[1]) || p[2] < 0 || p[2] > (double)BC_MAX_LEN)
                return fail(h, MKB_ERR_BAD_ARG, "RunLength: pairs, an integer srcType and srcSize 0 to 2^31 - 2");
            m = (int64_t)p[2];
        } else if (kind == K_FIXED || kind == K_INTERVAL) {
            if (kind == K_FIXED ? !(p[1] != 0) : !(p[3] >= 2))
                return fail(h, MKB_ERR_BAD_ARG, "FixedPoint factor 0 or IntervalQuantization numSteps < 2");
            ended = true;
            last.kind = kind == K_FIXED ? 1 : 2;
            last.a = p[1];
            last.b = kind == K_FIXED ? 0.0 : (p[2] - p[1]) / (p[3] - 1.0);
        } else {
            return fail(h, MKB_ERR_BAD_ARG, "step %lld: unknown kind %d", (long long)s, kind);
        }
        cap = std::max(cap, m);
    }
    if (cap > BC_MAX_LEN) return fail(h, MKB_ERR_BAD_ARG, "arrays of more than 2^31 - 2 values");
    const bool floats = !is_int || ended;
    if (mode == MODE_ROWS) {
        if (n_out > m || (n_out && !out)) return fail(h, MKB_ERR_BAD_ARG, "n_out rows must be 0 to the decoded length");
    } else if (mode == MODE_FRAMES) {
        if (!floats || natoms < 1 || m % natoms || atom_stride < n_out || (n_out && (!out || !frames)))
            return fail(h, MKB_ERR_BAD_ARG, "frames need floats, whole frames of natoms rows and atom_stride >= n_frames");
        for (int64_t k = 0; k < n_out; ++k)
            if (frames[k] < 0 || frames[k] >= m / natoms)
                return fail(h, MKB_ERR_BAD_ARG, "frames[%lld] = %lld is not a frame", (long long)k, (long long)frames[k]);
    } else if (mode == MODE_RUNS) {
        if (floats || (n_out && !out)) return fail(h, MKB_ERR_BAD_ARG, "runs need integers");
    } else {
        return fail(h, MKB_ERR_BAD_ARG, "unknown mode");
    }
    unsigned *val;
    long long *idx;
    void *tmp;
    size_t tmp_bytes;
    int rc;
    if ((rc = scratch_get(h, S_BCIF_VAL, (size_t)(2 * cap + 2), &val))) return rc;
    if ((rc = scratch_get(h, S_BCIF_IDX, (size_t)(cap + 2), &idx))) return rc;
    const size_t frame_bytes = mode == MODE_FRAMES ? sizeof(long long) * (size_t)n_out : 0;
    if ((rc = bc_scan_tmp(h, st, cap, frame_bytes, &tmp, &tmp_bytes))) return rc;
    long long *d_frames = reinterpret_cast<long long *>(h->scratch[S_BCIF_TMP].ptr);
    unsigned *a = val, *b = val + cap + 1;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemsetAsync(status, 0, 2 * sizeof(long long), st));
    if (frame_bytes)
        MKB_CUDA(h, cudaMemcpyAsync(d_frames, frames, frame_bytes, cudaMemcpyHostToDevice, st));
    m = nbytes / type_bytes(type0);
    if (m) {
        bc_bytes_kernel<<<bc_grid(m), BC_THREADS, 0, st>>>(data, m, type0, a);
        MKB_LAUNCHED(h);
    }
    long long *sd = reinterpret_cast<long long *>(status);
    for (int64_t s = 1; s < n_steps && conv.kind == 0; ++s) {
        const double *p = steps + s * BC_STEP_WORDS;
        const int kind = (int)p[0];
        if (kind == K_PACKING) {
            const int w = (int)p[1], u = p[2] != 0;
            const int64_t src = (int64_t)p[3];
            if (m) {
                bc_term_kernel<<<bc_grid(m), BC_THREADS, 0, st>>>((const int *)a, m, w, u, idx);
                MKB_LAUNCHED(h);
                MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, idx, (int)(m), st));
                bc_unpack_kernel<<<bc_grid(m), BC_THREADS, 0, st>>>((const int *)a, m, w, u, idx, src, b, sd);
                MKB_LAUNCHED(h);
            }
            std::swap(a, b);
            m = src;
            conv.u32 = 0;
        } else if (kind == K_DELTA) {
            const int type = (int)p[2];
            if (m) {
                MKB_CUDA(h, cub::DeviceScan::ExclusiveScan(tmp, tmp_bytes, a, b, cuda::std::plus<unsigned>{},
                                                           (unsigned)(long long)p[1], (int)(m), st));
                bc_delta_kernel<<<bc_grid(m), BC_THREADS, 0, st>>>(a, b, m, type);
                MKB_LAUNCHED(h);
                std::swap(a, b);
            }
            conv.u32 = type == T_U32;
        } else if (kind == K_RUN_LENGTH) {
            const int type = (int)p[1];
            const int64_t src = (int64_t)p[2], R = m / 2;
            bc_counts_kernel<<<bc_grid(R + 1), BC_THREADS, 0, st>>>(a, R, conv.u32, idx, sd);
            MKB_LAUNCHED(h);
            MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, idx, (int)(R + 1), st));
            bc_total_kernel<<<1, 1, 0, st>>>(idx, R, src, sd);
            MKB_LAUNCHED(h);
            if (src && R) {
                bc_expand_kernel<<<bc_grid(src), BC_THREADS, 0, st>>>(a, idx, R, src, type, b);
                MKB_LAUNCHED(h);
            }
            std::swap(a, b);
            m = src;
            conv.u32 = type == T_U32;
        } else {  // FixedPoint or IntervalQuantization, the last step: applied by the store below
            conv.kind = last.kind;
            conv.a = last.a;
            conv.b = last.b;
        }
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    if (mode == MODE_ROWS && n_out) {
        bc_rows_kernel<<<bc_grid(n_out), BC_THREADS, 0, st>>>(a, n_out, conv, (unsigned *)out);
        MKB_LAUNCHED(h);
    } else if (mode == MODE_FRAMES && n_out) {
        const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_out, 32), 65535));
        bc_frames_kernel<<<grid, dim3(32, 8), 0, st>>>(a, d_frames, n_out, natoms, conv, (unsigned *)out, atom_stride);
        MKB_LAUNCHED(h);
    } else if (mode == MODE_RUNS && m) {
        bc_runs_kernel<<<bc_grid(m), BC_THREADS, 0, st>>>(a, m, conv.u32, (long long *)out, n_out, sd);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_bcif_quantize(mkb_handle_t h, void *stream, const float *x, int64_t atom_stride, int64_t frame_stride,
                                 int64_t natoms, int64_t n_frames, double factor, int32_t *q) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (natoms < 0 || n_frames < 0 || atom_stride < 0 || frame_stride < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (natoms == 0 || n_frames == 0) return MKB_OK;
    if (!x || !q) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "x and q must be 4-byte aligned");
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, 32), 65535));
    bc_quantize_kernel<<<grid, dim3(32, 8), 0, st>>>(x, atom_stride, frame_stride, natoms, n_frames, factor, q);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_bcif_sizes(mkb_handle_t h, void *stream, const int32_t *v, int64_t period, int64_t step, int64_t n,
                              int64_t *sizes) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    Src s;
    int rc;
    if ((rc = bc_src(h, v, period, n, &s))) return rc;
    if (!sizes) return fail(h, MKB_ERR_BAD_ARG, "null sizes");
    s.step = step;
    long long *idx, *acc;
    void *tmp;
    size_t tmp_bytes;
    // rank_v, rank_d (n + 1 each), starts_v, starts_d (n each), then 20 accumulators
    if ((rc = scratch_get(h, S_BCIF_IDX, (size_t)(4 * n + 2 + 2 * 2 * BC_STATS), &idx))) return rc;
    if ((rc = bc_scan_tmp(h, st, n, 0, &tmp, &tmp_bytes))) return rc;
    long long *rank_v = idx, *rank_d = idx + n + 1, *starts_v = idx + 2 * n + 2, *starts_d = starts_v + n;
    acc = starts_d + n;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    bc_init_kernel<<<1, 32, 0, st>>>(acc);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    bc_stats_kernel<<<bc_grid(n + 1), BC_THREADS, 0, st>>>(s, n, rank_v, rank_d, acc);
    MKB_LAUNCHED(h);
    if ((rc = bc_run_starts(h, st, s, n, 0, rank_v, starts_v, tmp, tmp_bytes))) return rc;
    if ((rc = bc_run_starts(h, st, s, n, 1, rank_d, starts_d, tmp, tmp_bytes))) return rc;
    bc_run_stats_kernel<<<bc_grid(n), BC_THREADS, 0, st>>>(s, n, rank_v, starts_v, rank_d, starts_d,
                                                           acc + 2 * BC_STATS);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    long long got[4 * BC_STATS], runs[2];
    int32_t v0;
    MKB_CUDA(h, cudaMemcpyAsync(got, acc, sizeof(got), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaMemcpyAsync(&runs[0], rank_v + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaMemcpyAsync(&runs[1], rank_d + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaMemcpyAsync(&v0, v, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    // chains (a) the array, (b) its runs, (c) its deltas, (d) the deltas' runs: acc blocks 0, 2, 1, 3
    const int block[4] = {0, 2, 1, 3};
    const int64_t len[4] = {n, 2 * runs[0], n, 2 * runs[1]};
    sizes[0] = v0;
    for (int c = 0; c < 4; ++c) {
        int64_t *o = sizes + 1 + 6 * c;
        o[0] = len[c];
        for (int j = 0; j < BC_STATS; ++j) o[1 + j] = got[block[c] * BC_STATS + j];
    }
    return MKB_OK;
}

extern "C" int mkb_bcif_emit(mkb_handle_t h, void *stream, const int32_t *v, int64_t period, int64_t step, int64_t n,
                             int64_t chain, int64_t width, int64_t is_unsigned, int64_t n_packed, uint8_t *out,
                             int64_t out_bytes) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    Src s;
    int rc;
    if ((rc = bc_src(h, v, period, n, &s))) return rc;
    s.step = step;
    if (chain < 0 || chain > 3 || (width != 1 && width != 2 && width != 4))
        return fail(h, MKB_ERR_BAD_ARG, "chain 0 to 3 and width 1, 2 or 4");
    if (n_packed < 1 || n_packed > (chain & 1 ? 2 * n : n) || (chain & 1 ? n_packed & 1 : n_packed != n))
        return fail(h, MKB_ERR_BAD_ARG, "n_packed is not the chosen array's length");
    if (!out || (reinterpret_cast<uintptr_t>(out) & 3)) return fail(h, MKB_ERR_BAD_ARG, "out must be 4-byte aligned");
    if (width == 4 && out_bytes < 4 * n_packed) return fail(h, MKB_ERR_CAPACITY, "out holds %lld bytes", (long long)out_bytes);
    int *arr;
    long long *idx;
    void *tmp;
    size_t tmp_bytes;
    if ((rc = scratch_get(h, S_BCIF_VAL, (size_t)n_packed, &arr))) return rc;
    if ((rc = scratch_get(h, S_BCIF_IDX, (size_t)(2 * n + 2 + n_packed), &idx))) return rc;
    if ((rc = bc_scan_tmp(h, st, std::max(n, n_packed), 0, &tmp, &tmp_bytes))) return rc;
    const int use_delta = chain >= 2;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    if (chain & 1) {
        long long *rank = idx, *starts = idx + n + 1;
        bc_flags_kernel<<<bc_grid(n + 1), BC_THREADS, 0, st>>>(s, n, use_delta, rank);
        MKB_LAUNCHED(h);
        if ((rc = bc_run_starts(h, st, s, n, use_delta, rank, starts, tmp, tmp_bytes))) return rc;
        bc_rle_kernel<<<bc_grid(n), BC_THREADS, 0, st>>>(s, n, use_delta, rank, starts, arr);
        MKB_LAUNCHED(h);
    } else {
        bc_build_kernel<<<bc_grid(n), BC_THREADS, 0, st>>>(s, n, use_delta, arr);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    if (width == 4) {
        MKB_CUDA(h, cudaMemcpyAsync(out, arr, 4 * (size_t)n_packed, cudaMemcpyDeviceToDevice, st));
    } else {
        bc_cost_kernel<<<bc_grid(n_packed + 1), BC_THREADS, 0, st>>>(arr, n_packed, (int)width, is_unsigned != 0, idx);
        MKB_LAUNCHED(h);
        MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, idx, (int)(n_packed + 1), st));
        bc_pack_kernel<<<bc_grid(n_packed), BC_THREADS, 0, st>>>(arr, n_packed, (int)width, is_unsigned != 0, idx, out,
                                                                  out_bytes / width);
        MKB_LAUNCHED(h);
    }
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
