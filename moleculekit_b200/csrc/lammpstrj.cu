// lammpstrj.cu -- K32: LAMMPS dump trajectories (dump atom / dump custom text) indexed, parsed and formatted on the
// device.
//
// A frame is P lines: the header items of frame 0 (TIME, TIMESTEP, NUMBER OF ATOMS, BOX BOUNDS, ATOMS, H lines in all)
// and N atom lines whose columns are named by the ATOMS header.  Frame 0 may start with an ITEM: UNITS pair the others
// lack, so the running line count of the index starts at minus those lines and frame f >= 1 starts at line f P.
//
//   index   xl_lines.cuh's three newline passes record each frame's first byte (mkb_lammpstrj_index); then
//           lt_check_kernel, one thread per frame started in the chunk, walks the H header lines against frame 0's
//           (trailing whitespace stripped): every ITEM line byte for byte, the count line as N.  A mismatch, or a header
//           that runs past the bytes read, is left to the host.
//   head    lt_head_kernel, one thread per frame of the chunk (mkb_lammpstrj_head): TIMESTEP as int64, TIME and the
//           box lines as float64 (xyz_number.cuh's grammar, the value float() gives).  An undecided line is left to the
//           host.
//   decode  over staged whole frames (mkb_lammpstrj_decode): the newline emit pass stores every line start, then
//           lt_parse_kernel gives a warp 32 listed frames of one atom line: each lane walks the columns up to the last
//           one needed, places the line in its row by id (id - 1, or a binary search of frame 0's sorted ids), marks
//           the row in a per-frame bitmap (a duplicate or unknown id flags the frame) and converts the coordinates in
//           float64 with __dadd_rn / __dmul_rn in the order the module docstring states, rounded to float32 once.
//   encode  a length pass (one thread per line, the exact bytes of '%d %d %.9g ...'), a device scan and an emit pass
//           that formats each line at its offset (mkb_lammpstrj_encode); frame headers are built on the host.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "lammpstrj_g9.cuh"
#include "xl_lines.cuh"
#include "xyz_number.cuh"

namespace mkb {
namespace {

constexpr int LT_THREADS = 128;
constexpr int LT_WARPS = 8;  // decode: atom lines per CTA (one per warp), 32 listed frames per warp
enum LtRole { LT_SKIP = 0, LT_ID = 1, LT_POS = 2, LT_IMG = 5, LT_VEL = 8, LT_FRC = 11, LT_NROLE = 14 };

// bytes [p, end) of a 16-byte aligned buffer through a 16-byte window; '\n' at and past end
struct LtReader {
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

// the float32 nearest d; a NaN keeps its sign as a quiet 0x7fc00000, as numpy's float64 -> float32 cast gives it
__device__ __forceinline__ float lt_f32(double d) {
    if (isnan(d)) return __uint_as_float(((unsigned)(__double_as_longlong(d) >> 32) & 0x80000000u) | 0x7fc00000u);
    return __double2float_rn(d);
}

__device__ __forceinline__ bool lt_blank(unsigned c) { return c == ' ' || c == '\t' || c == '\r'; }

// the frames whose first line was started by a newline of this chunk: [f0, f1), f >= 1 and < frame_cap.  state[3]
// holds the line count before the chunk, state[0] after it.
__device__ __forceinline__ void lt_frame_range(const long long *state, long long P, long long frame_cap, long long &f0,
                                               long long &f1) {
    const long long before = state[3], after = state[0];  // lines [before + 1, after] start in this chunk
    f0 = max(1LL, (before + P) / P);
    f1 = min(frame_cap, (after + P) / P);  // the last f with f P <= after, plus one
}

// the end of the line at b[p] (its '\n'), or -1 when it does not end before n_read
__device__ __forceinline__ long long lt_eol(const unsigned char *b, long long p, long long n_read) {
    for (; p < n_read; ++p)
        if (b[p] == '\n') return p;
    return -1;
}

// [+-]?digits, at most 18 of them, then blanks to e -> v; false otherwise
__device__ __forceinline__ bool lt_int(LtReader &rd, long long &p, long long &v) {
    unsigned c = rd.at(p);
    bool neg = false;
    if (c == '+' || c == '-') {
        neg = c == '-';
        c = rd.at(++p);
    }
    int nd = 0;
    long long x = 0;
    for (; xyz_digit(c); c = rd.at(++p)) {
        if (++nd > 18) return false;
        x = 10 * x + (c - '0');
    }
    if (nd == 0 || !xyz_sep(c)) return false;
    v = neg ? -x : x;
    return true;
}

__device__ __forceinline__ unsigned lt_skip_sep(LtReader &rd, long long &p) {
    unsigned c = rd.at(p);
    while (xyz_sep(c) && c != '\n') c = rd.at(++p);
    return c;
}

// status[f] = 0 when the H header lines of frame f match the template (tmpl: frame 0's header lines without trailing
// whitespace, each ended by '\n'), the count line being natoms; else 1
__global__ void __launch_bounds__(LT_THREADS)
lt_check_kernel(const unsigned char *__restrict__ b, long long n_read, long long file_base, long long P,
                const long long *__restrict__ state, const long long *__restrict__ frame_off, long long frame_cap,
                const unsigned char *__restrict__ tmpl, int H, int count_line, long long natoms,
                unsigned char *__restrict__ status) {
    long long f0, f1;
    lt_frame_range(state, P, frame_cap, f0, f1);
    const long long f = f0 + (long long)blockIdx.x * LT_THREADS + threadIdx.x;
    if (f >= f1) return;
    long long p = frame_off[f] - file_base;
    int t = 0;
    unsigned char ok = 1;
    for (int j = 0; j < H && ok; ++j) {
        const long long e = p >= 0 ? lt_eol(b, p, n_read) : -1;
        if (e < 0) {
            ok = 0;
            break;
        }
        long long z = e;
        while (z > p && lt_blank(b[z - 1])) --z;
        const bool item = tmpl[t] == 'I' && tmpl[t + 1] == 'T' && tmpl[t + 2] == 'E' && tmpl[t + 3] == 'M' &&
                          tmpl[t + 4] == ':';
        if (item) {
            long long q = p;
            for (; tmpl[t] != '\n'; ++t, ++q)
                if (q >= z || b[q] != tmpl[t]) ok = 0;
            if (q != z) ok = 0;
        } else {
            while (tmpl[t] != '\n') ++t;
            if (j == count_line) {
                LtReader rd{reinterpret_cast<const uint4 *>(b), e};
                long long q = p, v = -1;
                lt_skip_sep(rd, q);
                if (!lt_int(rd, q, v) || v != natoms || lt_skip_sep(rd, q) != '\n') ok = 0;
            }
        }
        ++t;
        p = e + 1;
    }
    status[f] = ok ? 0 : 1;
}

// step[f], time[f], bounds[9 f ...] (lo, hi, tilt of each box line; tilt 0 without one) of each frame of the chunk;
// hstatus[f] = 1 when a line is left to the host
__global__ void __launch_bounds__(LT_THREADS)
lt_head_kernel(const unsigned char *__restrict__ b, long long n_read, long long file_base, long long P,
               const long long *__restrict__ state, const long long *__restrict__ frame_off, long long frame_cap,
               int step_line, int time_line, int box_line, int ntilt, long long *__restrict__ step,
               double *__restrict__ time, double *__restrict__ bounds, unsigned char *__restrict__ hstatus) {
    long long f0, f1;
    lt_frame_range(state, P, frame_cap, f0, f1);
    const long long f = f0 + (long long)blockIdx.x * LT_THREADS + threadIdx.x;
    if (f >= f1) return;
    long long p = frame_off[f] - file_base;
    bool ok = p >= 0;
    double bd[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    double tv = 0.0;
    long long sv = 0;
    const int last = max(box_line + 2, max(step_line, time_line));
    for (int j = 0; j <= last && ok; ++j) {
        const long long e = lt_eol(b, p, n_read);
        if (e < 0) {
            ok = false;
            break;
        }
        LtReader rd{reinterpret_cast<const uint4 *>(b), e};
        long long q = p;
        if (j == step_line) {
            lt_skip_sep(rd, q);
            ok = lt_int(rd, q, sv) && lt_skip_sep(rd, q) == '\n';
        } else if (j == time_line || j >= box_line) {
            const int nv = j == time_line ? 1 : 2 + ntilt;
            for (int i = 0; i < nv && ok; ++i) {
                unsigned long long bits;
                if (lt_skip_sep(rd, q) == '\n' || !xyz_number<true>(rd, q, bits)) {
                    ok = false;
                    break;
                }
                const double v = xyz_bits_f64(bits);
                if (j == time_line) tv = v;
                else bd[3 * (j - box_line) + i] = v;
            }
            if (ok && lt_skip_sep(rd, q) != '\n') ok = false;
        }
        p = e + 1;
    }
    step[f] = sv;
    time[f] = tv;
#pragma unroll
    for (int i = 0; i < 9; ++i) bounds[9 * f + i] = bd[i];
    hstatus[f] = ok ? 0 : 1;
}

// coords / vels / forces[(row*3 + d)*frame_stride + k] of atom line a of listed frame k (staged frame frame_of[k], lines
// starts[P u + H + a] ...).  role[c] (c < n_cols) names column c's use; params[9 k ...] = xlo ylo zlo lx ly lz xy xz yz.
// fstat[k] |= 1 when a line is left to the host, 2 for a duplicate or unknown id.
__global__ void __launch_bounds__(LT_WARPS * 32)
lt_parse_kernel(const uint4 *__restrict__ bytes, long long nbytes, const long long *__restrict__ starts,
                long long n_lines, const int *__restrict__ frame_of, int n_frames, int natoms, long long P, int H,
                const signed char *__restrict__ role, int n_cols, const long long *__restrict__ ids, int ids_dense,
                const double *__restrict__ params, int scaled, int unwrap, float *__restrict__ coords,
                float *__restrict__ vels, float *__restrict__ forces, long long frame_stride,
                unsigned *__restrict__ bitmap, long long bitmap_words, unsigned char *__restrict__ fstat) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long a = (long long)blockIdx.x * LT_WARPS + warp;
    if (a >= natoms) return;
    const int n_ft = (n_frames + 31) / 32;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k = ft * 32 + lane;
        if (k >= n_frames) continue;
        const long long li = P * frame_of[k] + H + a;
        const long long s = min(max(starts[li], 0LL), nbytes);
        const long long e = min(max(li + 1 < n_lines ? starts[li + 1] : nbytes, s), nbytes);
        LtReader rd{bytes, e};
        long long p = s, id = a + 1;
        double val[LT_NROLE];
        bool ok = true;
        for (int c = 0; c < n_cols && ok; ++c) {
            const int r = role[c];
            if (lt_skip_sep(rd, p) == '\n') {
                ok = false;
                break;
            }
            if (r == LT_SKIP) {
                for (unsigned ch = rd.at(p); !xyz_sep(ch); ch = rd.at(++p))
                    if (ch >= 0x80u) ok = false;
            } else if (r == LT_ID || (r >= LT_IMG && r < LT_IMG + 3)) {
                long long v;
                ok = lt_int(rd, p, v);
                if (r == LT_ID) id = v;
                else val[r] = (double)v;
            } else {
                unsigned long long bits;
                ok = xyz_number<true>(rd, p, bits);
                val[r] = xyz_bits_f64(bits);
            }
        }
        if (!ok) {
            atomicOr(reinterpret_cast<unsigned *>(fstat + (k & ~3)), 1u << (8 * (k & 3)));
            continue;
        }
        long long row = -1;
        if (ids_dense) {
            if (id >= 1 && id <= natoms) row = id - 1;
        } else {
            long long lo = 0, hi = natoms;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (__ldg(ids + mid) < id) lo = mid + 1;
                else hi = mid;
            }
            if (lo < natoms && __ldg(ids + lo) == id) row = lo;
        }
        bool dup = row < 0;
        if (!dup) {
            const unsigned bit = 1u << (row & 31);
            dup = atomicOr(bitmap + (long long)k * bitmap_words + (row >> 5), bit) & bit;
        }
        if (dup) {
            atomicOr(reinterpret_cast<unsigned *>(fstat + (k & ~3)), 2u << (8 * (k & 3)));
            continue;
        }
        const long long o = row * 3 * frame_stride + k;
        if (coords) {
            const double *pk = params + 9LL * k;
            double x = val[LT_POS], y = val[LT_POS + 1], z = val[LT_POS + 2];
            if (scaled) {
                const double xs = x, ys = y, zs = z;
                x = __dadd_rn(__dadd_rn(__dadd_rn(pk[0], __dmul_rn(xs, pk[3])), __dmul_rn(ys, pk[6])),
                              __dmul_rn(zs, pk[7]));
                y = __dadd_rn(__dadd_rn(pk[1], __dmul_rn(ys, pk[4])), __dmul_rn(zs, pk[8]));
                z = __dadd_rn(pk[2], __dmul_rn(zs, pk[5]));
            }
            if (unwrap) {
                const double ix = val[LT_IMG], iy = val[LT_IMG + 1], iz = val[LT_IMG + 2];
                x = __dadd_rn(x, __dadd_rn(__dadd_rn(__dmul_rn(ix, pk[3]), __dmul_rn(iy, pk[6])), __dmul_rn(iz, pk[7])));
                y = __dadd_rn(y, __dadd_rn(__dmul_rn(iy, pk[4]), __dmul_rn(iz, pk[8])));
                z = __dadd_rn(z, __dmul_rn(iz, pk[5]));
            }
            coords[o] = lt_f32(x);
            coords[o + frame_stride] = lt_f32(y);
            coords[o + 2 * frame_stride] = lt_f32(z);
        }
        if (vels) {
#pragma unroll
            for (int d = 0; d < 3; ++d) vels[o + d * frame_stride] = lt_f32(val[LT_VEL + d]);
        }
        if (forces) {
#pragma unroll
            for (int d = 0; d < 3; ++d) forces[o + d * frame_stride] = lt_f32(val[LT_FRC + d]);
        }
    }
}

// the line of item i (frame k = i / (N + 1), j = i % (N + 1); j = 0 is the frame's header, j >= 1 atom j - 1) into
// d, or its length alone when d is null
__device__ __forceinline__ int lt_line(long long i, long long N, const float *__restrict__ coords,
                                       const float *__restrict__ vels, long long frame_stride,
                                       const long long *__restrict__ ids, const long long *__restrict__ types,
                                       unsigned char *d) {
    const long long k = i / (N + 1), a = i - k * (N + 1) - 1;
    unsigned char tmp[2 * G9_INT_MAX + 6 * (G9_MAX + 1) + 2];
    unsigned char *o = d ? d : tmp;
    int n = g9_int(__ldg(ids + a), o);
    o[n++] = ' ';
    n += g9_int(__ldg(types + a), o + n);
    const long long base = a * 3 * frame_stride + k;
    for (int d3 = 0; d3 < 3; ++d3) {
        o[n++] = ' ';
        n += g9_format(__ldg(coords + base + d3 * frame_stride), o + n);
    }
    if (vels)
        for (int d3 = 0; d3 < 3; ++d3) {
            o[n++] = ' ';
            n += g9_format(__ldg(vels + base + d3 * frame_stride), o + n);
        }
    o[n++] = '\n';
    return n;
}

__global__ void __launch_bounds__(256)
lt_len_kernel(long long n_items, long long N, const float *__restrict__ coords, const float *__restrict__ vels,
              long long frame_stride, const long long *__restrict__ ids, const long long *__restrict__ types,
              const long long *__restrict__ head_off, long long *__restrict__ lens) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i > n_items) return;
    if (i == n_items) {
        lens[i] = 0;
        return;
    }
    const long long k = i / (N + 1);
    if (i == k * (N + 1)) lens[i] = head_off[k + 1] - head_off[k];
    else lens[i] = lt_line(i, N, coords, vels, frame_stride, ids, types, nullptr);
}

__global__ void __launch_bounds__(256)
lt_emit_kernel(long long n_items, long long N, const float *__restrict__ coords, const float *__restrict__ vels,
               long long frame_stride, const long long *__restrict__ ids, const long long *__restrict__ types,
               const unsigned char *__restrict__ head, const long long *__restrict__ head_off,
               const long long *__restrict__ offs, unsigned char *__restrict__ out) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n_items) return;
    const long long k = i / (N + 1);
    unsigned char *d = out + offs[i];
    if (i == k * (N + 1)) {
        for (long long c = head_off[k]; c < head_off[k + 1]; ++c) *d++ = head[c];
        return;
    }
    unsigned char line[2 * G9_INT_MAX + 6 * (G9_MAX + 1) + 2];
    const int n = lt_line(i, N, coords, vels, frame_stride, ids, types, line);
    for (int c = 0; c < n; ++c) d[c] = line[c];
}

int lt_chunk_grid(int64_t n, int64_t P, unsigned &blocks) {
    const int64_t frames = n / P + 2;  // a line holds at least its newline
    const int64_t g = cdiv(frames, LT_THREADS);
    if (g > INT32_MAX) return 1;
    blocks = (unsigned)std::max<int64_t>(1, g);
    return 0;
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_lammpstrj_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                                   int64_t file_base, int64_t P, int64_t natoms, const uint8_t *tmpl, int64_t H,
                                   int64_t count_line, int64_t *state, int64_t *frame_off, uint8_t *status,
                                   int64_t frame_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n < 0 || n_read < n || file_base < 0 || frame_cap < 0) return fail(h, MKB_ERR_BAD_ARG, "bad size");
    if (natoms < 1 || natoms > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to 2^31 - 1");
    if (H < 1 || H > INT32_MAX || P != H + natoms || count_line < 0 || count_line >= H)
        return fail(h, MKB_ERR_BAD_ARG, "bad frame layout");
    if (!bytes || !tmpl || !state || (frame_cap && (!frame_off || !status)))
        return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(state) & 7) return fail(h, MKB_ERR_BAD_ARG, "state must be 8-byte aligned");
    if (n == 0) return MKB_OK;
    unsigned blocks;
    if (lt_chunk_grid(n, P, blocks)) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(state + 3, state, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    int rc = xyz_lines<true>(h, st, bytes, n, n_read, file_base, P, natoms, frame_off, status, frame_cap, state,
                             nullptr, 0);
    if (rc) return rc;
    lt_check_kernel<<<blocks, LT_THREADS, 0, st>>>(bytes, n_read, file_base, P, reinterpret_cast<long long *>(state),
                                                   reinterpret_cast<long long *>(frame_off), frame_cap, tmpl, (int)H,
                                                   (int)count_line, natoms, status);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_lammpstrj_head(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                                  int64_t file_base, int64_t P, const int64_t *state, const int64_t *frame_off,
                                  int64_t frame_cap, int64_t step_line, int64_t time_line, int64_t box_line,
                                  int64_t ntilt, int64_t *step, double *time, double *bounds, uint8_t *hstatus) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n < 0 || n_read < n || file_base < 0 || frame_cap < 0 || P < 1) return fail(h, MKB_ERR_BAD_ARG, "bad size");
    if (step_line < 0 || box_line < 0 || box_line + 3 > P || step_line >= P || time_line >= P || time_line < -1 ||
        (ntilt != 0 && ntilt != 1))
        return fail(h, MKB_ERR_BAD_ARG, "bad frame layout");
    if (!bytes || !state || (frame_cap && (!frame_off || !step || !time || !bounds || !hstatus)))
        return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if (n == 0 || frame_cap == 0) return MKB_OK;
    unsigned blocks;
    if (lt_chunk_grid(n, P, blocks)) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    lt_head_kernel<<<blocks, LT_THREADS, 0, st>>>(bytes, n_read, file_base, P, reinterpret_cast<const long long *>(state),
                                                  reinterpret_cast<const long long *>(frame_off), frame_cap,
                                                  (int)step_line, (int)time_line, (int)box_line, (int)ntilt,
                                                  reinterpret_cast<long long *>(step), time, bounds, hstatus);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_lammpstrj_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes,
                                    int64_t n_staged, const int32_t *frame_of, int64_t n_frames, int64_t natoms,
                                    int64_t H, const int8_t *role, int64_t n_cols, const int64_t *ids,
                                    const double *params, int32_t scaled, int32_t unwrap, float *coords, float *vels,
                                    float *forces, int64_t frame_stride, uint8_t *fstat) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || n_staged < 0 || nbytes < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (n_frames >= (1ll << 31) - 32) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (H < 1 || n_cols < 1 || n_cols > 4096) return fail(h, MKB_ERR_BAD_ARG, "bad frame layout");
    if (!bytes || !frame_of || !role || !fstat || (coords && !params)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(vels) |
         reinterpret_cast<uintptr_t>(forces)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords, vels and forces must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(fstat) & 3) return fail(h, MKB_ERR_BAD_ARG, "fstat must be 4-byte aligned");
    for (int64_t k = 0; k < n_frames; ++k)
        if (frame_of[k] < 0 || frame_of[k] >= n_staged)
            return fail(h, MKB_ERR_BAD_ARG, "frame_of[%lld] = %d is not a staged frame (%lld staged)", (long long)k,
                        (int)frame_of[k], (long long)n_staged);
    const int64_t P = H + natoms, n_lines = n_staged * P, words = cdiv(natoms, 32);
    long long *starts, *state;
    int *d_map;
    unsigned *bitmap;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_STARTS, (size_t)n_lines + 1, &starts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_STATE, 1, &state))) return rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_map))) return rc;
    if ((rc = scratch_get(h, S_LMP_BITMAP, (size_t)(n_frames * words), &bitmap))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_map, frame_of, sizeof(int) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(state, 0, sizeof(long long), st));
    MKB_CUDA(h, cudaMemsetAsync(bitmap, 0, sizeof(unsigned) * (size_t)(n_frames * words), st));
    MKB_CUDA(h, cudaMemsetAsync(fstat, 0, (size_t)n_frames, st));
    if ((rc = xyz_lines<false>(h, st, bytes, nbytes, nbytes, 0, P, natoms, nullptr, nullptr, 0,
                               reinterpret_cast<int64_t *>(state), starts, n_lines + 1)))
        return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, LT_WARPS), (unsigned)std::min<int64_t>(cdiv(n_frames, 32), 65535));
    lt_parse_kernel<<<grid, LT_WARPS * 32, 0, st>>>(
        reinterpret_cast<const uint4 *>(bytes), nbytes, starts, n_lines, d_map, (int)n_frames, (int)natoms, P, (int)H,
        reinterpret_cast<const signed char *>(role), (int)n_cols, reinterpret_cast<const long long *>(ids),
        ids == nullptr, params, scaled, unwrap, coords, vels, forces, frame_stride, bitmap, words, fstat);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_lammpstrj_encode(mkb_handle_t h, void *stream, const float *coords, const float *vels,
                                    int64_t frame_stride, int64_t n_frames, int64_t natoms, const int64_t *ids,
                                    const int64_t *types, int64_t line_max, const uint8_t *head,
                                    const int64_t *head_off, int64_t head_bytes, uint8_t *out, int64_t out_capacity,
                                    int64_t *total) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || head_bytes < 0 || out_capacity < 0 || line_max < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (!total) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (!coords || !ids || !types || !out || !head_off || (head_bytes && !head))
        return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const int64_t most = 2 * G9_INT_MAX + 2 + (vels ? 6 : 3) * (G9_MAX + 1);
    if (line_max < 1 || line_max > most) return fail(h, MKB_ERR_BAD_ARG, "line_max must be 1 to %lld", (long long)most);
    if (head_bytes + n_frames * natoms * line_max > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames may take %lld",
                    (long long)out_capacity, (long long)(head_bytes + n_frames * natoms * line_max));
    const int64_t n_items = n_frames * (natoms + 1);
    long long *lens, *offs;
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (long long *)nullptr, (long long *)nullptr,
                                              n_items + 1, st));
    int rc;
    if ((rc = scratch_get(h, S_LMP_LEN, 2 * (size_t)(n_items + 1), &lens))) return rc;
    if ((rc = scratch_get(h, S_LMP_TMP, tmp_bytes, &tmp))) return rc;
    offs = lens + n_items + 1;
    const unsigned blocks = (unsigned)cdiv(n_items + 1, 256);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    lt_len_kernel<<<blocks, 256, 0, st>>>(n_items, natoms, coords, vels, frame_stride,
                                          reinterpret_cast<const long long *>(ids),
                                          reinterpret_cast<const long long *>(types),
                                          reinterpret_cast<const long long *>(head_off), lens);
    MKB_LAUNCHED(h);
    MKB_CUDA(h, cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, lens, offs, n_items + 1, st));
    MKB_CUDA(h, cudaMemcpyAsync(total, offs + n_items, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    lt_emit_kernel<<<(unsigned)cdiv(n_items, 256), 256, 0, st>>>(
        n_items, natoms, coords, vels, frame_stride, reinterpret_cast<const long long *>(ids),
        reinterpret_cast<const long long *>(types), head, reinterpret_cast<const long long *>(head_off), offs, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
