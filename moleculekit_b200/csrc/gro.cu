// gro.cu -- K29: multi-frame GROMACS GRO trajectories indexed, parsed and formatted on the device.
//
// Replaces the host path of a GRO reader that walks every line, slices the fixed-width position (and velocity) columns
// and calls float() on each.  A frame is P = N + 3 lines: a title, the atom count, N atom lines "%5d%-5s%5s%5d" then
// three position fields of width w (and optionally three velocity fields of width w), and a free-format box line.
// Atom lines have no fixed size across files (w and the velocities vary) and titles have none at all, so every line
// must be found before it can be parsed.
//
//   index   over the file in chunks (mkb_gro_index): K26's newline count and scan (xl_lines.cuh), then gro_emit_kernel
//           keeps the file offset of every title line (L % P == 0) and checks every count line (L % P == 1) against N
//           with xyz_count_line (gro_count_line); a CR not followed by LF atomicMins its file offset.  The running line
//           count makes the chunks independent of each other: no host sync per chunk.
//   decode  over staged whole frames (mkb_gro_decode): xyz_lines<false> stores every line start, so atom a of staged
//           frame u is line P u + 2 + a, and gro_parse_kernel maps K23's tile (32 frames x 32 atoms per CTA of 256
//           threads): a thread checks that its line holds the columns the file needs, parses its fields into shared
//           tiles, and the warps store the tiles along frames into the (N, 3, F) positions and velocities.  A line the
//           device does not decide is appended to a list for the host.
//   head    mkb_gro_head: one thread per staged frame parses its box line (3 or 9 tokens) and the numbers after " t= "
//           and " step= " in its title.
//   encode  the inverse (mkb_gro_encode): a CTA loads 32 frames x 32 atoms along frames, each warp builds its 32 atoms'
//           lines (the host's 20-byte prefix, '%8.3f' positions, '%8.4f' velocities) in a shared-memory image and
//           stores it with aligned 32-bit words; the CTAs of the first atom tile copy each frame's title and count
//           lines, those of the last format its box line ('%10.5f').
//
// Arithmetic: with w = 8 a position goes through K25's F8.3 fast path (md_parse) and a velocity through the F8.4 one
// (md_parse4, f83.cuh); any other width, and every field the fast paths reject, through K26's general grammar inside
// the field (gro_field), so every decided field is bit for bit np.float32(float(field)).  The title's time goes
// through the same grammar to a double, float(token).  The formats use md_format and f_format: rint(x 10^d) in double
// is exact for d <= 12 and rounds half to even, as printf does.
#include <cub/block/block_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "f83.cuh"
#include "frame_tile.cuh"
#include "xl_lines.cuh"
#include "xyz_number.cuh"

namespace mkb {
namespace {

constexpr int GRO_PREFIX = 20;     // "%5d%-5s%5s%5d": resid, resname, atom name, serial
constexpr int GRO_MAX_WIDTH = 32;  // widest field the decoder takes
constexpr int GRO_LINE_X = 45;     // a written atom line with positions, '\n' included
constexpr int GRO_LINE_XV = 69;    // ... with positions and velocities
constexpr int GRO_BOX_FIELD = 10;  // '%10.5f'
constexpr int GRO_HEAD_THREADS = 128;
// the (vector, component) of the box's GRO-order fields v1x v2y v3z v1y v1z v2x v2z v3x v3y, as 3 i + j per nibble
constexpr unsigned long long GRO_BOX_ORDER = 0x765321840ull;

// bytes [p, end) of a buffer one at a time; '\n' at and past end (the end of a fixed-width field)
struct GroFieldReader {
    const unsigned char *b;
    long long end;
    __device__ __forceinline__ unsigned at(long long p) const { return p < end ? __ldg(b + p) : '\n'; }
};

// The whitespace bytes.split() splits on and float() strips from bytes: \t \n \v \f \r and space.  K26's xyz_sep also
// takes 0x1c-0x1f (str.split() splits on them), but the GRO reader works on bytes, where float() and int() reject
// them, so a GRO field or token holding one is left to the host.
__device__ __forceinline__ bool gro_sep(unsigned c) { return c == ' ' || (c >= 9u && c <= 13u); }

// xyz_count_line's check of the count line at b[p], and 1 (the host decides) when the line holds a byte 0x1c-0x1f
// within the bytes that check reads
__device__ __forceinline__ unsigned char gro_count_line(const unsigned char *__restrict__ b, long long p,
                                                        long long n_read, long long natoms) {
    const long long e = min(n_read, p + XYZ_COUNT_WINDOW);
    for (long long q = p; q < e && b[q] != '\n'; ++q)
        if (b[q] - 0x1cu < 4u) return 1;
    return xyz_count_line(b, p, n_read, natoms);
}

// the fixed-width field b[s, s + width) as float() reads its bytes: gro_sep whitespace, one number of K26's grammar,
// gro_sep whitespace.  false: the host decides (an empty field, anything outside the grammar, an undecided rounding).
__device__ __forceinline__ bool gro_field(const unsigned char *__restrict__ b, long long s, int width, unsigned &bits) {
    GroFieldReader rd{b, s + width};
    long long p = s;
    while (p < rd.end && gro_sep(rd.at(p))) ++p;
    if (p == rd.end || !xyz_number(rd, p, bits)) return false;
    for (; p < rd.end; ++p)
        if (!gro_sep(rd.at(p))) return false;
    return true;
}

// INDEX: lines numbered from state[0]'s value before the scan; the title line of frame f (L = f P) gets frame_off[f] =
// file_base + its byte, its count line (L = f P + 1) status[f] = gro_count_line's check (f >= frame_cap: state[2] =
// max f + 1); a lone CR atomicMins file_base + its byte into state[1].
__global__ void __launch_bounds__(XL_THREADS)
gro_emit_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, const long long *__restrict__ base,
                long long file_base, long long P, long long natoms, long long *__restrict__ frame_off,
                unsigned char *__restrict__ status, long long frame_cap, long long *__restrict__ state) {
    using Scan = cub::BlockScan<unsigned, XL_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const unsigned char *b = reinterpret_cast<const unsigned char *>(bytes);
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    long long g0 = base[blockIdx.x];  // number of the first newline of the segment
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        unsigned nl = 0, cr = 0;
        if (p0 < n) {
            const uint4 v = __ldg(bytes + wi);
            const unsigned ok = xl_valid(p0, n);
            nl = xl_mask(v, '\n') & ok;
            cr = xl_mask(v, '\r') & ok;
        }
        unsigned ex, total;
        Scan(tmp).ExclusiveSum((unsigned)__popc(nl), ex, total);
        long long g = g0 + ex;
        for (; nl; nl &= nl - 1, ++g) {
            const long long pos = p0 + __ffs(nl) - 1, L = g + 1, r = L % P;
            if (r > 1 || pos + 1 >= n_read) continue;
            const long long f = L / P;
            if (f >= frame_cap) {
                atomicMax(reinterpret_cast<unsigned long long *>(state + 2), (unsigned long long)(f + 1));
            } else if (r == 0) {
                frame_off[f] = file_base + pos + 1;
            } else {
                status[f] = gro_count_line(b, pos + 1, n_read, natoms);
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

// The atom line [s, e) (e: its '\n' or the end of the bytes): false when it holds fewer than `cols` characters before
// its line end, or a field the device does not decide.  Field d (positions 0-2, velocities 3-5 with VEL) is stored at
// col[gro_slot(d)], col pointing at the atom's x position in the parse kernel's tile.
__device__ __forceinline__ int gro_slot(int d) { return (d >= 3 ? FT_W * (FT_T + 1) : 0) + (d % 3) * (FT_T + 1); }

template <bool VEL>
__device__ __forceinline__ bool gro_line(const unsigned char *__restrict__ b, long long s, long long e, int w, int cols,
                                         unsigned *col) {
    if (e > s && b[e - 1] == '\r') --e;
    if (e - s < cols) return false;
    constexpr int NF = VEL ? 6 : 3;
    unsigned miss = (1u << NF) - 1u;
    if (w == 8) {
        miss = 0;
#pragma unroll
        for (int d = 0; d < NF; ++d) {
            unsigned lo, hi, next;
            md_field(b + s + GRO_PREFIX + 8 * d, lo, hi, next);
            bool ok;
            col[gro_slot(d)] = d < 3 ? md_parse(lo, hi, ok) : md_parse4(lo, hi, ok);
            miss |= (unsigned)!ok << d;
        }
    }
#pragma unroll 1
    for (; miss; miss &= miss - 1) {
        const int d = __ffs(miss) - 1;
        unsigned bits;
        if (!gro_field(b, s + GRO_PREFIX + (long long)w * d, w, bits)) return false;
        col[gro_slot(d)] = bits;
    }
    return true;
}

// coords[(a*3 + d)*frame_stride + k] = position field d of atom line a of listed frame k, staged frame frame_of[k]
// (line starts[P u + 2 + a]); with VEL vels[...] = velocity field d the same way.  A line shorter than `cols`
// characters or with a field the device does not decide appends (frame_base + k) * natoms + a to flags[1 ...] (flags[0]
// counts them; entries past flag_cap are dropped).
template <bool VEL>
__global__ void __launch_bounds__(FT_WARPS * 32)
gro_parse_kernel(const unsigned char *__restrict__ bytes, long long nbytes, const long long *__restrict__ starts,
                 long long n_lines, const int *__restrict__ frame_of, int n_frames, int natoms, long long P, int w,
                 int cols, float *__restrict__ coords, float *__restrict__ vels, long long frame_stride,
                 long long frame_base, unsigned long long *__restrict__ flags, long long flag_cap) {
    constexpr int NT = VEL ? 2 : 1;
    __shared__ unsigned tile[NT][FT_W][FT_T + 1];  // [positions, velocities][value][frame]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a = blockIdx.x * 32 + lane, v0 = blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile is stored
#pragma unroll
        for (int j = 0; j < FT_T / FT_WARPS; ++j) {
            const int fl = warp + FT_WARPS * j, k = k0 + fl;
            if (k < n_frames && a < natoms) {
                const long long li = P * frame_of[k] + 2 + a;
                const long long s = min(max(starts[li], 0LL), nbytes);
                const long long e = min(max(li + 1 < n_lines ? starts[li + 1] - 1 : nbytes, s), nbytes);
                if (!gro_line<VEL>(bytes, s, e, w, cols, &tile[0][3 * lane][fl])) {
                    const unsigned long long slot = atomicAdd(flags, 1ull);
                    if ((long long)slot < flag_cap) flags[1 + slot] = (unsigned long long)((frame_base + k) * natoms + a);
                }
            }
        }
        __syncthreads();
        const int k = k0 + lane;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            unsigned *dst = reinterpret_cast<unsigned *>(t ? vels : coords);
#pragma unroll
            for (int i = 0; i < FT_ITEMS; ++i) {
                const int r = warp + FT_WARPS * i;
                if (v0 + r < 3 * natoms && k < n_frames)
                    __stcs(dst + (long long)(v0 + r) * frame_stride + k, tile[t][r][lane]);
            }
        }
    }
}

__host__ __device__ constexpr unsigned long long gro_tag(const char *s, int n) {
    unsigned long long w = 0;
    for (int i = n - 1; i >= 0; --i) w = (w << 8) | (unsigned char)s[i];
    return w;
}

// Staged frame u is bytes [at[u], at[u + 1]).  Its last line: up to 9 whitespace-separated tokens into box[9 u ...] in
// file order (float32 bits); the number after the first " t= " of its first line into time[u] (float64 bits, NaN
// without one), the integer after the first " step= " into step[u] (-1 without one).  status[u]: bit 0 the box line
// holds a token count other than 3 or 9 or a token the device does not decide, bit 1 the time token, bit 2 the step
// token is left to the host (a line holding a byte 0x1c-0x1f goes to the host whole).
__global__ void __launch_bounds__(GRO_HEAD_THREADS)
gro_head_kernel(const unsigned char *__restrict__ bytes, const long long *__restrict__ at, int n,
                unsigned *__restrict__ box, unsigned long long *__restrict__ time, long long *__restrict__ step,
                int *__restrict__ status) {
    const int u = blockIdx.x * GRO_HEAD_THREADS + threadIdx.x;
    if (u >= n) return;
    const long long s = at[u], e = at[u + 1];
    int st = 0;
    // the box line [bs, be)
    long long be = e;
    if (be > s && __ldg(bytes + be - 1) == '\n') --be;
    long long bs = be;
    bool odd = false;  // a byte 0x1c-0x1f, which xyz_sep takes as whitespace and bytes.split() does not
    while (bs > s && __ldg(bytes + bs - 1) != '\n') {
        --bs;
        odd |= __ldg(bytes + bs) - 0x1cu < 4u;
    }
    if (odd) {
        st |= 1;
    } else {  // xyz_sep is gro_sep on this line
        GroFieldReader rd{bytes, be};
        long long p = bs;
        int nt = 0;
        for (;;) {
            while (p < be && xyz_sep(rd.at(p))) ++p;
            if (p == be) break;
            unsigned bits;
            if (nt == 9 || !xyz_number(rd, p, bits)) {
                st |= 1;
                break;
            }
            box[9ll * u + nt++] = bits;
        }
        if (nt != 3 && nt != 9) st |= 1;
    }
    // the title [s, te): the first " t= " and " step= "
    constexpr unsigned T_TAG = (unsigned)gro_tag(" t= ", 4);
    constexpr unsigned long long STEP_TAG = gro_tag(" step= ", 7);
    long long te = s, tq = -1, sq = -1;
    unsigned w4 = 0;
    unsigned long long w8 = 0;
    odd = false;
    for (; te < e; ++te) {
        const unsigned c = __ldg(bytes + te);
        if (c == '\n') break;
        odd |= c - 0x1cu < 4u;
        w4 = (w4 >> 8) | (c << 24);
        w8 = (w8 >> 8) | ((unsigned long long)c << 56);
        if (tq < 0 && te - s >= 3 && w4 == T_TAG) tq = te + 1;
        if (sq < 0 && te - s >= 6 && (w8 >> 8) == STEP_TAG) sq = te + 1;
    }
    GroFieldReader rd{bytes, te};
    unsigned long long tb = 0x7ff8000000000000ull;  // NaN without " t= "
    if (odd) {  // the host splits the title's bytes
        st |= (tq >= 0 ? 2 : 0) | (sq >= 0 ? 4 : 0);
        tq = sq = -1;
    }
    if (tq >= 0) {
        long long p = tq;
        while (p < te && xyz_sep(rd.at(p))) ++p;
        if (p == te || !xyz_number<true>(rd, p, tb)) st |= 2;
    }
    long long sv = -1;
    if (sq >= 0) {
        long long p = sq;
        while (p < te && xyz_sep(rd.at(p))) ++p;
        unsigned c = rd.at(p);
        const bool neg = c == '-';
        if (c == '+' || c == '-') c = rd.at(++p);
        long long v = 0;
        int nd = 0;
        for (; xyz_digit(c) && nd < 18; c = rd.at(++p), ++nd) v = 10 * v + (c - '0');
        if (nd == 0 || !xyz_sep(c)) st |= 4;
        else sv = neg ? -v : v;
    }
    time[u] = tb;
    step[u] = sv;
    status[u] = st;
}

// Frame k of out is out[k*S ...], S = head_bytes + natoms*L + (box9 ? 91 : 31), L = 69 with VEL else 45: the frame's
// head_bytes bytes of head (head[k*head_bytes ...]: its title and count lines), per atom its 20-byte prefix
// prefix[a*20 ...], '%8.3f' of coords[(a*3 + d)*frame_stride + k] for d = 0, 1, 2, with VEL '%8.4f' of vels[...] the
// same way, and '\n'; then the box line: '%10.5f' of box[(3 i + j)*box_stride + k] for the GRO-order (i, j) of its 3
// or 9 fields, and '\n'.  prefix and out are 4-byte aligned.
template <bool VEL>
__global__ void __launch_bounds__(FT_WARPS * 32)
gro_encode_kernel(const float *__restrict__ coords, const float *__restrict__ vels, long long frame_stride,
                  int n_frames, int natoms, const unsigned char *__restrict__ head, int head_bytes,
                  const unsigned char *__restrict__ prefix, const float *__restrict__ box, long long box_stride,
                  int box9, long long S, unsigned char *__restrict__ out) {
    constexpr int NT = VEL ? 2 : 1, L = VEL ? GRO_LINE_XV : GRO_LINE_X;
    constexpr int ROW = (32 * L + 8 + 15) & ~15;
    __shared__ float tile[NT][FT_W][FT_T + 1];  // [positions, velocities][value][frame]
    __shared__ __align__(16) unsigned char img_all[FT_WARPS][ROW];
    __shared__ unsigned char box_all[FT_WARPS][9 * GRO_BOX_FIELD + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *img = img_all[warp];
    const int a0 = blockIdx.x * 32, v0 = blockIdx.x * FT_W, na = min(32, natoms - a0);
    const int nb = box9 ? 9 : 3, BL = nb * GRO_BOX_FIELD + 1;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile is formatted
#pragma unroll
        for (int t = 0; t < NT; ++t) {
            const float *src = t ? vels : coords;
#pragma unroll
            for (int i = 0; i < FT_ITEMS; ++i) {
                const int r = warp + FT_WARPS * i, k = k0 + lane;
                tile[t][r][lane] = v0 + r < 3 * natoms && k < n_frames
                                       ? __ldcs(src + (long long)(v0 + r) * frame_stride + k) : 0.f;
            }
        }
        __syncthreads();
        for (int j = 0; j < FT_T / FT_WARPS; ++j) {
            const int fl = warp + FT_WARPS * j, k = k0 + fl;
            if (k >= n_frames) break;
            if (blockIdx.x == 0)  // the frame's title and count lines
                for (int c = lane; c < head_bytes; c += 32)
                    out[(long long)k * S + c] = __ldg(head + (long long)k * head_bytes + c);
            if (a0 + na == natoms) {  // the last atom tile ends the frame with its box line
                unsigned char *bl = box_all[warp];
                if (lane < nb) {
                    const int ij = (int)((GRO_BOX_ORDER >> (4 * lane)) & 15u);
                    f_format<GRO_BOX_FIELD, 5>(__ldg(box + ij * box_stride + k), bl + GRO_BOX_FIELD * lane);
                }
                if (lane == 0) bl[BL - 1] = '\n';
                __syncwarp();
                for (int c = lane; c < BL; c += 32) out[(long long)k * S + S - BL + c] = bl[c];
                __syncwarp();
            }
            const long long g0 = (long long)k * S + head_bytes + (long long)a0 * L;
            const int sh = (int)(g0 & 3), span = na * L;
            if (lane < na) {
                unsigned char *d = img + sh + lane * L;
                const unsigned *pw = reinterpret_cast<const unsigned *>(prefix + (long long)(a0 + lane) * GRO_PREFIX);
#pragma unroll
                for (int m = 0; m < GRO_PREFIX / 4; ++m) {
                    const unsigned w = __ldg(pw + m);
#pragma unroll
                    for (int c = 0; c < 4; ++c) d[4 * m + c] = (unsigned char)(w >> (8 * c));
                }
#pragma unroll
                for (int x = 0; x < 3; ++x) {
                    unsigned lo, hi;
                    md_format(tile[0][3 * lane + x][fl], lo, hi);
                    md_put(d + GRO_PREFIX + 8 * x, lo, hi);
                }
                if (VEL) {
#pragma unroll
                    for (int x = 0; x < 3; ++x)
                        f_format<8, 4>(tile[NT - 1][3 * lane + x][fl], d + GRO_PREFIX + 24 + 8 * x);
                }
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

extern "C" int mkb_gro_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
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
    const int64_t n_seg = std::max<int64_t>(1, cdiv(n, XL_SEG));
    if (n_seg > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    unsigned *counts;
    long long *base;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_COUNTS, (size_t)n_seg, &counts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_BASE, (size_t)n_seg, &base))) return rc;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const uint4 *b = reinterpret_cast<const uint4 *>(bytes);
    xyz_count_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, counts);
    MKB_LAUNCHED(h);
    xyz_scan_kernel<<<1, XL_SCAN_THREADS, 0, st>>>(counts, (int)n_seg, base, reinterpret_cast<long long *>(state));
    MKB_LAUNCHED(h);
    gro_emit_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, n_read, base, file_base, natoms + 3, natoms,
                                                            reinterpret_cast<long long *>(frame_off), status, frame_cap,
                                                            reinterpret_cast<long long *>(state));
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_gro_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                              const int32_t *frame_of, int64_t n_frames, int64_t natoms, int64_t width,
                              int32_t velocities, float *coords, float *vels, int64_t frame_stride, int64_t frame_base,
                              int64_t *flags, int64_t flag_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || n_staged < 0 || nbytes < 0 || frame_base < 0 || flag_cap < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (width < 1 || width > GRO_MAX_WIDTH)
        return fail(h, MKB_ERR_BAD_ARG, "field width must be 1 to %d, got %lld", GRO_MAX_WIDTH, (long long)width);
    if (vels && !velocities) return fail(h, MKB_ERR_BAD_ARG, "vels needs a file with velocities");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!bytes || !frame_of || !coords || !flags) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if (((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(vels)) & 3) ||
        (reinterpret_cast<uintptr_t>(flags) & 7))
        return fail(h, MKB_ERR_BAD_ARG, "coords and vels must be 4-byte and flags 8-byte aligned");
    for (int64_t k = 0; k < n_frames; ++k)
        if (frame_of[k] < 0 || frame_of[k] >= n_staged)
            return fail(h, MKB_ERR_BAD_ARG, "frame_of[%lld] = %d is not a staged frame (%lld staged)", (long long)k,
                        (int)frame_of[k], (long long)n_staged);
    const int64_t P = natoms + 3, n_lines = n_staged * P;
    const int cols = GRO_PREFIX + (velocities ? 6 : 3) * (int)width;
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
    auto *fl = reinterpret_cast<unsigned long long *>(flags);
    if (vels)
        gro_parse_kernel<true><<<grid, FT_WARPS * 32, 0, st>>>(bytes, nbytes, starts, n_lines, d_map, (int)n_frames,
                                                               (int)natoms, P, (int)width, cols, coords, vels,
                                                               frame_stride, frame_base, fl, flag_cap);
    else
        gro_parse_kernel<false><<<grid, FT_WARPS * 32, 0, st>>>(bytes, nbytes, starts, n_lines, d_map, (int)n_frames,
                                                                (int)natoms, P, (int)width, cols, coords, nullptr,
                                                                frame_stride, frame_base, fl, flag_cap);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_gro_head(mkb_handle_t h, void *stream, const uint8_t *bytes, const int64_t *frame_at,
                            int64_t n_staged, float *box, double *time, int64_t *step, int32_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_staged < 0 || n_staged > INT32_MAX - GRO_HEAD_THREADS) return fail(h, MKB_ERR_BAD_ARG, "bad n_staged");
    if (n_staged == 0) return MKB_OK;
    if (!bytes || !frame_at || !box || !time || !step || !status) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (((reinterpret_cast<uintptr_t>(frame_at) | reinterpret_cast<uintptr_t>(time) |
          reinterpret_cast<uintptr_t>(step)) & 7) ||
        ((reinterpret_cast<uintptr_t>(box) | reinterpret_cast<uintptr_t>(status)) & 3))
        return fail(h, MKB_ERR_BAD_ARG, "frame_at, time and step must be 8-byte, box and status 4-byte aligned");
    gro_head_kernel<<<(unsigned)cdiv(n_staged, GRO_HEAD_THREADS), GRO_HEAD_THREADS, 0, st>>>(
        bytes, reinterpret_cast<const long long *>(frame_at), (int)n_staged, reinterpret_cast<unsigned *>(box),
        reinterpret_cast<unsigned long long *>(time), reinterpret_cast<long long *>(step), status);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_gro_encode(mkb_handle_t h, void *stream, const float *coords, const float *vels,
                              int64_t frame_stride, int64_t n_frames, int64_t natoms, const uint8_t *head,
                              int64_t head_bytes, const uint8_t *prefix, const float *box, int64_t box_stride,
                              int32_t box9, uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || head_bytes < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / GRO_LINE_XV) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 69");
    if (head_bytes > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "head too long");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!coords || !prefix || !box || !out || (head_bytes && !head)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(vels) | reinterpret_cast<uintptr_t>(prefix) |
         reinterpret_cast<uintptr_t>(box) | reinterpret_cast<uintptr_t>(out)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords, vels, prefix, box and out must be 4-byte aligned");
    if (frame_stride < n_frames || box_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const int64_t L = vels ? GRO_LINE_XV : GRO_LINE_X;
    const int64_t S = head_bytes + natoms * L + (box9 ? 9 : 3) * GRO_BOX_FIELD + 1;
    if (n_frames * S > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * S));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    if (vels)
        gro_encode_kernel<true><<<grid, FT_WARPS * 32, 0, st>>>(coords, vels, frame_stride, (int)n_frames, (int)natoms,
                                                                head, (int)head_bytes, prefix, box, box_stride,
                                                                box9 != 0, S, out);
    else
        gro_encode_kernel<false><<<grid, FT_WARPS * 32, 0, st>>>(coords, nullptr, frame_stride, (int)n_frames,
                                                                 (int)natoms, head, (int)head_bytes, prefix, box,
                                                                 box_stride, box9 != 0, S, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
