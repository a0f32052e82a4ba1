// pdb.cu -- K28: multi-model PDB trajectories indexed, parsed and formatted on the device.
//
// Replaces the host path of a PDB reader that walks every line, keeps the ATOM / HETATM records and calls float() on
// the column slices [30:38], [38:46] and [46:54] of each.  A frame is the atom records of one MODEL; other records (TER,
// ANISOU, REMARK, ...) can sit between them, so a frame has no fixed size and its atom lines must be found before they
// can be parsed.
//
//   records  a line start is byte 0 of the span (when the caller says it starts a line) or the byte after a '\n'; its
//            first six bytes classify it (pdb_record): ATOM / HETATM, MODEL, ENDMDL, END, CRYST1 or other.
//   index    over the file in chunks (mkb_pdb_index), in three launches per chunk: pdb_count_kernel counts the atom
//            records that start in each 32 KB segment, xl_lines.cuh's scan turns the counts into each segment's first
//            atom number and advances a running atom count kept on the device, and pdb_emit_kernel<true> appends every
//            MODEL / ENDMDL / END / CRYST1 record to a list as (file offset * 8 + kind, atom records before it).  A CR
//            not followed by LF atomicMins its file offset.  The chunks are independent of each other: no host sync per
//            chunk; the host derives the frames from the O(F) list.
//   decode   over staged whole frames (mkb_pdb_decode), each holding exactly natoms atom records: the same count and
//            scan, and pdb_emit_kernel<false> stores the start of every atom record by its rank, so a TER or ANISOU
//            between atoms costs nothing.  Then pdb_parse_kernel maps K23's tile (32 frames x 32 atoms per CTA of 256
//            threads): a thread parses the three fields of one atom line into a shared-memory tile, and the warps store
//            the tile along frames.  A line the device does not decide is appended to a list for the host.
//   cells    mkb_pdb_cell parses the six fields of staged CRYST1 lines (a, b, c: %9.3f in columns 7-33; alpha, beta,
//            gamma: %7.2f in columns 34-54), one thread per line.
//   encode   the inverse (mkb_pdb_encode): a CTA loads 32 frames x 32 atoms along frames, each warp copies its 32 atoms'
//            81-byte template lines into a shared-memory image, writes their three '%8.3f' fields and stores the image
//            with aligned 32-bit words; the CTAs of the first atom tile write each frame's MODEL and CRYST1 lines, those
//            of the last its ENDMDL line.
//
// Arithmetic: a field goes through K25's F8.3 fast path (md_parse, f83.cuh) first, and anything else through K26's
// general grammar (xyz_number.cuh) with the field's end as a separator, so every decided field is bit for bit
// np.float32(float(field)).  The formats use md_format ('%8.3f') and f_format ('%9.3f', '%7.2f'): rint(x 10^d) in
// double is exact for d <= 3 and rounds half to even, as printf does.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "f83.cuh"
#include "frame_tile.cuh"
#include "xl_lines.cuh"
#include "xyz_number.cuh"

namespace mkb {
namespace {

constexpr int PDB_LINE = 81;      // a written atom line, '\n' included
constexpr int PDB_COLS = 54;      // columns an atom line must hold (through the z field)
constexpr int PDB_MODEL = 15;     // "MODEL %8d\n"
constexpr int PDB_CRYST = 71;     // "CRYST1%9.3f%9.3f%9.3f%7.2f%7.2f%7.2f P 1           1\n"
constexpr int PDB_ENDMDL = 7;     // "ENDMDL\n"
constexpr int PDB_CELL_ROW = 64;  // bytes per staged CRYST1 line
constexpr int PDB_CELL_THREADS = 128;

enum : int { REC_OTHER = 0, REC_ATOM = 1, REC_MODEL = 2, REC_ENDMDL = 3, REC_END = 4, REC_CRYST1 = 5 };

__host__ __device__ constexpr unsigned long long pdb_tag(const char *s, int n) {
    unsigned long long w = 0;
    for (int i = n - 1; i >= 0; --i) w = (w << 8) | (unsigned char)s[i];
    return w;
}

// the record of the line starting at b[p]; bytes at and past n_read read as '\n'
__device__ __forceinline__ int pdb_record(const unsigned char *__restrict__ b, long long p, long long n_read) {
    unsigned long long w = 0;
#pragma unroll
    for (int i = 5; i >= 0; --i) w = (w << 8) | (p + i < n_read ? b[p + i] : (unsigned char)'\n');
    const unsigned c3 = (unsigned)(w >> 24) & 0xffu, c5 = (unsigned)(w >> 40) & 0xffu;
    const bool end3 = c3 == ' ' || c3 == '\r' || c3 == '\n', end5 = c5 == ' ' || c5 == '\r' || c5 == '\n';
    constexpr unsigned long long ATOM = pdb_tag("ATOM  ", 6), HETATM = pdb_tag("HETATM", 6), MODEL = pdb_tag("MODEL", 5),
                                 ENDMDL = pdb_tag("ENDMDL", 6), END = pdb_tag("END", 3), CRYST1 = pdb_tag("CRYST1", 6);
    if (w == ATOM || w == HETATM) return REC_ATOM;
    if ((w & 0xffffffffffull) == MODEL && end5) return REC_MODEL;
    if (w == ENDMDL) return REC_ENDMDL;
    if ((w & 0xffffffull) == END && end3) return REC_END;
    if (w == CRYST1) return REC_CRYST1;
    return REC_OTHER;
}

// counts[s] = the atom records starting in segment s of bytes[0, n) (a line start after a '\n' in the segment; byte 0
// too when `first`)
__global__ void __launch_bounds__(XL_THREADS) pdb_count_kernel(const uint4 *__restrict__ bytes, long long n,
                                                               long long n_read, int first,
                                                               unsigned *__restrict__ counts) {
    using Reduce = cub::BlockReduce<unsigned, XL_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    const unsigned char *b = reinterpret_cast<const unsigned char *>(bytes);
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    unsigned c = first && blockIdx.x == 0 && threadIdx.x == 0 && pdb_record(b, 0, n_read) == REC_ATOM;
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        if (p0 >= n) break;
        for (unsigned nl = xl_mask(__ldg(bytes + wi), '\n') & xl_valid(p0, n); nl; nl &= nl - 1)
            c += pdb_record(b, p0 + __ffs(nl), n_read) == REC_ATOM;
    }
    const unsigned total = Reduce(tmp).Sum(c);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// Atom records numbered from state[0]'s value before the scan (base[s]: the first of segment s).
// INDEX: every MODEL / ENDMDL / END / CRYST1 record at byte p appends ((file_base + p) * 8 + kind, atom records before
// it) to marks[2 j], marks[2 j + 1] for j = atomicAdd(state[2], 1) < mark_cap; a CR not followed by LF atomicMins
// file_base + its byte into state[1].  Otherwise: starts[r] = the byte of atom record r for r < starts_cap.
template <bool INDEX>
__global__ void __launch_bounds__(XL_THREADS)
pdb_emit_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, int first,
                const long long *__restrict__ base, long long file_base, long long *__restrict__ marks,
                long long mark_cap, long long *__restrict__ state, long long *__restrict__ starts,
                long long starts_cap) {
    using Scan = cub::BlockScan<unsigned, XL_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const unsigned char *b = reinterpret_cast<const unsigned char *>(bytes);
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    long long g0 = base[blockIdx.x];  // atom records before the segment
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        // line starts of this thread: bit j of nl (the byte after newline p0 + j), and byte 0 (zc) for the first one
        const bool zero = first && i == 0 && blockIdx.x == 0 && threadIdx.x == 0;
        const int zc = zero ? pdb_record(b, 0, n_read) : REC_OTHER;
        unsigned nl = 0, cr = 0, am = 0, mm = 0;
        if (p0 < n) {
            const uint4 v = __ldg(bytes + wi);
            const unsigned ok = xl_valid(p0, n);
            nl = xl_mask(v, '\n') & ok;
            if (INDEX) cr = xl_mask(v, '\r') & ok;
            for (unsigned m = nl; m; m &= m - 1) {
                const int j = __ffs(m) - 1, rc = pdb_record(b, p0 + j + 1, n_read);
                if (rc == REC_ATOM) am |= 1u << j;
                else if (rc != REC_OTHER) mm |= 1u << j;
            }
        }
        const unsigned za = zc == REC_ATOM;
        unsigned ex, total;
        Scan(tmp).ExclusiveSum(__popc(am) + za, ex, total);
        const long long g = g0 + ex;  // atom records before this thread's first line start
        if (INDEX) {
            auto mark = [&](long long p, int kind, long long before) {
                const unsigned long long j = atomicAdd(reinterpret_cast<unsigned long long *>(state + 2), 1ull);
                if ((long long)j < mark_cap) {
                    marks[2 * j] = (file_base + p) * 8 + kind;
                    marks[2 * j + 1] = before;
                }
            };
            if (zc != REC_OTHER && !za) mark(0, zc, g);
            for (; mm; mm &= mm - 1) {
                const int j = __ffs(mm) - 1;
                mark(p0 + j + 1, pdb_record(b, p0 + j + 1, n_read), g + za + __popc(am & ((1u << j) - 1u)));
            }
            for (; cr; cr &= cr - 1) {
                const long long pos = p0 + __ffs(cr) - 1;
                if (pos + 1 < n_read && b[pos + 1] != '\n')
                    atomicMin(reinterpret_cast<unsigned long long *>(state + 1), (unsigned long long)(file_base + pos));
            }
        } else {
            long long r = g;
            if (za && r < starts_cap) starts[r] = 0;
            r += za;
            for (; am; am &= am - 1, ++r)
                if (r < starts_cap) starts[r] = p0 + __ffs(am);
        }
        g0 += total;
        __syncthreads();  // tmp is reused by the next item's scan
    }
}

// a '\n' or '\r' among bytes [s, s + PDB_COLS) (the caller keeps s + PDB_COLS + 3 inside the buffer)
__device__ __forceinline__ bool pdb_short(const unsigned char *__restrict__ b, long long s) {
    const unsigned *w = reinterpret_cast<const unsigned *>(reinterpret_cast<uintptr_t>(b + s) & ~uintptr_t(3));
    const int sh = (int)(reinterpret_cast<uintptr_t>(b + s) & 3u);
    bool hit = false;
#pragma unroll
    for (int j = 0; j < (PDB_COLS + 3 + 3) / 4; ++j) {
        const unsigned x = __ldg(w + j);
        unsigned z = (~md_nonzero(x ^ 0x0a0a0a0au) | ~md_nonzero(x ^ 0x0d0d0d0du)) & 0x80808080u;
        if (j == 0) z &= 0x80808080u << (8 * sh);                          // bytes before s
        const int last = sh + PDB_COLS - 4 * j;                            // bytes of this word before s + PDB_COLS
        if (last < 4) z &= last <= 0 ? 0u : 0x80808080u >> (8 * (4 - last));
        hit |= z != 0u;
    }
    return hit;
}

// bytes [p, end) of a buffer one at a time; '\n' at and past end (the end of a fixed-width field)
struct PdbField {
    const unsigned char *b;
    long long end;
    __device__ __forceinline__ unsigned at(long long p) const { return p < end ? __ldg(b + p) : '\n'; }
};

// the fixed-width field b[s, s + width) as float() reads it: separators, a number in K26's grammar, separators.
// false: the host decides (an empty field, anything outside the grammar, an undecided rounding).
__device__ __forceinline__ bool pdb_general(const unsigned char *__restrict__ b, long long s, int width,
                                            unsigned &bits) {
    PdbField rd{b, s + width};
    long long p = s;
    while (p < rd.end && xyz_sep(rd.at(p))) ++p;
    if (p == rd.end || !xyz_number(rd, p, bits)) return false;
    for (; p < rd.end; ++p)
        if (!xyz_sep(rd.at(p))) return false;
    return true;
}

// the three coordinate fields of the atom line at s -> x, y, z: the F8.3 fast path for each, then one general-path loop
// over those it rejected (not unrolled: one copy of the general grammar)
__device__ __forceinline__ bool pdb_coords(const unsigned char *__restrict__ b, long long s, unsigned &x, unsigned &y,
                                           unsigned &z) {
    unsigned miss = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        unsigned lo, hi, next;
        md_field(b + s + 30 + 8 * d, lo, hi, next);
        bool ok;
        const unsigned bits = md_parse(lo, hi, ok);
        (d == 0 ? x : d == 1 ? y : z) = bits;
        miss |= (unsigned)!ok << d;
    }
#pragma unroll 1
    for (; miss; miss &= miss - 1) {
        const int d = __ffs(miss) - 1;
        unsigned bits;
        if (!pdb_general(b, s + 30 + 8 * d, 8, bits)) return false;
        if (d == 0) x = bits;
        else if (d == 1) y = bits;
        else z = bits;
    }
    return true;
}

// coords[(a*3 + d)*frame_stride + k] = field d (columns 31-38, 39-46, 47-54) of atom record a of listed frame k, staged
// frame frame_of[k] (its atom records are starts[natoms u ...]).  An undecided line, or one shorter than 54 columns,
// appends (frame_base + k) * natoms + a to flags[1 ...] (flags[0] counts them; entries past flag_cap are dropped).
__global__ void __launch_bounds__(FT_WARPS * 32)
pdb_parse_kernel(const unsigned char *__restrict__ bytes, long long nbytes, const long long *__restrict__ starts,
                 const int *__restrict__ frame_of, int n_frames, int natoms, float *__restrict__ coords,
                 long long frame_stride, long long frame_base, unsigned long long *__restrict__ flags,
                 long long flag_cap) {
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
                const long long s = starts[(long long)natoms * frame_of[k] + a];
                const bool ok = s >= 0 && s + PDB_COLS <= nbytes && !pdb_short(bytes, s) && pdb_coords(bytes, s, x, y, z);
                if (!ok) {
                    const unsigned long long slot = atomicAdd(flags, 1ull);
                    if ((long long)slot < flag_cap) flags[1 + slot] = (unsigned long long)((frame_base + k) * natoms + a);
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

// cells[6 i + d] = field d of the CRYST1 line rows[i * PDB_CELL_ROW ...] (its first 54 bytes); bad[i] = 1 when a field
// is left to the host or the line ends before column 54
__global__ void __launch_bounds__(PDB_CELL_THREADS)
pdb_cell_kernel(const unsigned char *__restrict__ rows, int n_cells, float *__restrict__ cells,
                int *__restrict__ bad) {
    const int i = blockIdx.x * PDB_CELL_THREADS + threadIdx.x;
    if (i >= n_cells) return;
    const unsigned char *r = rows + (long long)i * PDB_CELL_ROW;
    bool ok = !pdb_short(r, 0);
#pragma unroll
    for (int d = 0; d < 6; ++d) {
        unsigned bits = 0u;
        ok = ok && pdb_general(r, d < 3 ? 6 + 9 * d : 33 + 7 * (d - 3), d < 3 ? 9 : 7, bits);
        reinterpret_cast<unsigned *>(cells)[6 * i + d] = bits;
    }
    bad[i] = !ok;
}

// "%8d" of v (0 <= v < 10^8) into d[0 .. 8)
__device__ __forceinline__ void pdb_int8(unsigned v, unsigned char *d) {
    int c = 7;
    do {
        d[c--] = (unsigned char)('0' + v % 10u);
        v /= 10u;
    } while (v && c >= 0);
    for (; c >= 0; --c) d[c] = ' ';
}

// Frame k of out is out[k*S ...], S = H + natoms*81 + 7: "MODEL %8d\n" of model0 + k, with a box the CRYST1 line of
// box[d*box_stride + k] and angles[d*box_stride + k] (H = 15 + 71, else H = 15), per atom its template line
// tmpl[a*81 ...] with the '%8.3f' fields of coords[(a*3 + d)*frame_stride + k] in columns 31-54, and "ENDMDL\n".  tmpl
// is readable up to natoms*81 rounded up to 4; tmpl and out are 4-byte aligned.
__global__ void __launch_bounds__(FT_WARPS * 32)
pdb_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, int natoms,
                  const unsigned char *__restrict__ tmpl, const float *__restrict__ box,
                  const float *__restrict__ angles, long long box_stride, long long model0, long long S,
                  unsigned char *__restrict__ out) {
    constexpr int ROW = (32 * PDB_LINE + 8 + 15) & ~15;
    __shared__ float tile[FT_W][FT_T + 1];  // [value][frame]
    __shared__ __align__(16) unsigned char img_all[FT_WARPS][ROW];
    __shared__ unsigned char head_all[FT_WARPS][PDB_MODEL + PDB_CRYST + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char *img = img_all[warp];
    const int a0 = blockIdx.x * 32, v0 = blockIdx.x * FT_W, na = min(32, natoms - a0);
    const int H = PDB_MODEL + (box ? PDB_CRYST : 0);
    const unsigned *tw = reinterpret_cast<const unsigned *>(tmpl + (long long)a0 * PDB_LINE);  // a0 * 81: 4-aligned
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
            if (blockIdx.x == 0) {  // the frame's MODEL and CRYST1 lines
                unsigned char *hd = head_all[warp];
                if (lane == 0) {
                    const char *m = "MODEL ";
                    for (int c = 0; c < 6; ++c) hd[c] = (unsigned char)m[c];
                    pdb_int8((unsigned)(model0 + k), hd + 6);
                    hd[14] = '\n';
                    if (box) {
                        unsigned char *cl = hd + PDB_MODEL;
                        const char *t = "CRYST1";
                        for (int c = 0; c < 6; ++c) cl[c] = (unsigned char)t[c];
                        for (int d = 0; d < 3; ++d) {
                            f_format<9, 3>(box[d * box_stride + k], cl + 6 + 9 * d);
                            f_format<7, 2>(angles[d * box_stride + k], cl + 33 + 7 * d);
                        }
                        const char *sg = " P 1           1\n";
                        for (int c = 0; c < 17; ++c) cl[54 + c] = (unsigned char)sg[c];
                    }
                }
                __syncwarp();
                for (int c = lane; c < H; c += 32) out[(long long)k * S + c] = hd[c];
                __syncwarp();
            }
            if (a0 + na == natoms && lane < PDB_ENDMDL)  // the last atom tile ends the frame
                out[(long long)k * S + S - PDB_ENDMDL + lane] = (unsigned char)"ENDMDL\n"[lane];
            const long long g0 = (long long)k * S + H + (long long)a0 * PDB_LINE;
            const int sh = (int)(g0 & 3), span = na * PDB_LINE;
            for (int m = lane; 4 * m < span; m += 32) {
                const unsigned w = __ldg(tw + m);
#pragma unroll
                for (int c = 0; c < 4; ++c) img[sh + 4 * m + c] = (unsigned char)(w >> (8 * c));
            }
            __syncwarp();
            if (lane < na) {
                unsigned char *d = img + sh + lane * PDB_LINE + 30;
#pragma unroll
                for (int x = 0; x < 3; ++x) {
                    unsigned lo, hi;
                    md_format(tile[3 * lane + x][fl], lo, hi);
                    md_put(d + 8 * x, lo, hi);
                }
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

// the three passes over bytes[0, n); the scan reads and advances state[0]
template <bool INDEX>
int pdb_lines(mkb_ctx *h, cudaStream_t st, const uint8_t *bytes, int64_t n, int64_t n_read, int first,
              int64_t file_base, int64_t *marks, int64_t mark_cap, int64_t *state, long long *starts,
              int64_t starts_cap) {
    const int64_t n_seg = std::max<int64_t>(1, cdiv(n, XL_SEG));
    if (n_seg > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    unsigned *counts;
    long long *base;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_COUNTS, (size_t)n_seg, &counts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_BASE, (size_t)n_seg, &base))) return rc;
    const uint4 *b = reinterpret_cast<const uint4 *>(bytes);
    pdb_count_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, n_read, first, counts);
    MKB_LAUNCHED(h);
    xyz_scan_kernel<<<1, XL_SCAN_THREADS, 0, st>>>(counts, (int)n_seg, base, reinterpret_cast<long long *>(state));
    MKB_LAUNCHED(h);
    pdb_emit_kernel<INDEX><<<(unsigned)n_seg, XL_THREADS, 0, st>>>(
        b, n, n_read, first, base, file_base, reinterpret_cast<long long *>(marks), mark_cap,
        reinterpret_cast<long long *>(state), starts, starts_cap);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_pdb_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                             int64_t file_base, int64_t *state, int64_t *marks, int64_t mark_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n < 0 || n_read < n || file_base < 0 || mark_cap < 0) return fail(h, MKB_ERR_BAD_ARG, "bad size");
    if (!bytes || !state || (mark_cap && !marks)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(marks)) & 7)
        return fail(h, MKB_ERR_BAD_ARG, "state and marks must be 8-byte aligned");
    if (n == 0) return MKB_OK;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    int rc = pdb_lines<true>(h, st, bytes, n, n_read, file_base == 0, file_base, marks, mark_cap, state, nullptr, 0);
    if (rc) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_pdb_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
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
    const int64_t n_atoms = n_staged * natoms;
    long long *starts, *state;
    int *d_map;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_STARTS, (size_t)n_atoms, &starts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_STATE, 1, &state))) return rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_map))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_map, frame_of, sizeof(int) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(state, 0, sizeof(long long), st));
    // a staged frame that holds fewer atom records leaves its starts at -1: the parse flags those lines
    MKB_CUDA(h, cudaMemsetAsync(starts, 0xff, sizeof(long long) * (size_t)n_atoms, st));
    if ((rc = pdb_lines<false>(h, st, bytes, nbytes, nbytes, 1, 0, nullptr, 0, reinterpret_cast<int64_t *>(state),
                               starts, n_atoms)))
        return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    pdb_parse_kernel<<<grid, FT_WARPS * 32, 0, st>>>(bytes, nbytes, starts, d_map, (int)n_frames, (int)natoms, coords,
                                                     frame_stride, frame_base,
                                                     reinterpret_cast<unsigned long long *>(flags), flag_cap);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_pdb_cell(mkb_handle_t h, void *stream, const uint8_t *rows, int64_t n_cells, float *cells,
                            int32_t *bad) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_cells < 0 || n_cells > INT32_MAX - PDB_CELL_THREADS) return fail(h, MKB_ERR_BAD_ARG, "bad n_cells");
    if (n_cells == 0) return MKB_OK;
    if (!rows || !cells || !bad) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(rows) & 15) || ((reinterpret_cast<uintptr_t>(cells) | reinterpret_cast<uintptr_t>(bad)) & 3))
        return fail(h, MKB_ERR_BAD_ARG, "rows must be 16-byte, cells and bad 4-byte aligned");
    pdb_cell_kernel<<<(unsigned)cdiv(n_cells, PDB_CELL_THREADS), PDB_CELL_THREADS, 0, st>>>(rows, (int)n_cells, cells,
                                                                                           bad);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

extern "C" int mkb_pdb_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride,
                              int64_t n_frames, int64_t natoms, const uint8_t *tmpl, const float *box,
                              const float *angles, int64_t box_stride, int64_t model0, uint8_t *out,
                              int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / PDB_LINE) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 81");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (model0 < 0 || model0 + n_frames > 100000000ll) return fail(h, MKB_ERR_BAD_ARG, "model serials must be below 10^8");
    if (!coords || !tmpl || !out || (box && !angles)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(tmpl) | reinterpret_cast<uintptr_t>(out) |
         reinterpret_cast<uintptr_t>(box) | reinterpret_cast<uintptr_t>(angles)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords, tmpl, box, angles and out must be 4-byte aligned");
    if (frame_stride < n_frames || (box && box_stride < n_frames))
        return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const int64_t S = PDB_MODEL + (box ? PDB_CRYST : 0) + natoms * PDB_LINE + PDB_ENDMDL;
    if (n_frames * S > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * S));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    pdb_encode_kernel<<<grid, FT_WARPS * 32, 0, st>>>(coords, frame_stride, (int)n_frames, (int)natoms, tmpl, box,
                                                      angles, box_stride, model0 + 1, S, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
