// cif.cu -- K30: multi-model PDBx/mmCIF trajectories indexed, parsed and formatted on the device.
//
// Replaces the host path of an mmCIF reader that tokenizes every row of the _atom_site loop and calls float() on its
// Cartn_x, Cartn_y and Cartn_z tokens.  The loop is free-format: a row is a run of whitespace-separated tokens (a token
// may be a '...' or "..." string), the column order is the loop header's, and a frame is a run of rows with the same
// pdbx_PDB_model_num.  So the device work is a tokenizer, not column slices.
//
//   lines    a line start is byte 0 of the span (when the caller says it starts a line) or the byte after a '\n'; its
//            first non-blank byte classifies it (cif_line): a row, a skipped line (blank, or '#': a CIF comment) or the
//            line that ends the loop (a tag '_...', loop_, stop_, global_, data_..., save_...).
//   index    over the loop body in chunks (mkb_cif_index), in three launches per chunk: cif_count_kernel<true> counts the
//            rows that start in each 32 KB segment, tokenizes the segment's last row for its model number and
//            atomicMins the offset of every terminator line; cif_scan_kernel turns the counts into each segment's first
//            row rank and the model number of the row before it, both carried across chunks in device state; and
//            cif_index_emit_kernel ranks the segment's rows before the terminator into shared memory, then lets every
//            thread tokenize one row at a time (token count and model number) and, where a row's model number differs
//            from the row before it, append a mark (file offset, rank, model).  The first bad row and the first lone CR
//            are atomicMins; the terminator's rank is stored.  Only O(F) marks come back: the host derives the frames.
//   tokens   cif_fast walks a row in aligned 16-byte words with SWAR masks (blanks, newline, token starts); a row it
//            cannot decide that way (a quoted token with a blank inside, ';', control bytes) goes through cif_tokens,
//            the byte-at-a-time statement of the rule.
//   decode   over staged whole frames (mkb_cif_decode), each holding exactly natoms rows: the same count and scan, and
//            cif_emit_kernel stores the start of every row by its rank, so comment and blank lines cost nothing.
//            cif_parse_kernel maps K23's tile (32 frames x 32 atoms per CTA of 256 threads), one thread per row: it
//            tokenizes the row up to the furthest Cartn column and parses the three tokens with K26's grammar.  A row
//            the device does not decide is appended to a list for the host.
//   encode   the inverse (mkb_cif_encode): a CTA loads 32 frames x 32 atoms along frames, each warp copies its 32
//            atoms' fixed-width template rows into a shared-memory image, writes id, the three '%10.3f' fields and
//            pdbx_PDB_model_num, and stores the image with aligned 32-bit words.
//
// Arithmetic: a coordinate token goes through K26's general grammar (xyz_number.cuh) with the token's end as the line
// end, so every decided token is bit for bit np.float32(float(token)); '%10.3f' is f83.cuh's f_format.
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

constexpr long long CIF_NONE = (long long)(-0x7fffffffffffffffll - 1);  // "no row" in the model carry
constexpr int CIF_SEG_ROWS = 5472;  // rows of a 32 KB segment the index keeps: a row of 3 tokens takes 6 bytes or more
constexpr int CIF_MAX_ROW = 768;  // the widest written row, '\n' included (the encode image holds 32 of them per warp)
constexpr int CIF_MODEL_DIGITS = 18;
constexpr int CIF_SCAN_THREADS = 512;

enum : int { LINE_SKIP = 0, LINE_ROW = 1, LINE_TERM = 2 };
// index state (int64): running row count, first lone CR, marks, first bad row, first terminator, model carry,
// terminator rank
enum : int { ST_ROWS = 0, ST_CR = 1, ST_MARKS = 2, ST_BAD = 3, ST_TERM = 4, ST_PREV = 5, ST_TERM_RANK = 6 };

// bytes at and past n read as '\n'
struct CifBuf {
    const unsigned char *b;
    long long n;
    __device__ __forceinline__ unsigned at(long long p) const { return p < n ? __ldg(b + p) : '\n'; }
};

// the blanks of a line: what bytes.split() splits on, '\n' (the line end) aside
__device__ __forceinline__ bool cif_blank(unsigned c) { return c == ' ' || c == '\t' || c == '\v' || c == '\f' || c == '\r'; }
__device__ __forceinline__ unsigned cif_lower(unsigned c) { return c - 'A' < 26u ? c | 0x20u : c; }

__host__ __device__ constexpr unsigned long long cif_word(const char *s, int n) {
    unsigned long long w = 0;
    for (int i = n - 1; i >= 0; --i) w = (w << 8) | (unsigned char)s[i];
    return w;
}

// the kind of the line starting at p
__device__ __forceinline__ int cif_line(const CifBuf &rd, long long p) {
    unsigned c = rd.at(p);
    while (cif_blank(c)) c = rd.at(++p);
    if (c == '\n' || c == '#') return LINE_SKIP;
    if (c == '_') return LINE_TERM;
    unsigned long long w = 0;  // the first 8 bytes of the token, letters in lower case
    int n = 0;
    for (; n < 8 && !cif_blank(c) && c != '\n'; c = rd.at(++p), ++n) w |= (unsigned long long)cif_lower(c) << (8 * n);
    if (n == 8 && !cif_blank(c) && c != '\n') n = 9;  // longer than 8
    constexpr unsigned long long LOOP = cif_word("loop_", 5), STOP = cif_word("stop_", 5),
                                 GLOBAL = cif_word("global_", 7), DATA = cif_word("data_", 5), SAVE = cif_word("save_", 5);
    if ((n == 5 && (w == LOOP || w == STOP)) || (n == 7 && w == GLOBAL)) return LINE_TERM;
    if (n >= 5 && ((w & 0xffffffffffull) == DATA || (w & 0xffffffffffull) == SAVE)) return LINE_TERM;
    return LINE_ROW;
}

// The tokens of the row starting at p: on(i, s, e, quoted) for token i = bytes [s, e) (a quoted token without its
// quotes), until on returns false or token `stop` has been seen.  Returns the token count (up to stop + 1), -1 when a
// quoted token is not closed before the line's end or the row starts with ';', -2 when on returned false, and with
// ASCII_ONLY -2 for a byte >= 0x80.
template <bool ASCII_ONLY, class F>
__device__ __forceinline__ int cif_tokens(const CifBuf &rd, long long p, int stop, F &&on) {
    unsigned c = rd.at(p);
    for (int i = 0;; ++i) {
        while (cif_blank(c)) c = rd.at(++p);
        if (c == '\n' || i > stop) return i;
        long long s = p, e;
        const bool quoted = c == '\'' || c == '"';
        if (quoted) {  // closes at the first matching quote followed by a blank or the line's end
            const unsigned q = c;
            for (e = ++s;; ++e) {
                const unsigned d = rd.at(e);
                if (d == '\n') return -1;
                if (ASCII_ONLY && d >= 0x80u) return -2;
                if (d == q) {
                    const unsigned x = rd.at(e + 1);
                    if (cif_blank(x) || x == '\n') break;
                }
            }
            p = e + 1;
            c = rd.at(p);
        } else {
            if (c == ';' && i == 0) return -1;  // a text field: rows must be one line each
            for (; !cif_blank(c) && c != '\n'; c = rd.at(++p))
                if (ASCII_ONLY && c >= 0x80u) return -2;
            e = p;
        }
        if (!on(i, s, e, quoted)) return -2;
    }
}

// bit j of the result: bit 7 of byte j of the 16 bytes (z holds bit 7 per byte of each word)
__device__ __forceinline__ unsigned cif_bits(const unsigned z[4]) {
    unsigned m = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        m |= (((z[i] >> 7) & 1u) | ((z[i] >> 14) & 2u) | ((z[i] >> 21) & 4u) | ((z[i] >> 28) & 8u)) << (4 * i);
    return m;
}

// The row at p in 16-byte words (the fast path of cif_tokens): count = its tokens (counting stops past token stop) and
// s[d] = the first byte of token want[d] (want[d] < 0: none).  false: a byte the fast path leaves to cif_tokens --
// ';', a control byte other than \t, \r and \n, a quoted token with a blank inside, and with ASCII_ONLY a byte >=
// 0x80.  b is readable up to n
// rounded up to 16; bytes at and past n read as '\n'.
template <bool ASCII_ONLY>
__device__ __forceinline__ bool cif_fast(const unsigned char *__restrict__ b, long long n, long long p, int stop,
                                         const int want[3], int &count, long long s[3]) {
    unsigned carry = 0;  // the byte before the word is a token byte
    int cnt = 0;
    for (long long w = p & ~15ll;; w += 16) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(b + w));
        const unsigned x[4] = {v.x, v.y, v.z, v.w};
        unsigned lo[4], hi[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            lo[i] = ~(((x[i] & 0x7f7f7f7fu) + 0x60606060u) | x[i]) & 0x80808080u;  // bytes below 0x20
            hi[i] = x[i] & 0x80808080u;
        }
        const unsigned valid = xl_valid(w, n), live = w < p ? valid & (0xffffu << (int)(p - w)) : valid;
        const unsigned nl = (xl_mask(v, '\n') & live) | (0xffffu & ~valid);
        const unsigned blank = xl_mask(v, ' ') | xl_mask(v, '\t') | xl_mask(v, '\r');
        const unsigned row = live & (nl ? (nl & (0u - nl)) - 1u : 0xffffu);  // this word's bytes of the row
        const unsigned odd = (cif_bits(lo) & ~blank) | xl_mask(v, ';') | (ASCII_ONLY ? cif_bits(hi) : 0u);
        if (odd & row) return false;
        const unsigned tok = ~blank & row, st = tok & ~((tok << 1) | carry);
        // a token that opens a quote: the same token boundaries when it is 2 bytes or more and ends in that quote
        for (unsigned q = st & (xl_mask(v, '\'') | xl_mask(v, '"')); q; q &= q - 1) {
            const long long a = w + __ffs(q) - 1;
            const unsigned c = __ldg(b + a);
            long long e = a + 1;
            unsigned d = e < n ? __ldg(b + e) : '\n';
            for (; !cif_blank(d) && d != '\n'; d = e < n ? __ldg(b + e) : '\n') ++e;
            if (e - a < 2 || __ldg(b + e - 1) != c) return false;
        }
        const int k = __popc(st);
#pragma unroll
        for (int d = 0; d < 3; ++d)
            if (want[d] >= cnt && want[d] < cnt + k) s[d] = w + (int)__fns(st, 0, want[d] - cnt + 1);
        cnt += k;
        if (nl || cnt > stop) {
            count = cnt;
            return true;
        }
        carry = (tok >> 15) & 1u;
    }
}

// [+-]?digits (at most 18) -> v
__device__ __forceinline__ bool cif_int(const CifBuf &rd, long long s, long long e, long long &v) {
    unsigned c = rd.at(s);
    const bool neg = c == '-';
    if (c == '+' || c == '-') ++s;
    if (s == e || e - s > CIF_MODEL_DIGITS) return false;
    long long x = 0;
    for (; s < e; ++s) {
        c = rd.at(s);
        if (!xyz_digit(c)) return false;
        x = 10 * x + (c - '0');
    }
    v = neg ? -x : x;
    return true;
}

// the row at p: true when it holds n_tags tokens and (model_col >= 0) an integer model token -> model (0 without one)
__device__ __forceinline__ bool cif_row(const CifBuf &rd, long long p, int n_tags, int model_col, long long &model) {
    model = 0;
    const int want[3] = {model_col, -1, -1};
    long long s[3] = {-1, -1, -1};
    int n;
    if (cif_fast<false>(rd.b, rd.n, p, n_tags, want, n, s)) {
        if (n != n_tags) return false;
        if (model_col < 0) return true;
        long long e = s[0];
        while (!cif_blank(rd.at(e)) && rd.at(e) != '\n') ++e;
        return cif_int(rd, s[0], e, model);
    }
    bool ok = true;
    n = cif_tokens<false>(rd, p, n_tags, [&](int i, long long a, long long e, bool quoted) {
        if (i == model_col) ok = !quoted && cif_int(rd, a, e, model);
        return ok;
    });
    return ok && n == n_tags;
}

struct CifMax {
    __device__ __forceinline__ long long operator()(long long a, long long b) const { return a > b ? a : b; }
};

// Rows numbered from state[ST_ROWS]'s value before the scan.  counts[s] = the rows starting in segment s of bytes[0, n)
// (a line start after a '\n' in the segment; byte 0 too when `first`).  INDEX: last_model[s] = the model number of the
// segment's last row (CIF_NONE without one or for a bad row), and every terminator line atomicMins file_base + its
// byte into state[ST_TERM].
template <bool INDEX>
__global__ void __launch_bounds__(XL_THREADS)
cif_count_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, int first, long long file_base,
                 int n_tags, int model_col, unsigned *__restrict__ counts, long long *__restrict__ last_model,
                 long long *__restrict__ state) {
    using Reduce = cub::BlockReduce<unsigned, XL_THREADS>;
    using ReduceL = cub::BlockReduce<long long, XL_THREADS>;
    __shared__ union {
        typename Reduce::TempStorage r;
        typename ReduceL::TempStorage l;
    } tmp;
    const CifBuf rd{reinterpret_cast<const unsigned char *>(bytes), n_read};
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    unsigned c = 0;
    long long last = -1;
    auto line = [&](long long p) {
        const int k = cif_line(rd, p);
        if (k == LINE_ROW) {
            ++c;
            last = p;
        } else if (INDEX && k == LINE_TERM) {
            atomicMin(reinterpret_cast<unsigned long long *>(state + ST_TERM), (unsigned long long)(file_base + p));
        }
    };
    if (first && blockIdx.x == 0 && threadIdx.x == 0) line(0);
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        if (p0 >= n) break;
        for (unsigned nl = xl_mask(__ldg(bytes + wi), '\n') & xl_valid(p0, n); nl; nl &= nl - 1) line(p0 + __ffs(nl));
    }
    const unsigned total = Reduce(tmp.r).Sum(c);
    if (!INDEX) {
        if (threadIdx.x == 0) counts[blockIdx.x] = total;
        return;
    }
    __syncthreads();
    const long long at = ReduceL(tmp.l).Reduce(last, CifMax());
    if (threadIdx.x == 0) {
        counts[blockIdx.x] = total;
        long long m = CIF_NONE;
        if (at >= 0 && !cif_row(rd, at, n_tags, model_col, m)) m = CIF_NONE;
        last_model[blockIdx.x] = m;
    }
}

struct CifLast {  // the scan operator of the model carry: the last value that is not CIF_NONE
    __device__ __forceinline__ long long operator()(long long a, long long b) const { return b != CIF_NONE ? b : a; }
};

// base[s] = state[ST_ROWS] + the counts of segments before s; state[ST_ROWS] += all of them.  With last_model:
// prev[s] = the model number of the last row before segment s (state[ST_PREV] for the chunk's first rows), and
// state[ST_PREV] advances to the chunk's last row.
__global__ void __launch_bounds__(CIF_SCAN_THREADS)
cif_scan_kernel(const unsigned *__restrict__ counts, const long long *__restrict__ last_model, int n_seg,
                long long *__restrict__ base, long long *__restrict__ prev, long long *__restrict__ state) {
    using Scan = cub::BlockScan<unsigned, CIF_SCAN_THREADS>;
    using ScanL = cub::BlockScan<long long, CIF_SCAN_THREADS>;
    __shared__ union {
        typename Scan::TempStorage u;
        typename ScanL::TempStorage l;
    } tmp;
    long long carry = state[ST_ROWS], mcarry = last_model ? state[ST_PREV] : CIF_NONE;
    for (int s0 = 0; s0 < n_seg; s0 += CIF_SCAN_THREADS) {
        const int s = s0 + threadIdx.x;
        const unsigned cnt = s < n_seg ? counts[s] : 0u;
        unsigned ex, total;
        Scan(tmp.u).ExclusiveSum(cnt, ex, total);
        if (s < n_seg) base[s] = carry + ex;
        carry += total;
        if (last_model) {
            __syncthreads();
            long long before, agg;
            ScanL(tmp.l).ExclusiveScan(cnt ? last_model[s] : CIF_NONE, before, mcarry, CifLast(), agg);
            if (s < n_seg) prev[s] = before;
            mcarry = CifLast()(mcarry, agg);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        state[ST_ROWS] = carry;
        if (last_model) state[ST_PREV] = mcarry;
    }
}

// the row starts among the line starts of the 16-byte word at p0 (bit j: the line after byte p0 + j) and, for the first
// word of the span, byte 0 (zrow); line starts at and past `stop` are left out and has_stop tells whether one sits there
__device__ __forceinline__ unsigned cif_rows(const CifBuf &rd, const uint4 *__restrict__ bytes, long long wi, long long n,
                                             bool zero, long long stop, unsigned &zrow, bool &has_stop, unsigned &nl) {
    const long long p0 = 16 * wi;
    unsigned rows = 0;
    zrow = 0;
    has_stop = false;
    nl = 0;
    if (zero) {
        has_stop = stop == 0;
        zrow = !has_stop && cif_line(rd, 0) == LINE_ROW;
    }
    if (p0 < n) {
        nl = xl_mask(__ldg(bytes + wi), '\n') & xl_valid(p0, n);
        for (unsigned m = nl; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const long long p = p0 + j + 1;
            if (p >= stop) {
                has_stop |= p == stop;
                continue;
            }
            if (cif_line(rd, p) == LINE_ROW) rows |= 1u << j;
        }
    }
    return rows;
}

// starts[base[s] + r] = the byte of row r of segment s, for ranks below starts_cap
__global__ void __launch_bounds__(XL_THREADS)
cif_emit_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, int first,
                const long long *__restrict__ base, long long *__restrict__ starts, long long starts_cap) {
    using Scan = cub::BlockScan<unsigned, XL_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const CifBuf rd{reinterpret_cast<const unsigned char *>(bytes), n_read};
    const long long w0 = (long long)blockIdx.x * (XL_SEG / 16);
    long long g0 = base[blockIdx.x];  // rows before the segment
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        unsigned zrow, nl;
        bool has_stop;
        unsigned rows = cif_rows(rd, bytes, wi, n, first && i == 0 && blockIdx.x == 0 && threadIdx.x == 0,
                                 n_read + 1, zrow, has_stop, nl);
        unsigned ex, total;
        Scan(tmp).ExclusiveSum(__popc(rows) + zrow, ex, total);
        long long r = g0 + ex;
        if (zrow && r < starts_cap) starts[r] = 0;
        r += zrow;
        for (; rows; rows &= rows - 1, ++r)
            if (r < starts_cap) starts[r] = p0 + __ffs(rows);
        g0 += total;
        __syncthreads();  // tmp is reused by the next item's scan
    }
}

// The index's emit pass over one segment, in two phases.  Rows: every line start before the terminator (file offset
// below state[ST_TERM]) is classified and the segment's rows are ranked with a block scan, their starts kept in shared
// memory; the terminator stores its rank in state[ST_TERM_RANK] and a CR not followed by LF atomicMins its offset
// into state[ST_CR].  Tokens: the threads take the rows in turn, one row each, so a warp tokenizes 32 rows at once; a
// row whose model number differs from the row before it appends (file offset, rank, model) to marks[3 j ...] for j =
// state[ST_MARKS]++ < mark_cap, and a bad row (token count, model token, text field) atomicMins its offset into
// state[ST_BAD].  A segment holds at most CIF_SEG_ROWS rows of 6 bytes or more; a row past them is reported as bad.
__global__ void __launch_bounds__(XL_THREADS)
cif_index_emit_kernel(const uint4 *__restrict__ bytes, long long n, long long n_read, int first, long long file_base,
                      int n_tags, int model_col, const long long *__restrict__ base, const long long *__restrict__ prev,
                      long long *__restrict__ marks, long long mark_cap, long long *__restrict__ state) {
    using Scan = cub::BlockScan<unsigned, XL_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ int pos[CIF_SEG_ROWS];     // row starts, relative to the segment
    __shared__ long long mdl[XL_THREADS];  // the model numbers of one turn of rows
    const CifBuf rd{reinterpret_cast<const unsigned char *>(bytes), n_read};
    const long long s0 = (long long)blockIdx.x * XL_SEG, w0 = s0 / 16;
    const long long term = state[ST_TERM] - file_base;  // the terminator's byte in this span
    if (term <= s0) return;                              // the segment lies past the loop
    auto bad = [&](long long p) {
        atomicMin(reinterpret_cast<unsigned long long *>(state + ST_BAD), (unsigned long long)(file_base + p));
    };
    unsigned g0 = 0;  // rows of the segment before the item
    for (int i = 0; i < XL_ITEMS; ++i) {
        const long long wi = w0 + i * XL_THREADS + threadIdx.x, p0 = 16 * wi;
        unsigned zrow, nl;
        bool has_term;
        unsigned rows = cif_rows(rd, bytes, wi, n, first && i == 0 && blockIdx.x == 0 && threadIdx.x == 0, term,
                                 zrow, has_term, nl);
        unsigned ex, total;
        const unsigned nr = __popc(rows) + zrow;
        Scan(tmp).ExclusiveSum(nr, ex, total);
        unsigned r = g0 + ex;
        if (zrow) {
            if (r < CIF_SEG_ROWS) pos[r] = 0;
            else bad(0);
            ++r;
        }
        for (; rows; rows &= rows - 1, ++r) {
            const int off = (int)(p0 + __ffs(rows) - s0);
            if (r < CIF_SEG_ROWS) pos[r] = off;
            else bad(s0 + off);
        }
        if (has_term) state[ST_TERM_RANK] = base[blockIdx.x] + g0 + ex + nr;  // its thread's rows lie before it
        if (p0 < n) {
            for (unsigned cr = xl_mask(__ldg(bytes + wi), '\r') & xl_valid(p0, n); cr; cr &= cr - 1) {
                const long long at = p0 + __ffs(cr) - 1;
                if (at < term && at + 1 < n_read && rd.at(at + 1) != '\n')
                    atomicMin(reinterpret_cast<unsigned long long *>(state + ST_CR), (unsigned long long)(file_base + at));
            }
        }
        g0 += total;
        __syncthreads();  // tmp is reused by the next item's scan
    }
    const int R = (int)min(g0, (unsigned)CIF_SEG_ROWS);
    const long long rank0 = base[blockIdx.x];
    long long carry = prev[blockIdx.x];
    for (int t0 = 0; t0 < R; t0 += XL_THREADS) {
        const int r = t0 + threadIdx.x;
        long long m = CIF_NONE;
        if (r < R && !cif_row(rd, s0 + pos[r], n_tags, model_col, m)) {
            bad(s0 + pos[r]);
            m = CIF_NONE;
        }
        mdl[threadIdx.x] = m;
        __syncthreads();
        const long long before = threadIdx.x ? mdl[threadIdx.x - 1] : carry;
        if (r < R && m != CIF_NONE && m != before) {
            const unsigned long long j = atomicAdd(reinterpret_cast<unsigned long long *>(state + ST_MARKS), 1ull);
            if ((long long)j < mark_cap) {
                marks[3 * j] = file_base + s0 + pos[r];
                marks[3 * j + 1] = rank0 + r;
                marks[3 * j + 2] = m;
            }
        }
        carry = mdl[min(XL_THREADS, R - t0) - 1];
        __syncthreads();  // mdl is reused by the next turn
    }
}

// the three Cartn tokens (token columns cx, cy, cz) of the row at p -> x, y, z; false: the host decides (a quoted
// token, a token outside K26's grammar, a byte >= 0x80 before the last of them, an undecided rounding)
__device__ __forceinline__ bool cif_coords(const CifBuf &rd, long long p, int cx, int cy, int cz, unsigned &x,
                                           unsigned &y, unsigned &z) {
    const int stop = max(cx, max(cy, cz)), want[3] = {cx, cy, cz};
    long long s[3];
    int n;
    if (cif_fast<true>(rd.b, rd.n, p, stop, want, n, s)) {  // each token ends at a blank or '\n': xyz_number's end
        long long q0 = s[0], q1 = s[1], q2 = s[2];
        return n > stop && xyz_number(rd, q0, x) && xyz_number(rd, q1, y) && xyz_number(rd, q2, z);
    }
    int got = 0;
    n = cif_tokens<true>(rd, p, stop, [&](int i, long long a, long long e, bool quoted) {
        if (i != cx && i != cy && i != cz) return true;
        if (quoted) return false;
        CifBuf tok{rd.b, e};  // the token's end reads as the line's end
        unsigned bits;
        long long q = a;
        if (!xyz_number(tok, q, bits) || q != e) return false;
        if (i == cx) x = bits;
        if (i == cy) y = bits;
        if (i == cz) z = bits;
        ++got;
        return true;
    });
    return n > stop && got == 3;
}

// coords[(a*3 + d)*frame_stride + k] = Cartn token d of row a of listed frame k, staged frame frame_of[k] (its rows
// are starts[natoms u ...]).  A row the device does not decide appends (frame_base + k) * natoms + a to flags[1 ...]
// (flags[0] counts them; entries past flag_cap are dropped).
__global__ void __launch_bounds__(FT_WARPS * 32)
cif_parse_kernel(const unsigned char *__restrict__ bytes, long long nbytes, const long long *__restrict__ starts,
                 const int *__restrict__ frame_of, int n_frames, int natoms, int cx, int cy, int cz,
                 float *__restrict__ coords, long long frame_stride, long long frame_base,
                 unsigned long long *__restrict__ flags, long long flag_cap) {
    __shared__ unsigned tile[FT_W][FT_T + 1];  // [value][frame]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int a = blockIdx.x * 32 + lane, v0 = blockIdx.x * FT_W;
    const int n_ft = (n_frames + FT_T - 1) / FT_T;
    const CifBuf rd{bytes, nbytes};
    for (int ft = blockIdx.y; ft < n_ft; ft += gridDim.y) {
        const int k0 = ft * FT_T;
        __syncthreads();  // the previous tile is stored
#pragma unroll 1
        for (int j = 0; j < FT_T / FT_WARPS; ++j) {
            const int fl = warp + FT_WARPS * j, k = k0 + fl;
            unsigned x = 0u, y = 0u, z = 0u;
            if (k < n_frames && a < natoms) {
                const long long s = starts[(long long)natoms * frame_of[k] + a];
                if (!(s >= 0 && cif_coords(rd, s, cx, cy, cz, x, y, z))) {
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

// v right-justified in d[0 .. w) (v < 10^w)
__device__ __forceinline__ void cif_put_int(unsigned long long v, unsigned char *d, int w) {
    int c = w - 1;
    do {
        d[c--] = (unsigned char)('0' + v % 10u);
        v /= 10u;
    } while (v && c >= 0);
    for (; c >= 0; --c) d[c] = ' ';
}

// Frame k of out is out[k*S ...], S = natoms*R: per atom its template row tmpl[a*R ...] with id = (frame0 + k)*natoms
// + a + 1 right-justified in id_w bytes at col_id, the '%10.3f' fields of coords[(a*3 + d)*frame_stride + k] at col_x
// + 11 d, and pdbx_PDB_model_num = frame0 + k + 1 right-justified in model_w bytes at col_model.  tmpl is readable up to
// natoms*R rounded up to 4; tmpl and out are 4-byte aligned.  Dynamic shared memory: FT_WARPS images of 32 rows.
__global__ void __launch_bounds__(FT_WARPS * 32)
cif_encode_kernel(const float *__restrict__ coords, long long frame_stride, int n_frames, int natoms,
                  const unsigned char *__restrict__ tmpl, int R, int col_id, int id_w, int col_x, int col_model,
                  int model_w, long long frame0, unsigned char *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char img_all[];
    __shared__ float tile[FT_W][FT_T + 1];  // [value][frame]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int img_bytes = (32 * R + 4 + 15) & ~15;
    unsigned char *img = img_all + warp * img_bytes;
    const int a0 = blockIdx.x * 32, v0 = blockIdx.x * FT_W, na = min(32, natoms - a0);
    const long long S = (long long)natoms * R;
    const unsigned *tw = reinterpret_cast<const unsigned *>(tmpl + (long long)a0 * R);  // a0 * R: 4-aligned
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
            const long long g0 = (long long)k * S + (long long)a0 * R;
            const int sh = (int)(g0 & 3), span = na * R;
            for (int m = lane; 4 * m < span; m += 32) {
                const unsigned w = __ldg(tw + m);
#pragma unroll
                for (int c = 0; c < 4; ++c) img[sh + 4 * m + c] = (unsigned char)(w >> (8 * c));
            }
            __syncwarp();
            if (lane < na) {
                unsigned char *d = img + sh + lane * R;
                cif_put_int((unsigned long long)((frame0 + k) * natoms + a0 + lane + 1), d + col_id, id_w);
#pragma unroll
                for (int x = 0; x < 3; ++x) f_format<10, 3>(tile[3 * lane + x][fl], d + col_x + 11 * x);
                cif_put_int((unsigned long long)(frame0 + k + 1), d + col_model, model_w);
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

// the three passes over bytes[0, n); the scan reads and advances state
template <bool INDEX>
int cif_lines(mkb_ctx *h, cudaStream_t st, const uint8_t *bytes, int64_t n, int64_t n_read, int first,
              int64_t file_base, int n_tags, int model_col, int64_t *marks, int64_t mark_cap, int64_t *state,
              long long *starts, int64_t starts_cap) {
    const int64_t n_seg = std::max<int64_t>(1, cdiv(n, XL_SEG));
    if (n_seg > INT32_MAX) return fail(h, MKB_ERR_BAD_ARG, "span too long");
    unsigned *counts;
    long long *base, *seg = nullptr;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_COUNTS, (size_t)n_seg, &counts))) return rc;
    // INDEX: base, then each segment's last model, then the model before it
    if ((rc = scratch_get(h, S_XYZ_BASE, (size_t)n_seg * (INDEX ? 3 : 1), &base))) return rc;
    if (INDEX) seg = base + n_seg;
    const uint4 *b = reinterpret_cast<const uint4 *>(bytes);
    long long *s = reinterpret_cast<long long *>(state);
    cif_count_kernel<INDEX><<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, n_read, first, file_base, n_tags, model_col,
                                                                     counts, seg, s);
    MKB_LAUNCHED(h);
    cif_scan_kernel<<<1, CIF_SCAN_THREADS, 0, st>>>(counts, seg, (int)n_seg, base, INDEX ? seg + n_seg : nullptr, s);
    MKB_LAUNCHED(h);
    if (INDEX)
        cif_index_emit_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, n_read, first, file_base, n_tags, model_col,
                                                                      base, seg + n_seg,
                                                                      reinterpret_cast<long long *>(marks), mark_cap, s);
    else
        cif_emit_kernel<<<(unsigned)n_seg, XL_THREADS, 0, st>>>(b, n, n_read, first, base, starts, starts_cap);
    MKB_LAUNCHED(h);
    return MKB_OK;
}

}  // namespace
}  // namespace mkb

using namespace mkb;

extern "C" int mkb_cif_index(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t n, int64_t n_read,
                             int64_t file_base, int64_t first, int64_t n_tags, int64_t model_col, int64_t *state,
                             int64_t *marks, int64_t mark_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n < 0 || n_read < n || file_base < 0 || mark_cap < 0) return fail(h, MKB_ERR_BAD_ARG, "bad size");
    if (n_tags < 3 || n_tags > 1 << 20 || model_col < -1 || model_col >= n_tags)
        return fail(h, MKB_ERR_BAD_ARG, "n_tags must be 3 to 2^20 and model_col -1 or a column");
    if (!bytes || !state || (mark_cap && !marks)) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(state) | reinterpret_cast<uintptr_t>(marks)) & 7)
        return fail(h, MKB_ERR_BAD_ARG, "state and marks must be 8-byte aligned");
    if (n == 0) return MKB_OK;
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    int rc = cif_lines<true>(h, st, bytes, n, n_read, first != 0, file_base, (int)n_tags, (int)model_col, marks,
                             mark_cap, state, nullptr, 0);
    if (rc) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_cif_decode(mkb_handle_t h, void *stream, const uint8_t *bytes, int64_t nbytes, int64_t n_staged,
                              const int32_t *frame_of, int64_t n_frames, int64_t natoms, int64_t col_x, int64_t col_y,
                              int64_t col_z, float *coords, int64_t frame_stride, int64_t frame_base, int64_t *flags,
                              int64_t flag_cap) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || n_staged < 0 || nbytes < 0 || frame_base < 0 || flag_cap < 0)
        return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (col_x < 0 || col_y < 0 || col_z < 0 || col_x >= 1 << 20 || col_y >= 1 << 20 || col_z >= 1 << 20)
        return fail(h, MKB_ERR_BAD_ARG, "Cartn columns must be 0 to 2^20 - 1");
    if (!bytes || !frame_of || !coords || !flags) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (reinterpret_cast<uintptr_t>(bytes) & 15) return fail(h, MKB_ERR_BAD_ARG, "bytes must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(coords) & 3) || (reinterpret_cast<uintptr_t>(flags) & 7))
        return fail(h, MKB_ERR_BAD_ARG, "coords must be 4-byte and flags 8-byte aligned");
    for (int64_t k = 0; k < n_frames; ++k)
        if (frame_of[k] < 0 || frame_of[k] >= n_staged)
            return fail(h, MKB_ERR_BAD_ARG, "frame_of[%lld] = %d is not a staged frame (%lld staged)", (long long)k,
                        (int)frame_of[k], (long long)n_staged);
    const int64_t n_rows = n_staged * natoms;
    long long *starts, *state;
    int *d_map;
    int rc;
    if ((rc = scratch_get(h, S_XYZ_STARTS, (size_t)n_rows, &starts))) return rc;
    if ((rc = scratch_get(h, S_XYZ_STATE, 1, &state))) return rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &d_map))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_map, frame_of, sizeof(int) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(state, 0, sizeof(long long), st));
    // a staged frame that holds fewer rows leaves its starts at -1: the parse flags those rows
    MKB_CUDA(h, cudaMemsetAsync(starts, 0xff, sizeof(long long) * (size_t)n_rows, st));
    if ((rc = cif_lines<false>(h, st, bytes, nbytes, nbytes, 1, 0, 3, -1, nullptr, 0,
                               reinterpret_cast<int64_t *>(state), starts, n_rows)))
        return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    cif_parse_kernel<<<grid, FT_WARPS * 32, 0, st>>>(bytes, nbytes, starts, d_map, (int)n_frames, (int)natoms,
                                                     (int)col_x, (int)col_y, (int)col_z, coords, frame_stride,
                                                     frame_base, reinterpret_cast<unsigned long long *>(flags), flag_cap);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

extern "C" int mkb_cif_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride,
                              int64_t n_frames, int64_t natoms, const uint8_t *tmpl, int64_t row_bytes, int64_t col_id,
                              int64_t id_width, int64_t col_x, int64_t col_model, int64_t model_width, int64_t frame0,
                              uint8_t *out, int64_t out_capacity) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0 || frame0 < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0) return MKB_OK;
    if (natoms < 1 || natoms > INT32_MAX / 3) return fail(h, MKB_ERR_BAD_ARG, "natoms must be 1 to (2^31 - 1) / 3");
    if (n_frames >= (1ll << 31) - FT_T) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (row_bytes < 2 || row_bytes > CIF_MAX_ROW) return fail(h, MKB_ERR_BAD_ARG, "row_bytes must be 2 to %d", CIF_MAX_ROW);
    if (id_width < 1 || id_width > 19 || model_width < 1 || model_width > 19)
        return fail(h, MKB_ERR_BAD_ARG, "id and model widths must be 1 to 19");
    if (col_id < 0 || col_id + id_width > row_bytes || col_x < 0 || col_x + 32 > row_bytes || col_model < 0 ||
        col_model + model_width > row_bytes)
        return fail(h, MKB_ERR_BAD_ARG, "a field lies outside the row");
    if (!coords || !tmpl || !out) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if ((reinterpret_cast<uintptr_t>(coords) | reinterpret_cast<uintptr_t>(tmpl) | reinterpret_cast<uintptr_t>(out)) & 3)
        return fail(h, MKB_ERR_BAD_ARG, "coords, tmpl and out must be 4-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    const int64_t S = natoms * row_bytes;
    if (n_frames * S > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the frames take %lld", (long long)out_capacity,
                    (long long)(n_frames * S));
    const size_t smem = (size_t)FT_WARPS * ((32 * row_bytes + 4 + 15) & ~15);
    MKB_CUDA(h, cudaFuncSetAttribute(cif_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (h->timing) {
        MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
        MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    }
    const dim3 grid((unsigned)cdiv(natoms, 32), (unsigned)std::min<int64_t>(cdiv(n_frames, FT_T), FT_MAX_GRID_Y));
    cif_encode_kernel<<<grid, FT_WARPS * 32, smem, st>>>(coords, frame_stride, (int)n_frames, (int)natoms, tmpl,
                                                         (int)row_bytes, (int)col_id, (int)id_width, (int)col_x,
                                                         (int)col_model, (int)model_width, frame0, out);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
