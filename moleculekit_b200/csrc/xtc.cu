// xtc.cu -- K11 (SURVEY 8f row 4, second half): XTC compressed coordinates decoded on the device.
//
// Replaces the per-frame loop of xtc_read_new / xtc_read_frame (moleculekit/fileformats/xtc/src/xtc_src.cpp:195-258) around
// xdrfile_decompress_coord_float (src/xdrfile.cpp:750-982) and the frame-minor scatter it does on the host (xtc_src.cpp:236-
// 244).  The format (xdrfile "xdr3dfcoord"): per frame a bit stream, MSB first; every atom starts with a full-range integer
// triple stored as ONE mixed-radix number (or three plain fields when a range exceeds 24 bits), a flag bit and an optional
// 5-bit code that sets the run length (atoms coded as small offsets from their predecessor, again one mixed-radix number per
// atom) and adapts the small range up or down one step in a fixed table; the first atom of a run is emitted BEFORE the atom
// it was coded against (water oxygen / hydrogen order).  Coordinates are (float)int * (float)(1.0 / precision), in nm.
//
// Frames are independent and the stream of one frame is inherently sequential, so: ONE THREAD PER FRAME.  The output
// layout is frame-minor (natoms, 3, F): thread f writes element (a, d, f), so a warp that is in step writes 32
// consecutive floats.  Mixed-radix numbers are assembled in 64-bit registers (128-bit only for the rare > 64-bit triple)
// instead of the reference's byte-array long arithmetic.  A 10 000-frame, 5 000-atom trajectory is 10 000 threads of ~2 M
// instructions each: the device decodes it in milliseconds while the compressed file (about a third of the float32 size)
// is all that crosses PCIe.
#include <cmath>
#include <vector>

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace mkb {

__constant__ int c_xtc_magic[73] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 8, 10, 12, 16, 20, 25, 32, 40, 50, 64, 80, 101, 128, 161, 203, 256,
    322, 406, 512, 645, 812, 1024, 1290, 1625, 2048, 2580, 3250, 4096, 5060, 6501, 8192, 10321, 13003, 16384, 20642, 26007, 32768,
    41285, 52015, 65536, 82570, 104031, 131072, 165140, 208063, 262144, 330280, 416127, 524287, 660561, 832255, 1048576, 1321122,
    1664510, 2097152, 2642245, 3329021, 4194304, 5284491, 6658042, 8388607, 10568983, 13316085, 16777216};
constexpr int XTC_FIRSTIDX = 9, XTC_LASTIDX = 73;

struct XtcBits {
    const unsigned *p32;   // the block as big-endian 32-bit words (XDR pads every block to 4 bytes and starts it on a word)
    long long nwords;      // words that may be read (bits past the block read as zero)
    long long word;        // next word to fetch
    unsigned long long buf;  // upcoming bits, left-aligned
    int avail;               // valid bits in buf

    __device__ __forceinline__ void init(const unsigned char *data, long long nbytes) {
        p32 = reinterpret_cast<const unsigned *>(data);
        nwords = (nbytes + 3) >> 2;
        word = 0; buf = 0; avail = 0;
    }
    // n <= 32 bits, most significant first
    __device__ __forceinline__ unsigned take(int n) {
        if (avail < n) {  // avail <= 31 here: room for one more word
            const unsigned v = word < nwords ? __byte_perm(__ldg(p32 + word), 0, 0x0123) : 0u;
            ++word;
            buf |= (unsigned long long)v << (32 - avail);
            avail += 32;
        }
        const unsigned r = n ? (unsigned)(buf >> (64 - n)) : 0u;
        buf <<= n;
        avail -= n;
        return r;
    }
    // an nbits-bit field as stored (MSB first), nbits <= 64
    __device__ __forceinline__ unsigned long long take64(int nbits) {
        if (nbits <= 32) return take(nbits);
        const unsigned long long hi = take(nbits - 32);
        return (hi << 32) | take(32);
    }
    // three integers packed as one mixed-radix number of nbits bits, stored in 8-bit chunks with the LEAST significant
    // chunk first in the stream: k full chunks then r = nbits - 8k remaining bits (the most significant ones)
    __device__ __forceinline__ void take3(int nbits, unsigned s1, unsigned s2, int out[3]) {
        if (nbits <= 64) {
            const unsigned long long V = take64(nbits);
            const int k = (nbits - 1) >> 3, r = nbits - 8 * k;
            unsigned long long v = V;
            if (k > 0) {
                const unsigned long long W = V >> r;  // the k chunks, first chunk most significant
                const unsigned lo = (unsigned)W, hi = (unsigned)(W >> 32);
                const unsigned long long rev = ((unsigned long long)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
                v = ((V & ((1ull << r) - 1ull)) << (8 * k)) | (rev >> (64 - 8 * k));
            }
            if (v <= 0xffffffffull) {  // the common small-offset case: 32-bit divisions
                unsigned u = (unsigned)v;
                out[2] = (int)(u % s2); u /= s2;
                out[1] = (int)(u % s1); out[0] = (int)(u / s1);
            } else {
                out[2] = (int)(v % s2); v /= s2;
                out[1] = (int)(v % s1); out[0] = (int)(unsigned)(v / s1);
            }
        } else {
            unsigned __int128 v = 0;
            int shift = 0, left = nbits;
            while (left > 8) { v |= (unsigned __int128)take(8) << shift; shift += 8; left -= 8; }
            if (left > 0) v |= (unsigned __int128)take(left) << shift;
            out[2] = (int)(unsigned)(v % s2); v /= s2;
            out[1] = (int)(unsigned)(v % s1); out[0] = (int)(unsigned)(v / s1);
        }
    }
};

__device__ __forceinline__ int xtc_bits_of(unsigned size) {  // xdrfile.cpp:455-465
    int n = 0;
    unsigned long long num = 1;
    while (size >= num && n < 32) { ++n; num <<= 1; }
    return n;
}

__device__ __forceinline__ int xtc_bits_of3(unsigned a, unsigned b, unsigned c) {  // xdrfile.cpp:480-510
    unsigned __int128 t = (unsigned __int128)a * b * c;
    int nbytes = 0;
    while (t > 0xff) { t >>= 8; ++nbytes; }
    int nb = 0;
    unsigned num = 1;
    while ((unsigned)t >= num) { ++nb; num *= 2; }
    return nb + nbytes * 8;
}

struct XtcFrame {  // == mkb_xtc_frame
    long long data_offset;
    int nbytes, natoms;
    float precision;
    int minint[3], maxint[3];
    int smallidx;
};

__device__ __forceinline__ float xtc_be_float(const unsigned char *p) {
    return __uint_as_float(((unsigned)p[0] << 24) | ((unsigned)p[1] << 16) | ((unsigned)p[2] << 8) | (unsigned)p[3]);
}

__global__ void xtc_decode_kernel(const unsigned char *__restrict__ file, long long file_size,
                                  const XtcFrame *__restrict__ frames, long long F, long long natoms, float *__restrict__ out,
                                  long long fs, float scale, int *__restrict__ status) {
    const long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (f >= F) return;
    const XtcFrame fr = frames[f];
    float *col = out + f;  // element (a, d) of this frame: col[(a*3 + d) * fs]
    const bool rescale = scale != 1.0f;
    auto emit = [&](long long w, float v) { col[w * fs] = rescale ? __fmul_rn(v, scale) : v; };
    if (fr.natoms != natoms || fr.data_offset < 0 || fr.nbytes < 0 || fr.data_offset + fr.nbytes > file_size ||
        ((reinterpret_cast<unsigned long long>(file) + (unsigned long long)fr.data_offset) & 3ull)) {  // XDR: word aligned
        status[f] = -1;
        return;
    }
    const unsigned char *data = file + fr.data_offset;
    if (fr.smallidx < 0) {  // <= 9 atoms: plain big-endian floats (xdrfile.cpp:802-806)
        if (fr.nbytes != 12 * natoms) { status[f] = -1; return; }
        for (long long w = 0; w < 3 * natoms; ++w) emit(w, xtc_be_float(data + 4 * w));
        return;
    }
    // Lattice arithmetic is modulo 2^32, as the format defines it: a range of 2^31 or more, or a run next to INT_MIN,
    // overflows signed int, so sizes and sums are formed in unsigned and only the final coordinate is read as int.
    unsigned sizeint[3];
    int bitsizeint[3] = {0, 0, 0};
#pragma unroll
    for (int d = 0; d < 3; ++d) sizeint[d] = (unsigned)fr.maxint[d] - (unsigned)fr.minint[d] + 1u;
    if (!sizeint[0] || !sizeint[1] || !sizeint[2]) { status[f] = -2; return; }
    int bitsize;
    if ((sizeint[0] | sizeint[1] | sizeint[2]) > 0xffffffu) {
#pragma unroll
        for (int d = 0; d < 3; ++d) bitsizeint[d] = xtc_bits_of(sizeint[d]);
        bitsize = 0;
    } else {
        bitsize = xtc_bits_of3(sizeint[0], sizeint[1], sizeint[2]);
    }
    int smallidx = fr.smallidx;
    if (smallidx < XTC_FIRSTIDX || smallidx >= XTC_LASTIDX) { status[f] = -3; return; }
    int smaller = c_xtc_magic[max(smallidx - 1, XTC_FIRSTIDX)] / 2;
    int smallnum = c_xtc_magic[smallidx] / 2;
    unsigned sizesmall = (unsigned)c_xtc_magic[smallidx];
    const float inv_precision = (float)(1.0 / (double)fr.precision);
    XtcBits b;
    b.init(data, (long long)fr.nbytes);
    long long i = 0, w = 0;
    const long long wmax = 3 * natoms;
    int run = 0;
    while (i < natoms) {
        int cur[3], prev[3];
        if (bitsize == 0) {
#pragma unroll
            for (int d = 0; d < 3; ++d) cur[d] = (int)b.take(bitsizeint[d]);
        } else {
            b.take3(bitsize, sizeint[1], sizeint[2], cur);
        }
        ++i;
#pragma unroll
        for (int d = 0; d < 3; ++d) { cur[d] = (int)((unsigned)cur[d] + (unsigned)fr.minint[d]); prev[d] = cur[d]; }
        int is_smaller = 0;
        if (b.take(1)) {
            run = (int)b.take(5);
            is_smaller = run % 3;
            run -= is_smaller;
            --is_smaller;
        }
        if (run > 0) {
            for (int k = 0; k < run; k += 3) {
                int s[3];
                b.take3(smallidx, sizesmall, sizesmall, s);
                ++i;
#pragma unroll
                for (int d = 0; d < 3; ++d) s[d] = (int)((unsigned)s[d] + (unsigned)prev[d] - (unsigned)smallnum);
                if (w + (k == 0 ? 6 : 3) > wmax) { status[f] = -4; return; }
                if (k == 0) {  // the first atom of a run is written before the atom it was coded against
#pragma unroll
                    for (int d = 0; d < 3; ++d) { emit(w++, __fmul_rn((float)s[d], inv_precision)); prev[d] = s[d]; s[d] = cur[d]; }
                } else {
#pragma unroll
                    for (int d = 0; d < 3; ++d) prev[d] = s[d];
                }
#pragma unroll
                for (int d = 0; d < 3; ++d) emit(w++, __fmul_rn((float)s[d], inv_precision));
            }
        } else {
            if (w + 3 > wmax) { status[f] = -4; return; }
#pragma unroll
            for (int d = 0; d < 3; ++d) emit(w++, __fmul_rn((float)cur[d], inv_precision));
        }
        smallidx += is_smaller;
        if (smallidx < XTC_FIRSTIDX - 1 || smallidx >= XTC_LASTIDX) { status[f] = -3; return; }
        if (is_smaller < 0) {
            smallnum = smaller;
            smaller = smallidx > XTC_FIRSTIDX ? c_xtc_magic[smallidx - 1] / 2 : 0;
        } else if (is_smaller > 0) {
            smaller = smallnum;
            smallnum = c_xtc_magic[smallidx] / 2;
        }
        sizesmall = (unsigned)c_xtc_magic[smallidx];
        if (!sizesmall) { status[f] = -3; return; }
    }
    if (w != wmax) status[f] = -4;
}

}  // namespace mkb

using namespace mkb;

extern "C" int mkb_xtc_decode(mkb_handle_t h, void *stream, const uint8_t *file_bytes, int64_t file_size,
                              const mkb_xtc_frame *frames, int64_t n_frames, int64_t natoms, float *coords,
                              int64_t frame_stride, float scale, int32_t *status) {
    static_assert(sizeof(mkb_xtc_frame) == sizeof(XtcFrame) && sizeof(XtcFrame) == 48, "frame descriptor layout");
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || file_size < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0 || natoms == 0) return MKB_OK;
    if (!file_bytes || !frames || !coords || !status) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (natoms >= (1ll << 31) / 3) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    XtcFrame *d_frames;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames * sizeof(XtcFrame), (void **)&d_frames))) return rc;
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemcpyAsync(d_frames, frames, sizeof(XtcFrame) * (size_t)n_frames, cudaMemcpyHostToDevice, st));
    MKB_CUDA(h, cudaMemsetAsync(status, 0, sizeof(int32_t) * (size_t)n_frames, st));
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    xtc_decode_kernel<<<(unsigned)cdiv(n_frames, 64), 64, 0, st>>>(file_bytes, file_size, d_frames, n_frames, natoms, coords,
                                                                    frame_stride, scale, status);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// K21: XTC encode -- the writer's half of the codec (xdrfile_compress_coord_float, src/xdrfile.cpp; restated in
// oracle/xtc_writer.py::compress_frame, which the tests hold this kernel to byte for byte).
//
// The same mapping as the decoder: ONE THREAD PER FRAME, reading element (a, d, f) of the frame-minor array, so a warp in
// step reads 32 consecutive floats.  The length of a frame's stream is known only once it has been written, so the
// kernel runs twice: a size pass that takes the per-frame reductions (lattice ranges, the smallest consecutive distance,
// the overflow tests) and walks the stream counting bits, and, after an exclusive scan of the block lengths, a write pass
// that walks it again and stores 32-bit words at the frame's offset.  Blocks are therefore packed back to back with no
// slack, no scratch buffer and no copy.  All lattice arithmetic that the reference does in C `int` is done modulo 2^32
// here; every float step is individually rounded (the reference binary has no FMA).
namespace mkb {

constexpr long long XTC_ENC_MAX_ATOMS = 100000000;  // 102 bits per atom at most: the byte count of a block stays an int32

struct XtcEncHead {  // what the size pass found and the write pass needs
    int minint[3], maxint[3];
    int smallidx;
};

// MSB-first bit output in 32-bit big-endian words; without WRITE only the bit count is kept
template <bool WRITE>
struct XtcPut {
    unsigned *p32;           // next word of the stream
    unsigned long long acc;  // bits not stored yet, right-aligned
    int n;                   // how many: < 32 between calls
    long long nbits;         // bits sent in all

    __device__ __forceinline__ void init(unsigned char *p) {
        p32 = reinterpret_cast<unsigned *>(p);
        acc = 0; n = 0; nbits = 0;
    }
    // the w <= 32 low bits of v (v has no bit above them)
    __device__ __forceinline__ void put(int w, unsigned v) {
        nbits += w;
        if (WRITE) {
            acc = (acc << w) | v;
            n += w;
            if (n >= 32) {
                n -= 32;
                *p32++ = __byte_perm((unsigned)(acc >> n), 0, 0x0123);
            }
        }
    }
    // three integers as one mixed-radix number ((a*s1 + b)*s2 + c) of nbits <= 72 bits: 8-bit chunks, least significant
    // first, then the remaining high bits (encodeints; the inverse of XtcBits::take3).  The number is kept as a 128-bit
    // (hi, lo) pair whatever its size: one path for every triple.
    __device__ __forceinline__ void put3(int nbits3, unsigned a, unsigned b, unsigned c, unsigned s1, unsigned s2) {
        if (!WRITE) { nbits += nbits3; return; }
        const unsigned long long t = (unsigned long long)a * s1 + b;
        unsigned long long lo = t * s2, hi = __umul64hi(t, (unsigned long long)s2);
        lo += c;
        hi += lo < c;
        int left = nbits3;
        while (left > 8) {
            put(8, (unsigned)lo & 0xffu);
            lo = (lo >> 8) | (hi << 56);
            hi >>= 8;
            left -= 8;
        }
        put(left, (unsigned)lo);
    }
    // the last partial word, its unused bits zero: this is also the XDR padding of the block
    __device__ __forceinline__ void flush() {
        if (WRITE && n > 0) *p32 = __byte_perm((unsigned)(acc << (32 - n)), 0, 0x0123);
    }
};

__device__ __forceinline__ bool xtc_near(const int (&a)[3], const int (&b)[3], int lim) {  // C abs(): abs(INT_MIN) < 0
    return abs((int)((unsigned)a[0] - (unsigned)b[0])) < lim && abs((int)((unsigned)a[1] - (unsigned)b[1])) < lim &&
           abs((int)((unsigned)a[2] - (unsigned)b[2])) < lim;
}

template <bool WRITE>
__global__ void __launch_bounds__(64)
xtc_encode_kernel(const float *__restrict__ coords, long long fs, long long F, int natoms, float precision, float scale,
                  XtcEncHead *__restrict__ heads, unsigned char *__restrict__ out, long long *__restrict__ offsets,
                  int *__restrict__ nbytes_out, int *__restrict__ status) {
    const long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (f >= F) return;
    const float *col = coords + f;  // element (a, d) of this frame: col[(a*3 + d) * fs]
    const bool rescale = scale != 1.0f;
    auto real = [&](long long w) {
        const float x = __ldg(col + w * fs);
        return rescale ? __fmul_rn(x, scale) : x;
    };
    if (natoms <= 9) {  // plain big-endian floats (xdrfile.cpp: size <= 9)
        if (WRITE) {
            unsigned *o = reinterpret_cast<unsigned *>(out + offsets[f]);
            for (int w = 0; w < 3 * natoms; ++w) o[w] = __byte_perm(__float_as_uint(real(w)), 0, 0x0123);
        } else {
            nbytes_out[f] = 12 * natoms;
            offsets[f + 1] = 12 * natoms;
        }
        return;
    }
    // float -> lattice: lf = x * precision, +- 0.5 by the sign of x, truncate; |lf| > INT_MAX - 2 (or not a number, where
    // the reference's conversion is undefined) is the reference's "Internal overflow compressing coordinates"
    bool bad = false;
    auto lattice = [&](int a, int (&c)[3]) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float x = real(3ll * a + d);
            float lf = __fmul_rn(x, precision);
            lf = x >= 0.0f ? __fadd_rn(lf, 0.5f) : __fsub_rn(lf, 0.5f);
            bad |= !(fabs((double)lf) <= 2147483645.0);
            c[d] = (int)lf;
        }
    };
    XtcEncHead hd;
    if (!WRITE) {
        int mindiff = INT_MAX, old[3] = {0, 0, 0};
#pragma unroll
        for (int d = 0; d < 3; ++d) { hd.minint[d] = INT_MAX; hd.maxint[d] = INT_MIN; }
        for (int a = 0; a < natoms; ++a) {
            int c[3];
            lattice(a, c);
            unsigned diff = 0;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                hd.minint[d] = min(hd.minint[d], c[d]);
                hd.maxint[d] = max(hd.maxint[d], c[d]);
                diff += (unsigned)abs((int)((unsigned)c[d] - (unsigned)old[d]));
                old[d] = c[d];
            }
            if (a > 0) mindiff = min(mindiff, (int)diff);
        }
        int st = 0;
        hd.smallidx = XTC_FIRSTIDX;
        if (bad) {
            st = MKB_XTC_ENC_COORD_OVERFLOW;
        } else if (__fsub_rn((float)hd.maxint[0], (float)hd.minint[0]) >= 2147483648.0f ||  // (float)(INT_MAX - 2) = 2^31
                   __fsub_rn((float)hd.maxint[1], (float)hd.minint[1]) >= 2147483648.0f ||
                   __fsub_rn((float)hd.maxint[2], (float)hd.minint[2]) >= 2147483648.0f) {
            st = MKB_XTC_ENC_RANGE_OVERFLOW;
        } else {
            while (hd.smallidx < XTC_LASTIDX && c_xtc_magic[hd.smallidx] < mindiff) ++hd.smallidx;
            if (hd.smallidx + 8 >= XTC_LASTIDX) st = MKB_XTC_ENC_SMALLIDX_RANGE;  // the reference reads magicints[73]
        }
        if (st) {
            status[f] = st;
            nbytes_out[f] = 0;
            offsets[f + 1] = 0;
            return;
        }
        heads[f] = hd;
    } else {
        if (status[f] != 0) return;
        hd = heads[f];
    }
    unsigned sizeint[3];
    int bitsizeint[3] = {0, 0, 0};
#pragma unroll
    for (int d = 0; d < 3; ++d) sizeint[d] = (unsigned)hd.maxint[d] - (unsigned)hd.minint[d] + 1u;
    int bitsize;
    if ((sizeint[0] | sizeint[1] | sizeint[2]) > 0xffffffu) {
#pragma unroll
        for (int d = 0; d < 3; ++d) bitsizeint[d] = xtc_bits_of(sizeint[d]);
        bitsize = 0;
    } else {
        bitsize = xtc_bits_of3(sizeint[0], sizeint[1], sizeint[2]);
    }
    int smallidx = hd.smallidx;
    const int minidx = smallidx, maxidx = smallidx + 8;  // maxidx < LASTIDX was checked by the size pass
    const int larger = c_xtc_magic[maxidx] / 2;
    int smaller = c_xtc_magic[max(XTC_FIRSTIDX, smallidx - 1)] / 2;
    int smallnum = c_xtc_magic[smallidx] / 2;
    unsigned sizesmall = (unsigned)c_xtc_magic[smallidx];
    unsigned char *block = WRITE ? out + offsets[f] : nullptr;
    XtcPut<WRITE> b;
    b.init(WRITE ? block + 36 : nullptr);
    int prevrun = -1, prev[3] = {0, 0, 0}, nxt[3];
    lattice(0, nxt);  // nxt = atom i in the writer's order (the first two atoms of a run trade places) while i < natoms
    int i = 0;
    while (i < natoms) {
        int cur[3] = {nxt[0], nxt[1], nxt[2]};
        int is_smaller;
        if (smallidx < maxidx && i >= 1 && xtc_near(cur, prev, larger)) is_smaller = 1;
        else if (smallidx > minidx) is_smaller = -1;
        else is_smaller = 0;
        bool is_small = false;
        if (i + 1 < natoms) {
            int nn[3];
            lattice(i + 1, nn);
            is_small = xtc_near(cur, nn, smallnum);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                if (is_small) { nxt[d] = cur[d]; cur[d] = nn[d]; }  // water O then H: the second atom is sent in full
                else nxt[d] = nn[d];
            }
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) prev[d] = cur[d];
        ++i;
        if (!is_small && is_smaller == -1) is_smaller = 0;
        if (bitsize == 0) {
#pragma unroll
            for (int d = 0; d < 3; ++d) b.put(bitsizeint[d], (unsigned)cur[d] - (unsigned)hd.minint[d]);
        } else {
            b.put3(bitsize, (unsigned)cur[0] - (unsigned)hd.minint[0], (unsigned)cur[1] - (unsigned)hd.minint[1],
                   (unsigned)cur[2] - (unsigned)hd.minint[2], sizeint[1], sizeint[2]);
        }
        // the run: up to 8 atoms, each within smallnum of its predecessor, kept as their small offsets until the flag
        // that precedes them in the stream is known
        unsigned run[8][3];
        int nrun = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (is_small) {
                unsigned tmpsum = 0;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    const unsigned dd = (unsigned)nxt[d] - (unsigned)prev[d];
                    tmpsum += dd * dd;
                    run[k][d] = dd + (unsigned)smallnum;
                    prev[d] = nxt[d];
                }
                if (is_smaller == -1 && (int)tmpsum >= (int)((unsigned)smaller * (unsigned)smaller)) is_smaller = 0;
                ++i;
                nrun = k + 1;
                is_small = false;
                if (i < natoms) {
                    lattice(i, nxt);
                    is_small = xtc_near(nxt, prev, smallnum);
                }
            }
        }
        if (3 * nrun != prevrun || is_smaller != 0) {  // flag bit 1 and the 5-bit code
            prevrun = 3 * nrun;
            b.put(6, 32u | (unsigned)(3 * nrun + is_smaller + 1));
        } else {
            b.put(1, 0u);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < nrun) b.put3(smallidx, run[k][0], run[k][1], run[k][2], sizesmall, sizesmall);
        if (is_smaller != 0) {
            smallidx += is_smaller;
            smaller = is_smaller < 0 ? c_xtc_magic[smallidx - 1] / 2 : smallnum;
            smallnum = c_xtc_magic[smallidx] / 2;
            sizesmall = (unsigned)c_xtc_magic[smallidx];
        }
    }
    b.flush();
    const int nbytes = (int)((b.nbits + 7) >> 3);
    if (WRITE) {
        unsigned *hw = reinterpret_cast<unsigned *>(block);
        hw[0] = __byte_perm(__float_as_uint(precision), 0, 0x0123);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            hw[1 + d] = __byte_perm((unsigned)hd.minint[d], 0, 0x0123);
            hw[4 + d] = __byte_perm((unsigned)hd.maxint[d], 0, 0x0123);
        }
        hw[7] = __byte_perm((unsigned)hd.smallidx, 0, 0x0123);
        hw[8] = __byte_perm((unsigned)nbytes, 0, 0x0123);
    } else {
        const int len = 36 + ((nbytes + 3) & ~3);
        nbytes_out[f] = len;
        offsets[f + 1] = len;
    }
}

}  // namespace mkb

extern "C" int mkb_xtc_encode(mkb_handle_t h, void *stream, const float *coords, int64_t frame_stride, int64_t n_frames,
                              int64_t natoms, float precision, float scale, uint8_t *out_bytes, int64_t out_capacity,
                              int64_t *frame_offsets, int32_t *frame_nbytes, int32_t *status) {
    MKB_ENTER(h);
    cudaStream_t st = (cudaStream_t)stream;
    MKB_STREAM_ORDER(h, st);
    if (n_frames < 0 || natoms < 0 || out_capacity < 0) return fail(h, MKB_ERR_BAD_ARG, "negative size");
    if (n_frames == 0 || natoms == 0) return MKB_OK;
    if (!coords || !frame_offsets || !frame_nbytes || !status) return fail(h, MKB_ERR_BAD_ARG, "null argument");
    if (out_capacity > 0 && !out_bytes) return fail(h, MKB_ERR_BAD_ARG, "null out_bytes with a capacity");
    if (reinterpret_cast<uintptr_t>(out_bytes) & 3) return fail(h, MKB_ERR_BAD_ARG, "out_bytes must be 4-byte aligned");
    if (frame_stride < n_frames) return fail(h, MKB_ERR_BAD_ARG, "frame stride < n_frames");
    if (natoms > XTC_ENC_MAX_ATOMS) return fail(h, MKB_ERR_BAD_ARG, "too many atoms");
    if (n_frames >= (1ll << 31) - 1) return fail(h, MKB_ERR_BAD_ARG, "too many frames for one call");
    if (!(precision > 0.0f)) precision = 1000.0f;  // the reference's rule, before the float -> int step
    XtcEncHead *heads;
    int rc;
    if ((rc = scratch_get(h, S_DESC, (size_t)n_frames, &heads))) return rc;
    long long *offsets = reinterpret_cast<long long *>(frame_offsets);
    size_t tmp_bytes = 0;
    MKB_CUDA(h, cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, offsets + 1, offsets + 1, (int)n_frames, st));
    void *tmp = nullptr;
    if ((rc = scratch_get(h, S_SCAN_TMP, tmp_bytes, &tmp))) return rc;
    const unsigned grid = (unsigned)cdiv(n_frames, 64);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[0], st));
    MKB_CUDA(h, cudaMemsetAsync(status, 0, sizeof(int32_t) * (size_t)n_frames, st));
    MKB_CUDA(h, cudaMemsetAsync(offsets, 0, sizeof(long long), st));
    // size pass: block lengths into frame_nbytes and, as int64, into frame_offsets[1..], which the scan turns into offsets
    xtc_encode_kernel<false><<<grid, 64, 0, st>>>(coords, frame_stride, n_frames, (int)natoms, precision, scale, heads,
                                                  nullptr, offsets, frame_nbytes, status);
    MKB_LAUNCHED(h);
    MKB_CUDA(h, cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, offsets + 1, offsets + 1, (int)n_frames, st));
    h->launches++;
    long long total = 0;
    MKB_CUDA(h, cudaMemcpyAsync(&total, offsets + n_frames, sizeof(long long), cudaMemcpyDeviceToHost, st));
    MKB_CUDA(h, cudaStreamSynchronize(st));
    if (total > out_capacity)
        return fail(h, MKB_ERR_CAPACITY, "out_capacity is %lld bytes, the blocks take %lld (frame_offsets[n_frames])",
                    (long long)out_capacity, total);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[1], st));
    xtc_encode_kernel<true><<<grid, 64, 0, st>>>(coords, frame_stride, n_frames, (int)natoms, precision, scale, heads,
                                                 out_bytes, offsets, frame_nbytes, status);
    MKB_LAUNCHED(h);
    if (h->timing) MKB_CUDA(h, cudaEventRecord(h->ev[2], st));
    return MKB_OK;
}
