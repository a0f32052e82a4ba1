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
