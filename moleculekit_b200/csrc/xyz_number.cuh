// xyz_number.cuh -- K26's per-line grammar: the whitespace split of an XYZ atom line and the correctly rounded decimal ->
// double -> float32 conversion of its coordinate fields, the contract of np.float32(float(token)).
//
// Written for any byte reader R with `unsigned at(long long p)` that returns '\n' at and past the end of the line, so
// that the same code builds for the device (xyz.cu) and, with a host compiler, for a CPU check against Python's float().
//
//   separators  the bytes str.split() splits ASCII text on: \t \n \v \f \r, space and 0x1c-0x1f.
//   number      [+-]? (d+ .? d* | . d+) ([eE] [+-]? d+)?, or nan / inf / infinity in any case with an optional sign,
//               ended by a separator.  Anything else (an underscore, a byte >= 0x80, any other character) is left to the
//               host, which applies float() itself.
//   conversion  the first 19 significant digits w and the decimal exponent q: Clinger's fast path when w <= 2^53,
//               |q| <= 22 and no digit was dropped (one correctly rounded double product or quotient), else
//               Eisel-Lemire with the 128-bit powers of five of xyz_pow5.cuh (fast_float's compute_float).  With more
//               than 19 digits the value lies in [w, w + 1) 10^q: when w and w + 1 round to different doubles, or when
//               the 128-bit product cannot decide the rounding, the token is left to the host.  The double is then
//               rounded to float32 (to nearest even), which is np.float32(float(token)): two roundings, as the reference
//               does them.  NaN is 0x7fc00000 with the token's sign, as np.float32(float('-nan')) gives.
#pragma once

#include <type_traits>

#include "xyz_pow5.cuh"

#ifdef __CUDACC__
#define XYZ_FN __device__ __forceinline__
#else
#include <cstring>
#define XYZ_FN inline
#endif

namespace mkb {

XYZ_FN unsigned long long xyz_mulhi(unsigned long long a, unsigned long long b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (unsigned long long)(((unsigned __int128)a * b) >> 64);
#endif
}

XYZ_FN int xyz_clz(unsigned long long w) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)w);
#else
    return __builtin_clzll(w);
#endif
}

XYZ_FN unsigned long long xyz_p5(int i) {
#ifdef __CUDA_ARCH__
    return __ldg(&xyz_pow5[i]);
#else
    return xyz_pow5[i];
#endif
}

XYZ_FN unsigned xyz_f32_bits(double d) {
#ifdef __CUDA_ARCH__
    return __float_as_uint(__double2float_rn(d));
#else
    const float f = (float)d;  // to nearest even on the host's default rounding mode
    unsigned u;
    std::memcpy(&u, &f, 4);
    return u;
#endif
}

XYZ_FN unsigned long long xyz_f64_bits(double d) {
#ifdef __CUDA_ARCH__
    return (unsigned long long)__double_as_longlong(d);
#else
    unsigned long long u;
    std::memcpy(&u, &d, 8);
    return u;
#endif
}

XYZ_FN double xyz_bits_f64(unsigned long long u) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)u);
#else
    double d;
    std::memcpy(&d, &u, 8);
    return d;
#endif
}

XYZ_FN bool xyz_sep(unsigned c) { return c == ' ' || (c >= 9u && c <= 13u) || (c >= 0x1cu && c <= 0x1fu); }
XYZ_FN bool xyz_digit(unsigned c) { return c - '0' < 10u; }

// Eisel-Lemire: w != 0, the double nearest w 10^q as (biased exponent << 52 | mantissa); *undecided when the 128-bit
// product leaves the rounding open
XYZ_FN unsigned long long xyz_lemire(long long q, unsigned long long w, bool *undecided) {
    if (q < XYZ_POW5_MIN) return 0;
    if (q > XYZ_POW5_MAX) return 0x7ffull << 52;
    const int lz = xyz_clz(w);
    w <<= lz;
    const int idx = 2 * (int)(q - XYZ_POW5_MIN);
    const unsigned long long p5 = xyz_p5(idx);
    unsigned long long hi = xyz_mulhi(w, p5), lo = w * p5;
    if ((hi & 0x1ffull) == 0x1ffull) {  // the 9 bits below the 55 kept are all ones: add the low half's product
        const unsigned long long hi2 = xyz_mulhi(w, xyz_p5(idx + 1));
        lo += hi2;
        if (hi2 > lo) ++hi;
    }
    // 5^q is exact in 128 bits for -27 <= q <= 55; elsewhere a low word of all ones may hide a carry
    *undecided = lo == ~0ull && !(q >= -27 && q <= 55);
    const int upper = (int)(hi >> 63), shift = upper + 9;
    unsigned long long m = hi >> shift;
    int p2 = (int)((((152170 + 65536) * (int)q) >> 16) + 63) + upper - lz + 1023;
    if (p2 <= 0) {  // subnormal or zero
        if (-p2 + 1 >= 64) return 0;
        m >>= -p2 + 1;
        m += m & 1;
        m >>= 1;
        return m < (1ull << 52) ? m : (1ull << 52) | (m & ((1ull << 52) - 1));
    }
    // an exact halfway product (possible for -4 <= q <= 23 only) rounds to even
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << shift) == hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << 52)) {
        m = 1ull << 52;
        ++p2;
    }
    m &= ~(1ull << 52);
    if (p2 >= 0x7ff) return 0x7ffull << 52;
    return ((unsigned long long)p2 << 52) | m;
}

// The number starting at p -> *bits (float32, or with F64 the float64 that float() gives); p is left on the byte after
// it.  false: not in the device grammar, or undecided (the host re-reads the line).
template <bool F64 = false, class R>
XYZ_FN bool xyz_number(R &rd, long long &p, typename std::conditional<F64, unsigned long long, unsigned>::type &bits) {
    unsigned c = rd.at(p);
    bool neg = false;
    if (c == '+' || c == '-') {
        neg = c == '-';
        c = rd.at(++p);
    }
    const unsigned sign = neg ? 0x80000000u : 0u;
    if ((c | 0x20u) == 'n' || (c | 0x20u) == 'i') {  // nan, inf, infinity
        unsigned long long word = 0;
        int n = 0;
        while (n < 9 && !xyz_sep(c)) {
            word = (word << 8) | (c | 0x20u);  // lower case (a non-letter gives no match below)
            c = rd.at(++p);
            ++n;
        }
        if (!xyz_sep(c)) return false;
        if (n == 3 && word == 0x6e616eull) {  // "nan"
            if constexpr (F64) bits = (unsigned long long)sign << 32 | 0x7ff8000000000000ull;
            else bits = sign | 0x7fc00000u;
            return true;
        }
        if ((n == 3 && word == 0x696e66ull) || (n == 8 && word == 0x696e66696e697479ull)) {  // "inf", "infinity"
            if constexpr (F64) bits = (unsigned long long)sign << 32 | 0x7ff0000000000000ull;
            else bits = sign | 0x7f800000u;
            return true;
        }
        return false;
    }
    unsigned long long w = 0;
    long long q = 0;
    int nd = 0;
    bool any = false, dropped = false;
    for (; xyz_digit(c); c = rd.at(++p)) {
        any = true;
        if (w == 0 && c == '0') continue;  // leading zero
        if (nd < 19) {
            w = 10 * w + (c - '0');
            ++nd;
        } else {
            dropped = true;
            ++q;
        }
    }
    if (c == '.') {
        for (c = rd.at(++p); xyz_digit(c); c = rd.at(++p)) {
            any = true;
            if (w == 0 && c == '0') {
                --q;
            } else if (nd < 19) {
                w = 10 * w + (c - '0');
                ++nd;
                --q;
            } else {
                dropped = true;
            }
        }
    }
    if (!any) return false;
    if ((c | 0x20u) == 'e') {
        c = rd.at(++p);
        bool eneg = false;
        if (c == '+' || c == '-') {
            eneg = c == '-';
            c = rd.at(++p);
        }
        if (!xyz_digit(c)) return false;
        long long e = 0;
        for (; xyz_digit(c); c = rd.at(++p))
            if (e < 100000) e = 10 * e + (c - '0');  // saturates far beyond any finite, non-zero result
        q += eneg ? -e : e;
    }
    if (!xyz_sep(c)) return false;
    if (w == 0) {
        if constexpr (F64) bits = (unsigned long long)sign << 32;
        else bits = sign;
        return true;
    }
    double d;
    if (!dropped && q >= -22 && q <= 22 && w <= (1ull << 53)) {  // Clinger: both operands exact, one rounding
        double t = 1.0, s = 10.0;  // 10^|q| by squaring: every factor and product is a power of ten <= 1e22, exact
        for (int e = (int)(q < 0 ? -q : q); e; e >>= 1, s *= s)
            if (e & 1) t *= s;
        d = q < 0 ? (double)w / t : (double)w * t;
    } else {
        bool open = false;
        const unsigned long long u = xyz_lemire(q, w, &open);
        if (open) return false;
        if (dropped) {
            bool open1 = false;
            if (xyz_lemire(q, w + 1, &open1) != u || open1) return false;
        }
        d = xyz_bits_f64(u);
    }
    if constexpr (F64) bits = (unsigned long long)sign << 32 | xyz_f64_bits(d);
    else bits = sign | xyz_f32_bits(d);
    return true;
}

// the separators at p (c = the byte at p) and the number after them; false when the line ends first
template <class R>
XYZ_FN bool xyz_field(R &rd, long long &p, unsigned &c, unsigned &bits) {
    while (xyz_sep(c)) {
        if (c == '\n') return false;
        c = rd.at(++p);
    }
    if (!xyz_number(rd, p, bits)) return false;
    c = rd.at(p);
    return true;
}

// An atom line (from p to the reader's end): field 0 skipped, fields 1-3 -> x, y, z (float32 bits), the rest ignored.
// false: the host re-reads the line (fewer than four fields, a byte >= 0x80 up to field 3, or a field outside the
// device grammar).
template <class R>
XYZ_FN bool xyz_atom_line(R &rd, long long p, unsigned &x, unsigned &y, unsigned &z) {
    unsigned c = rd.at(p);
    while (xyz_sep(c)) {
        if (c == '\n') return false;
        c = rd.at(++p);
    }
    for (; !xyz_sep(c); c = rd.at(++p))
        if (c >= 0x80u) return false;
    return xyz_field(rd, p, c, x) && xyz_field(rd, p, c, y) && xyz_field(rd, p, c, z);
}

}  // namespace mkb
