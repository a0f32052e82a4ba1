// lammpstrj_g9.cuh -- K32's number formatter: '%.9g' % float(np.float32(v)) and '%d' of an int64, byte for byte
// Python's % formatting.  Builds for the device (lammpstrj.cu) and, with a host compiler, for a CPU check against Python.
//
// '%.9g' is the shortest %g precision that round-trips every float32, so a written file reads back to the same bits.
// The nine significant digits are exact: v = m 2^e (m < 2^24) is scaled by 10^s, s = 8 - k with k the decimal exponent,
// as the fraction A / B of two integers held in five 32-bit limbs -- A = 2 m 5^s 2^(e+s) and B = 1 or 2^-(e+s) for
// s >= 0, A = 2 m 2^(e-s') and B = 5^s' for s = -s' < 0 (then e >= s').  floor(A / B) is a shift or a chain of
// divisions by 5^13 and a smaller power (floors compose), and a sticky bit records a non-zero remainder; the low bit
// of the quotient is then the half-digit and the sticky bit decides above half or an exact tie (to the even digit, as
// Python's dtoa does).  No float64 product is involved.  The result is at most 15 bytes ("-1.23456789e-38").
#pragma once

#include "xyz_number.cuh"

namespace mkb {

constexpr int G9_MAX = 15;   // longest '%.9g' of a float32
constexpr int G9_INT_MAX = 20;  // longest '%d' of an int64

struct G9Big {
    unsigned w[5];  // little-endian 32-bit limbs
};

XYZ_FN void g9_mul(G9Big &a, unsigned x) {
    unsigned long long c = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
        c += (unsigned long long)a.w[i] * x;
        a.w[i] = (unsigned)c;
        c >>= 32;
    }
}

XYZ_FN void g9_shl(G9Big &a, int n) {  // 0 <= n < 160
    const int q = n >> 5, r = n & 31;
    for (int i = 4; i >= 0; --i) {
        const unsigned hi = i - q >= 0 ? a.w[i - q] : 0u, lo = i - q - 1 >= 0 ? a.w[i - q - 1] : 0u;
        a.w[i] = r ? (hi << r) | (lo >> (32 - r)) : hi;
    }
}

// a >>= n; sticky |= the bits shifted out were not all zero
XYZ_FN void g9_shr(G9Big &a, int n, bool &sticky) {
    if (n >= 160) {
        for (int i = 0; i < 5; ++i) {
            sticky |= a.w[i] != 0u;
            a.w[i] = 0u;
        }
        return;
    }
    const int q = n >> 5, r = n & 31;
    for (int i = 0; i < q; ++i) sticky |= a.w[i] != 0u;
    if (r) sticky |= (a.w[q] & ((1u << r) - 1u)) != 0u;
    for (int i = 0; i < 5; ++i) {
        const unsigned lo = i + q < 5 ? a.w[i + q] : 0u, hi = i + q + 1 < 5 ? a.w[i + q + 1] : 0u;
        a.w[i] = r ? (lo >> r) | (hi << (32 - r)) : lo;
    }
}

XYZ_FN void g9_div(G9Big &a, unsigned d, bool &sticky) {
    unsigned long long r = 0;
    for (int i = 4; i >= 0; --i) {
        const unsigned long long cur = (r << 32) | a.w[i];
        a.w[i] = (unsigned)(cur / d);
        r = cur % d;
    }
    sticky |= r != 0;
}

XYZ_FN unsigned g9_pow5(int n) {  // 0 <= n <= 13
    unsigned p = 1u;
    for (int i = 0; i < n; ++i) p *= 5u;
    return p;
}

// floor(m 2^e 10^s) and the value rounded to an integer, ties to even
XYZ_FN void g9_scaled(unsigned m, int e, int s, unsigned long long &fl, unsigned long long &rn) {
    G9Big a = {{m, 0u, 0u, 0u, 0u}};
    bool sticky = false;
    if (s >= 0) {
        for (int t = s; t > 0; t -= 13) g9_mul(a, g9_pow5(t < 13 ? t : 13));
        const int sh = e + s + 1;
        if (sh >= 0) g9_shl(a, sh);
        else g9_shr(a, -sh, sticky);
    } else {
        g9_shl(a, e + s + 1);  // e >= -s here: a float32 of at least 10^9 has e >= 6 and m 2^e >= 10^k
        for (int t = -s; t > 0; t -= 13) g9_div(a, g9_pow5(t < 13 ? t : 13), sticky);
    }
    const unsigned long long q2 = ((unsigned long long)a.w[1] << 32) | a.w[0];
    fl = q2 >> 1;
    rn = fl + ((q2 & 1ull) && (sticky || (fl & 1ull)) ? 1ull : 0ull);
}

// '%.9g' % float(x) into d (at least G9_MAX bytes) -> its length
XYZ_FN int g9_format(float x, unsigned char *d) {
    unsigned u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(x);
#else
    std::memcpy(&u, &x, 4);
#endif
    const bool neg = u >> 31;
    const unsigned ex = (u >> 23) & 0xffu, mant = u & 0x7fffffu;
    int n = 0;
    if (ex == 0xffu) {
        if (mant) {
            d[0] = 'n'; d[1] = 'a'; d[2] = 'n';
            return 3;
        }
        if (neg) d[n++] = '-';
        d[n] = 'i'; d[n + 1] = 'n'; d[n + 2] = 'f';
        return n + 3;
    }
    if (neg) d[n++] = '-';
    if (ex == 0u && mant == 0u) {
        d[n] = '0';
        return n + 1;
    }
    const unsigned m = ex ? mant | 0x800000u : mant;
    const int e = ex ? (int)ex - 150 : -149;
    const int b = e + 31 - xyz_clz((unsigned long long)m) + 32;  // floor(log2 |x|)
    int k = (b * 78913) >> 18;  // floor(b log10 2): the decimal exponent or one below it
    unsigned long long fl, D;
    g9_scaled(m, e, 8 - k, fl, D);
    if (fl >= 1000000000ull) {
        ++k;
        g9_scaled(m, e, 8 - k, fl, D);
    }
    if (D == 1000000000ull) {  // rounded up to the next power of ten
        D = 100000000ull;
        ++k;
    }
    unsigned char dig[9];
    unsigned long long t = D;
    for (int i = 8; i >= 0; --i) {
        dig[i] = (unsigned char)('0' + t % 10ull);
        t /= 10ull;
    }
    int last = 8;  // the last digit kept: trailing zeros are stripped
    while (last > 0 && dig[last] == '0') --last;
    if (k >= -4 && k < 9) {
        if (k >= 0) {
            for (int i = 0; i <= k; ++i) d[n++] = dig[i];
            if (last > k) {
                d[n++] = '.';
                for (int i = k + 1; i <= last; ++i) d[n++] = dig[i];
            }
        } else {
            d[n++] = '0';
            d[n++] = '.';
            for (int i = 0; i < -k - 1; ++i) d[n++] = '0';
            for (int i = 0; i <= last; ++i) d[n++] = dig[i];
        }
        return n;
    }
    d[n++] = dig[0];
    if (last > 0) {
        d[n++] = '.';
        for (int i = 1; i <= last; ++i) d[n++] = dig[i];
    }
    d[n++] = 'e';
    d[n++] = k < 0 ? '-' : '+';
    const int ak = k < 0 ? -k : k;
    d[n++] = (unsigned char)('0' + ak / 10);
    d[n++] = (unsigned char)('0' + ak % 10);
    return n;
}

// '%d' % v into d (at least G9_INT_MAX bytes) -> its length
XYZ_FN int g9_int(long long v, unsigned char *d) {
    unsigned long long t = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    unsigned char tmp[G9_INT_MAX];
    int n = 0;
    do {
        tmp[n++] = (unsigned char)('0' + t % 10ull);
        t /= 10ull;
    } while (t);
    int o = 0;
    if (v < 0) d[o++] = '-';
    while (n) d[o++] = tmp[--n];
    return o;
}

}  // namespace mkb
