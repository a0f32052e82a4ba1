// f83.cuh -- fixed-width decimal fields with SWAR code: Fortran F8.3 parsed and formatted (K25's mdcrd fields, K28's PDB
// coordinate columns, K29's GRO positions), F8.4 parsed (K29's GRO velocities), and the general '%W.Df' formatter K28
// uses for the CRYST1 fields and K29 for the velocities and the box.
//
// Arithmetic (the contract with Python's float() and '%W.Df'):
//   parse   the digits k of an F8.3 field (point removed, k < 10^7) give __double2float_rn((double)k / 1000.0), the sign
//           applied afterwards: the double division is correctly rounded like float(), so both round the decimal once
//           to double and once to float32, and '-0.000' gives -0.0.
//   format  k = rint((double)x * 10^D) is exact before the rounding for D <= 12 (a float32 times 10^D fits 53 bits) and
//           rounds half to even, which is what printf's correctly rounded '%.Df' does; the sign of x is printed even
//           when k == 0.
//
// The helpers have internal linkage, so each .cu that includes this header inlines its own copies.
#pragma once

namespace mkb {
namespace {

// per byte: bit 7 set where the byte is not zero
__device__ __forceinline__ unsigned md_nonzero(unsigned x) { return (((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u; }
// per byte of x ^ '0000': bit 7 set where the byte is not a digit
__device__ __forceinline__ unsigned md_nondigit(unsigned d) { return (((d & 0x7f7f7f7fu) + 0x76767676u) | d) & 0x80808080u; }

// The 8 characters of a field as two little-endian words (lo: characters 0-3, hi: 4-7) -> float32 bits.  ok = the
// field matches spaces, an optional '-', digits, '.', three digits.
__device__ __forceinline__ unsigned md_parse(unsigned lo, unsigned hi, bool &ok) {
    constexpr unsigned H = 0x80808080u;
    const unsigned dl = lo ^ 0x30303030u, dh = hi ^ 0x30303030u;
    const unsigned D = ~md_nondigit(dl) & H, Sp = ~md_nonzero(lo ^ 0x20202020u) & H, M = ~md_nonzero(lo ^ 0x2d2d2d2du) & H;
    const unsigned smask = (Sp >> 7) * 0xffu;  // 0xff in every space byte
    // the spaces are a prefix, a '-' (at most one) comes right after them, digits fill the rest
    ok = (D | Sp | M) == H && (smask & (smask + 1u)) == 0u && (M == 0u || (M >> 7) == smask + 1u) &&
         (hi & 0xffu) == 0x2eu && (md_nondigit(dh) & 0x80808000u) == 0u;
    const unsigned v = dl & ((D >> 7) * 0xffu);  // digit values, 0 in the other bytes
    const unsigned ip = (v & 0xffu) * 1000u + __dp4a(v, 0x010a6400u, 0u);
    const unsigned k = ip * 1000u + __dp4a(dh, 0x010a6400u, 0u);
    return __float_as_uint(__double2float_rn((double)k / 1000.0)) | (M ? 0x80000000u : 0u);
}

// The 8 characters of an F8.4 field (GRO's '%8.4f' velocities; lo: characters 0-3, hi: 4-7) -> float32 bits.  ok =
// the field matches spaces, an optional '-', digits (at most three characters before the point), '.' at character 3,
// four digits; the value is __double2float_rn(k / 10000.0) of the seven digits k, as md_parse does for three decimals.
__device__ __forceinline__ unsigned md_parse4(unsigned lo, unsigned hi, bool &ok) {
    constexpr unsigned H = 0x00808080u;  // characters 0-2
    const unsigned dl = lo ^ 0x30303030u, dh = hi ^ 0x30303030u;
    const unsigned D = ~md_nondigit(dl) & H, Sp = ~md_nonzero(lo ^ 0x20202020u) & H, M = ~md_nonzero(lo ^ 0x2d2d2d2du) & H;
    const unsigned smask = (Sp >> 7) * 0xffu;
    ok = (D | Sp | M) == H && (smask & (smask + 1u)) == 0u && (M == 0u || (M >> 7) == smask + 1u) &&
         (lo >> 24) == 0x2eu && md_nondigit(dh) == 0u;
    const unsigned v = dl & ((D >> 7) * 0xffu);
    const unsigned ip = __dp4a(v, 0x00010a64u, 0u);  // characters 0-2: 100, 10, 1
    const unsigned k = ip * 10000u + (dh & 0xffu) * 1000u + __dp4a(dh, 0x010a6400u, 0u);
    return __float_as_uint(__double2float_rn((double)k / 10000.0)) | (M ? 0x80000000u : 0u);
}

// The three aligned words covering bytes [a, a + 9) -> the field at a (lo, hi) and the byte at a + 8
__device__ __forceinline__ void md_field(const unsigned char *a, unsigned &lo, unsigned &hi, unsigned &next) {
    const unsigned *w = reinterpret_cast<const unsigned *>(reinterpret_cast<uintptr_t>(a) & ~uintptr_t(3));
    const unsigned s = reinterpret_cast<uintptr_t>(a) & 3u;
    const unsigned w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
    const unsigned sel = 0x3210u + 0x1111u * s;
    lo = __byte_perm(w0, w1, sel);
    hi = __byte_perm(w1, w2, sel);
    next = (w2 >> (8 * s)) & 0xffu;
}

// float32 -> the 8 characters of '%8.3f' (lo: characters 0-3, hi: 4-7); '********' (Fortran's overflow field) outside
// the writable range and for NaN / +-inf
__device__ __forceinline__ void md_format(float x, unsigned &lo, unsigned &hi) {
    const bool neg = signbit(x);
    const double a = fabs(rint((double)x * 1000.0));
    if (!(a <= (neg ? 999999.0 : 9999999.0))) {
        lo = hi = 0x2a2a2a2au;
        return;
    }
    const unsigned k = (unsigned)a, ip = k / 1000u, fp = k - 1000u * ip;
    hi = 0x3030302eu + ((fp / 100u) << 8) + ((fp / 10u % 10u) << 16) + ((fp % 10u) << 24);
    const unsigned digits = 0x30303030u + (ip / 1000u) + ((ip / 100u % 10u) << 8) + ((ip / 10u % 10u) << 16) +
                            ((ip % 10u) << 24);
    const int nd = ip >= 1000u ? 4 : ip >= 100u ? 3 : ip >= 10u ? 2 : 1;
    const unsigned keep = 0xffffffffu << (8 * (4 - nd));  // the last nd characters
    lo = (digits & keep) | (0x20202020u & ~keep);
    if (neg) {  // nd <= 3 here: k <= 999 999
        const int at = 8 * (3 - nd);
        lo = (lo & ~(0xffu << at)) | (0x2du << at);
    }
}

__device__ __forceinline__ void md_put(unsigned char *d, unsigned lo, unsigned hi) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        d[c] = (unsigned char)(lo >> (8 * c));
        d[4 + c] = (unsigned char)(hi >> (8 * c));
    }
}

__host__ __device__ constexpr double f_pow10(int d) { return d == 0 ? 1.0 : 10.0 * f_pow10(d - 1); }  // exact for d <= 22
__host__ __device__ constexpr int f_bits(unsigned long long v) { return v ? 1 + f_bits(v >> 1) : 0; }
__host__ __device__ constexpr unsigned long long f_pow5(int d) { return d == 0 ? 1ull : 5ull * f_pow5(d - 1); }

// '%W.Df' of x into d[0 .. W), the variant of md_format for other widths.  The caller has checked the range: rint(x
// 10^D) < 10^(W - 1), 10^(W - 2) when x is negative, and x finite.  x 10^D = x 2^D 5^D is exact in a double while the
// float32's 24-bit significand times 5^D fits 53 bits (D <= 12), so rint rounds the exact product once.
template <int W, int D>
__device__ __forceinline__ void f_format(float x, unsigned char *d) {
    static_assert(D >= 1 && 24 + f_bits(f_pow5(D)) <= 53 && W >= D + 2 && W <= 16,
                  "a float32 times 10^D must stay exact in a double");
    const bool neg = signbit(x);
    unsigned long long k = (unsigned long long)fabs(rint((double)x * f_pow10(D)));
#pragma unroll
    for (int c = W - 1; c >= W - D; --c) {
        d[c] = (unsigned char)('0' + k % 10u);
        k /= 10u;
    }
    d[W - D - 1] = '.';
    int c = W - D - 2;
    do {
        d[c--] = (unsigned char)('0' + k % 10u);
        k /= 10u;
    } while (k && c >= 0);
    if (neg && c >= 0) d[c--] = '-';
    for (; c >= 0; --c) d[c] = ' ';
}

}  // namespace
}  // namespace mkb
