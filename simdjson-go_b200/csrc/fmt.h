// fmt.h -- the text Iter.MarshalJSON writes for one tape value (parsed_json.go:394-556): decimal integers, the shortest
// round-trip text of a double in appendFloat's layout (parsed_json.go:1250-1272) and escapeBytes' string escapes
// (parsed_json.go:1171-1238).
//
// Portable C++ like bits.h: under nvcc the functions are __host__ __device__ and run in the marshal kernels
// (marshal.cuh); tests/emu/fmt_shim.cpp compiles the same source with g++ so the CPU tests check it against the oracle.
//
// The double's digits come from Schubfach (R. Giulietti, "The Schubfach way to render doubles", 2020; PAPERS.md): the
// shortest decimal in the rounding interval, the one closest to the exact value among those (ties to even digit).  Its
// 128-bit powers of ten g = floor(10^q * 2^(127 - floor(log2 10^q))) + 1 are derived from the Eisel-Lemire table
// (pow10_table.inc): that table holds the floor for q >= 0 and q < -27 and already holds floor + 1 for -27 <= q < 0.
#pragma once
#include "bits.h"

namespace sj {

constexpr int FMT_POW10_MIN = -348;
#if defined(__CUDACC__)
__device__ const uint64_t FMT_POW10[696][2] = {
#include "pow10_table.inc"
};
#else
static const uint64_t FMT_POW10[696][2] = {
#include "pow10_table.inc"
};
#endif

constexpr uint64_t FMT_ABS_1E_6 = 0x3eb0c6f7a0b5ed8dull;  // the bits of 1e-6 and 1e21: appendFloat's fixed-notation range
constexpr uint64_t FMT_ABS_1E21 = 0x444b1ae4d6e2ef50ull;

SJ_HD uint64_t fmt_umulhi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// Schubfach's g for 10^q, q in [-292, 324]
SJ_HD void fmt_pow10_g(int q, uint64_t* hi, uint64_t* lo) {
#if defined(__CUDA_ARCH__) || !defined(__CUDACC__)
    uint64_t h = FMT_POW10[q - FMT_POW10_MIN][0], l = FMT_POW10[q - FMT_POW10_MIN][1];
    if (q >= 0 || q < -27) {
        l += 1;
        h += l == 0;
    }
    *hi = h;
    *lo = l;
#else
    *hi = *lo = 0;  // nvcc's host pass: the library formats on the device only
#endif
}

// floor(g * cp / 2^128), with the lowest bit set when the discarded part is not (nearly) zero: "round to odd"
SJ_HD uint64_t fmt_round_to_odd(uint64_t ghi, uint64_t glo, uint64_t cp) {
    const uint64_t x1 = fmt_umulhi(cp, glo);
    const uint64_t y0a = cp * ghi, y1a = fmt_umulhi(cp, ghi);
    const uint64_t y0 = y0a + x1;
    const uint64_t y1 = y1a + (y0 < y0a);
    return y1 | (y0 > 1);
}

struct FmtDec {
    uint64_t s;  // digits, no trailing zero
    int32_t k;   // value = s * 10^k
};

// the shortest decimal of a finite, nonzero double (sign ignored)
SJ_HD FmtDec fmt_shortest(uint64_t bits) {
    const uint64_t f = bits & ((1ull << 52) - 1);
    const uint32_t e = (uint32_t)(bits >> 52) & 0x7ff;
    uint64_t c;
    int32_t q;
    if (e) {
        c = f | (1ull << 52);
        q = (int32_t)e - 1075;
    } else {
        c = f;
        q = -1074;
    }
    const bool even = (c & 1) == 0;
    const bool closer = f == 0 && e > 1;  // the gap to the next double below is half the one above
    const uint64_t cbl = 4 * c - 2 + closer, cb = 4 * c, cbr = 4 * c + 2;
    const int32_t k = (q * 1262611 - (closer ? 524031 : 0)) >> 22;  // floor(log10(2^q)), or of 3/4 2^q when closer
    const int32_t h = q + ((-k * 1741647) >> 19) + 1;                 // q + floor(log2(10^-k)) + 1, in [1, 4]
    uint64_t ghi, glo;
    fmt_pow10_g(-k, &ghi, &glo);
    const uint64_t vbl = fmt_round_to_odd(ghi, glo, cbl << h);
    const uint64_t vb = fmt_round_to_odd(ghi, glo, cb << h);
    const uint64_t vbr = fmt_round_to_odd(ghi, glo, cbr << h);
    const uint64_t lower = vbl + !even, upper = vbr - !even;
    FmtDec r;
    const uint64_t s = vb / 4;
    bool done = false;
    if (s >= 10) {  // one digit fewer fits in the interval?
        const uint64_t sp = s / 10;
        const bool up_in = lower <= 40 * sp, wp_in = 40 * sp + 40 <= upper;
        if (up_in != wp_in) {
            r.s = sp + wp_in;
            r.k = k + 1;
            done = true;
        }
    }
    if (!done) {
        const bool u_in = lower <= 4 * s, w_in = 4 * s + 4 <= upper;
        if (u_in != w_in) {
            r.s = s + w_in;
        } else {
            const uint64_t mid = 4 * s + 2;
            r.s = s + (vb > mid || (vb == mid && (s & 1) != 0));
        }
        r.k = k;
    }
    while (r.s % 10 == 0) {
        r.s /= 10;
        r.k++;
    }
    return r;
}

SJ_HD uint32_t fmt_digits(uint64_t v) {  // decimal digits of v (1 for 0)
    uint32_t n = 1;
    uint64_t p = 10;
    while (v >= p) {
        if (++n == 20) break;
        p *= 10;
    }
    return n;
}

// the nd digits of v at o[0..nd)
SJ_HD void fmt_put_digits(uint64_t v, uint32_t nd, uint8_t* o) {
    for (uint32_t i = nd; i-- > 0;) {
        o[i] = (uint8_t)('0' + v % 10);
        v /= 10;
    }
}

// strconv.AppendUint / AppendInt base 10; W = false: the length only
template <bool W>
SJ_HD uint32_t fmt_u64(uint64_t v, uint8_t* o) {
    const uint32_t n = fmt_digits(v);
    if (W) fmt_put_digits(v, n, o);
    return n;
}
template <bool W>
SJ_HD uint32_t fmt_i64(int64_t v, uint8_t* o) {
    if (v >= 0) return fmt_u64<W>((uint64_t)v, o);
    if (W) o[0] = '-';
    return 1 + fmt_u64<W>(0 - (uint64_t)v, W ? o + 1 : o);
}

// appendFloat of a finite double: fixed notation for 1e-6 <= |x| < 1e21 and for 0, else d[.ddd]e(+|-)N
template <bool W>
SJ_HD uint32_t fmt_double(uint64_t bits, uint8_t* o) {
    const uint32_t neg = (uint32_t)(bits >> 63);
    const uint64_t mag = bits & ~(1ull << 63);
    if (W && neg) *o++ = '-';
    if (mag == 0) {
        if (W) o[0] = '0';
        return neg + 1;
    }
    const FmtDec d = fmt_shortest(mag);
    const uint32_t nd = fmt_digits(d.s);
    const int32_t E = d.k + (int32_t)nd;  // value = 0.d1d2...dn * 10^E
    if (mag >= FMT_ABS_1E_6 && mag < FMT_ABS_1E21) {
        if (E <= 0) {  // 0.000ddd
            if (W) {
                o[0] = '0';
                o[1] = '.';
                for (int32_t i = 0; i < -E; i++) o[2 + i] = '0';
                fmt_put_digits(d.s, nd, o + 2 - E);
            }
            return neg + 2 + (uint32_t)(-E) + nd;
        }
        if ((uint32_t)E < nd) {  // ddd.ddd
            if (W) {
                uint64_t v = d.s;
                for (uint32_t i = nd; i-- > 0;) {
                    o[i < (uint32_t)E ? i : i + 1] = (uint8_t)('0' + v % 10);
                    v /= 10;
                }
                o[E] = '.';
            }
            return neg + nd + 1;
        }
        if (W) {  // ddd000
            fmt_put_digits(d.s, nd, o);
            for (uint32_t i = nd; i < (uint32_t)E; i++) o[i] = '0';
        }
        return neg + (uint32_t)E;
    }
    const int32_t x = E - 1;
    const uint32_t ax = (uint32_t)(x < 0 ? -x : x);
    const uint32_t nx = ax >= 100 ? 3 : ax >= 10 ? 2 : 1;
    const uint32_t m = nd + (nd > 1);  // d or d.ddd
    if (W) {
        uint64_t v = d.s;
        for (uint32_t i = nd; i-- > 0;) {
            o[i == 0 ? 0 : i + 1] = (uint8_t)('0' + v % 10);
            v /= 10;
        }
        if (nd > 1) o[1] = '.';
        o[m] = 'e';
        o[m + 1] = x < 0 ? '-' : '+';
        fmt_put_digits(ax, nx, o + m + 2);
    }
    return neg + m + 2 + nx;
}

// escapeBytes for one byte: the escaped length, and (W) the escape itself
SJ_HD uint32_t fmt_escaped_len(uint8_t c) {
    if (c >= 0x20) return (c == '"' || c == '\\') ? 2 : 1;
    return (c == '\b' || c == '\f' || c == '\n' || c == '\r' || c == '\t') ? 2 : 6;
}
SJ_HD uint32_t fmt_escape(uint8_t c, uint8_t* o) {
    const uint32_t n = fmt_escaped_len(c);
    if (n == 1) {
        o[0] = c;
        return 1;
    }
    o[0] = '\\';
    if (n == 2) {
        o[1] = c == '\b' ? 'b' : c == '\f' ? 'f' : c == '\n' ? 'n' : c == '\r' ? 'r' : c == '\t' ? 't' : c;
        return 2;
    }
    o[1] = 'u';
    o[2] = '0';
    o[3] = '0';
    o[4] = (uint8_t)("0123456789abcdef"[c >> 4]);
    o[5] = (uint8_t)("0123456789abcdef"[c & 15]);
    return 6;
}

}  // namespace sj
