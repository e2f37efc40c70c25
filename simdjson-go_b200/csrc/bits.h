// bits.h -- the bit and byte primitives that stage 1 (stage1.cuh), the per-structural stage 2 (stage2.cuh) and the
// streaming stage 2 (s2s_core.h, s2s_slab.h) share: portable intrinsics, the bit-plane transpose, prefix XOR, and the
// per-byte tables of the string and atom parsers.
//
// Portable C++ like s2s_core.h: under nvcc the functions are __host__ __device__, and tests/emu/s2s_emu.cpp compiles
// them with g++, so the code K1 runs is the code the emulation checks against the oracle.
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#if defined(__CUDACC__)
#define SJ_HD __host__ __device__ __forceinline__
#define SJ_HDC __host__ __device__ constexpr
#else
#define SJ_HD inline
#define SJ_HDC constexpr
#endif

namespace sj {

// the tape word of a string in Strings.B has it set (not one in the message): stage 2 writes it, tape.cuh reads it
constexpr uint64_t STRINGBUFBIT = 0x80000000000000ull;  // parsed_json.go:29

// ---------------------------------------------------------------------------------
// portable "intrinsics"
// ---------------------------------------------------------------------------------
namespace pi {
SJ_HD uint32_t popc32(uint32_t x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}
SJ_HD uint32_t popc64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popcll(x);
#else
    return (uint32_t)__builtin_popcountll(x);
#endif
}
SJ_HD uint32_t clz32(uint32_t x) {  // 32 for 0
#ifdef __CUDA_ARCH__
    return (uint32_t)__clz((int)x);
#else
    return x ? (uint32_t)__builtin_clz(x) : 32u;
#endif
}
SJ_HD uint32_t clz64(uint64_t x) {  // 64 for 0
#ifdef __CUDA_ARCH__
    return (uint32_t)__clzll((long long)x);
#else
    return x ? (uint32_t)__builtin_clzll(x) : 64u;
#endif
}
SJ_HD uint64_t umulhi64(uint64_t a, uint64_t b) {  // the upper 64 bits of a * b
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
SJ_HD double ddiv_rn(double a, double b) {  // a / b and a * b, rounded to nearest even (no FMA contraction)
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
SJ_HD double dmul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
SJ_HD uint64_t double_bits(double d) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t r;
    memcpy(&r, &d, 8);
    return r;
#endif
}
SJ_HD uint32_t ctz64(uint64_t x) {  // undefined for 0
#ifdef __CUDA_ARCH__
    return (uint32_t)__ffsll((long long)x) - 1u;
#else
    return (uint32_t)__builtin_ctzll(x);
#endif
}
SJ_HD uint32_t ctz32(uint32_t x) {  // undefined for 0
#ifdef __CUDA_ARCH__
    return (uint32_t)__ffs((int)x) - 1u;
#else
    return (uint32_t)__builtin_ctz(x);
#endif
}
SJ_HD uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t sel) {  // selectors 0..7 only
#ifdef __CUDA_ARCH__
    return __byte_perm(a, b, sel);
#else
    const uint64_t pool = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((pool >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
#endif
}
SJ_HD uint32_t shr_hi(uint32_t y, int s) {  // y >> s for 1 <= s <= 31, on the FMA pipe (IMAD.HI) on the device
#ifdef __CUDA_ARCH__
    return __umulhi(y, 1u << (32 - s));
#else
    return y >> s;
#endif
}
// (a & m) | (b & ~m) as ONE LOP3 (the compiler emits an AND and an OR-AND for the C expression because m and ~m are
// different immediates)
SJ_HD uint32_t bitsel(uint32_t m, uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, 0xE4;" : "=r"(d) : "r"(a), "r"(b), "r"(m));
    return d;
#else
    return (a & m) | (b & ~m);
#endif
}
SJ_HD uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t s) {  // lower word of (hi:lo) >> (s & 31)
#ifdef __CUDA_ARCH__
    return __funnelshift_r(lo, hi, s);
#else
    s &= 31;
    return s ? (lo >> s) | (hi << (32 - s)) : lo;
#endif
}
SJ_HD uint32_t funnel_l(uint32_t lo, uint32_t hi, uint32_t s) {  // upper word of (hi:lo) << (s & 31)
#ifdef __CUDA_ARCH__
    return __funnelshift_l(lo, hi, s);
#else
    s &= 31;
    return s ? (hi << s) | (lo >> (32 - s)) : hi;
#endif
}
}  // namespace pi

SJ_HD uint64_t mk64(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// ---------------------------------------------------------------------------------
// bit planes (find_whitespace_and_structurals_amd64.s:6-29 classifies bytes with VPSHUFB look-ups; here the 32 bytes
// are transposed into their 8 bit planes -- a 4x4 byte transpose with PRMT, then three mask/shift merge stages, the
// classic "s2p" of parallel bit streams -- and every class is a Boolean function of the planes)
// ---------------------------------------------------------------------------------
// rows a,b,c,d (4 bytes each) -> r_t = {a.b_t, b.b_t, c.b_t, d.b_t}
SJ_HD void transpose4x4(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    const uint32_t t0 = pi::byte_perm(a, b, 0x5140), t1 = pi::byte_perm(a, b, 0x7362);
    const uint32_t t2 = pi::byte_perm(c, d, 0x5140), t3 = pi::byte_perm(c, d, 0x7362);
    r0 = pi::byte_perm(t0, t2, 0x5410);
    r1 = pi::byte_perm(t0, t2, 0x7632);
    r2 = pi::byte_perm(t1, t3, 0x5410);
    r3 = pi::byte_perm(t1, t3, 0x7632);
}
// one merge step: hi keeps the m-bits of X in place and moves the m-bits of Y down by s;
// lo moves the ~m-bits of X up by s and keeps the ~m-bits of Y     (m >> s == ~m)
// Y >> s runs on the FMA pipe (pi::shr_hi): the classifiers are bound by the ALU pipe (LOP3 / SHF / PRMT issue every
// other cycle), the FMA pipe is nearly idle
SJ_HD void s2p_pair(uint32_t X, uint32_t Y, uint32_t m, int s, uint32_t& hi, uint32_t& lo) {
    hi = pi::bitsel(m, X, pi::shr_hi(Y, s));
    lo = pi::bitsel(m, X << s, Y);
}
// w[0..7]: 32 bytes (word k = bytes 4k..4k+3); pl[k] bit i = bit k of byte i
SJ_HD void bit_planes32(const uint32_t* w, uint32_t (&pl)[8]) {
    uint32_t R[8];  // R[t] = bytes {t, 8+t, 16+t, 24+t}
    transpose4x4(w[0], w[2], w[4], w[6], R[0], R[1], R[2], R[3]);
    transpose4x4(w[1], w[3], w[5], w[7], R[4], R[5], R[6], R[7]);
    uint32_t h1[4], l1[4];
#pragma unroll
    for (int t = 0; t < 4; t++) s2p_pair(R[t + 4], R[t], 0xF0F0F0F0u, 4, h1[t], l1[t]);
    uint32_t hh[2], hl[2], lh[2], ll[2];
    s2p_pair(h1[2], h1[0], 0xCCCCCCCCu, 2, hh[0], hl[0]);
    s2p_pair(h1[3], h1[1], 0xCCCCCCCCu, 2, hh[1], hl[1]);
    s2p_pair(l1[2], l1[0], 0xCCCCCCCCu, 2, lh[0], ll[0]);
    s2p_pair(l1[3], l1[1], 0xCCCCCCCCu, 2, lh[1], ll[1]);
    s2p_pair(hh[1], hh[0], 0xAAAAAAAAu, 1, pl[7], pl[6]);
    s2p_pair(hl[1], hl[0], 0xAAAAAAAAu, 1, pl[5], pl[4]);
    s2p_pair(lh[1], lh[0], 0xAAAAAAAAu, 1, pl[3], pl[2]);
    s2p_pair(ll[1], ll[0], 0xAAAAAAAAu, 1, pl[1], pl[0]);
}

// find_quote_mask_and_bits_amd64.s:66: carry-less multiply by all-ones == prefix XOR
SJ_HD uint64_t prefix_xor64(uint64_t x) {
    uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
    lo ^= lo << 1;
    hi ^= hi << 1;
    lo ^= lo << 2;
    hi ^= hi << 2;
    lo ^= lo << 4;
    hi ^= hi << 4;
    lo ^= lo << 8;
    hi ^= hi << 8;
    lo ^= lo << 16;
    hi ^= hi << 16;
    hi ^= (uint32_t)((int32_t)lo >> 31);  // parity of the low half carries into the high half
    return mk64(lo, hi);
}

// ---------------------------------------------------------------------------------
// atoms and escapes
// ---------------------------------------------------------------------------------
// atoms (stage2_build_tape_amd64.go:124-158, 455-476): the byte behind a literal must be structural / white / NUL
SJ_HD bool structural_or_ws_or_nul(uint32_t c) {
    return c == 0 || c == '\t' || c == '\n' || c == '\r' || c == ' ' || c == ',' || c == ':' || c == '[' || c == ']' ||
           c == '{' || c == '}';
}

// parse_string_amd64.s:4-69 digittoval: bytes below '0' map to 0 (no DATA line), hex digits to their value, everything
// else to -1
SJ_HD int32_t digit_to_val(uint32_t c) {
    if (c < 0x30) return 0;
    if (c <= '9') return (int32_t)c - '0';
    const uint32_t l = c | 0x20;
    if (c < 0x80 && l >= 'a' && l <= 'f' && c >= 'A') return (int32_t)l - 'a' + 10;
    return -1;
}
// parse_string_amd64.s:4-69 escape_map (+0x140): the byte a "\x" escape stands for, 0 = invalid ('u' is handled apart)
SJ_HD uint32_t escape_map(uint32_t e) {
    switch (e) {
    case '"': return 0x22;
    case '/': return 0x2f;
    case '\\': return 0x5c;
    case 'b': return 0x08;
    case 'f': return 0x0c;
    case 'n': return 0x0a;
    case 'r': return 0x0d;
    case 't': return 0x09;
    default: return 0;
    }
}

// the n (1..4) UTF-8 bytes of code point cp, first one in bits 0..7
SJ_HD uint32_t utf8_pack(uint32_t cp, uint32_t n) {
    if (n == 1) return cp;
    if (n == 2) return (0xC0u + (cp >> 6)) | ((0x80u | (cp & 63)) << 8);
    if (n == 3) return (0xE0u + (cp >> 12)) | ((0x80u | ((cp >> 6) & 63)) << 8) | ((0x80u | (cp & 63)) << 16);
    return (0xF0u + (cp >> 18)) | ((0x80u | ((cp >> 12) & 63)) << 8) | ((0x80u | ((cp >> 6) & 63)) << 16) | ((0x80u | (cp & 63)) << 24);
}

}  // namespace sj
