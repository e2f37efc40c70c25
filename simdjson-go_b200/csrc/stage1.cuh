// stage1.cuh -- K1 `stage1_flatten`: structural-index discovery + flatten_bits as ONE
// sm_90a kernel (the reference also fuses them: find_structural_bits_amd64.s:56-115).
//
// Replaces, per 64-byte block (SURVEY.md 3.4):
//   find_odd_backslash_sequences     find_odd_backslash_sequences_amd64.s:24-61
//   find_quote_mask_and_bits         find_quote_mask_and_bits_amd64.s:49-84   (CLMUL -> shift/xor prefix + warp ballot parity)
//   find_whitespace_and_structurals  find_whitespace_and_structurals_amd64.s:62-103 (VPSHUFB LUTs -> bit planes)
//   finalize_structurals             finalize_structurals_amd64.s:19-36
//   find_newline_delimiters          find_newline_delimiters_amd64.s:16-28    (NDJSON)
//   flatten_bits_incremental         flatten_bits_amd64.s:26-60               (serial tzcnt -> popcount + warp scan compaction)
// and the driver loop of stage1_find_marks_amd64.go:41-148.
//
// Shape: persistent cooperative grid (1 CTA per SM).  A CTA is S1_WARPS worker warps plus one
// scan warp and works on one 96 KiB TILE at a time (tiles are dealt round-robin to the CTAs);
// the tile is staged HBM -> shared memory by one 1-D TMA bulk copy into a double buffer (the
// next tile streams in while the current one is processed).  Each worker warp owns one 6 KiB
// slab of the tile; lane L owns the 64-byte block L of each of the slab's 2 KiB steps and reads
// it with four conflict-free 16-byte LDS.  Carries across blocks use ballots inside a warp;
// carries across slabs go through shared memory; carries across tiles use two decoupled
// look-back chains (in-string parity, then structural count) that the scan warp runs while the
// workers classify / flatten, so a look-back never stalls them; the odd-backslash and
// pseudo-predecessor carries are recovered from the 32 bytes in front of the slab (prefetched
// one tile ahead).  The 64-byte masks come from a bit-sliced classifier (byte transpose + bit
// planes + Boolean class functions) instead of per-byte compares.
#pragma once
#include "bits.h"
#include "common.cuh"
#include "s2s_slab.h"

namespace sj {

constexpr int S1_WARPS = 16;                     // warps per CTA = slabs per tile
// Pause between two polls of a look-back (ns); the first poll is not preceded by one.  With one descriptor slot per
// L2 line the chains are insensitive to it; with the descriptors of 128 tiles packed in one line a poll issued while
// the other CTAs published cost microseconds.
constexpr unsigned S1_SPIN_SLEEP_NS = 100;
constexpr int S1_CTAS_PER_SM = 1;
constexpr int S1_THREADS = (S1_WARPS + 1) * 32;  // worker warps + one scan warp (the look-backs)
constexpr int S1_STEPS = (int)S2S_STEPS;         // 2 KiB steps per slab (the streaming stage 2 walks the same slabs)
constexpr int S1_STEP_BYTES = 32 * 64;
constexpr int S1_SLAB_BYTES = S1_STEPS * S1_STEP_BYTES;  // 6 KiB per warp
constexpr int S1_TILE_BYTES = S1_WARPS * S1_SLAB_BYTES;  // one look-back per tile
constexpr int S1_BUFS = 2;
constexpr size_t S1_SMEM_BYTES = (size_t)S1_BUFS * S1_TILE_BYTES + 64;  // tiles + mbarriers

// K1's parse-mode section probe (tools/k1_probe.py builds it; the product build does not define SJ_K1_PROBE): a
// clock64() stamp at each section boundary of a worker iteration, each warp's sums added into sj_k1_probe_cycles when it
// leaves the loop.  The stamps cost time themselves, so the sums are for shares, not for K1's time.
enum : uint32_t {
    K1P_CARRIES,     // carries from the bytes in front of the slab
    K1P_TMA,         // wait for the tile's bytes
    K1P_CLASSIFY,    // phase A: load + classify every block
    K1P_PASS2,       // pass 2: escapes, quote parity
    K1P_WAIT,        // output offsets and in-string state from the scan warp (bar_S, bar_Q)
    K1P_B_CLASSIFY,  // phase B: the classes step_events reads
    K1P_B_ESCAPES,   // phase B: escapes inside strings -> dropped bytes
    K1P_EVENTS,      // step_events
    K1P_AGG,         // the slab's counts
    K1P_STORE,       // the SlabAgg store, slab count and last structural, bar_R
    K1P_SECTIONS
};
#if defined(SJ_K1_PROBE) && defined(__CUDACC__)
__device__ unsigned long long sj_k1_probe_cycles[K1P_SECTIONS];
#endif
#if defined(SJ_K1_PROBE) && defined(__CUDA_ARCH__)
// (lane k keeps the sum of section k; parse mode only)
#define K1_PROBE_START        \
    uint32_t probe_acc = 0;   \
    long long probe_t = clock64();
#define K1_PROBE(sec)                                              \
    do {                                                           \
        if (PARSE) {                                               \
            __syncwarp();                                          \
            const long long t_ = clock64();                        \
            if (lane == (sec)) probe_acc += (uint32_t)(t_ - probe_t); \
            probe_t = t_;                                          \
        }                                                          \
    } while (0)
#define K1_PROBE_FLUSH                                                                             \
    do {                                                                                           \
        if (PARSE && lane < K1P_SECTIONS) atomicAdd(&sj_k1_probe_cycles[lane], (unsigned long long)probe_acc); \
    } while (0)
#else
#define K1_PROBE_START
#define K1_PROBE(sec) \
    do {              \
    } while (0)
#define K1_PROBE_FLUSH \
    do {               \
    } while (0)
#endif

struct Stage1Result {
    uint32_t n_idx;           // total structurals found
    uint32_t error;           // != 0: control character (< 0x20) inside a string
    uint32_t ends_in_string;  // message ends inside an unterminated string
    uint32_t last_pos;        // position of the last structural (valid if n_idx > 0)
    uint32_t overflow;        // index buffer too small (n_idx is still exact)
    uint32_t last_char;       // message byte at last_pos (stage1_find_marks_amd64.go:140-146 tests it for '}' / ']')
    uint32_t pad[2];
};

// ---------------------------------------------------------------------------------
// byte classification: SWAR on 32-bit words, flags land in bit 7 of each byte
// ---------------------------------------------------------------------------------
struct WordFlags {
    uint32_t bs, qt, st, sp;
};

__device__ __forceinline__ WordFlags classify_word(uint32_t v, uint32_t& ctacc) {
    const uint32_t L7 = 0x7f7f7f7fu, H = 0x80808080u;
    uint32_t v7 = v & L7;
    // (x ^ C) + 0x7f: bit 7 set iff (byte & 0x7f) != C.  Bytes >= 0x80 are removed by "| v".
    uint32_t tbs = (v7 ^ 0x5c5c5c5cu) + L7;
    uint32_t tqt = (v7 ^ 0x22222222u) + L7;
    uint32_t tcm = (v7 ^ 0x2c2c2c2cu) + L7;
    uint32_t tcl = (v7 ^ 0x3a3a3a3au) + L7;
    uint32_t tsp = (v7 ^ 0x20202020u) + L7;
    // { } [ ] in one test: (b + 1) & 0xDD == 0x5C  <=>  b in {5b,5d,7b,7d}
    uint32_t tbr = (((v7 + 0x01010101u) & 0x5d5d5d5du) ^ 0x5c5c5c5cu) + L7;
    uint32_t tct = v7 + 0x60606060u;  // bit 7 set iff (byte & 0x7f) >= 0x20
    WordFlags f;
    f.bs = ~(tbs | v) & H;
    f.qt = ~(tqt | v) & H;
    f.st = ~((tbr & tcm & tcl) | v) & H;
    f.sp = ~(tsp | v) & H;
    ctacc |= ~(tct | v);
    return f;
}

struct WordFlagsSlow {
    uint32_t ct, wsc, nl;
};

__device__ __forceinline__ WordFlagsSlow classify_word_slow(uint32_t v) {
    const uint32_t L7 = 0x7f7f7f7fu, H = 0x80808080u;
    uint32_t v7 = v & L7;
    uint32_t tct = v7 + 0x60606060u;
    uint32_t ge9 = v7 + 0x77777777u;  // >= 0x09
    uint32_t geb = v7 + 0x75757575u;  // >= 0x0b
    uint32_t tcr = (v7 ^ 0x0d0d0d0du) + L7;
    uint32_t tnl = (v7 ^ 0x0a0a0a0au) + L7;
    WordFlagsSlow f;
    f.ct = ~(tct | v) & H;
    f.wsc = ((ge9 & ~geb) | ~tcr) & ~v & H;
    f.nl = ~(tnl | v) & H;
    return f;
}

// gather the four bit-7 flags of a word into the next nibble of an accumulator
// (words are fed most-significant first): acc = acc << 4 | flags
__device__ __forceinline__ uint32_t gather4(uint32_t flags, uint32_t acc) {
    return __funnelshift_l(flags * 0x00204081u, acc, 4);
}

// rotate a 64-bit mask left by 16*r bits (r = 0..3): undoes the bank-conflict-free
// chunk rotation used when a lane reads its 64 bytes from shared memory.  Two PRMTs: the four
// 16-bit pieces of (lo, hi) are re-ordered by per-lane selectors (rot_selectors) computed once per thread.
struct RotSel {
    uint32_t lo, hi;
};
__device__ __forceinline__ RotSel rot_selectors(uint32_t r) {
    // result piece k = source piece (k - r) & 3 ; piece q = bytes 2q, 2q+1 of the 8-byte pool {lo, hi}
    auto two = [](uint32_t q0, uint32_t q1) { return (2 * q0) | ((2 * q0 + 1) << 4) | ((2 * q1) << 8) | ((2 * q1 + 1) << 12); };
    RotSel s;
    s.lo = two((0 - r) & 3, (1 - r) & 3);
    s.hi = two((2 - r) & 3, (3 - r) & 3);
    return s;
}
__device__ __forceinline__ uint64_t rotl16x(uint32_t lo, uint32_t hi, const RotSel& s) {
    return mk64(__byte_perm(lo, hi, s.lo), __byte_perm(lo, hi, s.hi));
}

struct BlockMasks {
    uint64_t bs, qt, st, sp;
    uint32_t anyct;
};

// w[16]: the block's 16 words in slot order
__device__ __forceinline__ BlockMasks classify_block(const uint32_t (&w)[16]) {
    uint32_t bs_lo = 0, bs_hi = 0, qt_lo = 0, qt_hi = 0, st_lo = 0, st_hi = 0, sp_lo = 0, sp_hi = 0, ct = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) {
        WordFlags f = classify_word(w[k], ct);
        bs_lo = gather4(f.bs, bs_lo);
        qt_lo = gather4(f.qt, qt_lo);
        st_lo = gather4(f.st, st_lo);
        sp_lo = gather4(f.sp, sp_lo);
    }
#pragma unroll
    for (int k = 15; k >= 8; k--) {
        WordFlags f = classify_word(w[k], ct);
        bs_hi = gather4(f.bs, bs_hi);
        qt_hi = gather4(f.qt, qt_hi);
        st_hi = gather4(f.st, st_hi);
        sp_hi = gather4(f.sp, sp_hi);
    }
    BlockMasks m;
    m.bs = mk64(bs_lo, bs_hi);
    m.qt = mk64(qt_lo, qt_hi);
    m.st = mk64(st_lo, st_hi);
    m.sp = mk64(sp_lo, sp_hi);
    m.anyct = ct & 0x80808080u;
    return m;
}

struct SlowMasks {
    uint64_t ct, wsc, nl;
};

__device__ __forceinline__ SlowMasks classify_block_slow(const uint32_t (&w)[16]) {
    uint32_t a_lo = 0, a_hi = 0, b_lo = 0, b_hi = 0, c_lo = 0, c_hi = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) {
        WordFlagsSlow f = classify_word_slow(w[k]);
        a_lo = gather4(f.ct, a_lo);
        b_lo = gather4(f.wsc, b_lo);
        c_lo = gather4(f.nl, c_lo);
    }
#pragma unroll
    for (int k = 15; k >= 8; k--) {
        WordFlagsSlow f = classify_word_slow(w[k]);
        a_hi = gather4(f.ct, a_hi);
        b_hi = gather4(f.wsc, b_hi);
        c_hi = gather4(f.nl, c_hi);
    }
    SlowMasks m;
    m.ct = mk64(a_lo, a_hi);
    m.wsc = mk64(b_lo, b_hi);
    m.nl = mk64(c_lo, c_hi);
    return m;
}

// ---------------------------------------------------------------------------------
// Bit-sliced classification (default).  The 64 bytes of a block are transposed into their 8
// bit planes (bit_planes32 of bits.h, the same code the streaming stage 2 runs: a 4x4 byte
// transpose with PRMT, then three mask/shift merge stages -- the classic "s2p" of parallel
// bit streams), after which every class is a Boolean function of the planes evaluated for
// 32 bytes per LOP3: no per-class compares, no flag gathering, and tab / LF / CR / control
// masks come for free.  K1's class set differs from the streaming pass's (classify_planes2),
// so the Boolean functions stay apart; the parse mode takes the two planes it needs on top of
// them (parse_planes) from classify_planes2 on the same transpose.  About 230 instructions per 64-byte block for
// all six masks, against 464 (4 masks) to 750 (with the control-character pass) for the
// word-wise SWAR compares above; those stay as an independent second implementation that the
// test hook sj_test_block_masks cross-checks against this one on every block.
// ---------------------------------------------------------------------------------
struct PlaneMasks {
    uint64_t bs, qt, st, ws, ct, nl;
    uint64_t px, py;  // parse mode: X / Y of parse_planes (s2s_core.h)
};

struct HalfMasks {
    uint32_t bs, qt, st, ws, ct, nl;
};

// character classes of find_whitespace_and_structurals_amd64.s:6-29 / find_quote_mask_and_bits /
// find_odd_backslash_sequences / find_newline_delimiters as Boolean functions of the bit planes
__device__ __forceinline__ HalfMasks classify_planes(const uint32_t (&p)[8]) {
    const uint32_t A = ~p[7] & ~p[6];           // 0x00..0x3f
    const uint32_t hi2 = A & p[5] & ~p[4];      // 0x2_
    const uint32_t hi3 = A & p[5] & p[4];       // 0x3_
    const uint32_t hi01 = A & ~p[5];            // 0x00..0x1f  (control characters)
    const uint32_t hi0 = hi01 & ~p[4];          // 0x0_
    const uint32_t hi57 = ~p[7] & p[6] & p[4];  // 0x5_ or 0x7_
    const uint32_t hi5 = hi57 & ~p[5];
    const uint32_t c32 = p[3] & p[2], c30 = p[3] & ~p[2], z32 = ~p[3] & ~p[2];
    const uint32_t loC = c32 & ~p[1] & ~p[0], loD = c32 & ~p[1] & p[0];
    const uint32_t loA = c30 & p[1] & ~p[0], loB = c30 & p[1] & p[0], lo9 = c30 & ~p[1] & p[0];
    const uint32_t lo2 = z32 & p[1] & ~p[0], lo0 = z32 & ~p[1] & ~p[0];
    HalfMasks m;
    m.qt = hi2 & lo2;                                              // "
    m.bs = hi5 & loC;                                              // backslash
    m.st = (hi2 & loC) | (hi3 & loA) | (hi57 & (loB | loD));       // , : [ ] { }
    m.ws = (hi2 & lo0) | (hi0 & (lo9 | loA | loD));                // space \t \n \r
    m.ct = hi01;                                                   // < 0x20
    m.nl = hi0 & loA;                                              // \n
    return m;
}

// w[16]: the block's 16 words (any fixed order; masks come out in the same order)
__device__ __forceinline__ PlaneMasks classify_block_planes(const uint32_t (&w)[16]) {
    uint32_t p0[8], p1[8];
    bit_planes32(&w[0], p0);
    bit_planes32(&w[8], p1);
    HalfMasks a = classify_planes(p0), b = classify_planes(p1);
    const ParsePlanes pa = parse_planes(p0), pb = parse_planes(p1);
    PlaneMasks m;
    m.px = mk64(pa.x, pb.x);
    m.py = mk64(pa.y, pb.y);
    m.bs = mk64(a.bs, b.bs);
    m.qt = mk64(a.qt, b.qt);
    m.st = mk64(a.st, b.st);
    m.ws = mk64(a.ws, b.ws);
    m.ct = mk64(a.ct, b.ct);
    m.nl = mk64(a.nl, b.nl);
    return m;
}

// ---------------------------------------------------------------------------------
// 64-bit mask algebra (same formulas as the reference's scalar tail of each routine)
// ---------------------------------------------------------------------------------
// find_odd_backslash_sequences_amd64.s:27-58 ; prev in {0,1}
__device__ __forceinline__ uint64_t odd_backslash_ends(uint64_t bs, uint32_t prev, uint32_t* carry_out) {
    const uint64_t even_bits = 0x5555555555555555ull, odd_bits = 0xAAAAAAAAAAAAAAAAull;
    uint64_t p = prev;
    uint64_t starts = bs & ~(bs << 1);
    uint64_t even_starts = starts & (even_bits ^ p);
    uint64_t odd_starts = starts & (odd_bits ^ p);
    uint64_t even_carries = bs + even_starts;
    uint64_t odd_carries = bs + odd_starts;
    if (carry_out) *carry_out = odd_carries < bs;
    odd_carries |= p;
    return (even_carries & ~bs & odd_bits) | (odd_carries & ~bs & even_bits);
}

// finalize_structurals_amd64.s:19-36 ; pp_in in {0,1}; *pp_out = pseudo_pred >> 63
__device__ __forceinline__ uint64_t finalize_structurals(uint64_t st, uint64_t ws, uint64_t qm, uint64_t qb,
                                                         uint32_t pp_in, uint32_t* pp_out) {
    uint64_t s = (st & ~qm) | qb;
    uint64_t pred = s | ws;
    uint64_t shifted = (pred << 1) | pp_in;
    *pp_out = (uint32_t)(pred >> 63);
    uint64_t pseudo = shifted & ~ws & ~qm;
    s |= pseudo;
    s &= ~(qb & ~qm);
    return s;
}

// ---------------------------------------------------------------------------------
// flatten: one warp emits the structurals of one 2 KiB step (lane L holds the 64-bit
// mask of block L).  Positions are written in order at out[base + ...]; in delta mode
// each entry is the distance from the previous structural (reference format,
// flatten_bits_amd64.s:26-60: first delta of the message = position + 1).
// `prev_last` is the position of the last structural before this step (0xffffffff = none).
// Returns the number of structurals in the step; updates prev_last.
// ---------------------------------------------------------------------------------
// `stage` (optional): stage_cap x uint32 of shared memory private to the warp; the lanes drop their
// entries there and the warp then streams them out with fully coalesced 128-byte stores.
constexpr int S1_FLATTEN_UNROLL = 2;  // positions per half and trip of the extraction loops
// index of the highest set bit (0xffffffff for 0): one FLO
__device__ __forceinline__ uint32_t bfind(uint32_t x) {
    uint32_t b;
    asm("bfind.u32 %0, %1;" : "=r"(b) : "r"(x));
    return b;
}
// st.shared.u32 [addr], val  predicated on cond != 0
__device__ __forceinline__ void sts_if(uint32_t addr, uint32_t val, uint32_t cond) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p st.shared.u32 [%0], %1;\n\t}" ::"r"(addr), "r"(val), "r"(cond)
        : "memory");
}

template <bool DELTAS>
__device__ __forceinline__ uint32_t flatten_step(uint64_t S, uint32_t blockpos, uint32_t* __restrict__ out,
                                                 uint64_t base, uint64_t cap, uint32_t& prev_last, uint32_t& overflow,
                                                 uint32_t* stage = nullptr, uint32_t stage_cap = 0) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t lo = (uint32_t)S, hi = (uint32_t)(S >> 32);
    uint32_t c = __popc(lo) + __popc(hi);
    // warp inclusive scan of counts
    uint32_t inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(FULL, inc, d);
        if (lane >= d) inc += t;
    }
    uint32_t total = __shfl_sync(FULL, inc, 31);
    uint64_t off = base + (inc - c);
    // last structural of this lane and of the nearest non-empty lane below
    uint32_t own_last = blockpos + (hi ? 63 - __clz(hi) : 31 - __clz(lo | 1));
    uint32_t ne = __ballot_sync(FULL, c != 0);
    uint32_t below = ne & lanemask_lt();
    uint32_t src = below ? 31 - __clz(below) : 0;
    uint32_t got = __shfl_sync(FULL, own_last, src);
    uint32_t prev = below ? got : prev_last;
    uint32_t top = ne ? 31 - __clz(ne) : 0;
    uint32_t newlast = __shfl_sync(FULL, own_last, top);
    if (ne) prev_last = newlast;
    if (base + total > cap) {  // warp-uniform
        overflow = 1;
        return total;
    }
    uint32_t pos0 = blockpos;
    if (stage && total <= stage_cap) {  // warp-uniform
        // the two 32-bit halves are extracted side by side (two independent dependency chains,
        // half the trip count of the divergent loop); bit-reversed so that one FLO finds the
        // next position
        uint32_t alo = (uint32_t)__cvta_generic_to_shared(stage + (inc - c));
        uint32_t ahi = alo + 4 * __popc(lo);
        uint32_t prev_hi = lo ? pos0 + 31 - __clz(lo) : prev;
        const uint32_t pos1 = pos0 + 32;
        // branch-free body: an exhausted half keeps running on a zero mask with its store
        // predicated off (inline PTX: the compiler would branch around the four instructions)
        // (an exhausted half never uses its cursor again, so the cursors advance unconditionally)
        while (lo | hi) {
#pragma unroll
            for (int u = 0; u < S1_FLATTEN_UNROLL; u++) {
                {
                    const uint32_t p = pos0 + (__ffs(lo) - 1);
                    sts_if(alo + 4 * u, DELTAS ? p - prev : p, lo);
                    prev = p;
                    lo &= lo - 1;
                }
                {
                    const uint32_t p = pos1 + (__ffs(hi) - 1);
                    sts_if(ahi + 4 * u, DELTAS ? p - prev_hi : p, hi);
                    prev_hi = p;
                    hi &= hi - 1;
                }
            }
            alo += 4 * S1_FLATTEN_UNROLL;
            ahi += 4 * S1_FLATTEN_UNROLL;
        }
        __syncwarp();
        for (uint32_t k = lane; k < total; k += 32) out[base + k] = stage[k];
        __syncwarp();
        return total;
    }
    while (lo) {
        uint32_t b = __ffs(lo) - 1;
        lo &= lo - 1;
        uint32_t p = pos0 + b;
        out[off++] = DELTAS ? p - prev : p;
        prev = p;
    }
    pos0 += 32;
    while (hi) {
        uint32_t b = __ffs(hi) - 1;
        hi &= hi - 1;
        uint32_t p = pos0 + b;
        out[off++] = DELTAS ? p - prev : p;
        prev = p;
    }
    return total;
}

// Positions of the structurals of one 2 KiB step, staged into `chunk` (room for `cap` entries).  Extraction runs from the top bit down (one FLO per
// structural, no bit reversal) as two independent chains (the two 32-bit halves of the lane's
// mask) with predicated stores.  Returns the step's count (warp-uniform); nothing is staged if it
// exceeds `cap` (more than one structural per 4 bytes).
__device__ __forceinline__ uint32_t extract_step(uint64_t S, uint32_t pos0, uint32_t* chunk, uint32_t cap) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t lo = (uint32_t)S, hi = (uint32_t)(S >> 32);
    const uint32_t ch = __popc(hi);
    const uint32_t c = __popc(lo) + ch;
    uint32_t inc = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(FULL, inc, d);
        if (lane >= d) inc += t;
    }
    const uint32_t total = __shfl_sync(FULL, inc, 31);
    if (total > cap) return total;
    // cursors on the LAST slot of each half
    uint32_t ahi = (uint32_t)__cvta_generic_to_shared(chunk) + 4 * inc - 4;
    uint32_t alo = ahi - 4 * ch;
    const uint32_t pos1 = pos0 + 32;
    while (lo | hi) {
#pragma unroll
        for (int u = 0; u < S1_FLATTEN_UNROLL; u++) {
            {
                const uint32_t b = bfind(lo);
                sts_if(alo - 4 * u, pos0 + b, lo);
                lo &= ~(1u << (b & 31));
            }
            {
                const uint32_t b = bfind(hi);
                sts_if(ahi - 4 * u, pos1 + b, hi);
                hi &= ~(1u << (b & 31));
            }
        }
        alo -= 4 * S1_FLATTEN_UNROLL;
        ahi -= 4 * S1_FLATTEN_UNROLL;
    }
    return total;
}

// Coalesced copy-out of one staged step; deltas (flatten_bits_amd64.s:38-40) are formed here from
// neighbouring staged positions, so the divergent extraction loop carries no delta arithmetic.
template <bool DELTAS>
__device__ __forceinline__ void copy_out(const uint32_t* stage, uint32_t n, uint32_t* __restrict__ dst, uint32_t prev_last) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t k = lane;
    for (; k + 96 < n; k += 128) {  // four coalesced 128-byte rows per trip
        uint32_t v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            v[u] = stage[k + 32 * u];
            if (DELTAS) v[u] -= (k + 32 * u) ? stage[k + 32 * u - 1] : prev_last;
        }
#pragma unroll
        for (int u = 0; u < 4; u++) dst[k + 32 * u] = v[u];
    }
    for (; k < n; k += 32) {
        uint32_t v = stage[k];
        if (DELTAS) v -= k ? stage[k - 1] : prev_last;
        dst[k] = v;
    }
}

// Flatten of a whole slab through the warp's staging area.  Positions are extracted from the top
// bit down (one FLO per structural, no bit reversal) by two independent chains (the two 32-bit
// halves of the lane's mask) with predicated stores; the copy-out is coalesced and forms the
// deltas (flatten_bits_amd64.s:38-40) from neighbouring staged positions, so the divergent
// extraction loop carries no delta arithmetic at all.
//   slabpos   = message offset of the slab,  dst = out + (output offset of the slab)
//   prev_last = position of the last structural in front of the slab (0xffffffff: none yet)
template <bool DELTAS, int STEPS>
__device__ __forceinline__ void flatten_slab_staged(const uint64_t (&S)[STEPS], uint32_t slabpos, uint32_t* __restrict__ dst,
                                                    uint32_t prev_last, uint32_t* stage, uint32_t stage_cap) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(stage);
    uint32_t so = 0;  // entries staged and not yet copied out (warp-uniform)
    // coalesced copy-out of the staged positions (as deltas if asked for)
    auto flush = [&]() {
        __syncwarp();
#pragma unroll 4
        for (uint32_t k = lane; k < so; k += 32) {
            uint32_t v = stage[k];
            if (DELTAS) v -= k ? stage[k - 1] : prev_last;
            dst[k] = v;
        }
        if (DELTAS && so) prev_last = stage[so - 1];
        dst += so;
        so = 0;
        __syncwarp();
    };
#pragma unroll
    for (int s = 0; s < STEPS; s++) {
        uint32_t lo = (uint32_t)S[s], hi = (uint32_t)(S[s] >> 32);
        const uint32_t ch = __popc(hi);
        const uint32_t c = __popc(lo) + ch;
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(FULL, inc, d);
            if (lane >= d) inc += t;
        }
        const uint32_t total = __shfl_sync(FULL, inc, 31);
        const uint32_t pos0 = slabpos + s * S1_STEP_BYTES + 64 * lane, pos1 = pos0 + 32;
        if (so + total > stage_cap) {  // warp-uniform; only inputs with > 1 structural per 4 bytes get here
            flush();
            if (total > stage_cap) {  // this step alone does not fit: straight to global memory
                uint32_t overflow = 0;
                flatten_step<DELTAS>(S[s], pos0, dst, 0, ~0ull, prev_last, overflow);
                dst += total;
                continue;
            }
        }
        // cursors on the LAST slot of each half
        uint32_t ahi = sbase + 4 * (so + inc) - 4;
        uint32_t alo = ahi - 4 * ch;
        while (lo | hi) {
#pragma unroll
            for (int u = 0; u < S1_FLATTEN_UNROLL; u++) {
                {
                    const uint32_t b = bfind(lo);
                    sts_if(alo - 4 * u, pos0 + b, lo);
                    lo &= ~(1u << (b & 31));
                }
                {
                    const uint32_t b = bfind(hi);
                    sts_if(ahi - 4 * u, pos1 + b, hi);
                    hi &= ~(1u << (b & 31));
                }
            }
            alo -= 4 * S1_FLATTEN_UNROLL;
            ahi -= 4 * S1_FLATTEN_UNROLL;
        }
        so += total;
    }
    flush();
}

// ---------------------------------------------------------------------------------
// look-back chains over TILES (all slabs of one CTA iteration; only the scan warp of a CTA
// publishes and polls).  Every tile owns one descriptor SLOT per chain, and the slots are
// S1_DESC_STRIDE bytes apart, i.e. in different L2 lines: with the descriptors of 128 tiles packed
// into one line (the previous layout) every CTA of the grid published into and polled the same line
// at the same moment, and a poll issued during that burst took microseconds.
//   chain 1 (in-string parity): uint32 {bit0 valid, bit1 inclusive, bit2 parity}
//   chain 2 (structural count): 16 bytes {uint32 aggregate | bit31 valid, pad, uint64 inclusive
//            prefix | bit63 valid}
// A lane inspects S1_LB_PER_LANE predecessors per round (distance lane + 32 j), all loads in
// flight at once; with a grid of at most 32 * S1_LB_PER_LANE CTAs the tile this CTA published
// one iteration ago (always inclusive) is inside the first round.
// ---------------------------------------------------------------------------------
constexpr int S1_DESC_STRIDE = 128;
constexpr int S1_LB_PER_LANE = 5;
constexpr uint32_t DP_VALID = 1, DP_INCL = 2, DP_PAR = 4;
constexpr uint32_t DA_VALID = 0x80000000u;
constexpr uint64_t DI_VALID = 1ull << 63;

__device__ __forceinline__ uint4 ld_relaxed_v4(const void* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ uint32_t* par_slot(uint8_t* dpar, int tile) {
    return reinterpret_cast<uint32_t*>(dpar + (size_t)tile * S1_DESC_STRIDE);
}
__device__ __forceinline__ uint8_t* cnt_slot(uint8_t* dcnt, int tile) { return dcnt + (size_t)tile * S1_DESC_STRIDE; }

// quote parity of everything in front of `tile` (tile > 0)
__device__ __forceinline__ uint32_t lookback_parity(uint8_t* dpar, int tile) {
    const int lane = threadIdx.x & 31;
    uint32_t par = 0;
    for (int base = tile - 1;; base -= 32 * S1_LB_PER_LANE) {
        uint32_t d[S1_LB_PER_LANE];
        bool again = false;
        uint32_t ok;
        do {
            if (again) __nanosleep(S1_SPIN_SLEEP_NS);
            again = true;
            ok = 1;
#pragma unroll
            for (int j = 0; j < S1_LB_PER_LANE; j++) {
                const int t = base - lane - 32 * j;
                d[j] = t >= 0 ? ld_relaxed_u32(par_slot(dpar, t)) : (DP_VALID | DP_INCL);  // before the message: parity 0
                ok &= d[j];
            }
        } while (__any_sync(FULL, !(ok & DP_VALID)));
#pragma unroll
        for (int j = 0; j < S1_LB_PER_LANE; j++) {  // nearest predecessors first
            const uint32_t I = __ballot_sync(FULL, (d[j] & DP_INCL) != 0);
            const uint32_t P = __ballot_sync(FULL, (d[j] & DP_PAR) != 0);
            if (I == 0) {
                par ^= __popc(P) & 1;
            } else {  // the nearest inclusive descriptor: it and everything nearer
                const uint32_t f = __ffs(I) - 1;
                par ^= __popc(P & (0xffffffffu >> (31 - f))) & 1;
                return par;
            }
        }
    }
}

// number of structurals in all tiles in front of `tile` (tile > 0)
__device__ __forceinline__ uint64_t lookback_count(uint8_t* dcnt, int tile) {
    const int lane = threadIdx.x & 31;
    uint64_t total = 0;
    for (int base = tile - 1;; base -= 32 * S1_LB_PER_LANE) {
        uint32_t agg[S1_LB_PER_LANE];
        uint64_t inc[S1_LB_PER_LANE];
        bool again = false;
        uint32_t ok;
        do {
            if (again) __nanosleep(S1_SPIN_SLEEP_NS);
            again = true;
            ok = DA_VALID;
#pragma unroll
            for (int j = 0; j < S1_LB_PER_LANE; j++) {
                const int t = base - lane - 32 * j;
                if (t >= 0) {
                    const uint4 q = ld_relaxed_v4(cnt_slot(dcnt, t));
                    agg[j] = q.x;
                    inc[j] = ((uint64_t)q.w << 32) | q.z;
                } else {  // before the message: prefix 0
                    agg[j] = DA_VALID;
                    inc[j] = DI_VALID;
                }
                ok &= agg[j];
            }
        } while (__any_sync(FULL, !(ok & DA_VALID)));
#pragma unroll
        for (int j = 0; j < S1_LB_PER_LANE; j++) {  // nearest predecessors first
            const uint32_t I = __ballot_sync(FULL, (inc[j] & DI_VALID) != 0);
            const uint32_t f = I ? __ffs(I) - 1 : 32;  // nearest tile with an inclusive prefix
            uint32_t v = (uint32_t)lane < f ? (agg[j] & ~DA_VALID) : 0;
#pragma unroll
            for (int dd = 16; dd > 0; dd >>= 1) v += __shfl_xor_sync(FULL, v, dd);
            total += v;
            if (I) {
                const uint32_t lo = __shfl_sync(FULL, (uint32_t)inc[j], f), hi = __shfl_sync(FULL, (uint32_t)(inc[j] >> 32), f);
                return total + ((((uint64_t)hi << 32) | lo) & ~DI_VALID);
            }
        }
    }
}

// ---------------------------------------------------------------------------------
// carries recovered from the bytes in front of a slab: length of the run of backslashes
// that ends just before `end` (warp-cooperative, 32 bytes per round; one round in practice).
// Not backslash_run_before_p (s2s_slab.h): that one compiles to other bit-scan instructions.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t backslash_run_before(const uint8_t* __restrict__ msg, uint64_t end) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t run = 0;
    for (uint64_t off = 0;; off += 32) {
        uint64_t back = off + lane + 1;  // lane L looks at byte end-1-off-L
        uint32_t c = back <= end ? msg[end - back] : 0x20;
        uint32_t B = __ballot_sync(FULL, c == '\\');
        uint32_t n = B == FULL ? 32 : __ffs(~B) - 1;
        run += n;
        if (n < 32) return run;
    }
}

struct Stage1Params {
    const uint8_t* msg;  // 16-byte aligned, readable up to round_up(len, 16)
    uint64_t len;
    uint32_t* out;       // positions (or deltas)
    uint64_t out_cap;
    uint8_t* dpar;       // [ntiles * S1_DESC_STRIDE] zeroed: chain-1 descriptor slots
    uint8_t* dcnt;       // [ntiles * S1_DESC_STRIDE] zeroed: chain-2 descriptor slots
    uint32_t* lastp1;    // [ntiles] position + 1 of the tile's last structural (0 = none)
    uint32_t* bsmap;     // optional: bit k = 64-byte block k contains a backslash (lets stage 2 skip the string scan)
    uint32_t* slabpar;   // optional: [ntiles] bit w = "inside a string" in front of slab w of the tile (handed to the streaming stage 2)
    Stage1Result* result;
    int ntiles;
    // parse mode (the streaming stage 2 follows): no index; per slab the counts of stage 2 instead
    SlabAgg* agg;        // [slabs] what s2s_slab<W, false> adds up for the slab
    uint32_t* s2_error;  // an invalid escape (Stage2Result::error)
};

// message bytes for the escape decoder in parse mode: the slab's bytes from shared memory, others from global memory,
// 0 beyond the end of the message
struct SlabReader {
    const uint8_t* src;
    uint64_t start;
    uint32_t win;  // message bytes the image holds
    const uint8_t* msg;
    uint64_t len;
    __device__ __forceinline__ uint32_t operator()(uint64_t pos) const {
        const uint64_t d = pos - start;
        if (d < win) return src[d];
        return pos < len ? msg[pos] : 0u;
    }
};

__device__ __forceinline__ void load_block_words(const uint8_t* buf, uint32_t lane, uint32_t (&w)[16]) {
    // lane's 64 bytes live at buf + 64*lane; read the four 16-byte chunks in the rotated
    // order (j + lane/2) & 3 so that every quarter-warp touches all 32 banks once
    const uint4* base = reinterpret_cast<const uint4*>(buf + 64 * lane);
    const uint32_t r = (lane >> 1) & 3;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        uint4 q = base[(j + r) & 3];
        w[4 * j + 0] = q.x;
        w[4 * j + 1] = q.y;
        w[4 * j + 2] = q.z;
        w[4 * j + 3] = q.w;
    }
}

// bytes at or beyond `len` read as 0x20 (find_structural_bits_amd64.s:134-155).
// PARSE: the streaming parse's stage 1.  No index is extracted or written (out / out_cap are not used); phase B adds
// up, per slab, the counts stage 2 needs (SlabAgg: the same step_events / agg_lane_add / agg_warp_finish the emulator's
// counting pass runs) from one classification per block, run behind bar_P, with the slab's bytes still in shared memory.
template <bool NDJSON, bool DELTAS, bool PARSE = false>
__global__ void __launch_bounds__(S1_THREADS, S1_CTAS_PER_SM) stage1_flatten_kernel(const Stage1Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    // workers -> scan warp: quote parity, structural count, last structural (+1) of each slab
    __shared__ uint32_t s_par[S1_WARPS], s_cnt[S1_WARPS], s_last[S1_WARPS];
    // scan warp -> workers: in-string state in front of each slab of the current tile; output
    // offset and last structural (+1) in front of each slab of the previous tile
    __shared__ uint32_t s_parin[S1_WARPS], s_wlast[S1_WARPS];
    __shared__ unsigned long long s_off[S1_WARPS];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)S1_BUFS * S1_TILE_BYTES);
    // hand-shakes between the worker warps and the scan warp (one phase per iteration).  Workers
    // never wait for each other directly: they signal P / R and wait for the scan warp's S / Q.
    uint64_t* const bar_P = bars + 2;  // workers -> scan: slab parities of the tile are written   (count = workers)
    uint64_t* const bar_R = bars + 3;  // workers -> scan: slab counts of the tile are written     (count = workers)
    uint64_t* const bar_S = bars + 4;  // scan -> workers: output offsets of the previous tile     (count = 1)
    uint64_t* const bar_Q = bars + 5;  // scan -> workers: in-string state in front of every slab  (count = 1)
    const uint64_t len16 = (p.len + 15) & ~15ull;
    const int G = (int)gridDim.x;

    // Tiles are dealt round-robin to the CTAs of a COOPERATIVE launch (all CTAs co-resident), so
    // every predecessor a look-back waits for is owned by a running CTA; thread 0 issues one TMA
    // bulk copy per tile, one tile ahead.
    auto issue = [&](int t, int b) {
        if (t < p.ntiles) {
            uint64_t start = (uint64_t)t * S1_TILE_BYTES;
            uint32_t bytes = (uint32_t)min((uint64_t)S1_TILE_BYTES, len16 - start);
            // the buffer was last written through the generic proxy (staged positions)
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&bars[b], bytes);
            tma_load_1d(smem + (size_t)b * S1_TILE_BYTES, p.msg + start, bytes, &bars[b]);
        }
    };

    int tile = blockIdx.x;
    if (threadIdx.x == S1_WARPS * 32) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(bar_P, S1_WARPS);
        mbar_init(bar_R, S1_WARPS);
        mbar_init(bar_S, 1);
        mbar_init(bar_Q, 1);
        mbar_fence_init();
        issue(tile, 0);
    }
    __syncthreads();
    int b = 0;

    // ---------------------------------------------------------------------------------------
    // Scan warp: owns both decoupled look-backs and the TMA issue, so that neither chain ever
    // stalls the worker warps.  Per iteration (tile T_i, previous tile T_(i-1) of this CTA):
    //   while the workers classify T_i     : chain 2 (output offset) of T_(i-1)  -> s_off
    //   barrier (1)
    //   while the workers flatten T_(i-1)  : chain 1 (quote parity) of T_i       -> s_parin
    //   barrier (2), barrier (3)
    //   publish T_i's structural count (chain-2 aggregate)
    // ---------------------------------------------------------------------------------------
    if (warp == S1_WARPS) {
        bool have_prev = false;
        int prev_tile = 0;
        uint32_t prev_tile_count = 0, prev_par_out = 0;
        uint32_t prev_wbase = 0, prev_wlast = 0;  // lane w: structurals / last structural (+1) in the slabs below slab w
        uint32_t itpar = 0;                        // parity of the iteration = phase of the hand-shake barriers
        while (tile < p.ntiles || have_prev) {
            const bool cur = tile < p.ntiles;  // CTA-uniform
            uint64_t tb = 0;
            if (have_prev) {  // every tile in front of prev_tile published its count one iteration ago
                if (prev_tile > 0) tb = lookback_count(p.dcnt, prev_tile);
                if (lane == 0) {
                    st_relaxed_u64(reinterpret_cast<uint64_t*>(cnt_slot(p.dcnt, prev_tile) + 8), DI_VALID | (tb + prev_tile_count));
                    if (prev_tile == p.ntiles - 1) {
                        p.result->n_idx = (uint32_t)(tb + prev_tile_count);
                        p.result->ends_in_string = prev_par_out;
                    }
                }
            }
            if (lane < S1_WARPS) {
                s_off[lane] = tb + prev_wbase;
                s_wlast[lane] = prev_wlast;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_S);
            mbar_wait(bar_P, itpar);  // every worker has classified its slab: buffer b^1 (tile i-1) is dead
            if (lane == 0) issue(tile + G, b ^ 1);
            const uint32_t parbits = __ballot_sync(FULL, lane < S1_WARPS && s_par[lane < S1_WARPS ? lane : 0] != 0);
            const uint32_t tile_par = __popc(parbits) & 1;
            uint32_t tin = 0;
            if (cur) {
                if (lane == 0)
                    st_relaxed_u32(par_slot(p.dpar, tile), DP_VALID | (tile == 0 ? DP_INCL : 0) | (tile_par ? DP_PAR : 0));
                if (tile > 0) {
                    tin = lookback_parity(p.dpar, tile);
                    if (lane == 0) st_relaxed_u32(par_slot(p.dpar, tile), DP_VALID | DP_INCL | ((tile_par ^ tin) ? DP_PAR : 0));
                }
            }
            const uint32_t slab_in = tin ^ (__popc(parbits & lanemask_lt()) & 1);
            if (lane < S1_WARPS) s_parin[lane] = slab_in;
            if (p.slabpar) {  // (kernel-uniform)
                const uint32_t inbits = __ballot_sync(FULL, lane < S1_WARPS && slab_in != 0);
                if (cur && lane == 0) p.slabpar[tile] = inbits;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_Q);
            mbar_wait(bar_R, itpar);
            itpar ^= 1;
            // per-slab prefixes of the tile just finished (consumed by its flatten, next iteration)
            const uint32_t cnt = lane < S1_WARPS ? s_cnt[lane] : 0, l1 = lane < S1_WARPS ? s_last[lane] : 0;
            uint32_t incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                uint32_t t = __shfl_up_sync(FULL, incl, d);
                if (lane >= d) incl += t;
            }
            const uint32_t tile_count = __shfl_sync(FULL, incl, 31);
            const uint32_t nonempty = __ballot_sync(FULL, l1 != 0);
            const uint32_t below = nonempty & lanemask_lt();
            const uint32_t got = __shfl_sync(FULL, l1, below ? 31 - __clz(below) : 0);
            const uint32_t tile_last1 = __shfl_sync(FULL, l1, nonempty ? 31 - __clz(nonempty) : 0);
            prev_wbase = incl - cnt;
            prev_wlast = below ? got : 0;
            if (cur && lane == 0) {  // chain-2 aggregate; its look-back runs one iteration later
                p.lastp1[tile] = tile_last1;
                st_relaxed_u32(reinterpret_cast<uint32_t*>(cnt_slot(p.dcnt, tile)), DA_VALID | tile_count);
            }
            have_prev = cur;
            prev_tile = tile;
            prev_tile_count = tile_count;
            prev_par_out = tin ^ tile_par;
            tile += G;
            b ^= 1;
        }
        return;
    }

    uint32_t phasebits = 0;
    uint32_t itpar = 0;  // parity of the iteration = phase of the hand-shake barriers
    const RotSel rsel = rot_selectors((lane >> 1) & 3);  // undoes the bank-conflict-free chunk order of load_block_words

    // software pipeline: iteration i runs phase A / chain 1 / phase B of tile T_i and the chain-2
    // look-back + flatten of tile T_(i-1); one drain iteration flattens the last tile
    bool have_prev = false;
    uint64_t S_prev[S1_STEPS];
#pragma unroll
    for (int s = 0; s < S1_STEPS; s++) S_prev[s] = 0;
    int prev_tile = 0;
    uint32_t prev_slab_count = 0;

    // bytes in front of a warp's slab of tile t (0x20 = "nothing there": first slab, or no such slab)
    auto peek_load = [&](int t) -> uint32_t {
        const uint64_t ss = ((uint64_t)t * S1_WARPS + warp) * S1_SLAB_BYTES;
        return (t < p.ntiles && ss < p.len && ss > lane) ? (uint32_t)p.msg[ss - 1 - lane] : 0x20u;
    };
    uint32_t peekc = peek_load(tile);
    K1_PROBE_START

    while (tile < p.ntiles || have_prev) {
        const bool cur = tile < p.ntiles;  // CTA-uniform
        const int slab = tile * S1_WARPS + (int)warp;
        const uint64_t slab_start = (uint64_t)slab * S1_SLAB_BYTES;
        const bool active = cur && slab_start < p.len;  // warps past the end of the message only keep the barriers
        const bool tail_tile = tile >= p.ntiles - 1;
        const uint8_t* buf = smem + (size_t)b * S1_TILE_BYTES + (size_t)warp * S1_SLAB_BYTES;

        // carries that depend only on raw bytes in front of the slab: lane L holds byte
        // slab_start - 1 - L (loaded one iteration ago, under the flatten of the previous tile)
        uint32_t bs_carry, prevc_esc = 0;
        const uint32_t peek_bs = __ballot_sync(FULL, peekc == '\\');
        const uint32_t prevc = __shfl_sync(FULL, peekc, 0);
        if (peek_bs == FULL)
            bs_carry = backslash_run_before(p.msg, slab_start) & 1;  // a run of 32 or more: walk it
        else
            bs_carry = (__ffs(~peek_bs) - 1) & 1;
        if (prevc == '"') {  // warp-uniform; is that quote escaped?
            const uint32_t n = __ffs(~(peek_bs >> 1)) - 1;
            prevc_esc = n == 31 ? backslash_run_before(p.msg, slab_start - 1) & 1 : n & 1;
        }
        K1_PROBE(K1P_CARRIES);
        if (cur) {
            mbar_wait(&bars[b], (phasebits >> b) & 1);
            phasebits ^= 1u << b;
        }

        // the last tile: bytes past the end of the message read as spaces (find_structural_bits_amd64.s:167);
        // padded in shared memory so that the hot loop carries no tail handling at all
        if (tail_tile && active && p.len - slab_start < S1_SLAB_BYTES) {
            uint8_t* wbuf = smem + (size_t)b * S1_TILE_BYTES + (size_t)warp * S1_SLAB_BYTES;
            for (uint32_t o = (uint32_t)(p.len - slab_start) + lane; o < S1_SLAB_BYTES; o += 32) wbuf[o] = 0x20;
            __syncwarp();
        }
        K1_PROBE(K1P_TMA);

        // ---------------- phase A: classify, escape analysis, slab quote parity ----------------
        uint64_t qb[S1_STEPS], st[S1_STEPS], ws[S1_STEPS], ct[S1_STEPS], nl[S1_STEPS], bsm[S1_STEPS], qmr[S1_STEPS];
        uint64_t px[S1_STEPS], py[S1_STEPS];  // PARSE: the rest of the classes phase B reads (parse_planes)
        uint32_t slab_par = 0;
        uint32_t cinbits = 0;  // PARSE: bit s = escape carry into the lane's block of step s
        uint32_t ctbits = 0;   // PARSE: bit s / bit 8 + s = a control character inside / outside the slab-relative quote mask of step s
        uint32_t* const stage = reinterpret_cast<uint32_t*>(smem + (size_t)b * S1_TILE_BYTES + (size_t)warp * S1_SLAB_BYTES);
        const uint32_t pslab_pos = (uint32_t)(((uint64_t)prev_tile * S1_WARPS + warp) * S1_SLAB_BYTES);
#pragma unroll
        for (int s = 0; s < S1_STEPS; s++) {
            qb[s] = st[s] = ws[s] = ct[s] = nl[s] = bsm[s] = qmr[s] = px[s] = py[s] = 0;
            if (active && PARSE) {
                // parse mode: the quote parity first, from the quotes and backslashes alone (the word-wise classifier),
                // so that chain 1 starts early; the other classes come after bar_P, under the look-back
                uint32_t w[16];
                load_block_words(buf + s * S1_STEP_BYTES, lane, w);
                const BlockMasks m = classify_block(w);
                bsm[s] = rotl16x((uint32_t)m.bs, (uint32_t)(m.bs >> 32), rsel);
                qb[s] = rotl16x((uint32_t)m.qt, (uint32_t)(m.qt >> 32), rsel);
            } else if (active) {
                uint32_t w[16];
                load_block_words(buf + s * S1_STEP_BYTES, lane, w);
                PlaneMasks m = classify_block_planes(w);
                bsm[s] = rotl16x((uint32_t)m.bs, (uint32_t)(m.bs >> 32), rsel);
                qb[s] = rotl16x((uint32_t)m.qt, (uint32_t)(m.qt >> 32), rsel);  // raw quotes; escaped ones are removed in pass 2
                st[s] = rotl16x((uint32_t)m.st, (uint32_t)(m.st >> 32), rsel);
                ws[s] = rotl16x((uint32_t)m.ws, (uint32_t)(m.ws >> 32), rsel);
                ct[s] = rotl16x((uint32_t)m.ct, (uint32_t)(m.ct >> 32), rsel);
                if (NDJSON) nl[s] = rotl16x((uint32_t)m.nl, (uint32_t)(m.nl >> 32), rsel);
            }
        }
        K1_PROBE(K1P_CLASSIFY);
        if (active) {
            // pass 2: everything that needs votes across the warp
#pragma unroll
            for (int s = 0; s < S1_STEPS; s++) {
                const uint64_t bs = bsm[s];
                // odd-backslash carry into each lane's block (warp-uniform fast path: no backslashes at all)
                uint64_t odd_ends = 0;
                const uint32_t hasbs = __ballot_sync(FULL, bs != 0);
                if (hasbs || bs_carry) {
                    uint32_t allbs = bs == ~0ull;
                    uint32_t trail_odd = (bs == ~0ull) ? 0 : (__clzll(~bs) & 1);
                    uint32_t A = __ballot_sync(FULL, allbs);
                    uint32_t F = __ballot_sync(FULL, trail_odd);
                    uint32_t below = ~A & lanemask_lt();
                    uint32_t cin = below ? (F >> (31 - __clz(below))) & 1 : bs_carry;
                    uint32_t nonpass = ~A;
                    bs_carry = nonpass ? (F >> (31 - __clz(nonpass))) & 1 : bs_carry;
                    odd_ends = odd_backslash_ends(bs, cin, nullptr);
                    if (PARSE) cinbits |= cin << s;
                }
                qb[s] &= ~odd_ends;
                // quote mask relative to the start of the slab (find_quote_mask_and_bits_amd64.s:49-66); the
                // state in front of the slab is XORed in once chain 1 has delivered it (phase B)
                const uint32_t P = __ballot_sync(FULL, (__popcll(qb[s]) & 1) != 0);
                const uint32_t lane_rel = slab_par ^ (__popc(P & lanemask_lt()) & 1);
                slab_par ^= __popc(P) & 1;
                qmr[s] = prefix_xor64(qb[s]) ^ (lane_rel ? ~0ull : 0ull);
                if (p.bsmap && lane == 0) p.bsmap[slab * S1_STEPS + s] = hasbs;
            }
        }
        K1_PROBE(K1P_PASS2);
        // P: the slab's parity is written and the warp is done with buffer b^1.  When the last worker
        // has signalled, the scan warp issues the TMA of the next tile into b^1 and starts chain 1 of
        // this tile; nobody waits here, so the warps drift apart and the ALU-bound classification of
        // late warps overlaps the FLO / store-bound extraction of early ones.
        if (lane == 0) {
            s_par[warp] = slab_par;
            mbar_arrive(bar_P);
        }
        const uint32_t peek_next = peek_load(tile + G);
        if (PARSE && active) {
            // the classes phase B reads, from one bit-sliced classification of each block (the slab's bytes stay in
            // buffer b: parse mode stages nothing over them)
#pragma unroll
            for (int s = 0; s < S1_STEPS; s++) {
                uint32_t w[16];
                load_block_words(buf + s * S1_STEP_BYTES, lane, w);
                const PlaneMasks m = classify_block_planes(w);
                st[s] = rotl16x((uint32_t)m.st, (uint32_t)(m.st >> 32), rsel);
                ws[s] = rotl16x((uint32_t)m.ws, (uint32_t)(m.ws >> 32), rsel);
                if (NDJSON) nl[s] = rotl16x((uint32_t)m.nl, (uint32_t)(m.nl >> 32), rsel);
                px[s] = rotl16x((uint32_t)m.px, (uint32_t)(m.px >> 32), rsel);
                py[s] = rotl16x((uint32_t)m.py, (uint32_t)(m.py >> 32), rsel);
                const uint64_t ctm = rotl16x((uint32_t)m.ct, (uint32_t)(m.ct >> 32), rsel);
                ctbits |= ((ctm & qmr[s]) != 0 ? 1u : 0u) << s | ((ctm & ~qmr[s]) != 0 ? 1u : 0u) << (8 + s);
            }
            K1_PROBE(K1P_CLASSIFY);
        }
        // ---------------- extraction of the previous tile's structurals ----------------
        // the positions are staged over the warp's own slab of this tile (dead: this warp alone read
        // it, in phase A above)
        uint32_t staged = 0;  // entries staged (warp-uniform)
        uint32_t dense = 0;   // more than one structural per 4 bytes: the slab does not fit its own staging area
        if (!PARSE && have_prev) {
            __syncwarp();
#pragma unroll
            for (int s = 0; s < S1_STEPS; s++) {
                if (!dense) {
                    const uint32_t n = extract_step(S_prev[s], pslab_pos + s * S1_STEP_BYTES + 64 * lane, stage + staged,
                                                    S1_SLAB_BYTES / 4 - staged);
                    dense = n > S1_SLAB_BYTES / 4 - staged;
                    staged += n;
                }
            }
        }
        mbar_wait(bar_S, itpar);  // output offsets of the previous tile (chain 2, run by the scan warp under phase A)
        __syncwarp();            // staged positions of all lanes are visible

        // ---------------- copy-out of the previous tile's staged structurals ----------------
        if (!PARSE && have_prev) {
            // deltas: the first structural of a tile is written as pos + 1 here and rebased on the
            // previous tile's last structural by stage1_finish_kernel
            uint32_t prev_last = s_wlast[warp] - 1;  // 0xffffffff when nothing precedes inside the tile
            const uint64_t off = s_off[warp];
            if (off + prev_slab_count > p.out_cap) {  // warp-uniform
                if (lane == 0) atomicOr(&p.result->overflow, 1u);
            } else if (!dense) {
                copy_out<DELTAS>(stage, staged, p.out + off, prev_last);
            } else {  // more than one structural per 4 bytes somewhere in the slab: unstaged path
                flatten_slab_staged<DELTAS, S1_STEPS>(S_prev, pslab_pos, p.out + off, prev_last, stage, S1_SLAB_BYTES / 4);
            }
        }
        mbar_wait(bar_Q, itpar);  // quote parity in front of the tile (chain 1, run by the scan warp meanwhile)
        const uint32_t par_in = s_parin[warp];

        // pseudo-structural predecessor carry into the slab (finalize_structurals_amd64.s:24-27;
        // initial value 1: stage1_find_marks_amd64.go:54)
        uint32_t pp_carry = 1;
        if (slab > 0) {
            uint32_t is_q = prevc == '"' && !prevc_esc;
            uint32_t is_ws = prevc == 0x20 || prevc == 0x09 || prevc == 0x0a || prevc == 0x0d;
            uint32_t is_st = prevc == '{' || prevc == '}' || prevc == '[' || prevc == ']' || prevc == ':' || prevc == ',';
            // prevc not a quote: its quote_mask bit equals the in-string state after it (= par_in)
            pp_carry = is_q | is_ws | (is_st & (par_in ^ 1));
        }
        K1_PROBE(K1P_WAIT);

        // ---------------- phase B: quote mask, finalize, counts ----------------
        uint32_t err = 0;
        uint32_t slab_count = 0;
        const uint64_t flip = par_in ? ~0ull : 0ull;
        if constexpr (PARSE) {
            // stage 2's counts of the slab, as s2s_slab<W, false> adds them up (the carries into the slab are the ones
            // worked out above, or from the bytes in front of it as it does)
            DevWarp wp;
            const GlobalReader g{p.msg, p.len};
            const SlabReader rd{buf, slab_start, active ? (uint32_t)min((uint64_t)S1_SLAB_BYTES, p.len - slab_start) : 0u, p.msg, p.len};
            LaneAgg la = lane_agg_zero();
            uint32_t s2err = 0, hd_drop = 0;
            err = (par_in ? ctbits >> 8 : ctbits & 0xffu) != 0;  // find_quote_mask_and_bits_amd64.s:69-80
            uint32_t ppc = pp_carry;
            uint32_t recc = (NDJSON && active && !par_in && slab > 0) ? record_carry_in(wp, g, slab_start, peekc) : 0u;
            K1_PROBE(K1P_CARRIES);
#pragma unroll
            for (int s = 0; s < S1_STEPS; s++) {
                const uint64_t qm = qmr[s] ^ flip;
                const uint64_t step_start = slab_start + (uint64_t)s * S1_STEP_BYTES;
                uint64_t fin = 0;
                if (active && step_start < p.len) {  // warp-uniform
                    Class64 m = classes_from_parse_planes(st[s], px[s], py[s]);
                    m.ws = ws[s];
                    m.nl = nl[s];
                    K1_PROBE(K1P_B_CLASSIFY);
                    // escapes inside strings -> the bytes they drop from Strings.B; what an escape that starts in front
                    // of the step leaves behind its start: head_info at the slab start, the previous step's last lane
                    // inside the slab
                    const uint64_t Ein = escape_starts(bsm[s], (cinbits >> s) & 1u) & qm;
                    if (s == 0) {
                        const HeadInfo hd = head_info(wp, g, step_start, par_in != 0, peekc);
                        hd_drop = hd.drop;
                        s2err |= hd.bad;
                    }
                    uint64_t D = 0;
                    uint32_t next_drop = 0;
                    if (__any_sync(FULL, Ein != 0)) {
                        uint32_t spill = 0;  // dropped bytes of the lane's escapes that lie in the next block
                        const uint64_t bp = step_start + 64 * lane;
                        for (uint64_t r = Ein; r; r &= r - 1) {
                            const uint32_t j = (uint32_t)__ffsll((long long)r) - 1;
                            EscInfo ei;
                            if (!esc_u_fast(buf + s * S1_STEP_BYTES, 64 * lane + j, (uint32_t)min((uint64_t)S1_STEP_BYTES, p.len - step_start), ei,
                                            FlatLayout()))
                                ei = esc_decode(rd, g, bp + j);
                            if (ei.second) continue;
                            if (!ei.valid) {
                                s2err = 1;
                                continue;
                            }
                            const uint32_t hi = j + ei.c - ei.n;  // all c source bytes are dropped except the last n
                            D |= range64(j, hi < 64 ? hi : 64);
                            if (hi > 64) spill |= (uint32_t)below64(hi - 64);
                        }
                        const uint32_t up = __shfl_up_sync(FULL, spill, 1);
                        if (lane) D |= up;
                        next_drop = __shfl_sync(FULL, spill, 31);
                    }
                    if (lane == 0) D |= hd_drop;
                    hd_drop = next_drop;
                    const uint64_t K = qm & ~qb[s] & ~D;
                    K1_PROBE(K1P_B_ESCAPES);
                    const StepEvents e = step_events(wp, m, qm, qb[s], K, NDJSON ? 1u : 0u, ppc, recc);
                    K1_PROBE(K1P_EVENTS);
                    agg_lane_add(la, e, s);
                    K1_PROBE(K1P_AGG);
                    fin = e.S;
                }
                S_prev[s] = fin;
                slab_count += __popcll(fin);
            }
            if (__any_sync(FULL, s2err) && lane == 0) atomicOr(p.s2_error, 1u);
            if (active) {  // warp-uniform
                const SlabAgg run = agg_warp_finish(wp, la, S_prev, [&](uint32_t s, uint32_t o) { return (uint32_t)buf[s * S1_STEP_BYTES + o]; });
                K1_PROBE(K1P_AGG);
                if (lane == 0) p.agg[slab] = run;
            }
        } else {
#pragma unroll
        for (int s = 0; s < S1_STEPS; s++) {
            const uint64_t qm = qmr[s] ^ flip;
            if (ct[s] & qm) err = 1;  // find_quote_mask_and_bits_amd64.s:69-80
            // pseudo_pred bit of the previous block: previous lane, or the carry for lane 0
            uint64_t s0 = (st[s] & ~qm) | qb[s];
            uint32_t my_pp = (uint32_t)((s0 | ws[s]) >> 63);
            uint32_t up = __shfl_up_sync(FULL, my_pp, 1);
            uint32_t pp_in = lane == 0 ? pp_carry : up;
            pp_carry = __shfl_sync(FULL, my_pp, 31);
            uint32_t dummy;
            uint64_t fin = finalize_structurals(st[s], ws[s], qm, qb[s], pp_in, &dummy);
            if (NDJSON) fin |= nl[s] & ~qm;  // find_newline_delimiters_amd64.s:17-27
            if (!active) fin = 0;
            S_prev[s] = fin;  // flattened in the next iteration
            slab_count += __popcll(fin);
        }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) slab_count += __shfl_xor_sync(FULL, slab_count, d);
        if (__any_sync(FULL, err)) {
            if (lane == 0) atomicOr(&p.result->error, 1u);
        }

        // last structural of the slab (pos + 1, 0 = none)
        uint32_t own_last1 = 0;
#pragma unroll
        for (int s = S1_STEPS - 1; s >= 0; s--) {
            if (own_last1 == 0 && S_prev[s] != 0)
                own_last1 = (uint32_t)(slab_start + (uint64_t)s * S1_STEP_BYTES + 64 * lane + 63 - __clzll(S_prev[s])) + 1;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) own_last1 = max(own_last1, __shfl_xor_sync(FULL, own_last1, d));
        if (lane == 0) {
            s_cnt[warp] = slab_count;
            s_last[warp] = own_last1;
        }
        // R: slab counts of the tile are written (the same lane 0 wrote them)
        if (lane == 0) mbar_arrive(bar_R);
        itpar ^= 1;
        K1_PROBE(K1P_STORE);

        have_prev = cur;
        prev_tile = tile;
        prev_slab_count = slab_count;
        peekc = peek_next;
        tile += G;
        b ^= 1;
    }
    K1_PROBE_FLUSH;
}

// After K1: rebase the first delta of every tile on the last structural of the tiles in
// front of it (delta mode), and record the position of the last structural of the message.
template <bool DELTAS>
__global__ void stage1_finish_kernel(const Stage1Params p) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= p.ntiles) return;
    const uint32_t own = p.lastp1[s];
    if (s == p.ntiles - 1) {
        int t = s;
        uint32_t l = own;
        while (l == 0 && t > 0) l = p.lastp1[--t];
        p.result->last_pos = l - 1;
        p.result->last_char = l != 0 && (uint64_t)(l - 1) < p.len ? p.msg[l - 1] : 0;
    }
    if (!DELTAS || own == 0 || s == 0) return;
    int t = s - 1;
    uint32_t prev = p.lastp1[t];
    while (prev == 0 && t > 0) prev = p.lastp1[--t];
    if (prev == 0) return;  // no structural in front: the first delta stays pos + 1
    const uint64_t incl = *reinterpret_cast<const uint64_t*>(cnt_slot(p.dcnt, s) + 8) & ~DI_VALID;
    const uint64_t first = incl - (*reinterpret_cast<const uint32_t*>(cnt_slot(p.dcnt, s)) & ~DA_VALID);
    if (first < p.out_cap) p.out[first] -= prev;  // (pos + 1) - (prev_pos + 1)
}

}  // namespace sj
