// s2s_core.h -- streaming stage 2 ("K2p count / K2r emit"): the tape build as a bit-parallel pass over the MESSAGE,
// one warp per 6 KiB slab, lane L = 64-byte block L of each 2 KiB step -- the same decomposition as the stage-1
// kernel -- instead of one thread per structural.
//
// What the reference does serially per structural (unifiedMachine, stage2_build_tape_amd64.go:160-446; parseString,
// parse_string_amd64.s:72-479) is done here per 64-byte block with mask algebra:
//   * every count stage 2 needs in front of a block (tape words, string-buffer bytes, brackets, depth, records,
//     numbers) is a popcount of a class mask, so the offsets come from one scan over per-slab aggregates (K2q)
//     between a counting pass (K2p) and the emitting pass (K2r), both of which run the SAME analysis code below;
//   * Strings.B (copy_strings, options.go:13 default) is a byte compaction of the message under the mask "inside a
//     string, not a quote, not a consumed escape byte": escapes are decoded where their backslash sits (escape
//     starts = backslashes at an even offset of their run, the same parity argument as
//     find_odd_backslash_sequences_amd64.s:24-61) and their UTF-8 bytes patched into the compacted stream;
//   * a string is emitted at its CLOSING quote (no structural lies between the two quotes), which is where its
//     unescaped length and its end offset in Strings.B are known;
//   * the grammar (stage2...go:176-425) is checked per structural against the PREVIOUS structural only: strings are
//     refined into "follows '{' or ','" (a key in an object) and "follows anything else", so the transition depends
//     on one predecessor; what depends on the enclosing container is collected as a 3-bit mask {root, object, array}
//     ANDed per bracket-to-bracket segment and resolved once per bracket after the scope matching (K2t).
//
// This header is portable C++: under nvcc the functions are __host__ __device__, and tests/emu/s2s_emu.cpp compiles
// the very same templates with a 32-fiber "warp" to check them against the oracle on a machine without a GPU.
#pragma once
#include "bits.h"

namespace sj {

// ---------------------------------------------------------------------------------
// structural types (shared with the per-structural kernels of stage2.cuh) and the grammar
// ---------------------------------------------------------------------------------
enum : uint8_t {
    T_INVALID = 0,
    T_OBJ_OPEN = 1,
    T_ARR_OPEN = 2,
    T_OBJ_CLOSE = 3,
    T_ARR_CLOSE = 4,
    T_COLON = 5,
    T_COMMA = 6,
    T_STRING = 7,
    T_NUMBER = 8,
    T_TRUE = 9,
    T_FALSE = 10,
    T_NULL = 11,
    T_NEWLINE = 12,
    T_START = 13,
    T_STRING_KEYPOS = 14,  // streaming stage 2 only: a string whose predecessor is '{' or ','
};
enum : uint32_t { CTX_ROOT = 0, CTX_OBJ = 1, CTX_ARR = 2 };

SJ_HDC bool is_value_start(uint32_t c) {
    return c == T_STRING || c == T_NUMBER || c == T_TRUE || c == T_FALSE || c == T_NULL || c == T_OBJ_OPEN ||
           c == T_ARR_OPEN;
}
SJ_HDC bool is_scalar_or_close(uint32_t c) {
    return c == T_NUMBER || c == T_TRUE || c == T_FALSE || c == T_NULL || c == T_OBJ_CLOSE || c == T_ARR_CLOSE;
}

// stage2_build_tape_amd64.go:176-425, restated as "is c allowed after p (after pp) inside ctx"
SJ_HDC bool transition_ok(uint32_t ctx, uint32_t pp, uint32_t p, uint32_t c) {
    if (c == T_INVALID) return false;
    if (ctx == CTX_OBJ) {
        if (p == T_OBJ_OPEN) return c == T_STRING || c == T_OBJ_CLOSE;                // object_begin :225-240
        if (p == T_STRING) {
            const bool is_key = pp == T_OBJ_OPEN || pp == T_COMMA;
            return is_key ? c == T_COLON : (c == T_COMMA || c == T_OBJ_CLOSE);         // :242-248 / objectContinue :302-324
        }
        if (p == T_COLON) return is_value_start(c);                                      // :251-300
        if (is_scalar_or_close(p)) return c == T_COMMA || c == T_OBJ_CLOSE;             // objectContinue
        if (p == T_COMMA) return c == T_STRING;                                          // :309-316
        return false;
    }
    if (ctx == CTX_ARR) {
        if (p == T_ARR_OPEN) return is_value_start(c) || c == T_ARR_CLOSE;             // arrayBegin :347-353
        if (p == T_STRING || is_scalar_or_close(p)) return c == T_COMMA || c == T_ARR_CLOSE;  // arrayContinue :409-425
        if (p == T_COMMA) return is_value_start(c);                                      // mainArraySwitch :355-407
        return false;
    }
    // top level
    if (p == T_START) return c == T_OBJ_OPEN || c == T_ARR_OPEN;                       // continueRoot :176-188
    if (p == T_OBJ_CLOSE || p == T_ARR_CLOSE) return c == T_NEWLINE;                   // startContinue :196-198
    if (p == T_NEWLINE) return c == T_NEWLINE || c == T_OBJ_OPEN || c == T_ARR_OPEN;   // :200-221
    return false;
}

// the same grammar on REFINED types (strings carry "my predecessor was '{' or ','"): bit ctx of the result says
// whether c may follow p inside a container of kind ctx
SJ_HDC uint32_t transition_mask(uint32_t p, uint32_t c) {
    const uint32_t pb = p == T_STRING_KEYPOS ? (uint32_t)T_STRING : p;
    const uint32_t cb = c == T_STRING_KEYPOS ? (uint32_t)T_STRING : c;
    const uint32_t pp = p == T_STRING_KEYPOS ? (uint32_t)T_COMMA : (uint32_t)T_INVALID;  // only "is p a key" matters
    uint32_t m = 0;
    for (uint32_t ctx = 0; ctx < 3; ctx++)
        if (transition_ok(ctx, pp, pb, cb)) m |= 1u << ctx;
    return m;
}

// type of a structural from the byte it sits on (quotes: the string; the streaming pass looks at closing quotes)
SJ_HDC uint32_t char_type(uint32_t ch) {
    return ch == '{'   ? (uint32_t)T_OBJ_OPEN
           : ch == '[' ? (uint32_t)T_ARR_OPEN
           : ch == '}' ? (uint32_t)T_OBJ_CLOSE
           : ch == ']' ? (uint32_t)T_ARR_CLOSE
           : ch == ':' ? (uint32_t)T_COLON
           : ch == ',' ? (uint32_t)T_COMMA
           : ch == '"' ? (uint32_t)T_STRING
           : (ch == '-' || (ch >= '0' && ch <= '9')) ? (uint32_t)T_NUMBER
           : ch == 't' ? (uint32_t)T_TRUE
           : ch == 'f' ? (uint32_t)T_FALSE
           : ch == 'n' ? (uint32_t)T_NULL
           : ch == '\n' ? (uint32_t)T_NEWLINE
                        : (uint32_t)T_INVALID;
}

// 16 bytes moved as one vector access (LDS.128 / LDG.128 / STG.128 on the device)
struct alignas(16) V16 {
    uint32_t x, y, z, w;
};

SJ_HD uint64_t below64(uint32_t b) { return b >= 64 ? ~0ull : ((1ull << b) - 1ull); }  // bits [0, b)
SJ_HD uint64_t lt64(uint32_t b) { return (1ull << b) - 1ull; }                         // bits [0, b), b < 64
// the events of EV that follow an event of A (A a subset of EV; `cin`: the last event in front of the block is in A):
// adding (A << 1 | cin) to the complement of EV carries from the position behind each A-event to the next event
SJ_HD uint64_t next_event(uint64_t A, uint32_t cin, uint64_t EV) { return (((A << 1) | (uint64_t)cin) + ~EV) & EV; }
SJ_HD uint64_t range64(uint32_t lo, uint32_t hi) { return lo >= hi ? 0ull : below64(hi) & ~below64(lo); }  // bits [lo, hi)

// ---------------------------------------------------------------------------------
// geometry (the slab is the stage-1 kernel's slab: K1 hands over the in-string state in front of each one)
// ---------------------------------------------------------------------------------
constexpr uint32_t S2S_STEP_BYTES = 2048;                            // one warp pass: 32 lanes x 64 bytes
constexpr uint32_t S2S_STEPS = 3;  // 2 KiB steps per slab; stage 1 uses the same (S1_STEPS): its in-string bits are per slab
constexpr uint32_t S2S_SLAB_BYTES = S2S_STEPS * S2S_STEP_BYTES;      // == S1_SLAB_BYTES (static_assert in stage2_stream.cuh)
constexpr uint32_t S2S_IMAGE_BYTES = 2 * S2S_STEP_BYTES;              // two image buffers: the step at hand and the next one in flight
constexpr uint32_t S2S_SSTAGE_BYTES = S2S_STEP_BYTES + 32;           // compacted string bytes of one step (+ alignment shift)
// K2r's tape-staging area (8-byte words), which holds the escape scratch: more than the escapes need, and its size is
// part of K2r's shared memory per block, so it sets K2r's occupancy.  A step whose tape words (plus the destination's
// phase inside its 32-byte sector) fit is staged here and copied out in whole sectors; a denser one stores directly.
constexpr uint32_t S2S_TSTAGE_WORDS = 640;
// lists of a staged step's brackets and record starts, kept in the string staging area once Strings.B is out; a step
// with more of them leaves all its links to K2t
constexpr uint32_t S2S_LINK_BRK_CAP = 384, S2S_LINK_REC_CAP = 128;
constexpr uint32_t S2S_LINK_SCAN = 64;  // brackets a close looks back for its partner inside the step
// brk_kind bit: K2r has written both cross-links of this close (its partner lies in the same step), K2t skips them
constexpr uint8_t BRK_LINKED = 0x80;

// per-slab aggregate (K2p) / exclusive prefix (K2q).  `trail`: string-buffer bytes behind the last real quote of
// the slab (all of them if the slab holds no quote) -- scanned with the segmented operator below it gives, for a
// slab that starts inside a string, the bytes that string has contributed so far.
struct SlabAgg {
    uint32_t w;      // tape words
    uint32_t str;    // string-buffer bytes
    uint32_t brk;    // brackets
    uint32_t rec;    // record boundaries (NDJSON roots - 1)
    int32_t depth;   // opens - closes
    uint32_t last;   // the bytes under the last three stage-1 structurals (byte 0: the last one), their count (0..3) in bits 24..25
    uint32_t num;    // numbers
    uint32_t trail;  // bit 31: the slab holds a real quote; bits 0..30: bytes behind the last one
};
constexpr uint32_t TRAIL_HASQ = 0x80000000u;

// `last` of a in front of b: b's bytes are the later ones
SJ_HD uint32_t last_combine(uint32_t a, uint32_t b) {
    const uint32_t na = a >> 24, nb = b >> 24;
    if (nb >= 3) return b;
    const uint32_t n = na + nb < 3 ? na + nb : 3u;
    return (((a << (8 * nb)) | b) & 0xffffffu) | (n << 24);
}

SJ_HD SlabAgg agg_zero() { return SlabAgg{0, 0, 0, 0, 0, 0, 0, 0}; }
// a in front of b (not commutative in `trail`)
SJ_HD SlabAgg agg_combine(const SlabAgg& a, const SlabAgg& b) {
    SlabAgg r;
    r.w = a.w + b.w;
    r.str = a.str + b.str;
    r.brk = a.brk + b.brk;
    r.rec = a.rec + b.rec;
    r.depth = a.depth + b.depth;
    r.last = last_combine(a.last, b.last);
    r.num = a.num + b.num;
    r.trail = (b.trail & TRAIL_HASQ) ? b.trail : ((a.trail & TRAIL_HASQ) | (((a.trail & ~TRAIL_HASQ) + b.trail) & ~TRAIL_HASQ));
    return r;
}

// ---------------------------------------------------------------------------------
// byte classification: bit planes of 32 bytes (bit_planes32, bits.h), then every class as a Boolean function of the
// planes (find_whitespace_and_structurals_amd64.s:6-29 and the compares of the other stage-1 routines; same scheme as
// stage1.cuh, with the classes stage 2 needs on top: brackets by direction, first bytes of numbers / atoms)
// ---------------------------------------------------------------------------------
struct Half2 {
    uint32_t bs, qt, ws, nl, open, close, cc, comma, curly, numc, atomc;
};
SJ_HD Half2 classify_planes2(const uint32_t (&p)[8]) {
    const uint32_t n7 = ~p[7];
    const uint32_t A = n7 & ~p[6];              // 0x00..0x3f
    const uint32_t hi2 = A & p[5] & ~p[4];      // 0x2_
    const uint32_t hi3 = A & p[5] & p[4];       // 0x3_
    const uint32_t hi0 = A & ~p[5] & ~p[4];     // 0x0_
    const uint32_t hi57 = n7 & p[6] & p[4];     // 0x5_ or 0x7_
    const uint32_t hi5 = hi57 & ~p[5];
    const uint32_t hi7 = hi57 & p[5];
    const uint32_t hi6 = n7 & p[6] & p[5] & ~p[4];
    const uint32_t c32 = p[3] & p[2], c30 = p[3] & ~p[2], z32 = ~p[3] & ~p[2], n32 = ~p[3] & p[2];
    const uint32_t b00 = ~p[1] & ~p[0], b01 = ~p[1] & p[0], b10 = p[1] & ~p[0], b11 = p[1] & p[0];
    const uint32_t loC = c32 & b00, loD = c32 & b01, loE = c32 & b10;
    const uint32_t loA = c30 & b10, loB = c30 & b11, lo9 = c30 & b01;
    const uint32_t lo2 = z32 & b10, lo0 = z32 & b00;
    const uint32_t lo4 = n32 & b00, lo6 = n32 & b10;
    Half2 m;
    m.qt = hi2 & lo2;                                    // "
    m.bs = hi5 & loC;                                    // backslash
    m.open = hi57 & loB;                                 // [ {
    m.close = hi57 & loD;                                // ] }
    m.comma = hi2 & loC;                                 // ,
    m.cc = m.comma | (hi3 & loA);                        // , :
    m.curly = p[5];                                      // among [ ] { }: the curly ones (0x7b, 0x7d against 0x5b, 0x5d)
    m.ws = (hi2 & lo0) | (hi0 & (lo9 | loA | loD));      // space \t \n \r
    m.nl = hi0 & loA;                                    // \n
    m.numc = (hi3 & (~p[3] | (c30 & ~p[1]))) | (hi2 & loD);  // 0-9 -
    m.atomc = (hi7 & lo4) | (hi6 & (lo6 | loE));         // t f n
    return m;
}
struct Class64 {
    uint64_t bs, qt, ws, nl, open, close, cc, comma, curly, numc, atomc;
};
// w[16]: the block's 64 bytes in natural order
SJ_HD Class64 classify_block2(const uint32_t (&w)[16]) {
    uint32_t p0[8], p1[8];
    bit_planes32(&w[0], p0);
    bit_planes32(&w[8], p1);
    const Half2 a = classify_planes2(p0), b = classify_planes2(p1);
    Class64 m;
    m.bs = mk64(a.bs, b.bs);
    m.qt = mk64(a.qt, b.qt);
    m.ws = mk64(a.ws, b.ws);
    m.nl = mk64(a.nl, b.nl);
    m.open = mk64(a.open, b.open);
    m.close = mk64(a.close, b.close);
    m.cc = mk64(a.cc, b.cc);
    m.comma = mk64(a.comma, b.comma);
    m.curly = mk64(a.curly, b.curly);
    m.numc = mk64(a.numc, b.numc);
    m.atomc = mk64(a.atomc, b.atomc);
    return m;
}

// Stage 1's parse mode classifies each block once: next to its structurals st ({ } [ ] , :) it keeps two planes of the
// same transpose, X = brackets | first bytes of numbers and Y = opening brackets | first bytes of atoms.  No structural
// starts a number or an atom, so st takes them apart again (classes_from_parse_planes).
struct ParsePlanes {
    uint32_t x, y;
};
SJ_HD ParsePlanes parse_planes(const uint32_t (&p)[8]) {
    const Half2 m = classify_planes2(p);
    return ParsePlanes{m.open | m.close | m.numc, m.open | m.atomc};
}
// open, close, cc, numc, atomc of a block from st and its X / Y planes (the other members are left 0)
SJ_HD Class64 classes_from_parse_planes(uint64_t st, uint64_t x, uint64_t y) {
    Class64 m{};
    m.open = st & y;
    m.close = st & x & ~y;
    m.cc = st & ~x;
    m.numc = x & ~st;
    m.atomc = y & ~st;
    return m;
}

// Escape STARTS of a block: the backslashes that sit at an even offset inside their run (every second one, beginning
// with the first).  `first_escaped` = the block's first byte is consumed by an escape that started in front of the
// block (the carry of find_odd_backslash_sequences_amd64.s:27-58): a run beginning at bit 0 then starts at an odd offset.
SJ_HD uint64_t escape_starts(uint64_t bs, uint32_t first_escaped) {
    const uint64_t EVEN = 0x5555555555555555ull, ODD = 0xAAAAAAAAAAAAAAAAull;
    const uint64_t starts = bs & ~(bs << 1);
    const uint64_t even_starts = starts & (EVEN ^ (uint64_t)first_escaped);
    const uint64_t evenrun = bs & ~(bs + even_starts);  // members of the runs that start at an even position
    const uint64_t oddrun = bs & ~evenrun;
    return (evenrun & EVEN) | (oddrun & ODD);
}

// ---------------------------------------------------------------------------------
// escapes (parse_string_amd64.s:101-229; accept / reject behaviour as restated in stage2.cuh escape_step)
// ---------------------------------------------------------------------------------
struct EscInfo {
    uint32_t c;      // source bytes consumed (2, 6 or 12); 0 for the second half of a surrogate pair
    uint32_t n;      // UTF-8 bytes produced (1..4)
    uint32_t bytes;  // the produced bytes, first one in bits 0..7
    bool valid;
    bool second;     // "\uXXXX" that is the low half of a pair whose high half starts six bytes earlier
};

// four hex digits at x..x+3; 0xffffffff when one of them is a raw quote (the D >= 6 rule of parse_string_amd64.s:101-148)
// or not a hex digit (digit_to_val gives -1, which the range test then rejects)
template <class R>
SJ_HD uint32_t hex4_at(const R& rd, uint64_t x) {
    const uint32_t c0 = rd(x), c1 = rd(x + 1), c2 = rd(x + 2), c3 = rd(x + 3);
    if (c0 == '"' || c1 == '"' || c2 == '"' || c3 == '"') return 0xffffffffu;
    const uint32_t v = ((uint32_t)digit_to_val(c0) << 12) | ((uint32_t)digit_to_val(c1) << 8) | ((uint32_t)digit_to_val(c2) << 4) |
                       (uint32_t)digit_to_val(c3);
    return v > 0xffffu ? 0xffffffffu : v;
}
// number of consecutive backslashes immediately in front of x
template <class R>
SJ_HD uint32_t backslashes_before(const R& rd, uint64_t x) {
    uint32_t k = 0;
    while (x > k && rd(x - 1 - k) == '\\') k++;
    return k;
}
// is there a "\uD8xx".."\uDBxx" escape STARTING at y (a backslash at an even offset of its run)?  Cheapest test first:
// almost every "\u" escape is preceded by something that is not a high surrogate, and its third byte says so.  `near`
// may be the shared-memory image, which earlier escapes have patched in place: they put their output at the END of
// their own bytes (esc_out_pos), so the first three bytes of a 6-byte escape -- and all of the first half of a pair --
// still read as in the message; everything beyond the quick test is read from the message itself (`far`).
template <class N, class F>
SJ_HD bool high_escape_at(const N& near, const F& far, uint64_t y) {
    const uint32_t c0 = near(y), c1 = near(y + 1), c2 = near(y + 2);
    if (c0 != '\\' || c1 != 'u' || (c2 | 0x20u) != 'd') return false;
    if (far(y) != '\\' || far(y + 1) != 'u') return false;
    const uint32_t v = hex4_at(far, y + 2);
    if (v == 0xffffffffu || (v & 0xFC00u) != 0xD800u) return false;
    return (backslashes_before(far, y) & 1u) == 0;
}

// the escape whose backslash sits at x (x is known to be an escape start).  rd(pos) returns the ORIGINAL message
// byte, 0 beyond its end.  The sequential decoder consumes a surrogate pair in one step; here the "\u" of the low
// half is an escape start of its own, recognised by walking the chain of high surrogates in front of it: it is a
// second half iff an odd number of them precede it back to back (the reference does not range-check the low half,
// so "\ud800𐀀" is pair + lone low surrogate: parse_string_amd64.s:200-229).
// rd: the escape's own bytes and the quick look at what precedes it (may be the shared-memory image, patched in place
// by the escapes in front of x -- see high_escape_at); far: the original message
template <class R, class B>
SJ_HD EscInfo esc_decode(const R& rd, const B& far, uint64_t x) {
    EscInfo r;
    r.c = 2, r.n = 1, r.bytes = 0, r.valid = true, r.second = false;
    const uint32_t e = rd(x + 1);
    if (e != 'u') {
        const uint32_t m = escape_map(e);
        r.valid = m != 0;
        r.bytes = m;
        return r;
    }
    {
        uint32_t k = 0;
        uint64_t y = x;
        while (y >= 6 && high_escape_at(rd, far, y - 6)) {
            k++;
            y -= 6;
        }
        if (k & 1u) {
            r.second = true;
            r.c = 0, r.n = 0;
            return r;
        }
    }
    r.c = 6;
    uint32_t cp = hex4_at(rd, x + 2);
    if (cp == 0xffffffffu) {
        r.valid = false;
        return r;
    }
    if ((cp & 0xFC00u) == 0xD800u) {
        if (rd(x + 6) != '\\' || rd(x + 7) != 'u') {
            r.valid = false;
            return r;
        }
        const uint32_t cp2 = hex4_at(rd, x + 8);
        if (cp2 == 0xffffffffu) {
            r.valid = false;
            return r;
        }
        cp = (((cp << 10) + 0xFCA00000u) | (cp2 + 0xFFFF2400u)) + 0x10000u;  // low surrogate range NOT checked
        r.c = 12;
    }
    uint32_t n;
    if (cp < 0x80u)
        n = 1;
    else if (cp < 0x800u)
        n = 2;
    else if (cp < 0x10000u)
        n = 3;
    else if (cp <= 0x10FFFFu)
        n = 4;
    else {
        r.valid = false;
        return r;
    }
    r.n = n;
    r.bytes = utf8_pack(cp, n);
    return r;
}

// Where the produced bytes of the escape at x live among its c source bytes (the rest is dropped from Strings.B): at
// the escape's LAST n positions -- never over the first three bytes of a 6-byte escape nor over any byte of the first
// half or the "\u" of the second half of a pair, which later escapes (and the second half itself) still look at.  When
// the escape straddles the end of its 2 KiB step, each side patches the positions that fall into its own image.
SJ_HD uint64_t esc_out_pos(uint64_t x, uint32_t c, uint32_t n) { return x + c - n; }

// ---------------------------------------------------------------------------------
// parameters / outputs
// ---------------------------------------------------------------------------------
struct NumEntry {
    uint32_t pos;   // message offset of the number's first byte
    uint32_t slot;  // its tape slot (tag word; the value goes to slot + 1)
};

struct S2sParams {
    const uint8_t* msg;       // 16-byte aligned, readable up to round_up(len, 16)
    uint64_t len;
    uint32_t ndjson;
    const uint32_t* slabpar;  // per stage-1 tile: bit w = "inside a string" in front of slab w of the tile
    uint32_t slabs_per_tile;
    uint32_t nslabs;
    SlabAgg* agg;             // [nslabs] per-slab counts (stage 1's parse mode) -> K2q, and K2r's check of its own
    const SlabAgg* pre;       // [nslabs] exclusive prefix inside the slab's group of 1024 (K2q)
    const SlabAgg* grp_pre;   // [ngroups] exclusive prefix of the groups (K2q)
    // K2r outputs
    uint64_t* tape;
    uint8_t* strings;
    uint32_t* brk_tp;         // [nb] tape slot of bracket k
    int32_t* brk_depth;       // [nb] depth in front of it
    uint8_t* brk_kind;        // [nb] T_OBJ_OPEN .. T_ARR_CLOSE, | BRK_LINKED on a close K2r has cross-linked
    uint32_t* segmask;        // [(nb + 1 + 3) / 4] one byte per bracket-to-bracket segment, preset to 0xff: bit ctx = every
                              //   structural of the segment is allowed inside a container of kind ctx
    uint32_t* rootpos;        // [records + 1] tape slot of each record's root-open word
    uint32_t* rootlink;       // [(records + 1 + 31) / 32] preset to all ones; bit r cleared: K2r has written record r's two
                              //   root words (its open and the next record's open lie in one staged step), K2f skips them.
                              //   Optional: without it K2r writes no root words and K2f writes them all
    NumEntry* numlist;        // [numbers] in document order
    uint32_t* error;          // any stage-2 failure
    uint32_t* internal;       // optional: K2r's view of a slab differs from stage 1's (an internal error, never a verdict on
                              //   the input; the parse fails through `error` as well)
    // optional: stage 1's structural positions (absolute), where the caller has them (the host emulation); K2r then also
    // checks SlabAgg::last against the bytes under the last structurals in front of each slab.  The device parse has none.
    const uint32_t* idx;
    uint32_t n_idx;
    // NDJSON shards of ONE ParsedJson (simdjson_amd64.go:82-93): this parse's tape / Strings.B are the slices that
    // start at these offsets of the whole, so every index written INTO the tape is shifted by them
    // (root / scope pointers by tape_base, string offsets by str_base); both 0 for a stand-alone parse
    uint64_t tape_base, str_base;
    const uint64_t* bases_dev;  // optional: { msg_base, tape_base, str_base } in device memory (written by the ranks' exchange
                                // on the same stream, so no host round trip sits between the two halves); overrides the two above
};
SJ_HD uint64_t s2s_tape_base(const S2sParams& p) { return p.bases_dev ? p.bases_dev[1] : p.tape_base; }
SJ_HD uint64_t s2s_str_base(const S2sParams& p) { return p.bases_dev ? p.bases_dev[2] : p.str_base; }

// per-warp working memory (shared memory on the device)
struct S2sWarpMem {
    uint8_t* src;        // [S2S_IMAGE_BYTES] two step images, 16-byte chunks XOR-swizzled inside each 64-byte block pair
    uint8_t* sstage;     // [S2S_SSTAGE_BYTES] compacted string bytes of the current step
    uint64_t* tstage;    // [S2S_TSTAGE_WORDS] K2r's tape-staging area (esc points into it)
    const uint8_t* ctab;   // [256] char_type
    const uint8_t* oktab;  // [256] transition_mask(p, c) at [p * 16 + c]
    const uint32_t* cmptab;  // [16] compress_sel(m) | popcount(m) << 16
    uint8_t* esc;            // [S2S_ESC_SCRATCH] drop map + list of a step's escapes (K2r: the tape-staging area)
};
// scratch of a step's escapes: the drop map (one bit per image byte + one word behind the step), the record of the escape
// whose output runs past the end of the step, the list of escape positions (an escape is at least two bytes long)
constexpr uint32_t S2S_ESC_CAP = S2S_STEP_BYTES / 2;
constexpr uint32_t S2S_ESC_DMAP_WORDS = S2S_STEP_BYTES / 32 + 1;
constexpr uint32_t S2S_ESC_REC_OFS = 272, S2S_ESC_LIST_OFS = 288;
constexpr uint32_t S2S_ESC_SCRATCH = S2S_ESC_LIST_OFS + 2 * (S2S_ESC_CAP + 32);  // list + one spare slot per lane, 2400 bytes
static_assert(S2S_ESC_DMAP_WORDS * 4 <= S2S_ESC_REC_OFS, "drop map fits in front of the record");
// byte offset of message byte `o` of a step inside the swizzled step image: the four 16-byte chunks of block b are
// stored at chunk slots (j ^ ((b >> 1) & 3)) -- the pattern of a 64-byte TMA swizzle -- so that lane b reading its
// chunk j (LDS.128) is bank-conflict free for every j in NATURAL order (no mask rotation afterwards)
SJ_HD uint32_t swz(uint32_t o) {
    const uint32_t b = o >> 6, j = (o >> 4) & 3;
    return (b << 6) | ((j ^ ((b >> 1) & 3)) << 4) | (o & 15);
}

// 16-entry table for the byte compaction of one 4-byte word: PRMT selector that moves the kept bytes (mask m) to the
// low end and zero-fills the rest (selector nibble 4 = byte 0 of the second operand, which is 0)
SJ_HDC uint32_t compress_sel(uint32_t m) {
    uint32_t sel = 0, k = 0;
    for (uint32_t i = 0; i < 4; i++)
        if ((m >> i) & 1) {
            sel |= i << (4 * k);
            k++;
        }
    for (; k < 4; k++) sel |= 4u << (4 * k);
    return sel;
}

}  // namespace sj
