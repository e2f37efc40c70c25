// stage2.cuh -- tape construction (unifiedMachine, stage2_build_tape_amd64.go:160-446) as a
// data-parallel pipeline over the structural positions emitted by K1.
//
// The reference walks the structurals with a goto state machine and a scope stack.  Here
// every structural is handled by its own thread:
//   K2a classify_measure  type of each structural, atom validation (stage2...go:124-158),
//                         string validate-only pass (parse_string_amd64.s:72-258)
//                         -> per-structural tape-word / bracket / string-byte / record counts
//   K2b scans             exclusive prefix sums of those counts (tile sums -> 2-level scan; stage2_common.cuh)
//   K2c emit              tape slots, parse_number (parse_number.go:65), parse_string copy
//                         (parse_string_amd64.s:260-479), bracket compaction
//   K2d ansv              nearest-smaller-depth search over the brackets = the scope stack:
//                         gives every close its open and every value its enclosing container (stage2_common.cuh)
//   K2e grammar           the state machine's transition checks, evaluated locally from
//                         (previous two structurals, enclosing container); cross-links { } [ ]
//   K2f roots             root words and NDJSON root chaining (stage2...go:190-221, 428-441)
#pragma once
#include "common.cuh"
#include "number.h"
#include "s2s_core.h"
#include "stage2_common.cuh"

namespace sj {

// structural types and the grammar (transition_ok) live in s2s_core.h, STRINGBUFBIT and the atom and escape tables
// (structural_or_ws_or_nul, digit_to_val, escape_map) in bits.h: both are shared with the streaming kernels
constexpr uint32_t AUX_COPY = 0x80000000u;              // string goes to the string buffer
constexpr uint32_t AUX_ESC = 0x40000000u;               // string contains escapes (source length != unescaped length)
constexpr uint32_t AUX_LEN = 0x3fffffffu;
constexpr int S2_ITEMS = 4;                       // consecutive structurals per thread in K2a / K2c / K2e
constexpr int S2_TILE = S2_THREADS * S2_ITEMS;     // structurals per block = granularity of the K2b scan
// Strings that need the byte-exact slow paths (escapes, or no escape-free proof from K1's backslash
// map) are handled by their own thread up to this extent and by the whole warp beyond it: one long
// string per warp would otherwise keep 31 lanes idle for hundreds of serial iterations.
constexpr uint32_t S2_COOP_MIN = 64;
// number-heavy documents get their numbers parsed by dense kernels (K2g / K2h) when numbers << SHIFT >= structurals
// (one structural in 16)
constexpr int S2_DENSE_NUMBERS_SHIFT = 4;
constexpr int S2_EMIT_MIN_BLOCKS = 8;  // K2c: resident blocks per SM the register allocation must allow (8 = 32 registers)
// Long strings with escapes: the warp routines decode all escapes of a window at once (warp_string_fast).  K2c
// (unescape): windows with fewer backslashes than this take the exact step instead of decoding every window.  K2a
// (measure) calls warp_string_fast behind a call (inlined, it changes the code of the whole kernel).
constexpr int S2_FAST_MIN_BACKSLASHES = 3;

struct ScanVal {
    uint32_t w;     // tape words
    uint32_t brk;   // brackets
    uint32_t str;   // string-buffer bytes
    uint32_t rec;   // record boundaries (effective NDJSON newlines)
    int32_t depth;  // +1 open, -1 close
};

// agg_combine / agg_shfl_up: the operations of SlabAgg (s2s_core.h) for ScanVal, so that one block scan serves both
__device__ __forceinline__ ScanVal agg_combine(const ScanVal& a, const ScanVal& b) {
    ScanVal r;
    r.w = a.w + b.w;
    r.brk = a.brk + b.brk;
    r.str = a.str + b.str;
    r.rec = a.rec + b.rec;
    r.depth = a.depth + b.depth;
    return r;
}
__device__ __forceinline__ ScanVal sv_zero() { return ScanVal{0, 0, 0, 0, 0}; }
__device__ __forceinline__ ScanVal agg_shfl_up(const ScanVal& a, int d) {
    ScanVal r;
    r.w = __shfl_up_sync(FULL, a.w, d);
    r.brk = __shfl_up_sync(FULL, a.brk, d);
    r.str = __shfl_up_sync(FULL, a.str, d);
    r.rec = __shfl_up_sync(FULL, a.rec, d);
    r.depth = __shfl_up_sync(FULL, a.depth, d);
    return r;
}

// The block scan of stage2_common.cuh for the per-structural contributions of ONE block (K2a, K2c): every field but
// `str` is tiny (w <= 2, brk, rec <= 1, depth in {-1,0,1} per structural), so four of the five
// fields travel as 16-bit lanes of one 64-bit word (depth biased by +BIAS per thread, BIAS = number
// of structurals a thread contributes) and the scan moves 3 registers per step instead of 5.
// NT * BIAS <= 8192 keeps every lane below 2^16.
template <int NT, int BIAS>
__device__ __forceinline__ ScanVal block_exclusive_scan_small(const ScanVal& v, ScanVal& total) {
    constexpr int NW = NT / 32;
    __shared__ unsigned long long wp_pk[NW + 1];
    __shared__ uint32_t wp_str[NW + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned long long own = (unsigned long long)v.w | ((unsigned long long)v.brk << 16) | ((unsigned long long)v.rec << 32) |
                                   ((unsigned long long)(uint32_t)(v.depth + BIAS) << 48);
    unsigned long long pk = own;
    uint32_t st = v.str;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long tp = __shfl_up_sync(FULL, pk, d);
        const uint32_t ts = __shfl_up_sync(FULL, st, d);
        if (lane >= d) {
            pk += tp;
            st += ts;
        }
    }
    if (lane == 31) {
        wp_pk[warp + 1] = pk;
        wp_str[warp + 1] = st;
    }
    __syncthreads();
    if (warp == 0) {
        unsigned long long a = lane < NW ? wp_pk[lane + 1] : 0ull;
        uint32_t b = lane < NW ? wp_str[lane + 1] : 0u;
#pragma unroll
        for (int d = 1; d < NW; d <<= 1) {
            const unsigned long long ta = __shfl_up_sync(FULL, a, d);
            const uint32_t tb = __shfl_up_sync(FULL, b, d);
            if (lane >= d) {
                a += ta;
                b += tb;
            }
        }
        __syncwarp();
        if (lane < NW) {
            wp_pk[lane + 1] = a;  // inclusive: sum of warps <= lane
            wp_str[lane + 1] = b;
        }
        if (lane == 0) {
            wp_pk[0] = 0;
            wp_str[0] = 0;
        }
    }
    __syncthreads();
    const unsigned long long tot = wp_pk[NW];
    total.w = (uint32_t)(tot & 0xffff);
    total.brk = (uint32_t)((tot >> 16) & 0xffff);
    total.rec = (uint32_t)((tot >> 32) & 0xffff);
    total.depth = (int32_t)(tot >> 48) - NT * BIAS;
    total.str = wp_str[NW];
    const unsigned long long ex = wp_pk[warp] + pk - own;  // exclusive prefix of this thread
    ScanVal r;
    r.w = (uint32_t)(ex & 0xffff);
    r.brk = (uint32_t)((ex >> 16) & 0xffff);
    r.rec = (uint32_t)((ex >> 32) & 0xffff);
    r.depth = (int32_t)(ex >> 48) - (int32_t)threadIdx.x * BIAS;
    r.str = wp_str[warp] + st - v.str;
    __syncthreads();  // the shared arrays may be reused by the next call
    return r;
}

// exclusive scan of one contribution per lane across the WARP only (same packing; no shared memory,
// no barrier): K2c gets the prefix in front of its 32 structurals from K2a
__device__ __forceinline__ ScanVal warp_exclusive_scan_small(const ScanVal& v) {
    const int lane = threadIdx.x & 31;
    const unsigned long long own = (unsigned long long)v.w | ((unsigned long long)v.brk << 16) | ((unsigned long long)v.rec << 32) |
                                   ((unsigned long long)(uint32_t)(v.depth + 1) << 48);
    unsigned long long pk = own;
    uint32_t st = v.str;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long tp = __shfl_up_sync(FULL, pk, d);
        const uint32_t ts = __shfl_up_sync(FULL, st, d);
        if (lane >= d) {
            pk += tp;
            st += ts;
        }
    }
    const unsigned long long ex = pk - own;
    ScanVal r;
    r.w = (uint32_t)(ex & 0xffff);
    r.brk = (uint32_t)((ex >> 16) & 0xffff);
    r.rec = (uint32_t)((ex >> 32) & 0xffff);
    r.depth = (int32_t)(ex >> 48) - lane;
    r.str = st - v.str;
    return r;
}

struct Stage2Params {
    const uint8_t* msg;
    uint64_t len;
    const uint32_t* idx;  // structural positions
    const uint32_t* bsmap;  // from K1: bit k = 64-byte block k contains a backslash
    uint32_t n;
    uint32_t ndjson, copy_strings;
    // scratch
    uint8_t* typ;        // [n]
    uint32_t* aux;       // [n] strings: dst_len | AUX_COPY
    ScanVal* tile_sum;   // [ntiles]
    ScanVal* tile_pre;   // [ntiles] exclusive within its group of 1024 tiles
    ScanVal* sub_pre;    // [ntiles * S2_TILE / 32] exclusive prefix of every 32 structurals inside their tile (K2a)
    ScanVal* grp_sum;    // [ngroups]
    ScanVal* grp_pre;    // [ngroups] exclusive
    uint32_t ntiles, ngroups;
    // brackets
    uint32_t* brk_i;     // [nb] structural index
    uint32_t* brk_tp;    // [nb] tape slot
    int32_t* brk_depth;  // [nb] depth before the bracket  (= level 0 of the min hierarchy)
    int32_t* par;        // [nb] nearest previous bracket with smaller depth (-1 none)
    int32_t* enc_after;  // [nb] innermost scope that is open right AFTER bracket k (bracket index, -1 = top level)
    uint8_t* ctx_after;  // [nb] its kind (CTX_ROOT / CTX_OBJ / CTX_ARR)
    uint32_t* rootpos;   // [records + 1] tape slot of each record's root-open word
    uint32_t* numlist;   // [n_numbers] structural index of every number, or null: numbers are parsed inline by K2c
    // outputs
    uint64_t* tape;
    uint64_t tape_cap;
    uint8_t* strings;
    uint64_t strings_cap;
    Stage2Result* result;
    // this parse as a shard of ONE ParsedJson (see S2sParams): offsets added to every index written into the tape
    uint64_t tape_base, str_base, msg_base;
    const uint64_t* bases_dev;  // optional { msg_base, tape_base, str_base } in device memory: overrides the three above
};
__device__ __forceinline__ uint64_t s2_msg_base(const Stage2Params& p) { return p.bases_dev ? p.bases_dev[0] : p.msg_base; }
__device__ __forceinline__ uint64_t s2_tape_base(const Stage2Params& p) { return p.bases_dev ? p.bases_dev[1] : p.tape_base; }
__device__ __forceinline__ uint64_t s2_str_base(const Stage2Params& p) { return p.bases_dev ? p.bases_dev[2] : p.str_base; }

// ---------------------------------------------------------------------------------
// atoms (stage2_build_tape_amd64.go:124-158, 455-476)
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool atom_ok(const uint8_t* m, uint64_t pos, uint64_t len, const char* lit, int n) {
    if (pos + n + 1 > len) return false;  // needs one byte after the literal (len(buf) >= n+1)
    for (int i = 0; i < n; i++)
        if (m[pos + i] != (uint8_t)lit[i]) return false;
    return structural_or_ws_or_nul(m[pos + n]);
}

// ---------------------------------------------------------------------------------
// strings
// ---------------------------------------------------------------------------------
struct StrCursor {
    const uint8_t* body;  // first byte after the opening quote
    uint64_t avail;       // bytes readable from body; beyond that the reference reads zeros
    __device__ __forceinline__ uint32_t at(uint64_t i) const { return i < avail ? body[i] : 0; }
};

// One \-escape starting at body[b].  The window logic of the assembly reduces to: D = distance
// from the backslash to the next raw '"' byte (looked for within 12 bytes);  \uXXXX needs
// D >= 6, a surrogate pair D >= 12 (parse_string_amd64.s:101-148,178-180).  With body[b+1] == 'u'
// that is: no raw quote among the four hex positions (digit_to_val would read it as 0), and for a
// pair none among the second four either (positions 6 and 7 must be "\u" anyway) -- so the bytes
// the decoder loads anyway are enough and no separate 12-byte search is needed.
__device__ __forceinline__ bool escape_step(const StrCursor& s, uint64_t b, uint32_t* adv, uint32_t* cp_out,
                                            uint32_t* nbytes) {
    uint32_t e = s.at(b + 1);
    if (e != 'u') {
        uint32_t m = escape_map(e);
        if (m == 0) return false;
        *cp_out = m;
        *adv = 2;
        *nbytes = 1;
        return true;
    }
    const uint32_t c2 = s.at(b + 2), c3 = s.at(b + 3), c4 = s.at(b + 4), c5 = s.at(b + 5);
    if (c2 == '"' || c3 == '"' || c4 == '"' || c5 == '"') return false;  // D < 6
    uint32_t cp = ((uint32_t)digit_to_val(c2) << 12) | ((uint32_t)digit_to_val(c3) << 8) | ((uint32_t)digit_to_val(c4) << 4) |
                  (uint32_t)digit_to_val(c5);
    uint32_t a = 6;
    if ((cp & 0xFFFFFC00u) == 0xD800u) {
        if (s.at(b + 6) != '\\' || s.at(b + 7) != 'u') return false;
        const uint32_t c8 = s.at(b + 8), c9 = s.at(b + 9), c10 = s.at(b + 10), c11 = s.at(b + 11);
        if (c8 == '"' || c9 == '"' || c10 == '"' || c11 == '"') return false;  // D < 12
        uint32_t cp2 = ((uint32_t)digit_to_val(c8) << 12) | ((uint32_t)digit_to_val(c9) << 8) |
                       ((uint32_t)digit_to_val(c10) << 4) | (uint32_t)digit_to_val(c11);
        if ((cp | cp2) > 0xFFFFu) return false;
        cp = (((cp << 10) + 0xFCA00000u) | (cp2 + 0xFFFF2400u)) + 0x10000u;  // low surrogate range NOT checked
        a = 12;
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
    else
        return false;
    *cp_out = cp;
    *adv = a;
    *nbytes = n;
    return true;
}

// _parse_string_validate_only (parse_string_amd64.s:72-258): 32-byte windows starting at p;
// the bound `p < maxStringSize` is tested when a window is left, exactly like the assembly
__device__ __forceinline__ bool string_measure(const StrCursor& s, uint64_t max_string_size, uint64_t* src_len,
                                               uint64_t* dst_len) {
    if (max_string_size == 0) return false;
    uint64_t p = 0, dl = 0;
    for (;;) {
        uint32_t j = 0, c = 0;
        for (; j < 32; j++) {
            c = s.at(p + j);
            if (c == '"' || c == '\\') break;
        }
        if (j == 32) {
            p += 32;
            dl += 32;
        } else if (c == '"') {
            *src_len = p + j;
            *dst_len = dl + j;
            return true;
        } else {
            uint32_t adv, cp, n;
            if (!escape_step(s, p + j, &adv, &cp, &n)) return false;
            dl += j + n;
            p += j + adv;
        }
        if (!(p < max_string_size)) return false;
    }
}

// _parse_string (parse_string_amd64.s:260-479) for a string that already validated.  The UTF-8 bytes of an escape are
// stored one by one here and in warp_string_fast below: packing them with utf8_pack (bits.h) changes those stores.
__device__ __forceinline__ void string_copy(const StrCursor& s, uint8_t* dst) {
    uint64_t p = 0, dl = 0;
    for (;;) {
        uint32_t c = s.at(p);
        if (c == '"') return;
        if (c != '\\') {
            dst[dl++] = (uint8_t)c;
            p++;
            continue;
        }
        uint32_t adv, cp, n;
        if (!escape_step(s, p, &adv, &cp, &n)) return;  // cannot happen after validation
        if (n == 1) {
            dst[dl++] = (uint8_t)cp;
        } else if (n == 2) {
            dst[dl++] = (uint8_t)(0xC0 + (cp >> 6));
            dst[dl++] = (uint8_t)(0x80 | (cp & 63));
        } else if (n == 3) {
            dst[dl++] = (uint8_t)(0xE0 + (cp >> 12));
            dst[dl++] = (uint8_t)(0x80 | ((cp >> 6) & 63));
            dst[dl++] = (uint8_t)(0x80 | (cp & 63));
        } else {
            dst[dl++] = (uint8_t)(0xF0 + (cp >> 18));
            dst[dl++] = (uint8_t)(0x80 | ((cp >> 12) & 63));
            dst[dl++] = (uint8_t)(0x80 | ((cp >> 6) & 63));
            dst[dl++] = (uint8_t)(0x80 | (cp & 63));
        }
        p += adv;
    }
}

// ---- string_measure executed by a whole warp for ONE string (all 32 lanes call it with
// identical arguments; control flow is warp-uniform).  The reference's assembly works on 32-byte
// windows too (parse_string_amd64.s:84-100, 272-290): a window is loaded, the first '"' or '\\' in
// it decides what happens next.  Here lane j holds byte j of the window and two ballots replace
// VPCMPEQB / VPMOVMSKB; the escape itself is decoded redundantly by every lane (same addresses:
// the loads broadcast). ----
__device__ __forceinline__ bool warp_string_measure(const StrCursor& s, uint64_t max_string_size, uint64_t* src_len,
                                                    uint64_t* dst_len) {
    if (max_string_size == 0) return false;
    const uint32_t lane = threadIdx.x & 31;
    uint64_t p = 0, dl = 0;
    for (;;) {
        const uint32_t c = s.at(p + lane);
        const uint32_t qm = __ballot_sync(FULL, c == '"'), ev = qm | __ballot_sync(FULL, c == '\\');
        if (ev == 0) {
            p += 32;
            dl += 32;
        } else {
            const uint32_t j = __ffs(ev) - 1;
            if ((qm >> j) & 1) {
                *src_len = p + j;
                *dst_len = dl + j;
                return true;
            }
            uint32_t adv, cp, n;
            if (!escape_step(s, p + j, &adv, &cp, &n)) return false;
            dl += j + n;
            p += j + adv;
        }
        if (!(p < max_string_size)) return false;
    }
}

// ---- all escapes of a 32-byte window at once.  warp_string_measure pays one window (load, two
// ballots, a redundant decode) per ESCAPE; text that is escaped character by character (twitterescaped:
// "\u30c6\u30b9\u30c8...") makes that one window per six bytes.  Here every lane decodes "the escape
// that would start at my byte" from its neighbours (shuffles), the lanes that really start one are
// found from the parity of their backslash run, and prefix counts place every output byte -- about
// the same work per window whatever the number of escapes in it.
//   * a backslash starts an escape iff it sits at an even offset in its run of backslashes (the
//     window begins at an unconsumed byte), unless it is the "\u" of the second half of a surrogate
//     pair whose first half starts six bytes earlier;
//   * only starts at lanes <= 20 are decoded (a pair needs 12 bytes); the window is consumed up to
//     the closing quote or up to the first undecoded start (>= lane 21), whichever comes first;
//   * two high surrogates six bytes apart make "which one is the second half" a chain: such a
//     window takes one exact step instead (escape_step on the window's first event, as in
//     warp_string_measure), as does nothing else.
// Returns 0 = invalid, 1 = done (src_len / dst_len set), 2 = `bound` source bytes passed without a
// closing quote (the caller lets the exact routine decide).  The exact routines above stay the
// reference: the test hook runs all versions on every input. ----
template <bool COPY, int MIN_BACKSLASHES>
__device__ __forceinline__ int warp_string_fast(const StrCursor& s, uint64_t bound, uint8_t* dst, uint64_t* src_len,
                                                uint64_t* dst_len) {
    const uint32_t lane = threadIdx.x & 31, lt = lanemask_lt();
    uint64_t p = 0, dl = 0;
    for (;;) {
        if (p >= bound) return 2;
        const uint32_t c = s.at(p + lane);
        const uint32_t bs = __ballot_sync(FULL, c == '\\'), qm = __ballot_sync(FULL, c == '"');
        if (bs == 0) {  // plain window
            const uint32_t j = qm ? __ffs(qm) - 1 : 32;
            if (COPY && lane < j) dst[dl + lane] = (uint8_t)c;
            if (qm) {
                *src_len = p + j;
                *dst_len = dl + j;
                return 1;
            }
            p += 32;
            dl += 32;
            continue;
        }
        // fewer backslashes than MIN_BACKSLASHES: the exact step (first event of the window) instead of decoding all lanes
        bool single = __popc(bs) < MIN_BACKSLASHES;
        uint32_t SP = 0, um = 0, cpu = 0, H = 0, e = 0, cp2 = 0;
        bool uok = false, isu = false, uok2 = false;
        if (!single) {  // (warp-uniform: bs is a ballot)
            // escape starts by run parity
            bool sp = false;
            if ((bs >> lane) & 1) {
                const uint32_t below = ~bs & lt;
                const uint32_t run_start = below ? 32 - __clz(below) : 0;
                sp = ((lane - run_start) & 1) == 0;
            }
            SP = __ballot_sync(FULL, sp);
            um = __ballot_sync(FULL, c == 'u');
            // "\uXXXX starting at my byte": digits from lanes +2..+5 (meaningful for lanes <= 26)
            const int32_t dv = digit_to_val(c);
            const uint32_t d2 = (uint32_t)__shfl_down_sync(FULL, dv, 2), d3 = (uint32_t)__shfl_down_sync(FULL, dv, 3),
                           d4 = (uint32_t)__shfl_down_sync(FULL, dv, 4), d5 = (uint32_t)__shfl_down_sync(FULL, dv, 5);
            cpu = (d2 << 12) | (d3 << 8) | (d4 << 4) | d5;
            const bool in5 = lane + 5 < 32;
            uok = in5 && ((qm >> ((lane + 2) & 31)) & 0xFu) == 0 && cpu <= 0xFFFFu;  // no raw quote among the digits
            isu = lane < 31 && ((um >> ((lane + 1) & 31)) & 1);
            H = __ballot_sync(FULL, sp && isu && uok && (cpu & 0xFC00u) == 0xD800u);
            e = __shfl_down_sync(FULL, c, 1);
            cp2 = __shfl_down_sync(FULL, cpu, 6);
            uok2 = __shfl_down_sync(FULL, (int)uok, 6) != 0;
        }
        if (H & (H << 6)) single = true;  // chain of high surrogates: which one is a second half is sequential
        if (single) {
            // one exact step (first event of the window), then look again
            const uint32_t ev = bs | qm, j = __ffs(ev) - 1;
            if (COPY && lane < j) dst[dl + lane] = (uint8_t)c;
            if ((qm >> j) & 1) {
                *src_len = p + j;
                *dst_len = dl + j;
                return 1;
            }
            uint32_t adv1, cp1, n1;
            if (!escape_step(s, p + j, &adv1, &cp1, &n1)) return 0;
            if (COPY && lane == 0) {
                uint8_t* o = dst + dl + j;
                if (n1 == 1) {
                    o[0] = (uint8_t)cp1;
                } else if (n1 == 2) {
                    o[0] = (uint8_t)(0xC0 + (cp1 >> 6)), o[1] = (uint8_t)(0x80 | (cp1 & 63));
                } else if (n1 == 3) {
                    o[0] = (uint8_t)(0xE0 + (cp1 >> 12)), o[1] = (uint8_t)(0x80 | ((cp1 >> 6) & 63)), o[2] = (uint8_t)(0x80 | (cp1 & 63));
                } else {
                    o[0] = (uint8_t)(0xF0 + (cp1 >> 18)), o[1] = (uint8_t)(0x80 | ((cp1 >> 12) & 63));
                    o[2] = (uint8_t)(0x80 | ((cp1 >> 6) & 63)), o[3] = (uint8_t)(0x80 | (cp1 & 63));
                }
            }
            dl += j + n1;
            p += j + adv1;
            continue;
        }
        const uint32_t real = SP & ~(H << 6);  // second halves of pairs are not starts
        const bool mine = ((real >> lane) & 1) && lane <= 20;
        uint32_t adv = 0, n = 0, outcp = 0;
        bool ok = true;
        if (mine) {
            if (!isu) {
                outcp = escape_map(e);
                ok = outcp != 0;
                adv = 2;
                n = 1;
            } else if (!uok) {
                ok = false;
                adv = 6;
                n = 1;
            } else if ((cpu & 0xFC00u) == 0xD800u) {
                adv = 12;
                n = 4;
                if (!(((bs >> (lane + 6)) & 1) && ((um >> (lane + 7)) & 1) && uok2)) {
                    ok = false;
                } else {
                    const uint32_t x = (((cpu << 10) + 0xFCA00000u) | (cp2 + 0xFFFF2400u)) + 0x10000u;  // low surrogate range NOT checked
                    if (x > 0x10FFFFu) {
                        ok = false;
                    } else {
                        outcp = x;
                        n = x < 0x80u ? 1 : x < 0x800u ? 2 : x < 0x10000u ? 3 : 4;
                    }
                }
            } else {
                adv = 6;
                outcp = cpu;
                n = cpu < 0x80u ? 1 : cpu < 0x800u ? 2 : 3;
            }
        }
        const uint32_t consumed = __reduce_or_sync(FULL, mine ? (((1u << adv) - 1u) << lane) : 0u);
        const uint32_t late = SP & ~consumed & 0xFFE00000u;  // undecoded starts (lanes >= 21)
        const uint32_t Z = late ? __ffs(late) - 1 : 32;
        const uint32_t qreal = qm & ~consumed;
        const uint32_t Q = qreal ? __ffs(qreal) - 1 : 32;
        const uint32_t E = Q < Z ? Q : Z;
        if (__ballot_sync(FULL, mine && lane < E && !ok)) return 0;
        uint32_t cnt = 0;
        if (lane < E) cnt = mine ? n : (((consumed >> lane) & 1) ? 0u : 1u);
        const uint32_t b0 = __ballot_sync(FULL, cnt & 1), b1 = __ballot_sync(FULL, cnt & 2), b2 = __ballot_sync(FULL, cnt & 4);
        if (COPY && cnt) {
            uint8_t* o = dst + dl + __popc(b0 & lt) + 2 * __popc(b1 & lt) + 4 * __popc(b2 & lt);
            if (!mine) {
                o[0] = (uint8_t)c;
            } else if (n == 1) {
                o[0] = (uint8_t)outcp;
            } else if (n == 2) {
                o[0] = (uint8_t)(0xC0 + (outcp >> 6)), o[1] = (uint8_t)(0x80 | (outcp & 63));
            } else if (n == 3) {
                o[0] = (uint8_t)(0xE0 + (outcp >> 12)), o[1] = (uint8_t)(0x80 | ((outcp >> 6) & 63)), o[2] = (uint8_t)(0x80 | (outcp & 63));
            } else {
                o[0] = (uint8_t)(0xF0 + (outcp >> 18)), o[1] = (uint8_t)(0x80 | ((outcp >> 12) & 63));
                o[2] = (uint8_t)(0x80 | ((outcp >> 6) & 63)), o[3] = (uint8_t)(0x80 | (outcp & 63));
            }
        }
        dl += __popc(b0) + 2 * __popc(b1) + 4 * __popc(b2);
        if (Q < Z) {
            *src_len = p + Q;
            *dst_len = dl;
            return 1;
        }
        p += E;
    }
}

__device__ __noinline__ int warp_string_fast_measure_call(const uint8_t* body, uint64_t avail, uint64_t bound, uint64_t* src_len,
                                                          uint64_t* dst_len) {
    const StrCursor s{body, avail};
    return warp_string_fast<false, 1>(s, bound, nullptr, src_len, dst_len);
}

// element j (runtime index) of four registers
template <typename T>
__device__ __forceinline__ T sel4(const T (&a)[4], int j) {
    return j == 0 ? a[0] : j == 1 ? a[1] : j == 2 ? a[2] : a[3];
}

// ---------------------------------------------------------------------------------
// K2a
// ---------------------------------------------------------------------------------
__device__ __forceinline__ ScanVal contribution(uint32_t t, uint32_t aux, uint32_t next_t) {
    ScanVal v = sv_zero();
    switch (t) {
    case T_OBJ_OPEN:
    case T_ARR_OPEN:
        v.w = 1;
        v.brk = 1;
        v.depth = 1;
        break;
    case T_OBJ_CLOSE:
    case T_ARR_CLOSE:
        v.w = 1;
        v.brk = 1;
        v.depth = -1;
        break;
    case T_STRING:
        v.w = 2;
        v.str = (aux & AUX_COPY) ? (aux & AUX_LEN) : 0;
        break;
    case T_NUMBER: v.w = 2; break;
    case T_TRUE:
    case T_FALSE:
    case T_NULL: v.w = 1; break;
    case T_NEWLINE:
        // the last newline of a run closes the current root and opens the next one
        // (stage2_build_tape_amd64.go:200-219); trailing newlines produce nothing
        if (next_t != T_NEWLINE && next_t != T_START) {
            v.w = 2;
            v.rec = 1;
        }
        break;
    default: break;
    }
    return v;
}

// Four consecutive structurals per thread: their positions come with one 16-byte load, their first
// bytes are in flight together, and the block scan is paid once per four.
__global__ void __launch_bounds__(S2_THREADS) s2_classify_measure_kernel(const Stage2Params p) {
    const uint32_t i0 = (blockIdx.x * S2_THREADS + threadIdx.x) * S2_ITEMS;
    uint32_t pos[S2_ITEMS], nxt[S2_ITEMS], c[S2_ITEMS];  // position, position of the next structural, first byte
    uint32_t cn = 0;                                       // first byte of the structural after the thread's last one
    if (i0 + S2_ITEMS < p.n) {
        const uint4 q = *reinterpret_cast<const uint4*>(p.idx + i0);
        pos[0] = q.x, pos[1] = q.y, pos[2] = q.z, pos[3] = q.w;
        nxt[0] = q.y, nxt[1] = q.z, nxt[2] = q.w, nxt[3] = p.idx[i0 + 4];
    } else {
#pragma unroll
        for (int j = 0; j < S2_ITEMS; j++) {
            pos[j] = i0 + j < p.n ? p.idx[i0 + j] : 0;
            nxt[j] = i0 + j + 1 < p.n ? p.idx[i0 + j + 1] : pos[j];
        }
    }
#pragma unroll
    for (int j = 0; j < S2_ITEMS; j++) c[j] = i0 + j < p.n ? p.msg[pos[j]] : 0;
    if (i0 + S2_ITEMS < p.n) cn = p.msg[nxt[S2_ITEMS - 1]];
    uint32_t typ4 = 0;
    uint32_t auxv[S2_ITEMS] = {0, 0, 0, 0};
    uint32_t coop = 0;  // bit j: string j is long and needs the byte-exact scan -> measured by the whole warp below
#pragma unroll 1
    for (int j = 0; j < S2_ITEMS; j++) {
        const uint32_t i = i0 + j;
        if (i >= p.n) break;
        const uint64_t ps = sel4(pos, j);
        const bool has_next = i + 1 < p.n;
        const uint64_t next_pos = sel4(nxt, j);
        const uint32_t ch = sel4(c, j);
        uint32_t t = T_INVALID, aux = 0;
        switch (ch) {
        case '{': t = T_OBJ_OPEN; break;
        case '[': t = T_ARR_OPEN; break;
        case '}': t = T_OBJ_CLOSE; break;
        case ']': t = T_ARR_CLOSE; break;
        case ':': t = T_COLON; break;
        case ',': t = T_COMMA; break;
        case 't': t = atom_ok(p.msg, ps, p.len, "true", 4) ? T_TRUE : T_INVALID; break;
        case 'f': t = atom_ok(p.msg, ps, p.len, "false", 5) ? T_FALSE : T_INVALID; break;
        case 'n': t = atom_ok(p.msg, ps, p.len, "null", 4) ? T_NULL : T_INVALID; break;
        case '\n': t = p.ndjson ? T_NEWLINE : T_INVALID; break;
        case '"': {
            uint64_t sl = 0, dl = 0;
            bool ok = false, fast = false;
            if (has_next) {
                // Stage 1 succeeded, so the string closes before the next structural and only
                // whitespace separates its closing quote from that structural: the quote is the
                // last non-blank byte in front of it.  With no backslash in the blocks the body
                // touches (K1's per-block map) nothing needs scanning: src_len == dst_len.
                uint64_t e = next_pos - 1;
                while (e > ps) {
                    uint32_t ce = p.msg[e];
                    if (!(ce == 0x20 || ce == 0x0a || ce == 0x09 || ce == 0x0d)) break;
                    e--;
                }
                if (e > ps && p.msg[e] == '"') {
                    // any backslash block among blocks [b0, b1] of K1's map?  (one word in practice)
                    const uint32_t b0 = (uint32_t)((ps + 1) >> 6), b1 = (uint32_t)(e >> 6);
                    uint32_t hit = 0;
                    for (uint32_t wd = b0 >> 5; wd <= (b1 >> 5) && !hit; wd++) {
                        const uint32_t lo_bit = wd == (b0 >> 5) ? (b0 & 31) : 0, hi_bit = wd == (b1 >> 5) ? (b1 & 31) : 31;
                        hit = p.bsmap[wd] & ((0xffffffffu >> (31 - hi_bit)) & (0xffffffffu << lo_bit));
                    }
                    fast = hit == 0;
                    if (fast) {
                        sl = dl = e - ps - 1;
                        ok = true;
                    }
                }
            }
            if (!fast) {
                // peekSize: distance to the next structural, 0 when there is none (stage2...go:63-70)
                if (next_pos - ps >= S2_COOP_MIN) {
                    coop |= 1u << j;
                } else {
                    StrCursor sc{p.msg + ps + 1, p.len - ps - 1};
                    ok = string_measure(sc, next_pos - ps, &sl, &dl);
                }
            }
            if (ok) {
                t = T_STRING;
                aux = (uint32_t)dl | ((p.copy_strings || sl != dl) ? AUX_COPY : 0) |  // parse_string_amd64.go:40
                      (sl != dl ? AUX_ESC : 0);
            }
            break;
        }
        default:
            if (ch == '-' || (ch - '0') <= 9u) t = T_NUMBER;
            break;
        }
        typ4 |= t << (8 * j);
        if (j == 0) auxv[0] = aux; else if (j == 1) auxv[1] = aux; else if (j == 2) auxv[2] = aux; else auxv[3] = aux;
    }
    // long strings left over: one at a time, 32 bytes per step, by the whole warp (every thread of the
    // block gets here, so the full-mask ballots are safe)
#pragma unroll
    for (int j = 0; j < S2_ITEMS; j++) {
        uint32_t m = __ballot_sync(FULL, (coop >> j) & 1);
        while (m) {
            const int owner = __ffs(m) - 1;
            m &= m - 1;
            const uint64_t ps = __shfl_sync(FULL, pos[j], owner), next_pos = __shfl_sync(FULL, nxt[j], owner);
            const StrCursor sc{p.msg + ps + 1, p.len - ps - 1};
            uint64_t sl = 0, dl = 0;
            // the fast routine has no per-step bound test: its answer stands when the string closes inside the
            // bound (every step of the exact routine then starts below it); anything else the exact one decides
            const int r = warp_string_fast_measure_call(sc.body, sc.avail, next_pos - ps, &sl, &dl);
            bool ok = r == 1;
            if (r == 2 || (r == 1 && sl >= next_pos - ps)) ok = warp_string_measure(sc, next_pos - ps, &sl, &dl);
            if (ok && (int)(threadIdx.x & 31) == owner) {
                typ4 |= (uint32_t)T_STRING << (8 * j);  // was T_INVALID
                auxv[j] = (uint32_t)dl | ((p.copy_strings || sl != dl) ? AUX_COPY : 0) | (sl != dl ? AUX_ESC : 0);
            }
        }
    }
    ScanVal v = sv_zero();
#pragma unroll
    for (int j = 0; j < S2_ITEMS; j++) {
        const uint32_t i = i0 + j;
        if (i < p.n) {
            uint32_t next_t = T_START;  // only "newline or not" matters
            if (i + 1 < p.n) next_t = (j + 1 < S2_ITEMS ? c[(j + 1) & 3] : cn) == '\n' ? T_NEWLINE : T_INVALID;
            v = agg_combine(v, contribution((typ4 >> (8 * j)) & 0xff, auxv[j], next_t));
        }
    }
    if (i0 + S2_ITEMS <= p.n) {
        *reinterpret_cast<uint32_t*>(p.typ + i0) = typ4;
        *reinterpret_cast<uint4*>(p.aux + i0) = make_uint4(auxv[0], auxv[1], auxv[2], auxv[3]);
    } else {
#pragma unroll
        for (int j = 0; j < S2_ITEMS; j++)
            if (i0 + j < p.n) {
                p.typ[i0 + j] = (uint8_t)(typ4 >> (8 * j));
                p.aux[i0 + j] = auxv[j];
            }
    }
    // numbers of the block (decides whether they get their own dense kernel, K2g / K2h)
    __shared__ uint32_t s_nnum[S2_THREADS / 32];
    {
        uint32_t nnum = 0;
#pragma unroll
        for (int j = 0; j < S2_ITEMS; j++) nnum += ((typ4 >> (8 * j)) & 0xff) == T_NUMBER ? 1u : 0u;
        nnum = __reduce_add_sync(FULL, nnum);
        if ((threadIdx.x & 31) == 0) s_nnum[threadIdx.x >> 5] = nnum;
    }
    ScanVal total;
    const ScanVal ex = block_exclusive_scan_small<S2_THREADS, S2_ITEMS>(v, total);  // (its barriers publish s_nnum)
    if (threadIdx.x == 0) {
        uint32_t nn = 0;
#pragma unroll
        for (int w = 0; w < S2_THREADS / 32; w++) nn += s_nnum[w];
        if (nn) atomicAdd(&p.result->n_numbers, nn);
    }
    if (threadIdx.x == 0) p.tile_sum[blockIdx.x] = total;
    // K2c works warp by warp (32 structurals = 8 threads here): their prefix inside the tile
    if ((threadIdx.x & (32 / S2_ITEMS - 1)) == 0) p.sub_pre[i0 >> 5] = ex;
}

// ---------------------------------------------------------------------------------
// K2c
// ---------------------------------------------------------------------------------
// One structural per thread, warps independent of each other: with four structurals per thread the
// tape stores of a warp spread over 32 sectors.
__global__ void __launch_bounds__(S2_THREADS, S2_EMIT_MIN_BLOCKS) s2_emit_kernel(const Stage2Params p) {  // 8 blocks per SM = 32 registers: the kernel hides its load latency with occupancy
    const uint32_t i = blockIdx.x * S2_THREADS + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    uint32_t t = T_INVALID, aux = 0;
    ScanVal v = sv_zero();
    uint64_t pos = 0;
    // every global load of the thread is issued up front, in front of the scan's barriers
    if (i < p.n) {
        t = p.typ[i];
        aux = p.aux[i];
        pos = p.idx[i];
        uint32_t next_t = i + 1 < p.n ? p.typ[i + 1] : (uint32_t)T_START;
        v = contribution(t, aux, next_t);
    }
    // prefix in front of the warp's 32 structurals: K2b's tile prefix + K2a's prefix inside the tile;
    // the rest is a warp scan -- no shared memory, no barrier in this kernel
    const uint32_t tile = i / S2_TILE;
    const ScanVal blk = agg_combine(p.sub_pre[i >> 5], agg_combine(p.tile_pre[tile], p.grp_pre[tile >> 10]));
    ScanVal e = agg_combine(warp_exclusive_scan_small(v), blk);
    const uint64_t tp = 1 + (uint64_t)e.w;  // slot 0 is the first root word
    bool live = i < p.n;
    if (live && tp + v.w > p.tape_cap) {
        if (v.w) atomicOr(&p.result->overflow, 1u);
        live = false;
    }
    uint32_t fast_len = 0;  // escape-free string to be copied by the whole warp below
    bool coop_esc = false;  // long string with escapes: parse_string by the whole warp below
    if (live) {
        switch (t) {
        case T_OBJ_OPEN:
        case T_ARR_OPEN:
        case T_OBJ_CLOSE:
        case T_ARR_CLOSE:
            p.brk_i[e.brk] = i;
            p.brk_tp[e.brk] = (uint32_t)tp;
            p.brk_depth[e.brk] = e.depth;
            // the bracket itself (no need to re-read the message); payload cross-linked by K2e
            p.tape[tp] = (uint64_t)(t == T_OBJ_OPEN ? '{' : t == T_ARR_OPEN ? '[' : t == T_OBJ_CLOSE ? '}' : ']') << 56;
            break;
        case T_STRING: {
            const uint32_t dl = aux & AUX_LEN;
            if (aux & AUX_COPY) {
                p.tape[tp] = ((uint64_t)'"' << 56) | (STRINGBUFBIT + s2_str_base(p) + e.str);
                if ((uint64_t)e.str + dl <= p.strings_cap) {
                    if (aux & AUX_ESC) {
                        if (dl >= S2_COOP_MIN) {
                            coop_esc = true;  // unescaped by the whole warp below
                        } else {
                            StrCursor s{p.msg + pos + 1, p.len - pos - 1};
                            string_copy(s, p.strings + e.str);
                        }
                    } else {
                        fast_len = dl;  // copied by the warp below
                    }
                } else {
                    atomicOr(&p.result->overflow, 1u);
                }
            } else {
                p.tape[tp] = ((uint64_t)'"' << 56) | (s2_msg_base(p) + pos + 1);  // stage2...go:90-92
            }
            p.tape[tp + 1] = dl;
            break;
        }
        case T_NUMBER: {
            if (p.numlist) {  // number-heavy document: parsed by K2h in dense warps; leave the tape slot behind
                p.aux[i] = (uint32_t)tp;
                break;
            }
            uint64_t val = 0;
            uint64_t tag = parse_number(p.msg + pos, p.len - pos, &val);
            if (tag == 0) atomicOr(&p.result->error, 1u);
            p.tape[tp] = tag;
            p.tape[tp + 1] = val;
            break;
        }
        case T_TRUE: p.tape[tp] = (uint64_t)'t' << 56; break;
        case T_FALSE: p.tape[tp] = (uint64_t)'f' << 56; break;
        case T_NULL: p.tape[tp] = (uint64_t)'n' << 56; break;
        case T_NEWLINE:
            if (v.rec) p.rootpos[e.rec + 1] = (uint32_t)tp + 1;  // the new record's root-open slot
            break;
        default: break;
        }
    }
    else if (i < p.n && t == T_NUMBER && p.numlist) {
        p.aux[i] = 0xffffffffu;  // no room on the tape: K2h skips it
    }
    // ---- warp-cooperative copy of the warp's escape-free strings.  A string's own thread would copy
    // it byte by byte (one LSU transaction per byte and lane, trip count = the longest string of the
    // warp).  Instead the strings are queued in shared memory; strings of up to 32 bytes are copied
    // by groups of 8 lanes (four strings at a time, 8 consecutive bytes per group and step), longer
    // ones by the whole warp one after another (32 consecutive bytes per step). ----
    __shared__ uint4 s_q[S2_THREADS];
    uint4* q = s_q + (threadIdx.x & ~31u);
    const uint32_t shortm = __ballot_sync(FULL, fast_len != 0 && fast_len <= 32);
    const uint32_t longm = __ballot_sync(FULL, fast_len > 32);
    if (shortm | longm) {
        if (fast_len != 0 && fast_len <= 32) q[__popc(shortm & lanemask_lt())] = make_uint4((uint32_t)pos + 1, e.str, fast_len, 0);
        __syncwarp();
        const uint32_t ns = __popc(shortm), g = lane >> 3, b = lane & 7;
        for (uint32_t r = g; r < ns; r += 4) {
            const uint4 d = q[r];
            const uint8_t* src = p.msg + d.x;
            uint8_t* dst = p.strings + d.y;
#pragma unroll
            for (uint32_t o = 0; o < 32; o += 8)  // (a loop bounded by the length was measured: no difference)
                if (o + b < d.z) dst[o + b] = src[o + b];
        }
        uint32_t m = longm;
        while (m) {
            const int src_lane = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t sp = __shfl_sync(FULL, (uint32_t)pos + 1, src_lane), dp = __shfl_sync(FULL, e.str, src_lane),
                           ln = __shfl_sync(FULL, fast_len, src_lane);
            const uint8_t* src = p.msg + sp;
            uint8_t* dst = p.strings + dp;
            for (uint32_t o = lane; o < ln; o += 32) dst[o] = src[o];
        }
    }
    // ---- long strings with escapes: one at a time, 32 source bytes per step (parse_string_amd64.s:260-479) ----
    uint32_t em = __ballot_sync(FULL, coop_esc);
    while (em) {
        const int owner = __ffs(em) - 1;
        em &= em - 1;
        const uint64_t sp = __shfl_sync(FULL, (uint32_t)pos, owner);
        const uint32_t dp = __shfl_sync(FULL, e.str, owner);
        const StrCursor s{p.msg + sp + 1, p.len - sp - 1};
        uint64_t sl_unused, dl_unused;
        warp_string_fast<true, S2_FAST_MIN_BACKSLASHES>(s, ~0ull, p.strings + dp, &sl_unused, &dl_unused);  // validated by K2a
    }
}

// ---------------------------------------------------------------------------------
// K2g / K2h: numbers in dense warps.  In a number-heavy document (canada.json: every third
// structural) K2c's warps run parse_number with a third of their lanes.  K2g compacts the structural
// indexes of the numbers (one atomic per block; the order of the list is irrelevant, every entry
// carries its own tape slot in aux[]), K2h parses one number per thread with all lanes busy.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) s2_numlist_kernel(const Stage2Params p, uint32_t cap) {
    __shared__ uint32_t s_cnt[32];
    __shared__ uint32_t s_base;
    const uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool is_num = i < p.n && p.typ[i] == T_NUMBER;
    const uint32_t m = __ballot_sync(FULL, is_num);
    if (lane == 0) s_cnt[warp] = __popc(m);
    __syncthreads();
    if (warp == 0) {
        const uint32_t own = s_cnt[lane];
        uint32_t inc = own;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, inc, d);
            if (lane >= (uint32_t)d) inc += t;
        }
        s_cnt[lane] = inc - own;  // exclusive prefix of the warp counts
        if (lane == 31) s_base = inc ? atomicAdd(&p.result->num_fill, inc) : 0u;
    }
    __syncthreads();
    if (is_num) {
        const uint32_t slot = s_base + s_cnt[warp] + __popc(m & lanemask_lt());
        if (slot < cap) p.numlist[slot] = i;
    }
}

__global__ void __launch_bounds__(S2_THREADS) s2_numbers_kernel(const Stage2Params p, uint32_t count) {
    const uint32_t k = blockIdx.x * S2_THREADS + threadIdx.x;
    if (k >= count) return;
    const uint32_t i = p.numlist[k];
    const uint32_t tp = p.aux[i];
    if (tp == 0xffffffffu) return;
    const uint64_t pos = p.idx[i];
    uint64_t val = 0;
    const uint64_t tag = parse_number(p.msg + pos, p.len - pos, &val);  // parse_number.go:65
    if (tag == 0) atomicOr(&p.result->error, 1u);
    p.tape[tp] = tag;
    p.tape[tp + 1] = val;
}

// ---------------------------------------------------------------------------------
// K2e: grammar (the state machine's transitions) and bracket cross-links
// ---------------------------------------------------------------------------------
// transition_ok as a bit table, built at compile time: the previous-previous structural only
// matters as "was the string before us a key" (pp is '{' or ','), so the index is
// ((ctx * 2 + is_key) * 14 + p) * 14 + c  -- 1176 bits.  K2e copies it to shared memory and replaces
// ~100 branchy instructions per structural by one LDS.
constexpr uint32_t TRANS_NT = 14;  // T_INVALID .. T_START
constexpr uint32_t TRANS_WORDS = (3 * 2 * TRANS_NT * TRANS_NT + 31) / 32;
struct TransTable {
    uint32_t w[TRANS_WORDS];
};
__host__ __device__ constexpr uint32_t trans_index(uint32_t ctx, uint32_t is_key, uint32_t p, uint32_t c) {
    return ((ctx * 2 + is_key) * TRANS_NT + p) * TRANS_NT + c;
}
constexpr TransTable make_trans_table() {
    TransTable t{};
    for (uint32_t ctx = 0; ctx < 3; ctx++)
        for (uint32_t k = 0; k < 2; k++)
            for (uint32_t p = 0; p < TRANS_NT; p++)
                for (uint32_t c = 0; c < TRANS_NT; c++)
                    if (transition_ok(ctx, k ? (uint32_t)T_COMMA : (uint32_t)T_INVALID, p, c)) {
                        const uint32_t i = trans_index(ctx, k, p, c);
                        t.w[i >> 5] |= 1u << (i & 31);
                    }
    return t;
}
__constant__ TransTable c_trans = make_trans_table();

// Scope that is open right after each bracket: one thread per BRACKET does the pointer chase
// (bracket -> its open -> that open's parent) once, so that K2e -- one thread per structural, 10-40x
// more threads -- needs a single load of the result instead of a chain of five dependent ones.
__global__ void __launch_bounds__(S2_THREADS) s2_scope_kernel(const Stage2Params p, uint32_t nb) {
    const uint32_t k = blockIdx.x * S2_THREADS + threadIdx.x;
    if (k >= nb) return;
    const uint32_t bt = p.typ[p.brk_i[k]];
    int32_t enc;
    if (bt == T_OBJ_OPEN || bt == T_ARR_OPEN) {
        enc = (int32_t)k;
    } else {
        const int32_t m = p.par[k];  // the close's open
        enc = m >= 0 ? p.par[m] : -1;
    }
    p.enc_after[k] = enc;
    p.ctx_after[k] = enc >= 0 ? (p.typ[p.brk_i[enc]] == T_OBJ_OPEN ? CTX_OBJ : CTX_ARR) : CTX_ROOT;
}

// Four consecutive structurals per thread (the per-structural work is a handful of instructions
// behind two dependent loads, so one structural per thread is latency-bound): a block covers
// S2_TILE structurals = one K2b tile.
constexpr int S2E_ITEMS = S2_ITEMS;
__global__ void __launch_bounds__(S2_THREADS) s2_grammar_kernel(const Stage2Params p) {
    __shared__ uint32_t s_wcnt[S2_THREADS / 32];
    __shared__ uint32_t s_tr[TRANS_WORDS];
    if (threadIdx.x < TRANS_WORDS) s_tr[threadIdx.x] = c_trans.w[threadIdx.x];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t i0 = (blockIdx.x * S2_THREADS + threadIdx.x) * S2E_ITEMS;
    // types of the thread's structurals and of the two in front of them
    uint32_t c[S2E_ITEMS];
    if (i0 + S2E_ITEMS <= p.n) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(p.typ + i0);
#pragma unroll
        for (int j = 0; j < S2E_ITEMS; j++) c[j] = (w >> (8 * j)) & 0xff;
    } else {
#pragma unroll
        for (int j = 0; j < S2E_ITEMS; j++) c[j] = i0 + j < p.n ? p.typ[i0 + j] : (uint32_t)T_INVALID;
    }
    uint32_t pv = T_START, ppv = T_START;
    if (i0 >= 1 && i0 < p.n) pv = p.typ[i0 - 1];
    if (i0 >= 2 && i0 < p.n) ppv = p.typ[i0 - 2];
    // brackets of the tile in front of each structural: K2b's tile prefix + the other warp of the
    // tile + lower lanes of this warp + the thread's own earlier structurals
    uint32_t nbrk = 0;
#pragma unroll
    for (int j = 0; j < S2E_ITEMS; j++) nbrk += (c[j] >= T_OBJ_OPEN && c[j] <= T_ARR_CLOSE) ? 1u : 0u;
    const uint32_t b0 = __ballot_sync(FULL, nbrk & 1), b1 = __ballot_sync(FULL, nbrk & 2), b2 = __ballot_sync(FULL, nbrk & 4);
    const uint32_t lt = lanemask_lt();
    uint32_t before = __popc(b0 & lt) + 2 * __popc(b1 & lt) + 4 * __popc(b2 & lt);
    if (lane == 0) s_wcnt[warp] = __popc(b0) + 2 * __popc(b1) + 4 * __popc(b2);
    __syncthreads();
    if (i0 >= p.n) return;
#pragma unroll
    for (int w2 = 0; w2 < S2_THREADS / 32; w2++)
        if (w2 < (int)warp) before += s_wcnt[w2];
    const uint32_t tile = blockIdx.x;  // a block = one K2b tile of S2_TILE structurals
    before += p.tile_pre[tile].brk + p.grp_pre[tile >> 10].brk;
#pragma unroll
    for (int j = 0; j < S2E_ITEMS; j++) {
        const uint32_t i = i0 + j;
        if (i >= p.n) break;
        const uint32_t cj = c[j];
        const uint32_t k = before - 1;  // nearest bracket strictly before i; 0xffffffff when none
        // the scope this structural sits in = the scope open after the previous bracket (for a closing
        // bracket that is the scope it closes: its open is the nearest bracket of smaller depth)
        uint32_t ctx = CTX_ROOT;
        if (k != 0xffffffffu) ctx = p.ctx_after[k];
        const uint32_t ti = trans_index(ctx, (ppv == T_OBJ_OPEN || ppv == T_COMMA) ? 1u : 0u, pv, cj);
        if (!((s_tr[ti >> 5] >> (ti & 31)) & 1)) {  // transition_ok(ctx, ppv, pv, c)
            atomicOr(&p.result->error, 1u);
        } else if (cj == T_OBJ_CLOSE || cj == T_ARR_CLOSE) {  // scopeEnd, stage2...go:327-334
            const int32_t enclosing = p.enc_after[k];  // k exists: a close cannot follow T_START in a valid transition
            const uint32_t open_tp = p.brk_tp[enclosing], close_tp = p.brk_tp[k + 1];
            if (close_tp < p.tape_cap) {
                p.tape[open_tp] = ((uint64_t)(cj == T_OBJ_CLOSE ? '{' : '[') << 56) | (s2_tape_base(p) + close_tp + 1);
                p.tape[close_tp] = ((uint64_t)(cj == T_OBJ_CLOSE ? '}' : ']') << 56) | (s2_tape_base(p) + open_tp);
            }
        }
        if (cj >= T_OBJ_OPEN && cj <= T_ARR_CLOSE) before++;
        ppv = pv;
        pv = cj;
    }
}

// ---------------------------------------------------------------------------------
// K2f: root words.  Record r opens at rootpos[r]; its close sits right before the next
// record's open (or is the last word of the tape).  stage2...go:170,207-218,428-441
// (s2s_link_kernel writes the same words for the streaming path, bounded by tape_len instead of tape_cap)
// ---------------------------------------------------------------------------------
__global__ void s2_roots_kernel(const Stage2Params p, uint64_t n_records, uint64_t tape_len) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_records) return;
    const uint64_t R = (uint64_t)'r' << 56;
    const uint64_t open = r == 0 ? 0 : p.rootpos[r];
    const uint64_t next_open = r == n_records ? tape_len : p.rootpos[r + 1];
    if (next_open > p.tape_cap || next_open == 0) return;
    p.tape[open] = R | (s2_tape_base(p) + next_open);
    p.tape[next_open - 1] = R | (s2_tape_base(p) + open);
}

}  // namespace sj
