// s2s_slab.h -- streaming stage 2: what ONE WARP does with one 6 KiB slab, written once for the device (W = DevWarp,
// stage2_stream.cuh) and for the host emulation (W = FiberWarp, tests/emu/s2s_emu.cpp).  See s2s_core.h for the idea.
//
//   s2s_slab<W, false>   counts of the slab -> SlabAgg (the emulator's counting pass; on the device stage 1's parse mode
//                        counts, with step_events / agg_lane_add / agg_warp_finish below)
//   s2s_slab<W, true>    K2r: tape words, Strings.B bytes, bracket records, number list, grammar masks
//
// W provides: lane(), ballot(bool), any(bool), shfl / shfl_up (uint32_t), reduce_add(uint32_t), sync(),
// atomic_and(uint32_t*, uint32_t), atomic_or(uint32_t*, uint32_t), atomic_or_shared(uint32_t*, uint32_t).
// Every collective is reached by all 32 lanes (warp-uniform control flow around them).
#pragma once
#include "s2s_core.h"

namespace sj {

// K2r's section probe (tools/k2r_probe.py builds it; the product build does not define SJ_K2R_PROBE): a clock64()
// stamp at each section boundary of the slab loop, the per-slab sums added into sj_k2r_probe_cycles once per slab.
// The stamps cost time themselves, so the sums are for shares, not for K2r's time.
enum : uint32_t {
    K2R_PROLOGUE,   // slab prologue: carries, prefixes, pre-types
    K2R_IMAGE,      // image pipeline: issue the next step, wait for this one
    K2R_CLASSIFY,   // classify, escape starts, quote mask, escapes
    K2R_EVENTS,     // step_events and the scans of the step
    K2R_STRINGS,    // Strings.B compaction and copy-out
    K2R_GRAMMAR,    // pre-types and the grammar masks
    K2R_EMIT,       // emission loops
    K2R_LINK,       // in-step links and tape copy-out
    K2R_SECTIONS
};
#if defined(SJ_K2R_PROBE) && defined(__CUDACC__)
__device__ unsigned long long sj_k2r_probe_cycles[K2R_SECTIONS];
#endif
#if defined(SJ_K2R_PROBE) && defined(__CUDA_ARCH__)
// (lane k keeps the sum of section k: three registers in all)
#define K2R_PROBE_START        \
    uint32_t probe_acc = 0;    \
    long long probe_t = clock64();
#define K2R_PROBE(sec)                                        \
    do {                                                      \
        __syncwarp();                                         \
        const long long t_ = clock64();                       \
        if (lane == (sec)) probe_acc += (uint32_t)(t_ - probe_t); \
        probe_t = t_;                                         \
    } while (0)
#define K2R_PROBE_FLUSH                                                                          \
    do {                                                                                         \
        if (lane < K2R_SECTIONS) atomicAdd(&sj_k2r_probe_cycles[lane], (unsigned long long)probe_acc); \
    } while (0)
#else
#define K2R_PROBE_START
#define K2R_PROBE(sec) \
    do {               \
    } while (0)
#define K2R_PROBE_FLUSH \
    do {                \
    } while (0)
#endif

template <bool B>
struct BoolC {
    static constexpr bool value = B;
};

// original message bytes: the slab image in shared memory where it covers the position, global memory elsewhere,
// 0 beyond the end of the message (the reference reads zero padding there, stage2...go:75-86)
struct MsgReader {
    const uint8_t* msg;
    uint64_t len;
    const uint8_t* src;   // image of the current step (swizzled)
    uint64_t slab_start;  // message range the image holds: [slab_start, slab_end)
    uint64_t slab_end;
    SJ_HD uint32_t operator()(uint64_t pos) const {
        if (pos >= slab_start && pos < slab_end) return src[swz((uint32_t)(pos - slab_start))];
        return pos < len ? msg[pos] : 0u;
    }
};

// the same with 32-bit arithmetic on the hot path (messages are shorter than 2 GiB, so the low words decide)
struct ImageReader {
    const uint8_t* src;
    uint32_t start_lo;  // low word of the message offset the image starts at
    uint32_t win;       // message bytes the image holds
    const uint8_t* msg;
    uint64_t len;
    SJ_HD uint32_t operator()(uint64_t pos) const {
        const uint32_t d = (uint32_t)pos - start_lo;
        if (d < win) return src[swz(d)];
        return pos < len ? msg[pos] : 0u;
    }
};

struct GlobalReader {
    const uint8_t* msg;
    uint64_t len;
    SJ_HD uint32_t operator()(uint64_t pos) const { return pos < len ? msg[pos] : 0u; }
};

// atoms (stage2_build_tape_amd64.go:124-158, 455-476): literal + one following byte that is structural / white / NUL
template <class R>
SJ_HD bool atom_ok_p(const R& rd, uint64_t pos, uint64_t len, uint32_t type) {
    const char* lit = type == T_TRUE ? "true" : type == T_FALSE ? "false" : "null";
    const uint32_t n = type == T_FALSE ? 5 : 4;
    if (pos + n + 1 > len) return false;  // len(buf) >= n + 1
    for (uint32_t i = 0; i < n; i++)
        if (rd(pos + i) != (uint32_t)(uint8_t)lit[i]) return false;
    return structural_or_ws_or_nul(rd(pos + n));
}

// The same test for an atom that lies, with the byte behind it and then some, inside the step image (o + 8 <= avail):
// three aligned words, two funnel shifts, word compares; the byte behind the literal is looked up in a 128-bit set.
// Returns false when it does not apply (atom_ok_p is the definition); *ch = the atom's first byte.
SJ_HD bool atom_ok_fast(const uint8_t* img, uint32_t o, uint32_t avail, uint32_t* ch, bool* ok) {
    if (o + 8 > avail) return false;
    const uint32_t a = o & ~3u, sh = 8 * (o & 3u);
    const uint32_t a2 = a + 8 < S2S_STEP_BYTES ? a + 8 : a + 4;  // (the third word only matters when sh != 0, and then it is inside)
    const uint32_t w0 = *reinterpret_cast<const uint32_t*>(img + swz(a)), w1 = *reinterpret_cast<const uint32_t*>(img + swz(a + 4));
    const uint32_t w2 = *reinterpret_cast<const uint32_t*>(img + swz(a2));
    const uint32_t q0 = pi::funnel_r(w0, w1, sh), q1 = pi::funnel_r(w1, w2, sh);
    const uint32_t c = q0 & 0xffu;
    *ch = c;
    uint32_t follow;
    bool lit;
    if (c == 't') {
        lit = q0 == 0x65757274u, follow = q1 & 0xffu;
    } else if (c == 'n') {
        lit = q0 == 0x6c6c756eu, follow = q1 & 0xffu;
    } else if (c == 'f') {
        lit = q0 == 0x736c6166u && (q1 & 0xffu) == 'e', follow = (q1 >> 8) & 0xffu;
    } else {
        return false;
    }
    // NUL \t \n \r | space , : | [ ] | { }   (structural_or_ws_or_nul)
    const uint32_t set = follow < 32 ? 0x00002601u : follow < 64 ? 0x04001001u : follow < 96 ? 0x28000000u : 0x28000000u;
    *ok = lit && follow < 128 && ((set >> (follow & 31u)) & 1u) != 0;
    return true;
}

// esc_decode for the common case -- "\\uXXXX" with four proper hex digits, not a surrogate, and nothing that looks like a
// high surrogate six bytes in front of it -- straight from the step image with word accesses and register arithmetic
// only: four aligned words cover the twelve bytes [o - 6, o + 6), funnel shifts align them, the hex digits are checked
// and converted four at a time (SWAR).  No table look-ups: going through the 256-entry tables costs two dependent
// shared-memory loads per digit in a kernel that is bound by dependent latencies.  Returns false when it does not apply; esc_decode (s2s_core.h) is the definition and
// takes those cases -- including every digit quirk of parse_string_amd64.s:4-69, which is why only proper digits pass here.
//   o: offset of the backslash in the image; avail: image bytes that are message bytes
//   at: where image offset o lives (SwzLayout: K2r's swizzled step image; FlatLayout: stage 1's tile buffer)
struct SwzLayout {
    SJ_HD uint32_t operator()(uint32_t o) const { return swz(o); }
};
struct FlatLayout {
    SJ_HD uint32_t operator()(uint32_t o) const { return o; }
};
template <class A = SwzLayout>
SJ_HD bool esc_u_fast(const uint8_t* img, uint32_t o, uint32_t avail, EscInfo& r, A at = A()) {
    if (o < 6 || o + 6 > avail) return false;
    const uint32_t a = (o - 6) & ~3u, sh = 8 * ((o - 6) & 3u);
    const uint32_t a3 = a + 12 < S2S_STEP_BYTES ? a + 12 : a + 8;  // (the fourth word only matters when sh != 0, and then it is inside)
    const uint32_t w0 = *reinterpret_cast<const uint32_t*>(img + at(a)), w1 = *reinterpret_cast<const uint32_t*>(img + at(a + 4));
    const uint32_t w2 = *reinterpret_cast<const uint32_t*>(img + at(a + 8)), w3 = *reinterpret_cast<const uint32_t*>(img + at(a3));
    const uint32_t q0 = pi::funnel_r(w0, w1, sh), q1 = pi::funnel_r(w1, w2, sh), x = pi::funnel_r(w2, w3, sh);
    // q0 = bytes o-6 .. o-3, q1 = o-2 .. o+1, x = o+2 .. o+5 (the digits)
    if ((q1 >> 24) != 'u') return false;
    if ((q0 & 0x00DFFFFFu) == 0x0044755Cu) return false;  // "\\uD" / "\\ud" six bytes in front: perhaps the first half of a pair
    // bytes are proper hex digits: '0'..'9' (tested on x), 'A'..'F' / 'a'..'f' (tested on x | 0x20); every byte < 0x80,
    // so the per-byte additions do not carry into their neighbours (a byte >= 0x80 fails through ~x)
    const uint32_t l = x | 0x20202020u;
    const uint32_t isdig = (x + 0x50505050u) & ~(x + 0x46464646u);
    const uint32_t isalp = (l + 0x1f1f1f1fu) & ~(l + 0x19191919u);
    if ((((isdig | isalp) & ~x) & 0x80808080u) != 0x80808080u) return false;
    const uint32_t v = (x & 0x0f0f0f0fu) + 9u * ((x >> 6) & 0x01010101u);  // digit values, first digit in byte 0
    const uint32_t rv = pi::byte_perm(v, 0, 0x0123);                        // first digit in byte 3
    const uint32_t pr = (rv | (rv >> 4)) & 0x00ff00ffu;
    const uint32_t cp = (pr | (pr >> 8)) & 0xffffu;
    if ((cp & 0xF800u) == 0xD800u) return false;  // surrogates: the pair rules
    r.c = 6;
    r.n = cp < 0x80u ? 1u : cp < 0x800u ? 2u : 3u;
    r.bytes = utf8_pack(cp, r.n);
    r.valid = true;
    r.second = false;
    return true;
}

// What an escape that starts IN FRONT of position T (a step start) leaves behind it: `drop` = the bytes at T.. that
// belong to it and carry no output, `nhead` / `head` = its UTF-8 bytes when they live behind the edge (esc_out_pos).
// Lanes 0..10 each test one of the eleven positions in front of T (a pair is 12 bytes long); original bytes only.
struct HeadInfo {
    uint32_t drop;
    uint32_t nhead;
    uint32_t hpos;   // offset of the head bytes behind the edge
    uint32_t head;
    uint32_t bad;
};
// `behind`: the byte at T - 1 - lane for lanes 0..10 (asked for at the start of the slab, so its latency is long gone)
template <class W>
SJ_HD HeadInfo head_info(W& wp, const GlobalReader& g, uint64_t T, bool in_string, uint32_t behind) {
    HeadInfo h;
    h.drop = 0, h.nhead = 0, h.hpos = 0, h.head = 0, h.bad = 0;
    const uint32_t lane = wp.lane();
    uint32_t mine = 0;
    const uint64_t back = (uint64_t)lane + 1;
    if (lane < 11 && T >= back && in_string) mine = behind == '\\' ? 1u : 0u;
    if (!wp.any(mine != 0)) return h;  // no backslash among the last eleven bytes (or not inside a string): nothing straddles
    uint32_t drop = 0, nhead = 0, hpos = 0, head = 0, bad = 0;
    if (mine) {
        const uint64_t x = T - back;
        if ((backslashes_before(g, x) & 1u) == 0) {  // an escape start
            const EscInfo e = esc_decode(g, g, x);
            if (!e.second) {
                if (!e.valid) {
                    bad = 1;
                } else if (x + e.c > T) {
                    const uint32_t over = (uint32_t)(x + e.c - T);  // bytes of the escape at T..
                    const uint64_t op = esc_out_pos(x, e.c, e.n);
                    drop = (uint32_t)range64(0, over);
                    const uint32_t k0 = op < T ? (uint32_t)(T - op) : 0u;  // output bytes in front of the edge (patched there)
                    if (k0 < e.n) {
                        nhead = e.n - k0;
                        hpos = op < T ? 0u : (uint32_t)(op - T);
                        head = e.bytes >> (8 * k0);
                        drop &= ~(uint32_t)range64(hpos, hpos + nhead);
                    }
                }
            }
        }
    }
    // at most one escape can straddle the edge in a valid document; take the nearest one, OR the error flags
    const uint32_t have = wp.ballot(drop != 0 || nhead != 0);
    const uint32_t pick = have ? (uint32_t)(pi::ctz64(have)) : 0;  // lanes count backwards from the edge: the nearest start
    h.drop = have ? wp.shfl(drop, pick) : 0;
    h.nhead = have ? wp.shfl(nhead, pick) : 0;
    h.hpos = have ? wp.shfl(hpos, pick) : 0;
    h.head = have ? wp.shfl(head, pick) : 0;
    h.bad = wp.any(bad != 0) ? 1u : 0u;
    return h;
}

// length of the run of backslashes that ends just before `end` (32 bytes per round; one round in practice)
template <class W>
SJ_HD uint32_t backslash_run_before_p(W& wp, const GlobalReader& g, uint64_t end) {
    const uint32_t lane = wp.lane();
    uint32_t run = 0;
    for (uint64_t off = 0;; off += 32) {
        const uint64_t back = off + lane + 1;
        const uint32_t c = back <= end ? g(end - back) : 0x20u;
        const uint32_t B = wp.ballot(c == '\\');
        const uint32_t n = B == 0xffffffffu ? 32u : pi::ctz64((uint64_t)(~B));
        run += n;
        if (n < 32) return run;
    }
}

// NDJSON: is the last structural in front of the slab a newline?  Outside a string that is "the last byte that is not a
// blank, tab or CR is a newline" (every other byte is a structural of its own or belongs to a value that started behind
// the last newline).  `peekc`: lane L holds the byte at slab_start - 1 - L (0x20 in front of the message).
template <class W>
SJ_HD uint32_t record_carry_in(W& wp, const GlobalReader& g, uint64_t slab_start, uint32_t peekc) {
    const uint32_t lane = wp.lane();
    for (uint64_t off = 0;; off += 32) {
        const uint64_t back = off + lane + 1;
        const uint32_t c = off == 0 ? peekc : (back <= slab_start ? g(slab_start - back) : 0x7fu);
        const uint32_t solid = wp.ballot(!(c == 0x20 || c == 0x09 || c == 0x0d));
        if (solid) return wp.shfl(c, pi::ctz64((uint64_t)solid)) == '\n' ? 1u : 0u;
        if (back + 31 - lane >= slab_start) return 0;  // reached the start of the message: nothing but blanks
    }
}

// What one 2 KiB step holds once its quote mask and its dropped escape bytes are known: stage 1's structurals, the
// events of the tape, record starts, and the lane's counts.  The one definition of the counts: stage 1's parse mode
// adds them up into the slab's SlabAgg, K2r turns the same masks into offsets.
//   m: the classes of the lane's block (open, close, cc, ws, nl, numc, atomc are read); qm / qb: quote mask, real quotes;
//   K: bytes of Strings.B; ppc / recc: the pseudo-structural and record carries, passed on to the next step
struct StepEvents {
    uint64_t brk;     // brackets outside strings
    uint64_t st_out;  // brackets, commas, colons outside strings
    uint64_t closeq;  // closing quotes
    uint64_t V;       // value starts: atoms, numbers, garbage
    uint64_t NLS;     // newlines outside strings (NDJSON)
    uint64_t S;       // stage 1's structurals
    uint64_t EV;      // the same with every string moved to its closing quote
    uint64_t recst;   // record boundaries
    uint32_t n_brk, n_open, n_num, n_rec, w_lane, k_lane, t_lane;
    bool q_lane;
};
template <class W>
SJ_HD StepEvents step_events(W& wp, const Class64& m, uint64_t qm, uint64_t qb, uint64_t K, uint32_t ndjson, uint32_t& ppc,
                             uint32_t& recc) {
    const uint32_t lane = wp.lane();
    const uint32_t lt = (1u << lane) - 1u;
    StepEvents e;
    // finalize_structurals_amd64.s:19-36
    e.brk = (m.open | m.close) & ~qm;
    e.st_out = e.brk | (m.cc & ~qm);
    e.closeq = qb & ~qm;
    const uint64_t s0 = e.st_out | qb;
    uint64_t pseudo;
    {
        const uint64_t pred = s0 | m.ws;
        const uint32_t my_pp = (uint32_t)(pred >> 63);
        const uint32_t up = wp.shfl_up(my_pp, 1);
        const uint32_t pp_in = lane == 0 ? ppc : up;
        ppc = wp.shfl(my_pp, 31);
        pseudo = ((pred << 1) | pp_in) & ~m.ws & ~qm;
    }
    e.V = pseudo & ~s0;
    e.NLS = ndjson ? (m.nl & ~qm) : 0ull;  // find_newline_delimiters_amd64.s:17-27
    e.S = e.st_out | (qb & qm) | e.V | e.NLS;
    e.EV = e.st_out | e.closeq | e.V | e.NLS;
    // record boundaries: the first structural behind a run of newlines, if it is not a newline itself
    // (stage2...go:200-221).  (T + ~S) carries from the byte behind each newline to the next structural.  They are
    // counted where stage 1 sees that structural -- for a string at its OPENING quote -- so that the carry into
    // a slab never depends on what lies in front of an open string.
    e.recst = 0;
    if (ndjson) {
        const bool empty = e.S == 0;
        const bool gen = !empty && ((e.NLS >> (63 - pi::clz64(e.S))) & 1ull);
        const uint32_t Pm = wp.ballot(empty), G = wp.ballot(gen);
        const uint32_t below = ~Pm & lt;
        const uint32_t cin = below ? (G >> (31 - pi::clz32(below))) & 1u : recc;
        const uint32_t nonp = ~Pm;
        recc = nonp ? (G >> (31 - pi::clz32(nonp))) & 1u : recc;
        const uint64_t T = (e.NLS << 1) | cin;
        e.recst = (T + ~e.S) & e.S & ~e.NLS;
    }
    e.n_brk = pi::popc64(e.brk);
    e.n_open = pi::popc64(m.open & ~qm);
    const uint32_t n_str = pi::popc64(e.closeq), n_atom = pi::popc64(e.V & m.atomc);
    e.n_num = pi::popc64(e.V & m.numc);
    e.n_rec = pi::popc64(e.recst);
    e.w_lane = e.n_brk + 2 * n_str + 2 * e.n_num + n_atom + 2 * e.n_rec;
    e.k_lane = pi::popc64(K);
    e.q_lane = qb != 0;
    e.t_lane = e.q_lane ? pi::popc64(K & ~below64(64 - pi::clz64(qb))) : e.k_lane;  // bytes behind the lane's last quote
    return e;
}

// The lane's share of the slab's counts, added up over the slab's steps without a collective (agg_lane_add);
// agg_warp_finish turns the 32 shares into the slab's SlabAgg once per slab.
struct LaneAgg {
    uint32_t w, str, brk, rec, num;
    int32_t depth;
    uint32_t kstep;  // the lane's Strings.B bytes of step s in bits 8s..8s+7 (at most 64 per step)
    uint32_t tq;     // Strings.B bytes behind the lane's last real quote so far
    uint32_t qstep;  // 1 + the step of the lane's last real quote; 0: none yet
};
SJ_HD LaneAgg lane_agg_zero() { return LaneAgg{0, 0, 0, 0, 0, 0, 0, 0, 0}; }
SJ_HD void agg_lane_add(LaneAgg& a, const StepEvents& e, uint32_t s) {
    a.w += e.w_lane;
    a.str += e.k_lane;
    a.brk += e.n_brk;
    a.rec += e.n_rec;
    a.num += e.n_num;
    a.depth += (int32_t)(2 * e.n_open) - (int32_t)e.n_brk;
    a.kstep |= e.k_lane << (8 * s);
    if (e.q_lane) {
        a.tq = e.t_lane;
        a.qstep = s + 1;
    } else {
        a.tq += e.k_lane;
    }
}

// SlabAgg::last of one step's structurals S alone; byte(o) = the step's byte at offset o
template <class W, class B>
SJ_HD uint32_t last_of_step(W& wp, uint64_t S, const B& byte) {
    const uint32_t lane = wp.lane();
    uint32_t v = 0, n = 0;
    for (uint64_t r = S; r && n < 3; n++) {  // the lane's last three, the last one first
        const uint32_t b = 63 - pi::clz64(r);
        v |= byte(64 * lane + b) << (8 * n);
        r &= ~(1ull << b);
    }
    v |= n << 24;
    for (uint32_t d = 1; d < 32; d <<= 1) {  // lane 0 ends up with lanes 0..31 in order
        const uint32_t o = wp.shfl(v, lane + d < 32 ? lane + d : lane);
        if (lane + d < 32) v = last_combine(v, o);
    }
    return wp.shfl(v, 0);
}

// The slab's SlabAgg from the lanes' shares and the structurals S[s] of its steps (0 for steps behind the end of the
// message); byte(s, o) = the byte at offset o of step s.  SlabAgg::last is taken from the last steps that hold a
// structural, walking back only while fewer than three are found.
template <class W, class B>
SJ_HD SlabAgg agg_warp_finish(W& wp, const LaneAgg& a, const uint64_t (&S)[S2S_STEPS], const B& byte) {
    const uint32_t lane = wp.lane();
    SlabAgg r;
    r.w = wp.reduce_add(a.w);
    r.str = wp.reduce_add(a.str);
    r.brk = wp.reduce_add(a.brk);
    r.rec = wp.reduce_add(a.rec);
    r.num = wp.reduce_add(a.num);
    r.depth = (int32_t)wp.reduce_add((uint32_t)a.depth);
    // trail: the Strings.B bytes behind the slab's last real quote, which lies in the top lane among those whose last
    // quote is in the slab's last step with a quote; every step if the slab has none
    r.trail = r.str;
    for (uint32_t s = S2S_STEPS; s >= 1; s--) {
        const uint32_t Q = wp.ballot(a.qstep == s);
        if (Q) {  // warp-uniform
            const uint32_t top = 31 - pi::clz32(Q);
            const uint32_t from = lane > top ? s - 1 : s;  // the lane's blocks from this step on lie behind the quote
            uint32_t behind = 0;
            for (uint32_t t = from; t < S2S_STEPS; t++) behind += (a.kstep >> (8 * t)) & 0xffu;
            r.trail = TRAIL_HASQ | (wp.shfl(a.tq, top) + wp.reduce_add(lane == top ? 0u : behind));
            break;
        }
    }
    r.last = 0;
    for (uint32_t s = S2S_STEPS; s >= 1 && (r.last >> 24) < 3; s--) {
        if (wp.any(S[s - 1] != 0)) r.last = last_combine(last_of_step(wp, S[s - 1], [&](uint32_t o) { return byte(s - 1, o); }), r.last);
    }
    return r;
}

// Does SlabAgg::last in front of `slab` name the bytes under the last structurals of stage 1's index (p.idx) in front of
// it -- the ones K2r takes as the events in front of the slab (par ? 2 : 1: inside a string the last structural is
// that string's opening quote)?
SJ_HD bool last_matches_index(const S2sParams& p, const GlobalReader& g, uint32_t slab, uint32_t last) {
    const uint64_t slab_start = (uint64_t)slab * S2S_SLAB_BYTES;
    uint32_t lo = 0, hi = p.n_idx;  // structurals in front of the slab
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (p.idx[mid] < slab_start)
            lo = mid + 1;
        else
            hi = mid;
    }
    const uint32_t par = (p.slabpar[slab / p.slabs_per_tile] >> (slab % p.slabs_per_tile)) & 1u;
    const uint32_t back = par ? 2u : 1u, n = last >> 24;
    for (uint32_t k = back; k <= back + 1; k++) {
        const uint32_t want = lo >= k ? g(p.idx[lo - k]) : 0u, got = n >= k ? (last >> (8 * (k - 1))) & 0xffu : 0u;
        if (want != got) return false;
    }
    return true;
}

// Ask for the 2 KiB step that starts at message offset `first` into the image buffer `dst` (XOR-swizzled): whole
// 16-byte chunks inside the message travel asynchronously (LDGSTS on the device), the chunk that holds the end of the
// message and the chunks behind it are written directly, padded with spaces (find_structural_bits_amd64.s:167).
// first == ~0: nothing to ask for (an empty group keeps the wait's bookkeeping uniform).
template <class W>
SJ_HD void s2s_issue_step(W& wp, const S2sParams& p, uint64_t first, uint8_t* dst) {
    if (first != ~0ull) {
        const uint32_t lane = wp.lane();
        const uint64_t len16 = (p.len + 15) & ~15ull;
        for (uint32_t c = lane; c < S2S_STEP_BYTES / 16; c += 32) {
            const uint64_t gofs = first + 16ull * c;
            uint8_t* d = dst + swz(16u * c);
            if (gofs + 16 <= p.len) {
                wp.async_copy16(d, p.msg + gofs);
            } else {
                V16 q{0x20202020u, 0x20202020u, 0x20202020u, 0x20202020u};
                if (gofs < len16) {
                    q = *reinterpret_cast<const V16*>(p.msg + gofs);
                    uint32_t qq[4] = {q.x, q.y, q.z, q.w};
                    for (uint32_t k = 0; k < 16; k++)
                        if (gofs + k >= p.len) qq[k >> 2] = (qq[k >> 2] & ~(0xffu << (8 * (k & 3)))) | (0x20u << (8 * (k & 3)));
                    q = V16{qq[0], qq[1], qq[2], qq[3]};
                }
                *reinterpret_cast<V16*>(d) = q;
            }
        }
    }
    wp.async_commit();
}

// One slab.  `cur`: which of the two image buffers holds (will hold) the slab's first step -- the caller asked for it
// before the call (s2s_warp_loop) -- and, on return, the one that holds the first step of `next_slab`.
template <class W, bool EMIT>
SJ_HD void s2s_slab(W& wp, const S2sParams& p, uint32_t slab, const S2sWarpMem& sm, uint32_t& cur, uint32_t next_slab) {
    const uint32_t lane = wp.lane();
    const uint32_t lt = (1u << lane) - 1u;
    K2R_PROBE_START
    const uint64_t slab_start = (uint64_t)slab * S2S_SLAB_BYTES;
    const uint64_t slab_end = slab_start + S2S_SLAB_BYTES < p.len ? slab_start + S2S_SLAB_BYTES : p.len;
    const GlobalReader g{p.msg, p.len};

    // what the slab needs from global memory besides its own bytes is asked for first, so that these (dependent)
    // loads are in flight under the image fill
    uint32_t par = (p.slabpar[slab / p.slabs_per_tile] >> (slab % p.slabs_per_tile)) & 1u;  // in-string state in front of the slab (stage 1's chain 1)
    SlabAgg run = agg_zero();
    const uint64_t out_str_base = EMIT ? s2s_str_base(p) : 0;  // offset of this parse's Strings.B inside the whole (sharded ParseND)
    uint32_t pc1 = 0, pc2 = 0;   // K2r: the bytes under the last two events in front of the slab (0: none)
    bool have1 = false, have2 = false;
    if (EMIT) {
        run = agg_combine(p.grp_pre[slab >> 10], p.pre[slab]);
        // from stage 1's last structurals: inside a string the last one is that string's opening quote, whose event
        // (the closing quote) is still to come
        const uint32_t r = run.last >> 24, back = par ? 2u : 1u;
        have1 = r >= back, have2 = r >= back + 1;
        pc1 = have1 ? (run.last >> (8 * (back - 1))) & 0xffu : 0u;
        pc2 = have2 ? (run.last >> (8 * back)) & 0xffu : 0u;
    }
    const SlabAgg start = run;
    // the bytes in front of the slab (lanes 0..10: byte slab_start - 1 - lane), for an escape that straddles its start
    const uint32_t behind0 = (lane < 11 && slab_start > lane) ? g(slab_start - 1 - lane) : 0x20u;
    HeadInfo hd_next;
    hd_next.drop = 0, hd_next.nhead = 0, hd_next.hpos = 0, hd_next.head = 0, hd_next.bad = 0;
    MsgReader rd{p.msg, p.len, sm.src, slab_start, slab_end};

    // ---- carries into the slab ----
    // lane L: the byte at slab_start - 1 - L
    const uint32_t peekc = slab_start > lane ? g(slab_start - 1 - lane) : 0x20u;
    const uint32_t peek_bs = wp.ballot(peekc == '\\');
    const uint32_t prevc = wp.shfl(peekc, 0);
    uint32_t bsc;  // the slab's first byte is consumed by an escape that starts in front of it
    if (peek_bs == 0xffffffffu)
        bsc = backslash_run_before_p(wp, g, slab_start) & 1u;
    else
        bsc = pi::ctz64((uint64_t)(~peek_bs)) & 1u;
    uint32_t prevc_esc = 0;
    if (prevc == '"') {
        const uint32_t n = pi::ctz64((uint64_t)(~(peek_bs >> 1)));
        prevc_esc = n >= 31 ? backslash_run_before_p(wp, g, slab_start - 1) & 1u : n & 1u;
    }
    // pseudo-structural predecessor (finalize_structurals_amd64.s:24-27; 1 at the start: stage1_find_marks_amd64.go:54)
    uint32_t ppc = 1;
    if (slab > 0) {
        const uint32_t is_q = prevc == '"' && !prevc_esc;
        const uint32_t is_ws = prevc == 0x20 || prevc == 0x09 || prevc == 0x0a || prevc == 0x0d;
        const uint32_t is_st = prevc == '{' || prevc == '}' || prevc == '[' || prevc == ']' || prevc == ':' || prevc == ',';
        ppc = is_q | is_ws | (is_st & (par ^ 1u));
    }
    uint32_t recc = (p.ndjson && !par && slab > 0) ? record_carry_in(wp, g, slab_start, peekc) : 0u;

    // ---- running totals of the slab (K2p) / running prefixes (K2r) ----
    LaneAgg la = lane_agg_zero();  // counting pass: the lane's share of the slab's counts
    uint64_t S_step[S2S_STEPS] = {};  // counting pass: the structurals of each step, for SlabAgg::last
    uint32_t partial = 0;          // K2r: bytes the string that is open at the step start has contributed so far
    uint32_t pr = T_START;         // K2r: refined type of the last event in front of the step
    uint32_t err = 0;
    if (EMIT) {
        partial = run.trail & ~TRAIL_HASQ;
        if (have1) {
            const uint32_t t = sm.ctab[pc1], tp = have2 ? (uint32_t)sm.ctab[pc2] : (uint32_t)T_START;
            pr = (t == T_STRING && (tp == T_OBJ_OPEN || tp == T_COMMA)) ? (uint32_t)T_STRING_KEYPOS : t;
        }
    }

    K2R_PROBE(K2R_PROLOGUE);
    for (uint32_t s = 0; s < S2S_STEPS; s++) {
        const uint64_t step_start = slab_start + (uint64_t)s * S2S_STEP_BYTES;
        if (step_start >= p.len) break;  // warp-uniform
        const uint64_t step_end = step_start + S2S_STEP_BYTES;
        const uint64_t block_pos = step_start + 64ull * lane;
        // the image pipeline: ask for the NEXT step (of this slab or of the warp's next one) into the other buffer,
        // then wait for this step's bytes -- they were asked for one step ago
        {
            uint64_t nxt = step_end;
            if (s + 1 >= S2S_STEPS || nxt >= p.len) nxt = next_slab < p.nslabs ? (uint64_t)next_slab * S2S_SLAB_BYTES : ~0ull;
            wp.sync();  // (the readers of the buffer about to be overwritten -- the step before this one -- are done)
            s2s_issue_step(wp, p, nxt, sm.src + (cur ^ 1u) * S2S_STEP_BYTES);
            wp.async_wait_prev();
            wp.sync();
        }
        K2R_PROBE(K2R_IMAGE);
        const uint8_t* sbase = sm.src + cur * S2S_STEP_BYTES;
        cur ^= 1u;
        rd.src = sbase;
        rd.slab_start = step_start;
        rd.slab_end = step_end < p.len ? step_end : p.len;

        // ---------------- A: load + classify ----------------
        uint32_t w[16];
        {
            const uint32_t r = (lane >> 1) & 3;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const V16 q = *reinterpret_cast<const V16*>(sbase + 64 * lane + 16 * ((uint32_t)j ^ r));
                w[4 * j + 0] = q.x, w[4 * j + 1] = q.y, w[4 * j + 2] = q.z, w[4 * j + 3] = q.w;
            }
        }
        const Class64 m = classify_block2(w);

        // ---------------- B: escape starts, escaped bytes (find_odd_backslash_sequences_amd64.s:24-61) ----------------
        uint64_t E = 0, C = 0;
        {
            const uint32_t hasbs = wp.ballot(m.bs != 0);
            if (hasbs || bsc) {  // warp-uniform
                const bool allbs = m.bs == ~0ull;
                const uint32_t trail_odd = allbs ? 0u : (pi::clz64(~m.bs) & 1u);
                const uint32_t A = wp.ballot(allbs), F = wp.ballot(trail_odd != 0);
                const uint32_t below = ~A & lt;
                const uint32_t cin = below ? (F >> (31 - pi::clz32(below))) & 1u : bsc;
                const uint32_t nonpass = ~A;
                bsc = nonpass ? (F >> (31 - pi::clz32(nonpass))) & 1u : bsc;
                E = escape_starts(m.bs, cin);
                C = (E << 1) | cin;
            }
        }
        const uint64_t qb = m.qt & ~C;  // real quotes
        // ---------------- C: quote mask (find_quote_mask_and_bits_amd64.s:49-66) ----------------
        const bool par_step = par != 0;  // in-string state at the step start
        uint64_t qm;
        {
            const uint32_t P = wp.ballot((pi::popc64(qb) & 1u) != 0);
            const uint32_t lane_in = par ^ (pi::popc32(P & lt) & 1u);
            qm = prefix_xor64(qb) ^ (lane_in ? ~0ull : 0ull);
            par ^= pi::popc32(P) & 1u;
        }

        // ---------------- D: escapes inside strings -> dropped bytes ----------------
        uint64_t D = 0;
        const uint64_t Ein = E & qm;
        // what an escape that starts in front of this step leaves at its head: inside the slab the previous step saw it
        // and hands it over (hd_next); at the start of a slab -- another warp owns what precedes -- it is worked out
        // from the message (head_info)
        HeadInfo hd = hd_next;
        if (s == 0) hd = head_info(wp, g, step_start, par_step, behind0);
        err |= hd.bad;
        hd_next.drop = 0, hd_next.nhead = 0, hd_next.hpos = 0, hd_next.head = 0, hd_next.bad = 0;
        const bool any_esc = wp.any(Ein != 0);
        if (any_esc) {
            // Escape-heavy text is lumpy (a run of "\\uXXXX\\uXXXX..." puts eleven escapes into one block and none into its
            // neighbours), and a decode is a long dependent chain: with every lane decoding its own escapes the warp
            // waits for the fullest block.  So the step's escapes are listed in shared memory and decoded round-robin
            // by all lanes.  Whoever decodes an escape also publishes it: the UTF-8 bytes go straight into the image,
            // over the escape's own LAST bytes (esc_out_pos); its other bytes are marked in the step's DROP MAP (one
            // bit per image byte, red.shared.or); the one escape whose bytes run past the end of the step leaves a
            // record for the next step.  The owners then just read their 64 bits of the map -- no second walk.
            uint32_t* dmap = reinterpret_cast<uint32_t*>(sm.esc);
            uint32_t* rec = reinterpret_cast<uint32_t*>(sm.esc + S2S_ESC_REC_OFS);  // { nhead, hpos, head }
            uint16_t* epos = reinterpret_cast<uint16_t*>(sm.esc + S2S_ESC_LIST_OFS);
            dmap[2 * lane] = 0, dmap[2 * lane + 1] = 0;
            if (lane == 0) dmap[S2S_ESC_DMAP_WORDS - 1] = 0, rec[0] = 0, rec[1] = 0, rec[2] = 0;
            const uint32_t e_cnt = pi::popc64(Ein);
            uint32_t e_inc = e_cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = wp.shfl_up(e_inc, d);
                if ((int)lane >= d) e_inc += t;
            }
            const uint32_t e_tot = wp.shfl(e_inc, 31);
            {
                // the two 32-bit halves side by side (a 64-bit find-first-set is several instructions; two chains, half the trips)
                uint32_t lo = (uint32_t)Ein, hi = (uint32_t)(Ein >> 32);
                uint32_t k0 = e_inc - e_cnt, k1 = k0 + pi::popc32(lo);
                while (lo | hi) {  // branch-free body: an exhausted half writes into the lane's spare slot behind the list
                    const uint32_t s0 = lo ? k0 : S2S_ESC_CAP + lane, s1 = hi ? k1 : S2S_ESC_CAP + lane;
                    epos[s0] = (uint16_t)(64 * lane + pi::ctz32(lo | 0x80000000u));
                    epos[s1] = (uint16_t)(64 * lane + 32 + pi::ctz32(hi | 0x80000000u));
                    k0 += lo != 0, k1 += hi != 0;
                    lo &= lo - 1;
                    hi &= hi - 1;
                }
            }
            wp.sync();
            uint8_t* img = const_cast<uint8_t*>(sbase);
            const uint32_t avail = (uint32_t)(rd.slab_end - rd.slab_start);  // image bytes that are message bytes
            const ImageReader ird{sbase, (uint32_t)step_start, (uint32_t)(rd.slab_end - rd.slab_start), p.msg, p.len};
            // rounds of 32 escapes; in the emitting pass a round's patches wait until every lane has read what it needs (the
            // fast path reads whole words of the image, a patch writes bytes inside them), and the next round's reads wait
            // for the patches
            for (uint32_t base = 0; base < e_tot; base += 32) {  // warp-uniform trips
                const uint32_t i = base + lane;
                uint32_t o = 0;
                EscInfo ei;
                ei.c = 0, ei.n = 0, ei.bytes = 0, ei.valid = false, ei.second = false;
                bool live = false;
                if (i < e_tot) {
                    o = epos[i];
                    if (!esc_u_fast(sbase, o, avail, ei)) ei = esc_decode(ird, g, step_start + o);
                    if (!ei.second) {
                        if (!ei.valid)
                            err = 1;
                        else
                            live = true;
                    }
                }
                if (EMIT) wp.sync();
                if (live) {
                    const uint32_t op = o + ei.c - ei.n;  // first output position (image offset; may lie behind the step)
                    // all c source bytes are dropped except the last n, which hold the output
                    const uint32_t m = ((1u << ei.c) - 1u) & ~(((1u << ei.n) - 1u) << (ei.c - ei.n));
                    const uint32_t wd = o >> 5, sh = o & 31u;
                    wp.atomic_or_shared(dmap + wd, m << sh);
                    if (sh > 20 && (m >> (32 - sh))) wp.atomic_or_shared(dmap + wd + 1, m >> (32 - sh));  // (word 64: bytes of the next step)
                    if (EMIT) {
                        if ((op & 15u) + ei.n <= 16u && op + ei.n <= S2S_STEP_BYTES) {  // inside one 16-byte chunk of the image: one address
                            uint8_t* q = img + swz(op);
                            q[0] = (uint8_t)ei.bytes;
                            if (ei.n > 1) q[1] = (uint8_t)(ei.bytes >> 8);
                            if (ei.n > 2) q[2] = (uint8_t)(ei.bytes >> 16);
                            if (ei.n > 3) q[3] = (uint8_t)(ei.bytes >> 24);
                        } else {
                            for (uint32_t j = 0; j < ei.n; j++)
                                if (op + j < S2S_STEP_BYTES) img[swz(op + j)] = (uint8_t)(ei.bytes >> (8 * j));
                        }
                    }
                    if (op + ei.n > S2S_STEP_BYTES) {  // output bytes behind the end of the step: the next step patches them in
                        const uint32_t k0 = op < S2S_STEP_BYTES ? S2S_STEP_BYTES - op : 0u;
                        rec[0] = ei.n - k0;
                        rec[1] = op < S2S_STEP_BYTES ? 0u : op - S2S_STEP_BYTES;
                        rec[2] = ei.bytes >> (8 * k0);
                    }
                }
                if (EMIT) wp.sync();
            }
            wp.sync();
            D = mk64(dmap[2 * lane], dmap[2 * lane + 1]);
            hd_next.drop = dmap[S2S_ESC_DMAP_WORDS - 1];
            hd_next.nhead = rec[0], hd_next.hpos = rec[1], hd_next.head = rec[2];
            wp.sync();  // (the scratch is the tape staging area of the rest of the step)
        }
        if (lane == 0) D |= (uint64_t)hd.drop;
        const uint64_t K = qm & ~qb & ~D;  // bytes of Strings.B, at their source positions
        if (EMIT && (any_esc || hd.nhead)) {  // warp-uniform: the image was patched, the compaction wants the patched words
            if (hd.nhead && lane == 0) {
                uint8_t* img = const_cast<uint8_t*>(sbase);
                for (uint32_t i = 0; i < hd.nhead; i++) img[swz(hd.hpos + i)] = (uint8_t)(hd.head >> (8 * i));
            }
            wp.sync();
            const uint32_t r = (lane >> 1) & 3;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const V16 q = *reinterpret_cast<const V16*>(sbase + 64 * lane + 16 * ((uint32_t)j ^ r));
                w[4 * j + 0] = q.x, w[4 * j + 1] = q.y, w[4 * j + 2] = q.z, w[4 * j + 3] = q.w;
            }
        }

        K2R_PROBE(K2R_CLASSIFY);
        // ---------------- E: structurals (finalize_structurals_amd64.s:19-36), events, counts ----------------
        const StepEvents ev = step_events(wp, m, qm, qb, K, p.ndjson, ppc, recc);
        const uint64_t closeq = ev.closeq, V = ev.V, NLS = ev.NLS, EV = ev.EV, recst = ev.recst;
        const uint32_t n_brk = ev.n_brk, n_open = ev.n_open, n_num = ev.n_num, n_rec = ev.n_rec;
        const uint32_t w_lane = ev.w_lane, k_lane = ev.k_lane, t_lane = ev.t_lane;
        const bool q_lane = ev.q_lane;

        if (!EMIT) {
            agg_lane_add(la, ev, s);
            S_step[s] = ev.S;
            continue;
        }

        // =========================== K2r ===========================
        // exclusive prefixes of the lane inside the step: tape words (13 bits) | string bytes (12) | brackets (12) |
        // records (11) | depth, biased by 64 per lane (13) in one 64-bit word, numbers in a second one
        uint32_t w_ex, k_ex, b_ex, r_ex, n_ex;
        int32_t d_ex;
        uint32_t w_step, k_step, b_step, r_step, n_step;
        int32_t d_step;
        {
            const uint64_t own = (uint64_t)w_lane | ((uint64_t)k_lane << 13) | ((uint64_t)n_brk << 25) | ((uint64_t)n_rec << 37) |
                                 ((uint64_t)(2 * n_open + 64 - n_brk) << 48);
            uint64_t inc = own;
            uint32_t ninc = n_num;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t tl = wp.shfl_up((uint32_t)inc, d), th = wp.shfl_up((uint32_t)(inc >> 32), d);
                const uint32_t tn = wp.shfl_up(ninc, d);
                if ((int)lane >= d) {
                    inc += mk64(tl, th);
                    ninc += tn;
                }
            }
            const uint64_t ex = inc - own;
            w_ex = (uint32_t)(ex & 0x1fff), k_ex = (uint32_t)((ex >> 13) & 0xfff), b_ex = (uint32_t)((ex >> 25) & 0xfff);
            r_ex = (uint32_t)((ex >> 37) & 0x7ff);
            d_ex = (int32_t)(ex >> 48) - 64 * (int32_t)lane;
            n_ex = ninc - n_num;
            const uint64_t tot = mk64(wp.shfl((uint32_t)inc, 31), wp.shfl((uint32_t)(inc >> 32), 31));
            w_step = (uint32_t)(tot & 0x1fff), k_step = (uint32_t)((tot >> 13) & 0xfff), b_step = (uint32_t)((tot >> 25) & 0xfff);
            r_step = (uint32_t)((tot >> 37) & 0x7ff);
            d_step = (int32_t)(tot >> 48) - 64 * 32;
            n_step = wp.shfl(ninc, 31);
        }
        // bytes the string open at the lane's first byte has contributed so far
        uint32_t part_lane;
        {
            const uint32_t Q = wp.ballot(q_lane);
            const uint32_t v = t_lane - (k_ex + k_lane);  // (wraps; only differences are used)
            const uint32_t below = Q & lt;
            const uint32_t got = wp.shfl(v, below ? 31 - pi::clz32(below) : 0);
            part_lane = below ? k_ex + got : partial + k_ex;
            if (Q) {
                const uint32_t top = 31 - pi::clz32(Q);
                partial = k_step + wp.shfl(v, top);
            } else {
                partial += k_step;
            }
        }

        K2R_PROBE(K2R_EVENTS);
        // ---------------- Strings.B: byte compaction of the step into the staging area ----------------
        const uint32_t str_base = run.str;                 // offset of the step's bytes in Strings.B
        const uint32_t shift = (uint32_t)(reinterpret_cast<uintptr_t>(p.strings + str_base) & 15u);  // staging keeps the destination's 16-byte phase
        if (k_step) {                                      // warp-uniform
            // Every staging word in [shift / 4, (shift + k_step - 1) / 4] is stored exactly once, with a plain store, by
            // the lane that holds its first output byte: whole words as they fill, and the SEAM word a lane's bytes end
            // in after the lanes above have handed it the bytes they put into it.  Those lanes start their output in
            // the middle of the word (o & 3 != 0) and feed their first word's bytes (`feed`) instead of storing it; each
            // gives at least one byte, so at most three of them share the word with its owner.  The bytes in front of
            // `shift` and behind the step's last byte are never read.
            uint32_t* st32 = reinterpret_cast<uint32_t*>(sm.sstage);
            const uint32_t o = shift + k_ex;               // first output byte of the lane
            const uint32_t first = o >> 2;
            const bool feeds = (o & 3u) != 0 && o != shift;  // a lane below holds the first byte of the lane's first word
            uint32_t feed = 0, seam = 0, seam_at = ~0u;
            if (k_lane) {
                uint32_t ptr = first, fill = o & 3u, lo = 0;
                const uint32_t Klo = (uint32_t)K, Khi = (uint32_t)(K >> 32);
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    const uint32_t m4 = ((k < 8 ? Klo : Khi) >> (4 * (k & 7))) & 15u;
                    const uint32_t ce = sm.cmptab[m4];  // PRMT selector | kept bytes << 16
                    const uint32_t cw = pi::byte_perm(w[k], 0, ce & 0xffffu);
                    const uint32_t cnt = ce >> 16;
                    lo |= cw << (8 * fill);
                    const uint32_t hi = pi::funnel_l(cw, 0, 8 * fill);
                    fill += cnt;
                    if (fill >= 4) {
                        if (ptr == first && feeds)
                            feed = lo;
                        else
                            st32[ptr] = lo;
                        ptr++;
                        lo = hi;
                        fill -= 4;
                    }
                }
                if (fill) {
                    if (ptr == first && feeds)
                        feed = lo;
                    else
                        seam = lo, seam_at = ptr;
                }
            }
            // the next three lanes with output bytes: those whose first word is the seam word feed it
            uint32_t above = wp.ballot(k_lane != 0) & ~((2u << lane) - 1u);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const uint32_t src = above ? (uint32_t)pi::ctz32(above) : lane;
                const uint32_t f_src = wp.shfl(first, src), v_src = wp.shfl(feed, src);
                if (above && f_src == seam_at) seam |= v_src;
                above &= above - 1u;
            }
            if (seam_at != ~0u) st32[seam_at] = seam;
            wp.sync();
            // copy-out: head and tail bytes one by one, the 16-byte aligned middle as vectors
            {
                uint8_t* dst = p.strings + str_base;  // dst + i <-> sstage[shift + i]
                const uint32_t total = k_step;
                const uint32_t head_n = shift ? (16 - shift < total ? 16 - shift : total) : 0;
                if (lane < head_n) dst[lane] = sm.sstage[shift + lane];
                const uint32_t body = (total - head_n) & ~15u;
                const V16* s16 = reinterpret_cast<const V16*>(sm.sstage + shift + head_n);
                V16* d16 = reinterpret_cast<V16*>(dst + head_n);
                for (uint32_t i = lane; i < body / 16; i += 32) d16[i] = s16[i];
                const uint32_t tail0 = head_n + body;
                if (lane < total - tail0) dst[tail0 + lane] = sm.sstage[shift + tail0 + lane];
            }
        }

        K2R_PROBE(K2R_STRINGS);
        // ---------------- the lane's events, in order ----------------
        // The step's tape words [slot0, slot0 + w_step) go to the tape-staging area at the destination's 32-byte phase
        // and out in whole sectors behind the loops; scattered 8-byte stores straight to the tape would each land on a
        // sector of their own.  A step that does not fit (dense brackets: up to ~2048 words) stores directly.
        const uint32_t slot0 = 1 + run.w;                // tape slot of the step's first word (slot 0: the first root word)
        const uint32_t ph = (uint32_t)(reinterpret_cast<uintptr_t>(p.tape + slot0) >> 3) & 3u;  // (the tape is 8-byte aligned)
        const uint32_t sslot = slot0 - ph;               // slot of staging word 0 (modulo 2^32: it may lie in front of slot 0)
        const bool staged = ph + w_step <= S2S_TSTAGE_WORDS;  // warp-uniform, as are the two below
        // brackets and record starts of a staged step are listed in the string staging area, so that the pairs with both
        // ends in the step are linked here (K2t then skips them)
        const bool link_b = staged && b_step != 0 && b_step <= S2S_LINK_BRK_CAP;
        const bool link_r = staged && r_step >= 2 && r_step <= S2S_LINK_REC_CAP && p.rootlink != nullptr;
        uint32_t* const lst = reinterpret_cast<uint32_t*>(sm.sstage);  // [0, BRK_CAP): brackets, then record starts
        if (k_step && (link_b || link_r)) wp.sync();      // (Strings.B's copy-out has read the string staging area)
        auto put = [&](uint32_t slot, uint64_t v) {
            if (staged)
                sm.tstage[slot - sslot] = v;
            else
                p.tape[slot] = v;
        };
        {
            // refined type of the last event in front of the lane
            const uint32_t nev = pi::popc64(EV);
            uint32_t last_b = 0, prev_b = T_INVALID;  // base types of the lane's last event and of the one before it
            if (nev) {
                const uint32_t tb = 63 - pi::clz64(EV);
                last_b = sm.ctab[sbase[swz(64 * lane + tb)]];
                if (nev > 1) {
                    const uint64_t rest = EV & ~(1ull << tb);
                    prev_b = sm.ctab[sbase[swz(64 * lane + 63 - pi::clz64(rest))]];
                }
            }
            const uint32_t HE = wp.ballot(nev != 0);
            const uint32_t below = HE & lt;
            const uint32_t src = below ? 31 - pi::clz32(below) : 0;
            const uint32_t below_last_b = wp.shfl(last_b, src);
            const uint32_t pr_b = pr == T_STRING_KEYPOS ? (uint32_t)T_STRING : pr;
            if (nev == 1) prev_b = below ? below_last_b : pr_b;
            const uint32_t last_ref = (last_b == T_STRING && (prev_b == T_OBJ_OPEN || prev_b == T_COMMA)) ? (uint32_t)T_STRING_KEYPOS : last_b;
            const uint32_t below_last_ref = wp.shfl(last_ref, src);
            uint32_t pcur = below ? below_last_ref : pr;
            if (HE) pr = wp.shfl(last_ref, 31 - pi::clz32(HE));

            // ---- the grammar, bit-parallel (stage2...go:176-425 as restated by transition_ok): PRE_x = the events whose
            // previous event is of class x; an event is fine inside an object / an array / at the top level iff its
            // (previous class, own class) pair is in the respective set.  What depends on the container is decided
            // per bracket-to-bracket segment by K2t. ----
            const uint64_t O1 = m.open & m.curly & ~qm, O2 = m.open & ~m.curly & ~qm;
            const uint64_t C1 = m.close & m.curly & ~qm, C2 = m.close & ~m.curly & ~qm;
            const uint64_t COMMA = m.comma & ~qm, COLON = m.cc & ~m.comma & ~qm;
            const uint64_t NUM = V & m.numc, ATOM = V & m.atomc;
            const uint64_t BRK = O1 | O2 | C1 | C2;
            uint64_t BADR, BADO, BADA;
            {
                const uint64_t PRE_O1 = next_event(O1, pcur == T_OBJ_OPEN, EV), PRE_O2 = next_event(O2, pcur == T_ARR_OPEN, EV);
                const uint64_t PRE_COLON = next_event(COLON, pcur == T_COLON, EV), PRE_COMMA = next_event(COMMA, pcur == T_COMMA, EV);
                const uint64_t PRE_SCAL = next_event(NUM | ATOM, pcur >= T_NUMBER && pcur <= T_NULL, EV);
                const uint64_t PRE_CLOSE = next_event(C1 | C2, pcur == T_OBJ_CLOSE || pcur == T_ARR_CLOSE, EV);
                const uint64_t PRE_NL = next_event(NLS, pcur == T_NEWLINE, EV);
                const uint64_t PRE_START = pcur == T_START ? (EV & (0 - EV)) : 0ull;  // the very first event of the message
                const uint64_t STRK = closeq & (PRE_O1 | PRE_COMMA), STRV = closeq & ~STRK;  // strings in key position / elsewhere
                const uint64_t PRE_STRK = next_event(STRK, pcur == T_STRING_KEYPOS, EV), PRE_STRV = next_event(STRV, pcur == T_STRING, EV);
                const uint64_t VALSTART = closeq | NUM | ATOM | O1 | O2;
                const uint64_t VEND = PRE_SCAL | PRE_CLOSE;
                const uint64_t OKO = (PRE_O1 & (closeq | C1)) | (PRE_COLON & VALSTART) | (PRE_COMMA & closeq) | (PRE_STRK & COLON) |
                                     ((PRE_STRV | VEND) & (COMMA | C1));
                const uint64_t OKA = (PRE_O2 & (VALSTART | C2)) | (PRE_COMMA & VALSTART) | ((PRE_STRK | PRE_STRV | VEND) & (COMMA | C2));
                const uint64_t OKR = (PRE_START & (O1 | O2)) | (PRE_CLOSE & NLS) | (PRE_NL & (NLS | O1 | O2));
                BADR = EV & ~OKR, BADO = EV & ~OKO, BADA = EV & ~OKA;
            }
            if (V & ~m.numc & ~m.atomc) err = 1;  // a value that starts with neither a digit, '-' nor t / f / n
            K2R_PROBE(K2R_GRAMMAR);

            // ---- emission: one uniform loop per class of event; the tape slot of an event = words of the events below
            // it.  The block is handled as two 32-bit halves so that every mask operation is a single-register one. ----
            const uint64_t W1 = BRK | ATOM, W2 = closeq | NUM;  // one-word / two-word events
            const uint64_t OPENS = O1 | O2;
            const uint32_t lane_str = str_base + k_ex;          // Strings.B offset of the lane's first kept byte
            const uint64_t str_tag = (uint64_t)'"' << 56, str_buf = STRINGBUFBIT + out_str_base;
            uint32_t words_b = slot0 + w_ex;                     // tape slot of the half's first word
            uint32_t kb_b = run.brk + b_ex, rec_b = run.rec + r_ex, num_b = run.num + n_ex, rank_b = 0;
            int32_t depth_b = run.depth + d_ex;
            uint32_t pre_dl = part_lane;                         // bytes the string open at the start of the half has contributed
            uint32_t segbad = 0;                                 // contexts ruled out since the last bracket (bit 0 root, 1 object, 2 array)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const uint32_t w1 = (uint32_t)(W1 >> (32 * h)), w2 = (uint32_t)(W2 >> (32 * h)), rs = (uint32_t)(recst >> (32 * h));
                const uint32_t kk = (uint32_t)(K >> (32 * h)), qq = (uint32_t)(qb >> (32 * h)), cq = (uint32_t)(closeq >> (32 * h));
                const uint32_t brk = (uint32_t)(BRK >> (32 * h)), opn = (uint32_t)(OPENS >> (32 * h)), cur = (uint32_t)(m.curly >> (32 * h));
                const uint32_t num = (uint32_t)(NUM >> (32 * h)), atm = (uint32_t)(ATOM >> (32 * h));
                const uint32_t bdr = (uint32_t)(BADR >> (32 * h)), bdo = (uint32_t)(BADO >> (32 * h)), bda = (uint32_t)(BADA >> (32 * h));
                const uint64_t half_pos = block_pos + 32 * h;
                // record boundaries (root close + root open: the words themselves are written by K2f, or below)
                for (uint32_t mm = rs; mm; mm &= mm - 1) {
                    const uint32_t lo = (mm & (0u - mm)) - 1u;
                    const uint32_t below = pi::popc32(rs & lo);
                    const uint32_t open = words_b + pi::popc32(w1 & lo) + 2 * (pi::popc32(w2 & lo) + below) + 1;
                    p.rootpos[rec_b + below + 1] = open;
                    if (link_r) lst[S2S_LINK_BRK_CAP + rec_b - run.rec + below] = open;
                }
                // The tape slot of an event at bit j: words_b + one word per w1 event and two per w2 event below it + two
                // per record start below it (for brackets, numbers and atoms: at or below it -- their root words come
                // first).  A record start sits on stage 1's structural -- a bracket, an opening quote or a value start --
                // so it shares a bit with w2 only where a record starts with a number.  A lane whose half has no such bit
                // (FOLD) counts the record starts with w2 (w2r): two popcounts per slot instead of three.  On a bracket
                // or an atom w2 has no bit, so w2r up to and including the event's own bit counts its record start; on
                // a number rs has none.
                const uint32_t w2r = w2 | rs;
                const uint32_t str_lane = lane_str + rank_b;  // Strings.B offset of the half's first kept byte
                auto events = [&](auto fold) {
                    constexpr bool FOLD = decltype(fold)::value;
                    // brackets: records for the scope matching, the tape word, the grammar verdict of the segment they end
                    {
                        uint32_t prevm = 0;  // bits up to and including the previous bracket of the half
                        for (uint32_t mm = brk; mm; mm &= mm - 1) {
                            const uint32_t bit = mm & (0u - mm), lo = bit - 1u, upto = lo | bit;
                            const uint32_t slot = FOLD ? words_b + pi::popc32(w1 & lo) + 2 * pi::popc32(w2r & upto)
                                                       : words_b + pi::popc32(w1 & lo) + 2 * (pi::popc32(w2 & lo) + pi::popc32(rs & upto));
                            const uint32_t nb = pi::popc32(brk & lo), kb = kb_b + nb;
                            const bool curly = (cur & bit) != 0, opening = (opn & bit) != 0;
                            const int32_t dep = depth_b + 2 * (int32_t)pi::popc32(opn & lo) - (int32_t)nb;  // opens - closes below
                            const uint32_t kind = opening ? (curly ? T_OBJ_OPEN : T_ARR_OPEN) : (curly ? T_OBJ_CLOSE : T_ARR_CLOSE);
                            p.brk_tp[kb] = slot;
                            p.brk_depth[kb] = dep;
                            if (link_b)  // staging index (10 bits) | kind (3) | depth in front relative to the step's, + 4096 (13)
                                lst[kb - run.brk] = (slot - sslot) | (kind << 10) | ((uint32_t)(dep - run.depth + 4096) << 13);
                            else
                                p.brk_kind[kb] = (uint8_t)kind;
                            put(slot, (uint64_t)((opening ? 0x5bu : 0x5du) | (curly ? 0x20u : 0u)) << 56);  // payload: cross-linked below or by K2t
                            const uint32_t seg = upto & ~prevm;
                            const uint32_t bad = segbad | ((bdr & seg) ? 1u : 0u) | ((bdo & seg) ? 2u : 0u) | ((bda & seg) ? 4u : 0u);
                            if (bad) wp.atomic_and(p.segmask + (kb >> 2), ~(bad << (8 * (kb & 3))));
                            segbad = 0;
                            prevm = upto;
                        }
                        const uint32_t seg = ~prevm;  // behind the half's last bracket: the segment goes on
                        segbad |= ((bdr & seg) ? 1u : 0u) | ((bdo & seg) ? 2u : 0u) | ((bda & seg) ? 4u : 0u);
                    }
                    // strings, at their closing quote (stage2...go:72-113)
                    for (uint32_t mm = cq; mm; mm &= mm - 1) {
                        const uint32_t lo = (mm & (0u - mm)) - 1u;
                        const uint32_t slot = FOLD ? words_b + pi::popc32(w1 & lo) + 2 * pi::popc32(w2r & lo)
                                                   : words_b + pi::popc32(w1 & lo) + 2 * (pi::popc32(w2 & lo) + pi::popc32(rs & lo));
                        const uint32_t kbelow = pi::popc32(kk & lo);
                        const uint32_t lower = qq & lo;  // the opening quote is the highest quote below, if it is in this half
                        const uint32_t dl = lower ? pi::popc32(kk & lo & ~((1u << (31 - pi::clz32(lower))) - 1u)) : pre_dl + kbelow;
                        put(slot, str_tag | (str_buf + (uint64_t)(str_lane + kbelow - dl)));
                        put(slot + 1, dl);
                    }
                    // numbers: parsed by K2h from the list
                    for (uint32_t mm = num; mm; mm &= mm - 1) {
                        const uint32_t j = pi::ctz32(mm), bit = 1u << j, lo = bit - 1u;
                        NumEntry ne;
                        ne.pos = (uint32_t)(half_pos + j);
                        ne.slot = FOLD ? words_b + pi::popc32(w1 & lo) + 2 * pi::popc32(w2r & lo)
                                       : words_b + pi::popc32(w1 & lo) + 2 * (pi::popc32(w2 & lo) + pi::popc32(rs & (lo | bit)));
                        p.numlist[num_b + pi::popc32(num & lo)] = ne;
                    }
                    // atoms
                    for (uint32_t mm = atm; mm; mm &= mm - 1) {
                        const uint32_t j = pi::ctz32(mm), bit = 1u << j, lo = bit - 1u;
                        const uint32_t slot = FOLD ? words_b + pi::popc32(w1 & lo) + 2 * pi::popc32(w2r & (lo | bit))
                                                   : words_b + pi::popc32(w1 & lo) + 2 * (pi::popc32(w2 & lo) + pi::popc32(rs & (lo | bit)));
                        uint32_t ch;
                        bool ok;
                        if (!atom_ok_fast(sbase, 64 * lane + 32 * h + j, (uint32_t)(rd.slab_end - rd.slab_start), &ch, &ok)) {
                            ch = sbase[swz(64 * lane + 32 * h + j)];
                            ok = atom_ok_p(rd, half_pos + j, p.len, sm.ctab[ch]);
                        }
                        if (!ok) err = 1;
                        put(slot, (uint64_t)ch << 56);
                    }
                };
                if ((w2 & rs) == 0)  // per lane (no collective inside)
                    events(BoolC<true>());
                else
                    events(BoolC<false>());
                // totals of the half
                const uint32_t nk = pi::popc32(kk), nopn = pi::popc32(opn), nbr = pi::popc32(brk);
                words_b += pi::popc32(w1) + 2 * (pi::popc32(w2) + pi::popc32(rs));
                kb_b += nbr;
                depth_b += (int32_t)nopn - (int32_t)(nbr - nopn);
                rec_b += pi::popc32(rs);
                num_b += pi::popc32(num);
                pre_dl = qq ? pi::popc32(kk & ~((2u << (31 - pi::clz32(qq))) - 1u)) : pre_dl + nk;
                rank_b += nk;
            }
            // the segment behind the lane's last bracket goes on in the next lanes
            if (segbad) wp.atomic_and(p.segmask + (kb_b >> 2), ~(segbad << (8 * (kb_b & 3))));
        }
        K2R_PROBE(K2R_EMIT);
        if (staged) {
            wp.sync();
            if (link_b || link_r) {
                const uint64_t tb = s2s_tape_base(p);
                // a close whose partner -- the nearest bracket in front of it with a smaller depth in front, K2d's rule;
                // none for a close at the top level -- lies in the step gets both cross-links (K2t's words) and BRK_LINKED
                for (uint32_t i = lane; link_b && i < b_step; i += 32) {
                    const uint32_t e = lst[i], kind = (e >> 10) & 7u, t = e >> 13;
                    uint32_t linked = 0;
                    if ((kind == T_OBJ_CLOSE || kind == T_ARR_CLOSE) && run.depth + (int32_t)t - 4096 > 0) {
                        const uint32_t stop = i > S2S_LINK_SCAN ? i - S2S_LINK_SCAN : 0u;
                        for (uint32_t j = i; j > stop;) {
                            const uint32_t f = lst[j - 1], d = f >> 13;
                            if (d < t) {
                                const uint32_t o = f & 0x3ffu, c = e & 0x3ffu;  // staging indices of the pair
                                const bool curly = kind == T_OBJ_CLOSE;
                                sm.tstage[o] = ((uint64_t)(curly ? '{' : '[') << 56) | (tb + (uint32_t)(sslot + c + 1));
                                sm.tstage[c] = ((uint64_t)(curly ? '}' : ']') << 56) | (tb + (uint32_t)(sslot + o));
                                linked = BRK_LINKED;
                                break;
                            }
                            // the depth moves by one per bracket: the d - t brackets in front of this one are no shallower
                            const uint32_t skip = 1 + d - t;
                            j = j > stop + skip ? j - skip : stop;
                        }
                    }
                    p.brk_kind[run.brk + i] = (uint8_t)(kind | linked);
                }
                // records r = run.rec + 1 + i whose open (record start i of the step) and whose close (in front of record
                // start i + 1) both lie in the step: both root words (K2f's), and their rootlink bits cleared
                if (link_r) {
                    const uint64_t R = (uint64_t)'r' << 56;
                    const uint32_t* rl = lst + S2S_LINK_BRK_CAP;
                    for (uint32_t i = lane; i + 1 < r_step; i += 32) {
                        const uint32_t open = rl[i], next = rl[i + 1];
                        sm.tstage[open - sslot] = R | (tb + next);
                        sm.tstage[next - 1 - sslot] = R | (tb + open);
                    }
                    const uint32_t a = run.rec + 1, b = run.rec + r_step;  // records [a, b)
                    const uint32_t wd = (a >> 5) + lane;
                    if (wd <= ((b - 1) >> 5)) {
                        const uint32_t lo = wd == (a >> 5) ? (a & 31u) : 0u, hi = wd == ((b - 1) >> 5) ? ((b - 1) & 31u) : 31u;
                        const uint32_t m = (0xffffffffu >> (31 - hi)) & ~((1u << lo) - 1u);  // bits [lo, hi]
                        wp.atomic_and(p.rootlink + wd, ~m);
                    }
                }
                wp.sync();
            }
            // copy-out: staging word i is tape word sslot + i; the 16-byte aligned middle as vectors (8 lanes fill a
            // 128-byte line), at most one single word at each end
            if (w_step) {
                uint64_t* const d = p.tape + slot0;  // d[i - ph] <-> tstage[i]
                const uint32_t end = ph + w_step, a = (ph + 1) & ~1u, e = end & ~1u;
                if (lane == 0 && (ph & 1u)) d[0] = sm.tstage[ph];
                const V16* s16 = reinterpret_cast<const V16*>(sm.tstage + a);
                V16* d16 = reinterpret_cast<V16*>(d + (a - ph));
                for (uint32_t i = lane; i < (e - a) / 2; i += 32) d16[i] = s16[i];
                if (lane == 31 && (end & 1u)) d[e - ph] = sm.tstage[e];
            }
        }
        wp.sync();  // the staging areas and the escape scratch are reused by the next step
        K2R_PROBE(K2R_LINK);
        run.w += w_step;
        run.str += k_step;
        run.brk += b_step;
        run.rec += r_step;
        run.depth += d_step;
        run.num += n_step;
    }

    if (EMIT) K2R_PROBE_FLUSH;
    if (wp.any(err != 0) && lane == 0) wp.atomic_or(p.error, 1u);
    if (EMIT && lane == 0) {  // the counts K2r went by against the ones stage 1 added up for the slab
        const SlabAgg want = agg_combine(start, p.agg[slab]);
        bool miscount = run.w != want.w || run.str != want.str || run.brk != want.brk || run.rec != want.rec ||
                    run.depth != want.depth || run.num != want.num;
#ifndef __CUDA_ARCH__  // (the device parse has no index; compiled there, the test costs K2r registers)
        if (p.idx) miscount |= !last_matches_index(p, g, slab, start.last);
#endif
        if (miscount) {  // the tape is not to be trusted: the parse fails, and the internal word says why
            wp.atomic_or(p.error, 1u);
            if (p.internal) wp.atomic_or(p.internal, 1u);
        }
    }
    if (!EMIT) {  // (the step images are gone by now; structurals sit on original message bytes)
        const SlabAgg a = agg_warp_finish(wp, la, S_step, [&](uint32_t s, uint32_t o) { return g(slab_start + (uint64_t)s * S2S_STEP_BYTES + o); });
        if (lane == 0) p.agg[slab] = a;
    }
}

// What one warp does: slabs first, first + stride, ... with the image of the next step always in flight.
template <class W, bool EMIT>
SJ_HD void s2s_warp_loop(W& wp, const S2sParams& p, uint32_t first, uint32_t stride, const S2sWarpMem& sm) {
    if (first >= p.nslabs) return;  // warp-uniform
    uint32_t cur = 0;
    s2s_issue_step(wp, p, (uint64_t)first * S2S_SLAB_BYTES, sm.src);
    for (uint32_t slab = first; slab < p.nslabs; slab += stride) s2s_slab<W, EMIT>(wp, p, slab, sm, cur, slab + stride);
}

}  // namespace sj
