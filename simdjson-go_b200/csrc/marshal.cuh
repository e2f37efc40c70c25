// marshal.cuh -- Iter.MarshalJSON (parsed_json.go:394-556) on the device: a tape in HBM back to compact JSON text in HBM.
//
// The work is spread over tape words, not over roots, so a single-document tape runs as wide as an NDJSON one.  Each
// word-parallel step is one pass over the tape in tiles of MJ_TILE words (KM1's tiles, tape.cuh):
//   KM1 mj_heads_reduce (tape.cuh) / KM2 mj_depth   which words are heads and the depth in front of every head
//   K2d s2_min32 + s2_ansv (stage2_common.cuh)   the parent of every head: the nearest earlier head of smaller depth
//   KM3 mj_keys    F(j) = 1 for every non-close head whose parent is '{'; its per-tile counts and the in-tile parity of
//        its exclusive prefix (one bit per word).  A string in an object is a key when the parity over (object, string)
//        is even: a complete child container adds an even count, since every object inside it has an even number of
//        direct members
//   KM4 mj_measure  validation of the tape + every head's output length, per-tile sums
//   KM5 mj_emit     the exclusive scan of the lengths and the bytes
#pragma once
#include "common.cuh"
#include "fmt.h"
#include "tape.cuh"

namespace sj {

constexpr int MJ_THREADS = 1024;
constexpr int MJ_ROUNDS = 4;                        // a tile is MJ_ROUNDS rounds of one word per thread
constexpr uint64_t MJ_TILE = MJ_THREADS * MJ_ROUNDS;
static_assert(MJ_THREADS == TAPE_THREADS && MJ_ROUNDS == TAPE_ROUNDS, "KM2 .. KM5 run on KM1's tiles (tape.cuh)");
constexpr uint64_t MJ_SHORT = 32;                   // longer strings are escaped by their whole warp
constexpr int32_t MJ_PAYLOAD = 0x7fffffff;          // depth entry of a word that is not a head

// root words: the open one points forward (one past its close), the close one back at its open
__device__ __forceinline__ bool mj_is_close(uint64_t w, uint64_t i) {
    const uint32_t t = (uint32_t)(w >> 56);
    return t == '}' || t == ']' || (t == 'r' && (w & TAPE_VALUE_MASK) <= i);
}

// KM2: depth in front of every head (the tape starts at a head), MJ_PAYLOAD for the other words
__global__ void __launch_bounds__(MJ_THREADS) mj_depth_kernel(const uint64_t* tape, uint64_t n, const HAgg* tile_pre,
                                                             const HAgg* grp_pre, int32_t* depth) {
    const uint64_t base = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)threadIdx.x * MJ_ROUNDS;
    uint64_t w[MJ_ROUNDS];
    HAgg pre = tape_heads(tape, n, tile_pre, grp_pre, base, w);
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++) {
        if (base + j >= n) break;
        depth[base + j] = hagg_out(pre, 1) ? pre.d1 : MJ_PAYLOAD;
        pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
}

// KM3's words of a whole tape: F(i) = 1 for a non-close head whose parent is '{'
struct MjTapeWords {
    const uint64_t* tape;
    uint64_t n;
    __device__ __forceinline__ bool f(uint64_t i, const int32_t* depth, const int32_t* par) const {
        if (i >= n || depth[i] == MJ_PAYLOAD || mj_is_close(tape[i], i)) return false;
        const int32_t p = par[i];
        return p >= 0 && (tape[p] >> 56) == '{';
    }
};

// KM3: F per word; fbits = parity of F's in-tile exclusive prefix, tile_f = F's count per tile.  W is MjTapeWords, or
// the cells' virtual word space of the find's JSON paths (find_json.cuh)
template <class W>
__global__ void __launch_bounds__(MJ_THREADS) mj_keys_kernel(const W words, const int32_t* depth, const int32_t* par,
                                                            uint32_t* fbits, MSum* tile_f) {
    __shared__ uint32_t cnt[MJ_ROUNDS * 32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t b[MJ_ROUNDS];
#pragma unroll
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint64_t i = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS + threadIdx.x;
        const bool f = words.f(i, depth, par);
        b[r] = __ballot_sync(FULL, f);
        if (lane == 0) cnt[r * 32 + warp] = __popc(b[r]);
    }
    __syncthreads();
    if (warp == 0) {  // exclusive prefix of the 128 warp counts, in tape order (round-major)
        uint32_t v[MJ_ROUNDS], s = 0;
#pragma unroll
        for (int j = 0; j < MJ_ROUNDS; j++) {
            v[j] = cnt[lane * MJ_ROUNDS + j];
            s += v[j];
        }
        uint32_t inc = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(FULL, inc, d);
            if (lane >= d) inc += t;
        }
        uint32_t run = inc - s;
        __syncwarp();
#pragma unroll
        for (int j = 0; j < MJ_ROUNDS; j++) {
            cnt[lane * MJ_ROUNDS + j] = run;
            run += v[j];
        }
        if (lane == 31) tile_f[blockIdx.x] = MSum{inc};
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint32_t bit = (cnt[r * 32 + warp] + __popc(b[r] & lanemask_lt())) & 1;
        const uint32_t word = __ballot_sync(FULL, bit);
        if (lane == 0) fbits[((uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS) / 32 + warp] = word;
    }
}

struct MarshalParams {
    TapeView t;
    const int32_t* depth;
    const int32_t* par;
    const uint32_t* fbits;
    const MSum* f_tile_pre;
    const MSum* f_grp_pre;
    const HAgg* h_total;     // the transfer function of the whole tape
    MSum* len_tile;          // KM4: output bytes per tile
    const MSum* len_tile_pre;  // KM5: their exclusive scan
    const MSum* len_grp_pre;
    unsigned long long* err;  // any malformation
    uint8_t* out;
};

// parity of F's exclusive prefix at word j
__device__ __forceinline__ uint32_t mj_x(const MarshalParams& p, uint64_t j) {
    return (uint32_t)((tile_prefix(p.f_tile_pre, p.f_grp_pre, j / MJ_TILE).v + (p.fbits[j >> 5] >> (j & 31))) & 1);
}

struct MjItem {
    uint64_t len;       // output bytes of the word (a long string's body not yet included)
    const uint8_t* s;   // string body
    uint64_t slen;
    uint64_t payload;   // number value word
    uint32_t tag;       // 0: writes nothing
    uint32_t sep;       // 0, ':', ',' or '\n' behind the value
    bool long_str;
};

// The words [lo, hi) of the value a word belongs to (the whole tape, or one JSON cell of the find), and d = its tape
// index - its index in the per-word arrays (depth, par, fbits)
struct MjSpan {
    uint64_t lo, hi;
    int64_t d;
};

// What head i writes, after the checks of a foreign tape: false = malformed.  Every read stays inside the span, the
// string buffer or the message.  CELL: the span is one element's sub-tree, whose head alone sits at its top level and
// writes no separator, and which holds no root word.
template <bool CELL>
__device__ bool mj_item(const MarshalParams& p, uint64_t i, const MjSpan& s, MjItem& it) {
    const uint64_t w = p.t.tape[i];
    const uint32_t t = (uint32_t)(w >> 56);
    const uint64_t v = w & TAPE_VALUE_MASK;
    const int32_t pv = p.par[i - s.d];
    const int64_t pp = pv < 0 ? -1 : (int64_t)pv + s.d;  // the parent's tape index
    uint32_t pt = 0;
    if (pp >= 0) {
        const uint64_t pw = p.t.tape[pp];
        pt = (uint32_t)(pw >> 56);
        if (!(pt == '{' || pt == '[' || (pt == 'r' && (pw & TAPE_VALUE_MASK) > (uint64_t)pp))) return false;  // parent is no open
    }
    if (CELL) {
        if (t == 'r' || (pp < 0 && i != s.lo)) return false;
    } else {
        if (t == 'r' && v > i) return pp < 0;  // a root open writes nothing and sits at the top level
        if (pp < 0) return false;
    }
    if (t == '}' || t == ']' || t == 'r') {  // close: its parent is its open, and the two point at each other
        const uint32_t want = t == '}' ? '{' : t == ']' ? '[' : 'r';
        if (pt != want || v != (uint64_t)pp || (p.t.tape[pp] & TAPE_VALUE_MASK) != i + 1) return false;
        if (t == '}' && mj_x(p, i - s.d) != mj_x(p, pp + 1 - s.d)) return false;  // an object ends behind a key
        it.tag = t;
        if (t == 'r') {
            it.sep = i + 1 < s.hi ? '\n' : 0;
        } else {  // a container inside a container: the ',' in front of its next sibling goes behind the close
            const int32_t gv = p.par[pp - s.d];
            const uint32_t gt = gv >= 0 ? (uint32_t)(p.t.tape[gv + s.d] >> 56) : 0;
            if (gt == '{' || gt == '[') {
                if (i + 1 >= s.hi) return false;
                const uint32_t nt = (uint32_t)(p.t.tape[i + 1] >> 56);
                if (nt != '}' && nt != ']') it.sep = ',';
            }
        }
        it.len = (t != 'r') + (it.sep != 0);
        return true;
    }
    const bool key = pt == '{' && mj_x(p, i - s.d) == mj_x(p, pp + 1 - s.d);
    if (key && t != '"') return false;
    uint64_t end = i + 1;  // the word behind the value
    if (tape_value_tag(t)) {
        if (i + 1 >= s.hi) return false;
        const uint64_t pl = p.t.tape[i + 1];
        end = i + 2;
        it.payload = pl;
        if (t == '"') {
            if (!tape_string(p.t, w, pl, &it.s)) return false;
            it.slen = pl;
            it.len = 2;
            if (pl > MJ_SHORT)
                it.long_str = true;
            else
                for (uint64_t k = 0; k < pl; k++) it.len += fmt_escaped_len(it.s[k]);
        } else if (t == 'l') {
            it.len = fmt_i64<false>((int64_t)pl, nullptr);
        } else if (t == 'u') {
            it.len = fmt_u64<false>(pl, nullptr);
        } else {
            if (((pl >> 52) & 0x7ff) == 0x7ff) return false;  // NaN / Inf
            it.len = fmt_double<false>(pl, nullptr);
        }
    } else if (t == 't' || t == 'n') {
        it.len = 4;
    } else if (t == 'f') {
        it.len = 5;
    } else if (t == '{' || t == '[') {
        it.len = 1;
        it.tag = t;
        return true;  // (its ',' goes behind its close)
    } else {
        return false;  // unknown tag (the mutators' 'N' included)
    }
    it.tag = t;
    if (key) {
        it.sep = ':';
    } else if (pt == '{' || pt == '[') {  // (not behind a root's value, nor a cell's head)
        if (end <= i || end >= s.hi) return false;
        const uint32_t nt = (uint32_t)(p.t.tape[end] >> 56);
        if (nt != '}' && nt != ']') it.sep = ',';
    }
    it.len += it.sep != 0;
    return true;
}

// word i of the tape (when `in`): its item (tag 0 for value words) and, with the whole warp, a long string's escaped
// length
template <bool CELL>
__device__ __forceinline__ bool mj_load(const MarshalParams& p, bool in, uint64_t i, const MjSpan& s, MjItem& it, uint64_t& body) {
    it.len = 0;
    it.tag = 0;
    it.sep = 0;
    it.long_str = false;
    it.s = nullptr;
    it.slen = 0;
    bool ok = true;
    if (in && p.depth[i - s.d] != MJ_PAYLOAD) ok = mj_item<CELL>(p, i, s, it);
    if (!ok) it.long_str = false;
    body = 0;
    uint32_t m = __ballot_sync(FULL, it.long_str);
    const uint32_t lane = threadIdx.x & 31;
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(it.s), src));
        const uint64_t sl = __shfl_sync(FULL, it.slen, src);
        uint64_t acc = 0;
        for (uint64_t k = lane; k < sl; k += 32) acc += fmt_escaped_len(s[k]);
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(FULL, acc, d);
        if ((int)lane == src) body = acc;
    }
    it.len += body;
    return ok;
}

// KM4: checks + output bytes per tile
__global__ void __launch_bounds__(MJ_THREADS) mj_measure_kernel(const MarshalParams p) {
    __shared__ unsigned long long wsum[32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t acc = 0;
    bool bad = false;
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint64_t i = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS + threadIdx.x;
        MjItem it;
        uint64_t body;
        bad |= !mj_load<false>(p, i < p.t.n, i, MjSpan{0, p.t.n, 0}, it, body);
        acc += it.len;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && (p.h_total->d1 != 0 || hagg_out(*p.h_total, 1) != 1))
        bad = true;  // containers left open, or a string / number without its value word at the end
    if (__any_sync(FULL, bad) && lane == 0) atomicOr(p.err, 1ull);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(FULL, acc, d);
    if (lane == 0) wsum[warp] = acc;
    __syncthreads();
    if (warp == 0) {
        unsigned long long s = wsum[lane];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(FULL, s, d);
        if (lane == 0) p.len_tile[blockIdx.x] = MSum{s};
    }
}

__device__ __forceinline__ void mj_put(uint8_t* o, const char* s, uint32_t n) {
    for (uint32_t k = 0; k < n; k++) o[k] = (uint8_t)s[k];
}

// the bytes of item `it` at o, but for a long string's body (mj_put_long)
__device__ __forceinline__ void mj_put_item(const MjItem& it, uint64_t body, uint8_t* o) {
    switch (it.tag) {
    case '"':
        o[0] = '"';
        if (!it.long_str) {
            body = 0;
            for (uint64_t k = 0; k < it.slen; k++) body += fmt_escape(it.s[k], o + 1 + body);
        }
        o[1 + body] = '"';
        break;
    case 'l': fmt_i64<true>((int64_t)it.payload, o); break;
    case 'u': fmt_u64<true>(it.payload, o); break;
    case 'd': fmt_double<true>(it.payload, o); break;
    case 't': mj_put(o, "true", 4); break;
    case 'f': mj_put(o, "false", 5); break;
    case 'n': mj_put(o, "null", 4); break;
    case '{': case '}': case '[': case ']': o[0] = (uint8_t)it.tag; break;
    default: break;
    }
    if (it.sep) o[it.len - 1] = (uint8_t)it.sep;
}

// long strings: the warp escapes 32 bytes at a time, each lane one byte at its place in the scan of the lengths; the
// whole warp calls it, o is where the item of each lane goes
__device__ __forceinline__ void mj_put_long(const MjItem& it, uint8_t* o) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t m = __ballot_sync(FULL, it.long_str);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(it.s), src));
        const uint64_t sl = __shfl_sync(FULL, it.slen, src);
        uint8_t* d = reinterpret_cast<uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(o + 1), src));
        for (uint64_t k0 = 0; k0 < sl; k0 += 32) {
            const uint64_t k = k0 + lane;
            const uint8_t c = k < sl ? s[k] : 0;
            const uint32_t e = k < sl ? fmt_escaped_len(c) : 0;
            uint32_t inc = e;
#pragma unroll
            for (int dd = 1; dd < 32; dd <<= 1) {
                const uint32_t t = __shfl_up_sync(FULL, inc, dd);
                if ((int)lane >= dd) inc += t;
            }
            if (e) fmt_escape(c, d + inc - e);
            d += __shfl_sync(FULL, inc, 31);
        }
    }
}

// KM5: every word's bytes at the exclusive scan of the lengths
__global__ void __launch_bounds__(MJ_THREADS) mj_emit_kernel(const MarshalParams p) {
    uint64_t carry = tile_prefix(p.len_tile_pre, p.len_grp_pre, blockIdx.x).v;
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint64_t i = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS + threadIdx.x;
        MjItem it;
        uint64_t body;
        mj_load<false>(p, i < p.t.n, i, MjSpan{0, p.t.n, 0}, it, body);
        MSum total;
        const uint64_t off = carry + block_exclusive_scan(MSum{it.len}, total).v;
        carry += total.v;
        uint8_t* o = p.out + off;
        mj_put_item(it, body, o);
        mj_put_long(it, o);
    }
}

}  // namespace sj
