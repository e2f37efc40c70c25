// marshal.cuh -- Iter.MarshalJSON (parsed_json.go:394-556) on the device: a tape in HBM back to compact JSON text in HBM.
//
// The work is spread over tape words, not over roots, so a single-document tape runs as wide as an NDJSON one.  Each
// word-parallel step is one pass over the tape in tiles of MJ_TILE words:
//   KM1 mj_heads_reduce / KM2 mj_depth   which words are heads (not the value word of a string or number) and the
//        depth in front of every head: one scan of a per-word transfer function (HAgg), reduce then downsweep
//   K2d s2_min32 + s2_ansv (stage2_common.cuh)   the parent of every head: the nearest earlier head of smaller depth
//   KM3 mj_keys    F(j) = 1 for every non-close head whose parent is '{'; its per-tile counts and the in-tile parity of
//        its exclusive prefix (one bit per word).  A string in an object is a key when the parity over (object, string)
//        is even: a complete child container adds an even count, since every object inside it has an even number of
//        direct members
//   KM4 mj_measure  validation of the tape + every head's output length, per-tile sums
//   KM5 mj_emit     the exclusive scan of the lengths and the bytes
// The tile sums of KM1, KM3 and KM4 are scanned by scan_groups_kernel<T> (stage2_common.cuh), once per group of 1024
// tiles and once over the group totals.
#pragma once
#include "common.cuh"
#include "fmt.h"
#include "stage2_common.cuh"

namespace sj {

constexpr int MJ_THREADS = 1024;
constexpr int MJ_ROUNDS = 4;                        // a tile is MJ_ROUNDS rounds of one word per thread
constexpr uint64_t MJ_TILE = MJ_THREADS * MJ_ROUNDS;
constexpr uint64_t MJ_SHORT = 32;                   // longer strings are escaped by their whole warp
constexpr int32_t MJ_PAYLOAD = 0x7fffffff;          // depth entry of a word that is not a head
constexpr uint64_t MJ_VALUE_MASK = 0x00ffffffffffffffull;
constexpr uint64_t MJ_STRINGBUFBIT = 0x80000000000000ull;

// Transfer function of a run of tape words over the state "the next word is a head" (s = 1) or "is the value word of
// the string / number in front of it" (s = 0), and the depth change over the run in each case.  A word tagged
// '"', 'l', 'u' or 'd' flips the state, any other word sets it to 1, whatever it is.  T{} is the identity.
struct HAgg {
    uint32_t cst;  // 1: the state after the run is `val` whatever it was before; 0: it is s ^ val
    uint32_t val;
    int32_t d0, d1;  // depth change over the run when it starts in state 0 / 1
};
__device__ __forceinline__ uint32_t hagg_out(const HAgg& a, uint32_t s) { return a.cst ? a.val : (s ^ a.val); }
__device__ __forceinline__ HAgg agg_combine(const HAgg& a, const HAgg& b) {
    HAgg r;
    r.cst = a.cst | b.cst;
    r.val = b.cst ? b.val : (a.val ^ b.val);
    r.d0 = a.d0 + (hagg_out(a, 0) ? b.d1 : b.d0);
    r.d1 = a.d1 + (hagg_out(a, 1) ? b.d1 : b.d0);
    return r;
}
__device__ __forceinline__ HAgg agg_shfl_up(const HAgg& a, int d) {
    HAgg r;
    r.cst = __shfl_up_sync(FULL, a.cst, d);
    r.val = __shfl_up_sync(FULL, a.val, d);
    r.d0 = __shfl_up_sync(FULL, a.d0, d);
    r.d1 = __shfl_up_sync(FULL, a.d1, d);
    return r;
}

// a 64-bit count (KM3's F, KM4's output bytes)
struct MSum {
    uint64_t v;
};
__device__ __forceinline__ MSum agg_combine(const MSum& a, const MSum& b) { return MSum{a.v + b.v}; }
__device__ __forceinline__ MSum agg_shfl_up(const MSum& a, int d) { return MSum{__shfl_up_sync(FULL, a.v, d)}; }

__device__ __forceinline__ bool mj_value_tag(uint32_t t) { return t == '"' || t == 'l' || t == 'u' || t == 'd'; }
// root words: the open one points forward (one past its close), the close one back at its open
__device__ __forceinline__ bool mj_is_close(uint64_t w, uint64_t i) {
    const uint32_t t = (uint32_t)(w >> 56);
    return t == '}' || t == ']' || (t == 'r' && (w & MJ_VALUE_MASK) <= i);
}

__device__ __forceinline__ HAgg mj_word_agg(uint64_t w, uint64_t i) {
    const uint32_t t = (uint32_t)(w >> 56);
    HAgg a;
    a.cst = mj_value_tag(t) ? 0 : 1;
    a.val = 1;
    a.d0 = 0;
    a.d1 = (t == '{' || t == '[') ? 1 : (t == '}' || t == ']') ? -1 : t == 'r' ? ((w & MJ_VALUE_MASK) > i ? 1 : -1) : 0;
    return a;
}

// KM1: the transfer function of each tile (4 consecutive words per thread)
__global__ void __launch_bounds__(MJ_THREADS) mj_heads_reduce_kernel(const uint64_t* tape, uint64_t n, HAgg* tile_sum) {
    const uint64_t base = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)threadIdx.x * MJ_ROUNDS;
    HAgg a{};
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++)
        if (base + j < n) a = agg_combine(a, mj_word_agg(tape[base + j], base + j));
    HAgg total;
    block_exclusive_scan(a, total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// KM2: depth in front of every head (the tape starts at a head), MJ_PAYLOAD for the other words
__global__ void __launch_bounds__(MJ_THREADS) mj_depth_kernel(const uint64_t* tape, uint64_t n, const HAgg* tile_pre,
                                                             const HAgg* grp_pre, int32_t* depth) {
    const uint64_t base = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)threadIdx.x * MJ_ROUNDS;
    uint64_t w[MJ_ROUNDS];
    HAgg a{};
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++) {
        w[j] = base + j < n ? tape[base + j] : 0;
        if (base + j < n) a = agg_combine(a, mj_word_agg(w[j], base + j));
    }
    HAgg total;
    const HAgg ex = block_exclusive_scan(a, total);
    HAgg pre = agg_combine(agg_combine(grp_pre[blockIdx.x >> 10], tile_pre[blockIdx.x]), ex);
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++) {
        if (base + j >= n) break;
        depth[base + j] = hagg_out(pre, 1) ? pre.d1 : MJ_PAYLOAD;
        pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
}

// KM3: F per word; fbits = parity of F's in-tile exclusive prefix, tile_f = F's count per tile
__global__ void __launch_bounds__(MJ_THREADS) mj_keys_kernel(const uint64_t* tape, uint64_t n, const int32_t* depth,
                                                            const int32_t* par, uint32_t* fbits, MSum* tile_f) {
    __shared__ uint32_t cnt[MJ_ROUNDS * 32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t b[MJ_ROUNDS];
#pragma unroll
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint64_t i = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS + threadIdx.x;
        bool f = false;
        if (i < n && depth[i] != MJ_PAYLOAD && !mj_is_close(tape[i], i)) {
            const int32_t p = par[i];
            f = p >= 0 && (tape[p] >> 56) == '{';
        }
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
    const uint64_t* tape;
    uint64_t n;
    const uint8_t* msg;  // no-copy strings point into it
    uint64_t msg_len;
    const uint8_t* strings;  // Strings.B
    uint64_t strings_len;
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
    const uint64_t t = j / MJ_TILE;
    return (uint32_t)((p.f_grp_pre[t >> 10].v + p.f_tile_pre[t].v + (p.fbits[j >> 5] >> (j & 31))) & 1);
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

// What head i writes, after the checks of a foreign tape: false = malformed.  Every read stays inside the tape, the
// string buffer or the message.
__device__ bool mj_item(const MarshalParams& p, uint64_t i, MjItem& it) {
    const uint64_t w = p.tape[i];
    const uint32_t t = (uint32_t)(w >> 56);
    const uint64_t v = w & MJ_VALUE_MASK;
    const int32_t pp = p.par[i];
    uint32_t pt = 0;
    if (pp >= 0) {
        const uint64_t pw = p.tape[pp];
        pt = (uint32_t)(pw >> 56);
        if (!(pt == '{' || pt == '[' || (pt == 'r' && (pw & MJ_VALUE_MASK) > (uint64_t)pp))) return false;  // parent is no open
    }
    if (t == 'r' && v > i) return pp < 0;  // a root open writes nothing and sits at the top level
    if (pp < 0) return false;
    if (t == '}' || t == ']' || t == 'r') {  // close: its parent is its open, and the two point at each other
        const uint32_t want = t == '}' ? '{' : t == ']' ? '[' : 'r';
        if (pt != want || v != (uint64_t)pp || (p.tape[pp] & MJ_VALUE_MASK) != i + 1) return false;
        if (t == '}' && mj_x(p, i) != mj_x(p, pp + 1)) return false;  // an object ends behind a key
        it.tag = t;
        if (t == 'r') {
            it.sep = i + 1 < p.n ? '\n' : 0;
        } else {  // a container inside a container: the ',' in front of its next sibling goes behind the close
            const int32_t gp = p.par[pp];
            const uint32_t gt = gp >= 0 ? (uint32_t)(p.tape[gp] >> 56) : 0;
            if (gt == '{' || gt == '[') {
                if (i + 1 >= p.n) return false;
                const uint32_t nt = (uint32_t)(p.tape[i + 1] >> 56);
                if (nt != '}' && nt != ']') it.sep = ',';
            }
        }
        it.len = (t != 'r') + (it.sep != 0);
        return true;
    }
    const bool key = pt == '{' && mj_x(p, i) == mj_x(p, pp + 1);
    if (key && t != '"') return false;
    uint64_t end = i + 1;  // the word behind the value
    if (mj_value_tag(t)) {
        if (i + 1 >= p.n) return false;
        const uint64_t pl = p.tape[i + 1];
        end = i + 2;
        it.payload = pl;
        if (t == '"') {
            const bool sb = (v & MJ_STRINGBUFBIT) != 0;
            const uint64_t cap = sb ? p.strings_len : p.msg_len, off = sb ? v - MJ_STRINGBUFBIT : v;
            if (off > cap || pl > cap - off) return false;
            it.s = (sb ? p.strings : p.msg) + off;
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
    } else if (pt != 'r') {
        if (end <= i || end >= p.n) return false;
        const uint32_t nt = (uint32_t)(p.tape[end] >> 56);
        if (nt != '}' && nt != ']') it.sep = ',';
    }
    it.len += it.sep != 0;
    return true;
}

// word i of the tape: its item (tag 0 for value words) and, with the whole warp, a long string's escaped length
__device__ __forceinline__ bool mj_load(const MarshalParams& p, uint64_t i, MjItem& it, uint64_t& body) {
    it.len = 0;
    it.tag = 0;
    it.sep = 0;
    it.long_str = false;
    it.s = nullptr;
    it.slen = 0;
    bool ok = true;
    if (i < p.n && p.depth[i] != MJ_PAYLOAD) ok = mj_item(p, i, it);
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
        bad |= !mj_load(p, i, it, body);
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

// KM5: every word's bytes at the exclusive scan of the lengths
__global__ void __launch_bounds__(MJ_THREADS) mj_emit_kernel(const MarshalParams p) {
    const uint32_t lane = threadIdx.x & 31;
    uint64_t carry = p.len_grp_pre[blockIdx.x >> 10].v + p.len_tile_pre[blockIdx.x].v;
    for (int r = 0; r < MJ_ROUNDS; r++) {
        const uint64_t i = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)r * MJ_THREADS + threadIdx.x;
        MjItem it;
        uint64_t body;
        mj_load(p, i, it, body);
        MSum total;
        const uint64_t off = carry + block_exclusive_scan(MSum{it.len}, total).v;
        carry += total.v;
        uint8_t* o = p.out + off;
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
        // long strings: the warp escapes 32 bytes at a time, each lane one byte at its place in the scan of the lengths
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
}

}  // namespace sj
