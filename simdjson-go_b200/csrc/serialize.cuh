// serialize.cuh -- Serializer.Serialize / Deserialize (parsed_serialize.go:200-695) on the device, in the v3 wire format
// with uncompressed blocks (CompressNone): a tape in HBM to the stream in HBM, and the stream back to a tape.
//
// Stream layout (every block is its type byte 0 and the raw bytes):
//   3 | uvarint(bytes that follow) | uvarint(tape words) | 0 0 (no Strings.B block)
//   uvarint(message raw) uvarint(1 + raw) 0 <distinct string bytes>
//   uvarint(tags raw)    uvarint(1 + raw) 0 <one tag byte per head word>
//   uvarint(values raw)  uvarint(1 + raw) 0 <values, little endian>
// Per head word: '"' writes its offset into the message block and its length (8 bytes each); 'l' 'u' and a 'd' without
// flags their value word; a 'd' with flags is tag 'e' and writes the whole tag word and the value word; '{' '[' 'r' write
// payload - index (mod 2^64); '}' ']' 'n' 't' 'f' 'N' and tag 0 write nothing.
//
// String deduplication, the one intended difference from the reference: the reference keeps a 16 K-bucket table keyed
// by the per-process seeded runtime.memhash, so its output changes from run to run.  Here it is exact and
// first-occurrence: number the strings k = 0..m-1 in tape order, rep(k) = the smallest j with the same bytes; the message
// block is the bytes of every k with rep(k) == k in order of k, and string k points at rep(k)'s copy.  The output does
// not depend on thread scheduling nor on where a string's bytes lived (Strings.B or the message), and the message block
// is never larger than the reference's.
//
// Serialize, word-parallel passes over tiles of SZ_TILE words (= marshal.cuh's, so KM1's tile transfer functions serve):
//   KM1 mj_heads_reduce + scans          which words are heads
//   KS1 sz_count      checks + per-tile (tag bytes, value bytes, strings)
//   KS2 sz_index      the tape index of every string, by ordinal
//   KS3 sz_insert / KS4 sz_resolve, ordinal-parallel, one round per hash salt: every unresolved string's hash class
//       (an open-addressed table) takes its smallest ordinal by atomicMin; a string whose bytes equal that
//       representative's is resolved, the others (hash collisions) go to the next round with a new salt.  Strings
//       are hashed and compared by their whole warp, lanes with the same hash insert once.
//   KS5 sz_distinct   per-tile bytes of the distinct strings
//   KS6 sz_message    the message block and every distinct string's offset in it
//   KS7 sz_emit       tags and values
// Deserialize: KD0 dz_header (one thread) reads the block sizes; KD1 dz_count per tag (tape words, value bytes), scanned;
// KD2 dz_place marks which tag starts at each tape word; KD3 dz_check checks every open's close; KD4 dz_emit writes the tape.
#pragma once
#include "marshal.cuh"

namespace sj {

constexpr uint64_t SZ_TILE = 4096;   // words per tile of KS1 / KS2 / KS7 (MJ_TILE: KM1's tile sums are reused)
constexpr uint64_t SZ_OTILE = 4096;  // strings per tile of KS5 / KS6: 1024 threads x 4
constexpr int SZ_OTHREADS = 256;     // KS3 / KS4 blocks
constexpr uint64_t DZ_TILE = 4096;   // tags per tile of KD1 .. KD4: 1024 threads x 4
constexpr uint32_t SZ_UNRESOLVED = 0xffffffffu;
constexpr uint64_t SZ_EMPTY = ~0ull;
static_assert(SZ_TILE == MJ_TILE, "the serialize passes reuse KM1's tiles");

// ---------------------------------------------------------------------------------
// Serialize
// ---------------------------------------------------------------------------------
struct SzSum {
    uint64_t tags, vals, strs;
};
__device__ __forceinline__ SzSum agg_combine(const SzSum& a, const SzSum& b) { return SzSum{a.tags + b.tags, a.vals + b.vals, a.strs + b.strs}; }
__device__ __forceinline__ SzSum agg_shfl_up(const SzSum& a, int d) {
    return SzSum{__shfl_up_sync(FULL, a.tags, d), __shfl_up_sync(FULL, a.vals, d), __shfl_up_sync(FULL, a.strs, d)};
}

struct SerializeParams {
    const uint64_t* tape;
    uint64_t n;
    const uint8_t* msg;
    uint64_t msg_len;
    const uint8_t* strings;
    uint64_t strings_len;
    const HAgg* h_tile_pre;  // KM1's scans
    const HAgg* h_grp_pre;
    SzSum* c_tile;           // KS1 per-tile counts and their scans
    const SzSum* c_tile_pre;
    const SzSum* c_grp_pre;
    uint32_t* spos;          // tape index of string k
    uint32_t* rep;           // rep(k), SZ_UNRESOLVED until known
    uint32_t* slot;          // KS3: the table slot of string k
    uint64_t* keys;          // KS3: the hash table
    uint32_t* ords;          //      and the smallest ordinal of each hash
    uint64_t tab_mask;
    uint64_t hash_mask;      // the hash bits kept (all but for tests)
    uint64_t salt;
    uint64_t m;              // strings
    MSum* d_tile;            // KS5 per-tile distinct bytes and their scans
    const MSum* d_tile_pre;
    const MSum* d_grp_pre;
    uint64_t* moff;          // KS6: offset of string k's bytes in the message block (distinct strings only)
    unsigned long long* err;      // malformed tape
    unsigned long long* pending;  // KS4: strings left unresolved
    uint8_t* out;
    uint64_t msg_base, tags_base, vals_base;  // where the three blocks' bytes start in `out`
};

// what head word i writes: tag byte, value bytes, 1 if it is a string; false: the reference panics on it
__device__ __forceinline__ bool sz_item(const SerializeParams& p, uint64_t i, uint64_t w, uint32_t& tag, uint32_t& vals, uint32_t& str) {
    const uint32_t t = (uint32_t)(w >> 56);
    const uint64_t v = w & MJ_VALUE_MASK;
    tag = t;
    vals = 0;
    str = 0;
    switch (t) {
    case '"': {
        if (i + 1 >= p.n) return false;
        const uint64_t len = p.tape[i + 1];
        const bool sb = (v & MJ_STRINGBUFBIT) != 0;
        const uint64_t cap = sb ? p.strings_len : p.msg_len, off = v & (MJ_STRINGBUFBIT - 1);
        if (off > cap || len > cap - off) return false;
        vals = 16;
        str = 1;
        return true;
    }
    case 'l': case 'u': vals = 8; return i + 1 < p.n;
    case 'd':
        if (v) tag = 'e';
        vals = v ? 16 : 8;
        return i + 1 < p.n;
    case '{': case '[': case 'r': vals = 8; return true;
    case '}': case ']': case 'n': case 't': case 'f': case 'N': case 0: return true;
    default: return false;
    }
}

// the words of thread `threadIdx.x` of tile blockIdx.x (SZ_ROUNDS consecutive ones) and the head state in front of them
constexpr int SZ_ROUNDS = MJ_ROUNDS;
__device__ __forceinline__ HAgg sz_load(const SerializeParams& p, uint64_t base, uint64_t (&w)[SZ_ROUNDS]) {
    HAgg a{};
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++) {
        w[j] = base + j < p.n ? p.tape[base + j] : 0;
        if (base + j < p.n) a = agg_combine(a, mj_word_agg(w[j], base + j));
    }
    HAgg total;
    const HAgg ex = block_exclusive_scan(a, total);
    return agg_combine(agg_combine(p.h_grp_pre[blockIdx.x >> 10], p.h_tile_pre[blockIdx.x]), ex);
}

// KS1: checks and per-tile counts
__global__ void __launch_bounds__(MJ_THREADS) sz_count_kernel(const SerializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * SZ_TILE + (uint64_t)threadIdx.x * SZ_ROUNDS;
    uint64_t w[SZ_ROUNDS];
    HAgg pre = sz_load(p, base, w);
    SzSum s{0, 0, 0};
    bool bad = false;
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++) {
        if (base + j >= p.n) break;
        if (hagg_out(pre, 1)) {
            uint32_t tag, vals, str;
            bad |= !sz_item(p, base + j, w[j], tag, vals, str);
            s.tags++;
            s.vals += vals;
            s.strs += str;
        }
        pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
    if (__any_sync(FULL, bad) && (threadIdx.x & 31) == 0) atomicOr(p.err, 1ull);
    SzSum total;
    block_exclusive_scan(s, total);
    if (threadIdx.x == 0) p.c_tile[blockIdx.x] = total;
}

// KS2: spos[k] = tape index of string k
__global__ void __launch_bounds__(MJ_THREADS) sz_index_kernel(const SerializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * SZ_TILE + (uint64_t)threadIdx.x * SZ_ROUNDS;
    uint64_t w[SZ_ROUNDS];
    HAgg pre = sz_load(p, base, w);
    uint32_t str = 0;
    bool head[SZ_ROUNDS];
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++) {
        head[j] = base + j < p.n && hagg_out(pre, 1);
        str += head[j] && (w[j] >> 56) == '"';
        if (base + j < p.n) pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
    SzSum total;
    uint64_t k = p.c_grp_pre[blockIdx.x >> 10].strs + p.c_tile_pre[blockIdx.x].strs + block_exclusive_scan(SzSum{0, 0, str}, total).strs;
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++)
        if (head[j] && (w[j] >> 56) == '"') p.spos[k++] = (uint32_t)(base + j);
}

// the bytes of string k (checked by KS1)
__device__ __forceinline__ const uint8_t* sz_str(const SerializeParams& p, uint64_t k, uint64_t& len) {
    const uint32_t i = p.spos[k];
    const uint64_t v = p.tape[i] & MJ_VALUE_MASK;
    len = p.tape[i + 1];
    return (v & MJ_STRINGBUFBIT) ? p.strings + (v & (MJ_STRINGBUFBIT - 1)) : p.msg + v;
}

__host__ __device__ __forceinline__ uint64_t sz_mix(uint64_t x) {  // splitmix64's finalizer: a bijection
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// the hash of string (s, len) under `salt`, computed by the whole warp: a sum over (index, byte) pairs, so it does not
// depend on how the bytes are split among lanes
__device__ __forceinline__ uint64_t sz_warp_hash(const uint8_t* s, uint64_t len, uint64_t salt) {
    const uint32_t lane = threadIdx.x & 31;
    uint64_t h = 0;
    for (uint64_t k = lane; k < len; k += 32) h += sz_mix(((k << 8) | s[k]) ^ salt);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) h += __shfl_xor_sync(FULL, h, d);
    return sz_mix(h ^ sz_mix(len + salt));
}

// do (a, la) and (b, lb) hold the same bytes?  whole warp
__device__ __forceinline__ bool sz_warp_equal(const uint8_t* a, uint64_t la, const uint8_t* b, uint64_t lb) {
    if (la != lb) return false;
    const uint32_t lane = threadIdx.x & 31;
    bool eq = true;
    for (uint64_t k0 = 0; k0 < la && eq; k0 += 32) {
        const uint64_t k = k0 + lane;
        eq = __all_sync(FULL, k >= la || a[k] == b[k]);
    }
    return eq;
}

// KS3: every unresolved string's hash class takes its smallest ordinal
__global__ void __launch_bounds__(SZ_OTHREADS) sz_insert_kernel(const SerializeParams p) {
    const uint64_t k = (uint64_t)blockIdx.x * SZ_OTHREADS + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const bool act = k < p.m && p.rep[k] == SZ_UNRESOLVED;
    uint64_t h = 0;
    uint32_t m = __ballot_sync(FULL, act);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        uint64_t len;
        const uint8_t* s = sz_str(p, (uint64_t)blockIdx.x * SZ_OTHREADS + (threadIdx.x & ~31u) + src, len);
        const uint64_t hw = sz_warp_hash(s, len, p.salt);
        if ((int)lane == src) h = hw;
    }
    h &= p.hash_mask;
    if (h == SZ_EMPTY) h--;
    // lanes with the same hash insert once, through their first (smallest) ordinal
    const uint32_t act_mask = __ballot_sync(FULL, act);
    if (!act) return;
    const uint32_t same = __match_any_sync(act_mask, h);
    const int leader = __ffs(same) - 1;
    uint64_t sl = 0;
    if ((int)lane == leader) {
        sl = h & p.tab_mask;
        for (;;) {
            uint64_t cur = p.keys[sl];
            if (cur == SZ_EMPTY) cur = atomicCAS((unsigned long long*)&p.keys[sl], SZ_EMPTY, h);
            if (cur == SZ_EMPTY || cur == h) break;
            sl = (sl + 1) & p.tab_mask;
        }
        atomicMin(&p.ords[sl], (uint32_t)k);
    }
    sl = __shfl_sync(same, sl, leader);
    p.slot[k] = (uint32_t)sl;
}

// KS4: a string whose bytes equal its class's smallest ordinal's is resolved; the others wait for the next salt
__global__ void __launch_bounds__(SZ_OTHREADS) sz_resolve_kernel(const SerializeParams p) {
    const uint64_t k = (uint64_t)blockIdx.x * SZ_OTHREADS + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const bool act = k < p.m && p.rep[k] == SZ_UNRESOLVED;
    const uint32_t r = act ? p.ords[p.slot[k]] : 0;
    bool eq = false;
    uint32_t m = __ballot_sync(FULL, act);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint64_t ks = (uint64_t)blockIdx.x * SZ_OTHREADS + (threadIdx.x & ~31u) + src;
        const uint64_t rs = __shfl_sync(FULL, r, src);
        uint64_t la, lb;
        const uint8_t* a = sz_str(p, ks, la);
        const uint8_t* b = sz_str(p, rs, lb);
        const bool e = ks == rs || sz_warp_equal(a, la, b, lb);
        if ((int)lane == src) eq = e;
    }
    if (!act) return;
    if (eq)
        p.rep[k] = r;
    else
        atomicAdd(p.pending, 1ull);
}

// KS5: bytes of the distinct strings per tile of SZ_OTILE ordinals
__device__ __forceinline__ uint64_t sz_distinct_len(const SerializeParams& p, uint64_t k) {
    if (k >= p.m || p.rep[k] != k) return 0;
    return p.tape[p.spos[k] + 1];
}

__global__ void __launch_bounds__(1024) sz_distinct_kernel(const SerializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * SZ_OTILE + (uint64_t)threadIdx.x * 4;
    uint64_t s = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) s += sz_distinct_len(p, base + j);
    MSum total;
    block_exclusive_scan(MSum{s}, total);
    if (threadIdx.x == 0) p.d_tile[blockIdx.x] = total;
}

// KS6: the message block (by warps, one distinct string at a time) and moff of every distinct string
__global__ void __launch_bounds__(1024) sz_message_kernel(const SerializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * SZ_OTILE + (uint64_t)threadIdx.x * 4;
    const uint32_t lane = threadIdx.x & 31;
    uint64_t len[4], s = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        len[j] = sz_distinct_len(p, base + j);
        s += len[j];
    }
    MSum total;
    uint64_t off = p.d_grp_pre[blockIdx.x >> 10].v + p.d_tile_pre[blockIdx.x].v + block_exclusive_scan(MSum{s}, total).v;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const bool d = base + j < p.m && p.rep[base + j] == base + j;
        if (d) p.moff[base + j] = off;
        uint32_t m = __ballot_sync(FULL, d && len[j] > 0);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const uint64_t ks = __shfl_sync(FULL, base + j, src);
            const uint64_t o = __shfl_sync(FULL, off, src);
            uint64_t l;
            const uint8_t* str = sz_str(p, ks, l);
            uint8_t* dst = p.out + p.msg_base + o;
            for (uint64_t k = lane; k < l; k += 32) dst[k] = str[k];
        }
        off += len[j];
    }
}

__device__ __forceinline__ void sz_put64(uint8_t* o, uint64_t v) {
#pragma unroll
    for (int b = 0; b < 8; b++) o[b] = (uint8_t)(v >> (8 * b));
}

// KS7: one tag byte per head word and its values
__global__ void __launch_bounds__(MJ_THREADS) sz_emit_kernel(const SerializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * SZ_TILE + (uint64_t)threadIdx.x * SZ_ROUNDS;
    uint64_t w[SZ_ROUNDS];
    HAgg pre = sz_load(p, base, w);
    bool head[SZ_ROUNDS];
    SzSum s{0, 0, 0};
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++) {
        head[j] = base + j < p.n && hagg_out(pre, 1);
        if (head[j]) {
            uint32_t tag, vals, str;
            sz_item(p, base + j, w[j], tag, vals, str);
            s.tags++;
            s.vals += vals;
            s.strs += str;
        }
        if (base + j < p.n) pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
    SzSum total;
    const SzSum ex = block_exclusive_scan(s, total);
    SzSum at = agg_combine(agg_combine(p.c_grp_pre[blockIdx.x >> 10], p.c_tile_pre[blockIdx.x]), ex);
#pragma unroll
    for (int j = 0; j < SZ_ROUNDS; j++) {
        if (!head[j]) continue;
        const uint64_t i = base + j;
        uint32_t tag, vals, str;
        sz_item(p, i, w[j], tag, vals, str);
        p.out[p.tags_base + at.tags] = (uint8_t)tag;
        uint8_t* o = p.out + p.vals_base + at.vals;
        switch (tag) {
        case '"':
            sz_put64(o, p.moff[p.rep[at.strs]]);
            sz_put64(o + 8, p.tape[i + 1]);
            break;
        case 'e': sz_put64(o, w[j]); sz_put64(o + 8, p.tape[i + 1]); break;
        case 'l': case 'u': case 'd': sz_put64(o, p.tape[i + 1]); break;
        case '{': case '[': case 'r': sz_put64(o, (w[j] & MJ_VALUE_MASK) - i); break;
        default: break;
        }
        at.tags++;
        at.vals += vals;
        at.strs += str;
    }
}

// ---------------------------------------------------------------------------------
// Deserialize
// ---------------------------------------------------------------------------------
enum : uint32_t { DZ_OK = 0, DZ_BAD = 1, DZ_UNSUPPORTED = 2 };

struct DzHeader {
    uint32_t status;
    uint32_t pad;
    uint64_t tape_words, strings_len, msg_len, ntags, nvals;
    uint64_t strings_at, msg_at, tags_at, vals_at;  // where each block's raw bytes start in the stream
};

// binary.ReadUvarint: false on a short input or an overflow
__device__ __forceinline__ bool dz_uvarint(const uint8_t* s, uint64_t len, uint64_t& at, uint64_t& x) {
    x = 0;
    for (int i = 0, sh = 0; i < 10; i++, sh += 7) {
        if (at >= len) return false;
        const uint8_t b = s[at++];
        if (b < 0x80) {
            if (i == 9 && b > 1) return false;
            x |= (uint64_t)b << sh;
            return true;
        }
        x |= (uint64_t)(b & 0x7f) << sh;
    }
    return false;
}

// decBlock (parsed_serialize.go:697-756) for a block of `raw` bytes: DZ_OK with `data` at its bytes, DZ_BAD or
// DZ_UNSUPPORTED (S2 / zstd: the stream may be fine, but only uncompressed blocks are read here)
__device__ __forceinline__ uint32_t dz_block(const uint8_t* s, uint64_t len, uint64_t& at, uint64_t raw, uint64_t& data) {
    uint64_t size;
    if (!dz_uvarint(s, len, at, size)) return DZ_BAD;
    if (size > len - at) return DZ_BAD;
    data = at;
    if (size == 0 && raw == 0) return DZ_OK;
    if (size < 1) return DZ_BAD;
    const uint8_t typ = s[at++];
    size--;
    data = at;
    at += size;
    if (typ == 1 || typ == 2) return DZ_UNSUPPORTED;
    if (typ != 0 || size != raw) return DZ_BAD;
    return DZ_OK;
}

// KD0: the header, read as Deserialize reads it (parsed_serialize.go:466-570); S2 / zstd blocks are reported only
// when nothing else is wrong with what can be read
__global__ void dz_header_kernel(const uint8_t* s, uint64_t len, DzHeader* h) {
    DzHeader r{};
    uint64_t at = 0, c;
    uint32_t st = DZ_OK;
    r.status = DZ_BAD;
    if (len < 1 || s[at++] > 3) {
        *h = r;
        return;
    }
    if (!dz_uvarint(s, len, at, c) || (int64_t)c > (int64_t)(len - at)) {  // (Go compares int(c))
        *h = r;
        return;
    }
    uint32_t b;
    if (!dz_uvarint(s, len, at, r.tape_words) || !dz_uvarint(s, len, at, r.strings_len)) goto done;
    if ((b = dz_block(s, len, at, r.strings_len, r.strings_at)) == DZ_BAD) goto done;
    st |= b;
    if (!dz_uvarint(s, len, at, r.msg_len)) goto done;
    if ((b = dz_block(s, len, at, r.msg_len, r.msg_at)) == DZ_BAD) goto done;
    st |= b;
    if (!dz_uvarint(s, len, at, r.ntags)) goto done;
    if ((b = dz_block(s, len, at, r.ntags, r.tags_at)) == DZ_BAD) goto done;
    st |= b;
    if (!dz_uvarint(s, len, at, r.nvals)) goto done;
    if ((b = dz_block(s, len, at, r.nvals, r.vals_at)) == DZ_BAD) goto done;
    st |= b;
    r.status = st;
done:
    *h = r;
}

// per tag: tape words, value bytes, opens and closes, and the run of 'N' tags at the end
struct DzAgg {
    uint64_t words, vals;
    uint32_t opens, closes;
    uint32_t tags, trail;  // tags in the run; 'N' tags at its end
};
__device__ __forceinline__ DzAgg agg_combine(const DzAgg& a, const DzAgg& b) {
    return DzAgg{a.words + b.words, a.vals + b.vals, a.opens + b.opens, a.closes + b.closes, a.tags + b.tags,
                 b.trail == b.tags ? a.trail + b.trail : b.trail};
}
__device__ __forceinline__ DzAgg agg_shfl_up(const DzAgg& a, int d) {
    return DzAgg{__shfl_up_sync(FULL, a.words, d), __shfl_up_sync(FULL, a.vals, d), __shfl_up_sync(FULL, a.opens, d),
                 __shfl_up_sync(FULL, a.closes, d), __shfl_up_sync(FULL, a.tags, d), __shfl_up_sync(FULL, a.trail, d)};
}

// the aggregate of one tag; false for a tag Deserialize does not know
__device__ __forceinline__ bool dz_tag(uint32_t t, DzAgg& a) {
    a = DzAgg{1, 0, 0, 0, 1, 0};
    switch (t) {
    case '"': case 'e': a.words = 2; a.vals = 16; return true;
    case 'l': case 'u': case 'd': a.words = 2; a.vals = 8; return true;
    case '{': case '[': a.vals = 8; a.opens = 1; return true;
    case 'r': a.vals = 8; return true;
    case '}': case ']': a.closes = 1; return true;
    case 'n': case 't': case 'f': case 0: return true;
    case 'N': a.trail = 1; return true;
    default: return false;
    }
}

struct DeserializeParams {
    const uint8_t* in;
    const DzHeader* h;
    uint64_t ntags;
    DzAgg* tile;  // KD1 per-tile aggregates and their scans
    const DzAgg* tile_pre;
    const DzAgg* grp_pre;
    const DzAgg* total;
    uint8_t* ptag;     // KD2: the tag that starts at each tape word, 1 for a value word
    uint32_t* hit;     // KD3: one bit per tape word, set by the open that names it as its close
    unsigned long long* err;
    uint64_t* tape;
};

__device__ __forceinline__ uint64_t dz_get64(const uint8_t* s) {
    uint64_t v = 0;
#pragma unroll
    for (int b = 0; b < 8; b++) v |= (uint64_t)s[b] << (8 * b);
    return v;
}

// the DZ_ROUNDS tags of this thread, their aggregates and the aggregate in front of the first
constexpr int DZ_ROUNDS = 4;
__device__ __forceinline__ DzAgg dz_load(const DeserializeParams& p, uint64_t base, uint32_t (&t)[DZ_ROUNDS], bool with_pre,
                                         bool& bad) {
    const uint8_t* tags = p.in + p.h->tags_at;
    DzAgg s{};
    bad = false;
#pragma unroll
    for (int j = 0; j < DZ_ROUNDS; j++) {
        t[j] = base + j < p.ntags ? tags[base + j] : 0;
        if (base + j < p.ntags) {
            DzAgg a;
            bad |= !dz_tag(t[j], a);
            s = agg_combine(s, a);
        }
    }
    DzAgg total;
    const DzAgg ex = block_exclusive_scan(s, total);
    if (!with_pre) {
        if (threadIdx.x == 0) p.tile[blockIdx.x] = total;
        return s;
    }
    return agg_combine(agg_combine(p.grp_pre[blockIdx.x >> 10], p.tile_pre[blockIdx.x]), ex);
}

// KD1: per-tile aggregates; unknown tags
__global__ void __launch_bounds__(1024) dz_count_kernel(const DeserializeParams p) {
    uint32_t t[DZ_ROUNDS];
    bool bad;
    dz_load(p, (uint64_t)blockIdx.x * DZ_TILE + (uint64_t)threadIdx.x * DZ_ROUNDS, t, false, bad);
    if (__any_sync(FULL, bad) && (threadIdx.x & 31) == 0) atomicOr(p.err, 1ull);
}

// KD2: which tag starts at each tape word (the totals are checked first: with words == tape length every word is
// covered once)
__global__ void __launch_bounds__(1024) dz_place_kernel(const DeserializeParams p) {
    const uint64_t n = p.h->tape_words;
    if (p.total->words != n || p.total->vals != p.h->nvals || p.total->opens != p.total->closes) {
        if (threadIdx.x == 0) atomicOr(p.err, 1ull);
        return;
    }
    const uint64_t base = (uint64_t)blockIdx.x * DZ_TILE + (uint64_t)threadIdx.x * DZ_ROUNDS;
    uint32_t t[DZ_ROUNDS];
    bool bad;
    DzAgg at = dz_load(p, base, t, true, bad);
#pragma unroll
    for (int j = 0; j < DZ_ROUNDS; j++) {
        if (base + j >= p.ntags) break;
        DzAgg a;
        dz_tag(t[j], a);
        p.ptag[at.words] = (uint8_t)t[j];
        if (a.words == 2) p.ptag[at.words + 1] = 1;
        at = agg_combine(at, a);
    }
}

// KD3: every open names a later word that holds its matching close, no close is named twice, every root link stays
// inside the tape
__global__ void __launch_bounds__(1024) dz_check_kernel(const DeserializeParams p) {
    const uint64_t n = p.h->tape_words;
    if (p.total->words != n || p.total->vals != p.h->nvals || p.total->opens != p.total->closes) return;  // (KD2 said so)
    const uint64_t base = (uint64_t)blockIdx.x * DZ_TILE + (uint64_t)threadIdx.x * DZ_ROUNDS;
    const uint8_t* vals = p.in + p.h->vals_at;
    uint32_t t[DZ_ROUNDS];
    bool bad;
    DzAgg at = dz_load(p, base, t, true, bad);
    bad = false;
#pragma unroll
    for (int j = 0; j < DZ_ROUNDS; j++) {
        if (base + j >= p.ntags) break;
        DzAgg a;
        dz_tag(t[j], a);
        if (t[j] == '{' || t[j] == '[' || t[j] == 'r') {
            const uint64_t val = dz_get64(vals + at.vals) + at.words;
            if (val > n) {
                bad = true;
            } else if (t[j] != 'r') {
                const uint64_t c = val - 1;
                if (val == 0 || c <= at.words || p.ptag[c] != (t[j] == '{' ? '}' : ']')) {
                    bad = true;
                } else {
                    const uint32_t bit = 1u << (c & 31);
                    if (atomicOr(&p.hit[c >> 5], bit) & bit) bad = true;
                }
            }
        }
        at = agg_combine(at, a);
    }
    if (__any_sync(FULL, bad) && (threadIdx.x & 31) == 0) atomicOr(p.err, 1ull);
}

// KD4: the tape, as Deserialize writes it (parsed_serialize.go:581-683).  A run of k 'N' tags becomes 'N' words with
// k, k-1, .., 1, written by the thread of the tag behind the run (the last run by the last tag's thread).
__device__ __forceinline__ void dz_nops(uint64_t* tape, uint64_t end, uint32_t k) {
    for (uint32_t r = 0; r < k; r++) tape[end - k + r] = ((uint64_t)'N' << 56) | (uint64_t)(k - r);
}

__global__ void __launch_bounds__(1024) dz_emit_kernel(const DeserializeParams p) {
    const uint64_t base = (uint64_t)blockIdx.x * DZ_TILE + (uint64_t)threadIdx.x * DZ_ROUNDS;
    const uint8_t* vals = p.in + p.h->vals_at;
    uint32_t t[DZ_ROUNDS];
    bool bad;
    DzAgg at = dz_load(p, base, t, true, bad);
#pragma unroll
    for (int j = 0; j < DZ_ROUNDS; j++) {
        if (base + j >= p.ntags) break;
        DzAgg a;
        dz_tag(t[j], a);
        const uint64_t pos = at.words, tw = (uint64_t)t[j] << 56;
        const uint8_t* v = vals + at.vals;
        if (t[j] != 'N' && at.trail) dz_nops(p.tape, pos, at.trail);
        switch (t[j]) {
        case '"': p.tape[pos] = tw | dz_get64(v); p.tape[pos + 1] = dz_get64(v + 8); break;
        case 'l': case 'u': case 'd': p.tape[pos] = tw; p.tape[pos + 1] = dz_get64(v); break;
        case 'e': p.tape[pos] = dz_get64(v); p.tape[pos + 1] = dz_get64(v + 8); break;
        case 'n': case 't': case 'f': case 0: p.tape[pos] = tw; break;
        case '{': case '[': {
            const uint64_t val = dz_get64(v) + pos;
            p.tape[pos] = tw | val;
            p.tape[val - 1] = ((uint64_t)(t[j] == '{' ? '}' : ']') << 56) | pos;
            break;
        }
        case 'r': p.tape[pos] = tw | (dz_get64(v) + pos); break;
        default: break;  // '}' ']': written by their open; 'N': by the tag behind the run
        }
        at = agg_combine(at, a);
        if (base + j + 1 == p.ntags && at.trail) dz_nops(p.tape, at.words, at.trail);
    }
}

}  // namespace sj
