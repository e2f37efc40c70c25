// find_json.cuh -- the JSON cells of the device find (SJ_FIND_KIND_JSON): Element.Iter.MarshalJSON() of every found
// element (parsed_json.go:394-556), into the variable-length columns STRING cells use.
//
// A cell is the found element's restricted tape [head, head + len) (KF3, find.cuh).  Within one path these ranges are
// disjoint and in row order on every tape the parser or Deserialize writes, so laid end to end they form the path's
// virtual word space of W words, at most the tape.  The work is spread over those words, not over cells: one cell may
// be nearly the whole tape, and a million cells may be two words each.  A path's words run through marshal.cuh's
// passes in a segmented form, whose state restarts at every cell head, so nothing outside a cell changes its text:
//   KJ0 fj_prefix        V: the exclusive scan of every JSON cell's words (after fd_len_reduce and its scans); a
//       word's cell is a binary search in V
//   KJ1 fj_heads_reduce  KM1 with a reset at every cell head: the head state and the depth start over (FjAgg)
//   KJ2 fj_depth         the depth in front of every head, 0 at a cell head; at a cell's last word the check that it
//       ends at depth 0 in front of a head (no container left open, no string or number without its value word)
//   K2d                  the parents (each cell head at depth 0 is a parent of nothing outside its cell)
//   KM3 mj_keys          over FjWords: the key parity.  A key is told by the parity between it and its object's
//       first member, both inside the cell, so it needs no reset
//   KJ4 fj_measure       mj_item<true>'s checks and every word's output length, scanned in the tile; a cell head's
//       and a cell's last word's in-tile prefixes (length, malformed words) into c_lo / c_hi, per-tile totals
//   KJ5 fj_finish        per cell: its text length and status into KF3's slen / val / st, and its first byte's place
//       in the path's text scan (jbase)
//   KJ6 fj_emit          after KF5: each word's bytes at its cell's column offset + its place in the cell
#pragma once
#include "find.cuh"
#include "marshal.cuh"

namespace sj {

// JSON path j's virtual word space: word v lies in the cell r with V[cell0 + r] - v0 <= v < V[cell0 + r + 1] - v0
struct FjWords {
    const uint64_t* tape;
    uint64_t n;           // W
    const uint64_t* V;    // exclusive scan of the words of every JSON cell, one entry more than cells
    const int64_t* head;  // KF3's head index of the path's cells, by row
    uint64_t cell0, rows, v0;

    __device__ __forceinline__ uint64_t cell(uint64_t v) const {  // the last row whose start is <= v
        const uint64_t x = v0 + v;
        uint64_t lo = 0, hi = rows;
        while (hi - lo > 1) {
            const uint64_t mid = (lo + hi) >> 1;
            if (V[cell0 + mid] <= x) lo = mid;
            else hi = mid;
        }
        return lo;
    }
    // row r's first virtual word: row r's cell spans [vstart(r), vstart(r + 1))
    __device__ __forceinline__ uint64_t vstart(uint64_t r) const { return V[cell0 + r] - v0; }
    // KM3's F over the virtual words (mj_keys_kernel)
    __device__ __forceinline__ bool f(uint64_t v, const int32_t* depth, const int32_t* par) const;
};

// where virtual word v sits: its row, its tape index and its cell's span
struct FjWord {
    uint64_t r, i;
    MjSpan s;
    bool first, last;
};
__device__ __forceinline__ FjWord fj_at(const FjWords& m, uint64_t v) {
    FjWord x;
    x.r = m.cell(v);
    const uint64_t a = m.vstart(x.r), b = m.vstart(x.r + 1);
    const uint64_t lo = (uint64_t)m.head[x.r];
    x.s = MjSpan{lo, lo + (b - a), (int64_t)(lo - a)};
    x.i = v + (uint64_t)x.s.d;
    x.first = v == a;
    x.last = v + 1 == b;
    return x;
}

__device__ __forceinline__ bool FjWords::f(uint64_t v, const int32_t* depth, const int32_t* par) const {
    if (v >= n || depth[v] == MJ_PAYLOAD) return false;
    const FjWord x = fj_at(*this, v);
    if (mj_is_close(tape[x.i], x.i)) return false;
    const int32_t p = par[v];
    return p >= 0 && (tape[p + x.s.d] >> 56) == '{';
}

// HAgg with a reset: a cell head's word puts the state "head, depth 0" in front of itself, whatever came before
struct FjAgg {
    HAgg h;
    uint32_t reset;
};
__device__ __forceinline__ FjAgg agg_combine(const FjAgg& a, const FjAgg& b) {
    return b.reset ? b : FjAgg{agg_combine(a.h, b.h), a.reset};
}
__device__ __forceinline__ FjAgg agg_shfl_up(const FjAgg& a, int d) {
    return FjAgg{agg_shfl_up(a.h, d), __shfl_up_sync(FULL, a.reset, d)};
}
__device__ __forceinline__ FjAgg fj_word_agg(uint64_t w, uint64_t i, bool first) {
    const HAgg a = mj_word_agg(w, i);
    if (!first) return FjAgg{a, 0};
    return FjAgg{HAgg{1, hagg_out(a, 1), a.d1, a.d1}, 1};
}

// the (output bytes, malformed words) of a run of words
struct JSum {
    uint64_t len, bad;
};
__device__ __forceinline__ JSum agg_combine(const JSum& a, const JSum& b) { return JSum{a.len + b.len, a.bad + b.bad}; }
__device__ __forceinline__ JSum agg_shfl_up(const JSum& a, int d) {
    return JSum{__shfl_up_sync(FULL, a.len, d), __shfl_up_sync(FULL, a.bad, d)};
}

// KJ0: V[k] = the exclusive prefix of jlen at k, in place, and V[n] = the total (after fd_len_reduce and its scans)
__global__ void __launch_bounds__(TAPE_THREADS) fj_prefix_kernel(uint64_t* V, uint64_t n, const MSum* tile_pre, const MSum* grp_pre) {
    uint64_t carry = tile_prefix(tile_pre, grp_pre, blockIdx.x).v;
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        const uint64_t k = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)j * TAPE_THREADS + threadIdx.x;
        const uint64_t len = k < n ? V[k] : 0;
        MSum total;
        const uint64_t off = carry + block_exclusive_scan(MSum{len}, total).v;
        carry += total.v;
        if (k < n) V[k] = off;
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) V[n] = carry;
}

// this thread's TAPE_ROUNDS words from `base` on, with each one's place (0 past W)
__device__ __forceinline__ FjAgg fj_words_agg(const FjWords& m, uint64_t base, uint64_t (&w)[TAPE_ROUNDS], FjWord (&x)[TAPE_ROUNDS]) {
    FjAgg a{};
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        w[j] = 0;
        if (base + j >= m.n) continue;
        x[j] = j && !x[j - 1].last ? FjWord{x[j - 1].r, x[j - 1].i + 1, x[j - 1].s, false, x[j - 1].i + 2 == x[j - 1].s.hi}
                                   : fj_at(m, base + j);
        w[j] = m.tape[x[j].i];
        a = agg_combine(a, fj_word_agg(w[j], x[j].i, x[j].first));
    }
    return a;
}

// which of this thread's TAPE_ROUNDS words from `base` on are heads (bit j; a cell's first word is none), with their
// places in x: the words of fj_words_agg, judged by KJ1's segmented head scan (tile_pre / grp_pre); numeric: every
// other word from the one after the cell's first instead, without the scan (the heads of a numeric list's walk);
// direct: only the heads directly inside the cell's scope (depth 1).  The whole block calls it.
__device__ __forceinline__ uint32_t fj_heads(const FjWords& m, const FjAgg* tile_pre, const FjAgg* grp_pre, uint64_t base,
                                             FjWord (&x)[TAPE_ROUNDS], bool numeric, bool direct) {
    uint64_t w[TAPE_ROUNDS];
    const FjAgg a = fj_words_agg(m, base, w, x);
    uint32_t h = 0;
    if (numeric) {
#pragma unroll
        for (int j = 0; j < TAPE_ROUNDS; j++)
            if (base + j < m.n && !x[j].first && !((x[j].i - x[j].s.lo - 1) & 1)) h |= 1u << j;
        return h;
    }
    FjAgg total;
    FjAgg pre = agg_combine(tile_prefix(tile_pre, grp_pre, blockIdx.x), block_exclusive_scan(a, total));
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (base + j >= m.n) break;
        if (!x[j].first && hagg_out(pre.h, 1) && (!direct || pre.h.d1 == 1)) h |= 1u << j;
        pre = agg_combine(pre, fj_word_agg(w[j], x[j].i, x[j].first));
    }
    return h;
}

// a head at virtual word v that stops row r's walk lowers stop[r] to v with atomicMin (stop preset to ~0: none).  The
// whole warp calls it for its words j: a lane's word j lies behind the lower lanes' words j, so the lowest lane of a
// row has the warp's minimum and is the one that writes.
__device__ __forceinline__ void fj_lower_stop(uint64_t* stop, bool stops, uint64_t r, uint64_t v) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t g = __match_any_sync(FULL, stops ? r : ~0ull);
    if (stops && !(g & ((1u << lane) - 1)) && v < *(volatile uint64_t*)&stop[r])
        atomicMin(reinterpret_cast<unsigned long long*>(&stop[r]), (unsigned long long)v);
}

// a cell's scan in front of its first word a and behind its last word b - 1: the tile prefix (tiles of TILE words) of
// each word's tile with the cell's in-tile prefixes c_lo / c_hi
template <class A>
struct FjEnds {
    A lo, hi;
};
template <uint64_t TILE, class A>
__device__ __forceinline__ FjEnds<A> fj_ends(const A* tile_pre, const A* grp_pre, const A& c_lo, const A& c_hi, uint64_t a, uint64_t b) {
    return FjEnds<A>{agg_combine(tile_prefix(tile_pre, grp_pre, a / TILE), c_lo),
                     agg_combine(tile_prefix(tile_pre, grp_pre, (b - 1) / TILE), c_hi)};
}

// KJ1: the segmented transfer function of each tile
__global__ void __launch_bounds__(TAPE_THREADS) fj_heads_reduce_kernel(const FjWords m, FjAgg* tile_sum) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    uint64_t w[TAPE_ROUNDS];
    FjWord x[TAPE_ROUNDS];
    FjAgg total;
    block_exclusive_scan(fj_words_agg(m, base, w, x), total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// KJ2: depth in front of every head (0 at a cell head), MJ_PAYLOAD for the other words; cbad[r] = 1 when cell r does
// not end at depth 0 in front of a head
__global__ void __launch_bounds__(TAPE_THREADS) fj_depth_kernel(const FjWords m, const FjAgg* tile_pre, const FjAgg* grp_pre,
                                                               int32_t* depth, uint8_t* cbad) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    uint64_t w[TAPE_ROUNDS];
    FjWord x[TAPE_ROUNDS];
    FjAgg total;
    const FjAgg ex = block_exclusive_scan(fj_words_agg(m, base, w, x), total);
    FjAgg pre = agg_combine(tile_prefix(tile_pre, grp_pre, blockIdx.x), ex);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (base + j >= m.n) break;
        depth[base + j] = x[j].first ? 0 : hagg_out(pre.h, 1) ? pre.h.d1 : MJ_PAYLOAD;
        pre = agg_combine(pre, fj_word_agg(w[j], x[j].i, x[j].first));
        if (x[j].last) cbad[x[j].r] = !(hagg_out(pre.h, 1) && pre.h.d1 == 0);
    }
}

// KJ4: every word's checks and output length; c_lo[r] / c_hi[r] = the in-tile prefix in front of cell r's head / behind
// its last word, tile[] = the tile's totals
__global__ void __launch_bounds__(MJ_THREADS) fj_measure_kernel(const MarshalParams p, const FjWords m, JSum* c_lo, JSum* c_hi,
                                                               JSum* tile) {
    JSum carry{0, 0};
    for (int k = 0; k < MJ_ROUNDS; k++) {
        const uint64_t v = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)k * MJ_THREADS + threadIdx.x;
        const bool in = v < m.n;
        FjWord x{0, 0, MjSpan{0, 0, 0}, false, false};
        if (in) x = fj_at(m, v);
        MjItem it;
        uint64_t body;
        const bool ok = mj_load<true>(p, in, x.i, x.s, it, body);
        const JSum mine{it.len, ok ? 0u : 1u};
        JSum total;
        const JSum e = agg_combine(carry, block_exclusive_scan(mine, total));
        carry = agg_combine(carry, total);
        if (x.first) c_lo[x.r] = e;
        if (x.last) c_hi[x.r] = agg_combine(e, mine);
    }
    if (threadIdx.x == 0) tile[blockIdx.x] = carry;
}

struct FjCells {
    FjWords m;
    uint32_t path, sidx;
    const JSum* c_lo;
    const JSum* c_hi;
    const uint8_t* cbad;
    const JSum* len_tile_pre;  // KJ4's tile scan
    const JSum* len_grp_pre;
    uint64_t* jbase;           // the path's rows: the text scan in front of each cell
};

// KJ5: one thread per row of the path
__global__ void __launch_bounds__(256) fj_finish_kernel(const FjCells c, FindParams p) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= c.m.rows) return;
    const uint64_t a = c.m.vstart(r), b = c.m.vstart(r + 1);
    if (a == b) return;  // not found, or no element: KF3's status and 0 bytes stand
    const FjEnds<JSum> s = fj_ends<MJ_TILE>(c.len_tile_pre, c.len_grp_pre, c.c_lo[r], c.c_hi[r], a, b);
    uint64_t len = s.hi.len - s.lo.len;
    const uint64_t q = (uint64_t)c.path * p.roots.n + r;
    if (s.hi.bad != s.lo.bad || c.cbad[r]) {
        p.st[q] = FD_CORRUPT;
        len = 0;
    }
    p.val[q] = len;
    p.slen[(uint64_t)c.sidx * p.roots.n + r] = len;
    c.jbase[r] = s.lo.len;
}

// KJ6: the words' bytes, each OK cell's at its column offset (KF5) + its place in the cell
__global__ void __launch_bounds__(MJ_THREADS) fj_emit_kernel(const MarshalParams p, const FjCells c, const uint8_t* st,
                                                            const int64_t* col, uint8_t* out) {
    uint64_t carry = tile_prefix(c.len_tile_pre, c.len_grp_pre, blockIdx.x).len;
    for (int k = 0; k < MJ_ROUNDS; k++) {
        const uint64_t v = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)k * MJ_THREADS + threadIdx.x;
        const bool in = v < c.m.n;
        FjWord x{0, 0, MjSpan{0, 0, 0}, false, false};
        if (in) x = fj_at(c.m, v);
        MjItem it;
        uint64_t body;
        mj_load<true>(p, in, x.i, x.s, it, body);
        MSum total;
        const uint64_t off = carry + block_exclusive_scan(MSum{it.len}, total).v;
        carry += total.v;
        uint8_t* o = out;
        if (in && st[(uint64_t)c.path * c.m.rows + x.r] == FD_OK) {
            o = out + (uint64_t)col[x.r] + (off - c.jbase[x.r]);
            mj_put_item(it, body, o);
        } else {
            it.long_str = false;  // a CORRUPT cell writes nothing
        }
        mj_put_long(it, o);
    }
}

}  // namespace sj
