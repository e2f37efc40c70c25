// tape.cuh -- the device side of a tape in HBM that the tape consumers (consume.cuh, find.cuh, marshal.cuh,
// serialize.cuh) share: the tape format, the head scan and the root finder.
//
// The word-parallel passes run over tiles of TAPE_TILE words, TAPE_ROUNDS consecutive words per thread.  Their per-tile
// sums are scanned by scan_groups_kernel<T> (stage2_common.cuh), once per group of 1024 tiles and once over the group
// totals; tile_prefix() reads a tile's exclusive prefix back from the two levels.
//   KM1 mj_heads_reduce  which words are heads (not the value word of a string or number) and the depth in front of
//        every head: the transfer function (HAgg) of each tile; tape_heads() scans it inside a tile
//   KC1a tc_root_count   on any tape, the root opens ('r' words that point forward and are heads) per tile.  On every
//        tape the parser or Deserialize writes these are the roots ForEach visits.
//   KC1b tc_root_write   their slots, in tape order: the rows of countWhere (consume.cuh) and of the find (find.cuh)
#pragma once
#include "common.cuh"
#include "stage2_common.cuh"

namespace sj {

constexpr uint64_t TAPE_VALUE_MASK = 0x00ffffffffffffffull;  // JSONVALUEMASK, parsed_json.go:26
constexpr uint64_t TAPE_STRINGBUFMASK = STRINGBUFBIT - 1;     // parsed_json.go:30

constexpr int TAPE_THREADS = 1024;
constexpr int TAPE_ROUNDS = 4;  // a tile is TAPE_ROUNDS rounds of one word per thread
constexpr uint64_t TAPE_TILE = TAPE_THREADS * TAPE_ROUNDS;

// a tag whose value word follows it: string, int64, uint64, double
__device__ __forceinline__ bool tape_value_tag(uint32_t t) { return t == '"' || t == 'l' || t == 'u' || t == 'd'; }

// a tape and the two buffers its strings point into
struct TapeView {
    const uint64_t* tape;
    uint64_t n;
    const uint8_t* msg;  // no-copy strings point into it
    uint64_t msg_len;
    const uint8_t* strings;  // Strings.B
    uint64_t strings_len;
};

// stringByteAt (parsed_json.go:107-120): the `len` bytes of the string whose tape word is `word`; false when they do
// not lie inside their buffer (an offset + length that wraps makes the reference's slice panic)
__device__ __forceinline__ bool tape_string(const TapeView& t, uint64_t word, uint64_t len, const uint8_t** s) {
    const uint64_t v = word & TAPE_VALUE_MASK;
    if (!(v & STRINGBUFBIT)) {
        if (v + len < v || v + len > t.msg_len) return false;
        *s = t.msg + v;
        return true;
    }
    const uint64_t off = v & TAPE_STRINGBUFMASK;
    if (off + len < off || off + len > t.strings_len) return false;
    *s = t.strings + off;
    return true;
}
// the same without the check, for a string whose range has been checked (or, in countWhere, cannot be)
__device__ __forceinline__ const uint8_t* tape_string_ptr(const TapeView& t, uint64_t word) {
    const uint64_t v = word & TAPE_VALUE_MASK;
    return (v & STRINGBUFBIT) ? t.strings + (v & TAPE_STRINGBUFMASK) : t.msg + v;
}

// the exclusive prefix of tile `tile` from the two levels of a tile scan
template <class T>
__device__ __forceinline__ T tile_prefix(const T* tile_pre, const T* grp_pre, uint64_t tile) {
    return agg_combine(grp_pre[tile >> 10], tile_pre[tile]);
}

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

// a 64-bit count
struct MSum {
    uint64_t v;
};
__device__ __forceinline__ MSum agg_combine(const MSum& a, const MSum& b) { return MSum{a.v + b.v}; }
__device__ __forceinline__ MSum agg_shfl_up(const MSum& a, int d) { return MSum{__shfl_up_sync(FULL, a.v, d)}; }

__device__ __forceinline__ HAgg mj_word_agg(uint64_t w, uint64_t i) {
    const uint32_t t = (uint32_t)(w >> 56);
    HAgg a;
    a.cst = tape_value_tag(t) ? 0 : 1;
    a.val = 1;
    a.d0 = 0;
    a.d1 = (t == '{' || t == '[') ? 1 : (t == '}' || t == ']') ? -1 : t == 'r' ? ((w & TAPE_VALUE_MASK) > i ? 1 : -1) : 0;
    return a;
}

// KM1: the transfer function of each tile
__global__ void __launch_bounds__(TAPE_THREADS) mj_heads_reduce_kernel(const uint64_t* tape, uint64_t n, HAgg* tile_sum) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    HAgg a{};
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++)
        if (base + j < n) a = agg_combine(a, mj_word_agg(tape[base + j], base + j));
    HAgg total;
    block_exclusive_scan(a, total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// the TAPE_ROUNDS words of this thread of tile blockIdx.x, from `base` on (0 past n), and the head state in front of the
// first of them, from KM1's scan; the whole block calls it
__device__ __forceinline__ HAgg tape_heads(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre, const HAgg* h_grp_pre,
                                           uint64_t base, uint64_t (&w)[TAPE_ROUNDS]) {
    HAgg a{};
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        w[j] = base + j < n ? tape[base + j] : 0;
        if (base + j < n) a = agg_combine(a, mj_word_agg(w[j], base + j));
    }
    HAgg total;
    const HAgg ex = block_exclusive_scan(a, total);
    return agg_combine(tile_prefix(h_tile_pre, h_grp_pre, blockIdx.x), ex);
}

// which of this thread's words are root opens: 'r' words pointing forward that are heads.  A number whose value word
// happens to start with the byte 'r' (int64s from 0x72 << 56, doubles near 1e241-1e246) is no root.
__device__ __forceinline__ uint32_t tc_root_opens(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre, const HAgg* h_grp_pre,
                                                  uint64_t base) {
    uint64_t w[TAPE_ROUNDS];
    HAgg pre = tape_heads(tape, n, h_tile_pre, h_grp_pre, base, w);
    uint32_t open = 0;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (base + j < n && hagg_out(pre, 1) && (w[j] >> 56) == 'r' && (w[j] & TAPE_VALUE_MASK) > base + j) open |= 1u << j;
        pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
    return open;
}

// KC1a: root opens per tile, after KM1 and its scans
__global__ void __launch_bounds__(TAPE_THREADS) tc_root_count_kernel(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre,
                                                                   const HAgg* h_grp_pre, MSum* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    const uint32_t open = tc_root_opens(tape, n, h_tile_pre, h_grp_pre, base);
    MSum total;
    block_exclusive_scan(MSum{(uint64_t)__popc(open)}, total);
    if (threadIdx.x == 0) tile[blockIdx.x] = total;
}

// KC1b: the slots, in tape order
__global__ void __launch_bounds__(TAPE_THREADS) tc_root_write_kernel(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre,
                                                                   const HAgg* h_grp_pre, const MSum* tile_pre,
                                                                   const MSum* grp_pre, uint32_t* roots) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    const uint32_t open = tc_root_opens(tape, n, h_tile_pre, h_grp_pre, base);
    MSum total;
    uint64_t at = tile_prefix(tile_pre, grp_pre, blockIdx.x).v + block_exclusive_scan(MSum{(uint64_t)__popc(open)}, total).v;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++)
        if (open >> j & 1) roots[at++] = (uint32_t)(base + j);
}

// the rows of a tape: the slot of every root-open word, in tape order
struct TapeRows {
    const uint32_t* slot;
    uint32_t skip0;  // 1: slot[0] is not stored and means slot 0 (stage 2's rootpos array)
    uint64_t n;
};
__device__ __forceinline__ uint64_t tape_root(const TapeRows& r, uint64_t k) { return (r.skip0 && k == 0) ? 0 : r.slot[k]; }

}  // namespace sj
