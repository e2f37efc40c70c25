// stage2_common.cuh -- the stage-2 pieces both implementations run: the per-structural kernels (stage2.cuh) and the
// streaming kernels (stage2_stream.cuh).
//   Stage2Result          the totals and the verdict of stage 2
//   K2b / K2q scans       exclusive scan of the per-tile (ScanVal) or per-slab (SlabAgg) aggregates in groups of 1024,
//                         then of the group totals; grand totals -> Stage2Result
//   K2d s2_min32 + s2_ansv  scope matching on the brackets: nearest previous bracket of smaller depth
#pragma once
#include <type_traits>

#include "common.cuh"
#include "s2s_core.h"

namespace sj {

constexpr int S2_THREADS = 256;

struct Stage2Result {
    uint64_t tape_len;     // total tape words (including both root words of the last record)
    uint64_t strings_len;  // bytes of the string buffer
    uint64_t n_brackets;
    uint64_t n_records;    // record boundaries (roots - 1)
    int64_t final_depth;
    uint32_t error;        // any stage-2 failure
    uint32_t overflow;     // tape / string capacity exceeded
    uint32_t n_numbers;    // structurals that start a number (K2a)
    uint32_t num_fill;     // fill pointer of the number list (K2g)
    uint32_t internal;     // streaming stage 2: K2r's counts of a slab differ from stage 1's (a defect of the library, not of the input)
};

__device__ __forceinline__ SlabAgg agg_shfl_up(const SlabAgg& a, int d) {
    SlabAgg r;
    r.w = __shfl_up_sync(FULL, a.w, d);
    r.str = __shfl_up_sync(FULL, a.str, d);
    r.brk = __shfl_up_sync(FULL, a.brk, d);
    r.rec = __shfl_up_sync(FULL, a.rec, d);
    r.depth = __shfl_up_sync(FULL, a.depth, d);
    r.last = __shfl_up_sync(FULL, a.last, d);
    r.num = __shfl_up_sync(FULL, a.num, d);
    r.trail = __shfl_up_sync(FULL, a.trail, d);
    return r;
}

// block-wide exclusive scan of ScanVal (K2b) or SlabAgg (K2q), blockDim.x = 1024; returns the exclusive prefix of the
// calling thread and the block total.  agg_combine(a, b) puts a in front of b (SlabAgg's is not commutative in
// `trail`).  Warp totals are scanned by the first warp so every thread reads just two entries of shared memory.
template <class T>
__device__ __forceinline__ T block_exclusive_scan(const T& v, T& total) {
    __shared__ T warp_inc[33];  // [w] = sum of warps < w, [32] = block total
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T t = agg_shfl_up(inc, d);
        if (lane >= d) inc = agg_combine(t, inc);
    }
    if (lane == 31) warp_inc[warp + 1] = inc;  // provisional: the warp's own total
    __syncthreads();
    if (warp == 0) {
        T wv = warp_inc[lane + 1];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const T t = agg_shfl_up(wv, d);
            if (lane >= d) wv = agg_combine(t, wv);
        }
        __syncwarp();
        warp_inc[lane + 1] = wv;  // inclusive over warps <= lane
        if (lane == 0) warp_inc[0] = T{};
    }
    __syncthreads();
    total = warp_inc[32];
    T ex = agg_shfl_up(inc, 1);
    if (lane == 0) ex = T{};
    const T r = agg_combine(warp_inc[warp], ex);
    __syncthreads();  // the shared array is reused by the next call
    return r;
}

// ---------------------------------------------------------------------------------
// K2b (ScanVal per tile) / K2q (SlabAgg per slab): exclusive scan of `in[0..n)` in groups of 1024 (one block per group)
// ---------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(1024) scan_groups_kernel(const T* in, uint32_t n, T* pre, T* group_total) {
    const uint32_t i = blockIdx.x * 1024 + threadIdx.x;
    const T v = i < n ? in[i] : T{};
    T total;
    const T e = block_exclusive_scan(v, total);
    if (i < n) pre[i] = e;
    if (threadIdx.x == 0) group_total[blockIdx.x] = total;
}

// single block: exclusive scan of all group totals (looping), grand totals into `res` and, when given, into
// `totals_out` (sj_shard_totals in device memory, for an exchange that stays on the stream)
template <class T>
__global__ void __launch_bounds__(1024) scan_top_kernel(const T* in, uint32_t n, T* pre, Stage2Result* res, uint64_t* totals_out,
                                                        uint64_t msg_bytes) {
    T carry{};
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const T v = i < n ? in[i] : T{};
        T total;
        const T e = block_exclusive_scan(v, total);
        if (i < n) pre[i] = agg_combine(carry, e);
        carry = agg_combine(carry, total);
    }
    if (threadIdx.x == 0) {
        res->tape_len = (uint64_t)carry.w + 2;  // + root open + root close
        res->strings_len = carry.str;
        res->n_brackets = carry.brk;
        res->n_records = carry.rec;
        res->final_depth = carry.depth;
        if constexpr (std::is_same<T, SlabAgg>::value) res->n_numbers = carry.num;  // (K2a adds up its own count)
        if (totals_out) {
            totals_out[0] = msg_bytes;
            totals_out[1] = (uint64_t)carry.w + 2;
            totals_out[2] = carry.str;
            totals_out[3] = (uint64_t)carry.rec + 1;
        }
    }
}

// ---------------------------------------------------------------------------------
// K2d: min hierarchy + nearest-smaller-to-the-left
// ---------------------------------------------------------------------------------
constexpr int ANSV_MAX_LEVELS = 8;
struct AnsvLevels {
    const int32_t* lv[ANSV_MAX_LEVELS];
    uint32_t n[ANSV_MAX_LEVELS];
    int nlevels;
};

__global__ void s2_min32_kernel(const int32_t* in, uint32_t n_in, int32_t* out, uint32_t n_out) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n_out) return;
    const uint32_t j = w * 32 + lane;
    int32_t v = j < n_in ? in[j] : 0x7fffffff;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = min(v, __shfl_xor_sync(FULL, v, d));
    if (lane == 0) out[w] = v;
}

__global__ void __launch_bounds__(S2_THREADS) s2_ansv_kernel(AnsvLevels L, int32_t* par) {
    const uint32_t k = blockIdx.x * S2_THREADS + threadIdx.x;
    if (k >= L.n[0]) return;
    const int32_t* D = L.lv[0];
    const int32_t t = D[k];
    if (t <= 0) {
        // nothing in front of a bracket at depth 0 can be shallower unless an earlier close went below the top level --
        // which the grammar check rejects anyway (a close at the top level is in no legal transition), so the
        // answer "none" is exact for every accepted document and harmless for the others.  (Every NDJSON record
        // opens at depth 0: without this each of them walks the whole min hierarchy to find nothing.)
        par[k] = -1;
        return;
    }
    int64_t found = -1;
    {
        int64_t lo = k & ~31u;
        for (int64_t m = (int64_t)k - 1; m >= lo; m--)
            if (D[m] < t) {
                found = m;
                break;
            }
    }
    if (found < 0) {
        int lvl = 1;
        int64_t idx = (int64_t)(k >> 5) - 1;
        while (lvl < L.nlevels && idx >= 0) {
            const int32_t* A = L.lv[lvl];
            const int64_t lo = idx & ~31ll;
            int64_t hit = -1;
            for (int64_t j = idx; j >= lo; j--)
                if (A[j] < t) {
                    hit = j;
                    break;
                }
            if (hit >= 0) {
                int64_t cur = hit;
                for (int l = lvl; l >= 1; l--) {  // descend: last child below the bound
                    const int32_t* B = L.lv[l - 1];
                    int64_t base = cur * 32, hi = base + 31;
                    if (hi >= (int64_t)L.n[l - 1]) hi = (int64_t)L.n[l - 1] - 1;
                    int64_t c = hi;
                    while (c > base && !(B[c] < t)) c--;
                    cur = c;
                }
                found = cur;
                break;
            }
            idx = (lo >> 5) - 1;
            lvl++;
        }
    }
    par[k] = (int32_t)found;
}

}  // namespace sj
