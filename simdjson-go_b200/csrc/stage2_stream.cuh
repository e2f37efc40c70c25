// stage2_stream.cuh -- the streaming stage 2 on the device: kernels around the portable core (s2s_core.h, s2s_slab.h).
//
//   K1  stage1_flatten_kernel<., ., true> (stage1.cuh), the parse mode of stage 1: besides the in-string state of every
//                      slab, per-slab aggregate (tape words, string bytes, brackets, depth, records, the bytes under the
//                      last stage-1 structurals, numbers, bytes behind the last quote)
//   K2q scan_*_kernel<SlabAgg> (stage2_common.cuh)   exclusive scan of the aggregates (groups of 1024 + their
//                      totals), grand totals -> Stage2Result
//   K2r s2s_emit       the same analysis again, now with every offset known: tape words and Strings.B bytes (both
//                      staged in shared memory and streamed out with coalesced / 16-byte stores), the cross-links and
//                      root words of the pairs inside one step, bracket records for the scope matching, number list,
//                      per-segment grammar masks
//   K2h s2s_numbers    parse_number (parse_number.go:65) over the number list, one number per thread
//   K2t s2t_min + s2t_link (s2s_tile.h)   scope matching on the brackets, tile by tile; per bracket the cross-links of
//                      { } [ ] (stage2...go:327-334) and the grammar verdict of the segment in front of it against the
//                      container it lies in; the same launch writes the root words (K2f)
//
// The unifiedMachine of the reference (stage2_build_tape_amd64.go:160-446) walks one structural at a time; the
// per-structural kernels of stage2.cuh gave every structural a thread and spent ~460 warp-instructions per 32
// structurals on divergent per-type work.  Here the warp walks the MESSAGE like stage 1 does (lane = 64-byte block),
// and what is left per structural is a short loop.
#pragma once
#include "common.cuh"
#include "number.h"
#include "s2s_slab.h"
#include "s2s_tile.h"
#include "stage1.cuh"
#include "stage2_common.cuh"

namespace sj {

static_assert(S2S_SLAB_BYTES == (uint32_t)S1_SLAB_BYTES, "stage 2 takes the in-string state per stage-1 slab");
static_assert(S1_WARPS <= 32, "one bit per slab of a tile");

constexpr int S2S_WARPS = 8;  // slabs per CTA
constexpr int S2S_THREADS = S2S_WARPS * 32;
constexpr uint32_t S2S_SSTAGE_PAD = (S2S_SSTAGE_BYTES + 15u) & ~15u;
static_assert(S2S_TSTAGE_WORDS * 8 >= S2S_ESC_SCRATCH, "K2r decodes escapes in the tape-staging area");
constexpr uint32_t S2S_WARP_SMEM_EMIT = S2S_IMAGE_BYTES + S2S_SSTAGE_PAD + S2S_TSTAGE_WORDS * 8;
constexpr size_t S2S_SMEM_EMIT = (size_t)S2S_WARPS * S2S_WARP_SMEM_EMIT;
// resident blocks per SM the register allocation must allow; also the persistent grids' blocks per SM
constexpr int S2S_EMIT_MIN_BLOCKS = 2;

// character / transition / compaction tables of a CTA (shared memory)
struct S2sTables {
    uint8_t ctab[256];
    uint8_t oktab[256];
    uint32_t cmptab[16];
};
__device__ __forceinline__ void s2s_fill_tables(S2sTables& t) {
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        t.ctab[i] = (uint8_t)char_type(i);
        const uint32_t p = i >> 4, c = i & 15;
        t.oktab[i] = (p < 15 && c < 15) ? (uint8_t)transition_mask(p, c) : (uint8_t)0;
    }
    if (threadIdx.x < 16) t.cmptab[threadIdx.x] = compress_sel(threadIdx.x) | ((uint32_t)__popc(threadIdx.x) << 16);
}

__global__ void __launch_bounds__(S2S_THREADS, S2S_EMIT_MIN_BLOCKS) s2s_emit_kernel(const S2sParams p) {
    extern __shared__ __align__(128) uint8_t s2s_smem[];
    __shared__ S2sTables tabs;
    s2s_fill_tables(tabs);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5;
    S2sWarpMem sm;
    uint8_t* base = s2s_smem + (size_t)warp * S2S_WARP_SMEM_EMIT;
    sm.src = base;
    sm.sstage = base + S2S_IMAGE_BYTES;
    sm.tstage = reinterpret_cast<uint64_t*>(base + S2S_IMAGE_BYTES + S2S_SSTAGE_PAD);
    sm.esc = reinterpret_cast<uint8_t*>(sm.tstage);
    sm.ctab = tabs.ctab;
    sm.oktab = tabs.oktab;
    sm.cmptab = tabs.cmptab;
    DevWarp wp;
    s2s_warp_loop<DevWarp, true>(wp, p, blockIdx.x * S2S_WARPS + warp, gridDim.x * S2S_WARPS, sm);
}

// ---------------------------------------------------------------------------------
// K2h: parse_number over the number list
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(S2_THREADS) s2s_numbers_kernel(const uint8_t* msg, uint64_t len, const NumEntry* list, uint32_t count,
                                                                 uint64_t* tape, uint32_t* error) {
    const uint32_t k = blockIdx.x * S2_THREADS + threadIdx.x;
    if (k >= count) return;
    const NumEntry e = list[k];
    uint64_t val = 0;
    uint64_t tag = parse_number_fast(msg + e.pos, len - e.pos, &val);
    if (tag == PN_SLOW) tag = parse_number(msg + e.pos, len - e.pos, &val);  // parse_number.go:65
    if (tag == 0) atomicOr(error, 1u);
    tape[e.slot] = tag;
    tape[(uint64_t)e.slot + 1] = val;
}

// ---------------------------------------------------------------------------------
// K2t (s2s_tile.h): K2t-min builds the min hierarchy over the brackets' depths, one CTA per tile; K2t-link then gives
// every bracket of its tile its par, checks the tile's segments, writes the cross-links and, with the same grid, the
// root words of records lo .. lo + S2T_TILE - 1
// ---------------------------------------------------------------------------------
constexpr int S2T_THREADS = 1024;

__device__ __forceinline__ int32_t warp_min(int32_t v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = min(v, __shfl_xor_sync(FULL, v, d));
    return v;
}

__global__ void __launch_bounds__(S2T_THREADS) s2t_min_kernel(const int32_t* depth, uint32_t nb, const __grid_constant__ S2tLevels L) {
    __shared__ int32_t m1[S2T_TILE / 32], m2[S2T_TILE / 1024];
    const uint32_t lo = blockIdx.x * S2T_TILE, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t i = threadIdx.x; i < S2T_TILE; i += S2T_THREADS) {
        const int32_t v = warp_min(lo + i < nb ? depth[lo + i] : INT32_MAX);
        if (lane == 0) m1[i >> 5] = v;
    }
    __syncthreads();
    if (warp < S2T_TILE / 1024) {
        const uint32_t i = warp * 32 + lane;
        const int32_t v = m1[i];
        if (L.nlevels > 1 && (lo >> 5) + i < L.n[1]) L.lv[1][(lo >> 5) + i] = s2t_key(v);
        const int32_t w = warp_min(v);
        if (lane == 0) {
            if (L.nlevels > 2 && (lo >> 10) + warp < L.n[2]) L.lv[2][(lo >> 10) + warp] = s2t_key(w);
            m2[warp] = w;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && L.nlevels > 3) {
        int32_t v = m2[0];
        for (uint32_t q = 1; q < S2T_TILE / 1024; q++) v = min(v, m2[q]);
        for (int l = 3; l < L.nlevels; l++) atomicMin(L.lv[l] + (lo >> (5 * l)), s2t_key(v));
    }
}

__global__ void __launch_bounds__(S2T_THREADS) s2t_link_kernel(const S2sParams p, const __grid_constant__ S2tLevels L, uint32_t nb,
                                                               uint64_t n_records, uint64_t tape_len) {
    __shared__ int32_t d_s[S2T_TILE], par_s[S2T_TILE];
    __shared__ uint8_t k_s[S2T_TILE];
    const uint32_t lo = blockIdx.x * S2T_TILE;
    for (uint32_t i = threadIdx.x; i < S2T_TILE && lo + i < nb; i += S2T_THREADS) {
        d_s[i] = p.brk_depth[lo + i];
        k_s[i] = p.brk_kind[lo + i];
    }
    __syncthreads();
    const S2tTile v{p.brk_depth, p.brk_kind, d_s, k_s, par_s, lo, &L};
    for (uint32_t i = threadIdx.x; i < S2T_TILE && lo + i < nb; i += S2T_THREADS) par_s[i] = s2t_par(v, lo + i);
    __syncthreads();
    const uint64_t tape_base = s2s_tape_base(p);
    for (uint32_t i = threadIdx.x; i < S2T_TILE && lo + i <= nb; i += S2T_THREADS)
        if (!s2t_segment(p, v, nb, lo + i, tape_base)) atomicOr(p.error, 1u);
    for (uint32_t i = threadIdx.x; i < S2T_TILE && lo + i <= n_records; i += S2T_THREADS) s2t_root(p, lo + i, n_records, tape_len, tape_base);
}

}  // namespace sj
