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
//   K2d s2_min32 + s2_ansv (stage2_common.cuh)    scope matching on the brackets
//   K2e s2s_link       per bracket: cross-links of { } [ ] (stage2...go:327-334) and the grammar verdict of the segment
//                      in front of it against the container it lies in; the same launch writes the root words (K2f)
//
// The unifiedMachine of the reference (stage2_build_tape_amd64.go:160-446) walks one structural at a time; the
// per-structural kernels of stage2.cuh gave every structural a thread and spent ~460 warp-instructions per 32
// structurals on divergent per-type work.  Here the warp walks the MESSAGE like stage 1 does (lane = 64-byte block),
// and what is left per structural is a short loop.
#pragma once
#include "common.cuh"
#include "number.cuh"
#include "s2s_slab.h"
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
// K2e: per bracket k (and k = nb for the segment behind the last bracket): is every structural of segment k -- the
// ones behind bracket k-1 up to and including bracket k -- allowed inside the container that is open there?  That
// container is the scope open right after bracket k-1: the bracket itself if it opens, else the parent of the scope
// it closes (par = nearest previous bracket with a smaller depth in front of it, K2d).  Closing brackets cross-link
// the tape words of their pair (stage2...go:327-334), except those K2r has linked already (BRK_LINKED: both ends in
// one staged step).
// ---------------------------------------------------------------------------------
// The same launch writes the root words (K2f, stage2...go:170,207-218,428-441): record r opens at rootpos[r], its close
// sits right in front of the next record's open (or is the last word of the tape).  Records whose bit in rootlink K2r
// has cleared are written already.
__global__ void __launch_bounds__(S2_THREADS) s2s_link_kernel(const S2sParams p, const int32_t* par, uint32_t nb, uint64_t n_records,
                                                              uint64_t tape_len) {
    const uint32_t k = blockIdx.x * S2_THREADS + threadIdx.x;
    const uint64_t tape_base = s2s_tape_base(p);
    if (k <= n_records && ((p.rootlink[k >> 5] >> (k & 31)) & 1u)) {
        const uint64_t R = (uint64_t)'r' << 56;
        const uint64_t open = k == 0 ? 0 : p.rootpos[k];
        const uint64_t next_open = k == n_records ? tape_len : p.rootpos[k + 1];
        if (next_open <= tape_len && next_open != 0) {
            p.tape[open] = R | (tape_base + next_open);
            p.tape[next_open - 1] = R | (tape_base + open);
        }
    }
    if (k > nb) return;
    uint32_t ctx = CTX_ROOT;
    if (k > 0) {
        const uint32_t kd = p.brk_kind[k - 1] & ~BRK_LINKED;
        int32_t enc;
        if (kd == T_OBJ_OPEN || kd == T_ARR_OPEN) {
            enc = (int32_t)k - 1;
        } else {
            const int32_t m = par[k - 1];
            enc = m >= 0 ? par[m] : -1;
        }
        ctx = enc >= 0 ? ((p.brk_kind[enc] & ~BRK_LINKED) == T_OBJ_OPEN ? CTX_OBJ : CTX_ARR) : CTX_ROOT;
    }
    const uint32_t sg = (p.segmask[k >> 2] >> (8 * (k & 3))) & 0xffu;
    if (!((sg >> ctx) & 1u)) atomicOr(p.error, 1u);
    if (k < nb) {
        const uint32_t kd = p.brk_kind[k];  // (a linked close carries BRK_LINKED and matches neither kind)
        if (kd == T_OBJ_CLOSE || kd == T_ARR_CLOSE) {
            const int32_t m = par[k];
            if (m >= 0) {
                const uint32_t otp = p.brk_tp[m], ctp = p.brk_tp[k];
                p.tape[otp] = ((uint64_t)(kd == T_OBJ_CLOSE ? '{' : '[') << 56) | (tape_base + ctp + 1);
                p.tape[ctp] = ((uint64_t)(kd == T_OBJ_CLOSE ? '}' : ']') << 56) | (tape_base + otp);
            }
        }
    }
}

}  // namespace sj
