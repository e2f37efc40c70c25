// common.cuh -- small PTX wrappers (mbarrier, 1-D TMA bulk copy, relaxed/volatile
// global accesses) shared by the sm_90a kernels.  No CUTLASS/CUB dependency.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace sj {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ----------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {  // release
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)  // suspend-time hint (ns): the thread sleeps in
                                                             // hardware until the phase completes
            : "memory");
    } while (!done);
}

// ---- TMA: 1-D bulk copy global -> shared, completion on an mbarrier ------------
// (SASS: UBLKCP; src/dst 16-byte aligned, bytes a multiple of 16)
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- descriptor words for the decoupled look-back chains ----------------------
__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// named CTA barriers (id 1..15; id 0 is __syncthreads): producers arrive, consumers sync
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ uint32_t lanemask_lt() {
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// the warp of the portable stage-2 code (s2s_slab.h) on the device
struct DevWarp {
    __device__ __forceinline__ uint32_t lane() const { return threadIdx.x & 31; }
    __device__ __forceinline__ uint32_t ballot(bool p) { return __ballot_sync(FULL, p); }
    __device__ __forceinline__ bool any(bool p) { return __any_sync(FULL, p) != 0; }
    __device__ __forceinline__ uint32_t shfl(uint32_t v, uint32_t src) { return __shfl_sync(FULL, v, (int)src); }
    __device__ __forceinline__ uint32_t shfl_up(uint32_t v, int d) { return __shfl_up_sync(FULL, v, d); }
    __device__ __forceinline__ uint32_t reduce_add(uint32_t v) { return __reduce_add_sync(FULL, v); }
    __device__ __forceinline__ void sync() { __syncwarp(); }
    __device__ __forceinline__ void atomic_and(uint32_t* p, uint32_t v) { atomicAnd(p, v); }
    __device__ __forceinline__ void atomic_or(uint32_t* p, uint32_t v) { atomicOr(p, v); }
    // LDGSTS: 16 bytes global -> shared without a register round trip; .ca keeps the line in L1 for the byte look-ups
    __device__ __forceinline__ void async_copy16(void* dst, const void* src) {
        asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
    }
    __device__ __forceinline__ void async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
    __device__ __forceinline__ void async_wait_prev() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
    __device__ __forceinline__ void atomic_or_shared(uint32_t* p, uint32_t v) {
        asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
    }
};

#define SJ_CUDA_CHECK(expr)                                   \
    do {                                                      \
        cudaError_t _e = (expr);                              \
        if (_e != cudaSuccess) return -(1000 + (int)_e);      \
    } while (0)

}  // namespace sj
