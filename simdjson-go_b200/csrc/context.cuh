// context.cuh -- per-context CUDA stream, events, result block and grow-only device scratch.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#include "common.cuh"
#include "stage1.cuh"
#include "stage2_common.cuh"

// The context's result block: one device allocation (sj_ctx::result) and its pinned mirror (sj_ctx::host_result).  The
// kernels write s1 and s2; read_back copies a byte range of it to the mirror.
struct ResultBlock {
    sj::Stage1Result s1;
    uint8_t gap1[64 - sizeof(sj::Stage1Result)];
    sj::Stage2Result s2;
    uint8_t gap2[128 - sizeof(sj::Stage2Result)];
    uint64_t counters[2];  // mirror only: where the tape consumers (sj_consume.inl) land their two device counters
};
static_assert(offsetof(ResultBlock, s1) == 0, "result block layout");
static_assert(offsetof(ResultBlock, s2) == 64, "result block layout");
static_assert(offsetof(ResultBlock, counters) == 192, "result block layout");

struct S2Pending;  // sj_parse.inl

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    // grow-only; contents are not preserved
    int reserve(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + (bytes >> 3) + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            e = cudaMalloc(&p, bytes);  // retry without slack
            want = bytes;
        }
        if (e != cudaSuccess) return -(1000 + (int)e);
        cap = want;
        return 0;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

struct sj_ctx {
    int device = 0;
    int sm_count = 0;
    int s1_max_ctas = 0;  // co-resident CTAs of the stage-1 kernel (cooperative launch bound)
    cudaStream_t stream = nullptr;      // the stream the work runs on
    cudaStream_t own_stream = nullptr;  // the context's own one (sj_ctx_set_stream may point `stream` elsewhere)
    cudaEvent_t ev[2] = {nullptr, nullptr};
    uint64_t launches = 0;
    // stage 1
    DevBuf msg;      // device copy of the (trimmed) message, padded
    DevBuf idx;      // structural positions (uint32)
    DevBuf desc;     // K1 look-back descriptors (one 128-byte slot per tile and chain) + per-tile slab in-string bits
    const uint32_t* last_slabpar = nullptr;  // the in-string bits of the last stage-1 launch (inside desc), or null
    DevBuf result;                        // ResultBlock
    ResultBlock* host_result = nullptr;   // its pinned mirror
    // stage 2
    S2Pending* pending = nullptr;  // state between the counting and the emitting half of stage 2
    int s2_impl = 0;  // stage 2: 0 = streaming kernels (stage2_stream.cuh) when copy_strings is on, 1 = per-structural kernels (stage2.cuh) always
    DevBuf s2a, s2b, s2c;  // s2a/s2b: stage-2 scratch (before / after the totals are known), s2c: backslash block map
    DevBuf tape, strings;  // device outputs for the host-buffer API
    // tape consumers (consume.cuh): needles + counters, root list of a foreign tape
    DevBuf tc_small, tc_roots;
    // device MarshalJSON (marshal.cuh): scratch of the passes, the text of sj_parse_marshal before its copy to the host
    DevBuf mj, mj_out;
    // what the last successful stage 2 of this context left in device memory (valid until the next call)
    const uint32_t* last_rootpos = nullptr;  // stage 2's root list (slot of every record's root-open word, [0] implicit)
    uint64_t last_records = 0;               // record boundaries = roots - 1
    const uint64_t* last_tape = nullptr;
    uint64_t last_tape_len = 0;
    const uint8_t* last_strings = nullptr;
    const uint8_t* last_msg = nullptr;
    void* xchg = nullptr;  // SjExchange (sj_exchange.inl): the sharded ParseND's exchange over peer memory, if set up
    DevBuf test_in, test_out, test_aux;
};
