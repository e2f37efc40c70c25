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
    alignas(16) uint8_t back[128];  // mirror only: where the tape consumers' read-backs land (fetch, sj_tape.inl)
};
static_assert(offsetof(ResultBlock, s1) == 0, "result block layout");
static_assert(offsetof(ResultBlock, s2) == 64, "result block layout");
static_assert(offsetof(ResultBlock, back) == 192, "result block layout");

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
    // tape consumers (tape.cuh and its users), each alive within one call only: the call's arguments (countWhere's
    // needles, the find's paths), the scratch of its passes, the Serializer's string dedup, the root list of a foreign
    // tape and the scan that finds it, the output of an sj_parse_* call before its copy to the host, and the per-word
    // passes of the find's JSON paths (find_json.cuh), and the records and element rows of the find's array rows
    // (find_rows.cuh)
    DevBuf args, scratch, sz_tab, tc_roots, tc_scan, staging, fj, fr_rec, fr_row;
    uint64_t find_rows_serial = 0;  // the last array-rows call: records whose rows one thread walked (test hook)
    uint32_t sz_hash_bits = 0;  // test hook: keep only this many bits of the dedup hash (0 = all)
    // the Serializer's compress mode (SJ_COMPRESS_*) and, within one call, the S2 and zstd codecs' buffers (s2.cuh,
    // zstd.cuh): the uncompressed stream and the encoders' chunk slots; the chunk, frame and block lists and the
    // inflated blocks; the zstd encoder's sequences, and the decoder's literals, sequences and per-byte sources
    int compress_mode = 0;
    DevBuf s2_raw, s2_slots, s2_list, s2_out, zx_seq, zx_src;
    // what the last successful stage 2 of this context left in device memory.  The next parse clears last_tape, and so
    // does an sj_deserialize_device that writes over any part of that tape: tape_rows takes last_rootpos as the rows of
    // a tape at last_tape of last_tape_len words only while it is set.  A caller's own writes to that buffer are not
    // seen: the consumers take it as the tape the parse left there.
    const uint32_t* last_rootpos = nullptr;  // stage 2's root list (slot of every record's root-open word, [0] implicit)
    uint64_t last_records = 0;               // record boundaries = roots - 1
    const uint64_t* last_tape = nullptr;
    uint64_t last_tape_len = 0;
    const uint8_t* last_strings = nullptr;
    const uint8_t* last_msg = nullptr;
    void* xchg = nullptr;  // SjExchange (sj_exchange.inl): the sharded ParseND's exchange over peer memory, if set up
    DevBuf test_in, test_out, test_aux;
};
