// sj_api.cu -- C-ABI entry points (include/simdjson_b200.h), host orchestration.
//
// Host logic here mirrors the reference's parse driver (parse_json_amd64.go:28-127) and
// stage-1 driver epilogue (stage1_find_marks_amd64.go:115-148); all byte work runs in the
// sm_90a kernels of stage1.cuh and of the two stage-2 implementations (stage2_stream.cuh,
// stage2.cuh; what both run is in stage2_common.cuh).  There is NO CPU fallback: without a
// CUDA device every entry point returns SJ_ERR_NO_DEVICE.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <set>
#include <string>
#include <vector>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "../../include/simdjson_b200.h"
#include "context.cuh"
#include "stage1.cuh"
#include "stage2_stream.cuh"
#include "stage2.cuh"
#include "tape.cuh"
#include "consume.cuh"
#include "find.cuh"
#include "find_json.cuh"
#include "find_list.cuh"
#include "find_rows.cuh"
#include "marshal.cuh"
#include "serialize.cuh"
#include "zstd.cuh"
#include "gen.cuh"
#include "exchange.cuh"

using namespace sj;

// ---------------------------------------------------------------------------------
// test kernels (unit-test hooks)
// ---------------------------------------------------------------------------------
__global__ void test_block_masks_kernel(const uint8_t* blocks, size_t nblocks, const uint64_t* carry_in, uint64_t* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblocks) return;
    uint32_t w[16];
    const uint32_t* src = reinterpret_cast<const uint32_t*>(blocks + 64 * i);
#pragma unroll
    for (int k = 0; k < 16; k++) w[k] = src[k];
    PlaneMasks m = classify_block_planes(w);
    uint32_t prev_odd = (uint32_t)carry_in[4 * i + 0];
    uint64_t prev_inside = carry_in[4 * i + 1];
    uint32_t prev_pseudo = (uint32_t)carry_in[4 * i + 2];
    bool ndjson = carry_in[4 * i + 3] != 0;
    uint32_t odd_carry;
    uint64_t odd_ends = odd_backslash_ends(m.bs, prev_odd, &odd_carry);
    uint64_t qb = m.qt & ~odd_ends;
    uint64_t qm = prefix_xor64(qb) ^ prev_inside;
    uint64_t err = m.ct & qm;
    uint64_t ws = m.ws;
    uint32_t pp_out;
    uint64_t fin = finalize_structurals(m.st, ws, qm, qb, prev_pseudo, &pp_out);
    uint64_t nl = m.nl;  // raw newline mask; the fused result applies & ~quote_mask
    if (ndjson) fin |= nl & ~qm;
    // cross-check: the word-wise SWAR classifier must agree with the bit-sliced one
    {
        BlockMasks f = classify_block(w);
        SlowMasks sl = classify_block_slow(w);
        if (f.bs != m.bs || f.qt != m.qt || f.st != m.st || (f.sp | sl.wsc) != m.ws || sl.ct != m.ct || sl.nl != m.nl ||
            ((f.anyct != 0) != (m.ct != 0)))
            err = ~0ull;
    }
    uint64_t* o = out + 12 * i;
    o[0] = odd_ends;
    o[1] = qm;
    o[2] = qb;
    o[3] = err;
    o[4] = ws;
    o[5] = m.st;
    o[6] = fin;
    o[7] = nl;
    o[8] = odd_carry;
    o[9] = (uint64_t)((int64_t)qm >> 63);
    o[10] = pp_out;
    o[11] = m.ct != 0;
}

__global__ void test_finalize_kernel(const uint64_t* in, size_t n, uint64_t* out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t pp;
    out[2 * i] = finalize_structurals(in[5 * i], in[5 * i + 1], in[5 * i + 2], in[5 * i + 3], (uint32_t)in[5 * i + 4], &pp);
    out[2 * i + 1] = pp;
}

// one warp walks the mask sequence 32 masks (= one 2 KiB step) at a time through flatten_step,
// the stage-1 kernel's per-step path (the kernel's staged path is covered by sj_find_structural_indices)
__global__ void test_flatten_kernel(const uint64_t* masks, size_t nmasks, uint32_t* out, size_t cap, uint64_t* n_out) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t prev_last = 0xffffffffu, overflow = 0;
    uint64_t off = 0;
    for (size_t base = 0; base < nmasks; base += 32) {
        uint64_t S = base + lane < nmasks ? masks[base + lane] : 0;
        off += flatten_step<true>(S, (uint32_t)((base + lane) * 64), out, off, cap, prev_last, overflow);
    }
    if (lane == 0) {
        n_out[0] = off;
        n_out[1] = overflow;
    }
}

// ---------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------
extern "C" int sj_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" int sj_supported(void) {
    int n = sj_device_count();
    for (int d = 0; d < n; d++) {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, d) == cudaSuccess && prop.major == 9 && prop.minor == 0) return 1;
    }
    return 0;
}

extern "C" const char* sj_error_string(int rc) {
    switch (rc) {
    case SJ_OK: return "ok";
    case SJ_ERR_STAGE1: return "Failed to find all structural indices for stage 1";
    case SJ_ERR_STAGE2: return "Bad parsing while executing stage 2";
    case SJ_ERR_NO_DEVICE: return "Host does not have a usable sm_90 CUDA device";
    case SJ_ERR_CAPACITY: return "output buffer too small";
    case SJ_ERR_TOO_LARGE: return "message too large for one call";
    case SJ_ERR_ARGUMENT: return "bad argument";
    case SJ_STREAM_END: return "end of stream";
    case SJ_STREAM_EMPTY: return "no chunk in flight";
    case SJ_STREAM_BUSY: return "every stream slot is in use";
    case SJ_ERR_EXCHANGE: return "sharded ParseND: a peer's totals did not arrive in time";
    case SJ_ERR_PEER: return "sharded ParseND: a peer's shard failed";
    case SJ_ERR_UNSUPPORTED: return "serialized stream has S2 blocks in CompressNone mode, or zstd blocks in CompressNone / CompressFast mode";
    default: return rc < 0 ? cudaGetErrorString((cudaError_t)(-rc - 1000)) : "unknown error";
    }
}

extern "C" void sj_ctx_destroy(sj_ctx* c);
static void exchange_release(sj_ctx* c);  // sj_exchange.inl
static S2Pending* s2_pending_alloc();     // sj_parse.inl

extern "C" int sj_ctx_create(int device, sj_ctx** out) {
    if (!out) return SJ_ERR_ARGUMENT;
    *out = nullptr;
    int n = sj_device_count();
    if (n == 0) return SJ_ERR_NO_DEVICE;
    if (device < 0) {
        if (cudaGetDevice(&device) != cudaSuccess) return SJ_ERR_NO_DEVICE;
    }
    if (device >= n) return SJ_ERR_ARGUMENT;
    cudaDeviceProp prop;
    SJ_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return SJ_ERR_NO_DEVICE;  // sm_90a-only binary
    SJ_CUDA_CHECK(cudaSetDevice(device));
    sj_ctx* c = new (std::nothrow) sj_ctx();
    if (!c) return SJ_ERR_ARGUMENT;
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    // every failure below leaves through sj_ctx_destroy (stream, events, pinned result block, device scratch)
    const int rc = [&]() -> int {
        SJ_CUDA_CHECK(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
        c->stream = c->own_stream;
        SJ_CUDA_CHECK(cudaEventCreate(&c->ev[0]));
        SJ_CUDA_CHECK(cudaEventCreate(&c->ev[1]));
        SJ_CUDA_CHECK(cudaHostAlloc(&c->host_result, sizeof(ResultBlock), cudaHostAllocDefault));
        int r = c->result.reserve(sizeof(ResultBlock));
        if (r) return r;
        c->pending = s2_pending_alloc();
        if (!c->pending) return SJ_ERR_ARGUMENT;
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(stage1_flatten_kernel<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)S1_SMEM_BYTES));
        SJ_CUDA_CHECK(cudaFuncSetAttribute(s2s_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S2S_SMEM_EMIT));
        int per_sm = 0;
        SJ_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, stage1_flatten_kernel<true, true>, S1_THREADS,
                                                                    S1_SMEM_BYTES));
        if (per_sm < 1) return SJ_ERR_NO_DEVICE;
        if (per_sm > S1_CTAS_PER_SM) per_sm = S1_CTAS_PER_SM;
        c->s1_max_ctas = per_sm * c->sm_count;
        return SJ_OK;
    }();
    if (rc) {
        sj_ctx_destroy(c);
        return rc;
    }
    *out = c;
    return SJ_OK;
}

extern "C" void sj_ctx_destroy(sj_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    exchange_release(c);
    DevBuf* bufs[] = {&c->msg,     &c->idx,      &c->desc,     &c->result, &c->s2a,     &c->s2b,    &c->s2c,
                      &c->tape,    &c->strings,  &c->test_in,  &c->test_out, &c->test_aux, &c->args, &c->scratch,
                      &c->sz_tab,  &c->tc_roots, &c->tc_scan,  &c->staging, &c->fj, &c->s2_raw, &c->s2_slots, &c->s2_list,
                      &c->s2_out,  &c->zx_seq,   &c->zx_src,   &c->fr_rec, &c->fr_row};
    for (DevBuf* b : bufs) b->release();
    if (c->host_result) cudaFreeHost(c->host_result);
    free(c->pending);
    if (c->ev[0]) cudaEventDestroy(c->ev[0]);
    if (c->ev[1]) cudaEventDestroy(c->ev[1]);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

// stage-2 implementation of a context: 0 = streaming kernels when copy_strings is on (default), 1 = per-structural
// kernels always (the tests check the streaming kernels against them).
extern "C" int sj_ctx_set_stage2_impl(sj_ctx* c, int impl) {
    if (!c || impl < 0 || impl > 1) return SJ_ERR_ARGUMENT;
    c->s2_impl = impl;
    return SJ_OK;
}

// Host side of a rank: run the calling thread (and the threads it starts later) on the CPUs of the NUMA node the device
// hangs off, and prefer that node for its memory -- pinned staging buffers allocated afterwards (cudaHostAlloc,
// sj_host_alloc, the stream slots) then sit next to the GPU's PCIe root instead of across the socket link.  Reads
// /sys/bus/pci/devices/<bus id>/numa_node and /sys/devices/system/node/node<k>/cpulist; returns the node, or -1 when
// the topology is not exposed (single-node hosts, containers without sysfs) -- never an error.
extern "C" int sj_bind_to_device_numa(int device) {
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char* q = bus; *q; q++)
        if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
    char path[256];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return -1;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    char list[4096] = {0};
    const size_t got = fread(list, 1, sizeof list - 1, f);
    fclose(f);
    list[got] = 0;
    cpu_set_t allowed, want;
    CPU_ZERO(&want);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return -1;
    int any = 0;
    for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        const int k = sscanf(tok, "%d-%d", &a, &b);
        if (k < 1) continue;
        if (k == 1) b = a;
        for (int cpu = a; cpu <= b && cpu < CPU_SETSIZE; cpu++)
            if (CPU_ISSET(cpu, &allowed)) {
                CPU_SET(cpu, &want);
                any = 1;
            }
    }
    if (!any) return -1;  // the node's CPUs are outside this process's cpuset: leave everything as it is
    sched_setaffinity(0, sizeof want, &want);
#ifdef SYS_set_mempolicy
    if (node < 64) {
        unsigned long mask = 1ul << node;
        syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, sizeof(mask) * 8 + 1);
    }
#endif
    return node;
}

extern "C" int sj_ctx_set_stream(sj_ctx* c, void* cuda_stream) {
    if (!c) return SJ_ERR_ARGUMENT;
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : c->own_stream;
    return SJ_OK;
}

extern "C" void* sj_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void sj_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

extern "C" void sj_bounds(size_t len, size_t* tape_cap, size_t* strings_cap) {
    // tape <= 2 words per structural + 2 per record + 2; structurals <= len; records <= len/2 + 1
    if (tape_cap) *tape_cap = 2 * len + 8;
    if (strings_cap) *strings_cap = len + 64;
}

extern "C" int sj_ctx_sync(sj_ctx* c) {
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return SJ_OK;
}
extern "C" int sj_event_record(sj_ctx* c, int which) {
    SJ_CUDA_CHECK(cudaEventRecord(c->ev[which ? 1 : 0], c->stream));
    return SJ_OK;
}
extern "C" int sj_event_elapsed_ms(sj_ctx* c, float* ms) {
    SJ_CUDA_CHECK(cudaEventSynchronize(c->ev[1]));
    SJ_CUDA_CHECK(cudaEventElapsedTime(ms, c->ev[0], c->ev[1]));
    return SJ_OK;
}
extern "C" int sj_kernel_launches(sj_ctx* c, uint64_t* count) {
    *count = c->launches;
    return SJ_OK;
}

#ifdef SJ_K2R_PROBE
// K2r's section probe (s2s_slab.h; built by tools/k2r_probe.py only): the cycle sums so far into out[K2R_SECTIONS],
// then cleared
extern "C" int sj_k2r_probe_take(sj_ctx* c, unsigned long long* out) {
    static const unsigned long long zero[K2R_SECTIONS] = {};
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    SJ_CUDA_CHECK(cudaDeviceSynchronize());
    SJ_CUDA_CHECK(cudaMemcpyFromSymbol(out, sj_k2r_probe_cycles, sizeof(zero)));
    SJ_CUDA_CHECK(cudaMemcpyToSymbol(sj_k2r_probe_cycles, zero, sizeof(zero)));
    return SJ_OK;
}
#endif
#ifdef SJ_K1_PROBE
// K1's parse-mode section probe (stage1.cuh; built by tools/k1_probe.py only): the cycle sums so far into
// out[K1P_SECTIONS], then cleared
extern "C" int sj_k1_probe_take(sj_ctx* c, unsigned long long* out) {
    static const unsigned long long zero[K1P_SECTIONS] = {};
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    SJ_CUDA_CHECK(cudaDeviceSynchronize());
    SJ_CUDA_CHECK(cudaMemcpyFromSymbol(out, sj_k1_probe_cycles, sizeof(zero)));
    SJ_CUDA_CHECK(cudaMemcpyToSymbol(sj_k1_probe_cycles, zero, sizeof(zero)));
    return SJ_OK;
}
#endif

// ---------------------------------------------------------------------------------
// stage 1
// ---------------------------------------------------------------------------------
// `agg` given: the parse mode of the streaming stage 2 -- no index (d_out / cap unused), per-slab counts into agg, an
// invalid escape into *s2_error, the in-string bits of the slabs in the descriptor block (c->last_slabpar)
static int launch_stage1(sj_ctx* c, const uint8_t* d_msg, size_t len, bool ndjson, bool deltas, uint32_t* d_out,
                         size_t cap, uint32_t* d_bsmap = nullptr, SlabAgg* agg = nullptr, uint32_t* s2_error = nullptr) {
    if (len == 0 || len > SJ_MAX_MESSAGE) return SJ_ERR_TOO_LARGE;
    if ((reinterpret_cast<uintptr_t>(d_msg) & 15) != 0) return SJ_ERR_ARGUMENT;
    const int ntiles = (int)((len + S1_TILE_BYTES - 1) / S1_TILE_BYTES);
    // descriptor block: [lastp1 u32][chain-1 slots][chain-2 slots]; a slot per tile and chain
    const size_t n16 = ((size_t)ntiles + 15) & ~(size_t)15;
    const size_t off_last = 0, off_par = (n16 * 4 + 127) & ~(size_t)127, off_cnt = off_par + (size_t)ntiles * S1_DESC_STRIDE;
    const size_t off_slab = off_cnt + (size_t)ntiles * S1_DESC_STRIDE;  // per tile: in-string bits of its slabs
    const size_t desc_bytes = off_slab + n16 * 4;
    int rc = c->desc.reserve(desc_bytes);
    if (rc) return rc;
    SJ_CUDA_CHECK(cudaMemsetAsync(c->desc.p, 0, desc_bytes, c->stream));
    ResultBlock* const block = c->result.as<ResultBlock>();
    SJ_CUDA_CHECK(cudaMemsetAsync(&block->s1, 0, sizeof(Stage1Result), c->stream));
    Stage1Params p;
    p.msg = d_msg;
    p.len = len;
    p.out = d_out;
    p.out_cap = cap;
    p.lastp1 = reinterpret_cast<uint32_t*>(c->desc.as<uint8_t>() + off_last);
    p.dpar = c->desc.as<uint8_t>() + off_par;
    p.dcnt = c->desc.as<uint8_t>() + off_cnt;
    p.result = &block->s1;
    p.ntiles = ntiles;
    p.bsmap = d_bsmap;
    p.slabpar = agg ? reinterpret_cast<uint32_t*>(c->desc.as<uint8_t>() + off_slab) : nullptr;
    p.agg = agg;
    p.s2_error = s2_error;
    c->last_slabpar = p.slabpar;
    int grid = ntiles;
    if (grid > c->s1_max_ctas) grid = c->s1_max_ctas;
    // cooperative launch: the static tile deal needs every CTA of the grid resident at once
    void* args[] = {&p};
    const void* fn = agg ? (ndjson ? (const void*)stage1_flatten_kernel<true, false, true> : (const void*)stage1_flatten_kernel<false, false, true>)
                     : ndjson ? (deltas ? (const void*)stage1_flatten_kernel<true, true> : (const void*)stage1_flatten_kernel<true, false>)
                              : (deltas ? (const void*)stage1_flatten_kernel<false, true> : (const void*)stage1_flatten_kernel<false, false>);
    SJ_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(S1_THREADS), args, S1_SMEM_BYTES, c->stream));
    const int fgrid = (ntiles + 255) / 256;
    if (deltas)
        stage1_finish_kernel<true><<<fgrid, 256, 0, c->stream>>>(p);
    else
        stage1_finish_kernel<false><<<fgrid, 256, 0, c->stream>>>(p);
    c->launches += 2;
    SJ_CUDA_CHECK(cudaGetLastError());
    return SJ_OK;
}

// bytes [off, off + n) of the result block to the host, and the synchronisation that makes them valid there
static int read_back(sj_ctx* c, size_t off, size_t n) {
    SJ_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<uint8_t*>(c->host_result) + off, c->result.as<uint8_t>() + off, n,
                                  cudaMemcpyDeviceToHost, c->stream));
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return SJ_OK;
}

extern "C" int sj_stage1_launch(sj_ctx* c, const uint8_t* d_msg, size_t len, int ndjson, int deltas, uint32_t* d_out,
                                size_t cap) {
    if (!c) return SJ_ERR_ARGUMENT;
    return launch_stage1(c, d_msg, len, ndjson != 0, deltas != 0, d_out, cap);
}

extern "C" int sj_stage1_device(sj_ctx* c, const uint8_t* d_msg, size_t len, int ndjson, int deltas, uint32_t* d_out,
                                size_t cap, sj_stage1_info* info) {
    if (!c) return SJ_ERR_ARGUMENT;
    int rc = launch_stage1(c, d_msg, len, ndjson != 0, deltas != 0, d_out, cap);
    if (rc) return rc;
    rc = read_back(c, offsetof(ResultBlock, s1), sizeof(Stage1Result));
    if (rc) return rc;
    const Stage1Result r = c->host_result->s1;
    if (info) {
        info->n_idx = r.n_idx;
        info->error = r.error;
        info->ends_in_string = r.ends_in_string;
        info->last_pos = r.last_pos;
        info->overflow = r.overflow;
    }
    return SJ_OK;
}

// device copy of a host message: padded with 0x20 up to the next slab boundary so that
// look-ahead reads stay inside the allocation
static int upload_message(sj_ctx* c, const uint8_t* msg, size_t len) {
    size_t padded = ((len + S1_SLAB_BYTES - 1) / S1_SLAB_BYTES) * S1_SLAB_BYTES + 256;
    int rc = c->msg.reserve(padded);
    if (rc) return rc;
    SJ_CUDA_CHECK(cudaMemcpyAsync(c->msg.p, msg, len, cudaMemcpyHostToDevice, c->stream));
    SJ_CUDA_CHECK(cudaMemsetAsync(c->msg.as<uint8_t>() + len, 0x20, padded - len, c->stream));
    return SJ_OK;
}

// stage1_find_marks_amd64.go:115-147: the end-of-message checks
static bool stage1_ok(const Stage1Result& r, uint8_t last_char) {
    if (r.n_idx == 0) return false;
    if (r.error) return false;
    if (r.ends_in_string) return false;
    return last_char == '}' || last_char == ']';
}

extern "C" int sj_find_structural_indices(sj_ctx* c, const uint8_t* msg, size_t len, int ndjson, uint32_t* deltas,
                                          size_t cap, size_t* n) {
    if (!c || !n) return SJ_ERR_ARGUMENT;
    *n = 0;
    if (len == 0) return SJ_ERR_STAGE1;
    if (len > SJ_MAX_MESSAGE) return SJ_ERR_TOO_LARGE;
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    int rc = upload_message(c, msg, len);
    if (rc) return rc;
    size_t dcap = len / 4 + 1024;  // first guess; exact retry below if it overflows
    Stage1Result r;
    for (int attempt = 0; attempt < 2; attempt++) {
        rc = c->idx.reserve(dcap * sizeof(uint32_t));
        if (rc) return rc;
        rc = launch_stage1(c, c->msg.as<uint8_t>(), len, ndjson != 0, true, c->idx.as<uint32_t>(), dcap);
        if (rc) return rc;
        rc = read_back(c, offsetof(ResultBlock, s1), sizeof(Stage1Result));
        if (rc) return rc;
        r = c->host_result->s1;
        if (!r.overflow) break;
        dcap = (size_t)r.n_idx + 64;
    }
    *n = r.n_idx;
    if (r.n_idx > cap) return SJ_ERR_CAPACITY;
    if (r.n_idx) {
        SJ_CUDA_CHECK(cudaMemcpyAsync(deltas, c->idx.p, (size_t)r.n_idx * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                                      c->stream));
        SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    }
    uint8_t last_char = r.n_idx && r.last_pos < len ? msg[r.last_pos] : 0;
    return stage1_ok(r, last_char) ? SJ_OK : SJ_ERR_STAGE1;
}

// ---------------------------------------------------------------------------------
// unit-test hooks
// ---------------------------------------------------------------------------------
extern "C" int sj_test_block_masks(sj_ctx* c, const uint8_t* blocks, size_t nblocks, const uint64_t* carry_in,
                                   uint64_t* out) {
    if (!c || nblocks == 0) return SJ_ERR_ARGUMENT;
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    int rc = c->test_in.reserve(nblocks * 64);
    if (rc) return rc;
    rc = c->test_aux.reserve(nblocks * 4 * 8);
    if (rc) return rc;
    rc = c->test_out.reserve(nblocks * 12 * 8);
    if (rc) return rc;
    SJ_CUDA_CHECK(cudaMemcpyAsync(c->test_in.p, blocks, nblocks * 64, cudaMemcpyHostToDevice, c->stream));
    SJ_CUDA_CHECK(cudaMemcpyAsync(c->test_aux.p, carry_in, nblocks * 32, cudaMemcpyHostToDevice, c->stream));
    test_block_masks_kernel<<<(unsigned)((nblocks + 127) / 128), 128, 0, c->stream>>>(
        c->test_in.as<uint8_t>(), nblocks, c->test_aux.as<uint64_t>(), c->test_out.as<uint64_t>());
    c->launches++;
    SJ_CUDA_CHECK(cudaGetLastError());
    SJ_CUDA_CHECK(cudaMemcpyAsync(out, c->test_out.p, nblocks * 96, cudaMemcpyDeviceToHost, c->stream));
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return SJ_OK;
}

extern "C" void sj_test_geometry(uint32_t out[4]) {
    out[0] = 64;
    out[1] = S1_STEP_BYTES;
    out[2] = S1_SLAB_BYTES;
    out[3] = S1_TILE_BYTES;
}

extern "C" int sj_test_finalize(sj_ctx* c, const uint64_t* in, size_t n, uint64_t* out) {
    if (!c || n == 0) return SJ_ERR_ARGUMENT;
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    int rc = c->test_in.reserve(n * 40);
    if (rc) return rc;
    rc = c->test_out.reserve(n * 16);
    if (rc) return rc;
    SJ_CUDA_CHECK(cudaMemcpyAsync(c->test_in.p, in, n * 40, cudaMemcpyHostToDevice, c->stream));
    test_finalize_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c->stream>>>(c->test_in.as<uint64_t>(), n,
                                                                            c->test_out.as<uint64_t>());
    c->launches++;
    SJ_CUDA_CHECK(cudaGetLastError());
    SJ_CUDA_CHECK(cudaMemcpyAsync(out, c->test_out.p, n * 16, cudaMemcpyDeviceToHost, c->stream));
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return SJ_OK;
}

extern "C" int sj_test_flatten_bits(sj_ctx* c, const uint64_t* masks, size_t nmasks, uint32_t* deltas, size_t cap,
                                    size_t* n) {
    if (!c || nmasks == 0 || !n) return SJ_ERR_ARGUMENT;
    SJ_CUDA_CHECK(cudaSetDevice(c->device));
    int rc = c->test_in.reserve(nmasks * 8);
    if (rc) return rc;
    rc = c->test_out.reserve((cap + 1) * 4);
    if (rc) return rc;
    rc = c->test_aux.reserve(16);
    if (rc) return rc;
    SJ_CUDA_CHECK(cudaMemcpyAsync(c->test_in.p, masks, nmasks * 8, cudaMemcpyHostToDevice, c->stream));
    test_flatten_kernel<<<1, 32, 0, c->stream>>>(c->test_in.as<uint64_t>(), nmasks, c->test_out.as<uint32_t>(), cap,
                                                 c->test_aux.as<uint64_t>());
    c->launches++;
    SJ_CUDA_CHECK(cudaGetLastError());
    uint64_t res[2];
    SJ_CUDA_CHECK(cudaMemcpyAsync(res, c->test_aux.p, 16, cudaMemcpyDeviceToHost, c->stream));
    SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    *n = res[0];
    if (res[1] || res[0] > cap) return SJ_ERR_CAPACITY;
    if (res[0]) {
        SJ_CUDA_CHECK(cudaMemcpyAsync(deltas, c->test_out.p, res[0] * 4, cudaMemcpyDeviceToHost, c->stream));
        SJ_CUDA_CHECK(cudaStreamSynchronize(c->stream));
    }
    return SJ_OK;
}

#include "sj_exchange.inl"
#include "sj_parse.inl"
#include "sj_tape.inl"
#include "sj_consume.inl"
#include "sj_marshal.inl"
#include "sj_find.inl"
#include "sj_find_rows.inl"
#include "sj_s2.inl"
#include "sj_zstd.inl"
#include "sj_serialize.inl"
#include "sj_stream.inl"
#include "sj_gen.inl"
