// consume.cuh -- device-side consumers of the tape (SURVEY.md section 8(f), rank 2).
//
// The reference's NDJSON workloads parse a stream and then walk the tape on the host:
//   countWhere(key, value, pj)   ndjson_test.go:421-459   (BenchmarkNdjsonColdCountStarWithWhere,
//                                                          parse_json_amd64_test.go:134-157)
//   countObjects(pj)             ndjson_test.go:461-474
//   Object.FindKey               parsed_object.go:97-140
// With the tape built in HBM the walk can stay there too: the answer is two integers, so the
// D2H copy of a tape 1.7x the size of the input (the PCIe leg that bounds sj_parse) disappears.
//
//   KC1a tc_root_count   any device tape: root-open words ('r' whose payload points forward, and a head: not
//                        the value word of a string or number, by KM1 mj_heads_reduce and its scans) per tile
//                        of MJ_TILE words, whose counts scan_groups_kernel scans (twice).  On every tape the
//                        parser or Deserialize writes these are the roots ForEach visits.
//   KC1b tc_root_write   their slots, in tape order (the rows of the device find, find.cuh)
//   KC2 tc_count_where   one thread per root: FindKey over the top-level keys of the record's
//                        object, first match decides (FindKey returns the first element of that name)
#pragma once
#include "common.cuh"
#include "marshal.cuh"
#include "stage2_common.cuh"

namespace sj {

constexpr uint64_t TC_VALUE_MASK = 0x00ffffffffffffffull;  // JSONVALUEMASK, parsed_json.go:26
constexpr uint64_t TC_STRINGBUFBIT = 0x80000000000000ull;  // parsed_json.go:29

struct CountParams {
    const uint64_t* tape;
    uint64_t tape_len;
    const uint8_t* strings;  // Strings.B
    const uint8_t* msg;      // Message (no-copy strings point into it)
    const uint32_t* roots;   // tape slot of every root-open word
    uint32_t roots_skip0;    // 1: roots[0] is not stored and means slot 0 (stage 2's rootpos array)
    uint64_t n_roots;
    const uint8_t* key;      // device copies of the needle strings
    uint32_t key_len;
    const uint8_t* value;
    uint32_t value_len;
    unsigned long long* counters;  // [1] matches
};

__device__ __forceinline__ bool tc_is_root_open(uint64_t w, uint64_t i) { return (w >> 56) == 'r' && (w & TC_VALUE_MASK) > i; }

// which of a thread's MJ_ROUNDS consecutive words are root opens: 'r' words pointing forward that are heads, i.e. not the
// value word of the string or number in front of them (KM1's transfer function, scanned from word 0).  A number whose
// value word happens to start with the byte 'r' (int64s from 0x72 << 56, doubles near 1e241-1e246) is no root.
__device__ __forceinline__ uint32_t tc_root_opens(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre, const HAgg* h_grp_pre,
                                                  uint64_t base) {
    uint64_t w[MJ_ROUNDS];
    HAgg a{};
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++) {
        w[j] = base + j < n ? tape[base + j] : 0;
        if (base + j < n) a = agg_combine(a, mj_word_agg(w[j], base + j));
    }
    HAgg total;
    const HAgg ex = block_exclusive_scan(a, total);
    HAgg pre = agg_combine(agg_combine(h_grp_pre[blockIdx.x >> 10], h_tile_pre[blockIdx.x]), ex);
    uint32_t open = 0;
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++) {
        if (base + j < n && hagg_out(pre, 1) && tc_is_root_open(w[j], base + j)) open |= 1u << j;
        pre = agg_combine(pre, mj_word_agg(w[j], base + j));
    }
    return open;
}

// KC1a: root opens per tile of MJ_TILE words (MJ_ROUNDS consecutive words per thread), after KM1 and its scans
__global__ void __launch_bounds__(MJ_THREADS) tc_root_count_kernel(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre,
                                                                   const HAgg* h_grp_pre, MSum* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)threadIdx.x * MJ_ROUNDS;
    const uint32_t open = tc_root_opens(tape, n, h_tile_pre, h_grp_pre, base);
    MSum total;
    block_exclusive_scan(MSum{(uint64_t)__popc(open)}, total);
    if (threadIdx.x == 0) tile[blockIdx.x] = total;
}

// KC1b: the slots, in tape order
__global__ void __launch_bounds__(MJ_THREADS) tc_root_write_kernel(const uint64_t* tape, uint64_t n, const HAgg* h_tile_pre,
                                                                   const HAgg* h_grp_pre, const MSum* tile_pre,
                                                                   const MSum* grp_pre, uint32_t* roots) {
    const uint64_t base = (uint64_t)blockIdx.x * MJ_TILE + (uint64_t)threadIdx.x * MJ_ROUNDS;
    const uint32_t open = tc_root_opens(tape, n, h_tile_pre, h_grp_pre, base);
    MSum total;
    uint64_t at = grp_pre[blockIdx.x >> 10].v + tile_pre[blockIdx.x].v + block_exclusive_scan(MSum{(uint64_t)__popc(open)}, total).v;
#pragma unroll
    for (int j = 0; j < MJ_ROUNDS; j++)
        if (open >> j & 1) roots[at++] = (uint32_t)(base + j);
}

// the bytes of the string whose first tape word is w (parsed_json.go:107-120 stringByteAt)
__device__ __forceinline__ const uint8_t* tc_string_ptr(const CountParams& p, uint64_t w) {
    const uint64_t v = w & TC_VALUE_MASK;
    return (v & TC_STRINGBUFBIT) ? p.strings + (v - TC_STRINGBUFBIT) : p.msg + v;
}
__device__ __forceinline__ bool tc_bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t n) {
    for (uint32_t k = 0; k < n; k++)
        if (a[k] != b[k]) return false;
    return true;
}

__global__ void __launch_bounds__(256) tc_count_where_kernel(const CountParams p) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (r < p.n_roots) {
        const uint64_t open = (p.roots_skip0 && r == 0) ? 0 : p.roots[r];
        // iter.Root(): the element under the root; countWhere only looks at objects (ndjson_test.go:441-447)
        if (open + 2 < p.tape_len) {
            const uint64_t w1 = p.tape[open + 1];
            if ((w1 >> 56) == '{') {
                const uint64_t close = (w1 & TC_VALUE_MASK) - 1;  // '{' points one past its '}'
                uint64_t i = open + 2;
                // Object.FindKey (parsed_object.go:97-140): name, value, name, value ... up to the '}'
                while (i < close && i + 2 < p.tape_len) {
                    const uint64_t kw = p.tape[i];
                    if ((kw >> 56) != '"') break;
                    const uint64_t klen = p.tape[i + 1];
                    const uint64_t vi = i + 2;
                    const uint64_t vw = p.tape[vi];
                    const uint32_t vt = (uint32_t)(vw >> 56);
                    if (klen == p.key_len && tc_bytes_equal(tc_string_ptr(p, kw), p.key, p.key_len)) {
                        // first element of that name decides: elem.Type == TypeString && bytes == value
                        if (vt == '"' && vi + 1 < p.tape_len && p.tape[vi + 1] == p.value_len &&
                            tc_bytes_equal(tc_string_ptr(p, vw), p.value, p.value_len))
                            hit = true;
                        break;
                    }
                    // skip the value (Iter.Advance, parsed_json.go:158-214)
                    uint64_t next;
                    if (vt == '"' || vt == 'l' || vt == 'u' || vt == 'd')
                        next = vi + 2;
                    else if (vt == '{' || vt == '[')
                        next = vw & TC_VALUE_MASK;  // one past the matching close
                    else
                        next = vi + 1;  // t f n
                    if (next <= i) break;  // never loop on a corrupt tape
                    i = next;
                }
            }
        }
    }
    const uint32_t mh = __ballot_sync(FULL, hit);
    if ((threadIdx.x & 31) == 0 && mh) atomicAdd(&p.counters[1], (unsigned long long)__popc(mh));
}

}  // namespace sj
