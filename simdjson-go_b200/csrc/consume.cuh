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
//   KC2 tc_count_where   one thread per root (stage 2's root list, or KC1a / KC1b of tape.cuh): FindKey over the
//                        top-level keys of the record's object, first match decides (FindKey returns the first element
//                        of that name)
#pragma once
#include "common.cuh"
#include "tape.cuh"

namespace sj {

struct CountParams {
    // msg_len and strings_len are UINT64_MAX: sj_count_where_device takes no buffer lengths, so the string reads below
    // are not bounds-checked.  Checking them needs the lengths in the C ABI, a change of its own.
    TapeView t;
    TapeRows roots;
    const uint8_t* key;      // device copies of the needle strings
    uint32_t key_len;
    const uint8_t* value;
    uint32_t value_len;
    unsigned long long* counters;  // [1] matches
};

__device__ __forceinline__ bool tc_bytes_equal(const uint8_t* a, const uint8_t* b, uint32_t n) {
    for (uint32_t k = 0; k < n; k++)
        if (a[k] != b[k]) return false;
    return true;
}

__global__ void __launch_bounds__(256) tc_count_where_kernel(const CountParams p) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (r < p.roots.n) {
        const uint64_t open = tape_root(p.roots, r);
        // iter.Root(): the element under the root; countWhere only looks at objects (ndjson_test.go:441-447)
        if (open + 2 < p.t.n) {
            const uint64_t w1 = p.t.tape[open + 1];
            if ((w1 >> 56) == '{') {
                const uint64_t close = (w1 & TAPE_VALUE_MASK) - 1;  // '{' points one past its '}'
                uint64_t i = open + 2;
                // Object.FindKey (parsed_object.go:97-140): name, value, name, value ... up to the '}'
                while (i < close && i + 2 < p.t.n) {
                    const uint64_t kw = p.t.tape[i];
                    if ((kw >> 56) != '"') break;
                    const uint64_t klen = p.t.tape[i + 1];
                    const uint64_t vi = i + 2;
                    const uint64_t vw = p.t.tape[vi];
                    const uint32_t vt = (uint32_t)(vw >> 56);
                    if (klen == p.key_len && tc_bytes_equal(tape_string_ptr(p.t, kw), p.key, p.key_len)) {
                        // first element of that name decides: elem.Type == TypeString && bytes == value
                        if (vt == '"' && vi + 1 < p.t.n && p.t.tape[vi + 1] == p.value_len &&
                            tc_bytes_equal(tape_string_ptr(p.t, vw), p.value, p.value_len))
                            hit = true;
                        break;
                    }
                    // skip the value (Iter.Advance, parsed_json.go:158-214)
                    uint64_t next;
                    if (tape_value_tag(vt))
                        next = vi + 2;
                    else if (vt == '{' || vt == '[')
                        next = vw & TAPE_VALUE_MASK;  // one past the matching close
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
