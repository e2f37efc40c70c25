// fmt_shim.cpp -- the formatting of csrc/fmt.h (what the marshal kernels run), compiled with g++ for the CPU tests.
#include "../../simdjson-go_b200/csrc/fmt.h"

extern "C" {

// item i of n is written at out + 32 * i, its length to len[i]
void fmt_shim_doubles(const uint64_t* bits, size_t n, uint8_t* out, uint32_t* len) {
    for (size_t i = 0; i < n; i++) {
        const uint32_t m = sj::fmt_double<false>(bits[i], nullptr);
        len[i] = sj::fmt_double<true>(bits[i], out + 32 * i);
        if (m != len[i]) len[i] = 0xffffffffu;  // measured and written lengths must agree
    }
}

void fmt_shim_ints(const uint64_t* v, size_t n, int is_signed, uint8_t* out, uint32_t* len) {
    for (size_t i = 0; i < n; i++) {
        const uint32_t m = is_signed ? sj::fmt_i64<false>((int64_t)v[i], nullptr) : sj::fmt_u64<false>(v[i], nullptr);
        len[i] = is_signed ? sj::fmt_i64<true>((int64_t)v[i], out + 32 * i) : sj::fmt_u64<true>(v[i], out + 32 * i);
        if (m != len[i]) len[i] = 0xffffffffu;
    }
}

size_t fmt_shim_escape(const uint8_t* src, size_t n, uint8_t* out) {
    size_t o = 0;
    for (size_t i = 0; i < n; i++) {
        const uint32_t m = sj::fmt_escape(src[i], out + o);
        if (m != sj::fmt_escaped_len(src[i])) return (size_t)-1;
        o += m;
    }
    return o;
}

void fmt_shim_pow10_g(int q, uint64_t* hi, uint64_t* lo) { sj::fmt_pow10_g(q, hi, lo); }
}
