/* abi_example.c -- the C ABI used from plain C (what a cgo / JNI / FFI binding sees): compiled as C11 by the
 * CPU test-suite to prove that include/simdjson_b200.h is a C header and that the library links without any
 * C++ or CUDA types in the signatures.  Exit code 3 (SJ_ERR_NO_DEVICE) on a machine without an sm_90 GPU:
 * there is no CPU fallback.
 *   gcc -std=c11 -Wall -Wextra -Werror -Iinclude tools/abi_example.c -Lsimdjson-go_b200 -lsimdjson_b200 \
 *       -Wl,-rpath,$PWD/simdjson-go_b200 -o /tmp/abi_example */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "simdjson_b200.h"

int main(void) {
    static const char doc[] = " {\"Make\":\"HOND\",\"n\":[1,2.5,true]}\n{\"Make\":\"TOYT\"}\n";
    size_t start = 0, stop = 0;
    sj_trim_space((const uint8_t*)doc, sizeof doc - 1, &start, &stop); /* host-only helper: works everywhere */
    printf("trimmed window: [%zu, %zu)\n", start, stop);
    if (!sj_supported()) {
        sj_ctx* none = NULL;
        int rc = sj_ctx_create(0, &none);
        printf("no sm_90 device: sj_ctx_create -> %d (%s)\n", rc, sj_error_string(rc));
        return rc;
    }
    sj_ctx* ctx = NULL;
    int rc = sj_ctx_create(-1, &ctx);
    if (rc != SJ_OK) return rc;
    size_t tape_cap = 0, str_cap = 0, tape_len = 0, str_len = 0, off = 0, n = 0;
    sj_bounds(sizeof doc - 1, &tape_cap, &str_cap);
    uint64_t* tape = malloc(tape_cap * sizeof *tape);
    uint8_t* strings = malloc(str_cap);
    rc = sj_parse(ctx, (const uint8_t*)doc, sizeof doc - 1, SJ_FLAG_NDJSON | SJ_FLAG_COPY_STRINGS, tape, tape_cap, &tape_len,
                  strings, str_cap, &str_len, &off, &n);
    printf("sj_parse -> %d (%s): %zu tape words, %zu string bytes, message window [%zu, %zu)\n", rc, sj_error_string(rc),
           tape_len, str_len, off, off + n);
    uint64_t roots = 0, matches = 0;
    if (rc == SJ_OK)
        rc = sj_parse_count_where(ctx, (const uint8_t*)doc, sizeof doc - 1, SJ_FLAG_NDJSON | SJ_FLAG_COPY_STRINGS,
                                  (const uint8_t*)"Make", 4, (const uint8_t*)"HOND", 4, &roots, &matches);
    printf("sj_parse_count_where -> %d: %llu records, %llu with Make == HOND\n", rc, (unsigned long long)roots,
           (unsigned long long)matches);
    free(tape);
    free(strings);
    sj_ctx_destroy(ctx);
    return rc;
}
