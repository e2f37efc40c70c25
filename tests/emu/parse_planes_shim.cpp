// parse_planes_shim.cpp -- the classes stage 1's parse mode rebuilds from st and its two extra planes (parse_planes,
// classes_from_parse_planes in simdjson-go_b200/csrc/s2s_core.h) next to classify_block2, built with g++ (test
// infrastructure, NOT the product).
#include "../../simdjson-go_b200/csrc/s2s_core.h"

using namespace sj;

// blocks: n x 64 bytes.  out: 10 x uint64 per block -- open, close, cc, numc, atomc of classify_block2, then the same
// five rebuilt from st = open | close | cc (stage 1's structurals) and the X / Y planes of the same transpose
extern "C" void parse_planes_check(const uint8_t* blocks, size_t n, uint64_t* out) {
    for (size_t i = 0; i < n; i++) {
        uint32_t w[16];
        for (int k = 0; k < 16; k++)
            w[k] = (uint32_t)blocks[64 * i + 4 * k] | (uint32_t)blocks[64 * i + 4 * k + 1] << 8 |
                   (uint32_t)blocks[64 * i + 4 * k + 2] << 16 | (uint32_t)blocks[64 * i + 4 * k + 3] << 24;
        const Class64 c = classify_block2(w);
        uint32_t p0[8], p1[8];
        bit_planes32(&w[0], p0);
        bit_planes32(&w[8], p1);
        const ParsePlanes a = parse_planes(p0), b = parse_planes(p1);
        const Class64 r = classes_from_parse_planes(c.open | c.close | c.cc, mk64(a.x, b.x), mk64(a.y, b.y));
        uint64_t* o = out + 10 * i;
        o[0] = c.open, o[1] = c.close, o[2] = c.cc, o[3] = c.numc, o[4] = c.atomc;
        o[5] = r.open, o[6] = r.close, o[7] = r.cc, o[8] = r.numc, o[9] = r.atomc;
    }
}
