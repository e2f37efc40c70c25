// s2.cuh -- the S2 stream codec of the Serializer's CompressFast blocks (block type 1, parsed_serialize.go:791-833
// encBlock / :697-756 decBlock) on the device.
//
// An S2 stream is the identifier chunk ff 06 00 00 "S2sTwO" and then chunks of a type byte, a 3-byte little-endian
// length and the body.  A compressed (0x00) or stored (0x01) chunk's body starts with the masked CRC-32C of its
// uncompressed bytes, ((c >> 15) | (c << 17)) + 0xa282ead8; a compressed chunk's block is uvarint(decoded length) and
// then literals and copies.  Every chunk stands alone, so each is a warp's work:
//   KC1 sx_encode   one warp per chunk of S2_CHUNK input bytes: greedy matches from a hash table of positions in shared
//                   memory, 32 positions per step, in a fixed order (so the output does not depend on scheduling); only
//                   the Snappy subset (literals, copies with 1- and 2-byte offsets); stored when that is not shorter.
//                   The framed chunk goes into its own slot, its size into size[].
//   KC2 sx_gather   the slots laid end to end behind the block heads.
//   KX1 zx_list     (zstd.cuh) one thread per S2 block walks its chunk headers (sx_walk), applies the framing rules
//                   (s2.Reader's chunk loop) and lists the chunks that fill the block, with their output offsets.
//   KX2 sx_decode   one warp per listed chunk: literals and copies straight into global memory (a copy may reach back
//                   4 MiB), the decoded length and the CRC checked.
#pragma once
#include "serialize.cuh"

namespace sj {

constexpr uint32_t S2_CHUNK = 65536;         // input bytes per chunk KC1 writes (copies then need 2-byte offsets at most)
constexpr uint32_t S2_SLOT = 8 + S2_CHUNK + 8;  // a framed chunk KC1 writes: header, CRC, at most S2_CHUNK body bytes
constexpr uint32_t S2_MAX_DECODED = 4u << 20;   // a chunk of an S2 stream decodes to at most this
constexpr uint32_t S2_SNAPPY_MAX_DECODED = 65536;  // ... of a stream whose identifier is Snappy's
constexpr int S2_HASH_BITS = 13;
constexpr int S2_WARPS = 4;                  // warps per CTA of KC1 / KX2
constexpr uint32_t S2_IDENT_LEN = 10;
constexpr uint32_t S2_NONE = 0xff;           // SxBlock::type of a block with neither size nor type byte
static_assert(S2_CHUNK <= 65536, "KC1 keeps positions in uint16 and writes copies with 2-byte offsets");

// ---------------------------------------------------------------------------------
// CRC-32C (Castagnoli, reflected polynomial 0x82f63b78)
// ---------------------------------------------------------------------------------
constexpr uint32_t S2_CRC_POLY = 0x82f63b78u;

// x^(8 * 2^k) mod P, reflected: shifting a CRC over 2^k bytes of zeros is a multiplication by it
__constant__ uint32_t sx_x8pow[32] = {
    0x00800000, 0x00008000, 0x82f63b78, 0x6ea2d55c, 0x18b8ea18, 0x510ac59a, 0xb82be955, 0xb8fdb1e7,
    0x88e56f72, 0x74c360a4, 0xe4172b16, 0x0d65762a, 0x35d73a62, 0x28461564, 0xbf455269, 0xe2ea32dc,
    0xfe7740e6, 0xf946610b, 0x3c204f8f, 0x538586e3, 0x59726915, 0x734d5309, 0xbc1ac763, 0x7d0722cc,
    0xd289cabe, 0xe94ca9bc, 0x05b74f3f, 0xa51e1f42, 0x40000000, 0x20000000, 0x08000000, 0x00800000};

// a * b mod P (reflected: bit 31 is x^0)
__device__ __forceinline__ uint32_t sx_gf_mul(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        if (a & (0x80000000u >> i)) p ^= b;
        b = (b >> 1) ^ ((b & 1) ? S2_CRC_POLY : 0);
    }
    return p;
}

// the CRC register r carried over n more bytes of zeros: r * x^(8n) mod P
__device__ __forceinline__ uint32_t sx_crc_shift(uint32_t r, uint64_t n) {
    for (int k = 0; n && r; k++, n >>= 1)
        if (n & 1) r = sx_gf_mul(sx_x8pow[k & 31], r);
    return r;
}

__device__ __forceinline__ void sx_crc_table(uint32_t* tab) {
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t r = i;
        for (int k = 0; k < 8; k++) r = (r >> 1) ^ ((r & 1) ? S2_CRC_POLY : 0);
        tab[i] = r;
    }
}

// the masked CRC-32C of d[0, n), by the whole warp: each lane runs the table over its slice from register 0, the
// slices are joined by shifting each over the bytes behind it (the register is linear in the bytes), and the initial
// ~0 enters shifted over all n bytes
__device__ __forceinline__ uint32_t sx_crc_warp(const uint8_t* d, uint64_t n, const uint32_t* tab) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t slice = (n + 31) / 32, b = min(n, lane * slice), e = min(n, b + slice);
    uint32_t r = 0;
    for (uint64_t i = b; i < e; i++) r = tab[(r ^ d[i]) & 0xff] ^ (r >> 8);
    r = sx_crc_shift(r, n - e);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) r ^= __shfl_xor_sync(FULL, r, s);
    const uint32_t c = ~(r ^ sx_crc_shift(0xffffffffu, n));
    return ((c >> 15) | (c << 17)) + 0xa282ead8u;
}

// ---------------------------------------------------------------------------------
// KC1 / KC2: encode
// ---------------------------------------------------------------------------------
struct SxEncParams {
    const uint8_t* src[3];  // up to three inputs, each cut into chunks of S2_CHUNK bytes
    uint64_t len[3];
    uint32_t first[4];      // input b has chunks first[b] .. first[b + 1] - 1
    uint32_t codec[3];      // input b's block type: 1 (S2, KC1's chunks) or 2 (zstd, KZ1's: zstd.cuh)
    uint32_t nchunks;
    uint8_t* slots;         // S2_SLOT bytes per chunk
    uint32_t* size;         // framed bytes of each chunk
    const uint64_t* dst;    // KC2: where each chunk goes in out
    uint8_t* out;
};

__device__ __forceinline__ uint32_t sx_load32(const uint8_t* p) {
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}

// a literal of L bytes at out + o (lane 0 the tag, all lanes the bytes); false when it would end past `limit`
__device__ __forceinline__ bool sx_emit_literal(uint8_t* out, uint32_t& o, uint32_t limit, const uint8_t* s, uint32_t L) {
    if (L == 0) return true;
    const uint32_t x = L - 1, h = x < 60 ? 1 : x < 256 ? 2 : x < 65536 ? 3 : 4;
    if (o + h + L > limit) return false;
    if ((threadIdx.x & 31) == 0) {
        if (x < 60) {
            out[o] = (uint8_t)(x << 2);
        } else {
            out[o] = (uint8_t)((59 + h - 1) << 2);
            for (uint32_t k = 1; k < h; k++) out[o + k] = (uint8_t)(x >> (8 * (k - 1)));
        }
    }
    o += h;
    for (uint32_t k = threadIdx.x & 31; k < L; k += 32) out[o + k] = s[k];
    o += L;
    return true;
}

// a match of L >= 4 bytes at offset 1 <= off < 65536 as Snappy's emitCopy writes it: 64-byte copies while at least 68
// are left, a 60-byte one when 65 .. 67 are, then a 1-byte-offset copy for 4 .. 11 bytes at offsets below 2048, else a
// 2-byte-offset copy
__device__ __forceinline__ bool sx_emit_copy(uint8_t* out, uint32_t& o, uint32_t limit, uint32_t off, uint32_t L) {
    const bool lane0 = (threadIdx.x & 31) == 0;
    while (L > 0) {
        uint32_t l = L >= 68 ? 64 : L > 64 ? 60 : L;
        if (l < 12 && off < 2048) {
            if (o + 2 > limit) return false;
            if (lane0) {
                out[o] = (uint8_t)(1 | ((l - 4) << 2) | ((off >> 8) << 5));
                out[o + 1] = (uint8_t)off;
            }
            o += 2;
        } else {
            if (o + 3 > limit) return false;
            if (lane0) {
                out[o] = (uint8_t)(2 | ((l - 1) << 2));
                out[o + 1] = (uint8_t)off;
                out[o + 2] = (uint8_t)(off >> 8);
            }
            o += 3;
        }
        L -= l;
    }
    return true;
}

// The match finder of KC1 (and of the zstd encoder, zstd.cuh) over in[0, n), by the whole warp: e.literal(s, L) and
// e.copy(offset, L) in position order, false as soon as one of them is.  Steps of 32 positions: every position hashes
// its 4 bytes, its candidate is the last earlier position of the step with the same 4 bytes, else the table's
// (checked); then the table takes the step's positions (the last of each hash), and the matches are taken greedily in
// position order, each extended 32 bytes at a time.  The next step starts behind the step or behind the last match,
// whichever is later.  Matches are at least 4 bytes, offsets below n <= 65536.
template <class Emit>
__device__ bool sx_match_warp(const uint8_t* in, uint32_t n, uint16_t* tab, Emit& e) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = lane; i < (1u << S2_HASH_BITS) / 2; i += 32) reinterpret_cast<uint32_t*>(tab)[i] = 0xffffffffu;
    __syncwarp();
    uint32_t emit = 0;
    for (uint32_t s = 0; n >= 4 && s <= n - 4;) {
        const uint32_t pos = s + lane;
        const bool valid = pos <= n - 4;
        const uint32_t vm = __ballot_sync(FULL, valid);
        const uint32_t v = valid ? sx_load32(in + pos) : 0;
        const uint32_t h = (v * 0x1e35a7bdu) >> (32 - S2_HASH_BITS);
        const uint32_t below = __match_any_sync(FULL, v) & vm & ((1u << lane) - 1);
        uint32_t cand = 0;
        bool has = false;
        if (valid) {
            if (below) {
                cand = s + 31 - __clz(below);
                has = true;
            } else {
                cand = tab[h];
                has = cand != 0xffff && sx_load32(in + cand) == v;
            }
        }
        const uint32_t hs = __match_any_sync(FULL, h) & vm;
        __syncwarp();
        if (valid && 31 - __clz(hs) == lane) tab[h] = (uint16_t)pos;
        __syncwarp();
        uint32_t m = __ballot_sync(FULL, has && pos >= emit);
        while (m) {
            const int l = __ffs(m) - 1;
            const uint32_t p0 = s + l, c0 = __shfl_sync(FULL, cand, l);
            uint32_t len = 4;
            for (;;) {
                const uint32_t k = p0 + len + lane;
                const uint32_t ne = __ballot_sync(FULL, k >= n || in[k] != in[c0 + len + lane]);
                if (ne) {
                    len += __ffs(ne) - 1;
                    break;
                }
                len += 32;
            }
            if (!e.literal(in + emit, p0 - emit) || !e.copy(p0 - c0, len)) return false;
            emit = p0 + len;
            m &= emit - s >= 32 ? 0u : ~((1u << (emit - s)) - 1);
        }
        s = max(s + 32, emit);
    }
    return e.literal(in + emit, n - emit);
}

// sx_match_warp's elements as Snappy literals and copies at out + o, none ending past `limit`
struct SxSnappyEmit {
    uint8_t* out;
    uint32_t o, limit;
    __device__ bool literal(const uint8_t* s, uint32_t L) { return sx_emit_literal(out, o, limit, s, L); }
    __device__ bool copy(uint32_t off, uint32_t L) { return sx_emit_copy(out, o, limit, off, L); }
};

// The block of in[0, n) into out, by the whole warp: its length, or ~0u when it would not be shorter than n
__device__ uint32_t sx_compress_warp(const uint8_t* in, uint32_t n, uint8_t* out, uint16_t* tab) {
    const uint32_t lane = threadIdx.x & 31;
    uint32_t o = 0;
    for (uint32_t x = n; ; x >>= 7) {  // uvarint(n)
        if (lane == 0) out[o] = (uint8_t)(x >= 0x80 ? (x | 0x80) : x);
        o++;
        if (x < 0x80) break;
    }
    SxSnappyEmit e{out, o, n};
    return sx_match_warp(in, n, tab, e) ? e.o : ~0u;
}

// KC1: chunk ci of its input, framed, into slot ci
constexpr size_t S2_ENCODE_SMEM = 1024 + S2_WARPS * (2u << S2_HASH_BITS);  // the CRC table, a hash table per warp

__global__ void __launch_bounds__(S2_WARPS * 32) sx_encode_kernel(const SxEncParams p) {
    extern __shared__ uint32_t sx_smem[];
    uint32_t* crc_tab = sx_smem;
    sx_crc_table(crc_tab);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t ci = blockIdx.x * S2_WARPS + warp;
    if (ci >= p.nchunks) return;
    int b = 0;
    while (ci >= p.first[b + 1]) b++;
    if (p.codec[b] != 1) return;
    const uint64_t at = (uint64_t)(ci - p.first[b]) * S2_CHUNK;
    const uint32_t n = (uint32_t)min((uint64_t)S2_CHUNK, p.len[b] - at);
    const uint8_t* in = p.src[b] + at;
    uint8_t* slot = p.slots + (uint64_t)ci * S2_SLOT;
    uint32_t body = sx_compress_warp(in, n, slot + 8, reinterpret_cast<uint16_t*>(sx_smem + 256) + (warp << S2_HASH_BITS));
    const bool stored = body >= n;
    if (stored) {
        __syncwarp();
        for (uint32_t k = lane; k < n; k += 32) slot[8 + k] = in[k];
        body = n;
    }
    const uint32_t crc = sx_crc_warp(in, n, crc_tab);
    if (lane == 0) {
        const uint32_t L = body + 4;
        slot[0] = stored ? 1 : 0;
        slot[1] = (uint8_t)L;
        slot[2] = (uint8_t)(L >> 8);
        slot[3] = (uint8_t)(L >> 16);
        for (int k = 0; k < 4; k++) slot[4 + k] = (uint8_t)(crc >> (8 * k));
        p.size[ci] = 8 + body;
    }
}

// KC2: slot ci to out + dst[ci], one CTA per chunk
__global__ void __launch_bounds__(256) sx_gather_kernel(const SxEncParams p) {
    const uint32_t ci = blockIdx.x;
    const uint8_t* s = p.slots + (uint64_t)ci * S2_SLOT;
    uint8_t* d = p.out + p.dst[ci];
    const uint32_t n = p.size[ci];
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) d[k] = s[k];
}

// ---------------------------------------------------------------------------------
// KX1 / KX2: decode
// ---------------------------------------------------------------------------------
struct SxBlock {
    uint64_t at, size, raw;  // the block's bytes behind its type byte in the input, and its uncompressed size
    uint32_t type;           // 0, 1 (S2), 2 (zstd), S2_NONE
    uint32_t pad;
};

struct SxChunk {
    uint64_t src;  // the chunk's body (behind its 4-byte header) in the input
    uint64_t dst;  // its decoded bytes in its block's region
    uint32_t len;  // body bytes (CRC included)
    uint32_t n;    // decoded bytes
    uint32_t type; // 0 compressed, 1 stored
    uint32_t block;
};

// KX1's read-back; KX2 sets bad too
struct SxBack {
    uint32_t type[4];
    uint64_t total[4];  // decoded bytes of the chunks listed for each S2 block
    uint32_t count;     // chunks listed (only the first `cap` are stored)
    uint32_t bad;       // an S2 block breaks a framing rule (KX1) or a chunk does not decode (KX2)
};

// where each block's bytes are, read as KD0 read them (only called on a header KD0 accepted)
__device__ void sx_header_blocks(const uint8_t* s, uint64_t len, SxBlock* b) {
    uint64_t at = 1, x;
    dz_uvarint(s, len, at, x);
    dz_uvarint(s, len, at, x);
    for (int i = 0; i < 4; i++) {
        SxBlock r{};
        dz_uvarint(s, len, at, r.raw);
        dz_uvarint(s, len, at, r.size);
        r.type = S2_NONE;
        if (r.size) {
            r.type = s[at++];
            r.size--;
            r.at = at;
            at += r.size;
        }
        b[i] = r;
    }
}

// s2.Reader's chunk loop over block i (S2), until it has produced blk.raw bytes
__device__ bool sx_walk(const uint8_t* s, const SxBlock& blk, uint32_t i, SxChunk* list, uint32_t cap, SxBack* back) {
    uint64_t p = blk.at, filled = 0;
    const uint64_t end = blk.at + blk.size;
    bool first = true, snappy = false;
    while (filled < blk.raw) {
        if (end - p < 4) return false;  // out of chunks
        const uint32_t t = s[p], L = (uint32_t)s[p + 1] | (uint32_t)s[p + 2] << 8 | (uint32_t)s[p + 3] << 16;
        p += 4;
        if (L > end - p) return false;
        if (first && t != 0xff) return false;
        first = false;
        if (t == 0xff) {  // stream identifier
            if (L != 6) return false;
            const char* s2id = "S2sTwO";
            const char* snid = "sNaPpY";
            bool is_s2 = true, is_sn = true;
            for (int k = 0; k < 6; k++) {
                is_s2 &= s[p + k] == (uint8_t)s2id[k];
                is_sn &= s[p + k] == (uint8_t)snid[k];
            }
            if (!is_s2 && !is_sn) return false;
            snappy = is_sn;
        } else if (t == 0x00 || t == 0x01) {
            if (L < 4) return false;
            uint64_t n = L - 4;
            if (t == 0x00) {
                uint64_t at = p + 4;
                if (!dz_uvarint(s, p + L, at, n)) return false;
            }
            if (n > (snappy ? S2_SNAPPY_MAX_DECODED : S2_MAX_DECODED)) return false;
            const uint32_t k = atomicAdd(&back->count, 1u);
            if (k < cap) list[k] = SxChunk{p, filled, L, (uint32_t)n, t, i};
            filled += n;
        } else if (t < 0x80) {  // 0x02 .. 0x7f: reserved unskippable
            return false;
        }  // 0x80 .. 0xfe: skippable
        p += L;
    }
    back->total[i] = filled;
    return true;
}

// a copy of L bytes from `off` back, by the whole warp: 32 bytes a step when off >= 32 (each step reads only bytes
// written before it), else the period of `off` bytes in front of d
__device__ __forceinline__ void sx_copy_back(uint8_t* d, uint32_t off, uint64_t L) {
    const uint32_t lane = threadIdx.x & 31;
    if (off >= 32) {
        for (uint64_t k0 = 0; k0 < L; k0 += 32) {
            if (k0 + lane < L) d[k0 + lane] = d[k0 + lane - off];
            __syncwarp();
        }
    } else {
        for (uint64_t k = lane; k < L; k += 32) d[k] = (d - off)[k % off];
    }
}

// the block body s[0, len) into d[0, n), by the whole warp; false when it is corrupt
__device__ bool sx_decode_warp(const uint8_t* s, uint64_t len, uint8_t* d, uint64_t n) {
    const uint32_t lane = threadIdx.x & 31;
    uint64_t at = 0, x, o = 0;
    if (!dz_uvarint(s, len, at, x) || x != n) return false;
    uint32_t last = 0;
    while (at < len) {
        const uint32_t tag = s[at];
        uint64_t L;
        uint32_t off;
        if ((tag & 3) == 0) {
            x = tag >> 2;
            at++;
            if (x >= 60) {
                const uint32_t nb = (uint32_t)x - 59;
                if (nb > len - at) return false;
                x = 0;
                for (uint32_t k = 0; k < nb; k++) x |= (uint64_t)s[at + k] << (8 * k);
                at += nb;
            }
            L = x + 1;
            if (L > len - at || L > n - o) return false;
            for (uint64_t k = lane; k < L; k += 32) d[o + k] = s[at + k];
            __syncwarp();
            at += L;
            o += L;
            continue;
        }
        if ((tag & 3) == 1) {
            if (len - at < 2) return false;
            off = (tag >> 5) << 8 | s[at + 1];
            L = 4 + ((tag >> 2) & 7);
            at += 2;
            if (off == 0) {  // S2 repeat: the last offset again
                const uint32_t code = (tag >> 2) & 7;
                if (code >= 5) {
                    const uint32_t nb = code - 4;
                    if (nb > len - at) return false;
                    x = 0;
                    for (uint32_t k = 0; k < nb; k++) x |= (uint64_t)s[at + k] << (8 * k);
                    at += nb;
                    L = x + (code == 5 ? 8 : code == 6 ? 260 : 65540);
                }
                off = last;
            }
        } else if ((tag & 3) == 2) {
            if (len - at < 3) return false;
            off = (uint32_t)s[at + 1] | (uint32_t)s[at + 2] << 8;
            L = (tag >> 2) + 1;
            at += 3;
        } else {
            if (len - at < 5) return false;
            off = (uint32_t)s[at + 1] | (uint32_t)s[at + 2] << 8 | (uint32_t)s[at + 3] << 16 | (uint32_t)s[at + 4] << 24;
            L = (tag >> 2) + 1;
            at += 5;
        }
        if (off == 0 || off > o || L > n - o) return false;
        last = off;
        sx_copy_back(d + o, off, L);
        __syncwarp();
        o += L;
    }
    return o == n;
}

struct SxDecParams {
    const uint8_t* in;
    uint8_t* out;
    uint64_t base[4];  // each block's region in out
    const SxChunk* list;
    uint32_t nchunks;
    SxBack* back;
};

// KX2: listed chunk ci, decoded and checked
__global__ void __launch_bounds__(S2_WARPS * 32) sx_decode_kernel(const SxDecParams p) {
    __shared__ uint32_t crc_tab[256];
    sx_crc_table(crc_tab);
    __syncthreads();
    const uint32_t ci = blockIdx.x * S2_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (ci >= p.nchunks) return;
    const SxChunk k = p.list[ci];
    const uint8_t* s = p.in + k.src;
    uint8_t* d = p.out + p.base[k.block] + k.dst;
    bool ok = true;
    if (k.type == 1) {
        for (uint32_t j = lane; j < k.n; j += 32) d[j] = s[4 + j];
    } else {
        ok = sx_decode_warp(s + 4, k.len - 4, d, k.n);
    }
    __syncwarp();
    if (ok) ok = sx_crc_warp(d, k.n, crc_tab) == ((uint32_t)s[0] | (uint32_t)s[1] << 8 | (uint32_t)s[2] << 16 | (uint32_t)s[3] << 24);
    if (!ok && lane == 0) atomicOr(&p.back->bad, 1u);
}

}  // namespace sj
