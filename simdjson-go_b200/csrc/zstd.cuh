// zstd.cuh -- the zstd codec of the Serializer's CompressDefault / CompressBest blocks (block type 2,
// parsed_serialize.go:93-115 / :741-751) on the device, RFC 8878 without dictionaries.
//
// A zstd block of the stream is zero or more frames back to back (zstd or skippable).  A frame's blocks chain their
// window, their repeat offsets and their entropy tables, so no block stands alone; the decoder splits the work so that
// every step is parallel across blocks and only cheap scans run in frame order:
//   KX1 zx_list     one thread walks the frame and block headers of every zstd block of the stream (the S2 blocks'
//                   chunks are listed by the other threads, sx_walk) and lists frames and blocks
//   KZ2 zx_head     one thread per compressed block: literals header, Huffman description, sequences header and FSE
//                   descriptions are located and checked; which of the four tables the block defines
//   KZ3 zx_scan     one CTA: exclusive sums of literals and sequences (scratch offsets), and for each block the last
//                   block at or before it that defines each table (a max scan; it must lie in the block's frame)
//   KZ4 zx_entropy  one warp per compressed block: its tables built in shared memory from the defining blocks'
//                   descriptions, four lanes on four Huffman streams, one lane on the three-state sequence decode;
//                   literals and (ll, ml, offset_value) into scratch, the decoded size, and the block's effect on the
//                   repeat offsets as a function of the state it starts with
//   KZ3 zx_scan     again: output positions (sums of decoded sizes) and each block's starting repeat offsets (a scan of
//                   the composed functions, restarted at every frame); frame and block sizes checked
//   KZ5 zx_exec     one warp per block: literal bytes (raw and RLE blocks too) written, each match byte given its
//                   source byte's position; offsets made concrete and checked against the frame's start
//   KZ6 zx_jump     pointer jumping over the per-byte sources until every byte points at a written byte (at most
//                   log2 of the longest chain rounds, each a pass over the zstd output)
//   KZ7 zx_gather   every match byte copied from its source
//   KZ8 zx_xxh      XXH64 of each frame that carries a checksum, one warp per frame
// Encoder (Serialize): KZ1 zx_encode, one warp per ZX_CHUNK bytes of a zstd input, with KC1's match finder
// (sx_match_warp); raw literals, the predefined LL / OF / ML tables, new offsets only; a raw block when that is not
// shorter.  One frame per input, single segment with its content size, no checksum; KC2 gathers the blocks.
#pragma once
#include "s2.cuh"

namespace sj {

constexpr uint32_t ZX_BLOCK_MAX = 128u << 10;  // a zstd block's content and decoded size at most
constexpr uint32_t ZX_CHUNK = S2_CHUNK;         // input bytes per block KZ1 writes (KC1's match finder: uint16 positions)
constexpr uint32_t ZX_SEQ_CAP = ZX_CHUNK / 4 + 1;  // sequences of one KZ1 block (matches are at least 4 bytes)
constexpr uint32_t ZX_MAGIC = 0xFD2FB528u;
constexpr int ZX_WARPS = 4;                     // warps per CTA of KZ4 / KZ5 / KZ1
constexpr int ZX_SCAN = 256;                    // threads of KZ3
constexpr int ZX_LL_MAX = 35, ZX_ML_MAX = 52, ZX_OF_MAX = 31;
constexpr int ZX_LL_LOG = 9, ZX_ML_LOG = 9, ZX_OF_LOG = 8;
constexpr int64_t ZX_NEG = -(1ll << 60);

__constant__ int16_t zx_ll_default[36] = {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2,
                                          2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1};
__constant__ int16_t zx_ml_default[53] = {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                          1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1};
__constant__ int16_t zx_of_default[29] = {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1};
__constant__ uint32_t zx_ll_base[36] = {0,  1,  2,  3,  4,  5,  6,   7,   8,   9,   10,   11,   12,   13,   14,    15,    16,    18,
                                        20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536};
__constant__ uint8_t zx_ll_bits[36] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1,
                                       1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
__constant__ uint32_t zx_ml_base[53] = {3,  4,  5,  6,  7,  8,  9,  10,  11,  12,  13,  14,   15,   16,   17,   18,   19,    20,
                                        21, 22, 23, 24, 25, 26, 27, 28,  29,  30,  31,  32,   33,   34,   35,   37,   39,    41,
                                        43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539};
__constant__ uint8_t zx_ml_bits[53] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                       0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};

// ---------------------------------------------------------------------------------
// bits
// ---------------------------------------------------------------------------------
// n <= 57 bits of s[0, len) from bit `pos` on, zeros past the end
__device__ __forceinline__ uint64_t zx_peek(const uint8_t* s, uint64_t len, uint64_t pos, uint32_t n) {
    const uint64_t b = pos >> 3;
    uint64_t v = 0;
    for (uint32_t k = 0; k < 8 && b + k < len; k++) v |= (uint64_t)s[b + k] << (8 * k);
    v >>= pos & 7;
    return n >= 64 ? v : v & ((1ull << n) - 1);
}

// a bitstream read backwards from the padding bit of its last byte; `left` goes negative when it is read past its start
// (then zeros are read, and the stream cannot end exactly)
struct ZxBack {
    const uint8_t* s;
    uint64_t len;
    int64_t left;
    __device__ bool init(const uint8_t* p, uint64_t n) {
        s = p;
        len = n;
        if (n == 0 || p[n - 1] == 0) return false;
        left = 8 * (int64_t)n - (__clz((uint32_t)p[n - 1]) - 24) - 1;
        return true;
    }
    __device__ __forceinline__ uint32_t read(uint32_t n) {
        if (n == 0) return 0;
        left -= n;
        if (left >= 0) return (uint32_t)zx_peek(s, (uint64_t)(left + n + 7) >> 3, (uint64_t)left, n);
        if (left <= -(int64_t)n) return 0;
        const uint32_t have = (uint32_t)(left + n);
        return (uint32_t)(zx_peek(s, len, 0, have) << (n - have));
    }
};

// ---------------------------------------------------------------------------------
// FSE and Huffman tables
// ---------------------------------------------------------------------------------
struct ZxFse {
    uint16_t base;
    uint8_t sym, nb;
};

// the decoding table of normalized counts cnt[0, nsym) at accuracy log al (one thread); false when the spread does not
// come back to state 0
__device__ bool zx_fse_build(const int16_t* cnt, int nsym, int al, ZxFse* tab, uint16_t* nxt) {
    const uint32_t size = 1u << al;
    int high = (int)size - 1;
    for (int s = 0; s < nsym; s++) {
        if (cnt[s] == -1) {
            tab[high--].sym = (uint8_t)s;
            nxt[s] = 1;
        } else {
            nxt[s] = (uint16_t)max((int)cnt[s], 0);
        }
    }
    const uint32_t step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
    uint32_t pos = 0;
    for (int s = 0; s < nsym; s++)
        for (int i = 0; i < cnt[s]; i++) {
            tab[pos].sym = (uint8_t)s;
            do pos = (pos + step) & mask;
            while ((int)pos > high);
        }
    if (pos != 0) return false;
    for (uint32_t u = 0; u < size; u++) {
        const uint32_t x = nxt[tab[u].sym]++;
        const uint32_t nb = al - (31 - __clz(x));
        tab[u].nb = (uint8_t)nb;
        tab[u].base = (uint16_t)((x << nb) - size);
    }
    return true;
}

// an FSE table description at s[0, len): counts (nsym of them, max_sym + 1 at most), al, bytes; false when invalid
__device__ bool zx_ncount(const uint8_t* s, uint64_t len, int max_sym, int max_log, int16_t* cnt, int& nsym, int& al,
                          uint32_t& used) {
    if (len == 0) return false;
    uint64_t pos = 4;
    al = (s[0] & 15) + 5;
    if (al > max_log) return false;
    int remaining = (1 << al) + 1, threshold = 1 << al, nb = al + 1, n = 0;
    bool prev0 = false;
    while (remaining > 1 && n <= max_sym) {
        if (prev0) {
            uint32_t r;
            do {
                r = (uint32_t)zx_peek(s, len, pos, 2);
                pos += 2;
                if (n + (int)r > max_sym + 1) return false;
                for (uint32_t k = 0; k < r; k++) cnt[n++] = 0;
            } while (r == 3);
            if (n > max_sym) break;
        }
        const int mx = (2 * threshold - 1) - remaining;
        int v = (int)zx_peek(s, len, pos, nb);
        if ((v & (threshold - 1)) < mx) {
            v &= threshold - 1;
            pos += nb - 1;
        } else {
            if (v >= threshold) v -= mx;
            pos += nb;
        }
        const int c = v - 1;
        remaining -= c < 0 ? -c : c;
        cnt[n++] = (int16_t)c;
        prev0 = c == 0;
        while (remaining < threshold) {
            nb--;
            threshold >>= 1;
        }
    }
    if (remaining != 1) return false;
    used = (uint32_t)((pos + 7) >> 3);
    if (used > len) return false;
    nsym = n;
    return true;
}

struct ZxHufScratch {
    int16_t cnt[256];
    uint16_t nxt[256];
    ZxFse wtab[64];
    uint8_t w[256];
};

// a Huffman tree description at s[0, len) into the weights w (the last one implied) of nw symbols: its bytes, 0 when
// invalid (one thread)
__device__ uint32_t zx_huf_weights(const uint8_t* s, uint64_t len, ZxHufScratch& h, uint32_t& nw, uint32_t& maxbits) {
    if (len == 0) return 0;
    const uint32_t hb = s[0];
    uint32_t size, n = 0;
    if (hb < 128) {
        if (hb == 0 || 1 + (uint64_t)hb > len) return 0;
        int nsym, al;
        uint32_t used;
        if (!zx_ncount(s + 1, hb, 255, 6, h.cnt, nsym, al, used)) return 0;
        if (!zx_fse_build(h.cnt, nsym, al, h.wtab, h.nxt)) return 0;
        ZxBack br;
        if (!br.init(s + 1 + used, hb - used)) return 0;
        uint32_t s1 = br.read(al), s2 = br.read(al);
        for (;;) {
            if (n >= 255) return 0;
            h.w[n++] = h.wtab[s1].sym;
            s1 = h.wtab[s1].base + br.read(h.wtab[s1].nb);
            if (br.left < 0) {
                if (n >= 255) return 0;
                h.w[n++] = h.wtab[s2].sym;
                break;
            }
            if (n >= 255) return 0;
            h.w[n++] = h.wtab[s2].sym;
            s2 = h.wtab[s2].base + br.read(h.wtab[s2].nb);
            if (br.left < 0) {
                if (n >= 255) return 0;
                h.w[n++] = h.wtab[s1].sym;
                break;
            }
        }
        size = 1 + hb;
    } else {
        n = hb - 127;
        size = 1 + (n + 1) / 2;
        if (size > len) return 0;
        for (uint32_t k = 0; k < n; k++) {
            const uint8_t b = s[1 + k / 2];
            h.w[k] = (k & 1) ? (b & 15) : (b >> 4);
        }
    }
    uint32_t total = 0;
    for (uint32_t k = 0; k < n; k++) {
        if (h.w[k] > 11) return 0;
        if (h.w[k]) total += 1u << (h.w[k] - 1);
    }
    if (total == 0) return 0;
    maxbits = 32 - __clz(total);
    const uint32_t left = (1u << maxbits) - total;
    if (maxbits > 11 || (left & (left - 1)) != 0) return 0;
    h.w[n++] = (uint8_t)(32 - __clz(left));
    nw = n;
    return size;
}

// ---------------------------------------------------------------------------------
// the decoder's lists
// ---------------------------------------------------------------------------------
struct ZxFrame {
    uint64_t fcs;       // content size, when has_fcs
    uint32_t first, nblocks;  // its blocks in the block list
    uint32_t sblock;    // the stream block (0 .. 3) it is in
    uint32_t has_fcs, checksum, cks;  // content size present; checksum present and its value
};

// RepFn: the repeat offsets behind a run of sequences as a function of those in front of it, x; slot k is the constant
// d (src 3) or max(x[src] + d, f)
struct ZxRep {
    int64_t d[3], f[3];
    int32_t src[3];
    int32_t start;  // (KZ3) the block starts a frame
};

__device__ __forceinline__ ZxRep zx_rep_identity() {
    ZxRep r;
    for (int k = 0; k < 3; k++) {
        r.src[k] = k;
        r.d[k] = 0;
        r.f[k] = ZX_NEG;
    }
    r.start = 0;
    return r;
}

// g after f
__device__ __forceinline__ ZxRep zx_rep_compose(const ZxRep& f, const ZxRep& g) {
    ZxRep r;
    for (int k = 0; k < 3; k++) {
        if (g.src[k] == 3) {
            r.src[k] = 3;
            r.d[k] = g.d[k];
            r.f[k] = ZX_NEG;
            continue;
        }
        const int j = g.src[k];
        if (f.src[j] == 3) {
            r.src[k] = 3;
            r.d[k] = max(f.d[j] + g.d[k], g.f[k]);
            r.f[k] = ZX_NEG;
        } else {
            r.src[k] = f.src[j];
            r.d[k] = f.d[j] + g.d[k];
            r.f[k] = max(f.f[j] + g.d[k], g.f[k]);
        }
    }
    r.start = f.start | g.start;
    return r;
}

__device__ __forceinline__ int64_t zx_rep_slot(const ZxRep& r, int k, const int64_t* x) {
    return r.src[k] == 3 ? r.d[k] : max(x[r.src[k]] + r.d[k], r.f[k]);
}

enum : uint32_t { ZX_DEF_HUF = 1, ZX_DEF_LL = 2, ZX_DEF_OF = 4, ZX_DEF_ML = 8 };

struct ZxBlk {
    uint64_t src;         // its content in the input
    uint64_t out;         // (KZ3) its decoded bytes in the output
    uint64_t lit_off, seq_off;  // (KZ3) its literals and sequences in scratch
    uint32_t csize, n;    // content bytes; decoded bytes (raw / RLE: KX1, compressed: KZ4)
    uint32_t frame, type, limit;
    // KZ2: offsets into the content
    uint32_t lit_type, lit_n, lit_at, lit_end, nstreams;
    uint32_t nseq, modes, desc_at[3], seq_at, defines;
    int32_t huf_src, tab_src[3];  // (KZ3) the block whose description each table comes from
    int64_t rep[3];               // (KZ3) the repeat offsets in front of the block
    ZxRep fn;                     // (KZ4) its effect on them
};

// the zstd part of KX1's read-back
struct ZxCount {
    uint32_t blocks, frames;   // listed (only the first `cap` of each are stored)
    uint32_t first[4];         // each stream block's first listed block
    uint64_t lits, seqs;       // (KZ3) literal bytes and sequences of all compressed blocks
};

// KX1's read-back: the S2 part and the zstd part
struct XxBack {
    SxBack s;
    ZxCount z;
};

struct ZxList {
    ZxBlk* blk;
    ZxFrame* frm;
    uint32_t blk_cap, frm_cap;
    ZxCount* cnt;
};

// the frames of stream block i (zstd, one thread) into the lists; false on a framing rule
__device__ bool zx_walk(const uint8_t* s, const SxBlock& b, uint32_t i, ZxList L) {
    uint64_t p = b.at, produced = 0, most = 0;  // raw and RLE bytes; and what all blocks could decode to
    const uint64_t end = b.at + b.size;
    while (p < end) {
        if (end - p < 4) return false;
        const uint32_t magic = sx_load32(s + p);
        if ((magic & 0xfffffff0u) == 0x184D2A50u) {  // skippable
            if (end - p < 8) return false;
            const uint64_t n = sx_load32(s + p + 4);
            if (n > end - p - 8) return false;
            p += 8 + n;
            continue;
        }
        if (magic != ZX_MAGIC) return false;
        p += 4;
        if (p >= end) return false;
        const uint32_t fhd = s[p++];
        const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, cks = (fhd >> 2) & 1, did = fhd & 3;
        if (fhd & 8) return false;
        uint64_t window = 0;
        if (!single) {
            if (p >= end) return false;
            const uint32_t wd = s[p++];
            const uint64_t base = 1ull << (10 + (wd >> 3));
            window = base + (base >> 3) * (wd & 7);
        }
        const uint32_t dn = did == 3 ? 4 : did;
        if (end - p < dn) return false;
        for (uint32_t k = 0; k < dn; k++)
            if (s[p + k]) return false;  // no dictionaries
        p += dn;
        const uint32_t fn = fcs_flag == 0 ? single : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
        if (end - p < fn) return false;
        uint64_t fcs = 0;
        for (uint32_t k = 0; k < fn; k++) fcs |= (uint64_t)s[p + k] << (8 * k);
        if (fn == 2) fcs += 256;
        p += fn;
        if (single) window = fcs;
        const uint32_t limit = (uint32_t)min(window, (uint64_t)ZX_BLOCK_MAX);
        const uint32_t f = L.cnt->frames++;
        const uint32_t first = L.cnt->blocks;
        uint64_t known = 0;  // raw and RLE bytes of the frame
        for (;;) {
            if (end - p < 3) return false;
            const uint32_t bh = (uint32_t)s[p] | (uint32_t)s[p + 1] << 8 | (uint32_t)s[p + 2] << 16;
            p += 3;
            const uint32_t last = bh & 1, bt = (bh >> 1) & 3, bs = bh >> 3;
            if (bt == 3 || (bt == 2 && bs > limit)) return false;  // (raw and RLE blocks are not limited, as in libzstd)
            const uint64_t cs = bt == 1 ? 1 : bs;
            if (end - p < cs) return false;
            const uint32_t k = L.cnt->blocks++;
            if (k < L.blk_cap) {
                ZxBlk& x = L.blk[k];
                x.src = p;
                x.csize = (uint32_t)cs;
                x.n = bt == 2 ? 0 : bs;
                x.frame = f;
                x.type = bt;
                x.limit = limit;
                x.defines = 0;
                x.lit_n = x.nseq = 0;
            }
            if (bt != 2) known += bs;
            most += bt == 2 ? limit : bs;
            p += cs;
            if (last) break;
        }
        uint32_t ck = 0;
        if (cks) {
            if (end - p < 4) return false;
            ck = sx_load32(s + p);
            p += 4;
        }
        if (f < L.frm_cap) L.frm[f] = ZxFrame{fcs, first, L.cnt->blocks - first, i, fn != 0, cks, ck};
        if (fn && known > fcs) return false;
        produced += known;
    }
    // (the block's size then bounds the inflated region and the decoder's scratch)
    return produced <= b.raw && b.raw <= most;
}

// KX1: the blocks (from the header, or the one block `one`); thread i < 4 walks S2 block i's chunks, thread 4 every
// zstd block's frames in stream order (so a frame's blocks are listed together)
__global__ void zx_list_kernel(const uint8_t* s, uint64_t len, SxBlock one, bool from_header, SxChunk* list, uint32_t cap,
                               SxBack* back, ZxList zl) {
    __shared__ SxBlock b[4];
    if (threadIdx.x == 0) {
        if (from_header) {
            sx_header_blocks(s, len, b);
        } else {
            b[0] = one;
            for (int i = 1; i < 4; i++) b[i] = SxBlock{0, 0, 0, S2_NONE, 0};
        }
    }
    __syncthreads();
    const uint32_t i = threadIdx.x;
    if (i < 4) {
        back->type[i] = b[i].type;
        back->total[i] = 0;
        if (b[i].type == 1 && !sx_walk(s, b[i], i, list, cap, back)) atomicOr(&back->bad, 1u);
    } else if (i == 4 && zl.cnt) {
        for (int k = 0; k < 4; k++) {
            zl.cnt->first[k] = zl.cnt->blocks;
            if (b[k].type == 2 && !zx_walk(s, b[k], k, zl)) {
                atomicOr(&back->bad, 1u);
                return;
            }
        }
    }
}

// ---------------------------------------------------------------------------------
// KZ2: the sections of each compressed block
// ---------------------------------------------------------------------------------
__device__ bool zx_head(const uint8_t* in, ZxBlk& x) {
    const uint8_t* s = in + x.src;
    const uint32_t end = x.csize;
    uint32_t at = 0;
    if (at >= end) return false;
    const uint32_t b0 = s[0], t = b0 & 3, sf = (b0 >> 2) & 3;
    x.lit_type = t;
    x.nstreams = 1;
    if (t <= 1) {
        uint32_t n, hl;
        if ((sf & 1) == 0) {
            n = b0 >> 3;
            hl = 1;
        } else if (sf == 1) {
            if (end < 2) return false;
            n = (b0 >> 4) | (uint32_t)s[1] << 4;
            hl = 2;
        } else {
            if (end < 3) return false;
            n = (b0 >> 4) | (uint32_t)s[1] << 4 | (uint32_t)s[2] << 12;
            hl = 3;
        }
        if (n > ZX_BLOCK_MAX) return false;
        x.lit_n = n;
        x.lit_at = hl;
        x.lit_end = hl + (t == 0 ? n : 1);
        if (x.lit_end > end) return false;
    } else {
        const uint32_t hl = sf <= 1 ? 3 : sf + 2;
        if (end < hl) return false;
        uint64_t h = 0;
        for (uint32_t k = 0; k < hl; k++) h |= (uint64_t)s[k] << (8 * k);
        const uint32_t sb = sf <= 1 ? 10 : sf == 2 ? 14 : 18;
        const uint32_t n = (uint32_t)((h >> 4) & ((1u << sb) - 1)), cs = (uint32_t)((h >> (4 + sb)) & ((1u << sb) - 1));
        if (n > ZX_BLOCK_MAX) return false;
        x.nstreams = sf == 0 ? 1 : 4;
        x.lit_n = n;
        x.lit_at = hl;
        x.lit_end = hl + cs;
        if (x.lit_end > end) return false;
        if (t == 2) x.defines |= ZX_DEF_HUF;
    }
    at = x.lit_end;
    // sequences
    if (at >= end) return false;
    const uint32_t c0 = s[at];
    if (c0 == 0) {
        x.nseq = 0;
        return at + 1 == end;
    }
    if (c0 < 128) {
        x.nseq = c0;
        at += 1;
    } else if (c0 < 255) {
        if (end - at < 2) return false;
        x.nseq = ((c0 - 128) << 8) + s[at + 1];
        at += 2;
    } else {
        if (end - at < 3) return false;
        x.nseq = s[at + 1] + ((uint32_t)s[at + 2] << 8) + 0x7F00;
        at += 3;
    }
    if (at >= end) return false;
    x.modes = s[at++];
    if (x.modes & 3) return false;
    const int maxs[3] = {ZX_LL_MAX, ZX_OF_MAX, ZX_ML_MAX}, logs[3] = {ZX_LL_LOG, ZX_OF_LOG, ZX_ML_LOG};
    for (int k = 0; k < 3; k++) {
        const uint32_t m = (x.modes >> (6 - 2 * k)) & 3;
        x.desc_at[k] = at;
        if (m != 3) x.defines |= ZX_DEF_LL << k;
        if (m == 1) {
            if (at >= end || s[at] > (uint32_t)maxs[k]) return false;
            at++;
        } else if (m == 2) {
            int16_t cnt[64];
            int nsym, al;
            uint32_t used;
            if (!zx_ncount(s + at, end - at, maxs[k], logs[k], cnt, nsym, al, used)) return false;
            at += used;
        }
    }
    x.seq_at = at;
    return at < end;
}

struct ZxParams {
    const uint8_t* in;
    uint8_t* out;
    ZxBlk* blk;
    const ZxFrame* frm;
    ZxCount* cnt;
    uint32_t nblk, nfrm;
    uint8_t* lits;
    uint32_t* seqs;       // (ll, ml, offset_value) per sequence
    uint32_t* srcidx;     // per output byte: the position its byte comes from (itself when written)
    uint64_t base[4], raw[4];  // each stream block's region in out and its uncompressed size
    uint32_t ztype[4];    // the stream block is zstd
    unsigned long long* changed;
    uint32_t* bad;
};

__global__ void zx_head_kernel(const ZxParams p) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= p.nblk) return;
    ZxBlk x = p.blk[b];
    if (x.type != 2) return;
    bool ok = zx_head(p.in, x);
    // every sequence has a match of 3 or more bytes, so a block decodes to at least lit_n + 3 nseq
    ok = ok && (uint64_t)x.lit_n + 3ull * x.nseq <= x.limit;
    if (!ok) atomicOr(p.bad, 1u);
    p.blk[b] = x;
}

// ---------------------------------------------------------------------------------
// KZ3: the scans (one CTA of ZX_SCAN threads, chunks of ZX_SCAN blocks in order)
// ---------------------------------------------------------------------------------
template <class T, class Op>
__device__ T zx_cta_scan(T v, T* sh, Op op) {  // inclusive
    const uint32_t t = threadIdx.x;
    sh[t] = v;
    __syncthreads();
    for (uint32_t d = 1; d < ZX_SCAN; d <<= 1) {
        T x = v;
        if (t >= d) x = op(sh[t - d], v);
        __syncthreads();
        sh[t] = x;
        v = x;
        __syncthreads();
    }
    return v;
}

struct ZxS1 {
    uint64_t lits, seqs, need;  // need: the fewest bytes the blocks can decode to
    int32_t src[4];
};
struct ZxS1Op {
    __device__ ZxS1 operator()(const ZxS1& a, const ZxS1& b) const {
        ZxS1 r{a.lits + b.lits, a.seqs + b.seqs, a.need + b.need, {}};
        for (int k = 0; k < 4; k++) r.src[k] = max(a.src[k], b.src[k]);
        return r;
    }
};
struct ZxS2 {
    uint64_t n;
    ZxRep fn;
};
struct ZxS2Op {
    __device__ ZxS2 operator()(const ZxS2& a, const ZxS2& b) const {
        return ZxS2{a.n + b.n, b.fn.start ? b.fn : zx_rep_compose(a.fn, b.fn)};
    }
};

// (KZ3 phase 2, before the rebase) where block b's output starts, in the order of all listed blocks
__device__ __forceinline__ uint64_t zx_pos(const ZxParams& p, uint32_t b) {
    return b < p.nblk ? p.blk[b].out : p.nblk ? p.blk[p.nblk - 1].out + p.blk[p.nblk - 1].n : 0;
}

// phase 1: scratch offsets and table sources; phase 2: output positions, repeat offsets and the size checks
__global__ void __launch_bounds__(ZX_SCAN) zx_scan_kernel(const ZxParams p, int phase) {
    __shared__ ZxS1 sh1[ZX_SCAN];
    __shared__ ZxS2 sh2[ZX_SCAN];
    __shared__ ZxS1 c1;
    __shared__ ZxS2 c2;
    const uint32_t t = threadIdx.x;
    if (t == 0) {
        c1 = ZxS1{0, 0, 0, {-1, -1, -1, -1}};
        c2 = ZxS2{0, zx_rep_identity()};
    }
    __syncthreads();
    for (uint32_t b0 = 0; b0 < p.nblk; b0 += ZX_SCAN) {
        const uint32_t b = b0 + t;
        const bool in = b < p.nblk;
        ZxBlk* x = in ? &p.blk[b] : nullptr;
        if (phase == 1) {
            ZxS1 v{0, 0, 0, {-1, -1, -1, -1}};
            if (in) v.need = x->n;  // raw and RLE blocks; 0 for compressed ones until KZ4
            if (in && x->type == 2) {
                v.lits = x->lit_n;
                v.seqs = x->nseq;
                v.need = x->lit_n + 3ull * x->nseq;
                for (int k = 0; k < 4; k++)
                    if (x->defines & (1u << k)) v.src[k] = (int32_t)b;
            }
            ZxS1 r = ZxS1Op()(c1, zx_cta_scan(v, sh1, ZxS1Op()));
            if (in) {
                x->lit_off = r.lits - v.lits;
                x->seq_off = r.seqs - v.seqs;
                x->out = r.need - v.need;  // (phase 2 overwrites it with the block's position)
                const int32_t first = (int32_t)p.frm[x->frame].first;
                x->huf_src = r.src[0] >= first ? r.src[0] : -1;
                for (int k = 0; k < 3; k++) x->tab_src[k] = r.src[k + 1] >= first ? r.src[k + 1] : -1;
                if (x->type == 2) {
                    const bool treeless = x->lit_type == 3;
                    bool ok = !treeless || x->huf_src >= 0;
                    for (int k = 0; k < 3; k++) ok = ok && (x->nseq == 0 || x->tab_src[k] >= 0);
                    if (!ok) atomicOr(p.bad, 1u);
                }
            }
            __syncthreads();
            if (t == ZX_SCAN - 1) c1 = r;
        } else {
            ZxS2 v{0, zx_rep_identity()};
            if (in) {
                v.n = x->n;
                if (x->type == 2) v.fn = x->fn;
                v.fn.start = p.frm[x->frame].first == b;
            }
            ZxS2 r = ZxS2Op()(c2, zx_cta_scan(v, sh2, ZxS2Op()));
            if (in) {
                const uint64_t pos = r.n - v.n;  // exclusive: decoded bytes of all earlier blocks
                x->out = pos;
                x->fn = r.fn;  // inclusive, for the next block (below)
            }
            __syncthreads();
            if (t == ZX_SCAN - 1) c2 = r;
        }
        __syncthreads();
    }
    if (t == 0) {
        if (phase == 1) {
            p.cnt->lits = c1.lits;
            p.cnt->seqs = c1.seqs;
        }
    }
    if (phase == 1) {
        // every stream block's blocks must be able to decode to no more than its size before the scratch (literals,
        // sequences, per-byte sources) is sized from them
        __syncthreads();
        if (t < 4 && p.ztype[t]) {
            const uint32_t b0 = p.cnt->first[t], b1 = t < 3 ? p.cnt->first[t + 1] : p.nblk;
            const uint64_t a = b0 < p.nblk ? p.blk[b0].out : c1.need, e = b1 < p.nblk ? p.blk[b1].out : c1.need;
            if (e - a > p.raw[t]) atomicOr(p.bad, 1u);
        }
        return;
    }
    __syncthreads();
    // each block's starting repeat offsets: those behind the previous block of its frame; positions relative to the
    // stream block's first zstd block; frame content sizes and stream block totals.  (Every block reads its inclusive
    // function's predecessor before any is overwritten: the reads go to rep[], a separate field.)
    const int64_t init[3] = {1, 4, 8};
    for (uint32_t b = t; b < p.nblk; b += ZX_SCAN) {
        ZxBlk& x = p.blk[b];
        const ZxFrame& f = p.frm[x.frame];
        for (int k = 0; k < 3; k++) x.rep[k] = b == f.first ? init[k] : zx_rep_slot(p.blk[b - 1].fn, k, init);
    }
    __syncthreads();
    for (uint32_t fi = t; fi < p.nfrm; fi += ZX_SCAN) {
        const ZxFrame& f = p.frm[fi];
        if (f.has_fcs && zx_pos(p, f.first + f.nblocks) - zx_pos(p, f.first) != f.fcs) atomicOr(p.bad, 1u);
    }
    for (uint32_t i = t; i < 4; i += ZX_SCAN) {
        if (!p.ztype[i]) continue;
        const uint32_t b0 = p.cnt->first[i], b1 = i < 3 ? p.cnt->first[i + 1] : p.nblk;
        if (zx_pos(p, b1) - zx_pos(p, b0) != p.raw[i]) atomicOr(p.bad, 1u);
    }
    __shared__ uint64_t start[4];  // (read before any block's position is rebased)
    if (t < 4) start[t] = zx_pos(p, p.cnt->first[t]);
    __syncthreads();
    for (uint32_t b = t; b < p.nblk; b += ZX_SCAN) {
        ZxBlk& x = p.blk[b];
        const uint32_t sb = p.frm[x.frame].sblock;
        x.out = p.base[sb] + (x.out - start[sb]);
    }
}

// ---------------------------------------------------------------------------------
// KZ4: entropy decoding, one warp per compressed block
// ---------------------------------------------------------------------------------
struct ZxWarpSmem {
    uint16_t huf[1 << 11];  // symbol | nbits << 8, per 11-bit prefix (maxbits bits used)
    ZxFse ll[1 << ZX_LL_LOG], of[1 << ZX_OF_LOG], ml[1 << ZX_ML_LOG];
    ZxHufScratch hs;
    uint32_t maxbits, nw, hlen, logs[3];
    uint32_t ok;
};

// table k of block x (LL, OF, ML) from its source block's description (one thread)
__device__ bool zx_seq_table(const uint8_t* in, const ZxBlk* blk, const ZxBlk& x, int k, ZxFse* tab, uint32_t& al,
                             ZxHufScratch& h) {
    const ZxBlk& d = blk[x.tab_src[k]];
    const uint32_t m = (d.modes >> (6 - 2 * k)) & 3;
    const int maxs[3] = {ZX_LL_MAX, ZX_OF_MAX, ZX_ML_MAX}, logs[3] = {ZX_LL_LOG, ZX_OF_LOG, ZX_ML_LOG};
    if (m == 0) {
        const int16_t* c = k == 0 ? zx_ll_default : k == 1 ? zx_of_default : zx_ml_default;
        const int n = k == 0 ? 36 : k == 1 ? 29 : 53;
        for (int i = 0; i < n; i++) h.cnt[i] = c[i];
        al = k == 1 ? 5 : 6;
        return zx_fse_build(h.cnt, n, (int)al, tab, h.nxt);
    }
    const uint8_t* s = in + d.src;
    if (m == 1) {
        tab[0] = ZxFse{0, s[d.desc_at[k]], 0};
        al = 0;
        return true;
    }
    int nsym, a;
    uint32_t used;
    if (!zx_ncount(s + d.desc_at[k], d.csize - d.desc_at[k], maxs[k], logs[k], h.cnt, nsym, a, used)) return false;
    al = (uint32_t)a;
    return zx_fse_build(h.cnt, nsym, a, tab, h.nxt);
}

// one Huffman stream of n symbols (one lane); false unless it ends exactly at its padding
__device__ bool zx_huf_stream(const uint8_t* s, uint32_t len, const uint16_t* tab, uint32_t maxbits, uint8_t* d, uint32_t n) {
    ZxBack br;
    if (!br.init(s, len)) return false;
    for (uint32_t i = 0; i < n; i++) {
        const int64_t saved = br.left;
        const uint16_t e = tab[br.read(maxbits)];
        br.left = saved - (e >> 8);
        d[i] = (uint8_t)e;
    }
    return br.left == 0;
}

__global__ void __launch_bounds__(ZX_WARPS * 32) zx_entropy_kernel(const ZxParams p) {
    __shared__ ZxWarpSmem sm_all[ZX_WARPS];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    ZxWarpSmem& sm = sm_all[warp];
    const uint32_t b = blockIdx.x * ZX_WARPS + warp;
    if (b >= p.nblk) return;
    ZxBlk& x = p.blk[b];
    if (x.type != 2) return;
    const uint8_t* s = p.in + x.src;
    uint8_t* lit = p.lits + x.lit_off;
    // tables
    if (lane == 0) {
        bool ok = true;
        if (x.lit_type >= 2) {
            const ZxBlk& d = p.blk[x.huf_src];
            sm.hlen = zx_huf_weights(p.in + d.src + d.lit_at, d.lit_end - d.lit_at, sm.hs, sm.nw, sm.maxbits);
            ok = sm.hlen != 0;
        }
        if (ok && x.nseq) {
            ok = zx_seq_table(p.in, p.blk, x, 0, sm.ll, sm.logs[0], sm.hs) && zx_seq_table(p.in, p.blk, x, 1, sm.of, sm.logs[1], sm.hs) &&
                 zx_seq_table(p.in, p.blk, x, 2, sm.ml, sm.logs[2], sm.hs);
        }
        sm.ok = ok;
    }
    __syncwarp();
    if (!sm.ok) {
        if (lane == 0) atomicOr(p.bad, 1u);
        return;
    }
    // literals
    bool ok = true;
    if (x.lit_type == 0) {
        for (uint32_t k = lane; k < x.lit_n; k += 32) lit[k] = s[x.lit_at + k];
    } else if (x.lit_type == 1) {
        const uint8_t v = s[x.lit_at];
        for (uint32_t k = lane; k < x.lit_n; k += 32) lit[k] = v;
    } else {
        // the Huffman table: weight-1 symbols first, each weight's symbols in order, 2^(w-1) entries each.  The weights
        // were read into sm.hs.w (the ones of this block, or of the block whose table a treeless block reuses: they
        // were just re-read from that block's description)
        const uint32_t nw = sm.nw, mb = sm.maxbits;
        if (lane == 0) {
            uint32_t start[13], pos = 0;
            for (uint32_t w = 1; w <= mb; w++) {
                start[w] = pos;
                uint32_t c = 0;
                for (uint32_t k = 0; k < nw; k++) c += sm.hs.w[k] == w;
                pos += c << (w - 1);
            }
            for (uint32_t k = 0; k < nw; k++) {
                const uint32_t w = sm.hs.w[k];
                if (!w) continue;
                const uint16_t e = (uint16_t)(k | ((mb + 1 - w) << 8));
                for (uint32_t j = 0; j < (1u << (w - 1)); j++) sm.huf[start[w] + j] = e;
                start[w] += 1u << (w - 1);
            }
        }
        __syncwarp();
        const uint32_t h0 = x.lit_at + (x.lit_type == 2 ? sm.hlen : 0);
        const uint32_t body = x.lit_end - h0;
        if (x.nstreams == 1) {
            if (lane == 0) ok = zx_huf_stream(s + h0, body, sm.huf, mb, lit, x.lit_n);
        } else {
            uint32_t sz[4], at = h0 + 6;
            bool good = body >= 6;
            if (good) {
                sz[0] = s[h0] | (uint32_t)s[h0 + 1] << 8;
                sz[1] = s[h0 + 2] | (uint32_t)s[h0 + 3] << 8;
                sz[2] = s[h0 + 4] | (uint32_t)s[h0 + 5] << 8;
                const int64_t l4 = (int64_t)body - 6 - sz[0] - sz[1] - sz[2];
                good = l4 >= 0;
                sz[3] = (uint32_t)max(l4, (int64_t)0);
            }
            const uint32_t q = (x.lit_n + 3) / 4;
            good = good && x.lit_n >= 3 * q;
            if (good && lane < 4) {
                for (uint32_t k = 0; k < lane; k++) at += sz[k];
                const uint32_t nk = lane < 3 ? q : x.lit_n - 3 * q;
                ok = zx_huf_stream(s + at, sz[lane], sm.huf, mb, lit + lane * q, nk);
            }
            ok = ok && good;
        }
    }
    ok = __all_sync(FULL, ok);
    // sequences (lane 0)
    if (lane == 0 && ok) {
        uint32_t* q = p.seqs + 3 * x.seq_off;
        ZxRep fn = zx_rep_identity();
        uint64_t lsum = 0, msum = 0;
        if (x.nseq) {
            ZxBack br;
            ok = br.init(s + x.seq_at, x.csize - x.seq_at);
            if (ok) {
                uint32_t sl = br.read(sm.logs[0]), so = br.read(sm.logs[1]), smm = br.read(sm.logs[2]);
                for (uint32_t i = 0; i < x.nseq && ok; i++) {
                    const uint32_t oc = sm.of[so].sym, mc = sm.ml[smm].sym, lc = sm.ll[sl].sym;
                    if (oc > ZX_OF_MAX || mc > ZX_ML_MAX || lc > ZX_LL_MAX) {
                        ok = false;
                        break;
                    }
                    const uint32_t ofv = (1u << oc) + br.read(oc);
                    const uint32_t ml = zx_ml_base[mc] + br.read(zx_ml_bits[mc]);
                    const uint32_t ll = zx_ll_base[lc] + br.read(zx_ll_bits[lc]);
                    q[3 * i] = ll;
                    q[3 * i + 1] = ml;
                    q[3 * i + 2] = ofv;
                    lsum += ll;
                    msum += ml;
                    // the repeat offsets, symbolically
                    ZxRep g = zx_rep_identity();
                    if (ofv > 3) {
                        g.src[0] = 3;
                        g.d[0] = ofv - 3;
                        g.src[1] = 0;
                        g.src[2] = 1;
                    } else {
                        const uint32_t k = ofv - 1 + (ll == 0);
                        if (k == 1) {
                            g.src[0] = 1;
                            g.src[1] = 0;
                        } else if (k == 2) {
                            g.src[0] = 2;
                            g.src[1] = 0;
                            g.src[2] = 1;
                        } else if (k == 3) {  // rep1 - 1 (KZ5 rejects it when that is 0)
                            g.d[0] = -1;
                            g.src[1] = 0;
                            g.src[2] = 1;
                        }
                    }
                    fn = zx_rep_compose(fn, g);
                    if (i + 1 < x.nseq) {
                        sl = sm.ll[sl].base + br.read(sm.ll[sl].nb);
                        smm = sm.ml[smm].base + br.read(sm.ml[smm].nb);
                        so = sm.of[so].base + br.read(sm.of[so].nb);
                    }
                }
                ok = ok && br.left == 0;
            }
        }
        ok = ok && lsum <= x.lit_n && x.lit_n + msum <= x.limit;
        x.n = (uint32_t)(x.lit_n + msum);
        fn.start = 0;
        x.fn = fn;
    }
    if (!__all_sync(FULL, ok) && lane == 0) atomicOr(p.bad, 1u);
}

// ---------------------------------------------------------------------------------
// KZ5 .. KZ8: execution
// ---------------------------------------------------------------------------------
// KZ5: block b's literal bytes written and each of its match bytes pointed at its source; raw and RLE blocks written
__global__ void __launch_bounds__(ZX_WARPS * 32) zx_exec_kernel(const ZxParams p) {
    const uint32_t b = blockIdx.x * ZX_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= p.nblk) return;
    const ZxBlk& x = p.blk[b];
    const uint8_t* s = p.in + x.src;
    uint64_t o = x.out;
    if (x.type != 2) {
        for (uint32_t k = lane; k < x.n; k += 32) {
            p.out[o + k] = x.type == 0 ? s[k] : s[0];
            p.srcidx[o + k] = (uint32_t)(o + k);
        }
        return;
    }
    const uint64_t fs = p.blk[p.frm[x.frame].first].out;
    const uint8_t* lit = p.lits + x.lit_off;
    const uint32_t* q = p.seqs + 3 * x.seq_off;
    int64_t r[3] = {x.rep[0], x.rep[1], x.rep[2]};
    uint32_t li = 0;
    for (uint32_t i = 0; i < x.nseq; i++) {
        const uint32_t ll = q[3 * i], ml = q[3 * i + 1], ofv = q[3 * i + 2];
        for (uint32_t k = lane; k < ll; k += 32) {
            p.out[o + k] = lit[li + k];
            p.srcidx[o + k] = (uint32_t)(o + k);
        }
        li += ll;
        o += ll;
        int64_t off;
        if (ofv > 3) {
            off = ofv - 3;
            r[2] = r[1];
            r[1] = r[0];
            r[0] = off;
        } else {
            const uint32_t k = ofv - 1 + (ll == 0);
            if (k == 0) {
                off = r[0];
            } else {
                off = k == 3 ? r[0] - 1 : r[k];  // (rep1 - 1 = 0 is rejected below)
                if (k != 1) r[2] = r[1];
                r[1] = r[0];
                r[0] = off;
            }
        }
        if (off < 1 || (uint64_t)off > o - fs) {  // (no dictionary: nothing in front of the frame)
            if (lane == 0) atomicOr(p.bad, 1u);
            return;
        }
        for (uint32_t k = lane; k < ml; k += 32) p.srcidx[o + k] = (uint32_t)(o + k - off);
        o += ml;
    }
    for (uint32_t k = lane; li + k < x.lit_n; k += 32) {
        p.out[o + k] = lit[li + k];
        p.srcidx[o + k] = (uint32_t)(o + k);
    }
}

// KZ6: one round of pointer jumping over the zstd regions; *changed when a source moved
__global__ void zx_jump_kernel(const ZxParams p) {
    bool moved = false;
    for (int i = 0; i < 4; i++) {
        if (!p.ztype[i]) continue;
        for (uint64_t g = p.base[i] + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < p.base[i] + p.raw[i];
             g += (uint64_t)gridDim.x * blockDim.x) {
            const uint32_t a = p.srcidx[g];
            if (a == g) continue;
            const uint32_t c = p.srcidx[a];
            if (c != a) {
                p.srcidx[g] = c;
                moved = true;
            }
        }
    }
    if (__syncthreads_or(moved) && threadIdx.x == 0) *p.changed = 1;
}

// KZ7: every match byte from the written byte it points at
__global__ void zx_gather_kernel(const ZxParams p) {
    for (int i = 0; i < 4; i++) {
        if (!p.ztype[i]) continue;
        for (uint64_t g = p.base[i] + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < p.base[i] + p.raw[i];
             g += (uint64_t)gridDim.x * blockDim.x) {
            const uint32_t a = p.srcidx[g];
            if (a != g) p.out[g] = p.out[a];
        }
    }
}

// XXH64
constexpr uint64_t XX_P1 = 11400714785074694791ull, XX_P2 = 14029467366897019727ull, XX_P3 = 1609587929392839161ull,
                   XX_P4 = 9650029242287828579ull, XX_P5 = 2870177450012600261ull;
__device__ __forceinline__ uint64_t xx_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t v) { return xx_rotl(acc + v * XX_P2, 31) * XX_P1; }
__device__ __forceinline__ uint64_t xx_load64(const uint8_t* p) {
    uint64_t v = 0;
    for (int k = 0; k < 8; k++) v |= (uint64_t)p[k] << (8 * k);
    return v;
}

// KZ8: one warp per frame that carries a checksum; lanes 0 .. 3 run the four accumulators over the 32-byte stripes
__global__ void __launch_bounds__(ZX_WARPS * 32) zx_xxh_kernel(const ZxParams p) {
    const uint32_t fi = blockIdx.x * ZX_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (fi >= p.nfrm) return;
    const ZxFrame& f = p.frm[fi];
    if (!f.checksum) return;
    const ZxBlk& last = p.blk[f.first + f.nblocks - 1];
    const uint64_t a = p.blk[f.first].out, n = last.out + last.n - a;
    const uint8_t* d = p.out + a;
    const uint64_t stripes = n / 32;
    const uint64_t init[4] = {XX_P1 + XX_P2, XX_P2, 0, 0 - XX_P1};
    uint64_t v = lane < 4 ? init[lane] : 0;
    if (lane < 4)
        for (uint64_t j = 0; j < stripes; j++) v = xx_round(v, xx_load64(d + 32 * j + 8 * lane));
    const uint64_t v0 = __shfl_sync(FULL, v, 0), v1 = __shfl_sync(FULL, v, 1), v2 = __shfl_sync(FULL, v, 2),
                   v3 = __shfl_sync(FULL, v, 3);
    if (lane) return;
    uint64_t h;
    if (n >= 32) {
        h = xx_rotl(v0, 1) + xx_rotl(v1, 7) + xx_rotl(v2, 12) + xx_rotl(v3, 18);
        const uint64_t vs[4] = {v0, v1, v2, v3};
        for (int k = 0; k < 4; k++) h = (h ^ xx_round(0, vs[k])) * XX_P1 + XX_P4;
    } else {
        h = XX_P5;
    }
    h += n;
    uint64_t i = stripes * 32;
    for (; i + 8 <= n; i += 8) h = xx_rotl(h ^ xx_round(0, xx_load64(d + i)), 27) * XX_P1 + XX_P4;
    if (i + 4 <= n) {
        h = xx_rotl(h ^ ((uint64_t)sx_load32(d + i) * XX_P1), 23) * XX_P2 + XX_P3;
        i += 4;
    }
    for (; i < n; i++) h = xx_rotl(h ^ (d[i] * XX_P5), 11) * XX_P1;
    h = (h ^ (h >> 33)) * XX_P2;
    h = (h ^ (h >> 29)) * XX_P3;
    h ^= h >> 32;
    if ((uint32_t)h != f.cks) atomicOr(p.bad, 1u);
}

// ---------------------------------------------------------------------------------
// KZ1: encode
// ---------------------------------------------------------------------------------
// the predefined tables run backwards: enc[sym][next state] is the state in front of it, first[sym] a state of sym
struct ZxEncTables {
    ZxFse ll[64], of[32], ml[64];
    uint8_t ell[36][64], eof[32][32], eml[53][64];
    uint8_t fll[36], fof[32], fml[53];
};

__device__ void zx_enc_tables(ZxEncTables& t, ZxHufScratch& h) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < 36; i++) h.cnt[i] = zx_ll_default[i];
        zx_fse_build(h.cnt, 36, 6, t.ll, h.nxt);
        for (int i = 0; i < 29; i++) h.cnt[i] = zx_of_default[i];
        zx_fse_build(h.cnt, 29, 5, t.of, h.nxt);
        for (int i = 0; i < 53; i++) h.cnt[i] = zx_ml_default[i];
        zx_fse_build(h.cnt, 53, 6, t.ml, h.nxt);
    }
    __syncthreads();
    for (uint32_t u = threadIdx.x; u < 64 + 32 + 64; u += blockDim.x) {
        const ZxFse* tab = u < 64 ? t.ll : u < 96 ? t.of : t.ml;
        const uint32_t st = u < 64 ? u : u < 96 ? u - 64 : u - 96;
        const ZxFse e = tab[st];
        uint8_t* row = u < 64 ? t.ell[e.sym] : u < 96 ? t.eof[e.sym] : t.eml[e.sym];
        for (uint32_t x = e.base; x < e.base + (1u << e.nb); x++) row[x] = (uint8_t)st;
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int u = 63; u >= 0; u--) {
            t.fll[t.ll[u].sym] = (uint8_t)u;
            t.fml[t.ml[u].sym] = (uint8_t)u;
            if (u < 32) t.fof[t.of[u].sym] = (uint8_t)u;
        }
    __syncthreads();
}

// sx_match_warp's elements as zstd sequences: literals to lit, (ll, ml, offset) packed into seq
struct ZxSeqEmit {
    uint8_t* lit;
    uint64_t* seq;
    uint32_t nlit, nseq, pend;
    __device__ bool literal(const uint8_t* s, uint32_t L) {
        for (uint32_t k = threadIdx.x & 31; k < L; k += 32) lit[nlit + k] = s[k];
        nlit += L;
        pend += L;
        return true;
    }
    __device__ bool copy(uint32_t off, uint32_t L) {
        if ((threadIdx.x & 31) == 0) seq[nseq] = (uint64_t)pend | (uint64_t)L << 17 | (uint64_t)off << 34;
        nseq++;
        pend = 0;
        return true;
    }
};

// the code of v among bases[0, n) (the last base at or below v)
__device__ __forceinline__ uint32_t zx_code(const uint32_t* bases, uint32_t n, uint32_t v) {
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (bases[mid] <= v) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// forward bits, at most `limit` bytes
struct ZxBitW {
    uint8_t* d;
    uint32_t o, limit, nb;
    uint64_t acc;
    bool ok;
    __device__ void put(uint32_t v, uint32_t n) {
        acc |= (uint64_t)(v & ((1u << n) - 1)) << nb;
        nb += n;
        while (nb >= 8) {
            if (o >= limit) ok = false;
            else d[o] = (uint8_t)acc;
            o++;
            acc >>= 8;
            nb -= 8;
        }
    }
};

struct ZxEncParams {
    uint64_t* seqs;     // ZX_SEQ_CAP per chunk of a zstd input
    uint32_t zfirst[3];  // input b's first chunk among the zstd inputs' chunks
};

// KZ1: chunk ci of a zstd input as one block (block header included) into slot ci
constexpr size_t ZX_ENC_HS = (sizeof(ZxEncTables) + 15) & ~(size_t)15;
constexpr size_t ZX_ENC_HASH = ZX_ENC_HS + ((sizeof(ZxHufScratch) + 15) & ~(size_t)15);
constexpr size_t ZX_ENCODE_SMEM = ZX_ENC_HASH + S2_WARPS * (2u << S2_HASH_BITS);

__global__ void __launch_bounds__(S2_WARPS * 32) zx_encode_kernel(const SxEncParams p, const ZxEncParams z) {
    extern __shared__ uint32_t zx_smem[];
    ZxEncTables& t = *reinterpret_cast<ZxEncTables*>(zx_smem);
    ZxHufScratch& hs = *reinterpret_cast<ZxHufScratch*>(reinterpret_cast<uint8_t*>(zx_smem) + ZX_ENC_HS);
    uint16_t* hash = reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(zx_smem) + ZX_ENC_HASH);
    zx_enc_tables(t, hs);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t ci = blockIdx.x * S2_WARPS + warp;
    if (ci >= p.nchunks) return;
    int b = 0;
    while (ci >= p.first[b + 1]) b++;
    if (p.codec[b] != 2) return;
    const uint64_t at = (uint64_t)(ci - p.first[b]) * ZX_CHUNK;
    const uint32_t n = (uint32_t)min((uint64_t)ZX_CHUNK, p.len[b] - at);
    const bool last = ci + 1 == p.first[b + 1];
    const uint8_t* in = p.src[b] + at;
    uint8_t* slot = p.slots + (uint64_t)ci * S2_SLOT;
    uint64_t* seq = z.seqs + (uint64_t)(z.zfirst[b] + ci - p.first[b]) * ZX_SEQ_CAP;
    // content: raw literals with a 3-byte header, then the sequences section; kept only when shorter than n
    ZxSeqEmit e{slot + 6, seq, 0, 0, 0};
    sx_match_warp(in, n, hash + (warp << S2_HASH_BITS), e);
    __syncwarp();
    uint32_t size = 0;
    bool comp = false;
    if (lane == 0 && e.nseq) {
        const uint32_t L = e.nlit, N = e.nseq;
        slot[3] = (uint8_t)(0 | (3 << 2) | ((L & 15) << 4));
        slot[4] = (uint8_t)(L >> 4);
        slot[5] = (uint8_t)(L >> 12);
        ZxBitW w{slot, 6 + L, 3 + n, 0, 0, true};
        if (N < 128) {
            w.put(N, 8);
        } else {
            w.put(128 + (N >> 8), 8);
            w.put(N & 255, 8);
        }
        w.put(0, 8);  // LL, OF, ML: predefined
        // states from the last sequence back (the decoder reads initial states, then per sequence OF, ML, LL extra bits
        // and LL, ML, OF state updates; the writer goes in reverse)
        uint32_t sl = 0, so = 0, sm = 0;
        for (int32_t i = (int32_t)N - 1; i >= 0; i--) {
            const uint64_t v = seq[i];
            const uint32_t ll = (uint32_t)(v & 0x1ffff), ml = (uint32_t)((v >> 17) & 0x1ffff), ofv = (uint32_t)(v >> 34) + 3;
            const uint32_t lc = zx_code(zx_ll_base, 36, ll), mc = zx_code(zx_ml_base, 53, ml), oc = 31 - __clz(ofv);
            if (i == (int32_t)N - 1) {
                sl = t.fll[lc];
                so = t.fof[oc];
                sm = t.fml[mc];
            } else {
                const uint32_t pl = t.ell[lc][sl], po = t.eof[oc][so], pm = t.eml[mc][sm];
                w.put(so - t.of[po].base, t.of[po].nb);
                w.put(sm - t.ml[pm].base, t.ml[pm].nb);
                w.put(sl - t.ll[pl].base, t.ll[pl].nb);
                sl = pl;
                so = po;
                sm = pm;
            }
            w.put(ll - zx_ll_base[lc], zx_ll_bits[lc]);
            w.put(ml - zx_ml_base[mc], zx_ml_bits[mc]);
            w.put(ofv - (1u << oc), oc);
        }
        w.put(sm, 6);
        w.put(so, 5);
        w.put(sl, 6);
        w.put(1, 1);
        if (w.nb) w.put(0, 8 - w.nb);
        comp = w.ok && w.o < 3 + n;
        size = w.o;
    }
    comp = __shfl_sync(FULL, comp, 0);
    size = __shfl_sync(FULL, size, 0);
    __syncwarp();
    if (!comp) {
        for (uint32_t k = lane; k < n; k += 32) slot[3 + k] = in[k];
        size = 3 + n;
    }
    if (lane == 0) {
        const uint32_t bh = (last ? 1u : 0u) | (comp ? 2u : 0u) << 1 | (size - 3) << 3;
        slot[0] = (uint8_t)bh;
        slot[1] = (uint8_t)(bh >> 8);
        slot[2] = (uint8_t)(bh >> 16);
        p.size[ci] = size;
    }
}

}  // namespace sj
