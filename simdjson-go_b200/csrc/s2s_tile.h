// s2s_tile.h -- K2t, the tail of the streaming stage 2 behind K2r: the scope matching of the brackets, the grammar
// verdict of every bracket-to-bracket segment against the container it lies in, the cross-links of the closes K2r has
// not linked (stage2...go:327-334) and the root words of the records K2r has not linked (K2f, stage2...go:170,207-218,
// 428-441).
//
// par[k] = the nearest bracket in front of bracket k with a smaller depth in front of it (none for a bracket at depth
// 0 or above: a close at the top level is in no legal transition, so "none" is exact for every accepted document).
// For a close par is its open; the container open behind a close is par of that open.
//
// One CTA takes a tile of S2T_TILE brackets and keeps their depths, kinds and pars in shared memory, so the container
// of a segment is found inside the CTA: no CTA reads another CTA's output, and no ordering between CTAs is needed.  A
// search that leaves the tile climbs a hierarchy of 32-wide minima over the depths, built by one launch in front
// (K2t-min): levels 1 and 2 lie inside a tile and the tile stores them; a level above spans several tiles, and every
// tile puts its minimum there with an atomicMin.  That level memory is preset to all ones, so the minima are stored as
// order-preserving unsigned keys (s2t_key) and all ones is "no bracket".
//
// Portable C++ like s2s_core.h: tests/emu/s2s_tile_emu.cpp runs these functions tile by tile on the host.
#pragma once
#include "s2s_core.h"

namespace sj {

constexpr uint32_t S2T_TILE = 2048;  // brackets per CTA of K2t (1 024, 2 048, 4 096 and 8 192 measured: see DESIGN §6)
constexpr int S2T_MAX_LEVELS = 8;
static_assert(S2T_TILE % 1024 == 0 && 32768 % S2T_TILE == 0, "levels 1 and 2 lie inside one tile, level 3 covers whole tiles");

SJ_HD uint32_t s2t_key(int32_t d) { return (uint32_t)d ^ 0x80000000u; }
SJ_HD int32_t s2t_unkey(uint32_t key) { return (int32_t)(key ^ 0x80000000u); }

// the min hierarchy over the brackets' depths: level l >= 1 holds n[l] keys, entry i the minimum of entries 32 i ..
// 32 i + 31 of level l - 1 (level 0 = brk_depth itself).  Levels are added while a level has more than 32 entries.
struct S2tLevels {
    uint32_t* lv[S2T_MAX_LEVELS];
    uint32_t n[S2T_MAX_LEVELS];
    int nlevels;
};

// what one tile sees: its own brackets in shared memory, everything else in global memory
struct S2tTile {
    const int32_t* depth;  // [nb] brk_depth
    const uint8_t* kind;   // [nb] brk_kind
    const int32_t* d_s;    // [S2T_TILE] the tile's depths, kinds and pars
    const uint8_t* k_s;
    const int32_t* par_s;
    uint32_t lo;           // first bracket of the tile
    const S2tLevels* L;
    SJ_HD bool own(uint32_t i) const { return i - lo < S2T_TILE; }
    SJ_HD int32_t d(uint32_t i) const { return own(i) ? d_s[i - lo] : depth[i]; }
    SJ_HD uint32_t kd(uint32_t i) const { return (own(i) ? k_s[i - lo] : kind[i]) & ~BRK_LINKED; }
    SJ_HD int32_t at(int l, uint32_t i) const { return l == 0 ? d(i) : s2t_unkey(L->lv[l][i]); }
};

// par of bracket k, searched: its 32-group backwards, then up the hierarchy to the first earlier entry below the depth
// and down again to its last bracket below it.  On level 0 the search steps back by 1 + d - t: the depth moves by one
// per bracket, so the d - t brackets in front of one at depth d are no shallower than t.  Every loop leaves through its
// end, not by a return: the lanes of a warp that finish a loop at different trips meet again behind it, and the next
// loop runs once for the whole warp rather than once per group of lanes.
SJ_HD int32_t s2t_par(const S2tTile& v, uint32_t k) {
    const int32_t t = v.d(k);
    if (t <= 0) return -1;
    int64_t found = -1;
    for (int64_t m = (int64_t)k - 1, lo = k & ~31u; m >= lo;) {
        const int32_t d = v.d((uint32_t)m);
        if (d < t) {
            found = m;
            break;
        }
        m -= 1 + (int64_t)(d - t);
    }
    if (found < 0) {
        int64_t idx = (int64_t)(k >> 5) - 1;
        for (int l = 1; l < v.L->nlevels && idx >= 0; l++) {
            const int64_t lo = idx & ~31ll;
            int64_t hit = -1;
            for (int64_t j = idx; j >= lo; j--)
                if (v.at(l, (uint32_t)j) < t) {
                    hit = j;
                    break;
                }
            if (hit >= 0) {
                for (int m = l; m >= 1; m--) {  // descend: the last child below t (there is one)
                    const int64_t base = hit * 32, last = (int64_t)v.L->n[m - 1] - 1;
                    int64_t c = base + 31 < last ? base + 31 : last;
                    if (m == 1) {
                        for (int32_t d; c > base && (d = v.d((uint32_t)c)) >= t;) {
                            c -= 1 + (int64_t)(d - t);
                            if (c < base) c = base;
                        }
                    } else {
                        while (c > base && v.at(m - 1, (uint32_t)c) >= t) c--;
                    }
                    hit = c;
                }
                found = hit;
                break;
            }
            idx = (lo >> 5) - 1;
        }
    }
    return (int32_t)found;
}

SJ_HD int32_t s2t_par_of(const S2tTile& v, uint32_t i) { return v.own(i) ? v.par_s[i - v.lo] : s2t_par(v, i); }

// segment k -- the structurals behind bracket k - 1 up to and including bracket k; k = nb: behind the last bracket --
// against the container open right after bracket k - 1 (the bracket itself if it opens, else the parent of the scope
// it closes); then bracket k's cross-links when it is a close K2r has not linked (BRK_LINKED makes a close match
// neither kind).  k is one of the tile's own brackets, or nb.  Returns false when the segment breaks the grammar.
SJ_HD bool s2t_segment(const S2sParams& p, const S2tTile& v, uint32_t nb, uint32_t k, uint64_t tape_base) {
    uint32_t ctx = CTX_ROOT;
    if (k > 0) {
        const uint32_t kd = v.kd(k - 1);
        int32_t enc = (int32_t)k - 1;
        if (kd != T_OBJ_OPEN && kd != T_ARR_OPEN) {
            const int32_t m = s2t_par_of(v, k - 1);
            enc = m >= 0 ? s2t_par_of(v, (uint32_t)m) : -1;
        }
        ctx = enc >= 0 ? (v.kd((uint32_t)enc) == T_OBJ_OPEN ? CTX_OBJ : CTX_ARR) : CTX_ROOT;
    }
    if (k < nb) {
        const uint32_t kd = v.k_s[k - v.lo];
        const int32_t m = v.par_s[k - v.lo];
        if ((kd == T_OBJ_CLOSE || kd == T_ARR_CLOSE) && m >= 0) {
            const uint32_t otp = p.brk_tp[m], ctp = p.brk_tp[k];
            p.tape[otp] = ((uint64_t)(kd == T_OBJ_CLOSE ? '{' : '[') << 56) | (tape_base + ctp + 1);
            p.tape[ctp] = ((uint64_t)(kd == T_OBJ_CLOSE ? '}' : ']') << 56) | (tape_base + otp);
        }
    }
    const uint32_t sg = (p.segmask[k >> 2] >> (8 * (k & 3))) & 0xffu;
    return (sg >> ctx) & 1u;
}

// the root words of record r (r <= n_records): it opens at rootpos[r], its close sits right in front of the next
// record's open (or is the last word of the tape).  Records whose bit in rootlink K2r has cleared are written already.
SJ_HD void s2t_root(const S2sParams& p, uint64_t r, uint64_t n_records, uint64_t tape_len, uint64_t tape_base) {
    if (!((p.rootlink[r >> 5] >> (r & 31)) & 1u)) return;
    const uint64_t R = (uint64_t)'r' << 56;
    const uint64_t open = r == 0 ? 0 : p.rootpos[r];
    const uint64_t next_open = r == n_records ? tape_len : p.rootpos[r + 1];
    if (next_open <= tape_len && next_open != 0) {
        p.tape[open] = R | (tape_base + next_open);
        p.tape[next_open - 1] = R | (tape_base + open);
    }
}

}  // namespace sj
