// s2s_tile_emu.cpp -- the host emulation of the streaming stage 2 (s2s_emu.cpp, included whole: the fiber warp, the
// tables) with K2t as the device runs it (simdjson-go_b200/csrc/s2s_tile.h; test infrastructure, NOT the product).
//
// K2r runs as in the device parse; behind it, instead of a restatement of the scope matching and the links, the tiles of
// K2t-link run one after the other, last tile first (no tile reads another one's output), over a min hierarchy that
// restates K2t-min.  `k2r_links` = 0 runs K2r without the rootlink bitmap, so that K2t writes every root word; 1 runs it
// with the bitmap, as the device does.
#include "s2s_emu.cpp"

#include <algorithm>

#include "../../simdjson-go_b200/csrc/s2s_tile.h"

namespace {

void k2t_emu(const S2sParams& p, uint32_t nb, uint64_t nrec, uint64_t tlen, uint32_t* error) {
    S2tLevels L;
    memset(&L, 0, sizeof L);
    L.n[0] = nb;
    L.nlevels = 1;
    std::vector<std::vector<uint32_t>> lv(S2T_MAX_LEVELS);
    for (uint32_t sz = nb; sz > 32 && L.nlevels < S2T_MAX_LEVELS;) {
        const int l = L.nlevels;
        lv[l].assign((sz + 31) / 32, ~0u);
        for (uint32_t i = 0; i < sz; i++) lv[l][i / 32] = std::min(lv[l][i / 32], l == 1 ? s2t_key(p.brk_depth[i]) : lv[l - 1][i]);
        sz = (uint32_t)lv[l].size();
        L.lv[l] = lv[l].data();
        L.n[l] = sz;
        L.nlevels++;
    }
    const uint64_t items = std::max((uint64_t)nb + 1, nrec + 1);
    const uint64_t tb = s2s_tape_base(p);
    std::vector<int32_t> d_s(S2T_TILE), par_s(S2T_TILE);
    std::vector<uint8_t> k_s(S2T_TILE);
    for (uint64_t b = (items + S2T_TILE - 1) / S2T_TILE; b-- > 0;) {
        const uint32_t lo = (uint32_t)(b * S2T_TILE);
        for (uint32_t i = 0; i < S2T_TILE && lo + i < nb; i++) d_s[i] = p.brk_depth[lo + i], k_s[i] = p.brk_kind[lo + i];
        const S2tTile v{p.brk_depth, p.brk_kind, d_s.data(), k_s.data(), par_s.data(), lo, &L};
        for (uint32_t i = 0; i < S2T_TILE && lo + i < nb; i++) par_s[i] = s2t_par(v, lo + i);
        for (uint32_t i = 0; i < S2T_TILE && lo + i <= nb; i++)
            if (!s2t_segment(p, v, nb, lo + i, tb)) *error |= 1;
        for (uint32_t i = 0; i < S2T_TILE && lo + i <= nrec; i++) s2t_root(p, lo + i, nrec, tlen, tb);
    }
}

}  // namespace

// as s2s_emu_parse (0 ok, 2 stage-2 failure, 4 capacity; numbers as (position, slot) pairs)
extern "C" int s2s_emu_parse_tiled(const uint8_t* msg, size_t len, int ndjson, const uint32_t* idx, size_t n_idx, uint64_t* tape,
                                   size_t tape_cap, size_t* tape_len, uint8_t* strings, size_t strings_cap, size_t* strings_len,
                                   uint32_t* num_pos, uint32_t* num_slot, size_t num_cap, size_t* n_num, int k2r_links) {
    static Tables T;
    const uint32_t SPT = 16;
    const uint32_t nslabs = (uint32_t)((len + S2S_SLAB_BYTES - 1) / S2S_SLAB_BYTES);
    std::vector<uint32_t> slabpar((nslabs + SPT - 1) / SPT + 1, 0);
    {
        bool in = false, esc = false;
        for (size_t i = 0; i < len; i++) {
            if (i % S2S_SLAB_BYTES == 0 && in) slabpar[(i / S2S_SLAB_BYTES) / SPT] |= 1u << ((i / S2S_SLAB_BYTES) % SPT);
            const uint8_t c = msg[i];
            if (esc)
                esc = false;
            else if (c == '\\')
                esc = true;
            else if (c == '"')
                in = !in;
        }
    }
    std::vector<SlabAgg> agg(nslabs), pre(nslabs), grp_pre((nslabs + 1023) / 1024 + 1);
    std::vector<uint8_t> src(S2S_IMAGE_BYTES + 64), sstage(S2S_SSTAGE_BYTES + 64);
    std::vector<uint64_t> tstage(S2S_TSTAGE_WORDS + 8);
    uint32_t error = 0;
    S2sParams p;
    memset(&p, 0, sizeof p);
    p.msg = msg;
    p.len = len;
    p.ndjson = ndjson ? 1 : 0;
    p.idx = idx;
    p.n_idx = (uint32_t)n_idx;
    p.slabpar = slabpar.data();
    p.slabs_per_tile = SPT;
    p.nslabs = nslabs;
    p.agg = agg.data();
    p.pre = pre.data();
    p.grp_pre = grp_pre.data();
    p.error = &error;
    S2sWarpMem sm;
    sm.src = (uint8_t*)(((uintptr_t)src.data() + 15) & ~(uintptr_t)15);
    sm.sstage = (uint8_t*)(((uintptr_t)sstage.data() + 15) & ~(uintptr_t)15);
    sm.tstage = (uint64_t*)(((uintptr_t)tstage.data() + 15) & ~(uintptr_t)15);
    sm.esc = reinterpret_cast<uint8_t*>(sm.tstage);
    sm.ctab = T.ctab;
    sm.oktab = T.oktab;
    sm.cmptab = T.cmptab;
    FiberWarp W;
    for (uint32_t f = 0; f < 3; f++) W.run([&](FiberWarp& w) { s2s_warp_loop<FiberWarp, false>(w, p, f, 3, sm); });
    SlabAgg grand = agg_zero();
    for (uint32_t g0 = 0, gi = 0; g0 < nslabs; g0 += 1024, gi++) {
        grp_pre[gi] = grand;
        SlabAgg acc = agg_zero();
        for (uint32_t i = g0; i < nslabs && i < g0 + 1024; i++) {
            pre[i] = acc;
            acc = agg_combine(acc, agg[i]);
        }
        grand = agg_combine(grand, acc);
    }
    const uint64_t tlen = (uint64_t)grand.w + 2;
    *tape_len = tlen;
    *strings_len = grand.str;
    *n_num = grand.num;
    if (tlen > tape_cap || grand.str > strings_cap || grand.num > num_cap) return 4;
    const uint32_t nb = grand.brk;
    std::vector<uint32_t> brk_tp(nb + 1), segmask((nb + 1 + 3) / 4 + 1, 0xffffffffu), rootpos(grand.rec + 2, 0);
    std::vector<uint32_t> rootlink((grand.rec + 1 + 31) / 32, 0xffffffffu);
    std::vector<int32_t> brk_depth(nb + 1);
    std::vector<uint8_t> brk_kind(nb + 1);
    std::vector<NumEntry> numlist(grand.num + 1);
    memset(tape, 0, tlen * 8);
    p.tape = tape;
    p.strings = strings;
    p.brk_tp = brk_tp.data();
    p.brk_depth = brk_depth.data();
    p.brk_kind = brk_kind.data();
    p.segmask = segmask.data();
    p.rootpos = rootpos.data();
    p.rootlink = k2r_links ? rootlink.data() : nullptr;
    p.numlist = numlist.data();
    for (uint32_t f = 0; f < 3; f++) W.run([&](FiberWarp& w) { s2s_warp_loop<FiberWarp, true>(w, p, f, 3, sm); });
    p.rootlink = rootlink.data();
    for (uint32_t i = 0; i < grand.num; i++) {
        num_pos[i] = numlist[i].pos;
        num_slot[i] = numlist[i].slot;
    }
    k2t_emu(p, nb, grand.rec, tlen, &error);
    if (error || grand.depth != 0) return 2;
    return 0;
}
