// s2s_link_emu.cpp -- the host emulation of the streaming stage 2 (s2s_emu.cpp, included whole: the fiber warp, the
// tables, s2s_emu_parse) with K2r's root-word links switched on (test infrastructure, NOT the product).
//
// s2s_emu_parse runs K2r without a `rootlink` bitmap, so there K2r writes no root words and the K2f loop writes them all;
// its K2e loop already leaves the closes K2r has linked (BRK_LINKED makes them match neither close kind) alone.
// s2s_emu_parse_linked below is the same pipeline with the bitmap, as the device parse runs it: K2r writes the root
// words of the records that lie inside one staged step and clears their bits, and the K2f loop skips exactly those
// records -- so a wrong root word written by K2r reaches the tape and the comparison with the oracle.
#include "s2s_emu.cpp"

extern "C" int s2s_emu_parse_linked(const uint8_t* msg, size_t len, int ndjson, const uint32_t* idx, size_t n_idx, uint64_t* tape,
                                    size_t tape_cap, size_t* tape_len, uint8_t* strings, size_t strings_cap, size_t* strings_len,
                                    uint32_t* num_pos, uint32_t* num_slot, size_t num_cap, size_t* n_num, size_t* n_linked) {  // n_linked[0]: closes, [1]: records K2r has linked
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
    p.rootlink = rootlink.data();
    p.numlist = numlist.data();
    for (uint32_t f = 0; f < 3; f++) W.run([&](FiberWarp& w) { s2s_warp_loop<FiberWarp, true>(w, p, f, 3, sm); });
    for (uint32_t i = 0; i < grand.num; i++) {
        num_pos[i] = numlist[i].pos;
        num_slot[i] = numlist[i].slot;
    }
    // K2d
    std::vector<int32_t> par(nb + 1, -1), stack;
    for (uint32_t k = 0; k < nb; k++) {
        while (!stack.empty() && brk_depth[stack.back()] >= brk_depth[k]) stack.pop_back();
        par[k] = stack.empty() ? -1 : stack.back();
        stack.push_back((int32_t)k);
    }
    // K2e, as s2s_link_kernel: the flag masked where kinds are compared, linked closes skipped
    size_t linked = 0, linked_rec = 0;
    for (uint32_t k = 0; k <= nb; k++) {
        uint32_t ctx = CTX_ROOT;
        if (k > 0) {
            const uint32_t kd = brk_kind[k - 1] & ~BRK_LINKED;
            int32_t enc;
            if (kd == T_OBJ_OPEN || kd == T_ARR_OPEN)
                enc = (int32_t)k - 1;
            else {
                const int32_t m = par[k - 1];
                enc = m >= 0 ? par[m] : -1;
            }
            ctx = enc >= 0 ? ((brk_kind[enc] & ~BRK_LINKED) == T_OBJ_OPEN ? CTX_OBJ : CTX_ARR) : CTX_ROOT;
        }
        const uint32_t sg = (segmask[k >> 2] >> (8 * (k & 3))) & 0xff;
        if (!((sg >> ctx) & 1)) error |= 1;
        if (k < nb && (brk_kind[k] & BRK_LINKED)) linked++;
        if (k < nb && (brk_kind[k] == T_OBJ_CLOSE || brk_kind[k] == T_ARR_CLOSE)) {
            const int32_t m = par[k];
            if (m >= 0) {
                const uint32_t otp = brk_tp[m], ctp = brk_tp[k];
                tape[otp] = ((uint64_t)(brk_kind[k] == T_OBJ_CLOSE ? '{' : '[') << 56) | ((uint64_t)ctp + 1);
                tape[ctp] = ((uint64_t)(brk_kind[k] == T_OBJ_CLOSE ? '}' : ']') << 56) | otp;
            }
        }
    }
    // K2f, the records whose bit K2r has cleared skipped
    for (uint64_t r = 0; r <= grand.rec; r++) {
        if (!((rootlink[r >> 5] >> (r & 31)) & 1u)) {
            linked_rec++;
            continue;
        }
        const uint64_t R = (uint64_t)'r' << 56;
        const uint64_t open = r == 0 ? 0 : rootpos[r];
        const uint64_t next_open = r == grand.rec ? tlen : rootpos[r + 1];
        if (next_open > tlen || next_open == 0) continue;
        tape[open] = R | next_open;
        tape[next_open - 1] = R | open;
    }
    if (n_linked) n_linked[0] = linked, n_linked[1] = linked_rec;
    if (error || grand.depth != 0) return 2;
    return 0;
}
