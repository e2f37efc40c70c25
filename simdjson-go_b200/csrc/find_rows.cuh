// find_rows.cuh -- the array rows of the device find: for every record (a root, in the find's order), the array at a
// row path, and each of its elements one row of the find's columns.  A literal port of
//     elem.FindElement(row_path...) -> Element.Iter.Array    (parsed_json.go:833-864, :1022-1039), or elem.Array for a
//                                                            row path of 0 segments
//     Array.ForEach(func(i Iter) { i.FindElement(path...) ... })   (parsed_array.go:45-56, Advance :196-223)
// tests/find_rows_oracle.py is the same port in Python.
//
// A record's array is its tape [head, end), laid end to end with the other records' arrays in find_json.cuh's virtual
// word space (FjWords, KJ0's scan); the work is spread over those words, not over records, as one array may be nearly
// the whole tape.  The rows are proposed, then verified:
//   KR1 fr_record   one thread per record: its status, and its array's head and words (KF3's walk for the row path)
//   (KJ0 over the records' words, KJ1's segmented head scan over the array words)
//   KR2 fr_stop     the proposed walk: the heads directly inside each array (depth 1 in KJ1's scan).  The first of them
//       that ends ForEach there -- a TypeNone tag (']', '}', any unknown tag), a nop, or a scope whose link lies behind
//       it -- lowers the record's stop to its word with atomicMin; the heads in front of the stop are its candidates
//   KR3 fr_count    the candidates per tile (count and last word, RAgg), scanned; each record's in-tile prefixes
//   KR4 fr_verify   every candidate and every stop checks that Advance's successor of the candidate in front of it (a
//       scalar's off + 1 or + 2, a scope's link) is itself, and the first one that it is the word after '['.  So, by
//       induction from that word, the candidates are ForEach's elements
//   KR5 fr_finish   per record: its element count, and the last checks (a stop that is a nop, or no stop: the last
//       successor reaches the end).  A record that fails any check is walked literally by one thread (fr_walk) here
//   (the counts' scan: each record's first row)
//   KR6 fr_emit     each candidate of a verified record writes its row: (head, array end) as two uint32 words
//   KR7 fr_serial_emit   the rows of a record walked by one thread
//   (KF3 .. with rows = the elements: fd_walk_kernel<true> enters FindElement from each element's Iter)
//   KR8 fr_out      the record and row columns into the caller's buffers
//
// Member rows (an object's members, Object.ForEach, parsed_object.go:142-186, with Iter.Object, parsed_json.go:998-1018)
// are the same row source over each record's object: KR1<true> takes the Iter.Object branch, and KR2 .. KR4 verify
// that the heads directly inside it are Advance's sequence, which alternates key, value, key, value.  Then
//   KO1 fo_role     each candidate's rank in its record (KR3's scan) gives its role: a bit per word for the keys
//   KO2 fo_select   a key that fails ForEach's key checks marks its record for the one-thread walk (fo_walk); a key
//       whose value is a candidate and whose bytes are among only_keys (or every key) is selected: a bit per word,
//       counted per tile and scanned (MSum)
//   KR5<true>       a record's rows are its selected members, at most len(onlyKeys) of them
//   KO3 fo_emit     each selected key in front of that cut writes its row: (value head, object end) and its key head
//   KR7<true>       the rows of a record walked by one thread
//   (KF4 and the scans over the rows' key lengths)
//   KO4 fo_keys     the key column: offsets, and the keys' bytes (longer keys by their whole warp) behind KR8
#pragma once
#include "find.cuh"
#include "find_json.cuh"

namespace sj {

constexpr uint64_t FR_NO_STOP = ~0ull;

// the (candidates, last candidate's virtual word + 1, 0 for none) of a run of words
struct RAgg {
    uint64_t n, last;
};
__device__ __forceinline__ RAgg agg_combine(const RAgg& a, const RAgg& b) { return RAgg{a.n + b.n, b.last ? b.last : a.last}; }
__device__ __forceinline__ RAgg agg_shfl_up(const RAgg& a, int d) {
    return RAgg{__shfl_up_sync(FULL, a.n, d), __shfl_up_sync(FULL, a.last, d)};
}

// the last candidate's virtual word + 1 alone (KR4 reads no counts)
struct RLast {
    uint64_t v;
};
__device__ __forceinline__ RLast agg_combine(const RLast& a, const RLast& b) { return RLast{b.v ? b.v : a.v}; }
__device__ __forceinline__ RLast agg_shfl_up(const RLast& a, int d) { return RLast{__shfl_up_sync(FULL, a.v, d)}; }

struct FrCells {
    FjWords m;                // the records' arrays (m.rows = records, m.head = each array's '[')
    TapeView t;
    const FjAgg* h_tile_pre;  // KJ1's scan
    const FjAgg* h_grp_pre;
    uint64_t* stop;           // [records]: the virtual word ForEach's proposed walk stops on, FR_NO_STOP for none
    const RAgg* c_tile_pre;   // KR3's scan
    const RAgg* c_grp_pre;
    RAgg* c_lo;               // [records]: KR3's in-tile prefix in front of a record's '[' / behind its last word
    RAgg* c_hi;
    uint8_t* bad;             // [records]: 1 when a check failed
    uint8_t* serial;          // [records]: 1 when the record is walked by one thread
    uint64_t* E;              // [records + 1]: element counts, then their exclusive scan and total
    uint64_t* base;           // [records]: candidates in front of each record
    unsigned long long* n_serial;  // the records walked by one thread
    uint32_t* erow;           // [rows][2]
    // member rows
    uint32_t* krow;           // [rows]: each row's key head
    uint64_t* klen;           // [rows + 1]: each row's key length, then their exclusive scan and total
    uint8_t* st;              // [records]: each record's status (KR1's; a walked record's ForEach error)
    const FdSeg* kseg;        // only_keys: nkeys staged segments over kbytes, mkeys of them distinct (0: every key)
    const uint8_t* kbytes;
    uint32_t nkeys, mkeys;
    uint8_t* sel;             // [word tiles * TAPE_THREADS]: bit j of a thread: its word j is a selected key
    const MSum* s_tile_pre;   // KO2's scan
    const MSum* s_grp_pre;
    MSum* s_lo;               // [records]: KO2's in-tile prefix in front of a record's '{' / behind its last word
    MSum* s_hi;
};

// Advance's next offset after the element whose head is word i (calcNext(false) from off = i + 1)
__device__ __forceinline__ uint64_t fr_succ(const TapeView& t, uint64_t i) {
    const uint64_t w = t.tape[i];
    const uint32_t tag = (uint32_t)(w >> 56);
    if (tape_value_tag(tag)) return i + 2;
    if (fd_scope_tag(tag)) return w & TAPE_VALUE_MASK;
    return i + 1;
}
// Advance at head i ends ForEach: a TypeNone tag, a nop (which Advance skips: the record is walked by one thread), or
// a scope whose link lies behind its word (addNext < 0)
__device__ __forceinline__ bool fr_stops(const TapeView& t, uint64_t i) {
    const uint64_t w = t.tape[i];
    const uint32_t tag = (uint32_t)(w >> 56);
    return fd_type(tag) == 0 || (fd_scope_tag(tag) && (w & TAPE_VALUE_MASK) < i + 1);
}

// KR1: one thread per record.  FindElement(row path) as KF3 (no row path: the element itself), then Iter.Array, or
// with OBJ Iter.Object.
template <bool OBJ>
__global__ void __launch_bounds__(256) fr_record_kernel(const FindParams p, uint32_t row_path, uint8_t* st, int64_t* head,
                                                        uint64_t* words) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= p.roots.n) return;
    const FdPath path = p.paths[row_path];
    FdIt cp{0, 0, 0, 0, 0}, e{0, 0, 0, 0, 0};
    bool fresh = false;
    uint32_t s = FD_CORRUPT;
    if (fd_root_elem(p, tape_root(p.roots, r), cp)) {
        if (path.nseg == 0) {
            e = cp;
            s = FD_OK;
        } else {
            s = fd_find_element(p, cp, p.segs + path.seg0, p.seg_bytes, path.nseg, e, &fresh);
        }
    }
    uint64_t h = 0, n = 0;
    if (s == FD_OK) {
        if (fresh || e.t != (OBJ ? '{' : '[')) s = FD_CONVERT;  // a fresh Element, or "next item is not array / object"
        else if (OBJ && e.cur < e.off) s = FD_CORRUPT;          // "object ends at index before start"
        else if (e.n < e.cur) s = FD_CORRUPT;                    // "object extended beyond tape"
        else if (e.cur > e.off) h = e.off - 1, n = e.cur - h;  // a link at or behind the '[': Tape[:end] ends before
                                                                 // off, and ForEach's first Advance ends it (no rows)
    }
    st[r] = (uint8_t)s;
    head[r] = (int64_t)h;
    words[r] = n;
}

// KR2: every head that stops its walk lowers the record's stop to its word (stop preset to FR_NO_STOP)
__global__ void __launch_bounds__(TAPE_THREADS) fr_stop_kernel(const FrCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, false, true);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) fj_lower_stop(c.stop, (h >> j & 1) && fr_stops(c.t, x[j].i), x[j].r, base + j);
}

// this thread's candidates (bit j: a head directly inside its array in front of the record's stop) and their RAgg
__device__ __forceinline__ uint32_t fr_cands(const FrCells& c, uint64_t base, const FjWord (&x)[TAPE_ROUNDS], uint32_t h, RAgg* a) {
    uint32_t k = 0;
    *a = RAgg{0, 0};
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++)
        if ((h >> j & 1) && base + j < c.stop[x[j].r]) {
            k |= 1u << j;
            *a = agg_combine(*a, RAgg{1, base + j + 1});
        }
    return k;
}

// KR3: the candidates of each tile; c_lo / c_hi of every record: the in-tile prefix in front of its '[' / behind its
// last word
__global__ void __launch_bounds__(TAPE_THREADS) fr_count_kernel(const FrCells c, RAgg* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, false, true);
    RAgg a, total;
    const uint32_t k = fr_cands(c, base, x, h, &a);
    RAgg pre = block_exclusive_scan(a, total);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (base + j >= c.m.n) break;
        if (x[j].first) c.c_lo[x[j].r] = pre;
        if (k >> j & 1) pre = agg_combine(pre, RAgg{1, base + j + 1});
        if (x[j].last) c.c_hi[x[j].r] = pre;
    }
    if (threadIdx.x == 0) tile[blockIdx.x] = total;
}

// KR4: the successor check of every candidate and stop
__global__ void __launch_bounds__(TAPE_THREADS) fr_verify_kernel(const FrCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, false, true);
    RAgg a;
    const uint32_t k = fr_cands(c, base, x, h, &a);
    RLast total;
    RLast pre = agg_combine(RLast{tile_prefix(c.c_tile_pre, c.c_grp_pre, blockIdx.x).last}, block_exclusive_scan(RLast{a.last}, total));
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (!(h >> j & 1)) continue;
        if ((k >> j & 1) || base + j == c.stop[x[j].r]) {
            const uint64_t lo = x[j].s.lo, a0 = base + j - (x[j].i - lo);  // the record's first virtual word (its '[')
            if (pre.v > a0 ? fr_succ(c.t, pre.v - 1 - a0 + lo) != x[j].i : x[j].i != lo + 1) c.bad[x[j].r] = 1;
        }
        if (k >> j & 1) pre.v = base + j + 1;
    }
}

// Array.ForEach (parsed_array.go:45-56) over the array Tape[:hi] whose '[' is word lo, in one thread: its element
// count; with erow set it also writes each element's row there
__device__ uint64_t fr_walk(const TapeView& t, uint64_t lo, uint64_t hi, uint32_t* erow) {
    FindParams p;
    p.t = t;
    FdIt it{hi, lo + 1, 0, 0, 0};
    uint64_t n = 0;
    while (fd_advance(p, it) != 0) {
        if (erow) {
            erow[2 * n] = (uint32_t)(it.off - 1);
            erow[2 * n + 1] = (uint32_t)hi;
        }
        n++;
    }
    return n;
}

// the key at head k of an object Tape[:hi] passes ForEach's checks (parsed_object.go:150-163): a string with its value
// word and one more word in front of hi, whose bytes lie inside their buffer (*name, *len)
__device__ __forceinline__ bool fo_key(const TapeView& t, uint64_t k, uint64_t hi, const uint8_t** name, uint64_t* len) {
    const uint64_t w = t.tape[k];
    if ((w >> 56) != '"' || k + 2 >= hi) return false;
    *len = t.tape[k + 1];
    return tape_string(t, w, *len, name);
}
// the key is in onlyKeys, or onlyKeys is empty
__device__ __forceinline__ bool fo_match(const FrCells& c, const uint8_t* name, uint64_t len) {
    if (c.nkeys == 0) return true;
    for (uint32_t q = 0; q < c.nkeys; q++) {
        if (c.kseg[q].len != len) continue;
        const uint8_t* key = c.kbytes + c.kseg[q].off;
        uint64_t b = 0;
        while (b < len && name[b] == key[b]) b++;
        if (b == len) return true;
    }
    return false;
}

// Object.ForEach (parsed_object.go:142-186) over the object Tape[:hi] whose '{' is word lo, in one thread: its rows
// (the members fn is called for), and in *st FD_CORRUPT for its two errors ("unexpected name tag", "getting object
// name"), whose record keeps the rows in front of them; with erow set it also writes each row's (value head, hi), key
// head and key length
__device__ uint64_t fo_walk(const FrCells& c, uint64_t lo, uint64_t hi, uint32_t* erow, uint32_t* krow, uint64_t* klen,
                            uint32_t* st) {
    FindParams p;
    p.t = c.t;
    FdIt it{hi, lo + 1, 0, 0, 0};
    uint64_t n = 0;
    *st = FD_OK;
    for (;;) {
        const uint32_t typ = fd_advance(p, it);
        if (typ != 2 || it.off + 1 >= it.n) {
            if (typ != 0) *st = FD_CORRUPT;  // "object: unexpected name tag"
            return n;
        }
        const uint64_t k = it.off - 1, len = c.t.tape[it.off];
        const uint8_t* name;
        if (!tape_string(c.t, it.cur, len, &name)) {
            *st = FD_CORRUPT;  // "getting object name"
            return n;
        }
        const bool take = fo_match(c, name, len);
        if (fd_advance(p, it) == 0) return n;  // (a skipped value's Advance as well)
        if (!take) continue;
        if (erow) {
            erow[2 * n] = (uint32_t)(it.off - 1);
            erow[2 * n + 1] = (uint32_t)hi;
            krow[n] = (uint32_t)k;
            klen[n] = len;
        }
        n++;
        if (n == c.mkeys) return n;
    }
}

// KO1: each candidate's rank in its record gives its role: c.sel = the keys, the candidates of even rank
__global__ void __launch_bounds__(TAPE_THREADS) fo_role_kernel(const FrCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, false, true);
    RAgg a, total;
    const uint32_t k = fr_cands(c, base, x, h, &a);
    uint64_t g = agg_combine(tile_prefix(c.c_tile_pre, c.c_grp_pre, blockIdx.x), block_exclusive_scan(a, total)).n;
    uint32_t key = 0;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (!(k >> j & 1)) continue;
        const uint64_t a0 = base + j - (x[j].i - x[j].s.lo);  // the record's first virtual word (its '{')
        if (!((g++ - agg_combine(tile_prefix(c.c_tile_pre, c.c_grp_pre, a0 / TAPE_TILE), c.c_lo[x[j].r]).n) & 1)) key |= 1u << j;
    }
    c.sel[(uint64_t)blockIdx.x * TAPE_THREADS + threadIdx.x] = (uint8_t)key;
}

// KO2: a key failing ForEach's checks marks its record for the one-thread walk; a key whose value is a candidate and
// which onlyKeys takes is selected (c.sel, in place of KO1's keys), counted as KR3 counts (MSum)
__global__ void __launch_bounds__(TAPE_THREADS) fo_select_kernel(const FrCells c, MSum* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    const uint64_t t = (uint64_t)blockIdx.x * TAPE_THREADS + threadIdx.x;
    const uint32_t key = c.sel[t];
    uint64_t r[TAPE_ROUNDS];
    uint32_t sel = 0, first = 0, last = 0;
    FjWord x{0, 0, MjSpan{0, 0, 0}, false, false};
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        r[j] = 0;
        if (base + j >= c.m.n) continue;
        x = j && !x.last ? FjWord{x.r, x.i + 1, x.s, false, x.i + 2 == x.s.hi} : fj_at(c.m, base + j);
        r[j] = x.r;
        first |= (uint32_t)x.first << j;
        last |= (uint32_t)x.last << j;
        if (!(key >> j & 1)) continue;
        const uint8_t* name;
        uint64_t len;
        if (!fo_key(c.t, x.i, x.s.hi, &name, &len)) c.bad[x.r] = 1;
        else if (base + j + 2 < c.stop[x.r] && fo_match(c, name, len)) sel |= 1u << j;
    }
    MSum tot;
    MSum pre = block_exclusive_scan(MSum{(uint64_t)__popc(sel)}, tot);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (first >> j & 1) c.s_lo[r[j]] = pre;
        if (sel >> j & 1) pre.v++;
        if (last >> j & 1) c.s_hi[r[j]] = pre;
    }
    c.sel[t] = (uint8_t)sel;
    if (threadIdx.x == 0) tile[blockIdx.x] = tot;
}

// KR5: one thread per record; OBJ: its rows are its selected members (KO2), at most len(onlyKeys) of them
template <bool OBJ>
__global__ void __launch_bounds__(256) fr_finish_kernel(const FrCells c) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= c.m.rows) return;
    const uint64_t a = c.m.vstart(r), b = c.m.vstart(r + 1);
    c.serial[r] = 0;
    c.base[r] = 0;
    if (a == b) {  // no container: no rows
        c.E[r] = 0;
        return;
    }
    const uint64_t lo = (uint64_t)c.m.head[r], hi = lo + (b - a), s = c.stop[r];
    const FjEnds<RAgg> e = fj_ends<TAPE_TILE>(c.c_tile_pre, c.c_grp_pre, c.c_lo[r], c.c_hi[r], a, b);
    uint64_t n = e.hi.n - e.lo.n, first = e.lo.n;
    bool ok = !c.bad[r];
    if (s != FR_NO_STOP) ok = ok && (c.t.tape[lo + (s - a)] >> 56) != 'N';
    else ok = ok && (n ? fr_succ(c.t, e.hi.last - 1 - a + lo) >= hi : lo + 1 >= hi);
    if (OBJ) {
        const FjEnds<MSum> se = fj_ends<TAPE_TILE>(c.s_tile_pre, c.s_grp_pre, c.s_lo[r], c.s_hi[r], a, b);
        n = se.hi.v - se.lo.v;
        if (c.mkeys && n > c.mkeys) n = c.mkeys;  // ForEach returns at the len(onlyKeys)-th match
        first = se.lo.v;
    }
    if (!ok) {
        c.serial[r] = 1;
        atomicAdd(c.n_serial, 1ull);
        if (OBJ) {
            uint32_t st;
            n = fo_walk(c, lo, hi, nullptr, nullptr, nullptr, &st);
            c.st[r] = (uint8_t)st;
        } else {
            n = fr_walk(c.t, lo, hi, nullptr);
        }
    }
    c.E[r] = n;
    c.base[r] = first;
}

// KR6: each candidate of a verified record writes its row at the record's first row + its place among the candidates
__global__ void __launch_bounds__(TAPE_THREADS) fr_emit_kernel(const FrCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, false, true);
    RAgg a, total;
    const uint32_t k = fr_cands(c, base, x, h, &a);
    RAgg pre = agg_combine(tile_prefix(c.c_tile_pre, c.c_grp_pre, blockIdx.x), block_exclusive_scan(a, total));
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (!(k >> j & 1)) continue;
        const uint64_t r = x[j].r;
        if (!c.serial[r]) {
            const uint64_t q = c.E[r] + (pre.n - c.base[r]);
            c.erow[2 * q] = (uint32_t)x[j].i;
            c.erow[2 * q + 1] = (uint32_t)x[j].s.hi;
        }
        pre.n++;
    }
}

// KO3: each selected key of a verified record in front of its cut writes its row at the record's first row + its place
// among the record's selected keys: (value head, object end), its key head and key length
__global__ void __launch_bounds__(TAPE_THREADS) fo_emit_kernel(const FrCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    const uint32_t sel = c.sel[(uint64_t)blockIdx.x * TAPE_THREADS + threadIdx.x];
    MSum total;
    uint64_t g = tile_prefix(c.s_tile_pre, c.s_grp_pre, blockIdx.x).v + block_exclusive_scan(MSum{(uint64_t)__popc(sel)}, total).v;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (!(sel >> j & 1)) continue;
        const FjWord x = fj_at(c.m, base + j);
        const uint64_t r = x.r, rank = g++ - c.base[r];
        if (c.serial[r] || rank >= c.E[r + 1] - c.E[r]) continue;
        const uint64_t q = c.E[r] + rank;
        c.erow[2 * q] = (uint32_t)(x.i + 2);  // a verified key's successor: its value
        c.erow[2 * q + 1] = (uint32_t)x.s.hi;
        c.krow[q] = (uint32_t)x.i;
        c.klen[q] = c.t.tape[x.i + 1];
    }
}

// KR7: one thread per record walked by one thread
template <bool OBJ>
__global__ void __launch_bounds__(256) fr_serial_emit_kernel(const FrCells c) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= c.m.rows || !c.serial[r]) return;
    const uint64_t a = c.m.vstart(r), b = c.m.vstart(r + 1), lo = (uint64_t)c.m.head[r];
    if (OBJ) {
        uint32_t st;
        fo_walk(c, lo, lo + (b - a), c.erow + 2 * c.E[r], c.krow + c.E[r], c.klen + c.E[r], &st);
    } else {
        fr_walk(c.t, lo, lo + (b - a), c.erow + 2 * c.E[r]);
    }
}

// KR8: the record columns (status, rows' offsets) and the row columns (tag, head index) into the caller's buffers
__global__ void __launch_bounds__(256) fr_out_kernel(const uint64_t* tape, const uint8_t* st, const uint64_t* E, const uint32_t* erow,
                                                     uint64_t records, uint64_t rows, uint8_t* o_st, int64_t* o_off, uint8_t* o_tag,
                                                     int64_t* o_idx) {
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k < records) o_st[k] = st[k];
    if (k <= records) o_off[k] = (int64_t)E[k];
    if (k < rows) {
        const uint64_t h = erow[2 * k];
        o_tag[k] = (uint8_t)(tape[h] >> 56);
        o_idx[k] = (int64_t)h;
    }
}

// KO4: the key column: row k's key offset (KF4's scan of the key lengths) and its bytes (longer keys by the whole warp)
__global__ void __launch_bounds__(256) fo_keys_kernel(const TapeView t, const uint32_t* krow, const uint64_t* koff, uint64_t rows,
                                                      int64_t* o_off, uint8_t* o_bytes) {
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k <= rows) o_off[k] = (int64_t)koff[k];
    const uint8_t* s = nullptr;
    uint64_t copy = 0;
    uint8_t* d = o_bytes;
    if (k < rows) {
        d += koff[k];
        copy = koff[k + 1] - koff[k];
        s = tape_string_ptr(t, t.tape[krow[k]]);  // (checked by KO2 or fo_walk)
    }
    fd_copy(s, d, copy);
}

}  // namespace sj
