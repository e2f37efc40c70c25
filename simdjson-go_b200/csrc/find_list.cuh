// find_list.cuh -- the list cells of the device find: Iter.Array (parsed_json.go:1022-1039) of every found element,
// then Array.AsFloat / AsInteger / AsUint64 / AsString / AsStringCvt (parsed_array.go:145-344), into one pool of
// elements (and, for the string lists, the variable-length byte columns STRING cells use).
//
// A list cell is the array's tape [head, head + len) (KF3, find.cuh), laid end to end per path in find_json.cuh's
// virtual word space (FjWords, KJ0's scan).  The work is spread over those words, not over cells: one cell may be nearly
// the whole tape.  Up to the element that stops it, each walk reads exactly the heads of that space after the '[':
// AsFloat / AsInteger / AsUint64 read a tag at every even offset from the word after '[', and AsString / AsStringCvt step
// with AdvanceIter, which up to the first nested scope or nop visits the heads of KJ1's segmented head scan.  So
// fl_step() judges every such head on its own, and the first one that stops the walk decides the cell:
//   KJ1 fj_heads_reduce  (string lists) the head scan of the path's words, as for JSON cells
//   KL2 fl_stop          the stopping heads put their word into the cell's stop with atomicMin (one atomic per cell,
//       warp and round): the cell's minimum is the word its walk stops on
//   KL3 fl_measure       (string lists) the elements and bytes of the heads in front of the stop, scanned in the tile;
//       a cell's first and last word record their in-tile prefixes
//   KL4 fl_finish        per cell: its status from the stop word, its element count (numeric lists: half the words in
//       front of the stop) and byte length into KF3's st / val / slen / ecnt.  A cell whose AdvanceIter walk stops on a
//       nop (only foreign or Deserialize'd tapes have them) is finished here serially, by one thread, from that word on.
//   (KF4 .. : the element counts' scan gives each list cell its first element in the pool)
//   KL5 fl_offsets       the list offsets into the caller's columns
//   KL6 fl_emit          after KF5: each element's value or byte length into the pool and a string list's bytes behind
//       KF5's offsets (strings longer than FD_SHORT by their whole warp); KL7 fl_serial_emit the elements behind a nop
#pragma once
#include "find.cuh"
#include "find_json.cuh"

namespace sj {

enum : uint32_t { FL_ELEM = 8, FL_NOP = 9 };  // fl_step: an element / a nop of the AdvanceIter walk (else a cell status)
constexpr uint64_t FL_NO_STOP = ~0ull;

__host__ __device__ __forceinline__ bool fl_numeric(uint32_t kind) { return kind <= FD_ARRAY_UINT64; }

// the walk of list kind `kind` at tape word i, a head it reads after the array's '[', with the array's tape ending at
// hi: FL_ELEM with the element in *v (its value bits, or its byte length for the string lists), or the status the walk
// stops on there, or FL_NOP for a nop word of the AdvanceIter walk
__device__ uint32_t fl_step(const TapeView& t, uint32_t kind, uint64_t i, uint64_t hi, uint64_t* v) {
    const uint64_t w = t.tape[i];
    const uint32_t tag = (uint32_t)(w >> 56);
    if (fl_numeric(kind)) {  // AsFloat / AsInteger / AsUint64, parsed_array.go:145-283
        if (tag == ']') return FD_OK;
        if (tag != 'd' && tag != 'l' && tag != 'u') return FD_CONVERT;  // "unable to convert type %v to ..." (nops too)
        if (i + 1 >= hi) return FD_CORRUPT;                                // "corrupt input: ... but no more values"
        const uint32_t k = kind == FD_ARRAY_FLOAT64 ? FD_FLOAT64 : kind == FD_ARRAY_INT64 ? FD_INT64 : FD_UINT64;
        // (AsUint64's float bound is float64(MaxInt64) = 2^63)
        return fd_number(tag, t.tape[i + 1], k, 9223372036854775808.0, v) == FD_OK ? FL_ELEM : FD_CONVERT;
    }
    // AsString / AsStringCvt, parsed_array.go:287-344: AdvanceIter (parsed_json.go:291-347), then String / StringCvt
    const uint64_t cur = w & TAPE_VALUE_MASK;
    if (tag == 'N') return FL_NOP;
    // a scope: "element has negative offset" / "element extends beyond tape", else it is no string / cannot convert
    if (fd_scope_tag(tag)) return (cur < i + 1 || cur > hi) ? FD_CORRUPT : FD_CONVERT;
    if (fd_type(tag) == 0) return FD_OK;                       // TypeNone (']', or any unknown tag) ends the list
    if (tape_value_tag(tag) && i + 2 > hi) return FD_CORRUPT;  // "element extends beyond tape"
    if (tag == '"') {
        const uint64_t len = t.tape[i + 1];
        const uint8_t* s;
        if (!tape_string(t, w, len, &s)) return FD_CORRUPT;
        *v = len;
        return FL_ELEM;
    }
    if (kind == FD_ARRAY_STRING) return FD_CONVERT;  // "element in array is not string"
    const uint64_t pl = tape_value_tag(tag) ? t.tape[i + 1] : 0;
    if (tag == 'd' && !fd_finite(pl)) return FD_CONVERT;  // appendFloat: "INF or NaN number found"
    *v = fd_cvt_text<false>(tag, pl, nullptr);
    return FL_ELEM;
}

// the (bytes, elements) of a run of words
struct LSum {
    uint64_t bytes, elems;
};
__device__ __forceinline__ LSum agg_combine(const LSum& a, const LSum& b) { return LSum{a.bytes + b.bytes, a.elems + b.elems}; }
__device__ __forceinline__ LSum agg_shfl_up(const LSum& a, int d) {
    return LSum{__shfl_up_sync(FULL, a.bytes, d), __shfl_up_sync(FULL, a.elems, d)};
}

// list path l's cells
struct FlCells {
    FjWords m;
    TapeView t;
    uint32_t kind, path, sidx, lidx;
    const FjAgg* h_tile_pre;  // string lists: KJ1's scan
    const FjAgg* h_grp_pre;
    uint64_t* stop;           // [rows]: the virtual word each walk stops on, FL_NO_STOP for none
    const LSum* l_tile_pre;   // string lists: KL3's scan
    const LSum* l_grp_pre;
    LSum* c_lo;               // [rows]: KL3's in-tile prefixes in front of a cell's first word / behind its last
    LSum* c_hi;
    LSum* base;               // [rows]: KL3's scan in front of each cell
    LSum* pre;                // [rows]: each cell's elements and bytes in front of its stop
};

// this thread's TAPE_ROUNDS words from `base` on: their places, and which are heads the walk reads (bit j; a cell's
// '[' is none).  The whole block calls it.
__device__ __forceinline__ uint32_t fl_heads(const FlCells& c, uint64_t base, FjWord (&x)[TAPE_ROUNDS]) {
    return fj_heads(c.m, c.h_tile_pre, c.h_grp_pre, base, x, fl_numeric(c.kind), false);
}

// KL2: every head that stops its walk lowers the cell's stop to its word (stop preset to FL_NO_STOP)
__global__ void __launch_bounds__(TAPE_THREADS) fl_stop_kernel(const FlCells c) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fl_heads(c, base, x);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        uint64_t v;
        fj_lower_stop(c.stop, (h >> j & 1) && fl_step(c.t, c.kind, x[j].i, x[j].s.hi, &v) != FL_ELEM, x[j].r, base + j);
    }
}

// the elements (and bytes) of this thread's heads in front of their cell's stop, with each one's value in v[j]
__device__ __forceinline__ LSum fl_elems(const FlCells& c, uint64_t base, uint32_t h, const FjWord (&x)[TAPE_ROUNDS],
                                         uint64_t (&v)[TAPE_ROUNDS], uint32_t* el) {
    LSum s{0, 0};
    *el = 0;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        v[j] = 0;
        if ((h >> j & 1) && base + j < c.stop[x[j].r]) {  // every head in front of the stop is an element
            fl_step(c.t, c.kind, x[j].i, x[j].s.hi, &v[j]);
            *el |= 1u << j;
            s = agg_combine(s, LSum{fl_numeric(c.kind) ? 0 : v[j], 1});
        }
    }
    return s;
}

// KL3 (string lists): c_lo / c_hi of every cell, the tile's totals
__global__ void __launch_bounds__(TAPE_THREADS) fl_measure_kernel(const FlCells c, LSum* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fl_heads(c, base, x);
    uint64_t v[TAPE_ROUNDS];
    uint32_t el;
    LSum total;
    LSum e = block_exclusive_scan(fl_elems(c, base, h, x, v, &el), total);
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        if (base + j >= c.m.n) break;
        if (x[j].first) c.c_lo[x[j].r] = e;
        if (el >> j & 1) e = agg_combine(e, LSum{v[j], 1});
        if (x[j].last) c.c_hi[x[j].r] = e;
    }
    if (threadIdx.x == 0) tile[blockIdx.x] = total;
}

// the AdvanceIter walk of a string list from the nop at word i on, in one thread: the status it ends with, and the
// elements and bytes it adds to *n; with elems set it also writes them (element k at elems[k], its bytes at bytes + the
// bytes in front of it)
__device__ uint32_t fl_walk(const FindParams& p, uint32_t kind, uint64_t i, uint64_t hi, LSum* n, uint64_t* elems, uint8_t* bytes) {
    FdIt it{hi, i, 0, 0, 0}, el{0, 0, 0, 0, 0};
    for (;;) {
        uint32_t typ = 0;
        const uint32_t rc = fd_advance_iter(p, it, el, &typ);
        if (rc == FD_CORRUPT) return FD_CORRUPT;
        if (rc == FD_NOT_FOUND) return FD_OK;  // the array's tape ended exactly: TypeNone
        const uint64_t at = el.off - 1;
        uint64_t v;
        const uint32_t st = fl_step(p.t, kind, at, hi, &v);  // (AdvanceIter made the same checks of a scope's link)
        if (st != FL_ELEM) return st;
        if (elems) {
            elems[n->elems] = v;
            const uint8_t* s = fd_cell_text(p.t, at, bytes + n->bytes);
            if (s)
                for (uint64_t b = 0; b < v; b++) bytes[n->bytes + b] = s[b];
        }
        n->elems++;
        n->bytes += v;
    }
}

// KL4: one thread per row of the path
__global__ void __launch_bounds__(256) fl_finish_kernel(const FlCells c, FindParams p) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= c.m.rows) return;
    const uint64_t a = c.m.vstart(r), b = c.m.vstart(r + 1);
    if (a == b) return;  // no array: KF3's status, no elements and no bytes stand
    const uint64_t lo = (uint64_t)c.m.head[r], hi = lo + (b - a), s = c.stop[r];
    uint32_t st;
    uint64_t v;
    if (s == FL_NO_STOP)  // AsFloat & co. read past the array's tape (a panic); AdvanceIter met its end (TypeNone)
        st = fl_numeric(c.kind) ? FD_CORRUPT : FD_OK;
    else
        st = fl_step(c.t, c.kind, lo + (s - a), hi, &v);
    LSum n{0, 0};
    if (fl_numeric(c.kind)) {
        if (s != FL_NO_STOP) n.elems = (s - a - 1) / 2;
    } else {
        const FjEnds<LSum> e = fj_ends<TAPE_TILE>(c.l_tile_pre, c.l_grp_pre, c.c_lo[r], c.c_hi[r], a, b);
        n = LSum{e.hi.bytes - e.lo.bytes, e.hi.elems - e.lo.elems};
        c.base[r] = e.lo;
        c.pre[r] = n;
        if (st == FL_NOP) st = fl_walk(p, c.kind, lo + (s - a), hi, &n, nullptr, nullptr);
    }
    if (st != FD_OK) n = LSum{0, 0};
    const uint64_t q = (uint64_t)c.path * p.roots.n + r;
    p.st[q] = (uint8_t)st;
    p.val[q] = n.elems;
    if (!fl_numeric(c.kind)) p.slen[(uint64_t)c.sidx * p.roots.n + r] = n.bytes;
    p.ecnt[(uint64_t)c.lidx * p.roots.n + r] = n.elems;
}

// KL5: E = the exclusive scan of the element counts of all list cells (lidx-major) and their total; list path l's
// offsets column at o + l * (row_cap + 1)
__global__ void __launch_bounds__(256) fl_offsets_kernel(const uint64_t* E, uint64_t rows, uint32_t nl, int64_t* o, uint64_t row_cap) {
    const uint64_t k = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= rows * nl) return;
    const uint64_t l = k / rows, r = k - l * rows;
    o[l * (row_cap + 1) + r] = (int64_t)E[k];
    if (r + 1 == rows) o[l * (row_cap + 1) + rows] = (int64_t)E[k + 1];
}

// KL6: the elements of the OK cells in front of their stops: values or byte lengths at E[cell] + their index in the
// cell, a string list's bytes at its column offset (col) + their place in the row
__global__ void __launch_bounds__(TAPE_THREADS) fl_emit_kernel(const FlCells c, const uint8_t* st, const uint64_t* E, uint64_t* elems,
                                                              const int64_t* col, uint8_t* bytes) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x * TAPE_ROUNDS;
    FjWord x[TAPE_ROUNDS];
    const uint32_t h = fl_heads(c, base, x);
    uint64_t v[TAPE_ROUNDS];
    uint32_t el;
    const LSum mine = fl_elems(c, base, h, x, v, &el);
    const bool num = fl_numeric(c.kind);
    LSum e{0, 0};
    if (!num) {
        LSum total;
        e = agg_combine(tile_prefix(c.l_tile_pre, c.l_grp_pre, blockIdx.x), block_exclusive_scan(mine, total));
    }
    const uint64_t rows = c.m.rows;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        const uint8_t* s = nullptr;
        uint64_t copy = 0;
        uint8_t* d = bytes;
        if ((el >> j & 1) && st[(uint64_t)c.path * rows + x[j].r] == FD_OK) {
            const uint64_t r = x[j].r;
            const uint64_t k = num ? (x[j].i - x[j].s.lo - 1) / 2 : e.elems - c.base[r].elems;
            elems[E[(uint64_t)c.lidx * rows + r] + k] = v[j];
            if (!num) {
                d = bytes + (uint64_t)col[r] + (e.bytes - c.base[r].bytes);
                s = fd_cell_text(c.t, x[j].i, d);
                copy = s ? v[j] : 0;
            }
        }
        if (!num) {
            fd_copy(s, d, copy);
            if (el >> j & 1) e = agg_combine(e, LSum{v[j], 1});
        }
    }
}

// KL7 (string lists): one thread per row; an OK cell whose walk stopped on a nop writes the elements from it on
__global__ void __launch_bounds__(256) fl_serial_emit_kernel(const FlCells c, const FindParams p, const uint64_t* E, uint64_t* elems,
                                                             const int64_t* col, uint8_t* bytes) {
    const uint64_t r = (uint64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= c.m.rows || p.st[(uint64_t)c.path * c.m.rows + r] != FD_OK) return;
    const uint64_t a = c.m.vstart(r), b = c.m.vstart(r + 1), s = c.stop[r];
    if (a == b || s == FL_NO_STOP) return;
    const uint64_t lo = (uint64_t)c.m.head[r], i = lo + (s - a);
    if ((c.t.tape[i] >> 56) != 'N') return;
    LSum n = c.pre[r];
    fl_walk(p, c.kind, i, lo + (b - a), &n, elems + E[(uint64_t)c.lidx * c.m.rows + r], bytes + (uint64_t)col[r]);
}

}  // namespace sj
