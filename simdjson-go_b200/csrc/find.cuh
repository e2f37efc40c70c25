// find.cuh -- ParsedJson.ForEach + Iter.FindElement + the typed accessors on the device: every root's value at each of
// a set of key paths, into typed columns in HBM.
//
// The reference's NDJSON workload (ndjson_test.go:294-315, benchmarks_test.go:104-157) is
//     pj.ForEach(func(i Iter) { e, err := i.FindElement(e, path...); e.Iter.Int() / Float() / StringBytes() ... })
// Each (path, row) cell here is a literal port of those functions (tests/find_oracle.py is the same port in Python):
//   ForEach / AdvanceIter / AdvanceInto   parsed_json.go:125-138, :291-347, :228-258
//   FindElement -> Object -> FindPath     parsed_json.go:833-864, :998-1018, parsed_object.go:256-316
//   Advance / calcNext                    parsed_json.go:196-223, :268-278
// with the tape length each of them would see (the slices Tape[:n] the reference takes) carried as `n`.  Every tape read
// is below that length, every string read inside msg_len / strings_len, and every step moves strictly forward (a nop
// of AdvanceInto / AdvanceIter skips at least one word, Advance's at least its own), so a malformed tape terminates.
//
// Rows are the roots in tape order: stage 2's root list for the tape the context just built, else KC1a / KC1b
// (tape.cuh), as for countWhere.
//   KF3 fd_walk         one thread per (path, row), path-major, the path's segments staged in shared memory; the cell's
//       status, tag, head index and converted value into scratch, a STRING or STRING_CVT cell's length into `slen`, a
//       JSON or list cell's tape words into `jlen`
//   (JSON paths: the passes of find_json.cuh write each JSON cell's text length into `slen`, `val` and its status;
//    list paths: those of find_list.cuh write each list cell's element count, byte length and status)
//   KF4 fd_len_reduce   per-tile sums of `slen` (scan_groups_kernel twice)
//   KF5 fd_emit         the columns into the caller's buffers: the variable-length columns' offsets from the scan, the
//       STRING bytes (strings longer than FD_SHORT by their whole warp) and STRING_CVT text, and the fixed-size columns
//       with the caller's row stride
//   (JSON paths: find_json.cuh's KJ6 writes the text behind KF5's offsets; list paths: find_list.cuh's KL6 the elements)
#pragma once
#include "common.cuh"
#include "fmt.h"
#include "tape.cuh"

namespace sj {

constexpr int FD_THREADS = 256;     // KF3
constexpr uint64_t FD_SHORT = 32;   // longer strings are copied by their whole warp

// cell status (SJ_FIND_*) and path kind (SJ_FIND_KIND_*)
enum : uint32_t { FD_OK = 0, FD_NOT_FOUND = 1, FD_NOT_OBJECT = 2, FD_CONVERT = 3, FD_CORRUPT = 4 };
enum : uint32_t {
    FD_ELEMENT = 0, FD_INT64 = 1, FD_UINT64 = 2, FD_FLOAT64 = 3, FD_BOOL = 4, FD_STRING = 5, FD_JSON = 7,
    FD_ARRAY_FLOAT64 = 8, FD_ARRAY_INT64 = 9, FD_ARRAY_UINT64 = 10, FD_ARRAY_STRING = 11, FD_ARRAY_STRING_CVT = 12,
    FD_STRING_CVT = 13
};
__host__ __device__ __forceinline__ bool fd_list_kind(uint32_t k) { return k >= FD_ARRAY_FLOAT64 && k <= FD_ARRAY_STRING_CVT; }
// a variable-length byte column: STRING, JSON, STRING_CVT and the string lists
__host__ __device__ __forceinline__ bool fd_var_kind(uint32_t k) {
    return k == FD_STRING || k == FD_JSON || k == FD_STRING_CVT || k == FD_ARRAY_STRING || k == FD_ARRAY_STRING_CVT;
}

struct FdPath {
    uint32_t seg0, nseg;  // its segments: segs[seg0 .. seg0 + nseg)
    uint32_t kind;
    uint32_t sidx;        // variable-length paths (fd_var_kind): index among them (their column)
    uint32_t jidx;        // JSON and list paths: index among them (their cells are word ranges)
    uint32_t lidx;        // list paths: index among them
};
struct FdSeg {
    uint32_t off, len;    // bytes [off, off + len) of the segment bytes
};

struct FindParams {
    TapeView t;
    TapeRows roots;          // one row per root; with element rows (find_rows.cuh) roots.n is their count
    const uint32_t* erow;    // element or member rows: (head, container end) of row r at 2r, 2r + 1
    uint32_t n_paths;
    const FdPath* paths;
    const FdSeg* segs;
    const uint8_t* seg_bytes;
    // scratch, one entry per cell (p * rows + r)
    uint8_t* st;
    uint8_t* tag;
    int64_t* idx;
    uint64_t* val;
    uint64_t* slen;          // variable-length cells: bytes of the string or text (0 unless OK), at sidx * rows + r
    uint64_t* jlen;          // JSON and list cells: tape words of the found element (0 unless found), at jidx * rows + r
    uint64_t* ecnt;          // list cells: elements (0 unless OK), at lidx * rows + r
    const uint32_t* krow;    // member rows (an object's members, find_rows.cuh): the key head of row r; else nullptr
};

// the Iter fields the walk uses (parsed_json.go:180-195); n = length of its restricted tape
struct FdIt {
    uint64_t n, off;
    int64_t add;
    uint64_t cur;
    uint32_t t;
};

__device__ __forceinline__ bool fd_scope_tag(uint32_t t) { return t == 'r' || t == '{' || t == '['; }
// TagToType (parsed_json.go:1152-1163): TypeNone = 0; only String (2) and Object (7) are told apart by the walk
__device__ __forceinline__ uint32_t fd_type(uint32_t t) {
    switch (t) {
    case '"': return 2;
    case 'l': return 3;
    case 'u': return 4;
    case 'd': return 5;
    case 'n': return 1;
    case 't': case 'f': return 6;
    case '{': return 7;
    case '[': return 8;
    case 'r': return 9;
    default: return 0;
    }
}

// calcNext, parsed_json.go:268-278
__device__ __forceinline__ void fd_calc_next(FdIt& it, bool into) {
    it.add = 0;
    if (tape_value_tag(it.t))
        it.add = 1;
    else if (!into && fd_scope_tag(it.t))
        it.add = (int64_t)it.cur - (int64_t)it.off;
}
__device__ __forceinline__ void fd_move_to_end(FdIt& it) {  // moveToEnd, parsed_json.go:260-264
    it.off = it.n;
    it.add = 0;
    it.t = 0;
}

// Advance, parsed_json.go:196-223: the type of the next element, 0 = TypeNone
__device__ uint32_t fd_advance(const FindParams& p, FdIt& it) {
    it.off += (uint64_t)it.add;
    for (;;) {
        if (it.off >= it.n) {
            it.add = 0;
            it.t = 0;
            return 0;
        }
        const uint64_t v = p.t.tape[it.off];
        it.t = (uint32_t)(v >> 56);
        it.off++;
        it.cur = v & TAPE_VALUE_MASK;
        if (it.t == 'N') {
            it.off += it.cur;
            continue;
        }
        break;
    }
    fd_calc_next(it, false);
    if (it.add < 0) {
        fd_move_to_end(it);
        return 0;
    }
    return fd_type(it.t);
}

// AdvanceInto, parsed_json.go:228-258: the tag, 0 = TagEnd
__device__ uint32_t fd_advance_into(const FindParams& p, FdIt& it) {
    it.off += (uint64_t)it.add;
    for (;;) {
        if (it.off >= it.n) {
            it.add = 0;
            it.t = 0;
            return 0;
        }
        const uint64_t v = p.t.tape[it.off];
        it.t = (uint32_t)(v >> 56);
        it.cur = v & TAPE_VALUE_MASK;
        if (it.t == 'N') {
            if (it.cur == 0) {
                fd_move_to_end(it);
                return 0;
            }
            it.off += it.cur;
            continue;
        }
        it.off++;
        break;
    }
    fd_calc_next(it, true);
    return it.t;  // (addNext < 0 cannot follow calcNext(true))
}

// AdvanceIter, parsed_json.go:291-347, into dst (which may be it): FD_OK with *typ set, FD_NOT_FOUND when the tape
// ended exactly (TypeNone, nil error: dst untouched), FD_CORRUPT for its errors
__device__ uint32_t fd_advance_iter(const FindParams& p, FdIt& it, FdIt& dst, uint32_t* typ) {
    it.off += (uint64_t)it.add;
    for (;;) {
        if (it.off == it.n) {
            it.add = 0;
            it.t = 0;
            return FD_NOT_FOUND;
        }
        if (it.off > it.n) return FD_CORRUPT;  // "offset bigger than tape"
        const uint64_t v = p.t.tape[it.off];
        it.cur = v & TAPE_VALUE_MASK;
        it.t = (uint32_t)(v >> 56);
        it.off++;
        if (it.t == 'N') {
            if (it.cur == 0) return FD_CORRUPT;  // "invalid nop skip"
            it.off += it.cur;
            continue;
        }
        break;
    }
    fd_calc_next(it, false);
    if (it.add < 0) {
        fd_move_to_end(it);
        return FD_CORRUPT;  // "element has negative offset"
    }
    const uint64_t end = it.off + (uint64_t)it.add;
    *typ = fd_type(it.t);
    if (&dst != &it) dst = it;
    fd_calc_next(dst, true);
    if (end > dst.n) return FD_CORRUPT;  // "element extends beyond tape"
    dst.n = end;
    return FD_OK;
}

// Object.FindPath, parsed_object.go:256-316, over the object Tape[:n] whose members start at off; path = nseg >= 1
// staged segments.  FD_OK: e is the element's Iter, or *fresh when AdvanceIter met the end exactly.
__device__ uint32_t fd_find_path(const FindParams& p, uint64_t n, uint64_t off, const FdSeg* seg, const uint8_t* bytes,
                                 uint32_t nseg, FdIt& e, bool* fresh) {
    FdIt tmp{n, off, 0, 0, 0};
    uint32_t k = 0;
    for (;;) {
        const uint32_t typ = fd_advance(p, tmp);
        if (typ != 2 || tmp.off + 1 >= tmp.n) return FD_NOT_FOUND;
        const uint64_t offset = tmp.cur, length = p.t.tape[tmp.off];
        const uint32_t klen = seg[k].len;
        if (length != klen) {
            if (fd_advance(p, tmp) == 0) return FD_NOT_FOUND;
            continue;
        }
        const uint8_t* name;
        if (!tape_string(p.t, offset, length, &name)) return FD_CORRUPT;
        const uint8_t* key = bytes + seg[k].off;
        bool eq = true;
        for (uint32_t j = 0; j < klen; j++)
            if (name[j] != key[j]) {
                eq = false;
                break;
            }
        if (!eq) {
            fd_advance(p, tmp);
            continue;
        }
        uint32_t t = 0;
        if (k + 1 == nseg) {
            const uint32_t rc = fd_advance_iter(p, tmp, e, &t);
            *fresh = rc == FD_NOT_FOUND;
            return rc == FD_CORRUPT ? FD_CORRUPT : FD_OK;
        }
        const uint32_t rc = fd_advance_iter(p, tmp, tmp, &t);
        if (rc == FD_CORRUPT) return FD_CORRUPT;
        if (rc == FD_NOT_FOUND || t != 7) return FD_NOT_OBJECT;  // "value of key %v is not an object"
        k++;
    }
}

// ForEach's element for the root at slot `root` (parsed_json.go:125-138) into cp; false when AdvanceIter fails (the
// root word is read: it never "ends")
__device__ __forceinline__ bool fd_root_elem(const FindParams& p, uint64_t root, FdIt& cp) {
    FdIt it{p.t.n, root, 0, 0, 0};
    uint32_t typ;
    if (fd_advance_iter(p, it, cp, &typ) != FD_OK) return false;
    fd_advance_into(p, cp);
    return true;
}

// FindElement (parsed_json.go:833-864) from the Iter cp, with Object (:998-1018) and Root (:804-824)
__device__ __forceinline__ uint32_t fd_find_element(const FindParams& p, FdIt cp, const FdSeg* seg, const uint8_t* bytes,
                                                    uint32_t nseg, FdIt& e, bool* fresh) {
    if (nseg == 0) return FD_NOT_FOUND;
    for (;;) {
        if (cp.t == '{') {
            const uint64_t end = cp.cur;
            if (end < cp.off || cp.n < end) return FD_CORRUPT;  // "object ends at index before start" / "beyond tape"
            return fd_find_path(p, end, cp.off, seg, bytes, nseg, e, fresh);
        }
        if (cp.t == 'r') {
            if (cp.cur > cp.n || cp.cur == 0) return FD_CORRUPT;  // "root element extends beyond tape" / Tape[:0-1]
            cp.add = 0;
            cp.n = cp.cur - 1;
            fd_advance_into(p, cp);
            continue;
        }
        if (cp.t == 0) {
            if (fd_advance_into(p, cp) == 0) return FD_NOT_FOUND;
            continue;
        }
        return FD_NOT_OBJECT;  // "type %q found before object was found"
    }
}

// ForEach's element for the root at slot `root`, then FindElement
__device__ uint32_t fd_find(const FindParams& p, uint64_t root, const FdSeg* seg, const uint8_t* bytes, uint32_t nseg,
                            FdIt& e, bool* fresh) {
    FdIt cp{0, 0, 0, 0, 0};
    if (!fd_root_elem(p, root, cp)) return FD_CORRUPT;
    return fd_find_element(p, cp, seg, bytes, nseg, e, fresh);
}

// int64(x) as amd64 lowers it (CVTTSD2SQ): NaN and anything outside int64 give 0x8000000000000000, where CUDA's
// __double2ll_rz saturates
__device__ __forceinline__ uint64_t fd_cvttsd2sq(double x) {
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return 0x8000000000000000ull;
    return (uint64_t)__double2ll_rz(x);
}

// StringCvt's text (parsed_json.go:775-799) of a scalar other than a string, from its tag and value word (the value
// Int / Uint / Float return for 'l' / 'u' / 'd'); W = false: the length only.  A 'd' must be finite.
template <bool W>
__device__ __forceinline__ uint32_t fd_cvt_text(uint32_t t, uint64_t pl, uint8_t* o) {
    const char* lit = t == 't' ? "true" : t == 'f' ? "false" : "null";
    if (t == 'l') return fmt_i64<W>((int64_t)pl, o);
    if (t == 'u') return fmt_u64<W>(pl, o);
    if (t == 'd') return fmt_double<W>(pl, o);
    const uint32_t n = t == 'f' ? 5 : 4;
    if (W)
        for (uint32_t k = 0; k < n; k++) o[k] = (uint8_t)lit[k];
    return n;
}
__device__ __forceinline__ bool fd_finite(uint64_t bits) { return (bits & 0x7ff0000000000000ull) != 0x7ff0000000000000ull; }

// the text of the scalar at head h, a cell of a byte column: a string's bytes are returned for the caller to copy;
// any other scalar's StringCvt text (at most 24 bytes) is written to d, and nullptr returned
__device__ __forceinline__ const uint8_t* fd_cell_text(const TapeView& t, uint64_t h, uint8_t* d) {
    const uint64_t w = t.tape[h];
    const uint32_t tag = (uint32_t)(w >> 56);
    if (tag == '"') return tape_string_ptr(t, w);
    fd_cvt_text<true>(tag, tape_value_tag(tag) ? t.tape[h + 1] : 0, d);
    return nullptr;
}

// Float / Int / Uint (kind FD_FLOAT64 / FD_INT64 / FD_UINT64) of a number with tag t ('d', 'l' or 'u') and value word
// pl: FD_OK with *v, or FD_CONVERT.  uint_max: Uint's float bound, 2^64 for Iter.Uint (parsed_json.go:679-712) but
// float64(MaxInt64) = 2^63 for Array.AsUint64 (parsed_array.go:231-283), so there floats above 2^63 fail.
__device__ __forceinline__ uint32_t fd_number(uint32_t t, uint64_t pl, uint32_t kind, double uint_max, uint64_t* v) {
    const double d = __longlong_as_double((long long)pl);
    if (kind == FD_FLOAT64) {  // Float, parsed_json.go:560-583
        *v = t == 'd' ? pl : (uint64_t)__double_as_longlong(t == 'l' ? __ll2double_rn((long long)pl) : __ull2double_rn(pl));
        return FD_OK;
    }
    if (kind == FD_INT64) {  // Int, parsed_json.go:629-661
        if (t == 'd') {
            // v > math.MaxInt64 compares against float64(MaxInt64) = 2^63, so exactly 2^63 passes and CVTTSD2SQ makes
            // it math.MinInt64 (as it does NaN)
            if (d > 9223372036854775808.0 || d < -9223372036854775808.0) return FD_CONVERT;  // "float value overflows / underflows int64"
            *v = fd_cvttsd2sq(d);
            return FD_OK;
        }
        if (t == 'u' && pl > 0x7fffffffffffffffull) return FD_CONVERT;  // "unsigned integer value overflows int64"
        *v = pl;
        return FD_OK;
    }
    // Uint
    if (t == 'd') {
        if (d > uint_max || d < 0) return FD_CONVERT;  // "float value overflows uint64" / "is negative"
        // uint64(v) as Go lowers it on amd64 (cmd/compile/internal/ssagen/ssa.go, float64ToUint64):
        //   v < 2^63 ? int64(v) : int64(v - 2^63) | 1<<63
        // so exactly 2^64 or 2^63 (and NaN) give 1<<63, where __double2ull_rz saturates
        *v = d < 9223372036854775808.0 ? fd_cvttsd2sq(d) : (fd_cvttsd2sq(d - 9223372036854775808.0) | 0x8000000000000000ull);
        return FD_OK;
    }
    if (t == 'l' && (pl >> 63)) return FD_CONVERT;  // "int64 value is negative"
    *v = pl;
    return FD_OK;
}

// the accessor of `kind` on the found element e: FD_OK with *val (and the string's bytes for STRING), or its error
__device__ uint32_t fd_convert(const FindParams& p, const FdIt& e, uint32_t kind, uint64_t* val, const uint8_t** s) {
    const uint32_t t = e.t;
    *val = 0;
    if (kind == FD_ELEMENT) return FD_OK;
    if (kind == FD_BOOL) {  // Bool, parsed_json.go:867-875
        if (t != 't' && t != 'f') return FD_CONVERT;
        *val = t == 't';
        return FD_OK;
    }
    if (kind == FD_STRING || (kind == FD_STRING_CVT && t == '"')) {  // StringBytes, parsed_json.go:741-749
        if (t != '"') return FD_CONVERT;
        if (e.off >= e.n) return FD_CORRUPT;
        const uint64_t len = p.t.tape[e.off];
        if (!tape_string(p.t, e.cur, len, s)) return FD_CORRUPT;
        *val = len;
        return FD_OK;
    }
    if (kind == FD_STRING_CVT) {  // StringCvt, parsed_json.go:775-799 (strings above): the text of Int / Uint / Float
        if (t == 't' || t == 'f' || t == 'n') {
            *val = fd_cvt_text<false>(t, 0, nullptr);
            return FD_OK;
        }
        if (t != 'd' && t != 'l' && t != 'u') return FD_CONVERT;  // "cannot convert type %s to string"
        if (e.off >= e.n) return FD_CORRUPT;                       // "... no more values on tape"
        const uint64_t pl = p.t.tape[e.off];  // Int of 'l', Uint of 'u' and Float of 'd' return it unchanged
        if (t == 'd' && !fd_finite(pl)) return FD_CONVERT;         // appendFloat: "INF or NaN number found"
        *val = fd_cvt_text<false>(t, pl, nullptr);
        return FD_OK;
    }
    if (t != 'd' && t != 'l' && t != 'u') return FD_CONVERT;  // "unable to convert type %v to ..."
    if (e.off >= e.n) return FD_CORRUPT;  // "corrupt input: expected ..., but no more values on tape"
    return fd_number(t, p.t.tape[e.off], kind, 18446744073709551616.0, val);
}

// KF3: one thread per cell, path-major (neighbouring threads take neighbouring rows of one path).  The block stages
// the segments of the paths its cells belong to: their descriptors, then their bytes.  ELEMS: the rows are array
// elements or an object's members (find_rows.cuh), each an Iter that ForEach's Advance left on the element's (the
// member value's) head, over the container's tape.
template <bool ELEMS>
__global__ void __launch_bounds__(FD_THREADS) fd_walk_kernel(const FindParams p) {
    extern __shared__ uint8_t fd_smem[];
    const uint64_t cells = p.roots.n * p.n_paths;
    const uint64_t q0 = (uint64_t)blockIdx.x * FD_THREADS;
    const uint32_t p0 = (uint32_t)(q0 / p.roots.n);
    const uint64_t qlast = min(q0 + FD_THREADS, cells) - 1;
    const uint32_t p1 = (uint32_t)(qlast / p.roots.n);
    const uint32_t s_lo = p.paths[p0].seg0, s_hi = p.paths[p1].seg0 + p.paths[p1].nseg;
    const uint32_t b_lo = s_lo < s_hi ? p.segs[s_lo].off : 0;
    const uint32_t b_hi = s_lo < s_hi ? p.segs[s_hi - 1].off + p.segs[s_hi - 1].len : 0;
    FdSeg* sseg = reinterpret_cast<FdSeg*>(fd_smem);
    uint8_t* sbytes = fd_smem + sizeof(FdSeg) * (s_hi - s_lo);
    for (uint32_t k = threadIdx.x; k < s_hi - s_lo; k += FD_THREADS)
        sseg[k] = FdSeg{p.segs[s_lo + k].off - b_lo, p.segs[s_lo + k].len};
    for (uint32_t k = threadIdx.x; k < b_hi - b_lo; k += FD_THREADS) sbytes[k] = p.seg_bytes[b_lo + k];
    __syncthreads();
    const uint64_t q = q0 + threadIdx.x;
    if (q >= cells) return;
    const uint32_t pi = (uint32_t)(q / p.roots.n);
    const uint64_t r = q - (uint64_t)pi * p.roots.n;
    const FdPath path = p.paths[pi];
    FdIt e{0, 0, 0, 0, 0};
    bool fresh = false;
    uint32_t st;
    if (ELEMS) {
        const uint64_t h = p.erow[2 * r], w = p.t.tape[h];
        FdIt cp{p.erow[2 * r + 1], h + 1, 0, w & TAPE_VALUE_MASK, (uint32_t)(w >> 56)};
        fd_calc_next(cp, false);
        if (path.nseg == 0 && p.krow) {  // a member's value: the element Object.FindPath returns when it stops at the
                                         // member's key (AdvanceIter from the key, parsed_object.go:298-303)
            FdIt k{cp.n, (uint64_t)p.krow[r] + 1, 1, 0, '"'};
            uint32_t t;
            st = fd_advance_iter(p, k, e, &t);
            fresh = st == FD_NOT_FOUND;
            if (fresh) st = FD_OK;
        } else {
            st = fd_find_element(p, cp, sseg + (path.seg0 - s_lo), sbytes, path.nseg, e, &fresh);
        }
    } else {
        st = fd_find(p, tape_root(p.roots, r), sseg + (path.seg0 - s_lo), sbytes, path.nseg, e, &fresh);
    }
    uint32_t tag = 0;
    int64_t idx = -1;
    uint64_t val = 0;
    const uint8_t* s = nullptr;
    uint64_t words = 0;
    if (st == FD_OK && fresh) {
        st = path.kind == FD_ELEMENT ? FD_OK : FD_CONVERT;  // a fresh Element: Type None, a zero Iter
    } else if (st == FD_OK) {
        tag = e.t;
        idx = (int64_t)e.off - 1;
        if (path.kind == FD_JSON) {
            words = e.n - (uint64_t)idx;  // MarshalJSON's scope: the element's restricted tape [head, n)
        } else if (fd_list_kind(path.kind)) {  // Iter.Array, parsed_json.go:1022-1039: the array's tape [head, cur)
            if (e.t != '[') st = FD_CONVERT;          // "next item is not array"
            else if (e.n < e.cur) st = FD_CORRUPT;    // "object extended beyond tape"
            else words = e.cur - (uint64_t)idx;
        } else {
            st = fd_convert(p, e, path.kind, &val, &s);
            if (st != FD_OK) val = 0;
        }
    }
    p.st[q] = (uint8_t)st;
    p.tag[q] = (uint8_t)tag;
    p.idx[q] = idx;
    p.val[q] = val;
    if (fd_var_kind(path.kind)) p.slen[(uint64_t)path.sidx * p.roots.n + r] = val;
    if (path.kind == FD_JSON || fd_list_kind(path.kind)) p.jlen[(uint64_t)path.jidx * p.roots.n + r] = words;
    if (fd_list_kind(path.kind)) p.ecnt[(uint64_t)path.lidx * p.roots.n + r] = 0;
}

// KF4: per-tile sums of slen
__global__ void __launch_bounds__(TAPE_THREADS) fd_len_reduce_kernel(const uint64_t* slen, uint64_t n, MSum* tile) {
    const uint64_t base = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)threadIdx.x;
    uint64_t k = 0;
#pragma unroll
    for (int j = 0; j < TAPE_ROUNDS; j++)
        if (base + (uint64_t)j * TAPE_THREADS < n) k += slen[base + (uint64_t)j * TAPE_THREADS];
    MSum total;
    block_exclusive_scan(MSum{k}, total);
    if (threadIdx.x == 0) tile[blockIdx.x] = total;
}

struct FindEmit {
    TapeView t;
    uint64_t rows, row_cap;
    uint32_t n_paths, n_str;
    uint32_t str_ntiles;
    uint8_t str_path[64];        // the path of every variable-length column
    uint64_t str_later;          // bit s: column s is a JSON or string list path's (its bytes come from KJ6 / KL6)
    const uint8_t* st;
    const uint8_t* tag;
    const int64_t* idx;
    const uint64_t* val;
    const uint64_t* slen;
    const MSum* slen_tile_pre;
    const MSum* slen_grp_pre;
    // the caller's columns
    uint8_t* o_st;
    uint8_t* o_tag;
    int64_t* o_idx;
    uint64_t* o_val;
    int64_t* o_off;              // [n_str][row_cap + 1]
    uint8_t* o_bytes;
};

// `copy` bytes from s to d (none when copy is 0): the whole warp calls it, and copies its strings longer than FD_SHORT
// together, lane by lane
__device__ __forceinline__ void fd_copy(const uint8_t* s, uint8_t* d, uint64_t copy) {
    const uint32_t lane = threadIdx.x & 31;
    if (copy <= FD_SHORT)
        for (uint64_t b = 0; b < copy; b++) d[b] = s[b];
    uint32_t m = __ballot_sync(FULL, copy > FD_SHORT);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint8_t* ws = reinterpret_cast<const uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(s), src));
        uint8_t* wd = reinterpret_cast<uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(d), src));
        const uint64_t wl = __shfl_sync(FULL, copy, src);
        for (uint64_t b = lane; b < wl; b += 32) wd[b] = ws[b];
    }
}

// KF5: blocks [0, str_ntiles) write the string offsets and bytes of TAPE_TILE string cells each; the blocks behind
// them copy TAPE_TILE cells each of the fixed-size columns to the caller's row stride
__global__ void __launch_bounds__(TAPE_THREADS) fd_emit_kernel(const FindEmit p) {
    if (blockIdx.x >= p.str_ntiles) {
        const uint64_t cells = p.rows * p.n_paths;
        for (int j = 0; j < TAPE_ROUNDS; j++) {
            const uint64_t q = (uint64_t)(blockIdx.x - p.str_ntiles) * TAPE_TILE + (uint64_t)j * TAPE_THREADS + threadIdx.x;
            if (q >= cells) break;
            const uint64_t pi = q / p.rows, r = q - pi * p.rows, o = pi * p.row_cap + r;
            p.o_st[o] = p.st[q];
            p.o_tag[o] = p.tag[q];
            p.o_idx[o] = p.idx[q];
            p.o_val[o] = p.val[q];
        }
        return;
    }
    const uint64_t n = p.rows * p.n_str;
    uint64_t carry = tile_prefix(p.slen_tile_pre, p.slen_grp_pre, blockIdx.x).v;
    for (int j = 0; j < TAPE_ROUNDS; j++) {
        const uint64_t k = (uint64_t)blockIdx.x * TAPE_TILE + (uint64_t)j * TAPE_THREADS + threadIdx.x;
        const uint64_t len = k < n ? p.slen[k] : 0;
        MSum total;
        const uint64_t off = carry + block_exclusive_scan(MSum{len}, total).v;
        carry += total.v;
        const uint8_t* s = nullptr;
        uint64_t copy = 0;  // bytes of a STRING or STRING_CVT cell's string
        uint8_t* d = p.o_bytes + off;
        if (k < n) {
            const uint64_t si = k / p.rows, r = k - si * p.rows;
            int64_t* col = p.o_off + si * (p.row_cap + 1);
            col[r] = (int64_t)off;
            if (r + 1 == p.rows) col[p.rows] = (int64_t)(off + len);
            if (len && !(p.str_later >> si & 1)) {  // an OK cell: a string whose range was checked by KF3, or a scalar
                s = fd_cell_text(p.t, (uint64_t)p.idx[(uint64_t)p.str_path[si] * p.rows + r], d);
                copy = s ? len : 0;
            }
        }
        fd_copy(s, d, copy);
    }
}

}  // namespace sj
