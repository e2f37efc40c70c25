"""The find's list cells restated over a tape: Iter.Array of the element that ForEach + FindElement finds
(tests/find_oracle.py), then Array.AsFloat / AsInteger / AsUint64 / AsString / AsStringCvt, and Iter.StringCvt for
STRING_CVT cells.  Test infrastructure: the expected output of the device's list cells (find_list.cuh), cell for cell.

Each function ports one function of the reference line by line and names it with file:line.  Every error return ends
the cell with CONVERT or CORRUPT as the header sorts them, and a Go panic (an index out of range) with CORRUPT.

A list cell's value is (elements, bytes): the elements as uint64 bits (int64 / uint64 / float64 bits, or for the
string lists each element's byte length) and, for the string lists and STRING_CVT, the bytes of its text."""
import math

from tests.find_oracle import (CONVERT, CORRUPT, MIN_INT64, OK, TAG_END, TYPE_NONE, TYPE_STRING, VAL, Cell,
                               _advance_into, _advance_iter, _cvttsd2sq, _f64, _f64_bits, _Fail, _find_element, _It,
                               _string_bytes, find_cell, roots)

ARRAY_FLOAT64, ARRAY_INT64, ARRAY_UINT64, ARRAY_STRING, ARRAY_STRING_CVT, STRING_CVT = range(8, 14)
LIST_KINDS = (ARRAY_FLOAT64, ARRAY_INT64, ARRAY_UINT64, ARRAY_STRING, ARRAY_STRING_CVT)
STRING_LISTS = (ARRAY_STRING, ARRAY_STRING_CVT)
M64 = (1 << 64) - 1
MAX_INT64 = (1 << 63) - 1


def _read(tape, n, off):
    """Tape[off] of a tape restricted to n words: past it Go panics"""
    if off >= n:
        raise _Fail(CORRUPT)
    return int(tape[off])


def _array(e):
    """Iter.Array, parsed_json.go:1022-1039: (n, off) of the Array"""
    if e.t != ord("["):
        raise _Fail(CONVERT)  # "next item is not array"
    end = e.cur
    if e.n < end:
        raise _Fail(CORRUPT)  # "corrupt input: object extended beyond tape"
    return end, e.off


def _as_numbers(tape, n, off, kind):
    """Array.AsFloat / AsInteger / AsUint64, parsed_array.go:145-283: a tag word, its value word, the next tag word ..."""
    dst = []
    while True:
        tag = _read(tape, n, off) >> 56
        off += 1
        if tag == ord("]"):  # TagArrayEnd: break readArray
            return dst
        if tag not in (ord("d"), ord("l"), ord("u")):
            raise _Fail(CONVERT)  # "unable to convert type %v to float / integer"
        if n <= off:
            raise _Fail(CORRUPT)  # "corrupt input: expected float / integer, but no more values"
        p = int(tape[off])
        if kind == ARRAY_FLOAT64:  # :157-172
            if tag == ord("d"):
                dst.append(p)
            elif tag == ord("l"):
                dst.append(_f64_bits(float(p - (1 << 64) if p >> 63 else p)))  # float64(int64(x)), round to nearest
            else:
                dst.append(_f64_bits(float(p)))
        elif kind == ARRAY_INT64:  # :197-224
            if tag == ord("d"):
                v = _f64(p)
                if v > 2.0**63:  # val > math.MaxInt64 compares against float64(MaxInt64) = 2^63
                    raise _Fail(CONVERT)  # "float value overflows int64"
                if v < -2.0**63:
                    raise _Fail(CONVERT)  # "float value underflows int64"
                dst.append(_cvttsd2sq(v))  # int64(val): exactly 2^63 (and NaN) give math.MinInt64
            elif tag == ord("l"):
                dst.append(p)
            else:
                if p > MAX_INT64:
                    raise _Fail(CONVERT)  # "unsigned integer value overflows int64"
                dst.append(p)
        else:  # AsUint64, :248-275
            if tag == ord("d"):
                v = _f64(p)
                if v > 2.0**63:  # val > math.MaxInt64: floats above 2^63 fail, unlike Iter.Uint
                    raise _Fail(CONVERT)  # "float value overflows uint64"
                if v < 0:
                    raise _Fail(CONVERT)  # "float value is negative"
                # uint64(val) as amd64 Go lowers it: v < 2^63 ? int64(v) : int64(v - 2^63) | 1<<63 (NaN: 1<<63)
                dst.append(_cvttsd2sq(v) if v < 2.0**63 else _cvttsd2sq(v - 2.0**63) | MIN_INT64)
            elif tag == ord("l"):
                if p >> 63:
                    raise _Fail(CONVERT)  # "int64 value is negative"
                dst.append(p)
            else:
                dst.append(p)
        off += 1


def append_float(bits):
    """appendFloat, parsed_json.go:1250-1272 (floatToString :1243-1247)"""
    from tests.marshal_oracle import MalformedTape, format_float
    try:
        return format_float(_f64(bits))
    except MalformedTape:
        raise _Fail(CONVERT)  # "INF or NaN number found"


def string_cvt(tape, strings, message, it):
    """Iter.StringCvt, parsed_json.go:775-799, on an element's Iter: its text"""
    t = it.t
    if t == ord('"'):  # String, :729-738
        if it.off >= it.n:
            raise _Fail(CORRUPT)  # "corrupt input: no string offset"
        return _string_bytes(it.cur, int(tape[it.off]), strings, message)
    if t in (ord("l"), ord("u"), ord("d")):
        if it.off >= it.n:  # Int / Uint / Float: "corrupt input: expected ..., but no more values"
            raise _Fail(CORRUPT)
        p = int(tape[it.off])
        if t == ord("l"):
            return str(p - (1 << 64) if p >> 63 else p).encode()  # strconv.FormatInt
        if t == ord("u"):
            return str(p).encode()  # strconv.FormatUint
        return append_float(p)
    if t == ord("f"):
        return b"false"
    if t == ord("t"):
        return b"true"
    if t == ord("n"):
        return b"null"
    raise _Fail(CONVERT)  # "cannot convert type %s to string"


def _as_strings(tape, strings, message, n, off, kind):
    """Array.AsString / AsStringCvt, parsed_array.go:287-344: AdvanceIter over the Array's Iter (:37-43)"""
    i = _It(n, off)
    elem = _It(0)
    dst = []
    while True:
        t = _advance_iter(tape, i, elem)  # its errors raise CORRUPT
        if t is None or t == TYPE_NONE:
            return dst
        if kind == ARRAY_STRING:
            if t != TYPE_STRING:
                raise _Fail(CONVERT)  # "element in array is not string"
            dst.append(string_cvt(tape, strings, message, elem))  # elem.String()
        else:
            dst.append(string_cvt(tape, strings, message, elem))


def list_cell(tape, strings, message, root, path, kind):
    """one list or STRING_CVT cell: FindElement(path...) as find_cell, then Iter.Array and the accessor (or
    StringCvt).  Returns (Cell, elements, bytes): a list cell's Cell value is its element count, a STRING_CVT cell's
    its byte length; a cell that is not OK has no elements and no bytes."""
    it = _It(len(tape), root)
    elem = _It(0)
    try:
        _advance_iter(tape, it, elem)
        _advance_into(tape, elem)
        e = _find_element(tape, strings, message, elem, [bytes(s) for s in path])
    except _Fail as f:
        return Cell(f.status), [], b""
    if e.t == TAG_END and e.n == 0:  # a fresh Element
        return Cell(CONVERT), [], b""
    head = e.off - 1
    try:
        if kind == STRING_CVT:
            b = string_cvt(tape, strings, message, e)
            return Cell(OK, e.t, head, len(b)), [], b
        n, off = _array(e)
        if kind in STRING_LISTS:
            xs = _as_strings(tape, strings, message, n, off, kind)
            return Cell(OK, e.t, head, len(xs)), [len(x) for x in xs], b"".join(xs)
        xs = _as_numbers(tape, n, off, kind)
        return Cell(OK, e.t, head, len(xs)), [x & M64 for x in xs], b""
    except _Fail as f:
        return Cell(f.status, e.t, head, 0), [], b""


def find_lists(tape, strings, message, paths, kinds, rows=None):
    """every cell, path-major, as find(): a list or STRING_CVT path's cells are list_cell's triples, the others
    find_cell's Cells"""
    rs = roots(tape) if rows is None else rows
    return [[list_cell(tape, strings, message, int(r), path, kind) if kind in LIST_KINDS or kind == STRING_CVT else
             find_cell(tape, strings, message, int(r), path, kind) for r in rs] for path, kind in zip(paths, kinds)]
