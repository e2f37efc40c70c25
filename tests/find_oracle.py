"""ParsedJson.ForEach + Iter.FindElement + the typed accessors, restated line by line over a tape.  Test infrastructure:
the expected output of the device find (find.cuh), cell for cell.

Each function below ports one function of the reference and names it with file:line.  Go's iterator state (off,
addNext, cur, t) and the length of the restricted tape (the slices `Tape[:n]` the reference takes) are carried as
plain integers; every error return, and every panic on a malformed tape, ends the cell with a status.

Rows are the root-open words of the tape (tag 'r', value > own index) that are not the value word of a string or
number, in tape order (roots()): on every tape the parser or Deserialize writes, the roots ForEach visits
(foreach_roots()).  Each row is the element ForEach hands its callback for that root.
"""
import math
import struct

import numpy as np

VAL = (1 << 56) - 1                 # JSONVALUEMASK, parsed_json.go:26
STRINGBUFBIT = 1 << 55              # parsed_json.go:29
STRINGBUFMASK = (1 << 55) - 1       # parsed_json.go:30
M64 = (1 << 64) - 1
MIN_INT64 = 1 << 63                 # the bits of math.MinInt64

# statuses of a cell
OK, NOT_FOUND, NOT_OBJECT, CONVERT, CORRUPT = range(5)
# kinds of a path: which accessor reads the found element
ELEMENT, INT64, UINT64, FLOAT64, BOOL, STRING = range(6)

TAG_END, TAG_NOP = 0, ord("N")
_VALUE_TAGS = {ord('"'), ord("l"), ord("u"), ord("d")}
_SCOPE_TAGS = {ord("r"), ord("{"), ord("[")}
# TagToType (parsed_json.go:1152-1163); every other tag is TypeNone
TYPE_NONE, TYPE_STRING, TYPE_OBJECT = 0, 2, 7
_TAG_TO_TYPE = {ord('"'): 2, ord("l"): 3, ord("u"): 4, ord("d"): 5, ord("n"): 1, ord("t"): 6, ord("f"): 6,
                ord("{"): 7, ord("["): 8, ord("r"): 9}


class _Fail(Exception):
    def __init__(self, status):
        self.status = status


class _It:
    """Iter (parsed_json.go:180-195): tape restricted to its first `n` words."""
    __slots__ = ("n", "off", "add", "cur", "t")

    def __init__(self, n, off=0):
        self.n, self.off, self.add, self.cur, self.t = n, off, 0, 0, TAG_END


def roots(tape):
    """the rows of a tape: the slots of the root-open words ('r' pointing forward) that are heads -- not the value word
    of the string or number in front of them, reading from word 0 -- in tape order.  On every tape the parser or
    Deserialize writes these are foreach_roots(); a number's value word that starts with the byte 'r' is no row."""
    t = np.asarray(tape, dtype=np.uint64)
    tags = (t >> np.uint64(56)).astype(np.int64)
    head = np.ones(t.size, dtype=bool)
    value = np.isin(tags, list(_VALUE_TAGS))
    # sequential: a head with a value tag makes the next word its value word; any other word makes the next a head
    h = True
    for i, v in enumerate(value.tolist()):
        head[i] = h
        h = not (h and v)
    idx = np.arange(t.size, dtype=np.uint64)
    return np.nonzero(head & (tags == ord("r")) & ((t & np.uint64(VAL)) > idx))[0]


def foreach_roots(tape):
    """the roots ForEach visits (parsed_json.go:125-138): AdvanceIter from slot 0, one root after the other, until the
    tape ends, an element is not a root, or AdvanceIter fails.  On a tape the parser wrote these are the rows the
    context's own root list gives, and roots()."""
    n, out, i = len(tape), [], 0
    while i < n:
        w = int(tape[i])
        t, v = w >> 56, w & VAL
        if t == TAG_NOP:
            if v == 0:
                break
            i += 1 + v
            continue
        if t != ord("r") or v <= i or v > n:
            break
        out.append(i)
        i = v
    return np.array(out, dtype=np.int64)


def _calc_next(it, into):
    """calcNext, parsed_json.go:268-278"""
    it.add = 0
    if it.t in _VALUE_TAGS:
        it.add = 1
    elif it.t in _SCOPE_TAGS and not into:
        it.add = it.cur - it.off


def _move_to_end(it):
    """moveToEnd, parsed_json.go:260-264"""
    it.off, it.add, it.t = it.n, 0, TAG_END


def _advance(tape, it):
    """Advance, parsed_json.go:196-223: the TypeNone / type of the next element on this level"""
    it.off += it.add
    while True:
        if it.off >= it.n:
            it.add, it.t = 0, TAG_END
            return TYPE_NONE
        v = int(tape[it.off])
        it.t = v >> 56
        it.off += 1
        it.cur = v & VAL
        if it.t == TAG_NOP:
            it.off += it.cur
            continue
        break
    _calc_next(it, False)
    if it.add < 0:
        _move_to_end(it)
        return TYPE_NONE
    return _TAG_TO_TYPE.get(it.t, TYPE_NONE)


def _advance_into(tape, it):
    """AdvanceInto, parsed_json.go:228-258"""
    it.off += it.add
    while True:
        if it.off >= it.n:
            it.add, it.t = 0, TAG_END
            return TAG_END
        v = int(tape[it.off])
        it.t = v >> 56
        it.cur = v & VAL
        if it.t == TAG_NOP:
            if it.cur <= 0:
                _move_to_end(it)
                return TAG_END
            it.off += it.cur
            continue
        it.off += 1
        break
    _calc_next(it, True)
    if it.add < 0:
        _move_to_end(it)
        return TAG_END
    return it.t


def _advance_iter(tape, it, dst):
    """AdvanceIter, parsed_json.go:291-347 (dst may be it).  Returns the type, or None when the tape ended exactly
    (TypeNone with a nil error: dst is left as it was).  Errors raise CORRUPT."""
    it.off += it.add
    while True:
        if it.off == it.n:
            it.add, it.t = 0, TAG_END
            return None
        if it.off > it.n:
            raise _Fail(CORRUPT)  # "offset bigger than tape"
        v = int(tape[it.off])
        it.cur = v & VAL
        it.t = v >> 56
        it.off += 1
        if it.t == TAG_NOP:
            if it.cur <= 0:
                raise _Fail(CORRUPT)  # "invalid nop skip"
            it.off += it.cur
            continue
        break
    _calc_next(it, False)
    if it.add < 0:
        _move_to_end(it)
        raise _Fail(CORRUPT)  # "element has negative offset"
    end = it.off + it.add
    typ = _TAG_TO_TYPE.get(it.t, TYPE_NONE)
    if dst is not it:
        dst.n, dst.off, dst.add, dst.cur, dst.t = it.n, it.off, it.add, it.cur, it.t
    _calc_next(dst, True)
    if end > dst.n:
        raise _Fail(CORRUPT)  # "element extends beyond tape"
    dst.n = end
    return typ


def _string_bytes(offset, length, strings, message):
    """stringByteAt, parsed_json.go:107-120 (a Go slice out of range is a panic: CORRUPT too)"""
    if offset & STRINGBUFBIT == 0:
        if offset + length > len(message):
            raise _Fail(CORRUPT)
        return bytes(message[offset:offset + length])
    offset &= STRINGBUFMASK
    if offset + length > len(strings):
        raise _Fail(CORRUPT)
    return bytes(strings[offset:offset + length])


def _find_path(tape, strings, message, n, off, path):
    """Object.FindPath, parsed_object.go:256-316, on the object `Tape[:n]` whose members start at `off`.  Returns the
    found element's Iter, or a fresh (zero) Iter when AdvanceIter met the end of the tape exactly."""
    tmp = _It(n, off)
    key, rest = path[0], list(path[1:])
    while True:
        typ = _advance(tape, tmp)
        if typ != TYPE_STRING or tmp.off + 1 >= tmp.n:
            raise _Fail(NOT_FOUND)
        offset, length = tmp.cur, int(tape[tmp.off])
        if length != len(key):
            if _advance(tape, tmp) == TYPE_NONE:
                raise _Fail(NOT_FOUND)
            continue
        if _string_bytes(offset, length, strings, message) != key:
            _advance(tape, tmp)
            continue
        if not rest:
            dst = _It(0)
            _advance_iter(tape, tmp, dst)
            return dst
        if _advance_iter(tape, tmp, tmp) != TYPE_OBJECT:
            raise _Fail(NOT_OBJECT)  # "value of key %v is not an object"
        key, rest = rest[0], rest[1:]


def _find_element(tape, strings, message, cp, path):
    """Iter.FindElement, parsed_json.go:833-864, with Iter.Object (:998-1018) and Iter.Root (:804-824)"""
    if not path:
        raise _Fail(NOT_FOUND)
    while True:
        if cp.t == ord("{"):
            end = cp.cur
            if end < cp.off or cp.n < end:
                raise _Fail(CORRUPT)  # "object ends at index before start" / "object extended beyond tape"
            return _find_path(tape, strings, message, end, cp.off, path)
        if cp.t == ord("r"):
            if cp.cur > cp.n or cp.cur == 0:
                raise _Fail(CORRUPT)  # "root element extends beyond tape" / Tape[:cur-1] with cur 0 panics
            cp.add, cp.n = 0, cp.cur - 1
            _advance_into(tape, cp)
            continue
        if cp.t == TAG_END:
            if _advance_into(tape, cp) == TAG_END:
                raise _Fail(NOT_FOUND)
            continue
        raise _Fail(NOT_OBJECT)  # "type %q found before object was found"


def _f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def _f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _cvttsd2sq(x):
    """int64(x) as amd64 lowers it (CVTTSD2SQ): truncation, and 0x8000000000000000 (the 'integer indefinite' value)
    for NaN and for anything outside int64"""
    if math.isnan(x) or not -2.0**63 <= x < 2.0**63:
        return MIN_INT64
    return int(x) & M64


def _convert(tape, strings, message, e, kind):
    """the accessor of `kind` on the found element's Iter: (value bits, or bytes for STRING)"""
    t = e.t
    if kind == ELEMENT:
        return 0
    if kind == BOOL:  # Bool, parsed_json.go:867-875
        if t == ord("t"):
            return 1
        if t == ord("f"):
            return 0
        raise _Fail(CONVERT)
    if kind == STRING:  # StringBytes, parsed_json.go:741-749
        if t != ord('"'):
            raise _Fail(CONVERT)
        if e.off >= e.n:
            raise _Fail(CORRUPT)
        return _string_bytes(e.cur, int(tape[e.off]), strings, message)
    if t not in (ord("d"), ord("l"), ord("u")):
        raise _Fail(CONVERT)  # "unable to convert type %v to ..."
    if e.off >= e.n:
        raise _Fail(CORRUPT)  # "corrupt input: expected ..., but no more values on tape"
    p = int(tape[e.off])
    if kind == FLOAT64:  # Float, parsed_json.go:560-583
        if t == ord("d"):
            return p
        return _f64_bits(float(p - (1 << 64) if t == ord("l") and p >> 63 else p))
    if kind == INT64:  # Int, parsed_json.go:629-661
        if t == ord("d"):
            v = _f64(p)
            if v > 2.0**63 or v < -2.0**63:  # v > math.MaxInt64 compares against float64(MaxInt64) = 2^63
                raise _Fail(CONVERT)
            return _cvttsd2sq(v)  # exactly 2^63 (and NaN) convert to math.MinInt64
        if t == ord("u") and p > (1 << 63) - 1:
            raise _Fail(CONVERT)
        return p
    # Uint, parsed_json.go:679-712
    if t == ord("d"):
        v = _f64(p)
        if v > 2.0**64 or v < 0:
            raise _Fail(CONVERT)
        # uint64(v) as Go lowers it on amd64 (cmd/compile/internal/ssagen/ssa.go, float64ToUint64):
        # v < 2^63 ? int64(v) : int64(v - 2^63) | 1<<63 -- so exactly 2^64 (and NaN) give 1<<63
        if v < 2.0**63:
            return _cvttsd2sq(v)
        return _cvttsd2sq(v - 2.0**63) | MIN_INT64
    if t == ord("l") and p >> 63:
        raise _Fail(CONVERT)
    return p


class Cell:
    __slots__ = ("status", "tag", "index", "value")

    def __init__(self, status, tag=0, index=-1, value=0):
        self.status, self.tag, self.index, self.value = status, tag, index, value

    def astuple(self):
        return self.status, self.tag, self.index, self.value

    def __repr__(self):
        return "Cell%r" % (self.astuple(),)


def find_cell(tape, strings, message, root, path, kind):
    """one (row, path) cell: ForEach's element for the root at slot `root`, FindElement(path...), then the accessor"""
    n = len(tape)
    # ForEach (parsed_json.go:125-138): AdvanceIter onto the root word, then AdvanceInto
    it = _It(n, root)
    elem = _It(0)
    try:
        _advance_iter(tape, it, elem)
        _advance_into(tape, elem)
        e = _find_element(tape, strings, message, elem, [bytes(s) for s in path])
        if e.t == TAG_END and e.n == 0:  # AdvanceIter met the end exactly: a fresh Element, Type None
            if kind == ELEMENT:
                return Cell(OK)
            return Cell(CONVERT)
        head = e.off - 1
        try:
            return Cell(OK, e.t, head, _convert(tape, strings, message, e, kind))
        except _Fail as f:
            return Cell(f.status, e.t, head, b"" if kind == STRING else 0)
    except _Fail as f:
        return Cell(f.status, value=b"" if kind == STRING else 0)


def find(tape, strings, message, paths, kinds, rows=None):
    """every cell, path-major: result[p][r] is the Cell of path p on row r; rows = the root slots (default roots())"""
    rs = roots(tape) if rows is None else rows
    return [[find_cell(tape, strings, message, int(r), path, kind) for r in rs] for path, kind in zip(paths, kinds)]
