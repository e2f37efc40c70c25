"""The find's JSON cells (SJ_FIND_KIND_JSON) restated over a tape: Element.Iter.MarshalJSON() of the element that
ForEach + FindElement finds (tests/find_oracle.py).  Test infrastructure: the expected output of the device's JSON cells
(find_json.cuh), cell for cell.

marshal_json_buffer ports MarshalJSONBuffer line by line over the element's Iter, with file:line notes like the rest of
the port; subtree_ok restates the checks the device applies to a cell's sub-tree alone, which decide OK / CORRUPT."""
from tests.find_oracle import (CONVERT, CORRUPT, OK, TAG_END, TAG_NOP, VAL, _VALUE_TAGS, Cell, _advance_into,
                               _advance_iter, _f64, _Fail, _find_element, _It, _string_bytes, find_cell, roots)

JSON = 7  # SJ_FIND_KIND_JSON (6 is no kind)


def _peek_next_tag(tape, it):
    """PeekNextTag, parsed_json.go:373-391, on the Iter's restricted tape"""
    off = it.off + it.add
    while True:
        if off >= it.n:
            return TAG_END
        v = int(tape[off])
        t = v >> 56
        if t == TAG_NOP:
            skip = v & VAL
            if skip <= 0:
                return TAG_END
            off += skip
            continue
        return t


class MarshalError(Exception):
    pass


def marshal_json_buffer(tape, strings, message, it):
    """Iter.MarshalJSONBuffer, parsed_json.go:401-556, on the element's Iter.  Returns the text; every error return of the
    reference (and a panic of its accessors) raises MarshalError."""
    from tests.marshal_oracle import MalformedTape, escape, format_float
    NONE_, ARRAY, OBJECT, ROOT = range(4)  # :408-413
    stack = [NONE_]  # :405-407
    dst = bytearray()

    def string_bytes():  # StringBytes, :741-749
        if it.t != ord('"') or it.off >= it.n:
            raise MarshalError("expected string")
        try:
            return _string_bytes(it.cur, int(tape[it.off]), strings, message)
        except _Fail:
            raise MarshalError("string out of range")

    def payload():  # Int / Uint / Float on their own tag, :560-712
        if it.off >= it.n:
            raise MarshalError("no more values on tape")
        return int(tape[it.off])

    while True:  # writeloop, :415
        if stack[-1] == OBJECT and it.t != ord("}"):  # :417-429
            sb = string_bytes()
            dst += b'"' + escape(sb) + b'":'
            if _peek_next_tag(tape, it) == TAG_END:
                raise MarshalError("unexpected end of tape within object")
            _advance_into(tape, it)
        t = it.t
        if t == ord("r"):  # :433-459
            is_open = it.cur > it.off
            if len(stack) > 1:
                if is_open:
                    raise MarshalError("root tag open, but not at top of stack")
                if stack[-1] == ROOT:
                    if _peek_next_tag(tape, it) != TAG_END:
                        dst += b"\n"
                    stack.pop()
                    t = None  # break tagswitch
                elif stack[-1] == NONE_:
                    break
                else:
                    raise MarshalError("root tag, but not at top of stack")
            if t is not None:
                if is_open:
                    it.add = 0
                _advance_into(tape, it)
                stack.append(ROOT)
                continue
        elif t == ord('"'):  # :460-468
            dst += b'"' + escape(string_bytes()) + b'"'
        elif t == ord("l"):  # :469-474
            p = payload()
            dst += b"%d" % (p - (1 << 64) if p >> 63 else p)
        elif t == ord("u"):  # :475-480
            dst += b"%d" % payload()
        elif t == ord("d"):  # :481-490
            try:
                dst += format_float(_f64(payload()))
            except MalformedTape:
                raise MarshalError("INF or NaN number found")
        elif t == ord("n"):
            dst += b"null"
        elif t == ord("t"):
            dst += b"true"
        elif t == ord("f"):
            dst += b"false"
        elif t in (ord("{"), ord("[")):  # :497-501, :509-513
            dst += bytes([t])
            stack.append(OBJECT if t == ord("{") else ARRAY)
            _advance_into(tape, it)
            continue
        elif t in (ord("}"), ord("]")):  # :502-508, :514-520
            dst += bytes([t])
            if stack[-1] != (OBJECT if t == ord("}") else ARRAY):
                raise MarshalError("end of container with no container on stack")
            stack.pop()
        elif t == TAG_END:  # :521-526
            if _peek_next_tag(tape, it) == TAG_END:
                raise MarshalError("no content queued in iterator")
            _advance_into(tape, it)
            continue
        if _peek_next_tag(tape, it) == TAG_END:  # :529-532
            break
        _advance_into(tape, it)
        if stack[-1] in (ARRAY, OBJECT) and it.t not in (ord("]"), ord("}")):  # :534-549
            dst += b","
    if len(stack) > 1:  # :550-554
        raise MarshalError("objects or arrays not closed")
    return bytes(dst)


def subtree_ok(tape, strings, message, lo, hi):
    """the checks of the device marshal (marshal.cuh) on the sub-tree [lo, hi) alone: one value from lo to hi, closes
    linked to their opens both ways, objects of string keys not closed behind a key, value words inside [lo, hi), string
    ranges inside their buffer, finite floats, and no root, nop or unknown word"""
    stack = []  # [tag, members so far, index of the open]
    i = lo
    while i < hi:
        w = int(tape[i])
        t, v = w >> 56, w & VAL
        if i > lo and not stack:
            return False  # a second value at the cell's top level
        if t in (ord("}"), ord("]")):
            if not stack or stack[-1][0] != (ord("{") if t == ord("}") else ord("[")):
                return False
            o = stack[-1][2]
            if v != o or (int(tape[o]) & VAL) != i + 1 or (t == ord("}") and stack[-1][1] % 2):
                return False
            stack.pop()
            i += 1
            continue
        if stack:
            top = stack[-1]
            if top[0] == ord("{") and top[1] % 2 == 0 and t != ord('"'):
                return False
            top[1] += 1
        if t in _VALUE_TAGS:
            if i + 1 >= hi:
                return False
            p = int(tape[i + 1])
            if t == ord('"'):
                try:
                    _string_bytes(v, p, strings, message)
                except _Fail:
                    return False
            elif t == ord("d") and (p >> 52) & 0x7FF == 0x7FF:
                return False
            i += 2
        elif t in (ord("t"), ord("f"), ord("n")):
            i += 1
        elif t in (ord("{"), ord("[")):
            stack.append([t, 0, i])
            i += 1
        else:
            return False
    return not stack


def json_cell(tape, strings, message, root, path):
    """one JSON cell: FindElement(path...) as find_cell, then Element.Iter.MarshalJSON() on the element's Iter, when its
    sub-tree [head, n) passes subtree_ok (else CORRUPT); a fresh element (Type None) is CONVERT"""
    it = _It(len(tape), root)
    elem = _It(0)
    try:
        _advance_iter(tape, it, elem)
        _advance_into(tape, elem)
        e = _find_element(tape, strings, message, elem, [bytes(s) for s in path])
    except _Fail as f:
        return Cell(f.status, value=b"")
    if e.t == TAG_END and e.n == 0:
        return Cell(CONVERT, value=b"")
    head = e.off - 1
    if not subtree_ok(tape, strings, message, head, e.n):
        return Cell(CORRUPT, e.t, head, b"")
    cp = _It(e.n, e.off)
    cp.add, cp.cur, cp.t = e.add, e.cur, e.t
    # the well-formed sub-tree: the reference's walk must succeed (a MarshalError here is a defect of the checks)
    return Cell(OK, e.t, head, marshal_json_buffer(tape, strings, message, cp))


def find_json(tape, strings, message, paths, kinds, rows=None):
    """find() with JSON paths among the kinds"""
    rs = roots(tape) if rows is None else rows
    return [[json_cell(tape, strings, message, int(r), path) if kind == JSON else
             find_cell(tape, strings, message, int(r), path, kind) for r in rs] for path, kind in zip(paths, kinds)]
