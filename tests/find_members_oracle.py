"""The find's member rows restated over a tape: for every record (a root, as find() takes them), ForEach's element,
FindElement(row_path...) and Iter.Object (or elem.Object for a row path of 0 segments); then Object.ForEach(fn,
onlyKeys) over that object, each member fn receives a row with its key; then every (path, row) cell.  Test
infrastructure: the expected output of the device's member rows (find_rows.cuh), record for record and cell for cell.

Each function ports one function of the reference line by line and names it with file:line.  A cell of >= 1 segment is
tests/find_rows_oracle.py's element_cell from the member's Iter; a cell of 0 segments is the member's value, the element
Object.FindPath returns when it stops at the member's key."""
from tests.find_json_oracle import JSON, marshal_json_buffer, subtree_ok
from tests.find_lists_oracle import LIST_KINDS, M64, STRING_CVT, STRING_LISTS, _array, _as_numbers, _as_strings, string_cvt
from tests.find_oracle import (CONVERT, CORRUPT, OK, STRING, TAG_END, TYPE_NONE, _advance, _advance_into, _advance_iter,
                               _convert, _Fail, _find_element, _It, _string_bytes, foreach_roots)
from tests.find_rows_oracle import element_cell

TYPE_STRING = 2
TAG_OBJECT_START = ord("{")


def iter_object(e):
    """Iter.Object, parsed_json.go:998-1018: (end, off) of the object Tape[:end] whose members start at off"""
    if e.t != TAG_OBJECT_START:
        raise _Fail(CONVERT)  # "next item is not object"
    end = e.cur
    if end < e.off:
        raise _Fail(CORRUPT)  # "corrupt input: object ends at index before start"
    if e.n < end:
        raise _Fail(CORRUPT)  # "corrupt input: object extended beyond tape"
    return end, e.off


def record_object(tape, strings, message, root, row_path):
    """ForEach's element for the root at slot `root` (parsed_json.go:125-138), FindElement(row_path...) (:833-864) and
    Element.Iter.Object (:998-1018); with no row path elem.Object directly.  Returns (status, lo, end): the object's
    '{' at lo and its tape Tape[:end] (lo = end = 0 unless OK)."""
    it = _It(len(tape), root)
    elem = _It(0)
    try:
        _advance_iter(tape, it, elem)
        _advance_into(tape, elem)
        if row_path:
            e = _find_element(tape, strings, message, elem, [bytes(s) for s in row_path])
            if e.t == TAG_END and e.n == 0:  # a fresh Element: Object says "next item is not object"
                raise _Fail(CONVERT)
        else:
            e = elem
        end, off = iter_object(e)
        return OK, off - 1, end
    except _Fail as f:
        return f.status, 0, 0


def foreach_members(tape, strings, message, lo, end, only_keys=()):
    """Object.ForEach (parsed_object.go:142-186) over the object Tape[:end] whose '{' is word lo: o.tape.Iter() with
    off = lo + 1, then Advance (parsed_json.go:196-223) key by key.  Returns (members, status): (key bytes, key head,
    value Iter) of each member fn receives, and CORRUPT for ForEach's two errors (the members in front of them stay)."""
    keys = {bytes(k) for k in only_keys}  # map[string]struct{}: one entry per distinct key
    tmp = _It(end, lo + 1)
    out, n = [], 0
    while True:
        typ = _advance(tape, tmp)
        if typ != TYPE_STRING or tmp.off + 1 >= tmp.n:  # len(tmp.tape.Tape) = end
            if typ == TYPE_NONE:
                return out, OK
            return out, CORRUPT  # "object: unexpected name tag"
        offset, length = tmp.cur, int(tape[tmp.off])
        k = tmp.off - 1
        try:
            name = _string_bytes(offset, length, strings, message)
        except _Fail:
            return out, CORRUPT  # "getting object name"
        if len(keys) > 0 and name not in keys:
            if _advance(tape, tmp) == TYPE_NONE:  # skip the value
                return out, OK
            continue
        if _advance(tape, tmp) == TYPE_NONE:
            return out, OK
        e = _It(tmp.n, tmp.off)
        e.add, e.cur, e.t = tmp.add, tmp.cur, tmp.t
        out.append((name, k, e))
        n += 1
        if n == len(keys):
            return out, OK


def value_cell(tape, strings, message, k, end, kind):
    """a path of 0 segments on a member row: the element Object.FindPath returns when it stops at the key at head k
    (parsed_object.go:298-303: dst.Type, err = tmp.AdvanceIter(&dst.Iter), tmp left by Advance on the key), then the
    accessor of `kind` as element_cell (find_rows_oracle.py) applies it to a found element"""
    tmp = _It(end, k + 1)
    tmp.add, tmp.cur, tmp.t = 1, 0, ord('"')
    e = _It(0)
    try:
        if _advance_iter(tape, tmp, e) is None:  # the tape ended exactly: a fresh Element, Type None
            return (OK if kind == 0 else CONVERT), 0, -1, 0, [], b""
    except _Fail as f:
        return f.status, 0, -1, 0, [], b""
    head = e.off - 1
    try:
        if kind == JSON:
            if not subtree_ok(tape, strings, message, head, e.n):
                return CORRUPT, e.t, head, 0, [], b""
            c = _It(e.n, e.off)
            c.add, c.cur, c.t = e.add, e.cur, e.t
            b = marshal_json_buffer(tape, strings, message, c)
            return OK, e.t, head, len(b), [], b
        if kind == STRING_CVT:
            b = string_cvt(tape, strings, message, e)
            return OK, e.t, head, len(b), [], b
        if kind in LIST_KINDS:
            n, off = _array(e)
            if kind in STRING_LISTS:
                xs = _as_strings(tape, strings, message, n, off, kind)
                return OK, e.t, head, len(xs), [len(x) for x in xs], b"".join(xs)
            xs = _as_numbers(tape, n, off, kind)
            return OK, e.t, head, len(xs), [x & M64 for x in xs], b""
        v = _convert(tape, strings, message, e, kind)
        if kind == STRING:
            return OK, e.t, head, len(v), [], v
        return OK, e.t, head, v, [], b""
    except _Fail as f:
        return f.status, e.t, head, 0, [], b""


def member_cell(tape, strings, message, member, path, kind):
    """one (path, row) cell of a member row: element_cell from its value's Iter, or value_cell for 0 segments"""
    _, k, e = member
    if not path:
        return value_cell(tape, strings, message, k, e.n, kind)
    return element_cell(tape, strings, message, e, path, kind)


def find_members(tape, strings, message, row_path, paths, kinds, only_keys=(), records=None):
    """(rec_status, rec_offsets, row_tag, row_index, keys, cells): row_tag / row_index of each member's value head,
    keys[r] the key bytes of row r, cells[p][r] member_cell of path p on row r; records = the root slots (default
    foreach_roots())"""
    rs = foreach_roots(tape) if records is None else records
    rec_status, rec_offsets, members = [], [0], []
    for r in rs:
        st, lo, end = record_object(tape, strings, message, int(r), row_path)
        if st == OK:
            ms, st = foreach_members(tape, strings, message, lo, end, only_keys)
            members += ms
        rec_status.append(st)
        rec_offsets.append(len(members))
    row_tag = [e.t for _, _, e in members]
    row_index = [e.off - 1 for _, _, e in members]
    keys = [name for name, _, _ in members]
    cells = [[member_cell(tape, strings, message, m, list(path), kd) for m in members] for path, kd in zip(paths, kinds)]
    return rec_status, rec_offsets, row_tag, row_index, keys, cells
