"""The find's array rows restated over a tape: for every record (a root, as find() takes them), ForEach's element,
FindElement(row_path...) and Iter.Array (or elem.Array for a row path of 0 segments); then Array.ForEach over that
array, each element a row; then every (path, row) cell from the element's Iter.  Test infrastructure: the expected
output of the device's array rows (find_rows.cuh), record for record and cell for cell.

Each function ports one function of the reference line by line and names it with file:line.  The cells reuse the
ports of tests/find_oracle.py, tests/find_json_oracle.py and tests/find_lists_oracle.py from the point where those
have found their element."""
from tests.find_json_oracle import JSON, marshal_json_buffer, subtree_ok
from tests.find_lists_oracle import (LIST_KINDS, M64, STRING_CVT, STRING_LISTS, _array, _as_numbers, _as_strings,
                                     string_cvt)
from tests.find_oracle import (CONVERT, CORRUPT, OK, STRING, TAG_END, TYPE_NONE, _advance, _advance_into, _advance_iter,
                               _convert, _Fail, _find_element, _It, foreach_roots)


def record_array(tape, strings, message, root, row_path):
    """ForEach's element for the root at slot `root` (parsed_json.go:125-138), FindElement(row_path...) (:833-864) and
    Element.Iter.Array (:1022-1039); with no row path elem.Array directly.  Returns (status, lo, end): the array's '['
    at lo and its tape Tape[:end] (lo = end = 0 unless OK)."""
    it = _It(len(tape), root)
    elem = _It(0)
    try:
        _advance_iter(tape, it, elem)
        _advance_into(tape, elem)
        if row_path:
            e = _find_element(tape, strings, message, elem, [bytes(s) for s in row_path])
            if e.t == TAG_END and e.n == 0:  # a fresh Element: Array says "next item is not array"
                raise _Fail(CONVERT)
        else:
            e = elem
        end, off = _array(e)
        return OK, off - 1, end
    except _Fail as f:
        return f.status, 0, 0


def foreach_elements(tape, lo, end):
    """Array.ForEach (parsed_array.go:45-56) over the array Tape[:end] whose '[' is word lo: Array.Iter (:37-43) has
    off = lo + 1 and addNext 0, then Advance (parsed_json.go:196-223) until TypeNone.  The Iter of each element."""
    i = _It(end, lo + 1)
    out = []
    while _advance(tape, i) != TYPE_NONE:
        e = _It(i.n, i.off)
        e.add, e.cur, e.t = i.add, i.cur, i.t
        out.append(e)
    return out


def element_cell(tape, strings, message, it, path, kind):
    """one (path, row) cell from the element's Iter `it`: FindElement(path...) on a copy, then the accessor of `kind`.
    Returns (status, tag, index, value, elements, bytes) as the device writes them: value is the element count of a
    list cell and the byte length of a STRING / JSON / STRING_CVT cell."""
    cp = _It(it.n, it.off)
    cp.add, cp.cur, cp.t = it.add, it.cur, it.t
    try:
        e = _find_element(tape, strings, message, cp, [bytes(s) for s in path])
    except _Fail as f:
        return f.status, 0, -1, 0, [], b""
    if e.t == TAG_END and e.n == 0:  # AdvanceIter met the end exactly: a fresh Element, Type None
        return (OK if kind == 0 else CONVERT), 0, -1, 0, [], b""
    head = e.off - 1
    try:
        if kind == JSON:  # as json_cell (find_json_oracle.py)
            if not subtree_ok(tape, strings, message, head, e.n):
                return CORRUPT, e.t, head, 0, [], b""
            c = _It(e.n, e.off)
            c.add, c.cur, c.t = e.add, e.cur, e.t
            b = marshal_json_buffer(tape, strings, message, c)
            return OK, e.t, head, len(b), [], b
        if kind == STRING_CVT:  # as list_cell (find_lists_oracle.py)
            b = string_cvt(tape, strings, message, e)
            return OK, e.t, head, len(b), [], b
        if kind in LIST_KINDS:
            n, off = _array(e)
            if kind in STRING_LISTS:
                xs = _as_strings(tape, strings, message, n, off, kind)
                return OK, e.t, head, len(xs), [len(x) for x in xs], b"".join(xs)
            xs = _as_numbers(tape, n, off, kind)
            return OK, e.t, head, len(xs), [x & M64 for x in xs], b""
        v = _convert(tape, strings, message, e, kind)  # as find_cell (find_oracle.py)
        if kind == STRING:
            return OK, e.t, head, len(v), [], v
        return OK, e.t, head, v, [], b""
    except _Fail as f:
        return f.status, e.t, head, 0, [], b""


def find_rows(tape, strings, message, row_path, paths, kinds, records=None):
    """(rec_status, rec_offsets, row_tag, row_index, cells): cells[p][r] is element_cell of path p on row r; records =
    the root slots (default foreach_roots())"""
    rs = foreach_roots(tape) if records is None else records
    rec_status, rec_offsets, elems = [], [0], []
    for r in rs:
        st, lo, end = record_array(tape, strings, message, int(r), row_path)
        rec_status.append(st)
        es = foreach_elements(tape, lo, end) if st == OK else []
        elems += es
        rec_offsets.append(len(elems))
    row_tag = [e.t for e in elems]
    row_index = [e.off - 1 for e in elems]
    cells = [[element_cell(tape, strings, message, e, path, k) for e in elems] for path, k in zip(paths, kinds)]
    return rec_status, rec_offsets, row_tag, row_index, cells
