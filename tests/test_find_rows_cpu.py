"""Array rows of the find in the Python port (tests/find_rows_oracle.py): the array at a row path of every record,
Array.ForEach over it, and every cell from each element's Iter.  On every fixture that holds an array of objects, and
on NDJSON records with nested arrays, the rows and cells agree with Python's json; builder tapes pin each quirk of
Advance's walk with its rows written out.  The ctypes mirror of sj_find_rows_out matches the header.  CPU only."""
import ctypes as C
import json
import math
import os
import re

import numpy as np
import pytest

from tests import find_oracle as fo
from tests import find_rows_oracle as fr
from tests.find_json_oracle import JSON
from tests.tape_builder import word
from tests.test_find_json_cpu import harvest
from tests.test_find_lists_cpu import NDJSON_FIXTURES, _arr, _obj, ndjson_records
from tests.util import load_fixture

S = 1 << 55
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the fixtures whose documents hold arrays of objects, and the row path to each
DOC_ROWS = [("twitter", [b"statuses"]), ("citm_catalog", [b"performances"]), ("apache_builds", [b"jobs"]),
            ("random", [b"result"]), ("instruments", [b"instruments"]), ("instruments", [b"patterns"]),
            ("instruments", [b"samples"]), ("payload-large", [b"users"]), ("github_events", [])]
# NDJSON records (tests/test_find_lists_cpu.py) and a nested array of objects in each
ND_ROWS = {"twitter": [b"entities", b"hashtags"], "github_events": [b"payload", b"commits"], "random": [b"friends"],
           "update-center": [b"developers"]}


def _expect(v, path):
    """(status, value) of FindElement(path...) on the element v, from json"""
    if not path:
        return fo.NOT_FOUND, None
    for k in path:
        if not isinstance(v, dict):
            return fo.NOT_OBJECT, None
        k = k.decode("utf-8", "surrogatepass")
        if k not in v:
            return fo.NOT_FOUND, None
        v = v[k]
    return fo.OK, v


def _subpaths(elems):
    seen, out = set(), []
    for e in elems[:20]:
        for p in harvest(json.dumps(e).encode(), 40):
            if tuple(p) not in seen:
                seen.add(tuple(p))
                out.append(p)
    return out


def agree(tape, strs, msg, row_path, arrays):
    """rows and the STRING / INT64 / FLOAT64 / BOOL / JSON cells of sub-paths against json; arrays[k] = record k's
    array (None: no array there).  Returns the OK cells checked."""
    elems = [e for a in arrays if a is not None for e in a]
    paths = _subpaths([e for e in elems if isinstance(e, dict)] or elems)
    kinds = [fo.STRING, fo.INT64, fo.FLOAT64, fo.BOOL, JSON]
    ps, ks = [p for p in paths for _ in kinds], [k for _ in paths for k in kinds]
    st, offs, tags, idx, cells = fr.find_rows(tape, strs, msg, row_path, ps, ks)
    assert len(st) == len(arrays)
    for k, a in enumerate(arrays):
        assert (st[k] == fo.OK) == (a is not None), k
        assert offs[k + 1] - offs[k] == (len(a) if a is not None else 0), k
    assert len(idx) == len(elems)
    ok = 0
    for p, kind, col in zip(ps, ks, cells):
        for e, (s, t, i, v, _, b) in zip(elems, col):
            es, ev = _expect(e, p)
            if es != fo.OK:
                assert s == es, (p, kind, e)
                continue
            if kind == JSON:
                assert s == fo.OK and json.loads(b) == ev, (p, b[:80])
            elif kind == fo.STRING:
                assert (s == fo.OK) == isinstance(ev, str), (p, kind)
                if s == fo.OK:
                    assert b == ev.encode("utf-8", "surrogatepass")
            elif kind == fo.BOOL:
                assert (s == fo.OK) == isinstance(ev, bool), (p, kind)
                if s == fo.OK:
                    assert v == int(ev)
            elif kind == fo.INT64:
                if isinstance(ev, int) and not isinstance(ev, bool) and -2**63 <= ev < 2**63:
                    assert s == fo.OK and v == ev & (2**64 - 1), (p, ev, v)
                elif not isinstance(ev, (int, float)) or isinstance(ev, bool):
                    assert s == fo.CONVERT, (p, kind)
            else:
                if isinstance(ev, (int, float)) and not isinstance(ev, bool):
                    assert s == fo.OK and math.isclose(fo._f64(v), float(ev), rel_tol=1e-15), (p, ev)
                else:
                    assert s == fo.CONVERT, (p, kind)
            ok += s == fo.OK
    return ok


def _arrays(v, row_path):
    for k in row_path:
        v = v.get(k.decode()) if isinstance(v, dict) else None
    return v if isinstance(v, list) else None


@pytest.mark.parametrize("name,row_path", DOC_ROWS)
def test_documents_against_json(oracle_native, name, row_path):
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc)
    assert rc == 0
    arrays = [_arrays(json.loads(doc), row_path)]
    assert arrays[0] and len(arrays[0]) > 1
    assert agree(tape, strs, doc[off:off + ln], row_path, arrays) > 0


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
def test_ndjson_nested_arrays_against_json(oracle_native, name):
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(nd, ndjson=True)
    assert rc == 0
    arrays = [_arrays(r, ND_ROWS[name]) for r in recs]
    assert sum(len(a) for a in arrays if a) > 0
    agree(tape, strs, nd[off:off + ln], ND_ROWS[name], arrays)


def _rows(items, paths=(), kinds=(), row_path=(b"a",), strs=b"abcdefgh"):
    """the records' statuses, rows and cells of r { "a": [ items ] } r (the '[' at word 4)"""
    t = np.array(_obj(_arr(items)), dtype=np.uint64)
    st, offs, tags, idx, cells = fr.find_rows(t, strs, b"", list(row_path), list(paths), list(kinds), [0])
    return st, offs, idx, cells


def test_nop_skips_one_more_word_than_advance_into():
    """Advance: `i.off++ ... if i.t == TagNop { i.off += int(i.cur) }` (parsed_json.go:207-213) skips 1 + skip words:
    the nop at 7 with skip 1 lands on 9, not on the unknown tag at 8"""
    assert _rows([word("l"), 1, word("N", 1), word("x"), word("l"), 2])[:3] == ([fo.OK], [0, 2], [5, 9])


def test_delete_elems_nop_run_lands_past_the_next_head():
    """DeleteElems (parsed_array.go:60-76) writes skips 2, 1 over a 2-word element: ForEach lands on 5 + 1 + 2 = 8,
    one word past the 't' at 7, which it never hands out"""
    assert _rows([word("N", 2), word("N", 1), word("t"), word("l"), 3])[:3] == ([fo.OK], [0, 1], [8])


def test_nop_jump_past_the_end_ends_the_walk():
    """`if i.off >= len(i.tape.Tape) { ... return TypeNone }` (parsed_json.go:200-204)"""
    assert _rows([word("l"), 1, word("N", 10)])[:3] == ([fo.OK], [0, 1], [5])


def test_link_behind_its_word_ends_the_walk_silently():
    """`if i.addNext < 0 { i.moveToEnd(); return TypeNone }` (parsed_json.go:216-219): no error, no CORRUPT record"""
    assert _rows([word("t"), word("{", 3), word("}", 6)])[:3] == ([fo.OK], [0, 1], [5])


def test_unknown_tag_ends_and_root_is_an_element():
    """an 'r' is TypeRoot (an element, stepped over by its link), an unknown tag TypeNone; the cell of the 'r' enters
    it through Root (parsed_json.go:853-858), whose tape Tape[:cur - 1] (:822) ends at word 7: NOT_FOUND"""
    st, offs, idx, cells = _rows([word("t"), word("r", 8), word("t"), word("x"), word("t")], [[b"a"]], [fo.INT64])
    assert (st, offs, idx) == ([fo.OK], [0, 2], [5, 6])
    assert [c[0] for c in cells[0]] == [fo.NOT_OBJECT, fo.NOT_FOUND]


def test_nested_arrays_are_rows_with_not_object_cells():
    st, offs, idx, cells = _rows([word("[", 7), word("]", 5), word("l"), 3], [[b"a"], []], [fo.INT64, fo.ELEMENT])
    assert (st, offs, idx) == ([fo.OK], [0, 2], [5, 7])
    assert [c[0] for c in cells[0]] == [fo.NOT_OBJECT, fo.NOT_OBJECT]
    assert [c[0] for c in cells[1]] == [fo.NOT_FOUND, fo.NOT_FOUND]  # FindElement of 0 segments


def test_empty_array_has_no_rows():
    assert _rows([])[:3] == ([fo.OK], [0, 0], [])


def test_cells_of_object_elements():
    """{"a": [{"a": 7}, {"b": 1}]}: FindElement(["a"]) from each element"""
    obj1 = [word("{", 11), word('"', S), 1, word("l"), 7, word("}", 5)]
    obj2 = [word("{", 17), word('"', S | 1), 1, word("l"), 1, word("}", 11)]
    st, offs, idx, cells = _rows(obj1 + obj2, [[b"a"]], [fo.INT64])
    assert (st, offs, idx) == ([fo.OK], [0, 2], [5, 11])
    assert [(c[0], c[3]) for c in cells[0]] == [(fo.OK, 7), (fo.NOT_FOUND, 0)]


def test_zero_segment_row_path():
    """elem.Array directly: an object root is "next item is not array" (CONVERT); a root array gives its elements"""
    assert _rows([word("t")], row_path=())[:2] == ([fo.CONVERT], [0, 0])
    t = np.array([word("r", 6), word("[", 5), word("t"), word("f"), word("]", 1), word("r", 0)], dtype=np.uint64)
    st, offs, tags, idx, _ = fr.find_rows(t, b"", b"", [], [], [], [0])
    assert (st, offs, idx, tags) == ([fo.OK], [0, 2], [2, 3], [ord("t"), ord("f")])


def test_record_statuses():
    """NOT_FOUND, NOT_OBJECT and CONVERT records have no rows"""
    assert _rows([word("t")], row_path=(b"b",))[:2] == ([fo.NOT_FOUND], [0, 0])
    assert _rows([word("t")], row_path=(b"a", b"b"))[:2] == ([fo.NOT_OBJECT], [0, 0])
    t = np.array(_obj([word("t")]), dtype=np.uint64)
    assert fr.find_rows(t, b"abc", b"", [b"a"], [], [], [0])[:2] == ([fo.CONVERT], [0, 0])


def test_rows_out_struct_matches_header():
    """the ctypes mirror's fields are the header's, in order, at the same size"""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
    from simdjson_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "simdjson_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} sj_find_rows_out;", hdr).group(1)
    names = re.findall(r"(\w+);", body)
    assert names == [f[0] for f in _lib.FindRowsOut._fields_]
    assert C.sizeof(_lib.FindRowsOut) == 5 * 8
    assert "sj_find_rows_device" in _lib.EXPORTS and "sj_parse_find_rows" in _lib.EXPORTS
