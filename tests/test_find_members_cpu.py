"""Member rows of the find in the Python port (tests/find_members_oracle.py): the object at a row path of every record,
Object.ForEach over it, and every cell from each member.  On update-center's plugins, citm_catalog's maps, github_events
payloads and NDJSON records exploded with a row path of 0 segments, the rows, keys and cells agree with Python's json;
builder tapes pin each quirk of ForEach's walk with its rows written out.  CPU only."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from tests import find_members_oracle as fm
from tests import find_oracle as fo
from tests.find_json_oracle import JSON
from tests.find_rows_oracle import element_cell
from tests.tape_builder import word
from tests.test_find_lists_cpu import NDJSON_FIXTURES, ndjson_records
from tests.util import load_fixture

S = 1 << 55
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRS = b"abcdefgh"

# documents whose objects are maps keyed by an id or a name, and the row path to each
DOC_MEMBERS = [("update-center", [b"plugins"]), ("citm_catalog", [b"events"]), ("citm_catalog", [b"seatCategoryNames"]),
               ("citm_catalog", [b"areaNames"]), ("citm_catalog", [b"topicNames"])]


def K(c):
    """the key "c" (one byte of STRS)"""
    return [word('"', S | (ord(c) - ord("a"))), 1]


def rec(members, link=None):
    """r { members } r, the members from word 2; link: the '{' word's link if not one past the '}'"""
    n = 2 + len(members)
    return [word("r", n + 2), word("{", n + 1 if link is None else link)] + list(members) + [word("}", 1), word("r", 0)]


def members_of(members, only_keys=(), paths=(), kinds=(), link=None):
    t = np.array(rec(members, link), dtype=np.uint64)
    st, offs, tags, idx, keys, cells = fm.find_members(t, STRS, b"", [], list(paths), list(kinds), list(only_keys), [0])
    return st, offs, idx, keys, cells


# builder tapes of ForEach's quirks: (name, members, only_keys, '{' link, want (status, offsets, value heads, keys))
QUIRKS = [
    ("non_string_key_keeps_rows", K("a") + [word("t")] + K("b") + [word("f"), word("l"), 5, word("t")], (), None,
     ([fo.CORRUPT], [0, 2], [4, 7], [b"a", b"b"])),
    ("value_missing_at_close", K("a") + [word("t")] + K("b"), (), None, ([fo.OK], [0, 1], [4], [b"a"])),
    ("key_at_end_of_tape", K("a") + [word("t")] + K("b"), (), 7, ([fo.CORRUPT], [0, 1], [4], [b"a"])),
    ("nop_between_key_and_value", K("a") + [word("N", 0), word("t")] + K("b") + [word("f")], (), None,
     ([fo.OK], [0, 2], [5, 8], [b"a", b"b"])),
    ("link_behind_its_word", K("a") + [word("t")] + K("b") + [word("{", 3), word("}", 7)], (), None,
     ([fo.OK], [0, 1], [4], [b"a"])),
    ("unknown_tag_as_key", K("a") + [word("t"), word("x")] + K("b") + [word("f")], (), None, ([fo.OK], [0, 1], [4], [b"a"])),
    ("unknown_tag_as_value", K("a") + [word("x")] + K("b") + [word("f")], (), None, ([fo.OK], [0, 0], [], [])),
    ("duplicate_keys_counted", K("a") + [word("l"), 1] + K("a") + [word("l"), 2] + K("b") + [word("l"), 3], (b"a", b"b"),
     None, ([fo.OK], [0, 2], [4, 8], [b"a", b"a"])),
    ("cut_before_error_key", K("a") + [word("t")] + K("b") + [word("f"), word("n")], (b"a", b"b"), None,
     ([fo.OK], [0, 2], [4, 7], [b"a", b"b"])),
    ("error_key_before_cut", K("a") + [word("t")] + K("b") + [word("f"), word("n")], (b"a", b"b", b"c"), None,
     ([fo.CORRUPT], [0, 2], [4, 7], [b"a", b"b"])),
    ("error_key_inside_cut", K("a") + [word("t"), word("n")] + K("b") + [word("f")], (b"a", b"b"), None,
     ([fo.CORRUPT], [0, 1], [4], [b"a"])),
    ("duplicate_only_keys", K("a") + [word("l"), 1] + K("b") + [word("l"), 2] + K("a") + [word("l"), 3], (b"a", b"a"), None,
     ([fo.OK], [0, 1], [4], [b"a"])),
    ("duplicate_only_keys_two", K("a") + [word("l"), 1] + K("c") + [word("t")] + K("b") + [word("l"), 2] + K("a") +
     [word("l"), 3], (b"b", b"a", b"b"), None, ([fo.OK], [0, 2], [4, 11], [b"a", b"b"])),
    ("key_outside_its_buffer", K("a") + [word("t"), word('"', S | 7), 2, word("f")], (), None,
     ([fo.CORRUPT], [0, 1], [4], [b"a"])),
    ("skipped_key_outside_the_set", K("c") + [word("t")] + K("a") + [word("f")], (b"a",), None, ([fo.OK], [0, 1], [7], [b"a"])),
    ("empty_object", [], (), None, ([fo.OK], [0, 0], [], [])),
]


@pytest.mark.parametrize("name,members,only,link,w", QUIRKS, ids=[q[0] for q in QUIRKS])
def test_quirks(name, members, only, link, w):
    assert members_of(members, only, link=link)[:4] == w


def test_zero_segment_cell_after_a_zero_nop_is_corrupt():
    """AdvanceIter refuses a nop of skip 0 ("invalid nop skip", parsed_json.go:309-312) where Advance stepped over it:
    the row is there, its value cell of 0 segments is CORRUPT, a [key] cell from the value is NOT_OBJECT"""
    st, offs, idx, keys, cells = members_of(K("a") + [word("N", 0), word("t")], paths=[[], [b"a"]],
                                            kinds=[fo.BOOL, fo.BOOL])
    assert (st, offs, idx) == ([fo.OK], [0, 1], [5])
    assert cells[0][0][0] == fo.CORRUPT and cells[1][0][0] == fo.NOT_OBJECT


def test_zero_segment_row_path_and_record_statuses():
    """elem.Object directly for 0 segments; an array record is "next item is not object" (CONVERT); a '{' whose link
    lies in front of its members is "object ends at index before start" (CORRUPT)"""
    t = np.array([word("r", 5), word("[", 4), word("t"), word("]", 1), word("r", 0)], dtype=np.uint64)
    assert fm.find_members(t, b"", b"", [], [], [], (), [0])[:2] == ([fo.CONVERT], [0, 0])
    assert members_of(K("a") + [word("t")], link=1)[:2] == ([fo.CORRUPT], [0, 0])
    assert members_of(K("a") + [word("t")], link=2)[:2] == ([fo.OK], [0, 0])  # end == off: no members, no error


def _objects(v, row_path):
    for k in row_path:
        v = v.get(k.decode()) if isinstance(v, dict) else None
    return v if isinstance(v, dict) else None


def agree(tape, strs, msg, row_path, objs, only_keys=()):
    """rows, keys and the value cells (0 segments) against json; objs[k] = record k's object (None: none there); each
    value cell also equals the [key] cell from the record's object.  Returns the rows."""
    kinds = [JSON, fo.STRING, fo.INT64, fo.ELEMENT]
    st, offs, tags, idx, keys, cells = fm.find_members(tape, strs, msg, row_path, [[]] * len(kinds), kinds, only_keys)
    assert len(st) == len(objs)
    want = []
    for k, o in enumerate(objs):
        assert (st[k] == fo.OK) == (o is not None), k
        items = [(a, b) for a, b in (o or {}).items() if not only_keys or a.encode() in only_keys]
        assert offs[k + 1] - offs[k] == len(items), k
        want += items
    assert [k.decode("utf-8", "surrogatepass") for k in keys] == [a for a, _ in want]
    for r, (a, v) in enumerate(want):
        s, t, i, n, _, b = cells[0][r]
        assert s == fo.OK and i == idx[r] and json.loads(b) == v, (a, b[:80])
        assert (cells[1][r][0] == fo.OK) == isinstance(v, str)
        if isinstance(v, str):
            assert cells[1][r][5] == v.encode("utf-8", "surrogatepass")
    # the identity for unique keys: the value cell is FindElement([key]) from the record's object
    r, roots = 0, fo.foreach_roots(tape)
    for k, o in enumerate(objs[:50]):
        root = roots[k]
        s, lo, end = fm.record_object(tape, strs, msg, int(root), row_path)
        it = fo._It(end, lo + 1)
        it.t, it.cur = ord("{"), end
        for a in (o or {}):
            if only_keys and a.encode() not in only_keys:
                continue
            for p, kind in enumerate(kinds):
                assert element_cell(tape, strs, msg, it, [a.encode("utf-8", "surrogatepass")], kind) == cells[p][r]
            r += 1
    return len(want)


@pytest.mark.parametrize("name,row_path", DOC_MEMBERS)
def test_documents_against_json(oracle_native, name, row_path):
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc)
    assert rc == 0
    objs = [_objects(json.loads(doc), row_path)]
    assert objs[0] and len(objs[0]) > 1
    assert agree(tape, strs, doc[off:off + ln], row_path, objs) == len(objs[0])


def test_update_center_plugins_with_only_keys(oracle_native):
    doc = load_fixture("update-center")
    rc, tape, strs, (off, ln) = oracle_native.parse(doc)
    names = list(json.loads(doc)["plugins"])
    only = (names[3].encode(), names[100].encode(), b"\x00nowhere")
    assert agree(tape, strs, doc[off:off + ln], [b"plugins"], [_objects(json.loads(doc), [b"plugins"])], only) == 2


def test_github_events_payloads(oracle_native):
    recs, nd = ndjson_records("github_events")
    rc, tape, strs, (off, ln) = oracle_native.parse(nd, ndjson=True)
    assert rc == 0
    assert agree(tape, strs, nd[off:off + ln], [b"payload"], [_objects(r, [b"payload"]) for r in recs]) > 0


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
def test_ndjson_explode(oracle_native, name):
    """a row path of 0 segments: every key of every record, with its value"""
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(nd, ndjson=True)
    assert rc == 0
    assert agree(tape, strs, nd[off:off + ln], [], recs) == sum(len(r) for r in recs)


def test_escaped_keys_match_their_unescaped_bytes(oracle_native):
    doc = b'{"a\\"b": 1, "\\u00e9": 2, "x": 3, "\\u00e9": 4}'
    rc, tape, strs, (off, ln) = oracle_native.parse(doc)
    st, offs, tags, idx, keys, cells = fm.find_members(tape, strs, doc[off:off + ln], [], [[]], [fo.INT64],
                                                       [b'a"b', "é".encode()])
    assert (st, offs, keys) == ([fo.OK], [0, 2], [b'a"b', "é".encode()])
    assert [c[3] for c in cells[0]] == [1, 2]


def test_keys_out_struct_matches_header():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
    from simdjson_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "simdjson_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} sj_find_keys_out;", hdr).group(1)
    assert re.findall(r"(\w+);", body) == [f[0] for f in _lib.FindKeysOut._fields_]
    assert C.sizeof(_lib.FindKeysOut) == 3 * 8
    assert "sj_find_members_device" in _lib.EXPORTS and "sj_parse_find_members" in _lib.EXPORTS
