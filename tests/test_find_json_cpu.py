"""JSON cells of the find (SJ_FIND_KIND_JSON) in the Python port (tests/find_json_oracle.py): Element.Iter.MarshalJSON() of
the found element.  On every fixture's and fuzz seed's oracle tape every OK cell's text agrees three ways: the port of
MarshalJSONBuffer, the whole-tape marshal restatement (tests/marshal_oracle.py) of the sub-tree alone under a root, and
json.loads of the source document at that path.  Builder tapes pin one status rule each.  CPU only."""
import json

import numpy as np
import pytest

from tests import find_json_oracle as fj
from tests import find_oracle as fo
from tests.marshal_oracle import marshal
from tests.tape_builder import TapeBuilder, word
from tests.util import TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson


def harvest(doc, limit=80):
    """key paths through objects down to depth 4 of a JSON document, plus paths that are not there"""
    out = []

    def walk(v, path):
        if not isinstance(v, dict) or len(path) >= 4:
            return
        for k, x in v.items():
            p = path + [k.encode("utf-8", "surrogatepass")]
            out.append(p)
            walk(x, p)

    try:
        v = json.loads(doc)
    except Exception:
        v = None
    walk(v if isinstance(v, dict) else {}, [])
    return out[:limit] + [[b"\x00missing"], [b""], []]


def as_root(tape, lo, hi):
    """the words [lo, hi) alone under a root at slot 0, links moved by 1 - lo"""
    out, k = [word("r", hi - lo + 2)], lo
    while k < hi:
        w = int(tape[k])
        if (w >> 56) in b'"lud':
            out += [w, int(tape[k + 1])]
            k += 2
            continue
        out.append(w + 1 - lo if (w >> 56) in b"{[}]" else w)
        k += 1
    return np.array(out + [word("r", 0)], dtype=np.uint64)


class _Dup(Exception):
    pass


def _first_pairs(pairs):
    keys = [k for k, _ in pairs]
    if len(set(keys)) != len(keys):
        raise _Dup()
    return dict(pairs)


def _fits(v):
    if isinstance(v, bool) or v is None or isinstance(v, (float, str)):
        return True
    if isinstance(v, int):
        return -(1 << 63) <= v < (1 << 64)
    if isinstance(v, list):
        return all(_fits(x) for x in v)
    return all(_fits(x) for x in v.values())


def _same(a, b):
    """equal JSON values, where a float and the integer appendFloat writes for it are the same number"""
    if isinstance(a, bool) or isinstance(b, bool) or a is None or b is None:
        return a is b or a == b and type(a) is type(b)
    if isinstance(a, (int, float)) and isinstance(b, (int, float)):
        return float(a) == float(b)
    if isinstance(a, list) and isinstance(b, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict) and isinstance(b, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return a == b


def _at(v, path):
    for k in path:
        if not isinstance(v, dict) or k.decode("utf-8", "surrogatepass") not in v:
            return None, False
        v = v[k.decode("utf-8", "surrogatepass")]
    return v, True


def three_ways(tape, strs, msg, paths, docs=None):
    """every OK JSON cell: the port's text == marshal of the sub-tree under a root (== json.loads of its document at
    the path, for docs[r] with unique keys and 64-bit integers).  Returns the number of OK cells."""
    rows = fo.foreach_roots(tape)
    cells = fj.find_json(tape, strs, msg, paths, [fj.JSON] * len(paths), rows)
    n = 0
    for p, path in enumerate(paths):
        for r, c in enumerate(cells[p]):
            if c.status != fo.OK:
                assert c.value == b""
                continue
            n += 1
            t = int(tape[c.index]) >> 56
            hi = (int(tape[c.index]) & fo.VAL) if t in b"{[" else c.index + (2 if t in b'"lud' else 1)
            assert marshal(as_root(tape, c.index, hi), strs, msg) == c.value, (path, r)
            if docs is None:
                continue
            try:
                whole = json.loads(docs[r], object_pairs_hook=_first_pairs)
            except (_Dup, ValueError):
                continue
            want, found = _at(whole, path)
            if found and _fits(want) and not (isinstance(want, float) and want != want):
                assert _same(json.loads(c.value), want), (path, r)
    return n


@pytest.mark.parametrize("name", TAPE_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures_three_ways(oracle, name, copy):
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle.parse(doc, copy_strings=copy)
    assert rc == 0
    assert three_ways(tape, strs, doc[off:off + ln], harvest(doc), [doc]) > 0 or not harvest(doc)[:-3]


@pytest.mark.parametrize("copy", [True, False])
def test_fuzz_seeds_three_ways(oracle, copy):
    n = 0
    for name, data in fuzz_corpus("corpus", max_size=1 << 14):
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson, copy_strings=copy)
            if rc:
                continue
            msg = data[off:off + ln]
            docs = [x for x in data.split(b"\n") if x.strip()] if ndjson else [data]
            n += three_ways(tape, strs, msg, harvest(data, 20), docs if len(docs) == len(fo.foreach_roots(tape)) else None)
    assert n > 100


def test_tricky_ndjson(oracle):
    nd, recs = tricky_ndjson()
    for copy in (True, False):
        rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
        paths = [[b"Make"], [b"a"], [b"a", b"Make"], [b""], [b"t"], [b"d"], [b"x"], [b"nope"]]
        assert three_ways(tape, strs, nd[off:off + ln], paths, recs) > 0


def test_scalars_and_containers():
    """a scalar gives its own text; containers their compact text; the cell's tag and head index are the element's"""
    b = TapeBuilder()
    b.open("r"); b.open("{")
    b.string(b"s"); b.string(b'a"b\n\x01')
    b.string(b"l"); b.number("l", (1 << 64) - 12)
    b.string(b"u"); b.number("u", 1 << 63)
    b.string(b"d"); b.number("d", fo._f64_bits(1e21))
    b.string(b"t"); b.atom("t")
    b.string(b"o"); b.open("{"); b.string(b"k"); b.open("["); b.atom("n"); b.atom("f"); b.close(); b.close()
    b.string(b"e"); b.open("["); b.close()
    b.close(); b.close()
    tape, strs, msg = b.build()
    want = {b"s": b'"a\\"b\\n\\u0001"', b"l": b"-12", b"u": b"9223372036854775808", b"d": b"1e+21", b"t": b"true",
            b"o": b'{"k":[null,false]}', b"e": b"[]"}
    for k, text in want.items():
        (c,) = fj.find_json(tape, strs, msg, [[k]], [fj.JSON])[0]
        assert (c.status, c.value) == (fo.OK, text), k
        assert int(tape[c.index]) >> 56 == c.tag


def test_fresh_element_is_convert():
    """AdvanceIter that meets the end of the object's tape exactly (over a nop) gives a fresh element, Type None:
    MarshalJSON's "no content queued in iterator" """
    t = np.array([word("r", 7), word("{", 6), word('"', 1 << 55), 1, word("N", 1), word("n"), word("}", 1), word("r", 0)],
                 dtype=np.uint64)
    (c,) = fj.find_json(t, b"a", b"", [[b"a"]], [fj.JSON], [0])[0]
    assert c.astuple() == (fo.CONVERT, 0, -1, b"")


def _cell(words, strs=b"a", rows=(0,)):
    t = np.array(words, dtype=np.uint64)
    return fj.find_json(t, strs, b"", [[b"a"]], [fj.JSON], list(rows))[0]


def _obj(inner, extra=()):
    """r { "a": <inner> } r with inner's links relative to its first word at 4"""
    n = 4 + len(inner)
    return [word("r", n + 2), word("{", n + 1), word('"', 1 << 55), 1] + list(inner) + [word("}", 1), word("r", 0)] + list(extra)


S = 1 << 55


@pytest.mark.parametrize("what,inner", [
    ("close not linked back", [word("[", 6), word("]", 3)]),
    ("open links past its close", [word("[", 7), word("]", 4), word("t")]),
    ("wrong close kind", [word("[", 6), word("}", 4)]),
    ("object closed behind a key", [word("{", 8), word('"', S), 1, word("}", 4)]),
    ("non-string key", [word("{", 8), word("l"), 1, word("}", 4)]),
    ("string range outside Strings.B", [word("[", 8), word('"', S), 9, word("]", 4)]),
    ("NaN", [word("[", 8), word("d"), 0x7FF8000000000000, word("]", 4)]),
    ("Inf", [word("[", 8), word("d"), 0x7FF0000000000000, word("]", 4)]),
    ("nop inside", [word("[", 7), word("N", 0), word("]", 4)]),
    ("root word inside", [word("[", 7), word("r", 0), word("]", 4)]),
    ("unknown tag", [word("[", 7), word("x"), word("]", 4)]),
])
def test_each_check_fails_as_corrupt(what, inner):
    (c,) = _cell(_obj(inner))
    assert c.status == fo.CORRUPT and c.value == b"" and c.index == 4, what


def _shift(words, n0):
    """a root's words moved n0 words on: the links of opens, closes and the root open"""
    out = [(w & ~fo.VAL) | ((w & fo.VAL) + n0) if (w >> 56) in b"{[}]" or ((w >> 56) == ord("r") and (w & fo.VAL) > 0)
           else w for w in words]
    out[-1] = word("r", n0)  # the root close points at its open
    return out


def test_well_formed_cell_beside_malformed_regions():
    """a malformed root in front and a malformed region behind leave the cell's text alone, where the whole-tape
    marshal rejects the tape"""
    bad_root = [word("r", 3), word("x"), word("r", 0)]
    words = bad_root + _shift(_obj([word("[", 9), word("l"), 5, word("t"), word("]", 4)]), 3)
    words += [word("{", 0), word("d"), 0x7FF0000000000000]
    cells = _cell(words, rows=(0, 3))
    assert cells[1].status == fo.OK and cells[1].value == b"[5,true]"
    with pytest.raises(Exception):
        marshal(np.array(words, dtype=np.uint64), b"a", b"")


def test_malformed_cell_next_to_a_good_one():
    """two rows: the first cell malformed, the second's text right"""
    a = _obj([word("[", 7), word("x"), word("]", 4)])
    cells = _cell(a + _shift(_obj([word("[", 6), word("]", 4)]), len(a)), rows=(0, len(a)))
    assert [c.status for c in cells] == [fo.CORRUPT, fo.OK]
    assert cells[1].value == b"[]"
