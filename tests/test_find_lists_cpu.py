"""List cells of the find in the Python port (tests/find_lists_oracle.py): Iter.Array + Array.AsFloat / AsInteger /
AsUint64 / AsString / AsStringCvt, and Iter.StringCvt.  Builder tapes pin each quirk of the literal port, quoting the
Go line they follow; on every fixture as a single document and on the fixtures whose root holds an array of objects
re-emitted as NDJSON, every cell agrees with Python's json.  CPU only."""
import json
import struct

import numpy as np
import pytest

from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import fmt_values
from tests.marshal_oracle import format_float
from tests.tape_builder import TapeBuilder, word
from tests.test_find_json_cpu import _at, _Dup, _first_pairs, harvest
from tests.util import TAPE_FILES, load_fixture

S = 1 << 55
LISTS = list(fl.LIST_KINDS)


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _obj(inner):
    """r { "a": <inner> } r, inner's links relative to its first word at 4"""
    n = 4 + len(inner)
    return [word("r", n + 2), word("{", n + 1), word('"', S), 1] + list(inner) + [word("}", 1), word("r", 0)]


def _cell(inner, kind, strs=b"abcdefgh"):
    t = np.array(_obj(inner), dtype=np.uint64)
    c, elems, data = fl.find_lists(t, strs, b"", [[b"a"]], [kind], [0])[0][0]
    return c.status, elems, data


def _arr(items):
    """[ items ] at word 4: items' words in between, the close linked back"""
    return [word("[", 4 + len(items) + 2)] + list(items) + [word("]", 4)]


def test_zero_length_array_is_ok_everywhere():
    """`[]`: AsFloat reads TagArrayEnd first (parsed_array.go:173 `case TagArrayEnd: break readArray`); AsString's first
    AdvanceIter gives TypeNone (:299 `case TypeNone: return dst, nil`)"""
    for k in LISTS:
        assert _cell(_arr([]), k) == (fo.OK, [], b""), k


def test_nop_inside_as_float_is_convert_but_skipped_by_as_string():
    """AsFloat walks word by word: a nop is `default: return nil, fmt.Errorf("unable to convert type %v to float", tag)`
    (parsed_array.go:175-176); AsString steps with AdvanceIter, which skips it (parsed_json.go:306-311
    `if i.t == TagNop { ... i.off += int(i.cur) }`)"""
    nop = [word('"', S | 0), 1, word("N", 1), word("x"), word('"', S | 1), 2]  # the nop skips itself and 1 word
    assert _cell(_arr([word("l"), 1, word("N", 1), word("l"), 2]), fl.ARRAY_FLOAT64)[0] == fo.CONVERT
    assert _cell(_arr(nop), fl.ARRAY_STRING) == (fo.OK, [1, 2], b"abc")
    # a nop skip of 0: AdvanceIter's "invalid nop skip" (parsed_json.go:308-310)
    assert _cell(_arr([word('"', S), 1, word("N", 0), word('"', S | 1), 2]), fl.ARRAY_STRING)[0] == fo.CORRUPT


def test_as_string_ends_ok_at_an_unknown_tag():
    """the first TypeNone ends the list: parsed_array.go:299-300 `case TypeNone: return dst, nil`, and TagToType of an
    unknown tag is TypeNone"""
    items = [word('"', S), 1, word("x"), word('"', S | 1), 2]
    assert _cell(_arr(items), fl.ARRAY_STRING) == (fo.OK, [1], b"a")
    assert _cell(_arr(items), fl.ARRAY_STRING_CVT) == (fo.OK, [1], b"a")
    # AsFloat meets it as a tag: `default: ... unable to convert type` (parsed_array.go:175-176)
    assert _cell(_arr([word("l"), 1, word("x")]), fl.ARRAY_FLOAT64)[0] == fo.CONVERT


def test_as_uint64_at_two_to_the_63():
    """`if val > math.MaxInt64 { ... overflows uint64 }` (parsed_array.go:254) compares with float64(MaxInt64) = 2^63:
    exactly 2^63 passes and `uint64(val)` gives 1<<63; the next double above fails; NaN passes both checks and gives
    1<<63 too (amd64's float64ToUint64)"""
    two63 = _bits(2.0**63)
    assert _cell(_arr([word("d"), two63]), fl.ARRAY_UINT64) == (fo.OK, [1 << 63], b"")
    assert _cell(_arr([word("d"), two63 + 1]), fl.ARRAY_UINT64)[0] == fo.CONVERT
    assert _cell(_arr([word("d"), 0x7FF8000000000000]), fl.ARRAY_UINT64) == (fo.OK, [1 << 63], b"")
    # AsInteger: `if val > math.MaxInt64` (:203) lets 2^63 through and int64(val) is math.MinInt64
    assert _cell(_arr([word("d"), two63]), fl.ARRAY_INT64) == (fo.OK, [1 << 63], b"")
    assert _cell(_arr([word("d"), _bits(-2.0**63)]), fl.ARRAY_INT64) == (fo.OK, [1 << 63], b"")
    assert _cell(_arr([word("d"), _bits(-2.0**63) + 1]), fl.ARRAY_INT64)[0] == fo.CONVERT


def test_negative_ints():
    """AsUint64: `if val < 0 { return nil, errors.New("int64 value is negative") }` (parsed_array.go:265-267) and
    `if val < 0 { ... "float value is negative" }` (:257-259); AsInteger and AsFloat take them"""
    m5 = (1 << 64) - 5
    assert _cell(_arr([word("l"), m5]), fl.ARRAY_UINT64)[0] == fo.CONVERT
    assert _cell(_arr([word("d"), _bits(-0.5)]), fl.ARRAY_UINT64)[0] == fo.CONVERT
    assert _cell(_arr([word("l"), m5]), fl.ARRAY_INT64) == (fo.OK, [m5], b"")
    assert _cell(_arr([word("l"), m5]), fl.ARRAY_FLOAT64) == (fo.OK, [_bits(-5.0)], b"")
    # `float64(int64(...))` rounds to nearest (:164); `float64(uint64)` too (:169)
    assert _cell(_arr([word("l"), (1 << 53) + 1]), fl.ARRAY_FLOAT64) == (fo.OK, [_bits(2.0**53)], b"")
    m = (1 << 64) - 1
    assert _cell(_arr([word("u"), m]), fl.ARRAY_FLOAT64) == (fo.OK, [_bits(float(m))], b"")
    assert _cell(_arr([word("u"), 1 << 63]), fl.ARRAY_INT64)[0] == fo.CONVERT  # "unsigned integer value overflows int64"


def test_first_error_wins():
    """the walk returns at the first failing element: a CORRUPT string range behind a CONVERT element is CONVERT"""
    items = [word("t"), word('"', S), 99]
    assert _cell(_arr(items), fl.ARRAY_STRING)[0] == fo.CONVERT
    assert _cell(_arr([word('"', S), 99, word("t")]), fl.ARRAY_STRING)[0] == fo.CORRUPT


def test_nested_scopes():
    """AsFloat: a nested `[` is a tag like any other, `unable to convert type` (parsed_array.go:175-176).  AsString /
    AsStringCvt: AdvanceIter steps over it by its link (parsed_json.go:325-341), then `element in array is not string`
    (parsed_array.go:307-308) / StringCvt's `cannot convert type` (parsed_json.go:798); a link outside the array's tape
    is AdvanceIter's `element extends beyond tape` (:340-342)"""
    items = [word('"', S), 1] + [word("[", 9), word("]", 7)] + [word('"', S), 1]
    assert _cell(_arr([word("[", 7), word("]", 5)]), fl.ARRAY_FLOAT64)[0] == fo.CONVERT
    assert _cell(_arr(items), fl.ARRAY_STRING)[0] == fo.CONVERT
    assert _cell(_arr(items), fl.ARRAY_STRING_CVT)[0] == fo.CONVERT
    bad = [word('"', S), 1] + [word("[", 99), word("]", 7)] + [word('"', S), 1]
    assert _cell(_arr(bad), fl.ARRAY_STRING_CVT)[0] == fo.CORRUPT


def test_truncated_array():
    """the array's tape is Tape[:cur] (parsed_json.go:1032): AsFloat reading a tag past it panics, a value word past it
    is `corrupt input: expected integer, but no more values` (parsed_array.go:163-165); AsString's AdvanceIter meets
    its end exactly and returns TypeNone with no error (parsed_json.go:296-300)"""
    # [ l 1 t   with '[' pointing one past the t: no ']' inside the array's tape
    t = [word("[", 8), word("l"), 1, word("t")]
    assert _cell(t + [word("]", 4)], fl.ARRAY_FLOAT64)[0] == fo.CONVERT   # 't' is read as a tag
    t2 = [word("[", 7), word("l"), 1, word("]", 4)]  # '[' ends the array's tape at the ']'
    assert _cell(t2, fl.ARRAY_INT64)[0] == fo.CORRUPT
    t3 = [word("[", 6), word("l"), word("]", 4)]  # the value word of `l` lies past the array's tape
    assert _cell(t3, fl.ARRAY_UINT64)[0] == fo.CORRUPT
    t4 = [word("[", 7), word("t"), word("f"), word("]", 4)]
    assert _cell(t4, fl.ARRAY_STRING_CVT) == (fo.OK, [4, 5], b"truefalse")


def test_not_an_array_and_fresh_element():
    """Iter.Array: `if i.t != TagArrayStart { ... "next item is not array" }` (parsed_json.go:1024-1026)"""
    assert _cell([word("t")], fl.ARRAY_FLOAT64)[0] == fo.CONVERT
    assert _cell([word("{", 6), word("}", 4)], fl.ARRAY_STRING)[0] == fo.CONVERT
    t = np.array([word("r", 7), word("{", 6), word('"', S), 1, word("N", 1), word("n"), word("}", 1), word("r", 0)],
                 dtype=np.uint64)
    ((c, e, d),) = fl.find_lists(t, b"a", b"", [[b"a"]], [fl.ARRAY_FLOAT64], [0])[0]
    assert (c.status, e, d) == (fo.CONVERT, [], b"")


def test_string_cvt_scalars_and_lists():
    """StringCvt (parsed_json.go:775-799): strings raw, l / u in decimal, true / false / null as written, floats as
    appendFloat, whose INF / NaN is an error (:1251-1253)"""
    b = TapeBuilder()
    b.open("r"); b.open("{")
    b.string(b"s"); b.string(b'a"b\n')
    b.string(b"l"); b.number("l", (1 << 64) - 12)
    b.string(b"u"); b.number("u", (1 << 64) - 1)
    b.string(b"d"); b.number("d", _bits(1e21))
    b.string(b"n"); b.atom("n")
    b.string(b"i"); b.number("d", 0x7FF0000000000000)
    b.string(b"o"); b.open("{"); b.close()
    b.string(b"v"); b.open("["); b.string(b"x"); b.number("l", 7); b.atom("t"); b.number("d", _bits(0.1)); b.close()
    b.close(); b.close()
    tape, strs, msg = b.build()
    want = {b"s": b'a"b\n', b"l": b"-12", b"u": b"18446744073709551615", b"d": b"1e+21", b"n": b"null"}
    for k, text in want.items():
        ((c, _, d),) = fl.find_lists(tape, strs, msg, [[k]], [fl.STRING_CVT])[0]
        assert (c.status, c.value, d) == (fo.OK, len(text), text), k
    for k in (b"i", b"o"):
        assert fl.find_lists(tape, strs, msg, [[k]], [fl.STRING_CVT])[0][0][0].status == fo.CONVERT
    ((c, e, d),) = fl.find_lists(tape, strs, msg, [[b"v"]], [fl.ARRAY_STRING_CVT])[0]
    assert (c.status, e, d) == (fo.OK, [1, 1, 4, 3], b"x7true0.1")


def test_string_cvt_matches_the_formatter_cases():
    """STRING_CVT of every double of fmt_values' formatter cases is appendFloat's text"""
    xs = np.concatenate([fmt_values.powers_of_two()[::7], fmt_values.notation_edges(), fmt_values.integers_near_2_53()[::50]])
    t = np.array(_obj([word("[", 4 + 2 * len(xs) + 2)] + [w for x in xs.tolist() for w in (word("d"), x)] + [word("]", 4)]),
                 dtype=np.uint64)
    ((c, e, d),) = fl.find_lists(t, b"a", b"", [[b"a"]], [fl.ARRAY_STRING_CVT], [0])[0]
    want = [format_float(fo._f64(x)) for x in xs.tolist()]
    assert c.status == fo.OK and e == [len(w) for w in want] and d == b"".join(want)


# ---- against Python's json -----------------------------------------------------------------------------------------

def _num(x):
    return isinstance(x, (int, float)) and not isinstance(x, bool)


def expected(v, kind):
    """(status, elems, bytes) the list cell of JSON value v gives, or None where json alone cannot tell (float to
    integer conversions)"""
    if not isinstance(v, list):
        return fo.CONVERT, [], b""
    if kind == fl.ARRAY_FLOAT64:
        return (fo.OK, [_bits(x) for x in v], b"") if all(_num(x) for x in v) else (fo.CONVERT, [], b"")
    if kind in (fl.ARRAY_INT64, fl.ARRAY_UINT64):
        lo = -(1 << 63) if kind == fl.ARRAY_INT64 else 0
        hi = 1 << 63 if kind == fl.ARRAY_INT64 else 1 << 64
        if all(isinstance(x, int) and not isinstance(x, bool) and lo <= x < hi for x in v):
            return fo.OK, [x & fl.M64 for x in v], b""
        for x in v:  # the first element json can judge decides, if it comes before any float
            if isinstance(x, float):
                return None
            if not (isinstance(x, int) and not isinstance(x, bool)):
                return fo.CONVERT, [], b""
            if not lo <= x < hi:
                return (fo.CONVERT, [], b"") if -(1 << 63) <= x < 1 << 64 else None
        return None
    if kind == fl.ARRAY_STRING:
        if all(isinstance(x, str) for x in v):
            xs = [x.encode("utf-8", "surrogatepass") for x in v]
            return fo.OK, [len(x) for x in xs], b"".join(xs)
        return fo.CONVERT, [], b""
    xs = []
    for x in v:
        if isinstance(x, (list, dict)):
            return fo.CONVERT, [], b""
        if isinstance(x, str):
            xs.append(x.encode("utf-8", "surrogatepass"))
        elif x is None or isinstance(x, bool):
            xs.append(json.dumps(x).encode())
        elif isinstance(x, int) and -(1 << 63) <= x < 1 << 64:
            xs.append(str(x).encode())
        else:
            xs.append(format_float(float(x)))
    return fo.OK, [len(x) for x in xs], b"".join(xs)


def agree(tape, strs, msg, paths, docs):
    """every list cell of every path against json.loads of its row's document; returns the cells checked that hold a
    list"""
    rows = fo.foreach_roots(tape)
    assert len(rows) == len(docs)
    n = 0
    for kind in LISTS:
        cells = fl.find_lists(tape, strs, msg, paths, [kind] * len(paths), rows)
        for p, path in enumerate(paths):
            for r, (c, elems, data) in enumerate(cells[p]):
                if c.status != fo.OK:
                    assert (elems, data, c.value) == ([], b"", 0)
                v, found = _at(docs[r], path)
                if not found or not path:  # (a path of 0 segments is ErrPathNotFound)
                    assert c.status in (fo.NOT_FOUND, fo.NOT_OBJECT), (path, r)
                    continue
                want = expected(v, kind)
                if want is None:
                    continue
                assert (c.status, elems, data) == want, (kind, path, r, c, elems[:5], want[1][:5])
                assert c.status != fo.OK or c.value == len(elems)
                n += isinstance(v, list)
    return n


def _load(doc):
    try:
        return json.loads(doc, object_pairs_hook=_first_pairs)
    except (_Dup, ValueError):
        return None


@pytest.mark.parametrize("name", TAPE_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures_against_json(oracle, name, copy):
    doc = load_fixture(name)
    v = _load(doc)
    if v is None:
        pytest.skip("duplicate keys")
    rc, tape, strs, (off, ln) = oracle.parse(doc, copy_strings=copy)
    assert rc == 0
    agree(tape, strs, doc[off:off + ln], harvest(doc), [v])


def test_mesh_columns(oracle):
    """mesh.json: positions / normals / tex0 bit-exact floats, indices / colors ints, influences ([[1.0, 0], ...]) not
    numbers"""
    doc = load_fixture("mesh")
    v = json.loads(doc)
    rc, tape, strs, (off, ln) = oracle.parse(doc)
    msg = doc[off:off + ln]
    for key, kind, conv in [("positions", fl.ARRAY_FLOAT64, _bits), ("normals", fl.ARRAY_FLOAT64, _bits),
                            ("tex0", fl.ARRAY_FLOAT64, _bits), ("indices", fl.ARRAY_INT64, int),
                            ("colors", fl.ARRAY_INT64, int), ("indices", fl.ARRAY_UINT64, int)]:
        ((c, e, _),) = fl.find_lists(tape, strs, msg, [[key.encode()]], [kind])[0]
        assert c.status == fo.OK and e == [conv(x) for x in v[key]], key
    for kind in LISTS:
        ((c, e, _),) = fl.find_lists(tape, strs, msg, [[b"influences"]], [kind])[0]
        assert (c.status, e) == (fo.CONVERT, []), kind


def ndjson_records(name):
    """the fixtures whose root holds an array of objects, as (records, NDJSON bytes)"""
    v = json.loads(load_fixture(name))
    recs = {"twitter": lambda: v["statuses"], "github_events": lambda: v, "random": lambda: v["result"],
            "update-center": lambda: list(v["plugins"].values())}[name]()
    return recs, b"\n".join(json.dumps(r, ensure_ascii=False).encode("utf-8", "surrogatepass") for r in recs)


NDJSON_FIXTURES = ["twitter", "github_events", "random", "update-center"]


def ndjson_paths(recs):
    seen, out = set(), []
    for r in recs[:20]:
        for p in harvest(json.dumps(r).encode(), 60):
            if tuple(p) not in seen:
                seen.add(tuple(p))
                out.append(p)
    return out


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
@pytest.mark.parametrize("copy", [True, False])
def test_ndjson_against_json(oracle, name, copy):
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
    assert rc == 0
    assert agree(tape, strs, nd[off:off + ln], ndjson_paths(recs), recs) > 0
    if name == "update-center":
        cells = fl.find_lists(tape, strs, nd[off:off + ln], [[b"labels"]], [fl.ARRAY_STRING])[0]
        assert sum(c.status == fo.OK and len(e) > 0 for c, e, _ in cells) > 100
