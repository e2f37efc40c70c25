"""The restatement of ForEach + FindElement + the accessors (tests/find_oracle.py) pinned on the reference's own
expectations: TestObject_FindPath (parsed_object_test.go:10-131), ExampleIter_FindElement and ExampleParsedJson_ForEach
(parsed_json_test.go:1235-1315), the parking-citations count (ndjson_test.go:294-315), countWhere, and the error cases
of the functions it ports.  CPU only: tapes come from the oracle's parse, the tape builder and the Deserialize
restatement."""
import struct

import numpy as np
import pytest

from tests import find_oracle as fo
from tests.marshal_oracle import marshal
from tests.tape_builder import STRINGBUFBIT, TapeBuilder, word
from tests.util import golden, load_fixture, tricky_ndjson

IMAGE = b"""{
    "Image":
    {
        "Animated": false,
        "Height": 600,
        "IDs":
        [
            116,
            943,
            234,
            38793
        ],
        "Thumbnail":
        {
            "Height": 125,
            "Url": "http://www.example.com/image/481989943",
            "Width": 100
        },
        "Title": "View from 15th Floor",
        "Width": 800
    },
\t"Alt": "Image of city"
}"""


def _parse(oracle, msg, ndjson=False, copy=True):
    rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
    assert rc == 0
    return tape, strs, msg[off:off + ln]


def _cells(tape, strs, msg, path, kind=fo.ELEMENT):
    return fo.find(tape, strs, msg, [path], [kind])[0]


def _as_root(tape, i):
    """the element whose head word is at i, alone under a root at slot 0 (links moved by 1 - i)"""
    t = int(tape[i]) >> 56
    end = (int(tape[i]) & fo.VAL) if t in b"{[" else i + (2 if t in b'"lud' else 1)
    out, k = [word("r", end - i + 2)], i
    while k < end:
        w = int(tape[k])
        if (w >> 56) in b'"lud':
            out += [w, int(tape[k + 1])]
            k += 2
            continue
        out.append(w + 1 - i if (w >> 56) in b"{[}]" else w)
        k += 1
    return out + [word("r", 0)]


def _f(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


@pytest.mark.parametrize("copy", [True, False])
def test_object_find_path_table(oracle, copy):
    """every row of TestObject_FindPath: type, and the value through the MarshalJSON restatement; "404" is NOT_FOUND"""
    tape, strs, msg = _parse(oracle, IMAGE, copy=copy)
    rows = [([b"Alt"], ord('"'), b'"Image of city"'), ([b"Image", b"Animated"], ord("f"), b"false"),
            ([b"Image", b"Thumbnail", b"Url"], ord('"'), b'"http://www.example.com/image/481989943"'),
            ([b"Image", b"Height"], ord("l"), b"600"),
            ([b"Image", b"Thumbnail"], ord("{"), b'{"Height":125,"Url":"http://www.example.com/image/481989943","Width":100}'),
            ([b"Image", b"IDs"], ord("["), b"[116,943,234,38793]")]
    for path, tag, text in rows:
        (c,) = _cells(tape, strs, msg, path)
        assert (c.status, c.tag) == (fo.OK, tag), path
        wrapped = _as_root(tape, c.index)
        assert marshal(np.array(wrapped, dtype=np.uint64), strs, msg) == text, path
    assert _cells(tape, strs, msg, [b"Image", b"NonEx"])[0].status == fo.NOT_FOUND


def test_example_iter_find_element(oracle):
    """ExampleIter_FindElement: Image/Thumbnail/Width is int 100"""
    tape, strs, msg = _parse(oracle, IMAGE)
    (c,) = _cells(tape, strs, msg, [b"Image", b"Thumbnail", b"Width"], fo.INT64)
    assert (c.status, c.tag, c.value) == (fo.OK, ord("l"), 100)
    (c,) = _cells(tape, strs, msg, [b"Image", b"Thumbnail", b"Width"], fo.FLOAT64)
    assert c.value == _f(100.0)


def test_example_foreach(oracle):
    """ExampleParsedJson_ForEach: one row, Image/URL is the string http://example.com/example.gif"""
    tape, strs, msg = _parse(oracle, b'{"Image":{"URL":"http://example.com/example.gif"}}')
    (c,) = _cells(tape, strs, msg, [b"Image", b"URL"], fo.STRING)
    assert (c.status, c.tag, c.value) == (fo.OK, ord('"'), b"http://example.com/example.gif")


@pytest.mark.parametrize("copy", [True, False])
def test_parking_citations_make_hond(oracle, copy):
    """ndjson_test.go:294-315: 1000 rows, Make == HOND in 116 of them"""
    g = golden("G18_G19_fixtures")["parking_citations"]
    tape, strs, msg = _parse(oracle, load_fixture("parking-citations"), ndjson=True, copy=copy)
    cells = _cells(tape, strs, msg, [b"Make"], fo.STRING)
    assert len(cells) == g["roots"] == 1000
    assert sum(c.status == fo.OK and c.value == b"HOND" for c in cells) == g["make_hond"] == 116


@pytest.mark.parametrize("copy", [True, False])
def test_agrees_with_count_where(oracle, copy):
    """countWhere(key, value) counts the rows whose FindElement(key) is a string equal to value, for every key of the
    tricky records"""
    nd, recs = tricky_ndjson()
    tape, strs, msg = _parse(oracle, nd, ndjson=True, copy=copy)
    keys = {b"Make", b"", b"x", b"a", b"make", b"Make ", b"Mak", b"t", b"nope"}
    for key in sorted(keys):
        cells = _cells(tape, strs, msg, [key], fo.STRING)
        assert len(cells) == len(recs)
        for value in (b"HOND", b"TOYT", b"", b"HOND "):
            want = oracle.count_where(tape, strs, msg, key, value)
            assert (len(cells), sum(c.status == fo.OK and c.value == value for c in cells)) == want, (key, value)
    # non-object roots are NOT_OBJECT, not NOT_FOUND
    st = [c.status for c in _cells(tape, strs, msg, [b"Make"])]
    assert st[recs.index(b'["Make","HOND"]')] == st[recs.index(b"[]")] == fo.NOT_OBJECT
    assert st[recs.index(b"{}")] == fo.NOT_FOUND


def test_duplicates_and_non_object_first():
    """the first member with the key decides, even when its value is not an object and a later one is"""
    b = TapeBuilder()
    b.open("r"); b.open("{")
    b.string(b"a"); b.number("l", 1)
    b.string(b"a"); b.open("{"); b.string(b"b"); b.number("l", 2); b.close()
    b.close(); b.close()
    tape, strs, msg = b.build()
    (c,) = _cells(tape, strs, msg, [b"a"], fo.INT64)
    assert (c.status, c.value) == (fo.OK, 1)
    assert _cells(tape, strs, msg, [b"a", b"b"])[0].status == fo.NOT_OBJECT
    assert _cells(tape, strs, msg, [])[0].status == fo.NOT_FOUND  # a path of 0 segments
    assert _cells(tape, strs, msg, [b"a", b"b", b"c"])[0].status == fo.NOT_OBJECT


@pytest.mark.parametrize("copy", [True, False])
def test_escaped_and_empty_keys(oracle, copy):
    """keys compare on their unescaped bytes, read from Strings.B or (no-copy, no escape) from the message"""
    tape, strs, msg = _parse(oracle, b'{"M\\u0061ke":"x","":{"":true},"q\\"":[1],"plain":{"y":2}}', copy=copy)
    from_msg = [(int(w) >> 56) == ord('"') and not int(w) & STRINGBUFBIT for w in tape[2::2]]
    assert any(from_msg) != copy  # the no-copy parse leaves the unescaped keys in the message
    assert _cells(tape, strs, msg, [b"Make"], fo.STRING)[0].value == b"x"
    assert _cells(tape, strs, msg, [b"", b""], fo.BOOL)[0].astuple()[::3] == (fo.OK, 1)
    assert _cells(tape, strs, msg, [b'q"'])[0].tag == ord("[")
    assert _cells(tape, strs, msg, [b'q"', b"0"])[0].status == fo.NOT_OBJECT  # arrays are never entered
    assert _cells(tape, strs, msg, [b"plain", b"y"], fo.INT64)[0].astuple()[::3] == (fo.OK, 2)


ROOT_LOOKALIKES = (b'{"a":8214565720323785000,"b":"x"}\n{"a":1,"b":"y"}\n{"a":1e242,"b":"z"}\n'
                   b'{"a":[8286623314361712639,-1.5e241],"b":"w"}\n{"a":{"c":8214565720323784704},"b":"v"}')


@pytest.mark.parametrize("copy", [True, False])
def test_rows_skip_value_words_that_look_like_roots(oracle, copy):
    """int64s from 0x72 << 56 and doubles near 1e242-1e246 have value words whose top byte is 'r': they are no rows"""
    tape, strs, msg = _parse(oracle, ROOT_LOOKALIKES, ndjson=True, copy=copy)
    lookalikes = [i for i in range(1, len(tape)) if (int(tape[i]) >> 56) == ord("r") and (int(tape[i]) & fo.VAL) > i
                  and (int(tape[i - 1]) >> 56) in b"lud"]
    assert len(lookalikes) == 3  # (0x72 << 56 itself points at slot 0: no root open)
    assert list(fo.roots(tape)) == list(fo.foreach_roots(tape))
    assert [c.value for c in _cells(tape, strs, msg, [b"b"], fo.STRING)] == [b"x", b"y", b"z", b"w", b"v"]


def test_rows_are_foreach_roots_on_parsed_tapes(oracle):
    from tests.util import TAPE_FILES
    for name in ["parking-citations"] + TAPE_FILES[:6]:
        tape, strs, msg = _parse(oracle, load_fixture(name), ndjson=name == "parking-citations")
        assert list(fo.roots(tape)) == list(fo.foreach_roots(tape)), name


def test_nop_runs():
    """N words are skipped as each function skips them: AdvanceInto by their value, AdvanceIter by one more than their
    value (0 is "invalid nop skip"), Advance by one more than their value (0 included)"""
    S = STRINGBUFBIT

    def cell(t, kind=fo.INT64):
        (c,) = fo.find(np.array(t, dtype=np.uint64), b"ab", b"", [[b"a"]], [kind])[0]
        return c.status, c.index, c.value

    # in front of the root's object (ForEach's AdvanceInto)
    assert cell([word("r", 10), word("N", 2), word("N", 1), word("{", 9), word('"', S), 1, word("l"), 7, word("}", 3),
                 word("r", 0)]) == (fo.OK, 6, 7)
    # between a key and its value (FindPath's AdvanceIter)
    t2 = [word("r", 10), word("{", 9), word('"', S), 1, word("N", 1), word("n"), word("l"), 5, word("}", 1), word("r", 0)]
    assert cell(t2) == (fo.OK, 6, 5)
    t2[4] = word("N", 0)
    assert cell(t2)[0] == fo.CORRUPT
    # in front of a skipped value (FindPath's Advance)
    assert cell([word("r", 13), word("{", 12), word('"', S | 1), 1, word("N", 0), word("l"), 9, word('"', S), 1,
                 word("l"), 4, word("}", 1), word("r", 0)]) == (fo.OK, 9, 4)


def test_nop_runs_from_deserialize():
    """Deserialize writes N runs for skipped tags (parsed_serialize.go); the rows and their values do not change"""
    from tests import serialize_oracle as so
    b = TapeBuilder()
    for k in range(3):
        b.open("r"); b.open("{"); b.string(b"k"); b.number("l", k); b.close(); b.close()
    tape, strs, msg = b.build()
    src = so.serialize(tape, strs, msg)
    t2, s2, m2 = so.deserialize(src)
    t2 = np.array(t2, dtype=np.uint64)
    cells = fo.find(t2, s2, m2, [[b"k"]], [fo.INT64])[0]
    assert [(c.status, c.value) for c in cells] == [(fo.OK, k) for k in range(3)]
    # the same tape with its first member turned into a run of nops
    t3 = t2.copy()
    first = [c.index for c in cells]
    for r, hi in enumerate(first):
        t3[hi - 2:hi + 2] = [word("N", 4), word("N", 3), word("N", 2), word("N", 1)]
    assert [c.status for c in fo.find(t3, s2, m2, [[b"k"]], [fo.INT64])[0]] == [fo.NOT_FOUND] * 3


def _one_value(tag, payload):
    b = TapeBuilder()
    b.open("r"); b.open("{"); b.string(b"v"); b.number(tag, payload); b.close(); b.close()
    return b.build()


@pytest.mark.parametrize("tag,payload,kind,want", [
    # Int: d > 2^63 or < -2^63 is an error; exactly 2^63 passes the check and CVTTSD2SQ gives math.MinInt64
    ("d", _f(2.0 ** 63), fo.INT64, (fo.OK, 1 << 63)),
    ("d", _f(-2.0 ** 63), fo.INT64, (fo.OK, 1 << 63)),
    ("d", _f(2.0 ** 63 * (1 + 2 ** -52)), fo.INT64, (fo.CONVERT, 0)),
    ("d", _f(-2.0 ** 63 * (1 + 2 ** -52)), fo.INT64, (fo.CONVERT, 0)),
    ("d", _f(-1.9), fo.INT64, (fo.OK, (1 << 64) - 1)),
    ("d", _f(-0.0), fo.INT64, (fo.OK, 0)),
    ("u", (1 << 63) - 1, fo.INT64, (fo.OK, (1 << 63) - 1)),
    ("u", 1 << 63, fo.INT64, (fo.CONVERT, 0)),
    ("l", (1 << 64) - 1, fo.INT64, (fo.OK, (1 << 64) - 1)),
    # Uint: negative l, negative d, d > 2^64 are errors; exactly 2^64 gives 1<<63 (Go's float64ToUint64 lowering)
    ("d", _f(2.0 ** 64), fo.UINT64, (fo.OK, 1 << 63)),
    ("d", _f(2.0 ** 64 * (1 + 2 ** -52)), fo.UINT64, (fo.CONVERT, 0)),
    ("d", _f(2.0 ** 63), fo.UINT64, (fo.OK, 1 << 63)),
    ("d", _f(2.0 ** 64 - 2048), fo.UINT64, (fo.OK, (1 << 64) - 2048)),
    ("d", _f(-0.0), fo.UINT64, (fo.OK, 0)),
    ("d", _f(-0.5), fo.UINT64, (fo.CONVERT, 0)),
    ("l", (1 << 64) - 1, fo.UINT64, (fo.CONVERT, 0)),
    ("l", (1 << 63) - 1, fo.UINT64, (fo.OK, (1 << 63) - 1)),
    ("u", (1 << 64) - 1, fo.UINT64, (fo.OK, (1 << 64) - 1)),
    # Float: integers rounded to nearest
    ("l", (1 << 63) - 1, fo.FLOAT64, (fo.OK, _f(2.0 ** 63))),
    ("l", (1 << 63), fo.FLOAT64, (fo.OK, _f(-2.0 ** 63))),
    ("u", (1 << 64) - 1, fo.FLOAT64, (fo.OK, _f(2.0 ** 64))),
    ("u", (1 << 53) + 1, fo.FLOAT64, (fo.OK, _f(2.0 ** 53))),
    ("d", _f(-0.0), fo.FLOAT64, (fo.OK, _f(-0.0))),
    ("l", 5, fo.BOOL, (fo.CONVERT, 0)),
    ("l", 5, fo.STRING, (fo.CONVERT, b"")),
])
def test_conversion_boundaries(tag, payload, kind, want):
    tape, strs, msg = _one_value(tag, payload)
    (c,) = fo.find(tape, strs, msg, [[b"v"]], [kind])[0]
    assert (c.status, c.value) == want
    assert (c.tag, c.index) == (ord(tag), 4)


def test_number_texts_convert_like_the_parse(oracle):
    """int64 / uint64 borders of tests/number_values.py through the parse: the accessors see what the parser wrote"""
    from tests.number_values import integers
    for text in integers():
        rc, tape, strs, (off, ln) = oracle.parse(b'{"v":' + text + b"}")
        if rc:
            continue
        (ci,) = fo.find(tape, strs, b"", [[b"v"]], [fo.INT64])[0]
        t, p = int(tape[4]) >> 56, int(tape[5])
        if t == ord("l"):
            assert (ci.status, ci.value) == (fo.OK, p), text
        elif t == ord("u"):
            assert ci.status == (fo.OK if p < 1 << 63 else fo.CONVERT), text


def test_corrupt_tapes():
    ok = [word("r", 6), word("{", 5), word('"', STRINGBUFBIT), 1, word("l"), 3, word("}", 1), word("r", 0)]
    ok[0], ok[1], ok[6] = word("r", 8), word("{", 7), word("}", 1)
    base = np.array(ok, dtype=np.uint64)

    def status(t, strs=b"a", path=(b"a",), kind=fo.INT64):
        return fo.find(np.array(t, dtype=np.uint64), strs, b"", [list(path)], [kind])[0][0].status

    assert status(base) == fo.OK
    assert status(base, strs=b"") == fo.CORRUPT                   # key range outside Strings.B
    t = base.copy(); t[2] = word('"', 5)                           # key range outside the (empty) message
    assert status(t) == fo.CORRUPT
    t = base.copy(); t[1] = word("{", 1)                           # object ends before its start
    assert status(t) == fo.CORRUPT
    t = base.copy(); t[1] = word("{", 99)                          # object beyond the root's tape
    assert status(t) == fo.CORRUPT
    t = base.copy(); t[0] = word("r", 99)                          # root beyond the tape
    assert len(fo.find(t, b"a", b"", [[b"a"]], [fo.INT64])[0]) == 1 and status(t) == fo.CORRUPT
    t = base.copy(); t[4] = word("{", 2)                           # the found value points backwards
    assert status(t, kind=fo.ELEMENT) == fo.CORRUPT
    t = base.copy(); t[1] = word("r", 0)                           # a root word whose value is 0: Tape[:0-1] panics
    assert status(t) == fo.CORRUPT
    t = base.copy(); t[1] = word("N", 0)                           # AdvanceInto's nop of 0 ends the iterator
    assert status(t) == fo.NOT_FOUND
    t = base.copy(); t[1] = word("l")                              # the root holds a number
    assert status(t) == fo.NOT_OBJECT
    t = base.copy(); t[5] = word("N", 50)                          # the value word is past the object: still read
    assert status(t) == fo.OK


def test_fresh_element_when_the_tape_ends_exactly():
    """AdvanceIter that meets the end of the object's tape returns TypeNone with a nil error: the Element is a fresh one"""
    t = np.array([word("r", 7), word("{", 6), word('"', STRINGBUFBIT), 1, word("N", 1), word("n"), word("}", 1),
                  word("r", 0)], dtype=np.uint64)
    t[4] = word("N", 1)  # AdvanceIter: off 5 + 1 = 6 = end of Tape[:6]
    t[1] = word("{", 6)
    (c,) = fo.find(t, b"a", b"", [[b"a"]], [fo.ELEMENT])[0]
    assert c.astuple() == (fo.OK, 0, -1, 0)
    assert fo.find(t, b"a", b"", [[b"a"]], [fo.INT64])[0][0].status == fo.CONVERT


def test_rows_in_tape_order():
    b = TapeBuilder()
    for k in range(5):
        b.open("r"); b.open("{"); b.string(b"k"); b.number("l", k); b.close(); b.close()
    tape, strs, msg = b.build()
    assert list(fo.roots(tape)) == [8 * k for k in range(5)]
    assert [c.value for c in fo.find(tape, strs, msg, [[b"k"]], [fo.INT64])[0]] == list(range(5))
