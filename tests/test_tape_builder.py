"""The tape builder (tests/tape_builder.py) writes what the parser writes: for random documents JSON can express, in both
copy modes, its tape and Strings.B equal the oracle parse's.  This is what lets the device MarshalJSON tests trust tapes
the builder places at their edges."""
import struct

import numpy as np
import pytest

from tests import marshal_oracle as mo
from tests.tape_builder import STRINGBUFBIT, TapeBuilder

# escapes and what they stand for; a string with any of them is unescaped into Strings.B even without copy_strings
_ESCAPES = [(b'\\"', b'"'), (b"\\\\", b"\\"), (b"\\/", b"/"), (b"\\b", b"\b"), (b"\\f", b"\f"), (b"\\n", b"\n"),
            (b"\\r", b"\r"), (b"\\t", b"\t"), (b"\\u0001", b"\x01"), (b"\\u00e9", b"\xc3\xa9"), (b"\\u20ac", b"\xe2\x82\xac")]
_PLAIN = [b"a", b"Z", b"0", b" ", b"~", b"\xc3\xa9", b"\xe2\x82\xac", b"\xf0\x9f\x98\x80"]


def _string(rng, b, copy):
    parts = [(_ESCAPES[rng.integers(len(_ESCAPES))] if rng.random() < 0.15 else (p, p))
             for p in (_PLAIN[rng.integers(len(_PLAIN))] for _ in range(int(rng.choice([0, 1, 3, 31, 32, 33, 70]))))]
    text = b"".join(t for t, _ in parts)
    body = b"".join(u for _, u in parts)
    b.message += b'"'
    if copy or text != body:
        b.string(body, copy=True)
        b.message += text
    else:
        b.string(body, copy=False)
    b.message += b'"'


def _number(rng, b):
    k = rng.integers(4)
    if k == 0:
        v = int(rng.integers(-(1 << 63), 1 << 63, dtype=np.int64))
        b.number("l", v)
        b.message += b"%d" % v
    elif k == 1:
        v = int(rng.integers(1 << 63, 1 << 64, dtype=np.uint64))
        b.number("u", v)
        b.message += b"%d" % v
    else:
        x = float(10.0 ** rng.uniform(-30, 30) * rng.choice([-1, 1])) if k == 2 else struct.unpack(
            "<d", struct.pack("<Q", int(rng.integers(0, 0x7FF0000000000000, dtype=np.uint64))))[0]
        b.number("d", struct.unpack("<Q", struct.pack("<d", x))[0])
        b.message += repr(x).encode()


def _value(rng, b, copy, depth):
    k = rng.integers(9) if depth < 6 else 2 + rng.integers(7)
    if k in (0, 1):
        kind = "{[" [k]
        b.open(kind)
        b.message += kind.encode()
        for j in range(int(rng.choice([0, 1, 2, 5]))):
            if j:
                b.message += b","
            if kind == "{":
                _string(rng, b, copy)
                b.message += b":"
            _value(rng, b, copy, depth + 1)
        b.close()
        b.message += b"}" if kind == "{" else b"]"
    elif k in (2, 3):
        _string(rng, b, copy)
    elif k in (4, 5):
        _number(rng, b)
    else:
        t = "tfn"[k - 6]
        b.atom(t)
        b.message += {"t": b"true", "f": b"false", "n": b"null"}[t]


def _document(rng, copy, ndjson):
    """a builder holding the tape of a random document, and the document's text as its message"""
    b = TapeBuilder()
    for r in range(int(rng.integers(1, 4)) if ndjson else 1):
        if r:
            b.message += b"\n"
        b.open("r")
        kind = "{["[rng.integers(2)]
        b.open(kind)
        b.message += kind.encode()
        for j in range(int(rng.integers(0, 4))):
            if j:
                b.message += b","
            if kind == "{":
                _string(rng, b, copy)
                b.message += b":"
            _value(rng, b, copy, 1)
        b.close(2)
        b.message += b"}" if kind == "{" else b"]"
    return b


@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("ndjson", [False, True])
def test_builder_writes_the_parsers_tape(oracle, copy, ndjson):
    rng = np.random.default_rng(20261015 + 2 * copy + ndjson)
    for _ in range(300):
        b = _document(rng, copy, ndjson)
        tape, strs, msg = b.build()
        rc, want, want_strs, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
        assert rc == 0 and (off, ln) == (0, len(msg)), msg
        assert np.array_equal(tape, want), msg
        assert strs == want_strs, msg
        assert mo.marshal(tape, strs, msg) == mo.marshal(want, want_strs, msg)


def _resolved(tape, strs, msg):
    """the tape with every string offset replaced by the bytes it points at"""
    out, i = [], 0
    while i < len(tape):
        w = int(tape[i])
        if w >> 56 == ord('"'):
            v, n = w & ((1 << 56) - 1), int(tape[i + 1])
            buf, off = (strs, v - STRINGBUFBIT) if v & STRINGBUFBIT else (msg, v)
            out += ['"', bytes(buf[off:off + n])]
            i += 2
        else:
            out.append(w)
            i += 1
    return out


def test_bulk_items_match_the_parser(oracle):
    """the numpy-written runs (nesting, numbers, fillers) hold the parser's words; their keys share one copy in
    Strings.B, so strings are compared by their bytes"""
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    b.nest("[", 5)
    b.close(5)
    b.nest("{", 4, key=b"ab")
    b.close(4)
    d = [0.5, -1e-7, 5e-324, 1.7976931348623157e308]
    b.numbers("d", [struct.unpack("<Q", struct.pack("<d", x))[0] for x in d])
    b.numbers("l", [0, 1, (1 << 64) - 1, 1 << 63])
    b.open("{")
    b.numbers("u", [1 << 63, (1 << 64) - 1], key=b"k")
    assert b.pad_members_to(b.n + 11) == (1, 2)
    b.close()
    assert b.pad_to(b.n + 3, "t") == 3
    b.atoms("fn")
    b.close(2)
    tape, strs, _ = b.build()
    text = (b'[[[[[[]]]]],{"ab":{"ab":{"ab":{}}}},' + b",".join(repr(x).encode() for x in d) +
            b',0,1,-1,-9223372036854775808,{"k":9223372036854775808,"k":18446744073709551615,"k":null,"k":0,"k":0},'
            b'true,true,true,false,null]')
    rc, want, want_strs, (off, ln) = oracle.parse(text)
    assert rc == 0 and (off, ln) == (0, len(text))
    assert _resolved(tape, strs, b"") == _resolved(want, want_strs, text)
    assert mo.marshal(tape, strs) == mo.marshal(want, want_strs, text)


def test_grammar_mode_refuses_what_json_cannot_express():
    b = TapeBuilder()
    with pytest.raises(AssertionError):
        b.atom("n")  # outside a root
    b.open("r")
    b.open("{")
    with pytest.raises(AssertionError):
        b.number("l", 1)  # a key that is no string
    b.string(b"k")
    with pytest.raises(AssertionError):
        b.close()  # an object closed behind its key
    r = TapeBuilder(raw=True)
    r.open("r")
    r.open("{")
    r.number("l", 1)
    r.close(2)
    tape, strs, msg = r.build()
    with pytest.raises(mo.MalformedTape):
        mo.marshal(tape, strs, msg)
