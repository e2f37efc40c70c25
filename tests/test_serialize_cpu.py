"""The serializer oracle (tests/serialize_oracle.py) checked without a GPU: streams pinned byte for byte from the layout
of parsed_serialize.go, the size varint, and round trips through the oracle's Deserialize."""
import struct

import pytest

from tests import marshal_oracle as mo
from tests import serialize_oracle as so
from tests.tape_builder import STRINGBUFBIT, TapeBuilder, word
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, golden, load_fixture, unhex

Q = lambda *v: struct.pack("<%dQ" % len(v), *[x & so.M64 for x in v])  # noqa: E731


def test_pinned_flagged_float():
    # r [ e ] r : 0 r|5  1 [|4  2 d|flags  3 payload  4 ]|1  5 r|0 ... as written by hand from Serialize (:275-342)
    tape = [word("r", 6), word("[", 5), word("d", 3), 0x3FF0000000000000, word("]", 1), word("r", 0)]
    s = so.serialize(tape)
    tags = b"r[e]r"
    vals = Q(6, 4, word("d", 3), 0x3FF0000000000000, -5)
    body = b"\x06\0\0" + b"\0\x01\0" + b"\x05\x06\0" + tags + b"\x28\x29\0" + vals
    assert s == b"\x03" + bytes([len(body)]) + body
    assert so.deserialize(s)[0] == tape


def test_pinned_two_roots():
    # two NDJSON roots r "a" r r l 7 r with the string in the message
    tape = [word("r", 4), word('"', 0), 1, word("r", 0), word("r", 8), word("l"), 7, word("r", 4)]
    s = so.serialize(tape, b"", b"a")
    vals = Q(4, 0, 1, -3, 4, 7, -3)  # the last root close: 4 - 7
    body = b"\x08\0\0" + b"\x01\x02\0a" + b"\x06\x07\0" + b'r"rrlr' + b"\x38\x39\0" + vals
    assert s == b"\x03" + bytes([len(body)]) + body
    assert so.deserialize(s) == (tape, b"", b"a")


def test_pinned_nop_run():
    tape = [word("r", 6), word("N", 3), word("N", 2), word("N", 1), word("n"), word("r", 0)]
    s = so.serialize(tape)
    body = b"\x06\0\0" + b"\0\x01\0" + b"\x06\x07\0" + b"rNNNnr" + b"\x10\x11\0" + Q(6, -5)
    assert s == b"\x03" + bytes([len(body)]) + body
    assert so.deserialize(s)[0] == tape


def test_empty_tape():
    assert so.serialize([]) == bytes.fromhex("030c000000000100000100000100")
    assert so.deserialize(so.serialize([])) == ([], b"", b"")


@pytest.mark.parametrize("k", [126, 127, 128, 129, 16382, 16383, 16384, 16385])
def test_size_varint(k):
    """message, tag and value blocks with 1 + raw sizes around 127/128 and 16 383/16 384"""
    for which in ("msg", "tags"):
        b = TapeBuilder()
        b.open("r")
        b.open("[")
        if which == "msg":
            b.string(b"x" * (k - 1))
        else:
            b.atoms(("n", max(k - 5, 1)))
        b.close(2)
        tape, strs, msg = b.build()
        s = so.serialize(tape, strs, msg)
        r = so._Reader(s)
        r.byte()
        assert r.uvarint() == len(s) - r.at
        assert mo.marshal(*so.deserialize(s)) == mo.marshal(tape, strs, msg)


def _oracle_round_trip(tape, strs, msg):
    want = mo.marshal(tape, strs, msg)
    for dedup, seed in (("exact", 0), ("ref", 3), ("none", 0)):
        t2, s2, m2 = so.device_result(so.serialize(tape, strs, msg, dedup=dedup, seed=seed))
        assert mo.marshal(t2, s2, m2) == want


def test_round_trip_fixtures(oracle):
    for name in TAPE_FILES + SMALL_FILES + ["parking-citations"]:
        msg = load_fixture(name)
        for copy in (True, False):
            rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=name == "parking-citations", copy_strings=copy)
            assert rc == 0
            _oracle_round_trip(tape, strs, msg[off:off + ln])


def test_round_trip_golden(oracle):
    g = golden("G16_G17_documents")
    n = 0
    for group, nd in (("parse_nd", True), ("pass_cases", False)):
        for tc in g[group]:
            if tc["want"] is None:
                continue
            js = unhex(tc["js"])
            for copy in (True, False):
                rc, tape, strs, (off, ln) = oracle.parse(js, ndjson=nd, copy_strings=copy)
                _oracle_round_trip(tape, strs, js[off:off + ln])
            n += 1
    assert n == 19


def test_round_trip_fuzz_seeds(oracle):
    parsed = 0
    for name, data in fuzz_corpus("go-corpus"):
        for nd in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=nd)
            if rc == 0:
                parsed += 1
                _oracle_round_trip(tape, strs, data[off:off + ln])
                break
    assert parsed > 50


def test_twitter_and_twitterescaped(oracle):
    out = []
    for name in ("twitter", "twitterescaped"):
        msg = load_fixture(name)
        rc, tape, strs, (off, ln) = oracle.parse(msg)
        out.append(so.serialize(tape, strs, msg[off:off + ln]))
    assert out[0] == out[1]


def test_parking_citations_counts(oracle):
    msg = load_fixture("parking-citations")
    rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=True)
    s = so.serialize(tape, strs, msg[off:off + ln])
    ts, _, m, tags, vals, _ = so.header(s)
    assert (len(m), len(tags), len(vals), len(s)) == (35442, 42000, 632000, 709472)


def test_rejections():
    ok = so.serialize([word("r", 4), word("[", 3), word("]", 1), word("r", 0)])
    so.device_result(ok)
    bad = {
        "version 4": b"\x04" + ok[1:],
        "cut": ok[:-1],
        "unknown tag": ok.replace(b"r[]r", b"r[]x"),
        "block type 3": ok.replace(b"\x04\x05\x00r", b"\x04\x05\x03r"),
    }
    for name, s in bad.items():
        with pytest.raises(so.Rejected):
            so.device_result(s)
    s2 = ok.replace(b"\x04\x05\x00r", b"\x04\x05\x01r")
    with pytest.raises(so.Unsupported):
        so.device_result(s2)
    so.device_result(ok + b"trailing")
    for v in range(4):
        assert so.device_result(bytes([v]) + ok[1:])[0] == [word("r", 4), word("[", 3), word("]", 1), word("r", 0)]
    # an open naming a word that is no close is accepted by the reference when the close is written in time, but not here
    assert STRINGBUFBIT  # (the builder's constants are the oracle's)
