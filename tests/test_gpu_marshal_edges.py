"""Device MarshalJSON (marshal.cuh, fmt.h) at the places where it can go wrong, on tapes written by tests/tape_builder.py
and checked against a plain sequential reference: tests/marshal_oracle.py, and Python's repr / float for doubles.

- the formatter on every double and integer the CPU formatter test runs (tests/fmt_values.py);
- value words whose top byte looks like a tag, at tile edges;
- strings of every byte, every length up to 130 and dense escapes, as keys and values, in Strings.B and the message,
  and the two ends of the string range check;
- heads, value words, opens, closes and keys at word E + s for the tile and group edges E, so that the scans' carries
  (depth, head state, key parity, output offsets) cross them; nesting and arrays wider than a group;
- malformed tapes away from tile 0 and across group edges, capacity and the tape-length limit.

Tapes longer than about a million words get their expected text from string operations, not from the oracle's walk."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

from tests import fmt_values as fv
from tests import marshal_oracle as mo
from tests.tape_builder import STRINGBUFBIT, TapeBuilder, word

gpu = pytest.mark.gpu

OK, ERR_CAPACITY, ERR_TOO_LARGE, ERR_ARGUMENT = 0, 4, 5, 6

_CUH = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "simdjson-go_b200", "csrc", "marshal.cuh")).read()
THREADS = int(re.search(r"constexpr int MJ_THREADS = (\d+);", _CUH).group(1))
ROUNDS = int(re.search(r"constexpr int MJ_ROUNDS = (\d+);", _CUH).group(1))
SHORT = int(re.search(r"constexpr uint64_t MJ_SHORT = (\d+);", _CUH).group(1))
T = THREADS * ROUNDS  # words per tile
G = 1024 * T          # words per group of tiles (one block of scan_groups_kernel)
EDGES = [T, 2 * T, 1023 * T, G, G + T, 2 * G]
SHIFTS = range(-3, 3)


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _upload(tape, strs=b"", msg=b""):
    """device copies; the byte buffers are views of exactly their length, with a byte behind them"""
    import torch
    d_tape = torch.from_numpy(np.ascontiguousarray(tape, dtype=np.uint64).view(np.int64)).cuda()
    d_strs = torch.from_numpy(np.frombuffer(bytes(strs) + b"\0", dtype=np.uint8).copy()).cuda()[:len(strs)]
    d_msg = torch.from_numpy(np.frombuffer(bytes(msg) + b"\0", dtype=np.uint8).copy()).cuda()[:len(msg)]
    torch.cuda.synchronize()
    return d_tape, d_strs, d_msg


def _marshal(ctx, tape, strs=b"", msg=b""):
    rc, n, out = ctx.marshal_device(*_upload(tape, strs, msg))
    return rc, (out.cpu().numpy().tobytes() if rc == OK else None)


def _canary(n):
    import torch
    return torch.full((n,), 0xA5, dtype=torch.uint8, device="cuda")


def _first_difference(got, want, sep=b","):
    g, w = got.split(sep), want.split(sep)
    for k, (a, b) in enumerate(zip(g, w)):
        if a != b:
            return k, a, b
    return len(g), len(g), len(w)


def _doubles_of(bits):
    return np.asarray(bits, dtype=np.uint64).view(np.float64).tolist()


# ---- a. the formatter on the device ---------------------------------------------------------------------------------
def _sig_digits(text):
    m = text.lstrip(b"-").split(b"e")[0].replace(b".", b"").strip(b"0")
    return len(m)


@gpu
def test_formatter_doubles(ctx):
    bits = fv.all_doubles()
    texts = [mo.format_float(x) for x in _doubles_of(bits)]
    for key in (None, b"k"):
        b = TapeBuilder()
        b.open("r")
        b.open("[" if key is None else "{")
        b.numbers("d", bits, key=key)
        b.close(2)
        tape, strs, _ = b.build()
        rc, got = _marshal(ctx, tape, strs)
        pre = b"" if key is None else b'"k":'
        want = (b"[" if key is None else b"{") + b",".join(pre + t for t in texts) + (b"]" if key is None else b"}")
        assert rc == OK
        if got != want:
            k, g, w = _first_difference(got[1:-1], want[1:-1])
            pytest.fail("double %d (bits %#x): device %r, oracle %r" % (k, int(bits[k]), g, w))
    # what needs no restatement: the text reads back as the same double, with no more digits than repr's
    vals = _doubles_of(bits)
    for x, t in zip(vals, got[1:-1].split(b",")):
        t = t[len(b'"k":'):]
        y = float(t)
        assert struct.pack("<d", y) == struct.pack("<d", x), (t, x)
        assert _sig_digits(t) <= _sig_digits(repr(abs(x)).encode()), (t, repr(x))


@gpu
def test_formatter_integers(ctx):
    ints = fv.INTEGERS + [2 ** 63 + 1, 2 ** 64 - 2, 2 ** 63 - 2] + [2 ** 64 - x for x in fv.INTEGERS if x]
    for tag in "lu":
        b = TapeBuilder()
        b.open("r")
        b.open("[")
        b.numbers(tag, ints)
        b.close(2)
        tape, _, _ = b.build()
        signed = [x - (1 << 64) if tag == "l" and x >> 63 else x for x in ints]
        assert _marshal(ctx, tape) == (OK, b"[" + b",".join(b"%d" % x for x in signed) + b"]"), tag


# ---- b. payload words that look like tags ---------------------------------------------------------------------------
LOOKALIKE = b'{}[]r"ludtfn\x00\xff'


def test_lookalike_payloads_are_finite_doubles():
    for top in LOOKALIKE:
        p = top << 56 | 0x0012_3456_789A_BC
        assert (p >> 52) & 0x7FF != 0x7FF


@gpu
def test_payloads_that_look_like_tags_at_tile_edges(ctx):
    """every value word with such a top byte lands as the last word of a tile, the first, and the second"""
    items = [(tag, top << 56 | 0x0012_3456_789A_BC) for tag in "lud" for top in LOOKALIKE]
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    k = 1
    for a in (-1, 0, 1):
        for tag, p in items:
            b.pad_to(k * T + a - 1)  # the head in front of the value word
            b.number(tag, p)
            k += 1
    b.close(2)
    tape, strs, msg = b.build()
    assert _marshal(ctx, tape, strs, msg) == (OK, mo.marshal(tape, strs, msg))


# ---- c. strings -----------------------------------------------------------------------------------------------------
SIX = bytes(c for c in range(0x20) if c not in b"\b\f\n\r\t")  # escaped as \u00XX
TWO = b'"\\\b\f\n\r\t'


def _bodies():
    rng = np.random.default_rng(7)
    out = [bytes([c]) for c in range(256)] + [bytes(range(256)), bytes(range(255, -1, -1))]
    for n in range(0, 131):
        out.append(bytes(rng.integers(0x20, 0x7F, size=n, dtype=np.uint8)).replace(b'"', b"a").replace(b"\\", b"b"))
        out.append(bytes(SIX[i % len(SIX)] for i in range(n)))
        out.append(bytes(TWO[i % len(TWO)] for i in range(n)))
        out.append(bytes(rng.choice(np.frombuffer(SIX + TWO + b"a\x7f\x80\xff", dtype=np.uint8), size=n)))
        out.append(bytes(rng.integers(0, 256, size=n, dtype=np.uint8)))
    return out


@gpu
def test_strings(ctx):
    """as keys and values, in Strings.B and in the message, mixed in one tape that crosses a tile edge"""
    bodies = _bodies()
    assert max(len(s) for s in bodies) > 4 * SHORT
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    b.pad_to(T - 301)
    b.open("{")
    for i, s in enumerate(bodies):
        b.string(s, copy=i % 2 == 0)
        b.string(bodies[-1 - i], copy=i % 4 < 2)
    b.close()
    for i, s in enumerate(bodies):
        b.string(s, copy=i % 3 == 0)
    b.close(2)
    tape, strs, msg = b.build()
    assert _marshal(ctx, tape, strs, msg) == (OK, mo.marshal(tape, strs, msg))


@gpu
@pytest.mark.parametrize("copy", [True, False])
def test_string_range_edges(ctx, copy):
    """a string may end at its buffer's end, and be empty at offset == length; one byte further is malformed"""
    buf = b"0123456789abcdef"
    base = STRINGBUFBIT if copy else 0

    def tape_of(off, n):
        return np.array([word("r", 4), word('"', base | off), n, word("r", 0)], dtype=np.uint64)

    strs, msg = (buf, b"") if copy else (b"", buf)
    for off, n, ok in ((0, 16, True), (10, 6, True), (16, 0, True), (0, 17, False), (10, 7, False), (17, 0, False),
                       (16, 1, False), (1 << 40, 0, False), (0, 1 << 63, False)):
        t = tape_of(off, n)
        want = b'"' + mo.escape(buf[off:off + n]) + b'"' if ok else None
        if ok:
            assert mo.marshal(t, strs, msg) == want
        else:
            with pytest.raises(mo.MalformedTape):
                mo.marshal(t, strs, msg)
        assert _marshal(ctx, t, strs, msg) == ((OK, want) if ok else (ERR_ARGUMENT, None)), (off, n)


# ---- d. geometry ----------------------------------------------------------------------------------------------------
def _probe_key(b):
    b.open("{")
    b.string(b"kk")
    b.number("d", fv.double_bits([-0.5])[0])
    b.close()


def _probe_long_key(b):
    b.open("{")
    b.string(b"key\n" + b"x" * SHORT, copy=False)
    b.string(b"\x01\"" * SHORT)
    b.close()


def _probe_number(b):
    b.number("d", fv.double_bits([1e-7])[0])


def _probe_open(b):
    b.open("[")
    b.atoms("tf")
    b.close()


def _probe_empty(b):
    b.open("{")
    b.close()


# name -> (emit, offset of the word placed at E + s); each probe is followed by a sibling
PROBES = {
    "key head": (_probe_key, 1),
    "long key and value heads": (_probe_long_key, 1),
    "number head": (_probe_number, 0),
    "open": (_probe_open, 0),
    "close with a sibling": (_probe_open, 3),
    "empty container": (_probe_empty, 0),
}


def _text_of(emit):
    b = TapeBuilder()
    b.open("r")
    emit(b)
    b.close()
    return mo.marshal(*b.build())


def _array_with_probes(emit, offset, s):
    """r [ null ... probe at each E + s ... ] r, and its text"""
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    text = _text_of(emit)
    parts = []
    for E in EDGES:
        k = b.pad_to(E + s - offset)
        parts.append(b"null," * k + text + b",")
        emit(b)
    b.atoms("n")
    b.close(2)
    return b, b"[" + b"".join(parts) + b"null]"


@gpu
@pytest.mark.parametrize("probe", list(PROBES))
def test_probe_at_tile_and_group_edges(ctx, probe):
    emit, offset = PROBES[probe]
    for s in SHIFTS:
        b, want = _array_with_probes(emit, offset, s)
        tape, strs, msg = b.build()
        assert _marshal(ctx, tape, strs, msg) == (OK, want), (probe, s)


@gpu
def test_object_members_across_edges(ctx):
    """one object over all edges: a member's key head at E + s, so the key parity is carried across tiles and groups"""
    for s in SHIFTS:
        b = TapeBuilder()
        b.open("r")
        b.open("{")
        parts = []
        for E in EDGES:
            n3, n4 = b.pad_members_to(E + s)
            parts.append(b'"k":null,' * n3 + b'"k":0,' * n4 + b'"kk":-7,')
            b.string(b"kk")
            b.number("l", -7)
        b.close(2)
        tape, strs, msg = b.build()
        assert _marshal(ctx, tape, strs, msg) == (OK, b"{" + b"".join(parts)[:-1] + b"}"), s


@gpu
def test_root_close_at_edges(ctx):
    """NDJSON-shaped: many roots, one of them closing at E + s"""
    for s in SHIFTS:
        b = TapeBuilder()
        lines = []
        for E in EDGES + [2 * G + 50]:
            b.open("r")
            b.open("[")
            k = b.pad_to(E + s - 1)
            b.close(2)
            lines.append(b"[" + b",".join([b"null"] * k) + b"]")
            b.open("r")  # a small root behind it
            b.open("{")
            b.string(b"a")
            b.atom("t")
            b.close(2)
            lines.append(b'{"a":true}')
        tape, strs, msg = b.build()
        assert int(tape[EDGES[0] + s]) >> 56 == ord("r")
        assert _marshal(ctx, tape, strs, msg) == (OK, b"\n".join(lines)), s


@gpu
@pytest.mark.parametrize("kind", ["[", "{"])
def test_nesting_deeper_than_a_group(ctx, kind):
    D = G + 3
    b = TapeBuilder()
    b.open("r")
    b.nest(kind, D)
    b.close(D + 1)
    tape, strs, msg = b.build()
    want = b"[" * D + b"]" * D if kind == "[" else b'{"a":' * (D - 1) + b"{" + b"}" * D
    assert _marshal(ctx, tape, strs, msg) == (OK, want)


@gpu
def test_array_wider_than_a_group(ctx):
    n = G + 5
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    b.atoms("tfn" * (n // 3) + "t" * (n % 3))
    b.close(2)
    tape, _, _ = b.build()
    want = b"[" + b"true,false,null," * (n // 3) + b"true," * (n % 3)
    assert _marshal(ctx, tape) == (OK, want[:-1] + b"]")


@gpu
@pytest.mark.parametrize("n", [2, 3, 4, T - 1, T, T + 1, G - 1, G, G + 1])
def test_tape_lengths(ctx, n):
    b = TapeBuilder()
    b.open("r")
    if n == 3:
        b.atom("f")
    elif n > 3:
        b.open("[")
        b.atoms(("n", n - 4))
        b.close()
    b.close()
    tape, _, _ = b.build()
    assert len(tape) == n
    want = b"" if n == 2 else b"false" if n == 3 else b"[" + b",".join([b"null"] * (n - 4)) + b"]"
    assert _marshal(ctx, tape) == (OK, want)


@gpu
def test_one_word_tapes(ctx):
    """a root takes two words, so no one-word tape is valid"""
    for w in (word("r", 1), word("r", 0), word("n"), word("["), word("]"), word('"')):
        t = np.array([w], dtype=np.uint64)
        with pytest.raises(mo.MalformedTape):
            mo.marshal(t)
        assert _marshal(ctx, t)[0] == ERR_ARGUMENT, hex(w)


# ---- e. malformed tapes away from tile 0 ----------------------------------------------------------------------------
_DOC = b'{"a":[1,2.5,"x"],"b":{}}'
# 0 r 1 { 2 " 3 . 4 [ 5 l 6 . 7 d 8 . 9 " 10 . 11 ] 12 " 13 . 14 { 15 } 16 } 17 r
PLACES = {"tile 2 of group 1": G + 2 * T + 100, "across the group edge": G - 9}


def _doc_tape():
    b = TapeBuilder()
    b.open("r")
    b.open("{")
    b.string(b"a")
    b.open("[")
    b.number("l", 1)
    b.number("d", fv.double_bits([2.5])[0])
    b.string(b"x")
    b.close()
    b.string(b"b")
    b.open("{")
    b.close(3)
    return b.build()


def _around(base, doc):
    """a root of nulls, `doc` (a tape of roots that starts at 0) at word `base`, the root [null]: (tape, text in front)"""
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    k = b.pad_to(base - 2)
    b.close(2)
    t = np.concatenate([b.build()[0], doc + np.where(_links(doc), np.uint64(base), np.uint64(0))])
    m = len(t)
    tail = np.array([word("r", m + 5), word("[", m + 4), word("n"), word("]", m + 1), word("r", m)], dtype=np.uint64)
    return np.concatenate([t, tail]), b"[" + b",".join([b"null"] * k) + b"]"


def _links(t):
    return np.isin(t >> np.uint64(56), np.frombuffer(b"{}[]r", dtype=np.uint8).astype(np.uint64))


def _malformed_cases(place):
    """(name, tape) for each malformed tape, with the Strings.B and message of the document"""
    doc, strs, _ = _doc_tape()
    base = PLACES[place]
    tape, _ = _around(base, doc)
    n = len(tape)
    cases = {
        "unknown tag": {5: word("x")},
        "nop tag": {14: word("N", 2), 15: word("N", 1)},
        "open link out of range": {4: word("[", n + 1000)},
        "open link not at its close": {4: word("[", base + 10)},
        "close pointing elsewhere": {11: word("]", base + 2)},
        "root link broken": {0: word("r", base + 12)},
        "root close pointing elsewhere": {17: word("r", base + 1)},
        "string outside Strings.B": {9: int(doc[9]) + 100},
        "string length outside Strings.B": {10: 1 << 40},
        "string outside the message": {9: word('"', 1000)},
        "key not a string": {2: word("t"), 3: word("t")},
        "float NaN": {8: 0x7FF8000000000000},
        "float Inf": {8: 0x7FF0000000000000},
    }
    for name, change in cases.items():
        bad = tape.copy()
        for k, v in change.items():
            bad[base + k] = v
        yield name, bad
    yield "cut at the end", tape[:-1]
    yield "cut at the start", tape[1:]
    yield "cut inside the document", tape[:base + 9]
    yield "a word behind the last root", np.concatenate([tape, tape[:1]])
    dangling = np.array([word("r", 6), word("{", 5), word('"', STRINGBUFBIT), 1, word("}", 1), word("r", 0)], dtype=np.uint64)
    yield "an object closed behind a key", _around(base, dangling)[0]


def _odd_object_across_groups():
    """r { "k":null ... "k" } r with the last key in group 0 and the close in group 1"""
    b = TapeBuilder(raw=True)
    b.open("r")
    b.open("{")
    b.pad_members_to(G - 2)
    b.string(b"k")
    b.close(2)
    tape, strs, msg = b.build()
    assert int(tape[G - 2]) >> 56 == ord('"') and int(tape[G]) >> 56 == ord("}")
    return tape, strs


def _string_head_last():
    """r [ null ... " as a 2T-word tape: the string head is its last word, the links point where the closes would be"""
    tape = np.full(2 * T, word("n"), dtype=np.uint64)
    tape[0] = word("r", 2 * T + 2)
    tape[1] = word("[", 2 * T + 1)
    tape[-1] = word('"', STRINGBUFBIT)
    return tape


def test_oracle_rejects_the_malformed_tapes():
    """the oracle's walk raises on every tape the device must reject (no GPU needed)"""
    _, strs, _ = _doc_tape()
    for place in PLACES:
        for name, bad in _malformed_cases(place):
            with pytest.raises(mo.MalformedTape):
                mo.marshal(bad, strs, _DOC)
    t, s = _odd_object_across_groups()
    with pytest.raises(mo.MalformedTape):
        mo.marshal(t, s)
    with pytest.raises(mo.MalformedTape):
        mo.marshal(_string_head_last(), b"x")


def _assert_rejected(ctx, tape, strs, msg, what):
    d_tape, d_strs, d_msg = _upload(tape, strs, msg)
    buf = _canary(len(tape) * 6 + 64)
    rc, n, _ = ctx.marshal_device(d_tape, d_strs, d_msg, out=buf)
    assert rc == ERR_ARGUMENT, what
    assert bool((buf == 0xA5).all()), what


@gpu
@pytest.mark.parametrize("place", list(PLACES))
def test_malformed_tapes_away_from_tile_0(ctx, place):
    doc, strs, _ = _doc_tape()
    tape, head = _around(PLACES[place], doc)
    want = head + b"\n" + _DOC + b"\n[null]"
    assert _marshal(ctx, tape, strs, _DOC) == (OK, want)  # the valid tape the cases start from
    for name, bad in _malformed_cases(place):
        _assert_rejected(ctx, bad, strs, _DOC, (place, name))


@gpu
def test_malformed_across_group_edges(ctx):
    t, s = _odd_object_across_groups()
    _assert_rejected(ctx, t, s, b"", "odd object")
    _assert_rejected(ctx, _string_head_last(), b"x", b"", "string head last")


# ---- f. capacity and limits -----------------------------------------------------------------------------------------
@gpu
def test_capacity_on_a_multi_group_tape(ctx):
    doc, strs, _ = _doc_tape()
    tape, head = _around(G + 2 * T + 100, doc)
    want = head + b"\n" + _DOC + b"\n[null]"
    d_tape, d_strs, d_msg = _upload(tape, strs, _DOC)
    buf = _canary(len(want) + 64)
    rc, n, _ = ctx.marshal_device(d_tape, d_strs, d_msg, out=buf[:len(want) - 1])
    assert (rc, n) == (ERR_CAPACITY, len(want))
    assert bool((buf == 0xA5).all())
    rc, n, out = ctx.marshal_device(d_tape, d_strs, d_msg, out=buf[:len(want)])
    assert (rc, n) == (OK, len(want)) and out.cpu().numpy().tobytes() == want
    assert bool((buf[len(want):] == 0xA5).all())


@gpu
def test_tape_too_large(ctx):
    """the length is checked before any word is read: a one-word tensor stands for 2^31 words"""
    import torch
    one = torch.zeros(1, dtype=torch.int64, device="cuda")
    n = C.c_size_t(7)
    rc = ctx.L.sj_marshal_device(ctx.h, None, 0, one.data_ptr(), 1 << 31, None, 0, None, 0, C.byref(n))
    assert (rc, n.value) == (ERR_TOO_LARGE, 0)
