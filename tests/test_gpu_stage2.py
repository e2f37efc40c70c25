"""GPU parity tests for the whole parse (K1 + K2a..K2f) through the C ABI: tape and string
buffer bit-exact against the CPU oracle, plus the reference's goldens (G11..G19) and its fuzz
seed corpora (G20)."""
import struct

import numpy as np
import pytest

from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, golden, load_fixture, unhex

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _same_parse(ctx, oracle, msg, ndjson=False, copy=True):
    rc_g, tape_g, str_g, win_g = ctx.parse(msg, ndjson=ndjson, copy_strings=copy)
    rc_o, tape_o, str_o, win_o = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
    assert rc_g == rc_o, (rc_g, rc_o, bytes(msg[:80]))
    assert win_g == win_o
    if rc_o == 0:
        assert len(tape_g) == len(tape_o)
        if not np.array_equal(tape_g, tape_o):
            bad = int(np.nonzero(tape_g != tape_o)[0][0])
            raise AssertionError("tape differs at %d: gpu %016x oracle %016x" % (bad, int(tape_g[bad]), int(tape_o[bad])))
        assert str_g == str_o
    return rc_g


def test_g11_stage2_tapes(ctx):
    for i, tc in enumerate(golden("G11_tapes")):
        rc, tape, strs, _ = ctx.parse(unhex(tc["input"]), copy_strings=False)
        assert rc == 0 and [int(x) for x in tape] == tc["tape"], i


def test_g12_demo_ndjson_tape(ctx):
    g = golden("G12_ndjson_tape")
    rc, tape, _, _ = ctx.parse(unhex(g["input"]), ndjson=True, copy_strings=False)
    assert rc == 0 and [int(x) for x in tape] == list(g["tape"])


def test_g13_atoms(ctx, oracle):
    g = golden("G13_atoms")
    for kind in ("true", "false", "null"):
        for tc in g[kind]:
            txt = unhex(tc["input"])
            doc = b"[" + txt.rstrip(b" ") + b"]" if tc["expected"] else b"[" + txt.rstrip(b" ") + b" ]"
            _same_parse(ctx, oracle, doc)


def test_g14_strings(ctx):
    tcs = golden("G14_strings")
    items = [b'"' + unhex(tc["str"]) + b'"' for tc in tcs]
    res = ctx.parse_strings(items)
    for tc, (ok, sl, dl, out) in zip(tcs, res):
        assert ok == tc["success"], tc["name"]
        if ok:
            assert out == unhex(tc["want"]) and dl == len(out), tc["name"]


def test_strings_random_vs_oracle(ctx, oracle):
    rng = np.random.default_rng(99)
    alphabet = [b"a", b"\\", b'"', b"u", b"d", b"8", b"0", b"F", b"c", b"\\u", b"\\ud83d", b"\\ude00", b"n", b"/", b"\x00",
                b"-", b"\xc3\xa9", b"\\\\", b'\\"', b"xyz" * 5, b"t" * 31, b"q" * 33]
    items, maxs = [], []
    for _ in range(6000):
        body = b"".join(alphabet[j] for j in rng.integers(0, len(alphabet), rng.integers(0, 14)))
        tail = b'"' if rng.integers(0, 8) else b""
        it = b'"' + body + tail + b"," * int(rng.integers(0, 3))
        items.append(it)
        maxs.append(int(rng.integers(0, len(it) + 40)))
    res = ctx.parse_strings(items, maxs)
    for it, mx, (ok, sl, dl, out) in zip(items, maxs, res):
        ok_o, sl_o, dl_o = oracle.parse_string_validate_only(it, mx)
        assert ok == ok_o, (it, mx)
        if ok:
            assert (sl, dl) == (sl_o, dl_o), it
            assert out == oracle.parse_string(it)[1], it


def test_strings_long_random_vs_oracle(ctx, oracle):
    """multi-window strings: the warp-cooperative measure / unescape (32 source bytes per step) and the
    thread-serial routines both run in the hook and must agree with each other and with the oracle"""
    rng = np.random.default_rng(424242)
    alphabet = [b"a", b"\\", b'"', b"u", b"8", b"F", b"\\u", b"\\ud83d", b"\\ude00", b"\\uD800", b"n", b"/", b"\x00", b" ",
                b"\xc3\xa9", b"\\\\", b'\\"', b"\\n", b"\\/", b"\\u00e9", b"\\u20AC", b"xyz" * 5, b"t" * 31, b"q" * 33, b"w" * 64,
                b"0123456789abcdef" * 9]
    items, maxs = [], []
    for _ in range(4000):
        body = b"".join(alphabet[j] for j in rng.integers(0, len(alphabet), rng.integers(0, 48)))
        tail = b'"' if rng.integers(0, 10) else b""
        it = b'"' + body + tail + b" " * int(rng.integers(0, 3)) + b","
        items.append(it)
        maxs.append(max(0, int(rng.integers(len(it) - 8, len(it) + 40))) if rng.integers(0, 4) else int(rng.integers(0, len(it) + 1)))
    res = ctx.parse_strings(items, maxs)
    for it, mx, (ok, sl, dl, out) in zip(items, maxs, res):
        ok_o, sl_o, dl_o = oracle.parse_string_validate_only(it, mx)
        assert ok == ok_o, (it, mx)
        if ok:
            assert (sl, dl) == (sl_o, dl_o), it
            assert out == oracle.parse_string(it)[1], it


def _tagname(tag):
    return chr(tag >> 56) if tag else ""


def test_g15_numbers(ctx):
    g = golden("G15_numbers")
    res = ctx.parse_numbers([tc["input"].encode() + b":" for tc in g["parse_number"]])
    for tc, (tag, val) in zip(g["parse_number"], res):
        assert _tagname(tag) == tc["tag"] and tag & ((1 << 56) - 1) == tc["flags"], tc
        if tc["tag"] == "d":
            assert struct.pack("<Q", val) == struct.pack("<d", float(tc["d"])), tc
        elif tc["tag"] == "l":
            assert val == tc["i"] & M64, tc
        else:
            assert val == tc["u"], tc
    res = ctx.parse_numbers([tc["input"].encode() + b":" for tc in g["parse_int64"]])
    for tc, (tag, val) in zip(g["parse_int64"], res):
        assert _tagname(tag) == tc["tag"], tc
        if tc["tag"] == "l":
            assert val == tc["out"] & M64, tc
    res = ctx.parse_numbers([tc["input"].encode() + b":" for tc in g["atof"]])
    for tc, (tag, val) in zip(g["atof"], res):
        t = _tagname(tag)
        if t == "":
            assert tc["err"], tc
        elif t == "d":
            want = float(tc["out"].replace("+Inf", "inf").replace("-Inf", "-inf"))
            assert struct.pack("<Q", val) == struct.pack("<d", want), tc
        else:
            assert str(val if t == "u" else struct.unpack("<q", struct.pack("<Q", val))[0]) == tc["out"], tc
    for (tag, _), s in zip(ctx.parse_numbers([s.encode() for s in g["valid"]]), g["valid"]):
        assert tag != 0, s
    for (tag, _), s in zip(ctx.parse_numbers([s.encode() if s else b" " for s in g["invalid"]]), g["invalid"]):
        assert tag == 0, s


def test_numbers_random_vs_oracle(ctx, oracle):
    """bit-exact float64 (not just 1 ULP): Clinger / Eisel-Lemire / exact decimal paths"""
    rng = np.random.default_rng(2024)
    items = []
    for _ in range(40000):
        kind = rng.integers(0, 8)
        nd = int(rng.integers(1, 25 if kind < 6 else 60))
        digits = "".join(str(d) for d in rng.integers(0, 10, nd))
        s = digits.lstrip("0") or "0"
        if kind in (1, 3, 5, 7):
            k = int(rng.integers(0, len(s) + 1))
            s = (s[:k] or "0") + "." + (s[k:] or "0")
        if kind in (2, 3, 6, 7):
            s += "eE"[rng.integers(0, 2)] + ["", "+", "-"][rng.integers(0, 3)] + str(int(rng.integers(0, 340)))
        if rng.integers(0, 2):
            s = "-" + s
        items.append(s.encode() + b",")
    # doubles printed with 17 significant digits, their neighbours' midpoints, subnormals, extremes
    raw = rng.integers(0, 1 << 63, 20000, dtype=np.int64).view(np.float64)
    for x in raw[np.isfinite(raw)]:
        items.append(("%.17g" % x).replace("inf", "1e999").encode() + b"]")
        items.append(("%.25e" % x).encode() + b"]")
    for s in ("4.9e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623157e308",
              "1.7976931348623158e308", "1.797693134862315807e308", "8.98846567431158e307", "2.2250738585072011e-308",
              "0.000000000000000000000000000000000000000000000000000001e-290", "9007199254740993", "9007199254740992.5",
              "9007199254740993.0000000000000000000000000001", "1e23", "8.5e-323", "123456789012345678901234567890e-30"):
        items.append(s.encode() + b" ")
    res = ctx.parse_numbers(items)
    for it, (tag, val) in zip(items, res):
        otag, oval = oracle.parse_number(it)
        assert (tag, val) == (otag, oval), (it, hex(tag), hex(val), hex(otag), hex(oval))


def test_g16_g17_documents(ctx, oracle):
    g = golden("G16_G17_documents")
    for key, nd in (("fail_cases", False), ("pass_cases", False), ("parse_nd", True)):
        for tc in g[key]:
            for copy in (True, False):
                rc = _same_parse(ctx, oracle, unhex(tc["js"]), ndjson=nd, copy=copy)
                assert (rc != 0) == tc["want_err"], (key, tc["name"], rc)
    for hx in g["ndjson_emptylines"]:
        assert _same_parse(ctx, oracle, unhex(hx), ndjson=True) == 0


@pytest.mark.parametrize("name", TAPE_FILES + SMALL_FILES)
def test_g19_fixture_tapes_vs_oracle(ctx, oracle_native, name):
    """BASELINE configs 2 and 3 live here: canada (number-heavy), twitterescaped (bit-exact tape check)"""
    msg = load_fixture(name)
    for copy in (True, False):
        assert _same_parse(ctx, oracle_native, msg, copy=copy) == 0


def test_g18_parking_citations_ndjson(ctx, oracle_native):
    msg = load_fixture("parking-citations")
    for copy in (True, False):
        assert _same_parse(ctx, oracle_native, msg, ndjson=True, copy=copy) == 0
    rc, tape, strs, (off, ln) = ctx.parse(msg, ndjson=True)
    roots = int((tape >> np.uint64(56) == ord("r")).sum()) // 2
    assert roots == golden("G18_G19_fixtures")["parking_citations"]["roots"]


def test_twitter_vs_twitterescaped_identical(ctx):
    a = ctx.parse(load_fixture("twitter"))
    b = ctx.parse(load_fixture("twitterescaped"))
    assert a[0] == b[0] == 0 and np.array_equal(a[1], b[1]) and a[2] == b[2]


def test_structure_edge_cases(ctx, oracle):
    docs = [b"{}", b"[]", b"[[]]", b"[{}]", b'{"a":{}}', b"[" * 300 + b"]" * 300, b"[" * 300 + b"]" * 299, b"[" * 2 + b"]" * 3,
            b'{"a":[1,2,{"b":[]}],"c":null}', b"[1,2,3", b"[1,,2]", b'{"a" 1}', b'{"a":1,}', b"[1 2]", b'["a":1]', b'{"a":1}}',
            b"[}", b"{]", b"[true,false,null,tru,falsee]", b"[nul]", b'{"a":truex}', b'{1:2}', b"[-]", b"[1e]", b"[01]", b"[-0]",
            b"[1.]", b'["\\x"]', b'["\\ud800"]', b'["\\ud800\\u0041"]', b'["a\\"b"]', b" \n\t [1] \r\n", b"\xc2\xa0[1]\xe2\x80\x83",
            b"", b"   ", b"[\x80]", b'{"k":"v"} x', b'"str"', b"123", b"[1]x", b'[{"a":[{"b":[{"c":[1,2,3]}]}]}]',
            b'[' + b",".join(b"[%d,%d]" % (i, i) for i in range(5000)) + b"]",      # canada-like: long runs of siblings
            b'{"a":' * 70 + b"1" + b"}" * 70, b'[' + b'"s",' * 40000 + b'"e"]',      # long flat array: multi-level ANSV
            ]
    for d in docs:
        for copy in (True, False):
            _same_parse(ctx, oracle, d, copy=copy)
    nd = [b'{"a":1}\n{"b":2}', b'{"a":1}\n\n\n{"b":2}\n[3]', b'{"a":1}{"b":2}', b'{"a":1}\n', b'{"a":\n1}', b'{"a":1}\n2',
          b'[1]\n[2]\n[3]\n[4]', b'\n\n[1]\n\n', b'{"a":"x\\ny"}\n{"b":2}', b"[1]\n]", b"[1]\n[", b'{"a":1} \n {"b":2}']
    for d in nd:
        for copy in (True, False):
            _same_parse(ctx, oracle, d, ndjson=True, copy=copy)
        _same_parse(ctx, oracle, d, ndjson=False)


def test_long_and_escaped_strings_in_documents(ctx, oracle):
    """strings of 0..400 bytes with and without escapes, mixed inside the same warps: the short ones take the
    thread-serial measure / unescape, the long ones (>= S2_COOP_MIN bytes) the warp-cooperative one; invalid
    escapes and unterminated \\u sequences must fail exactly where the oracle fails"""
    rng = np.random.default_rng(20240923)
    pieces = [b"a", b"bc", b"\\n", b"\\/", b'\\"', b"\\\\", b"\\u00e9", b"\\ud83d\\ude00", b"\xe2\x82\xac", b" ", b"x" * 17, b"y" * 40,
              b"http:\\/\\/t.co\\/", b"0123456789" * 7]

    def rand_string(maxtok):
        return b'"' + b"".join(pieces[j] for j in rng.integers(0, len(pieces), rng.integers(0, maxtok))) + b'"'

    for trial in range(12):
        maxtok = (3, 12, 40)[trial % 3]
        vals = [rand_string(maxtok) for _ in range(700)]
        doc = b"[" + b",".join(vals) + b"]"
        obj = b"{" + b",".join(rand_string(maxtok) + b" : " + rand_string(maxtok) for _ in range(300)) + b"}"
        for d in (doc, obj, doc[:-1] + b"," + obj + b"]"):
            for copy in (True, False):
                assert _same_parse(ctx, oracle, d, copy=copy) == 0
    bad = [b'["' + b"x" * 100 + b'\\q' + b"y" * 100 + b'"]', b'["' + b"x" * 100 + b'\\u12"]', b'["' + b"x" * 90 + b'\\ud800\\n' + b"z" * 70 + b'"]',
           b'["' + b"x" * 70 + b'\\ud800' + b"z" * 70 + b'"]', b'["' + b"x" * 64 + b'\\uZZZZ' + b"z" * 64 + b'"]',
           b'["' + b"k" * 200 + b'\\u00e9' * 30 + b'", "' + b"k" * 31 + b'\\', b'["' + b"s" * 300 + b'\\ud83d\\ude00' * 20 + b'"]']
    for d in bad:
        for copy in (True, False):
            _same_parse(ctx, oracle, d, copy=copy)


def test_number_heavy_documents_dense_kernel(ctx, oracle):
    """documents where at least one structural in 16 is a number take the dense number kernels (K2g / K2h);
    sparse ones keep the inline parse in K2c -- both must give the oracle's tape, and a bad number anywhere must
    fail the document"""
    rng = np.random.default_rng(5150)

    def rand_number():
        k = int(rng.integers(0, 8))
        if k == 0:
            return str(int(rng.integers(-2**63, 2**63 - 1, dtype=np.int64))).encode()
        if k == 1:
            return str(int(rng.integers(0, 2**64 - 1, dtype=np.uint64))).encode()
        if k == 2:
            return repr(float(rng.standard_normal() * 10.0 ** int(rng.integers(-300, 300)))).encode()
        if k == 3:
            return b"%d.%de%d" % (rng.integers(0, 10**9), rng.integers(0, 10**9), rng.integers(-330, 290))
        if k == 4:
            return b"-%d.%018d" % (rng.integers(0, 200), rng.integers(0, 10**18))
        if k == 5:
            return b"%d" % rng.integers(-1000, 1000)
        if k == 6:
            return b"0.%s" % (b"".join(b"%d" % d for d in rng.integers(0, 10, rng.integers(1, 40))))
        return b"%dE+%d" % (rng.integers(1, 10**6), rng.integers(0, 30))

    nums = [rand_number() for _ in range(20000)]
    dense = b"[" + b",".join(nums) + b"]"
    pairs = b"[" + b",".join(b"[%s,%s]" % (nums[i], nums[i + 1]) for i in range(0, 6000, 2)) + b"]"
    sparse = b"[" + b",".join(b'{"k%d":"v","n":%s,"t":true,"s":"%s"}' % (i, nums[i], b"x" * (i % 50)) for i in range(1500)) + b"]"
    nd = b"\n".join(b'{"a":%s,"b":[%s,%s]}' % (nums[i], nums[i + 1], nums[i + 2]) for i in range(0, 9000, 3))
    for d, isnd in ((dense, False), (pairs, False), (sparse, False), (nd, True)):
        for copy in (True, False):
            assert _same_parse(ctx, oracle, d, ndjson=isnd, copy=copy) == 0
    for badnum in (b"1e", b"-", b"01", b"1.", b"--1", b"1e400", b"0x10", b"1_000", b"+1", b".5"):
        for where in (0, 7777, 19999):
            bad = list(nums)
            bad[where] = badnum
            _same_parse(ctx, oracle, b"[" + b",".join(bad) + b"]")


def test_large_documents(ctx, oracle_native):
    tw = load_fixture("twitter")
    big = b"[" + b",".join([tw] * 24) + b"]"           # ~15 MB single document, 60 k brackets per copy
    assert _same_parse(ctx, oracle_native, np.frombuffer(big, dtype=np.uint8)) == 0
    pk = load_fixture("parking-citations").strip()
    nd = b"\n".join([pk] * 30)                          # 30 000 NDJSON records
    assert _same_parse(ctx, oracle_native, np.frombuffer(nd, dtype=np.uint8), ndjson=True) == 0
    ca = load_fixture("canada")
    assert _same_parse(ctx, oracle_native, b"[" + b",".join([ca] * 4) + b"]") == 0


@pytest.mark.parametrize("which,expect", [("corpus", 8000), ("go-corpus", 300)])
def test_g20_fuzz_corpus_differential(ctx, oracle_native, which, expect):
    """fuzz_test.go:40-94 FuzzParse seeds -- ALL of them (8 680 + 356 inputs, no size cap): same accept / reject and the
    same tape and string buffer as the oracle, as a single document and as NDJSON, and (every 16th seed) with
    copy_strings off"""
    n = 0
    for name, data in fuzz_corpus(which):
        for nd in (False, True):
            _same_parse(ctx, oracle_native, data, ndjson=nd)
        if n % 16 == 0:
            _same_parse(ctx, oracle_native, data, ndjson=False, copy=False)
        n += 1
    assert n > expect, n


def test_concurrent_contexts(oracle_native):
    """parse_json_amd64.go is re-entrant on distinct ParsedJson values (ParseNDStream runs several
    parses at once, simdjson_amd64.go:132): distinct contexts must be usable from distinct threads"""
    import threading
    import simdjson_b200 as sj
    names = ["twitter", "canada", "citm_catalog", "random"]
    want = {n: oracle_native.parse(load_fixture(n)) for n in names}
    errs = []

    def work(name):
        try:
            c = sj.Context(0)
            for _ in range(4):
                rc, tape, strs, _ = c.parse(load_fixture(name))
                assert rc == 0 and np.array_equal(tape, want[name][1]) and strs == want[name][2]
            c.close()
        except Exception as e:  # noqa: BLE001
            errs.append((name, repr(e)))

    ts = [threading.Thread(target=work, args=(n,)) for n in names]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs


def test_too_large_and_empty(ctx):
    import ctypes as C
    tl, sl, mo, ml = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    rc = ctx.L.sj_parse(ctx.h, None, 0, 0, None, 0, C.byref(tl), None, 0, C.byref(sl), C.byref(mo), C.byref(ml))
    assert rc == 1  # empty input: stage-1 failure, like the reference
    assert ctx.L.sj_stage1_launch(ctx.h, 16, (1 << 31) + 5, 0, 0, 16, 0) == 5  # SJ_ERR_TOO_LARGE before touching memory


def test_parse_nd_stream(oracle_native):
    """ParseNDStream (simdjson_amd64.go:116): newline-aligned chunks, several in flight, results in
    input order, each an independent ParsedJson; ndjson_test.go:250 countWhere(Make == HOND) = 116 per copy"""
    import io
    from simdjson_b200.stream import ParseNDStream
    pk = load_fixture("parking-citations").strip()
    copies = 7
    stream = b"\n".join([pk] * copies) + b"\n"
    hond = roots = 0
    pos = 0
    for pj in ParseNDStream(io.BytesIO(stream), chunk_bytes=300_000, inflight=3):
        # the chunk this result came from is the next newline-aligned window of the stream
        chunk_len = len(pj.Message)
        start = stream.index(pj.Message[:64], pos)
        rc, tape, strs, _ = oracle_native.parse(stream[start:start + chunk_len], ndjson=True)
        assert rc == 0 and np.array_equal(pj.Tape, tape) and pj.Strings == strs
        pos = start + chunk_len
        it = pj.Iter()
        hond += it.count_where("Make", "HOND")
        roots += sum(1 for _ in it.roots())
    assert roots == 1000 * copies and hond == 116 * copies
    with pytest.raises(Exception):
        list(ParseNDStream(io.BytesIO(b'{"a":1}\n{"b":\n'), chunk_bytes=1 << 20))


@pytest.mark.parametrize("chunk,inflight", [(300_000, 3), (50_000, 1), (1_500_000, 4)])
def test_parse_nd_stream_native(oracle_native, chunk, inflight):
    """the same ParseNDStream contract through the library's own pipeline (sj_stream_*): chunks cut at record
    boundaries, several in flight, ordered delivery, every chunk bit-equal to the oracle's parse of the same bytes,
    the whole stream covered exactly once"""
    import io
    from simdjson_b200.stream import ParseNDStreamNative
    pk = load_fixture("parking-citations").strip()
    copies = 7
    stream = b"\n".join([pk] * copies) + b"\n\n  \n"
    hond = roots = 0
    pos = 0
    nchunks = 0
    for pj in ParseNDStreamNative(io.BytesIO(stream), chunk_bytes=chunk, inflight=inflight, read_bytes=777_777):
        start = stream.index(pj.Message[:64], pos)
        assert stream[start:start + len(pj.Message)] == pj.Message       # consecutive windows of the input
        assert stream[pos:start].strip() == b""                           # nothing but blanks skipped in between
        rc, tape, strs, _ = oracle_native.parse(pj.Message, ndjson=True)
        assert rc == 0 and np.array_equal(pj.Tape, tape) and pj.Strings == strs
        pos = start + len(pj.Message)
        it = pj.Iter()
        hond += it.count_where("Make", "HOND")
        roots += sum(1 for _ in it.roots())
        nchunks += 1
    assert stream[pos:].strip() == b""
    assert roots == 1000 * copies and hond == 116 * copies
    assert nchunks >= len(stream) // (chunk + 400) and nchunks <= len(stream) // chunk + 2


def test_parse_nd_stream_native_errors_and_big_records():
    import io
    from simdjson_b200.stream import ParseNDStreamNative
    from simdjson_b200 import ParseError
    with pytest.raises(ParseError):
        list(ParseNDStreamNative(io.BytesIO(b'{"a":1}\n{"b":\n'), chunk_bytes=1 << 20))
    with pytest.raises(ParseError):   # the second chunk fails: the first one is still delivered, then the error ends the stream
        got = []
        for pj in ParseNDStreamNative(io.BytesIO(b'{"a":1}\n' * 100 + b'{"b" 2}\n' * 100), chunk_bytes=800, inflight=2):
            got.append(pj)
    assert len(got) >= 1
    assert list(ParseNDStreamNative(io.BytesIO(b""), chunk_bytes=1 << 20)) == []
    assert list(ParseNDStreamNative(io.BytesIO(b" \n\n "), chunk_bytes=1 << 20)) == []
    # one record much larger than the chunk size: the chunk grows until a record boundary shows up
    big = b'{"k":"' + b"x" * 100_000 + b'"}'
    out = list(ParseNDStreamNative(io.BytesIO(big + b"\n" + big + b"\n" + b'{"s":1}'), chunk_bytes=10_000, inflight=2, read_bytes=4096))
    assert sum(sum(1 for _ in pj.Iter().roots()) for pj in out) == 3
    # blank lines in front of a record larger than the chunk: the cut at the last newline would leave a whitespace-only
    # chunk (stage-1 failure); the reference skips blank lines (stage2_build_tape_amd64.go:200-205)
    out = list(ParseNDStreamNative(io.BytesIO(b"\n \n" + big + b"\n\n" + big + b"\n"), chunk_bytes=10_000, inflight=2, read_bytes=4096))
    assert sum(sum(1 for _ in pj.Iter().roots()) for pj in out) == 2


def test_streaming_and_per_structural_stage2_agree(ctx, oracle_native):
    """the two stage-2 implementations (streaming kernels, stage2_stream.cuh = the default with copy_strings;
    per-structural kernels, stage2.cuh) give the same tape and string buffer -- on inputs far larger than the oracle
    comfortably checks, in every BASELINE shape"""
    import simdjson_b200 as sj
    legacy = sj.Context(0)
    legacy.set_stage2_impl(1)
    try:
        docs = []
        for name, k in (("twitter", 40), ("twitterescaped", 40), ("canada", 10), ("gsoc-2018", 8), ("citm_catalog", 12), ("marine_ik", 6)):
            d = load_fixture(name).strip()
            docs.append((b"[" + b",".join([d] * k) + b"]", False))
        pk = load_fixture("parking-citations").strip()
        docs.append((b"\n".join([pk] * 60), True))
        for doc, nd in docs:
            a = ctx.parse(np.frombuffer(doc, dtype=np.uint8), ndjson=nd)
            b = legacy.parse(np.frombuffer(doc, dtype=np.uint8), ndjson=nd)
            assert a[0] == b[0] == 0
            assert np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]
        # and both agree with the oracle on a mid-sized one
        d = load_fixture("twitterescaped").strip()
        assert _same_parse(ctx, oracle_native, b"[" + b",".join([d] * 6) + b"]") == 0
        assert _same_parse(legacy, oracle_native, b"[" + b",".join([d] * 6) + b"]") == 0
    finally:
        legacy.close()


def test_streaming_stage2_edges(ctx, oracle_native):
    """the emulation suite's edge cases (tests/test_s2s_emulation.py) through the real kernels: escapes and strings
    straddling block / step / slab edges, invalid escapes, grammar soup, NDJSON corner cases"""
    import tests.test_s2s_emulation as emu
    import tests.emu_util as eu
    orig = eu.same_as_oracle
    calls = [0]

    def via_gpu(oracle, msg, ndjson=False):
        calls[0] += 1
        return _same_parse(ctx, oracle, msg, ndjson=ndjson, copy=True)

    emu.same_as_oracle = via_gpu
    try:
        emu.test_escapes_across_every_edge(oracle_native)
        emu.test_invalid_escapes_and_strings(oracle_native)
        emu.test_strings_across_edges(oracle_native)
        emu.test_structure_and_grammar(oracle_native)
        emu.test_ndjson(oracle_native)
        emu.test_golden_documents(oracle_native)
    finally:
        emu.same_as_oracle = orig
    assert calls[0] > 2500


@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("world", [2, 3])
def test_parse_nd_sharded_is_one_parsed_json(oracle_native, copy, world):
    """sj_parse_nd_sharded_count / _emit (SURVEY.md 8e): the shards' slices, laid end to end, are bit for bit the tape and
    string buffer the reference's ParseND returns for the whole stream (simdjson_amd64.go:82-93; root chaining
    stage2_build_tape_amd64.go:190-221) -- `world` contexts on this GPU stand in for the ranks, the exchange of the totals
    is done by hand (over NCCL it is parallel.ShardedParse.exchange)"""
    import torch
    import simdjson_b200 as sj
    from simdjson_b200.parallel import ShardedParse, split_at_newlines, trimmed_window
    pk = load_fixture("parking-citations").strip()
    stream = b"\n".join([pk] * 7) + b"\n\n" + b'{"esc":"a\\u00e9\\n","n":[1,2.5,-3],"t":true}\n' + pk[:30000].rsplit(b"\n", 1)[0]
    rc, tape_o, str_o, (off_o, len_o) = oracle_native.parse(stream, ndjson=True, copy_strings=copy)
    assert rc == 0
    dev = torch.device("cuda:0")
    ranks = []
    for a, b in split_at_newlines(stream, world):
        a, b = trimmed_window(stream, a, b)
        c = sj.Context(0)
        d_msg = torch.full((b - a + 256,), 0x20, dtype=torch.uint8, device=dev)
        d_msg[: b - a] = torch.frombuffer(bytearray(stream[a:b]), dtype=torch.uint8).to(dev)
        sp = ShardedParse(c)
        rc, tot = sp.count(d_msg.data_ptr(), b - a, copy)
        assert rc == 0
        ranks.append((c, sp, d_msg, a, tot))
    tapes, strs = [], []
    tb = sb = 0
    for c, sp, d_msg, a, tot in ranks:
        d_tape = torch.empty(tot[1] + 8, dtype=torch.int64, device=dev)
        d_str = torch.empty(tot[2] + 64, dtype=torch.uint8, device=dev)
        assert sp.emit(a - off_o, tb, sb, d_tape.data_ptr(), d_tape.numel(), d_str.data_ptr(), d_str.numel()) == 0
        tapes.append(d_tape[: tot[1]].cpu().numpy().view(np.uint64))
        strs.append(d_str[: tot[2]].cpu().numpy().tobytes())
        tb += tot[1]
        sb += tot[2]
    assert sum(t[4][3] for t in ranks) == stream.count(b"\n{") + 1
    got = np.concatenate(tapes)
    assert len(got) == len(tape_o)
    assert np.array_equal(got, tape_o), int(np.nonzero(got != tape_o)[0][0])
    assert b"".join(strs) == str_o
    for c, *_ in ranks:
        c.close()


def _run_ranks(world, fn):
    """fn(rank, barrier) on `world` host threads (ctypes calls release the GIL): the ranks of one process"""
    import threading
    bar = threading.Barrier(world)
    out, errs = [None] * world, []

    def body(r):
        try:
            out[r] = fn(r, bar)
        except BaseException as e:  # noqa: BLE001 -- reported below; a rank that dies must not leave the others at a barrier
            errs.append((r, e))
            bar.abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    return out


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("world", [2, 5])
def test_parse_nd_sharded_exchange_over_peer_memory(oracle_native, copy, world, impl):
    """the same claim with the exchange done by the library (exchange.cuh): the counting half ends with a kernel that pushes
    the shard's totals into every peer's buffer, waits for the peers' and leaves the bases in device memory; the emitting
    half reads them there.  `world` host threads with one context each stand in for the ranks (their buffers are plain
    device pointers to each other: sj_exchange_connect_ptrs); three parses in a row exercise the epochs' double buffering"""
    import ctypes as C
    import torch
    import simdjson_b200 as sj
    from simdjson_b200.parallel import ShardedParse, split_at_newlines, trimmed_window
    pk = load_fixture("parking-citations").strip()
    stream = b"\n".join([pk] * 5) + b"\n\n" + b'{"esc":"a\\u00e9\\n","n":[1,2.5,-3],"t":true}\n' + pk[:30000].rsplit(b"\n", 1)[0]
    rc, tape_o, str_o, (off_o, len_o) = oracle_native.parse(stream, ndjson=True, copy_strings=copy)
    assert rc == 0
    dev = torch.device("cuda:0")
    wins = [trimmed_window(stream, a, b) for a, b in split_at_newlines(stream, world)]
    ctxs = [sj.Context(0) for _ in range(world)]
    for r, c in enumerate(ctxs):
        c.set_stage2_impl(impl)
        assert c.L.sj_exchange_create(c.h, r, world, 1, None) == 0
    locs = (C.c_void_p * world)(*[c.L.sj_exchange_local(c.h) for c in ctxs])

    def rank(r, bar):
        c = ctxs[r]
        a, b = wins[r]
        assert c.L.sj_exchange_connect_ptrs(c.h, locs) == 0
        assert c.L.sj_exchange_set_gap(c.h, wins[r + 1][0] - b if r + 1 < world else 0) == 0
        d_msg = torch.full((b - a + 256,), 0x20, dtype=torch.uint8, device=dev)
        d_msg[: b - a] = torch.frombuffer(bytearray(stream[a:b]), dtype=torch.uint8).to(dev)
        torch.cuda.synchronize()
        sp = ShardedParse(c)
        res = None
        for it in range(3):
            bar.wait()
            rc, tot = sp.count(d_msg.data_ptr(), b - a, copy)
            assert rc == 0, rc
            rc, ex = sp.exchange_result()
            assert rc == 0 and ex[8] == 0 and ex[9] == it + 1, ex
            d_tape = torch.empty(tot[1] + 8, dtype=torch.int64, device=dev)
            d_str = torch.empty(tot[2] + 64, dtype=torch.uint8, device=dev)
            assert sp.emit(0, 0, 0, d_tape.data_ptr(), d_tape.numel(), d_str.data_ptr(), d_str.numel(), c.L.sj_exchange_bases(c.h)) == 0
            res = (d_tape[: tot[1]].cpu().numpy().view(np.uint64), d_str[: tot[2]].cpu().numpy().tobytes(), tot, ex)
        return res

    out = _run_ranks(world, rank)
    got = np.concatenate([o[0] for o in out])
    assert len(got) == len(tape_o)
    assert np.array_equal(got, tape_o), int(np.nonzero(got != tape_o)[0][0])
    assert b"".join(o[1] for o in out) == str_o
    for r, o in enumerate(out):
        ex = o[3]
        assert ex[0] == wins[r][0] - off_o and ex[1] == sum(q[2][1] for q in out[:r]) and ex[2] == sum(q[2][2] for q in out[:r])
        assert ex[4] == len_o and ex[5] == len(tape_o) and ex[6] == len(str_o) and ex[7] == sum(q[2][3] for q in out)
    for c in ctxs:
        c.close()


def test_sharded_exchange_failures_do_not_hang():
    """a rank whose shard fails (stage 1: unterminated string; stage 2 counting pass: invalid escape; empty shard) still
    publishes, so its peers return SJ_ERR_PEER instead of waiting; a rank that never calls costs the others the time limit
    and SJ_ERR_EXCHANGE (the ranks' epochs then differ: the exchange has to be set up again)"""
    import ctypes as C
    import time
    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    from simdjson_b200.parallel import ShardedParse
    dev = torch.device("cuda:0")
    world = 3
    good = b'{"a":1}\n{"b":[true,null]}'
    cases = [(b'{"a":"unterminated}', _lib.ERR_STAGE1), (b'{"a":"bad \\q escape"}', _lib.ERR_STAGE2), (b"", _lib.ERR_STAGE1), (None, None)]
    ctxs = [sj.Context(0) for _ in range(world)]
    for r, c in enumerate(ctxs):
        assert c.L.sj_exchange_create(c.h, r, world, 1, None) == 0
    locs = (C.c_void_p * world)(*[c.L.sj_exchange_local(c.h) for c in ctxs])

    def rank(r, bar):
        c = ctxs[r]
        assert c.L.sj_exchange_connect_ptrs(c.h, locs) == 0
        sp = ShardedParse(c)
        got = []
        for doc, want in cases:
            mine = doc if r == 1 else good
            bar.wait()
            if mine is None:
                got.append(None)  # this rank skips the call: the others time out, and the epochs no longer agree ...
                bar.wait()
                continue
            d = torch.full((len(mine) + 256,), 0x20, dtype=torch.uint8, device=dev)
            if mine:
                d[: len(mine)] = torch.frombuffer(bytearray(mine), dtype=torch.uint8).to(dev)
            torch.cuda.synchronize()
            t0 = time.time()
            rc, tot = sp.count(d.data_ptr(), len(mine), True)
            got.append((rc, time.time() - t0))
            if doc is None:
                bar.wait()
        return got

    out = _run_ranks(world, rank)
    for i, (doc, want) in enumerate(cases[:3]):
        assert out[1][i][0] == want, (i, out[1][i])
        assert out[0][i][0] == _lib.ERR_PEER and out[2][i][0] == _lib.ERR_PEER, (i, out[0][i], out[2][i])
        assert max(o[i][1] for o in out) < 1.0
    assert out[0][3][0] == _lib.ERR_EXCHANGE and out[2][3][0] == _lib.ERR_EXCHANGE and 1.5 < out[0][3][1] < 4.0, out[0][3]
    for c in ctxs:
        c.close()


def test_numbers_fast_path_shapes(ctx, oracle):
    """the one-pass fast path of K2h ([-]digits[.digits], at most 18 digits, no exponent) and its borders: the hook runs it
    beside the full routine on every item and poisons the tag on a disagreement; the full routine is checked against the oracle"""
    rng = np.random.default_rng(77)
    items = []
    for _ in range(30000):
        nd = int(rng.integers(1, 21))
        s = "".join(str(d) for d in rng.integers(0, 10, nd))
        if rng.integers(0, 4):
            s = s.lstrip("0") or "0"
        if rng.integers(0, 3):
            k = int(rng.integers(0, len(s) + 1))
            s = s[:k] + "." + s[k:]
        if rng.integers(0, 2):
            s = "-" + s
        items.append(s.encode() + [b",", b"]", b"}", b" ", b"\n", b":", b"\t", b"x", b"e5,", b"-"][int(rng.integers(0, 10))])
    for s in ("0", "-0", "0.0", "-0.0", "00.5", "-00.5", "0.5", "01", "-01", "1.", ".5", "-.5", "1.5.5", "1-", "-", "12x", "9007199254740992.0",
              "9007199254740993.0", "900719925474099.25", "0.000000000000000001", "123456789012345678", "1234567890123456789",
              "12345678901234567.8", "999999999999999999", "-999999999999999999", "0.1", "0.2", "0.3", "2.5", "1e5", "1E5", "1+5", "+1"):
        for term in (b",", b"]", b" "):
            items.append(s.encode() + term)
    items += [b"1234567890.123456," + b"   " * 10] * 3  # (pads the tail so the last real items have 26 readable bytes)
    res = ctx.parse_numbers(items)
    for it, (tag, val) in zip(items, res):
        otag, oval = oracle.parse_number(it)
        assert (tag, val) == (otag, oval), (it, hex(tag), hex(val), hex(otag), hex(oval))
