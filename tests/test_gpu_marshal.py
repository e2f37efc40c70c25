"""GPU tests of MarshalJSON on the device (marshal.cuh): Iter.MarshalJSON (parsed_json.go:394-556) of the tape in HBM,
against the reference's expected texts and the oracle's walk of the oracle's tape (tests/marshal_oracle.py)."""
import ctypes as C

import numpy as np
import pytest

from tests import marshal_oracle as mo
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, golden, load_fixture, tricky_ndjson, unhex

pytestmark = pytest.mark.gpu

OK, ERR_CAPACITY, ERR_ARGUMENT = 0, 4, 6


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _want(oracle, msg, ndjson, copy=True):
    rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
    return rc, (mo.marshal(tape, strs, msg[off:off + ln]) if rc == 0 else None)


def _upload(tape, strs, msg):
    import torch
    d_tape = torch.from_numpy(np.ascontiguousarray(tape).view(np.int64).copy()).cuda()
    d_strs = torch.from_numpy(np.frombuffer(strs + b"\0", dtype=np.uint8).copy()).cuda()
    d_msg = torch.from_numpy(np.frombuffer(msg + b"\0", dtype=np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    return d_tape, d_strs[:len(strs)], d_msg[:len(msg)]


def _marshal_device(ctx, tape, strs, msg):
    d_tape, d_strs, d_msg = _upload(tape, strs, msg)
    rc, n, out = ctx.marshal_device(d_tape, d_strs, d_msg)
    return rc, (out.cpu().numpy().tobytes() if rc == OK else None)


def _golden_cases():
    g = golden("G16_G17_documents")
    for tc in g["parse_nd"]:
        if tc["want"] is not None:
            yield tc["name"], unhex(tc["js"]), True, unhex(tc["want"])
    for tc in g["pass_cases"]:
        if tc["want"] is not None:
            yield tc["name"], unhex(tc["js"]), False, unhex(tc["want"])


@pytest.mark.parametrize("impl", [0, 1])
def test_golden_texts(ctx, impl):
    cases = list(_golden_cases())
    assert len(cases) == 19
    ctx.set_stage2_impl(impl)
    try:
        for name, js, ndjson, want in cases:
            for copy in (True, False):
                assert ctx.parse_marshal(js, ndjson=ndjson, copy_strings=copy) == (OK, want), (name, copy, impl)
    finally:
        ctx.set_stage2_impl(0)


def test_fixtures_vs_oracle(ctx, oracle_native):
    for name in TAPE_FILES + SMALL_FILES + ["parking-citations"]:
        msg = load_fixture(name)
        nd = name == "parking-citations"
        for copy in (True, False):
            rc, want = _want(oracle_native, msg, nd, copy)
            assert rc == 0
            got = ctx.parse_marshal(msg, ndjson=nd, copy_strings=copy)
            assert got == (OK, want), (name, copy, len(got[1]), len(want))


def test_tricky_records_and_empty_lines(ctx, oracle):
    nd, _ = tricky_ndjson()
    for msg in (nd, b"\n\n" + nd.replace(b"\n", b"\n\n\n") + b"\n  \n", b'{"a":"\\u0001\\u001f\\"\\\\\\/\\b\\f\\n\\r\\t\\u007f\\u00ff"}'):
        for copy in (True, False):
            rc, want = _want(oracle, msg, True, copy)
            assert rc == 0 and ctx.parse_marshal(msg, ndjson=True, copy_strings=copy) == (OK, want)
    assert ctx.parse_marshal(b'{"a":1}\n{"b":\n', ndjson=True)[0] == 1
    assert ctx.parse_marshal(b'{"a":1}\n{"b" 2}\n', ndjson=True)[0] == 2
    assert ctx.parse_marshal(b"  \n ")[0] == 1


@pytest.mark.parametrize("which,expect", [("corpus", 8000), ("go-corpus", 300)])
def test_fuzz_seeds_vs_oracle(ctx, oracle_native, which, expect):
    n = parsed = 0
    for name, data in fuzz_corpus(which):
        n += 1
        rc, want = _want(oracle_native, data, False)
        got = ctx.parse_marshal(data)
        if rc != 0:
            assert got[0] == rc, name
            continue
        parsed += 1
        assert got == (OK, want), name
    assert n > expect and parsed > 0, (n, parsed)


def test_foreign_tapes(ctx, oracle):
    """oracle tapes uploaded with torch, through sj_marshal_device, in both copy modes"""
    nd, _ = tricky_ndjson()
    pk = load_fixture("parking-citations").strip()
    for msg, ndjson in ((nd, True), (pk, True), (load_fixture("twitterescaped"), False), (load_fixture("canada"), False),
                        (b'[[],{},[[{}]],{"a":[]},"",0,-0.0,1e300]', False)):
        for copy in (True, False):
            rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
            assert rc == 0
            want = mo.marshal(tape, strs, msg[off:off + ln])
            assert _marshal_device(ctx, tape, strs, msg[off:off + ln]) == (OK, want)
    import torch
    rc, n, out = ctx.marshal_device(torch.zeros(0, dtype=torch.int64, device="cuda"))
    assert (rc, n) == (OK, 0)


def test_capacity_leaves_the_buffer_alone(ctx, oracle):
    import torch
    msg = load_fixture("twitter")
    rc, tape, strs, (off, ln) = oracle.parse(msg)
    want = mo.marshal(tape, strs, msg[off:off + ln])
    d_tape, d_strs, d_msg = _upload(tape, strs, msg[off:off + ln])
    buf = torch.full((len(want) + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc, n, _ = ctx.marshal_device(d_tape, d_strs, d_msg, out=buf[:len(want) - 1])
    assert (rc, n) == (ERR_CAPACITY, len(want))
    assert bool((buf == 0xA5).all())
    rc, n, out = ctx.marshal_device(d_tape, d_strs, d_msg, out=buf[:len(want)])
    assert (rc, n) == (OK, len(want)) and out.cpu().numpy().tobytes() == want
    assert bool((buf[len(want):] == 0xA5).all())  # the canary behind the text
    out_len = C.c_size_t(0)
    host = np.full(len(want) + 8, 0xA5, dtype=np.uint8)
    rc = ctx.L.sj_parse_marshal(ctx.h, msg, len(msg), 2, host.ctypes.data, len(want) - 1, C.byref(out_len))
    assert (rc, out_len.value) == (ERR_CAPACITY, len(want)) and (host == 0xA5).all()


def _word(tag, v=0):
    return (ord(tag) << 56) | v


def test_malformed_tapes(ctx, oracle):
    msg = b'{"a":[1,2.5,"x"],"b":{}}'
    rc, tape, strs, (off, ln) = oracle.parse(msg)
    assert rc == 0
    m = msg[off:off + ln]
    assert _marshal_device(ctx, tape, strs, m) == (OK, mo.marshal(tape, strs, m))
    # 0 r 1 { 2 " 3 . 4 [ 5 l 6 . 7 d 8 . 9 " 10 . 11 ] 12 " 13 . 14 { 15 } 16 } 17 r
    assert [chr(int(w) >> 56) for w in tape[[0, 1, 2, 4, 5, 7, 9, 11, 12, 14, 15, 16, 17]]] == list('r{"[ld"]"{}}r')
    cases = {
        "unknown tag": {5: _word("x")},
        "nop tag": {14: _word("N", 2), 15: _word("N", 1)},
        "open link out of range": {4: _word("[", 1000)},
        "open link not at its close": {4: _word("[", 10)},
        "close pointing elsewhere": {11: _word("]", 2)},
        "root link broken": {0: _word("r", 12)},
        "root close pointing elsewhere": {17: _word("r", 1)},
        "string outside Strings.B": {9: int(tape[9]) + 100},
        "string length outside Strings.B": {10: 1 << 40},
        "string outside the message": {9: _word('"', 1000)},
        "key not a string": {2: _word("t"), 3: _word("t")},
        "float NaN": {8: 0x7FF8000000000000},
        "float Inf": {8: 0x7FF0000000000000},
    }
    for name, change in cases.items():
        bad = tape.copy()
        for k, v in change.items():
            bad[k] = v
        with pytest.raises(mo.MalformedTape):
            mo.marshal(bad, strs, m)
        assert _marshal_device(ctx, bad, strs, m)[0] == ERR_ARGUMENT, name
    for bad in (tape[:-1], tape[1:], tape[:9], np.concatenate([tape, tape[:1]])):  # cut or unbalanced tapes
        assert _marshal_device(ctx, bad, strs, m)[0] == ERR_ARGUMENT
    # an object that ends behind a key: r { "a" } r
    dangling = np.array([_word("r", 6), _word("{", 5), _word('"', 1 << 55), 1, _word("}", 1), _word("r", 0)], dtype=np.uint64)
    with pytest.raises(mo.MalformedTape):
        mo.marshal(dangling, strs, m)
    assert _marshal_device(ctx, dangling, strs, m)[0] == ERR_ARGUMENT
    # a string at the very end of the tape has no length word
    assert _marshal_device(ctx, np.array([_word('"')], dtype=np.uint64), strs, m)[0] == ERR_ARGUMENT


def test_fixed_point(ctx):
    for name in ("twitter", "canada", "citm_catalog", "twitterescaped"):
        rc, a = ctx.parse_marshal(load_fixture(name))
        assert rc == 0
        assert ctx.parse_marshal(a) == (OK, a), name
    rc, a = ctx.parse_marshal(load_fixture("parking-citations"), ndjson=True)
    assert rc == 0 and ctx.parse_marshal(a, ndjson=True) == (OK, a)


def test_iter_marshal_json(oracle):
    import simdjson_b200 as sj
    msg = load_fixture("citm_catalog")
    pj = sj.Parse(msg)
    assert pj.Iter().MarshalJSON() == _want(oracle, msg, False)[1]
    nd, _ = tricky_ndjson()
    pj = sj.ParseND(nd, copy_strings=False)
    assert pj.Iter().MarshalJSON() == _want(oracle, nd, True, False)[1]


def test_scale_replicated_ndjson(ctx):
    pk = load_fixture("parking-citations").strip()
    rc, m = ctx.parse_marshal(pk, ndjson=True)
    assert rc == 0
    big = b"\n".join([pk] * 700)  # about 260 MB, 700 000 records
    rc, got = ctx.parse_marshal(big, ndjson=True)
    assert rc == 0 and got == b"\n".join([m] * 700)


def test_scale_single_document(ctx):
    """one root of about 0.5 GiB: the work is spread over tape words, not over roots"""
    tw = load_fixture("twitter")
    rc, m = ctx.parse_marshal(tw)
    assert rc == 0
    k = (512 << 20) // len(tw)
    big = b"[" + b",".join([tw] * k) + b"]"
    del tw
    rc, got = ctx.parse_marshal(big)
    assert rc == 0 and got == b"[" + b",".join([m] * k) + b"]"
