"""Stage 1's per-slab counts (parse mode) against stage 2's tape writer.

In the streaming parse, stage 1 adds up for every 6 KiB slab what stage 2 needs to know about it (tape words, string
bytes, brackets, depth, records, numbers, the bytes under its last structurals) and the tape writer (K2r) takes its
offsets from the scan of those counts.  K2r recounts every slab with the same function and records any disagreement in
an internal-error word.  These tests put the carries between slabs -- strings, escapes and backslash runs that straddle
slab and tile edges, record boundaries and blank runs at a slab edge, a string over several tiles, a message of one
slab -- at every offset around the edges and require the oracle's tape and strings and an internal-error word of 0,
then the same over the whole fuzz corpus."""
import ctypes as C

import numpy as np
import pytest

from tests.util import fuzz_corpus

pytestmark = pytest.mark.gpu

SLAB = 6 * 1024       # stage 1's slab (one warp) = stage 2's slab
TILE = 16 * SLAB      # stage 1's tile (one look-back)


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _internal(ctx):
    w = C.c_uint32(0xFFFFFFFF)
    assert ctx.L.sj_test_stage2_internal(ctx.h, C.byref(w)) == 0
    return w.value


def _check(ctx, oracle, msg, ndjson):
    rc_g, tape_g, str_g, win_g = ctx.parse(msg, ndjson=ndjson, copy_strings=True)
    assert _internal(ctx) == 0, ("stage 1's and K2r's slab counts differ", len(msg), bytes(msg[:60]))
    rc_o, tape_o, str_o, win_o = oracle.parse(msg, ndjson=ndjson, copy_strings=True)
    assert rc_g == rc_o, (rc_g, rc_o, len(msg), bytes(msg[:60]))
    assert win_g == win_o
    if rc_o == 0:
        assert len(tape_g) == len(tape_o) and np.array_equal(tape_g, tape_o)
        assert str_g == str_o


def _place(edge, feature, at, head=b'{"k":"', tail=b'"}'):
    """one record whose `feature` starts `at` bytes in front of message offset `edge` (negative: behind it)"""
    pad = edge - at - len(head)
    assert pad >= 0
    return head + b"x" * pad + feature + tail


EDGES = [SLAB, 2 * SLAB, TILE, TILE + SLAB]
FEATURES = [
    b'\\u00e9\\n\\"z',              # escapes, an escaped quote
    b'\\ud83d\\ude00\\u0041',        # a surrogate pair
    b'\\\\\\\\"',                     # even backslash runs, then the closing quote
    b'\\uZZZZ',                      # an invalid escape
    b'ab","n":[1,-2.5e3,true,null,{"x":false}],"s":"',  # structurals of every kind
]


@pytest.mark.parametrize("edge", EDGES)
def test_features_across_slab_and_tile_edges(ctx, oracle_native, edge):
    for f in FEATURES:
        for at in range(-14, 15):
            doc = _place(edge, f, at)
            _check(ctx, oracle_native, doc, False)
            _check(ctx, oracle_native, doc + b"\n" + doc, True)


def test_backslash_runs(ctx, oracle_native):
    for run in list(range(1, 40)) + [63, 64, 65, 127, 128, 129, 200]:
        for at in (run + 1, run, run - 1, run // 2, 1, 0, -1):
            for edge in (SLAB, TILE):
                if edge - at - 6 < 0:
                    continue
                doc = _place(edge, b"\\" * run + b"q", at)
                _check(ctx, oracle_native, doc, False)


def test_record_boundaries_and_blank_runs_at_slab_edges(ctx, oracle_native):
    rec = b'{"a":[1,2,{"b":"c"}],"t":true}'
    for edge in (SLAB, 2 * SLAB, TILE):
        for blanks in (0, 1, 31, 32, 33, 100):
            for d in range(-3, 4):
                first = _place(edge + d - blanks, b"", 0)
                msg = first + b"\n" + (b" \t\r" * blanks)[:blanks] + rec + b"\n" + rec
                _check(ctx, oracle_native, msg, True)
                msg2 = first + (b" \t\r" * blanks)[:blanks] + b"\n" + rec
                _check(ctx, oracle_native, msg2, True)


def test_string_over_several_tiles(ctx, oracle_native):
    body = (b"abc\\u00e9\\\\" * (3 * TILE // 11 + 1))[: 3 * TILE + 123]
    doc = b'{"long":"' + body + b'","n":7}'
    _check(ctx, oracle_native, doc, False)
    _check(ctx, oracle_native, doc + b"\n" + doc, True)


def test_single_slab_messages(ctx, oracle_native):
    for n in (1, 100, SLAB - 10, SLAB - 1, SLAB):
        doc = _place(n - 2, b"", 0) if n > 8 else b'{"a":1}'
        assert len(doc) <= SLAB
        _check(ctx, oracle_native, doc, False)
        _check(ctx, oracle_native, doc, True)


@pytest.mark.parametrize("which,expect", [("corpus", 8000), ("go-corpus", 300)])
def test_internal_word_over_fuzz_corpus(ctx, oracle_native, which, expect):
    n = 0
    for _, data in fuzz_corpus(which):
        for nd in (False, True):
            ctx.parse(data, ndjson=nd, copy_strings=True)
            assert _internal(ctx) == 0, (which, n, bytes(data[:60]))
        n += 1
    assert n > expect, n
