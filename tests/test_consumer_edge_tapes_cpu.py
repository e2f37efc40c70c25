"""The intentions of tests/consumer_edge_tapes.py against the sequential ports: every feature sits where it is meant
to, the recorded rows are the ones fo.roots (the head scan, on windows of the large tapes) and fo.foreach_roots find,
the recorded cells are fo.find's, and the countWhere counts are the C oracle's.  No GPU."""
import math

import numpy as np
import pytest

from tests import consumer_edge_tapes as ce
from tests import find_oracle as fo

_TAG = np.uint64(56)


def _tag(w):
    return chr(int(w) >> 56)


def _cells_equal(tape, strs, msg, paths, rows, want, shift=0, what=""):
    got = fo.find(tape, strs, msg, [p for p, _ in paths], [k for _, k in paths], rows)
    for p in range(len(paths)):
        for r in range(len(rows)):
            g, w = got[p][r].astuple(), want[p][r].astuple()
            g = (g[0], g[1], g[2] + shift if g[2] >= 0 else g[2], g[3])
            assert g == w, (what, paths[p], r, g, w)


def _check_feature(tape, f, rows):
    """the feature word of f sits at E + offset and is what its family says"""
    F, t = f.at, tape
    assert F == f.E + f.offset and f.E == ce.EDGES[f.edge]
    rows = set(int(r) for r in rows)
    ws, we = f.window
    assert ws < F < we or ws <= F - 1
    if f.family == "root_open":
        assert _tag(t[F]) == "r" and int(t[F]) & ce.VAL > F and F in rows
    elif f.family == "root_close":
        assert _tag(t[F]) == "r" and int(t[F]) & ce.VAL < F and F not in rows and F + 1 in rows
    elif f.family == "lookalike_num":
        assert _tag(t[F - 1]) == f.detail and _tag(t[F]) == "r" and int(t[F]) & ce.VAL > F and F not in rows
    elif f.family == "lookalike_str":
        assert _tag(t[F - 1]) == '"' and int(t[F]) == 5 and F not in rows
    elif f.family == "parity":
        k = int(f.detail.split()[-1])
        run = (t[F - 2 * k + 1:F + 1] >> _TAG).astype(np.int64)
        assert (run[:-1] == ord("d")).all() and run[-1] == ord("r") and int(t[F]) & ce.VAL > F and F not in rows
        assert k >= 64 or f.E == ce.T          # every run but the first tile's is long
    elif f.family == "key_straddle":
        assert _tag(t[F - 1]) == '"' and int(t[F]) == 1 and F - 6 in rows
    elif f.family == "value_straddle":
        assert _tag(t[F - 1]) == f.detail.split()[-1] and _tag(t[F - 3]) == '"' and int(t[F - 2]) == 1 and F - 8 in rows
    else:
        raise AssertionError(f.family)


def _check_windows(et):
    """fo.roots, the head scan, on the window of every feature, read from its first word; fo.foreach_roots from the
    window's first row; both equal the recorded rows inside the window"""
    for f in et.features:
        ws, we = f.window
        w = ce.window(et.tape, ws, we)
        inside = et.rows[(et.rows >= ws) & (et.rows < we)]
        assert len(inside) >= 2, (et.name, f)
        assert np.array_equal(fo.roots(w) + ws, inside), (et.name, f.edge)
        r0 = int(inside[0])
        assert np.array_equal(fo.foreach_roots(ce.window(et.tape, r0, we)) + r0, inside), (et.name, f.edge)


def _check_tape(et, oracle, full_scan):
    for f in et.features:
        _check_feature(et.tape, f, et.rows)
    assert np.array_equal(fo.foreach_roots(et.tape), et.rows), et.name
    if full_scan:
        assert np.array_equal(fo.roots(et.tape), et.rows), et.name
    _check_windows(et)
    _cells_equal(et.tape, et.strings, et.message, ce.EDGE_PATHS, et.rows, et.cells, what=et.name)
    for (key, value), n in et.count_where.items():
        assert oracle.count_where(et.tape, et.strings, et.message, key, value) == (len(et.rows), n), (et.name, key)


def test_geometry():
    assert ce.T == ce.TAPE_THREADS * ce.TAPE_ROUNDS and ce.G == ce.GROUP_TILES * ce.T
    assert ce.KC2_BLOCK % 32 == 0 and ce.FD_THREADS % 32 == 0
    assert [ce.EDGES[k] for k in ce.EDGE_KINDS] == [ce.T, 2 * ce.T, 1023 * ce.T, ce.G, ce.G + ce.T, 2 * ce.G]


def test_small_edge_tapes(oracle):
    """tapes under 100k words: rows and cells against the whole-tape ports"""
    n = 0
    for et in ce.edge_tapes(large=False):
        assert len(et.tape) < 100_000
        _check_tape(et, oracle, full_scan=True)
        n += 1
    assert n == len(ce.FAMILIES) * len(ce.OFFSETS)


@pytest.mark.parametrize("family", ce.FAMILIES)
def test_large_edge_tapes(oracle, family):
    """tapes of more than 2G words: the head scan on windows, ForEach's walk, every cell and the counts on the whole
    tape (every record but the ones around the edges is a long filler that the walks step over)"""
    for o in ce.OFFSETS:
        et = ce.edge_tape(family, o)
        assert len(et.tape) > 2 * ce.G
        assert [f.edge for f in et.features] == list(ce.EDGE_KINDS)
        _check_tape(et, oracle, full_scan=False)


def test_every_family_reaches_every_edge():
    seen = set()
    for et in ce.edge_tapes(large=False):
        seen.update((f.family, f.edge, f.offset) for f in et.features)
    for fam in ce.FAMILIES:
        for o in ce.OFFSETS:
            assert {(fam, e, o) for e in ce.SMALL_EDGES} <= seen
            et = ce.edge_tape(fam, o, ("T", "G+T"))   # the large layout's edges are the same generator's
            assert [(f.edge, f.at) for f in et.features] == [("T", ce.T + o), ("G+T", ce.G + ce.T + o)]
    # the look-alike numbers meet every tag, the value straddles every kind of value
    tags = {f.detail for f in ce.edge_tape("lookalike_num", 0).features}
    vals = {f.detail for f in ce.edge_tape("value_straddle", 0).features}
    assert tags == set("lud") and vals == {"value " + c for c in '"udl'}


# ---- conversions ---------------------------------------------------------------------------------------------------
def test_conversion_table_against_the_port():
    et, specs = ce.conversion_tape()
    paths = [([b"k"], k) for k in ce.KINDS]
    assert np.array_equal(fo.roots(et.tape), et.rows)
    _cells_equal(et.tape, et.strings, et.message, paths, et.rows, et.cells, what="conversions")
    tags = {s[0][0] for s in specs}
    assert tags == set('lud"tfn[{')


def _cell(specs, cells, spec, kind):
    return cells[kind][specs.index(spec)]


def test_conversion_table_spot_values():
    """the edges written out by hand"""
    et, specs = ce.conversion_tape()
    b = ce.f64_bits

    def c(spec, kind):
        x = _cell(specs, et.cells, spec, kind)
        return x.status, x.value

    MIN = 1 << 63
    assert c(("d", b(2.0 ** 63)), ce.INT64) == (ce.OK, MIN)                     # passes the > MaxInt64 test, then CVTTSD2SQ
    assert c(("d", b(math.nextafter(2.0 ** 63, math.inf))), ce.INT64)[0] == ce.CONVERT
    assert c(("d", b(math.nextafter(2.0 ** 63, 0))), ce.INT64) == (ce.OK, 2 ** 63 - 1024)
    assert c(("d", b(-(2.0 ** 63))), ce.INT64) == (ce.OK, MIN)
    assert c(("d", b(2.0 ** 64)), ce.UINT64) == (ce.OK, MIN)                    # int64(2^63) | 1 << 63
    assert c(("d", b(math.nextafter(2.0 ** 64, 0))), ce.UINT64) == (ce.OK, 2 ** 64 - 2048)
    assert c(("d", b(-0.0)), ce.UINT64) == (ce.OK, 0)
    assert c(("d", b(-0.5)), ce.UINT64)[0] == ce.CONVERT
    assert c(("d", b(-0.5)), ce.INT64) == (ce.OK, 0)
    assert c(("d", b(-1 + 2.0 ** -53)), ce.INT64) == (ce.OK, 0)
    assert c(("d", 0x7FF8000000000000), ce.INT64) == (ce.OK, MIN)             # NaN compares false both ways
    assert c(("d", 0xFFF8000000000000), ce.UINT64) == (ce.OK, MIN)
    assert c(("d", 0x7FF0000000000000), ce.INT64)[0] == ce.CONVERT
    assert c(("d", 0xFFF0000000000000), ce.UINT64)[0] == ce.CONVERT
    assert c(("l", 2 ** 53 + 1), ce.FLOAT64) == (ce.OK, b(2.0 ** 53))          # ties to even
    assert c(("l", 2 ** 53 + 3), ce.FLOAT64) == (ce.OK, b(2.0 ** 53 + 4))
    assert c(("u", 2 ** 62 + 2 ** 9), ce.FLOAT64) == (ce.OK, b(2.0 ** 62))
    assert c(("u", 2 ** 62 + 2 ** 9 + 1), ce.FLOAT64) == (ce.OK, b(2.0 ** 62 + 2 ** 10))
    assert c(("l", 2 ** 64 - 1), ce.FLOAT64) == (ce.OK, b(-1.0))
    assert c(("u", 2 ** 64 - 1), ce.FLOAT64) == (ce.OK, b(2.0 ** 64))
    assert c(("u", 2 ** 63), ce.INT64)[0] == ce.CONVERT and c(("u", 2 ** 63 - 1), ce.INT64) == (ce.OK, 2 ** 63 - 1)
    assert c(("l", 2 ** 63), ce.UINT64)[0] == ce.CONVERT
    assert c(('"', b"1", True), ce.INT64)[0] == ce.CONVERT and c(("t",), ce.STRING) == (ce.CONVERT, b"")
    assert c(("l", 1), ce.BOOL)[0] == ce.CONVERT and c(("f",), ce.BOOL) == (ce.OK, 0)


# ---- countWhere ----------------------------------------------------------------------------------------------------
def test_count_where_messages(oracle):
    """the matches of every message are the oracle's count and the rows whose [key] STRING cell is the value"""
    cases = ce.cw_cases()
    assert {n for n, _, _, _ in cases} == set(ce.CW_COUNTS) and {p for _, p, _, _ in cases} == set(ce.PATTERNS)
    assert {(k, v) for _, _, k, v in cases} >= {(k, v) for k in ce.CW_LENS for v in ce.CW_LENS}
    for n, pat, kl, vl in cases:
        msg, key, value, hits = ce.cw_message(n, pat, kl, vl)
        assert len(key) == kl and len(value) == vl
        rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=True)
        assert rc == 0
        assert oracle.count_where(tape, strs, msg[off:off + ln], key, value) == (n, len(hits)), (n, pat, kl, vl)
        if n <= ce.KC2_BLOCK + 1:
            rows = fo.foreach_roots(tape)
            cells = fo.find(tape, strs, msg[off:off + ln], [[key]], [fo.STRING], rows)[0]
            assert [r for r, c in enumerate(cells) if c.status == fo.OK and c.value == value] == hits


def test_count_where_group_message(oracle):
    msg, matches, words = ce.cw_group_message("lane0", n=70_000)
    rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=True)
    assert rc == 0 and len(tape) == words
    assert oracle.count_where(tape, strs, msg[off:off + ln], b"a", b"b") == (70_000, matches)
    # the device test's message is the same generator at more than G words
    assert ce.cw_group_message("lane0")[2] > ce.G


# ---- KF3 and KF5 ---------------------------------------------------------------------------------------------------
def test_kf3_paths_fill_the_limits():
    paths, kinds = ce.kf3_paths()
    assert len(paths) == ce.FD_MAX_PATHS and len({tuple(p) for p in paths}) == ce.FD_MAX_PATHS
    assert sum(len(s) for p in paths for s in p) == ce.FD_MAX_SEG_BYTES
    assert [] in paths and sum(len(p) == ce.FD_MAX_SEGS for p in paths) == 2
    longs = [p[0] for p in paths if len(p) == 1]
    assert len({len(k) for k in longs}) == 2   # one length (and one longer key): only their bytes tell them apart


def test_kf3_rows_repeat_their_templates():
    """row r is template r % KF3_TEMPLATES: the same words as that template's first row, moved; so fo.find on the first
    rows gives every cell.  Each template finds what it holds."""
    tape, strs, msg, slots = ce.kf3_tape(2 * ce.KF3_TEMPLATES + 1)
    assert np.array_equal(fo.roots(tape), slots)
    ends = list(slots[1:]) + [len(tape)]
    first = [ce.window(tape, int(slots[t]), int(ends[t])) for t in range(ce.KF3_TEMPLATES)]
    for r in range(len(slots)):
        w = ce.window(tape, int(slots[r]), int(ends[r]))
        f = first[r % ce.KF3_TEMPLATES]
        assert len(w) == len(f)
        # strings may sit at other offsets of Strings.B; every other word is the same
        tags = (w >> _TAG).astype(np.int64)
        same = (w == f) | (tags == ord('"'))
        assert same.all(), r
    paths, kinds = ce.kf3_paths()
    got = fo.find(tape, strs, msg, paths, kinds, slots[:ce.KF3_TEMPLATES])
    sts = {c.status for col in got for c in col}
    assert {fo.OK, fo.NOT_FOUND, fo.NOT_OBJECT, fo.CONVERT} <= sts
    for p, path in enumerate(paths):
        for t in range(ce.KF3_TEMPLATES):
            if len(path) == 1:
                assert (got[p][t].status == fo.NOT_FOUND) == ((p + t) % 5 == 0), (p, t)


def test_kf5_tapes():
    tape, strs, msg, paths, kinds, want = ce.kf5_mixed(rows=64)
    got = fo.find(tape, strs, msg, paths, kinds)
    for col, w in zip(got[:2], want[:2]):
        assert [c.value for c in col] == w
    assert {len(s) for s in want[0] + want[1]} == set(ce.KF5_LENS)
    for w0 in range(0, 64, 32):     # every warp of the first two mixes short and long strings
        assert {len(s) > ce.FD_SHORT for s in want[0][w0:w0 + 32]} == {True, False}
    rows = 300
    tape, strs, gpaths, slots, offs, lens = ce.kf5_group(rows)
    assert np.array_equal(fo.roots(tape), slots)
    got = fo.find(tape, strs, b"", gpaths[:4], [fo.STRING] * 4, slots)
    for k in range(4):
        assert b"".join(c.value for c in got[k]) == ce.gather(strs, offs[k], lens[k])
        assert all(c.status == fo.OK for c in got[k])
    assert ce.FD_MAX_PATHS * (ce.G // ce.FD_MAX_PATHS + 1) > ce.G


def test_boundary_messages(oracle):
    n = 0
    for name, msg, nd in ce.boundary_messages():
        rc, tape, strs, _ = oracle.parse(msg, ndjson=nd)
        assert rc == 0, name
        n += 1
    assert n > 60
