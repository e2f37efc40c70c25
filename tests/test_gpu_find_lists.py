"""GPU tests of the find's list cells (SJ_FIND_KIND_ARRAY_* and STRING_CVT, find_list.cuh): device against the Python
port (tests/find_lists_oracle.py) cell for cell -- status, tag, index, value, list offsets, elements and bytes -- on
fixtures as documents and as NDJSON, fuzz seeds, the tricky records and foreign tapes with nops inside arrays; builder
tapes that put cell edges and stop words on the list passes' tile (4 096 virtual words) and group (1 024 tiles) edges,
cells of 0, 1 and 2 elements beside one of more than 2^24, and strings longer than FD_SHORT; mixed path sets; the
capacity contract and the kind split; and a 0.5 GiB one-array document against its generator."""
import ctypes as C

import numpy as np
import pytest

from tests import find_json_oracle as fj
from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import fmt_values
from tests.tape_builder import TapeBuilder, word
from tests.test_find_json_cpu import harvest
from tests.test_find_lists_cpu import NDJSON_FIXTURES, ndjson_paths, ndjson_records
from tests.util import TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu
TILE, GROUP = 4096, 4096 * 1024
VAR = (fo.STRING, fj.JSON, fl.STRING_CVT, fl.ARRAY_STRING, fl.ARRAY_STRING_CVT)
ALL = list(fl.LIST_KINDS) + [fl.STRING_CVT]


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _dev(a, dtype=np.uint8):
    import torch
    a = np.frombuffer(bytes(a), dtype=np.uint8) if not isinstance(a, np.ndarray) else a
    return torch.from_numpy(np.ascontiguousarray(a).view(dtype).copy()).cuda() if a.size else None


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def want_cells(tape, strs, msg, paths, kinds, rows=None):
    """per path, per row: (status, tag, index, value, elements, bytes) from the ports"""
    rs = fo.foreach_roots(tape) if rows is None else rows
    out = []
    for path, k in zip(paths, kinds):
        col = []
        for r in rs:
            if k in fl.LIST_KINDS or k == fl.STRING_CVT:
                c, e, b = fl.list_cell(tape, strs, msg, int(r), path, k)
            elif k == fj.JSON:
                c = fj.json_cell(tape, strs, msg, int(r), path)
                e, b = [], c.value
            else:
                c = fo.find_cell(tape, strs, msg, int(r), path, k)
                e, b = [], c.value if k == fo.STRING else b""
            v = len(b) if k in (fo.STRING, fj.JSON) else c.value
            col.append((c.status, c.tag, c.index, v, e, b))
        out.append(col)
    return out


def check(cols, rows, want, kinds, what):
    """every cell; the byte columns' offsets and the list offsets are checked to be contiguous across their columns"""
    at_s = at_e = 0
    for p, k in enumerate(kinds):
        c = cols[p]
        st, tag, idx, val = _np(c.status), _np(c.tag), _np(c.index), _np(c.value).view(np.uint64)
        assert len(want[p]) == rows, what
        if k in VAR:
            off, data = _np(c.offsets), _np(c.data).tobytes()
            assert int(off[0]) == at_s, (what, p)
            at_s = int(off[rows])
        if k in fl.LIST_KINDS:
            lo, el = _np(c.list_offsets), _np(c.elems).view(np.uint64)
            assert int(lo[0]) == at_e, (what, p)
            at_e = int(lo[rows])
        for r, (s, t, i, v, e, b) in enumerate(want[p]):
            got = (int(st[r]), int(tag[r]), int(idx[r]), int(val[r]))
            assert got == (s, t, i, v), (what, p, k, r, got, (s, t, i, v))
            if k in fl.LIST_KINDS:
                assert np.array_equal(el[lo[r]:lo[r + 1]], np.array(e, dtype=np.uint64)), (what, p, k, r)
            if k in VAR:
                assert data[off[r]:off[r + 1]] == b, (what, p, k, r, data[off[r]:off[r + 1]][:100], b[:100])


def _foreign(ctx, tape, strs, msg, paths, kinds, what, rows=None):
    rc, n, cols = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), paths, kinds)
    assert rc == 0, (what, rc)
    check(cols, n, want_cells(tape, strs, msg, paths, kinds, rows), kinds, what)


def _kinds(n):
    return [ALL[i % len(ALL)] for i in range(n)]


def _per_kind(paths):
    """every path under every list kind and STRING_CVT, in calls of at most 60 paths"""
    ps, ks = [p for p in paths for _ in ALL], [k for _ in paths for k in ALL]
    return [(ps[i:i + 60], ks[i:i + 60]) for i in range(0, len(ps), 60)]


@pytest.mark.parametrize("name", TAPE_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures(ctx, oracle_native, name, copy):
    """own tape (sj_parse_find_lists) and the oracle's tape as a foreign one"""
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc, copy_strings=copy)
    assert rc == 0
    msg = doc[off:off + ln]
    for paths, kinds in _per_kind(harvest(doc, 60)[:12] + harvest(doc, 60)[-3:]):
        want = want_cells(tape, strs, msg, paths, kinds)
        rc, rows, cols = ctx.parse_find(doc, paths, kinds, ndjson=False, copy_strings=copy)
        assert rc == 0
        check(cols, rows, want, kinds, name)
        _foreign(ctx, tape, strs, msg, paths, kinds, name)


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
@pytest.mark.parametrize("copy", [True, False])
def test_ndjson_fixtures(ctx, oracle, name, copy):
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
    assert rc == 0
    for paths, kinds in _per_kind(ndjson_paths(recs)[:30]):
        rc, rows, cols = ctx.parse_find(nd, paths, kinds, copy_strings=copy)
        assert rc == 0 and rows == len(recs)
        check(cols, rows, want_cells(tape, strs, nd[off:off + ln], paths, kinds), kinds, name)


def test_mesh_is_bit_exact(ctx):
    import json
    doc = load_fixture("mesh")
    v = json.loads(doc)
    paths = [[b"positions"], [b"normals"], [b"tex0"], [b"indices"], [b"colors"], [b"influences"]]
    kinds = [fl.ARRAY_FLOAT64] * 3 + [fl.ARRAY_INT64] * 2 + [fl.ARRAY_FLOAT64]
    rc, rows, cols = ctx.parse_find(doc, paths, kinds, ndjson=False)
    assert rc == 0 and rows == 1
    for p, (path, k) in enumerate(zip(paths[:5], kinds)):
        e = cols[p].elems[cols[p].list_offsets[0]:cols[p].list_offsets[1]]
        assert np.array_equal(e, np.array(v[path[0].decode()], dtype=e.dtype)), path
    assert cols[5].status[0] == fo.CONVERT


def test_tricky_ndjson(ctx, oracle):
    nd, recs = tricky_ndjson()
    paths = [[b"Make"], [b"a"], [b"a", b"Make"], [b""], [b"t"], [b"f"], [b"n"], [b"d"], [b"l"], [b"u"], [b"x"], [b"nope"], []]
    for copy in (True, False):
        rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
        for ps, kinds in _per_kind(paths):
            rc, rows, cols = ctx.parse_find(nd, ps, kinds, copy_strings=copy)
            assert rc == 0 and rows == len(recs)
            check(cols, rows, want_cells(tape, strs, nd[off:off + ln], ps, kinds), kinds, "tricky")


def test_fuzz_seeds(ctx, oracle):
    n = 0
    for name, data in fuzz_corpus("corpus", max_size=1 << 14):
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson)
            if rc:
                continue
            paths = harvest(data, 24)
            kinds = _kinds(len(paths))
            rc, rows, cols = ctx.parse_find(data, paths, kinds, ndjson=ndjson)
            assert rc == 0, name
            check(cols, rows, want_cells(tape, strs, data[off:off + ln], paths, kinds), kinds, name)
            n += 1
    assert n > 20


def _obj(inner, at=0):
    """r { "a": <inner> } r at word `at`, inner's links relative to its first word at at + 4"""
    n = 4 + len(inner)
    return [word("r", at + n + 2), word("{", at + n + 1), word('"', 1 << 55), 1] + list(inner) + [word("}", at + 1), word("r", at)]


def test_nops_inside_arrays(ctx):
    """foreign tapes with nops inside arrays: AsFloat stops on them, AsString's AdvanceIter skips them (one thread
    finishes that cell), a nop skip of 0 is CORRUPT; Deserialize's output as a foreign tape"""
    import simdjson_b200 as sj
    S = 1 << 55
    rows_words, at = [], 0
    for inner in ([word("l"), 1, word("N", 1), word("l"), 2],
                  [word('"', S), 1, word("N", 1), word("x"), word('"', S | 1), 2, word("N", 2), 0, 0, word('"', S | 2), 3],
                  [word('"', S), 1, word("N", 0), word('"', S | 1), 2],
                  [word("N", 1), word("x"), word("t"), word("l"), 7, word("[", 0), word("]", 0)],
                  [word('"', S | 3), 40, word("N", 1), word("x"), word('"', S | 3), 40]):
        arr = [word("[", at + 4 + len(inner) + 2)] + inner + [word("]", at + 4)]
        rows_words.append(_obj(arr, at))
        at += len(rows_words[-1])
    # the nested '[' of row 3 needs its links: fix them in place
    words = [w for r in rows_words for w in r]
    k = [i for i, w in enumerate(words) if w == word("[", 0)][0]
    words[k], words[k + 1] = word("[", k + 2), word("]", k)
    tape = np.array(words, dtype=np.uint64)
    strs = bytes(range(48, 48 + 50))
    rows = fo.roots(tape)
    assert len(rows) == 5
    for kinds in ([fl.ARRAY_FLOAT64], [fl.ARRAY_STRING], [fl.ARRAY_STRING_CVT], [fl.ARRAY_INT64]):
        _foreign(ctx, tape, strs, b"", [[b"a"]], kinds, ("nops", kinds), rows)
    doc = load_fixture("update-center")
    pj = sj.Parse(doc, ctx=ctx)
    back = sj.Serializer(ctx).Deserialize(sj.Serializer(ctx).Serialize(pj))
    tape, strs, msg = (np.asarray(back.Tape, dtype=np.uint64), bytes(back.Strings), bytes(back.Message))
    ((paths, kinds),) = _per_kind([[b"core", b"name"], [b"signature", b"certificates"], [b"plugins", b"AdaptivePlugin", b"labels"]])
    _foreign(ctx, tape, strs, msg, paths, kinds, "deserialize")


def _rows_tape(arrays):
    """one root { "a": [...] } per array of (tag, payload) items; returns the tape and Strings.B"""
    b = TapeBuilder()
    for items in arrays:
        b.open("r"); b.open("{"); b.string(b"a"); b.open("[")
        for t, v in items:
            if t in "lud":
                b.number(t, v)
            elif t == '"':
                b.string(v)
            else:
                b.atom(t)
        b.close(); b.close(); b.close()
    tape, strs, msg = b.build()
    return tape, strs, msg


def test_cell_edges_and_stops_on_tile_edges(ctx):
    """the path's virtual words are the arrays laid end to end: cell heads, last words and stop words (a `t` among
    numbers, a number among strings) at every offset -2 .. +2 of tile edges"""
    rng = np.random.default_rng(7)
    arrays, v = [], 0
    for edge in range(1, 6):
        for d in (-2, -1, 0, 1, 2):
            # pad to edge * TILE + d with one array of numbers, then a short array whose stop lands there
            target = edge * TILE + d
            k = max(0, (target - v - 2) // 2)
            arrays.append([("l", int(x)) for x in rng.integers(-5, 5, k)])
            v += 2 + 2 * k
            arrays.append([("l", 1), ("t", 0), ("l", 2)] if d % 2 else [('"', b"x" * 40), ("l", 3), ('"', b"yz")])
            v += 2 + (5 if d % 2 else 6)
    tape, strs, msg = _rows_tape(arrays)
    for k in ALL:
        _foreign(ctx, tape, strs, msg, [[b"a"]], [k], ("tile edges", k))


def test_small_cells_beside_a_huge_one_across_group_edges(ctx):
    """cells of 0, 1 and 2 elements on both sides of one of 2^24 + 5 int64s, which crosses eight group edges; the
    expected columns come from the generator"""
    rng = np.random.default_rng(11)
    big = rng.integers(-(1 << 40), 1 << 40, (1 << 24) + 5)
    b = TapeBuilder()
    small = [[], [5], [6, -7]]
    for arr in small + [big] + small[::-1]:
        b.open("r"); b.open("{"); b.string(b"a"); b.open("[")
        b.numbers("l", np.asarray(arr, dtype=np.int64).view(np.uint64))
        b.close(); b.close(); b.close()
    tape, strs, msg = b.build()
    kinds = [fl.ARRAY_FLOAT64, fl.ARRAY_INT64, fl.ARRAY_UINT64, fl.ARRAY_STRING_CVT]
    rc, rows, cols = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), [[b"a"]] * 4, kinds)
    assert rc == 0 and rows == 7
    arrays = small + [big] + small[::-1]
    for p, k in enumerate(kinds):
        c = cols[p]
        lo, el = _np(c.list_offsets), _np(c.elems)
        for r, arr in enumerate(arrays):
            a = np.asarray(arr, dtype=np.int64)
            if k == fl.ARRAY_UINT64 and (a < 0).any():
                assert (int(c.status[r]), lo[r + 1] - lo[r]) == (fo.CONVERT, 0)
                continue
            assert int(c.status[r]) == fo.OK and int(c.value[r]) == a.size, (k, r)
            got = el[lo[r]:lo[r + 1]]
            if k == fl.ARRAY_STRING_CVT:
                off, data = _np(c.offsets), _np(c.data)
                text = "".join(str(x) for x in a.tolist()).encode()
                assert data[off[r]:off[r + 1]].tobytes() == text, r
                assert np.array_equal(got, np.char.str_len(a.astype(str)).astype(np.int64)), r
            else:
                assert np.array_equal(got, a.astype(got.dtype)), (k, r)


def test_long_strings_and_formatted_doubles(ctx):
    """string lists whose strings are longer than FD_SHORT (copied by the whole warp) beside short ones, and
    STRING_CVT of fmt_values' doubles"""
    rng = np.random.default_rng(3)
    arrays = []
    for n in range(60):
        arrays.append([('"', bytes(rng.integers(97, 123, int(x)).astype(np.uint8))) for x in rng.integers(0, 200, n % 13)])
    xs = np.concatenate([fmt_values.powers_of_two()[::5], fmt_values.notation_edges()])
    arrays.append([("d", int(x)) for x in xs])
    tape, strs, msg = _rows_tape(arrays)
    for k in (fl.ARRAY_STRING, fl.ARRAY_STRING_CVT):
        _foreign(ctx, tape, strs, msg, [[b"a"]], [k], ("long strings", k))
    # STRING_CVT scalars: one root per double
    b = TapeBuilder()
    for x in xs.tolist():
        b.open("r"); b.open("{"); b.string(b"a"); b.number("d", x); b.close(); b.close()
    tape, strs, msg = b.build()
    _foreign(ctx, tape, strs, msg, [[b"a"]], [fl.STRING_CVT], "string_cvt doubles")


def test_mixed_path_sets_equal_paths_alone(ctx):
    recs, nd = ndjson_records("twitter")
    paths = [[b"text"], [b"entities", b"hashtags"], [b"user"], [b"id"], [b"coordinates", b"coordinates"],
             [b"user", b"name"], [b"contributors"], [b"id_str"]]
    kinds = [fo.STRING, fl.ARRAY_STRING_CVT, fj.JSON, fo.INT64, fl.ARRAY_FLOAT64, fl.STRING_CVT, fl.ARRAY_STRING, fl.ARRAY_INT64]
    rc, rows, mixed = ctx.parse_find(nd, paths, kinds)
    assert rc == 0
    for p, (path, k) in enumerate(zip(paths, kinds)):
        rc, rows2, (alone,) = ctx.parse_find(nd, [path], [k])
        assert rc == 0 and rows2 == rows
        m = mixed[p]
        for f in range(4):
            assert np.array_equal(m[f], alone[f]), (path, f)
        if k in VAR:
            assert [m.data[m.offsets[r]:m.offsets[r + 1]].tobytes() for r in range(rows)] == \
                   [alone.data[alone.offsets[r]:alone.offsets[r + 1]].tobytes() for r in range(rows)], path
        if k in fl.LIST_KINDS:
            assert np.array_equal(np.diff(m.list_offsets), np.diff(alone.list_offsets)), path
            assert np.array_equal(m.elems[m.list_offsets[0]:m.list_offsets[rows]], alone.elems), path


def test_capacity_and_kind_split(ctx):
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    recs, nd = ndjson_records("update-center")
    paths = [[b"labels"], [b"name"], [b"dependencies"]]
    kinds = [fl.ARRAY_STRING, fl.STRING_CVT, fl.ARRAY_STRING_CVT]
    rc, rows, cols = ctx.parse_find(nd, paths, kinds)
    assert rc == 0
    nb = int(cols[2].offsets[rows])
    ne = int(cols[0].list_offsets[rows]) + int(cols[2].list_offsets[rows] - cols[2].list_offsets[0])
    pj = sj.ParseND(nd, ctx=ctx)
    tape, strs, msg = _dev(np.asarray(pj.Tape, dtype=np.uint64), np.int64), _dev(bytes(pj.Strings)), _dev(bytes(pj.Message))
    cpaths, keep = sj._find_paths(paths, kinds)
    r, b, e = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    L = ctx.L
    args = (ctx.h, msg.data_ptr(), msg.numel(), tape.data_ptr(), tape.numel(), strs.data_ptr(), strs.numel(), cpaths, 3)
    # sizes only: lists NULL
    rc = L.sj_find_lists_device(*args, None, None, C.byref(r), C.byref(b), C.byref(e))
    assert (rc, r.value, b.value, e.value) == (_lib.ERR_CAPACITY, rows, nb, ne)
    # one element short: SJ_ERR_CAPACITY with exact sizes, and nothing written
    import torch
    o = [torch.full((3, rows), 0xAB, dtype=torch.uint8, device="cuda"), torch.full((3, rows), 0xAB, dtype=torch.uint8, device="cuda"),
         torch.full((3, rows), -3, dtype=torch.int64, device="cuda"), torch.full((3, rows), -3, dtype=torch.int64, device="cuda"),
         torch.full((3, rows + 1), -3, dtype=torch.int64, device="cuda"), torch.full((nb,), 0xAB, dtype=torch.uint8, device="cuda"),
         torch.full((2, rows + 1), -3, dtype=torch.int64, device="cuda"), torch.full((ne,), -3, dtype=torch.int64, device="cuda")]
    fo_ = _lib.FindOut(*(t.data_ptr() for t in o[:6]), rows, nb)
    lo = _lib.FindListsOut(o[6].data_ptr(), o[7].data_ptr(), ne - 1)
    rc = L.sj_find_lists_device(*args, C.byref(fo_), C.byref(lo), C.byref(r), C.byref(b), C.byref(e))
    assert (rc, r.value, b.value, e.value) == (_lib.ERR_CAPACITY, rows, nb, ne)
    torch.cuda.synchronize()
    assert all(bool((t == (0xAB if t.dtype == torch.uint8 else -3)).all()) for t in o)
    lo = _lib.FindListsOut(o[6].data_ptr(), o[7].data_ptr(), ne)
    rc = L.sj_find_lists_device(*args, C.byref(fo_), C.byref(lo), C.byref(r), C.byref(b), C.byref(e))
    assert rc == 0
    # list kinds through the old entry points, and kind 6 anywhere
    for k in list(fl.LIST_KINDS) + [6]:
        cp, keep2 = sj._find_paths([[b"labels"]], [k])
        rc = L.sj_find_device(ctx.h, msg.data_ptr(), msg.numel(), tape.data_ptr(), tape.numel(), strs.data_ptr(), strs.numel(),
                              cp, 1, C.byref(fo_), C.byref(r), C.byref(b))
        assert rc == _lib.ERR_ARGUMENT, k
        rc = L.sj_parse_find(ctx.h, nd, len(nd), 1, cp, 1, None, C.byref(r), C.byref(b))
        assert rc == _lib.ERR_ARGUMENT, k
    cp, keep2 = sj._find_paths([[b"labels"]], [6])
    rc = L.sj_find_lists_device(*args[:-2], cp, 1, None, None, C.byref(r), C.byref(b), C.byref(e))
    assert rc == _lib.ERR_ARGUMENT
    # STRING_CVT goes through the old entry point
    cp, keep2 = sj._find_paths([[b"name"]], [fl.STRING_CVT])
    rc = L.sj_find_device(ctx.h, msg.data_ptr(), msg.numel(), tape.data_ptr(), tape.numel(), strs.data_ptr(), strs.numel(),
                          cp, 1, None, C.byref(r), C.byref(b))
    assert rc == _lib.ERR_CAPACITY and r.value == rows
    # no rows: every list offsets column is its one 0
    rc, rows0, cols0 = ctx.find_device(_dev(np.array([word("N", 0)], dtype=np.uint64), np.int64), None, None, paths, kinds)
    assert rc == 0 and rows0 == 0 and [int(c.list_offsets[0]) for c in (cols0[0], cols0[2])] == [0, 0]


def test_one_array_of_half_a_gib(ctx):
    """{"a":[...]} of 0.5 GiB, about 4.5e7 numbers k / 4 from a numpy seed: AsFloat equals the generator's float64 bits
    (every k / 4 below 2^24 is exact in decimal and in binary)"""
    rng = np.random.default_rng(2024)
    x = rng.integers(0, 1 << 26, 45_000_000) / 4.0
    doc = b'{"a":[' + ",".join(map(repr, x.tolist())).encode() + b"]}"
    assert len(doc) > 400 << 20
    rc, rows, (col,) = ctx.parse_find(doc, [[b"a"]], [fl.ARRAY_FLOAT64], ndjson=False)
    assert rc == 0 and rows == 1 and int(col.status[0]) == fo.OK and int(col.value[0]) == x.size
    assert np.array_equal(col.elems.view(np.uint64), x.view(np.uint64))
