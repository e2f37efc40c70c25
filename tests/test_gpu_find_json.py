"""GPU tests of the find's JSON cells (SJ_FIND_KIND_JSON, find_json.cuh): device against the Python port
(tests/find_json_oracle.py) cell for cell -- text, offsets, status, tag, index and length -- on fixtures, fuzz seeds, the
tricky records and foreign tapes; mixed STRING + JSON path sets; the capacity contract and the kind 7 / kind 6 split;
builder tapes that put cell starts, ends and long strings on the segmented passes' tile (4 096 virtual words) and group
(1 024 tiles) edges; a malformed region beside well-formed cells at scale; and two checks at 0.5 GiB."""
import ctypes as C
import json

import numpy as np
import pytest

from tests import find_json_oracle as fj
from tests import find_oracle as fo
from tests.tape_builder import TapeBuilder, word
from tests.test_find_json_cpu import harvest
from tests.util import TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu
TILE, GROUP = 4096, 4096 * 1024


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


def _check(cols, rows, want, kinds, what):
    """every cell; the STRING and JSON columns' offsets are checked to be contiguous across columns"""
    assert all(len(w) == rows for w in want), what
    at = 0
    for p, k in enumerate(kinds):
        c = cols[p]
        st, tag, idx, val = _np(c.status), _np(c.tag), _np(c.index), _np(c.value).view(np.uint64)
        var = k in (fo.STRING, fj.JSON)
        if var:
            off, data = _np(c.offsets), _np(c.data).tobytes()
            assert int(off[0]) == at, (what, p)
            at = int(off[rows])
        for r, w in enumerate(want[p]):
            got = (int(st[r]), int(tag[r]), int(idx[r]))
            assert got == (w.status, w.tag, w.index), (what, p, r, got, w)
            if var:
                assert data[off[r]:off[r + 1]] == w.value, (what, p, r, data[off[r]:off[r + 1]][:200], w.value[:200])
                assert int(val[r]) == len(w.value), (what, p, r)
            else:
                assert int(val[r]) == w.value, (what, p, r)


def _foreign(ctx, tape, strs, msg, paths, kinds, what, rows=None):
    rc, n, cols = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), paths, kinds)
    assert rc == 0, (what, rc)
    want = fj.find_json(tape, strs, msg, paths, kinds, rows)
    _check(cols, n, want, kinds, what)


def _kinds(n):
    return [fj.JSON if i % 3 else fo.STRING for i in range(n)]


@pytest.mark.parametrize("name", TAPE_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures(ctx, oracle_native, name, copy):
    """own tape (sj_parse_find) and the oracle's tape as a foreign one, JSON paths mixed with STRING paths"""
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc, copy_strings=copy)
    assert rc == 0
    msg = doc[off:off + ln]
    paths = harvest(doc, 60)
    for kinds in ([fj.JSON] * len(paths), _kinds(len(paths))):
        want = fj.find_json(tape, strs, msg, paths, kinds, fo.foreach_roots(tape))
        rc, rows, cols = ctx.parse_find(doc, paths, kinds, ndjson=False, copy_strings=copy)
        assert rc == 0
        _check(cols, rows, want, kinds, name)
        _foreign(ctx, tape, strs, msg, paths, kinds, name)


def test_tricky_ndjson(ctx, oracle):
    nd, recs = tricky_ndjson()
    paths = [[b"Make"], [b"a"], [b"a", b"Make"], [b"Make", b"Make"], [b""], [b"t"], [b"f"], [b"n"], [b"d"], [b"l"],
             [b"u"], [b"x"], [b"nope"], []]
    for copy in (True, False):
        rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
        for kinds in ([fj.JSON] * len(paths), _kinds(len(paths))):
            rc, rows, cols = ctx.parse_find(nd, paths, kinds, copy_strings=copy)
            assert rc == 0 and rows == len(recs)
            _check(cols, rows, fj.find_json(tape, strs, nd[off:off + ln], paths, kinds, fo.foreach_roots(tape)), kinds, "tricky")


def test_fuzz_seeds(ctx, oracle):
    n = 0
    for name, data in fuzz_corpus("corpus", max_size=1 << 14):
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson)
            if rc:
                continue
            paths = harvest(data, 20)
            kinds = _kinds(len(paths))
            rc, rows, cols = ctx.parse_find(data, paths, kinds, ndjson=ndjson)
            assert rc == 0, name
            _check(cols, rows, fj.find_json(tape, strs, data[off:off + ln], paths, kinds, fo.foreach_roots(tape)), kinds, name)
            n += 1
    assert n > 20


def test_deserialize_output_is_a_foreign_tape(ctx, oracle):
    """Deserialize's tape (with its own Strings.B and message) through sj_find_device"""
    import simdjson_b200 as sj
    doc = load_fixture("citm_catalog")
    pj = sj.Parse(doc, ctx=ctx)
    back = sj.Serializer(ctx).Deserialize(sj.Serializer(ctx).Serialize(pj))
    tape, strs, msg = (np.asarray(back.Tape, dtype=np.uint64), bytes(back.Strings), bytes(back.Message))
    paths = harvest(doc, 40)
    _foreign(ctx, tape, strs, msg, paths, [fj.JSON] * len(paths), "deserialize")


def test_own_tape_equals_foreign(ctx):
    nd, recs = tricky_ndjson()
    paths = [[b"a"], [b"Make"], [b"t"]]
    kinds = [fj.JSON, fo.STRING, fj.JSON]
    rc, rows, own = ctx.parse_find(nd, paths, kinds)
    pj = __import__("simdjson_b200").ParseND(nd, ctx=ctx)
    rc2, rows2, cols = ctx.find_device(_dev(np.asarray(pj.Tape, dtype=np.uint64), np.int64), _dev(bytes(pj.Strings)),
                                       _dev(bytes(pj.Message)), paths, kinds)
    assert rc == rc2 == 0 and rows == rows2
    for a, b in zip(own, cols):
        for x, y in zip(a[:5], b[:5]):
            assert x is y is None or np.array_equal(_np(x), _np(y))
        if a.offsets is not None:
            end = int(_np(a.offsets)[rows])
            assert _np(a.data)[:end].tobytes() == _np(b.data)[:end].tobytes()


def test_no_rows_still_writes_the_first_offset(ctx):
    import torch
    tape = np.array([word("N", 0)], dtype=np.uint64)  # no root
    out = (torch.zeros((2, 4), dtype=torch.uint8, device="cuda"), torch.zeros((2, 4), dtype=torch.uint8, device="cuda"),
           torch.zeros((2, 4), dtype=torch.int64, device="cuda"), torch.zeros((2, 4), dtype=torch.int64, device="cuda"),
           torch.full((2, 5), 7, dtype=torch.int64, device="cuda"), torch.zeros(4, dtype=torch.uint8, device="cuda"))
    rc, rows, cols = ctx.find_device(_dev(tape, np.int64), None, None, [[b"a"], [b"b"]], [fj.JSON, fo.STRING], out)
    assert rc == 0 and rows == 0
    o = out[4].cpu().numpy()
    assert o[0, 0] == 0 and o[1, 0] == 0 and (o[:, 1:] == 7).all()


def test_capacity_and_kind_split(ctx):
    """sizes exact on SJ_ERR_CAPACITY and nothing written; kind 7 is JSON, kind 6 is refused"""
    import torch
    import simdjson_b200 as sj
    doc = b'{"a":{"b":[1,2.5,"x\\u0001"]},"s":"str"}\n{"a":true}'
    pj = sj.ParseND(doc, ctx=ctx)
    t, s, m = _dev(np.asarray(pj.Tape, dtype=np.uint64), np.int64), _dev(bytes(pj.Strings)), _dev(bytes(pj.Message))
    paths, kinds = [[b"a"], [b"s"]], [fj.JSON, fo.STRING]
    rc, rows, cols = ctx.find_device(t, s, m, paths, kinds)
    assert rc == 0 and rows == 2
    data = _np(cols[0].data).tobytes()
    off = _np(cols[0].offsets)
    assert data[off[0]:off[1]] == b'{"b":[1,2.5,"x\\u0001"]}' and data[off[1]:off[2]] == b"true"
    total = int(_np(cols[1].offsets)[2])
    small = (torch.zeros((2, 2), dtype=torch.uint8, device="cuda"), torch.zeros((2, 2), dtype=torch.uint8, device="cuda"),
             torch.zeros((2, 2), dtype=torch.int64, device="cuda"), torch.zeros((2, 2), dtype=torch.int64, device="cuda"),
             torch.full((2, 3), 9, dtype=torch.int64, device="cuda"), torch.full((total - 1,), 9, dtype=torch.uint8, device="cuda"))
    rc, rows, _ = ctx.find_device(t, s, m, paths, kinds, small)
    assert rc == sj.ERR_CAPACITY and rows == 2
    assert (small[4].cpu().numpy() == 9).all() and (small[5].cpu().numpy() == 9).all()
    cpaths, keep = sj._find_paths([[b"a"]], [6])
    r, b = C.c_size_t(0), C.c_size_t(0)
    assert ctx.L.sj_find_device(ctx.h, None, 0, t.data_ptr(), t.numel(), None, 0, cpaths, 1, None, C.byref(r), C.byref(b)) == sj._lib.ERR_ARGUMENT
    cpaths, keep = sj._find_paths([[b"a"]], [7])
    assert ctx.L.sj_find_device(ctx.h, m.data_ptr(), m.numel(), t.data_ptr(), t.numel(), s.data_ptr(), s.numel(), cpaths, 1,
                                None, C.byref(r), C.byref(b)) == sj.ERR_CAPACITY  # (no out: the sizes only)
    assert b.value == len(b'{"b":[1,2.5,"x\\u0001"]}') + 4


# ---- builder tapes on the segmented passes' edges ------------------------------------------------------------------

def _rows_of_cells(sizes, long_at=(), bad=()):
    """one root per size: {"a": [<size - 2 words>]}, the array's words `t`, with a long string (40 bytes with escapes)
    where long_at names (row, word in the cell) and a malformed word where bad names it.  Returns (tape, strs, msg)."""
    b = TapeBuilder()
    for r, size in enumerate(sizes):
        b.open("r"); b.open("{"); b.string(b"a")
        if size == 1:
            b.atom("t")
        else:
            b.open("[")
            k = 1
            while k < size - 1:
                if (r, k) in long_at and k + 2 <= size - 1:
                    b.string(b'"q\\' * 13 + b"z")
                    k += 2
                else:
                    b.atom("t")
                    k += 1
            b.close()
        b.close(); b.close()
    tape, strs, msg = b.build()
    tape = tape.copy()
    for i in bad:
        tape[i] = word("x")
    return tape, strs, msg


def _cell_heads(tape):
    return [int(r) + 4 for r in fo.roots(tape)]


def test_cell_edges_on_tiles_and_a_group(ctx):
    """cells of 1, 2, 3 and many words whose starts and ends fall at E-2 .. E+1 of tile and group edges of the virtual
    word space, long strings across those edges, and one cell longer than a group"""
    sizes = []
    v = 0
    for e in (TILE, 2 * TILE, 3 * TILE, GROUP, GROUP + TILE):
        for target in (e - 2, e - 1, e, e + 1):
            if target > v:
                sizes.append(target - v)
                v = target
    sizes += [1, 2, 3, 2, 1] * 40 + [GROUP + 5, 7]
    long_at = {(r, k) for r, s in enumerate(sizes) for k in (1, s - 3, s // 2) if s > 6}
    tape, strs, msg = _rows_of_cells(sizes, long_at)
    _foreign(ctx, tape, strs, msg, [[b"a"], [b"b"]], [fj.JSON, fj.JSON], "edges")


def test_millions_of_small_cells(ctx):
    sizes = ([1, 2] * (1 << 20))[: 1 << 21]
    tape, strs, msg = _rows_of_cells(sizes)
    rc, rows, cols = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), [[b"a"]], [fj.JSON])
    assert rc == 0 and rows == len(sizes)
    off, data = _np(cols[0].offsets), _np(cols[0].data).tobytes()
    assert (_np(cols[0].status) == fo.OK).all()
    want = [b"true", b"[]"]
    assert np.array_equal(np.diff(off), np.array([len(want[s - 1]) for s in sizes]))
    assert data == b"".join(want[s - 1] for s in sizes)


def test_deep_nesting(ctx):
    """nesting deep enough for several levels of the parents' min hierarchy"""
    b = TapeBuilder()
    b.open("r"); b.open("{"); b.string(b"a")
    b.nest("[", 40000)
    b.atom("n")
    b.close(40000)
    b.string(b"b"); b.nest("{", 3000, key=b"k"); b.string(b"k"); b.atom("t"); b.close(3000)
    b.close(); b.close()
    tape, strs, msg = b.build()
    _foreign(ctx, tape, strs, msg, [[b"a"], [b"b"]], [fj.JSON, fj.JSON], "deep")


def test_malformed_elsewhere_at_scale(ctx):
    """malformed words inside some cells and outside all of them: the other cells keep their text"""
    sizes = [3, 5000, 2, GROUP // 3, 9, 4096, 1] * 6
    tape, strs, msg = _rows_of_cells(sizes)
    heads = _cell_heads(tape)
    bad = [heads[1] + 7, heads[8] + 100, heads[20] + 1, heads[30] - 2, heads[31] - 4]  # inside cells, and the key words
    tape, strs, msg = _rows_of_cells(sizes, bad=bad)
    _foreign(ctx, tape, strs, msg, [[b"a"]], [fj.JSON], "malformed elsewhere", fo.roots(tape))


# ---- 0.5 GiB ----------------------------------------------------------------------------------------------------

def test_one_cell_of_half_a_gib(ctx):
    """(a) {"a": [twitter.json x K]}: the one cell of ["a"] is sj_marshal_device's text of the same tape without its
    first 5 bytes and its last byte"""
    import torch
    tw = load_fixture("twitter").strip()
    k = (512 << 20) // len(tw)
    doc = b'{"a":[' + b",".join([tw] * k) + b"]}"
    from simdjson_b200 import _lib
    d_msg = torch.from_numpy(np.frombuffer(doc + b" " * 64, dtype=np.uint8).copy()).cuda()
    tcap, scap, tl, sl = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    ctx.L.sj_bounds(len(doc), C.byref(tcap), C.byref(scap))
    d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
    assert ctx.L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(doc), _lib.FLAG_COPY_STRINGS, d_tape.data_ptr(), d_tape.numel(),
                                 C.byref(tl), d_str.data_ptr(), d_str.numel(), C.byref(sl)) == 0
    tape, strs = d_tape[:tl.value], d_str[:sl.value]
    rc, rows, cols = ctx.find_device(tape, strs, d_msg, [[b"a"]], [fj.JSON])
    assert rc == 0 and rows == 1 and int(_np(cols[0].status)[0]) == fo.OK
    rc, _, text = ctx.marshal_device(tape, strs, d_msg)
    assert rc == 0
    n = int(_np(cols[0].offsets)[1])
    assert n == text.numel() - 6
    assert torch.equal(cols[0].data[:n], text[5:-1])


def test_twitter_statuses_half_a_gib(ctx, oracle):
    """(b) NDJSON of twitter.json's statuses, one per line, repeated to about 512 MiB: the user / entities / id cells of
    row g are the port's cells of template line g mod K"""
    tw = json.loads(load_fixture("twitter"))
    lines = [json.dumps(s, ensure_ascii=False, separators=(",", ":")).encode() for s in tw["statuses"]]
    block = b"\n".join(lines)
    reps = (512 << 20) // (len(block) + 1)
    nd = b"\n".join([block] * reps)
    paths, kinds = [[b"user"], [b"entities"], [b"id"]], [fj.JSON, fj.JSON, fj.JSON]
    rc, tape, strs, (off, ln) = oracle.parse(block, ndjson=True)
    want = fj.find_json(tape, strs, block[off:off + ln], paths, kinds, fo.foreach_roots(tape))
    rc, rows, cols = ctx.parse_find(nd, paths, kinds)
    assert rc == 0 and rows == len(lines) * reps
    K = len(lines)
    for p in range(3):
        off, data = cols[p].offsets, cols[p].data
        assert (cols[p].status == fo.OK).all()
        texts = [w.value for w in want[p]]
        lens = np.tile(np.array([len(t) for t in texts]), reps)
        assert np.array_equal(np.diff(off), lens)
        assert data[off[0]:off[rows]].tobytes() == b"".join(texts) * reps
