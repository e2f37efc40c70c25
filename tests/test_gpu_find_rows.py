"""GPU tests of the find's array rows (sj_find_rows_device / sj_parse_find_rows, find_rows.cuh): device against the
Python port (tests/find_rows_oracle.py) record for record and cell for cell -- RowIndex (record statuses and offsets,
row tags and head indexes) and every column -- on fixtures as documents and as NDJSON, fuzz seeds, the tricky records,
the context's own tape against the same tape passed as foreign, builder tapes with nops, failing links and unknown tags
among the elements, a Deserialize'd tape, element heads and stops around tile edges, arrays of 0, 1 and 2 elements
beside one of more than 2^24 objects, a 0.5 GiB document against its generator, and the capacity and argument
contract with the launch count of one configuration."""
import ctypes as C
import json

import numpy as np
import pytest

from tests import find_json_oracle as fj
from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import find_rows_oracle as fr
from tests.tape_builder import word
from tests.test_find_json_cpu import harvest
from tests.test_find_lists_cpu import NDJSON_FIXTURES, _arr, _obj, ndjson_records
from tests.test_find_rows_cpu import DOC_ROWS, ND_ROWS
from tests.test_gpu_find_lists import _dev, _np, check
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu
S = 1 << 55
ALL = [fo.ELEMENT, fo.INT64, fo.UINT64, fo.FLOAT64, fo.BOOL, fo.STRING, fj.JSON] + list(fl.LIST_KINDS) + [fl.STRING_CVT]


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def want(tape, strs, msg, row_path, paths, kinds, records=None):
    """(rec_status, rec_offsets, row_tag, row_index, cells in check()'s form) from the port"""
    st, offs, tags, idx, cells = fr.find_rows(tape, strs, msg, row_path, paths, kinds, records)
    return st, offs, tags, idx, [[(s, t, i, v, e, b) for s, t, i, v, e, b in col] for col in cells]


def check_rows(res, w, kinds, what):
    rc, n_rec, n_rows, index, cols = res
    st, offs, tags, idx, cells = w
    assert rc == 0, (what, rc)
    assert (n_rec, n_rows) == (len(st), len(idx)), (what, n_rec, n_rows, len(st), len(idx))
    assert _np(index.rec_status).tolist() == st, what
    assert _np(index.rec_offsets).tolist() == offs, what
    assert _np(index.row_tag).tolist() == tags, what
    assert _np(index.row_index).tolist() == idx, what
    check(cols, n_rows, cells, kinds, what)


def foreign(ctx, tape, strs, msg, row_path, paths, kinds, what, records=None):
    res = ctx.find_rows_device(_dev(tape, np.int64), _dev(strs), _dev(msg), row_path, paths, kinds)
    check_rows(res, want(tape, strs, msg, row_path, paths, kinds, records), kinds, what)
    return res


def _row_path(name, doc):
    for n, p in DOC_ROWS:
        if n == name:
            return p
    v = json.loads(doc)
    if isinstance(v, dict):
        for k, x in v.items():
            if isinstance(x, list):
                return [k.encode()]
    return []


def _sub(doc, row_path, n=6):
    """sub-paths of the row path's first elements, and two that are nowhere"""
    v = json.loads(doc)
    for k in row_path:
        v = v.get(k.decode(), []) if isinstance(v, dict) else []
    seen, out = set(), []
    for e in (v if isinstance(v, list) else [])[:10]:
        for p in harvest(json.dumps(e).encode(), 20)[:-3]:
            if tuple(p) not in seen:
                seen.add(tuple(p))
                out.append(p)
    return out[:n] + [[b"\x00missing"], []]


def _per_kind(paths):
    ps, ks = [p for p in paths for _ in ALL], [k for _ in paths for k in ALL]
    return [(ps[i:i + 60], ks[i:i + 60]) for i in range(0, len(ps), 60)]


@pytest.mark.parametrize("name", TAPE_FILES + SMALL_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures(ctx, oracle_native, name, copy):
    """sj_parse_find_rows on the own tape, and the oracle's tape as a foreign one, under every kind"""
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc, copy_strings=copy)
    assert rc == 0
    msg = doc[off:off + ln]
    rp = _row_path(name, doc)
    for paths, kinds in _per_kind(_sub(doc, rp, 4 if name in ("random", "apache_builds", "citm_catalog") else 6)):
        w = want(tape, strs, msg, rp, paths, kinds)
        check_rows(ctx.parse_find_rows(doc, rp, paths, kinds, ndjson=False, copy_strings=copy), w, kinds, (name, "own"))
        assert ctx.find_rows_serial() == 0, name  # every record of a parser's tape passes propose / verify
        res = ctx.find_rows_device(_dev(tape, np.int64), _dev(strs), _dev(msg), rp, paths, kinds)
        check_rows(res, w, kinds, (name, "foreign"))
        assert ctx.find_rows_serial() == 0, name


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
def test_ndjson_nested_rows(ctx, oracle, name):
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True)
    assert rc == 0
    rp = ND_ROWS[name]
    elems = [e for r in recs for e in (r.get(rp[0].decode(), {}) or {}).get(rp[1].decode(), [])] if len(rp) == 2 else \
        [e for r in recs for e in (r.get(rp[0].decode()) or [])]
    paths = []
    for e in elems[:10]:
        for p in harvest(json.dumps(e).encode(), 10)[:-3]:
            if p not in paths:
                paths.append(p)
    paths = paths[:5] + [[b"nope"]]
    kinds = [ALL[i % len(ALL)] for i in range(len(paths))]
    w = want(tape, strs, nd[off:off + ln], rp, paths, kinds)
    assert len(w[3]) > 0
    check_rows(ctx.parse_find_rows(nd, rp, paths, kinds), w, kinds, name)


def test_fuzz_seeds_and_tricky(ctx, oracle):
    n = 0
    docs = [(nm, d) for nm, d in fuzz_corpus("corpus", max_size=1 << 14)] + [("tricky", tricky_ndjson()[0])]
    for name, data in docs:
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson)
            if rc:
                continue
            keys = harvest(data, 6)[:-3]
            for rp in ([], keys[0] if keys else [b"a"]):
                paths = harvest(data, 12)
                kinds = [ALL[i % len(ALL)] for i in range(len(paths))]
                w = want(tape, strs, data[off:off + ln], rp, paths, kinds)
                check_rows(ctx.parse_find_rows(data, rp, paths, kinds, ndjson=ndjson), w, kinds, (name, ndjson, rp))
                n += 1
    assert n > 40


def test_own_tape_equals_foreign_and_parse(ctx):
    """the same output for the context's own tape (stage 2's root list) and a copy passed as foreign, and from
    sj_parse_find_rows; the launch count of this configuration is pinned"""
    import torch
    doc = load_fixture("twitter")
    L = ctx.L
    d_msg = torch.full((len(doc) + 4096,), 0x20, dtype=torch.uint8, device="cuda")
    d_msg[:len(doc)].copy_(torch.frombuffer(bytearray(doc), dtype=torch.uint8))
    tcap, scap = C.c_size_t(0), C.c_size_t(0)
    L.sj_bounds(len(doc), C.byref(tcap), C.byref(scap))
    d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    assert L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(doc), 2, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                             d_str.data_ptr(), d_str.numel(), C.byref(sl)) == 0
    tape, strs, msg = d_tape[:tl.value], d_str[:sl.value], d_msg[:len(doc)]
    paths, kinds = [[b"user", b"screen_name"], [b"retweet_count"], [b"id"]], [fo.STRING, fo.INT64, fo.UINT64]
    l0 = ctx.launches()
    own = ctx.find_rows_device(tape, strs, msg, [b"statuses"], paths, kinds)
    l1 = ctx.launches()
    fgn = ctx.find_rows_device(tape.clone(), strs, msg, [b"statuses"], paths, kinds)
    l2 = ctx.launches()
    # two calls each (sizes, then the columns): KR1 .. KR7 (20) and KF3, KF4 + 2 scans (4); the second adds KR8 and KF5;
    # a foreign tape adds KM1, KC1a, KC1b and their scans (7) to each
    assert (l1 - l0, l2 - l1) == (24 + 26, (7 + 24) + (7 + 26))
    assert own[:3] == fgn[:3] == (0, 1, 100)
    for a, b in zip(list(own[3]) + [x for c in own[4] for x in c], list(fgn[3]) + [x for c in fgn[4] for x in c]):
        assert (a is None and b is None) or torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
    t = tape.cpu().numpy().view(np.uint64)
    w = want(t, strs.cpu().numpy().tobytes(), doc, [b"statuses"], paths, kinds)
    check_rows(own, w, kinds, "own")
    check_rows(ctx.parse_find_rows(doc, [b"statuses"], paths, kinds, ndjson=False), w, kinds, "parse")


def _tape_of(records):
    """r { "a": [ items ] } r per record, laid end to end, links moved to each record's place"""
    words, at = [], 0
    for items in records:
        for w in _obj(_arr(items)):
            t = w >> 56
            if t in b"r{[}]":
                w += at
            words.append(w)
        at = len(words)
    return np.array(words, dtype=np.uint64)


QUIRKS = [[word("l"), 1, word("N", 1), word("x"), word("l"), 2],
          [word("N", 2), word("N", 1), word("t"), word("l"), 3],
          [word("l"), 1, word("N", 10)],
          [word("t"), word("{", 3), word("}", 6)],
          [word("t"), word("r", 8), word("t"), word("x"), word("t")],
          [word("[", 7), word("]", 5), word("l"), 3],
          [],
          [word("{", 11), word('"', S), 1, word("l"), 7, word("}", 5), word("{", 17), word('"', S | 1), 1, word("l"), 1,
           word("}", 11)],
          [word("t"), word("{", 9), word("}", 6), word("t")],  # a link past the next candidate: verification fails
          [word("]", 4), word("t")]]


def test_foreign_quirk_tapes(ctx):
    """the builder tapes of tests/test_find_rows_cpu.py as records of one foreign tape: nops among the elements (the
    record walked by one thread), links that fail verification, unknown tags, nested arrays, empty arrays"""
    import simdjson_b200 as sj
    tape = _tape_of(QUIRKS)
    strs = b"abcdefgh"
    recs = fo.roots(tape)  # (the 'r' among the elements is a root open too: one record more)
    paths, kinds = [[b"a"], [b"a"], [b"a"], []], [fo.INT64, fj.JSON, fl.ARRAY_INT64, fo.ELEMENT]
    foreign(ctx, tape, strs, b"", [b"a"], paths, kinds, "quirks", recs)
    assert ctx.find_rows_serial() >= 4  # the nop records, the 'r' record and the link past the next candidate
    doc = load_fixture("github_events")
    back = sj.Serializer(ctx).Deserialize(sj.Serializer(ctx).Serialize(sj.Parse(doc, ctx=ctx)))
    t, s, m = np.asarray(back.Tape, dtype=np.uint64), bytes(back.Strings), bytes(back.Message)
    foreign(ctx, t, s, m, [], [[b"type"], [b"payload"], [b"actor", b"login"]], [fo.STRING, fj.JSON, fl.STRING_CVT], "deserialize")


def test_heads_and_stops_around_tile_edges(ctx, oracle):
    """element heads, scope links, stop words and array ends at every offset around the 4 096-word tiles of the
    array words: records of arrays whose element sizes shift by one word each"""
    rng = np.random.default_rng(5)
    items = [b'{"k":%d}', b'"s%d"', b"[%d]", b"%d.5", b"true", b"{}", b'{"k":{"k":%d}}']
    recs = []
    words = 0
    while words < 3 * 4096 + 500:
        n = int(rng.integers(0, 40))
        els = [items[int(rng.integers(0, len(items)))].replace(b"%d", str(int(rng.integers(0, 99))).encode()) for _ in range(n)]
        recs.append(b'{"p":' + [b"1", b"true", b"null"][int(rng.integers(0, 3))] + b',"a":[' + b",".join(els) + b"]}")
        words += 8 + 3 * n
    nd = b"\n".join(recs)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True)
    assert rc == 0 and len(tape) > 3 * 4096
    paths, kinds = [[b"k"], [b"k"], [b"k", b"k"]], [fo.INT64, fj.JSON, fo.ELEMENT]
    w = want(tape, strs, nd[off:off + ln], [b"a"], paths, kinds)
    check_rows(ctx.parse_find_rows(nd, [b"a"], paths, kinds), w, kinds, "tiles")
    # the same tape with the records shifted by 0 .. 4 leading nops, so every head meets every tile offset
    for shift in range(1, 5):
        t = np.concatenate([np.array([word("N", 1)] * shift, dtype=np.uint64), tape])
        tags = t >> np.uint64(56)
        link = np.isin(tags, [ord(c) for c in "r{[}]"]) & np.r_[np.zeros(shift, bool), _heads(tape)]
        t[link] += np.uint64(shift)
        foreign(ctx, t, strs, nd[off:off + ln], [b"a"], paths, kinds, ("shift", shift), fo.roots(t))


def _heads(tape):
    tags = (np.asarray(tape, dtype=np.uint64) >> np.uint64(56)).astype(np.int64)
    value = np.isin(tags, [ord(c) for c in '"lud'])
    head = np.ones(len(tags), bool)
    h = True
    for i, v in enumerate(value.tolist()):
        head[i] = h
        h = not (h and v)
    return head


def test_small_arrays_beside_a_huge_one(ctx):
    """root arrays of 0, 1 and 2 objects before and after one of 2^24 + 3 objects (a record covering more than 1 024
    tiles of array words), row path []: every row's head index from the generator"""
    big = (1 << 24) + 3
    recs = [b"[]", b"[{}]", b"[{},{}]", b"[" + b",".join([b"{}"] * big) + b"]", b"[]", b"[{}]", b"[{},{}]"]
    counts = [0, 1, 2, big, 0, 1, 2]
    rc, n_rec, n_rows, index, cols = ctx.parse_find_rows(b"\n".join(recs), [], [[b"a"]], [fo.INT64])
    assert rc == 0 and n_rec == 7 and n_rows == sum(counts)
    offs = _np(index.rec_offsets)
    assert offs.tolist() == np.concatenate([[0], np.cumsum(counts)]).tolist()
    idx = _np(index.row_index)
    at = 0  # each record: r [ {} ... ] r, an empty object being 2 words
    for k, n in enumerate(counts):
        got = idx[offs[k]:offs[k + 1]]
        assert np.array_equal(got, at + 2 + 2 * np.arange(n)), k
        at += 4 + 2 * n
    assert (_np(index.row_tag) == ord("{")).all()
    assert (_np(cols[0].status) == fo.NOT_FOUND).all()
    assert ctx.find_rows_serial() == 0


def test_array_links_at_or_behind_the_head(ctx):
    """an array whose link lies at or behind its '[' (a malformed foreign tape): reached by elem.Array (a row path of 0
    segments), Iter.Array's Tape[:end] ends before the Array's off, so ForEach's first Advance ends the walk -- an OK
    record with no rows, beside records that have rows"""
    words, at = [], 0
    for inner in ([word("t")], "at", [word("l"), 3], "behind", [word("f"), word("n")]):
        if isinstance(inner, str):
            arr = [word("[", 4 if inner == "at" else 2), word("t"), word("]", 4)]
        else:
            arr = _arr(inner)
        rec = _obj(arr)
        words += [w + at if (w >> 56) in b"r{[}]" else w for w in rec]
        at = len(words)
    # root arrays (row path []): a link at the '[' and one behind it, between two good ones
    for link in (None, 0, -1, None):
        n = at
        if link is None:
            words += [word("r", n + 5), word("[", n + 4), word("t"), word("]", n + 1), word("r", n)]
        else:
            words += [word("r", n + 5), word("[", n + 1 + link), word("t"), word("]", n + 1), word("r", n)]
        at = len(words)
    tape = np.array(words, dtype=np.uint64)
    for rp in ([b"a"], []):
        res = foreign(ctx, tape, b"abcdefgh", b"", rp, [[b"a"], []], [fo.INT64, fo.ELEMENT], ("links", rp), fo.roots(tape))
        st = _np(res[3].rec_status).tolist()
        # through a key path FindPath's AdvanceIter meets the link first: "element has negative offset" (CORRUPT);
        # elem.Array of a root array checks no link behind the '[' (AdvanceInto does not), so those records are OK
        want_st = [fo.OK, fo.CORRUPT, fo.OK, fo.CORRUPT, fo.OK] if rp else [fo.OK] * 4
        assert (st[:5] if rp else st[-4:]) == want_st, (rp, st)


def test_empty_and_rootless_tapes_ask_for_sizes(ctx):
    """NULL outputs on a tape of 0 words and on a foreign tape without roots: SJ_OK with no records and no rows"""
    import simdjson_b200 as sj
    cp, _k = sj._find_paths([[b"a"]], [fo.INT64])
    rp, _r = sj._find_paths([[b"a"]], [fo.ELEMENT])
    n = [C.c_size_t(7) for _ in range(4)]
    assert ctx.L.sj_find_rows_device(ctx.h, None, 0, None, 0, None, 0, rp, cp, 1, None, None, None,
                                     *(C.byref(x) for x in n)) == 0
    assert [x.value for x in n] == [0, 0, 0, 0]
    t = _dev(np.array([word("n"), word("t"), word("l"), 5], dtype=np.uint64), np.int64)
    n = [C.c_size_t(7) for _ in range(4)]
    assert ctx.L.sj_find_rows_device(ctx.h, None, 0, t.data_ptr(), t.numel(), None, 0, rp, cp, 1, None, None, None,
                                     *(C.byref(x) for x in n)) == 0
    assert [x.value for x in n] == [0, 0, 0, 0]
    rc, N, R, index, cols = ctx.find_rows_device(t, None, None, [b"a"], [[b"a"]], [fo.INT64])
    assert (rc, N, R) == (0, 0, 0) and _np(index.rec_offsets).tolist() == [0]


def test_heads_and_stops_around_a_group_edge(ctx, oracle_native):
    """heterogeneous records whose heads, links, stops and array ends sit at -2 .. +2 (and around) of word 4 194 304
    of the array word space, the edge of the first group of 1 024 tiles: a filler record of numbers in front, shifted
    word by word by trailing `true`s"""
    rng = np.random.default_rng(11)
    items = [b'{"k":%d}', b'"s%d"', b"[%d]", b"%d.5", b"true", b"{}", b'{"k":{"k":%d}}', b"[]"]
    tail = []
    for _ in range(40):
        n = int(rng.integers(0, 6))
        els = [items[int(rng.integers(0, len(items)))].replace(b"%d", str(int(rng.integers(0, 99))).encode()) for _ in range(n)]
        tail.append(b'{"a":[' + b",".join(els) + b"]}")
    edge = 4096 * 1024
    paths, kinds = [[b"k"], [b"k"]], [fo.INT64, fj.JSON]
    for shift in range(5):
        nf = (edge - 60) // 2
        filler = b'{"a":[' + b",".join([b"1"] * nf + [b"true"] * shift) + b"]}"
        nd = b"\n".join([filler] + tail)
        rc, tape, strs, (off, ln) = oracle_native.parse(nd, ndjson=True)
        assert rc == 0
        roots = fo.foreach_roots(tape)
        rc, N, R, index, cols = ctx.parse_find_rows(nd, [b"a"], paths, kinds)
        assert rc == 0 and N == len(tail) + 1 and ctx.find_rows_serial() == 0
        n0 = nf + shift
        offs, idx = _np(index.rec_offsets), _np(index.row_index)
        assert offs[1] == n0 and np.array_equal(idx[:nf], 5 + 2 * np.arange(nf))
        st, woffs, tags, widx, cells = want(tape, strs, nd[off:off + ln], [b"a"], paths, kinds, roots[1:])
        assert _np(index.rec_status).tolist()[1:] == st, shift
        assert (offs[1:] - n0).tolist() == woffs and idx[n0:].tolist() == widx and _np(index.row_tag)[n0:].tolist() == tags
        for p, k in enumerate(kinds):
            c = cols[p]
            got = list(zip(_np(c.status)[n0:].tolist(), _np(c.tag)[n0:].tolist(), _np(c.index)[n0:].tolist(),
                           _np(c.value).view(np.uint64)[n0:].tolist()))
            assert got == [(s, t, i, v) for s, t, i, v, _, _ in cells[p]], (shift, p)
            if k == fj.JSON:
                o, d = _np(c.offsets), _np(c.data).tobytes()
                assert [d[o[r]:o[r + 1]] for r in range(n0, R)] == [b for *_, b in cells[p]], shift


def test_half_a_gib_document(ctx):
    """{"statuses": [twitter's statuses x k]} of 0.5 GiB: rows, ids and screen names against the generator"""
    v = json.loads(load_fixture("twitter"))
    body = b",".join(json.dumps(s).encode() for s in v["statuses"])
    k = (1 << 29) // len(body)
    doc = b'{"statuses":[' + b",".join([body] * k) + b"]}"
    paths, kinds = [[b"id"], [b"user", b"screen_name"]], [fo.UINT64, fo.STRING]
    rc, n_rec, n_rows, index, cols = ctx.parse_find_rows(doc, [b"statuses"], paths, kinds, ndjson=False)
    assert rc == 0 and (n_rec, n_rows) == (1, 100 * k)
    ids = np.array([s["id"] for s in v["statuses"]], dtype=np.uint64)
    assert np.array_equal(cols[0].value, np.tile(ids, k))
    names = [s["user"]["screen_name"].encode() for s in v["statuses"]]
    lens = np.tile(np.array([len(x) for x in names]), k)
    assert np.array_equal(np.diff(cols[1].offsets), lens)
    assert bytes(cols[1].data[:cols[1].offsets[100]]) == b"".join(names)
    assert ctx.find_rows_serial() == 0


def test_capacity_and_arguments(ctx):
    """sizes exact and nothing written on SJ_ERR_CAPACITY with each cap too small in turn; NULL outputs ask for the
    sizes; SJ_ERR_ARGUMENT for a row path kind other than ELEMENT, more than 32 segments, list paths without lists"""
    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    nd = b"\n".join([b'{"a":[{"s":"xy","n":[1,2]},{"s":"z"}]}', b'{"a":[]}', b'{"b":1}', b'{"a":[{"n":[3]}]}'])
    paths, kinds = [[b"s"], [b"n"]], [fo.STRING, fl.ARRAY_INT64]
    rc, tape, strs, (off, ln) = ctx.parse(nd, ndjson=True)
    assert rc == 0
    t, s, m = _dev(tape, np.int64), _dev(strs), _dev(nd[off:off + ln])
    assert ctx.find_rows_device(t, s, m, [b"a"], paths, kinds)[:3] == (0, 4, 3)
    full = _out_of(ctx, t, s, m, paths, kinds)
    sizes = (4, 3, 3, 3)  # records, rows, bytes, elements
    cpaths, _k = sj._find_paths(paths, kinds)
    rpath, _r = sj._find_paths([[b"a"]], [fo.ELEMENT])

    def call(rec_cap, row_cap, str_cap, elem_cap, lists=True):
        out = [torch.full_like(x, 0x5A) if x.dtype == torch.uint8 else torch.full_like(x, 0x5A5A) for x in full]
        o = _lib.FindOut(*(x.data_ptr() for x in out[:6]), row_cap, str_cap)
        lo = _lib.FindListsOut(out[6].data_ptr(), out[7].data_ptr(), elem_cap)
        ro = _lib.FindRowsOut(*(x.data_ptr() for x in out[8:12]), rec_cap)
        n = [C.c_size_t(0) for _ in range(4)]
        tp, sp, mp = t.data_ptr(), s.data_ptr(), m.data_ptr()
        rc = ctx.L.sj_find_rows_device(ctx.h, mp, m.numel(), tp, t.numel(), sp, s.numel(), rpath, cpaths, 2, C.byref(o),
                                       C.byref(lo) if lists else None, C.byref(ro), *(C.byref(x) for x in n))
        torch.cuda.synchronize()
        return rc, tuple(x.value for x in n), out
    for k in range(4):
        caps = list(sizes)
        caps[k] -= 1
        rc, got, out = call(*caps)
        assert rc == _lib.ERR_CAPACITY and got == sizes, k
        for x in out:
            assert (x.view(torch.uint8) == 0x5A).all() or (x == 0x5A5A).all(), k
    rc, got, out = call(*sizes)
    assert rc == 0 and got == sizes
    assert _np(out[9]).tolist() == [0, 2, 2, 2, 3] and _np(out[8]).tolist() == [fo.OK, fo.OK, fo.NOT_FOUND, fo.OK]
    n = [C.c_size_t(0) for _ in range(4)]
    assert ctx.L.sj_find_rows_device(ctx.h, m.data_ptr(), m.numel(), t.data_ptr(), t.numel(), s.data_ptr(), s.numel(), rpath,
                                     cpaths, 2, None, None, None, *(C.byref(x) for x in n)) == _lib.ERR_CAPACITY
    assert tuple(x.value for x in n) == sizes
    # arguments
    for bad_path, bad_kind in (([b"a"], fo.INT64), ([b"a"] * 33, fo.ELEMENT)):
        rp, _r2 = sj._find_paths([bad_path], [bad_kind])
        assert ctx.L.sj_find_rows_device(ctx.h, m.data_ptr(), m.numel(), t.data_ptr(), t.numel(), s.data_ptr(), s.numel(), rp,
                                         cpaths, 2, None, None, None, *(C.byref(x) for x in n)) == _lib.ERR_ARGUMENT
    # a list path that finds nothing has no elements: without `lists` that is SJ_ERR_ARGUMENT, not a capacity
    lp, _l = sj._find_paths([[b"nope"]], [fl.ARRAY_INT64])
    o = _lib.FindOut(*(x.data_ptr() for x in full[:6]), 4, 3)
    ro = _lib.FindRowsOut(*(x.data_ptr() for x in full[8:12]), 4)
    assert ctx.L.sj_find_rows_device(ctx.h, m.data_ptr(), m.numel(), t.data_ptr(), t.numel(), s.data_ptr(), s.numel(), rpath,
                                     lp, 1, C.byref(o), None, C.byref(ro), *(C.byref(x) for x in n)) == _lib.ERR_ARGUMENT


def _out_of(ctx, t, s, m, paths, kinds):
    """the 12 output tensors of find_rows_device at the exact sizes"""
    import torch
    rc, N, R, index, cols = ctx.find_rows_device(t, s, m, [b"a"], paths, kinds)
    assert rc == 0
    u8, i64 = torch.uint8, torch.int64
    nb = int(cols[0].offsets[-1]) if cols[0].offsets is not None else 0
    ne = int(cols[1].list_offsets[-1])
    return (torch.empty((2, R), dtype=u8, device="cuda"), torch.empty((2, R), dtype=u8, device="cuda"),
            torch.empty((2, R), dtype=i64, device="cuda"), torch.empty((2, R), dtype=i64, device="cuda"),
            torch.empty((1, R + 1), dtype=i64, device="cuda"), torch.empty(nb, dtype=u8, device="cuda"),
            torch.empty((1, R + 1), dtype=i64, device="cuda"), torch.empty(ne, dtype=i64, device="cuda"),
            torch.empty(N, dtype=u8, device="cuda"), torch.empty(N + 1, dtype=i64, device="cuda"),
            torch.empty(R, dtype=u8, device="cuda"), torch.empty(R, dtype=i64, device="cuda"))
