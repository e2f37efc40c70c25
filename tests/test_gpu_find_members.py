"""GPU tests of the find's member rows (sj_find_members_device / sj_parse_find_members, find_rows.cuh): device against
the Python port (tests/find_members_oracle.py) record for record and cell for cell -- MemberIndex (record statuses and
offsets, value tags and heads, keys) and every column -- on map-like fixtures in both copy modes, NDJSON records
exploded with a row path of 0 segments, fuzz seeds, the own tape against a foreign copy and a Deserialize'd tape,
ForEach's quirk tapes, keys and values around the tile and first group edges, objects of 0, 1 and 2 members beside one
of 2^22 + 3, a 0.5 GiB document, empty and rootless tapes, and the capacity and argument contract with the launch count of one call."""
import ctypes as C
import json

import numpy as np
import pytest

from tests import find_json_oracle as fj
from tests import find_lists_oracle as fl
from tests import find_members_oracle as fm
from tests import find_oracle as fo
from tests.tape_builder import word
from tests.test_find_json_cpu import harvest
from tests.test_find_lists_cpu import NDJSON_FIXTURES, ndjson_records
from tests.test_find_members_cpu import DOC_MEMBERS, K, QUIRKS, STRS, rec
from tests.test_gpu_find_lists import _dev, _np, check
from tests.util import fuzz_corpus, load_fixture

pytestmark = pytest.mark.gpu
S = 1 << 55
ALL = [fo.ELEMENT, fo.INT64, fo.UINT64, fo.FLOAT64, fo.BOOL, fo.STRING, fj.JSON] + list(fl.LIST_KINDS) + [fl.STRING_CVT]
# the quirk tapes whose record the device hands to the one-thread walk
WALKED = {"non_string_key_keeps_rows", "key_at_end_of_tape", "nop_between_key_and_value", "cut_before_error_key",
          "error_key_before_cut", "error_key_inside_cut", "key_outside_its_buffer"}


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def want(tape, strs, msg, row_path, paths, kinds, only_keys=(), records=None):
    st, offs, tags, idx, keys, cells = fm.find_members(tape, strs, msg, row_path, paths, kinds, only_keys, records)
    return st, offs, tags, idx, keys, [[tuple(c) for c in col] for col in cells]


def check_members(res, w, kinds, what):
    rc, n_rec, n_rows, index, cols = res
    st, offs, tags, idx, keys, cells = w
    assert rc == 0, (what, rc)
    assert (n_rec, n_rows) == (len(st), len(idx)), (what, n_rec, n_rows, len(st), len(idx))
    assert _np(index.rec_status).tolist() == st, what
    assert _np(index.rec_offsets).tolist() == offs, what
    assert _np(index.row_tag).tolist() == tags, what
    assert _np(index.row_index).tolist() == idx, what
    ko = _np(index.key_offsets).tolist()
    data = _np(index.key_data).tobytes()
    assert len(ko) == n_rows + 1 and ko[0] == 0, what
    assert [data[ko[r]:ko[r + 1]] for r in range(n_rows)] == keys, what
    check(cols, n_rows, cells, kinds, what)


def foreign(ctx, tape, strs, msg, row_path, paths, kinds, what, only_keys=(), records=None):
    res = ctx.find_members_device(_dev(tape, np.int64), _dev(strs), _dev(msg), row_path, paths, kinds, list(only_keys))
    check_members(res, want(tape, strs, msg, row_path, paths, kinds, only_keys, records), kinds, what)
    return res


def _value_paths(objs, n=4):
    """[] (the member's value) and sub-paths of the first values"""
    seen, out = set(), [[]]
    for o in objs[:5]:
        for v in list(o.values())[:10]:
            for p in harvest(json.dumps(v).encode(), 10)[:-3]:
                if tuple(p) not in seen:
                    seen.add(tuple(p))
                    out.append(p)
    return out[:n] + [[b"\x00missing"]]


@pytest.mark.parametrize("name,row_path", DOC_MEMBERS)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures(ctx, oracle_native, name, row_path, copy):
    """sj_parse_find_members on the own tape, and the oracle's tape as a foreign one, under every kind"""
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc, copy_strings=copy)
    assert rc == 0
    msg = doc[off:off + ln]
    v = json.loads(doc)[row_path[0].decode()]
    ps = _value_paths([v], 2)
    paths, kinds = [p for p in ps for _ in ALL], [k for _ in ps for k in ALL]
    for only in ((), tuple(k.encode() for k in list(v)[1:4]) + (b"\x00none",)):
        w = want(tape, strs, msg, row_path, paths, kinds, only)
        assert len(w[3]) == (3 if only else len(v))
        check_members(ctx.parse_find_members(doc, row_path, paths, kinds, list(only), ndjson=False, copy_strings=copy), w,
                      kinds, (name, "own", only))
        assert ctx.find_rows_serial() == 0, name  # every record of a parser's tape passes propose / verify
        check_members(ctx.find_members_device(_dev(tape, np.int64), _dev(strs), _dev(msg), row_path, paths, kinds, list(only)),
                      w, kinds, (name, "foreign", only))
        assert ctx.find_rows_serial() == 0, name


@pytest.mark.parametrize("name", NDJSON_FIXTURES)
def test_ndjson_explode(ctx, oracle, name):
    """a row path of 0 segments: every key of every record; with two only_keys"""
    recs, nd = ndjson_records(name)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True)
    assert rc == 0
    paths = _value_paths(recs)
    kinds = [ALL[(3 * i) % len(ALL)] for i in range(len(paths))] + [fj.JSON, fl.STRING_CVT]
    paths += [[], []]
    keys = list(recs[0])
    for only in ((), (keys[0].encode(), keys[-1].encode())):
        w = want(tape, strs, nd[off:off + ln], [], paths, kinds, only)
        assert len(w[3]) == (sum(len(r) for r in recs) if not only else len(w[3])) > 0
        check_members(ctx.parse_find_members(nd, [], paths, kinds, list(only)), w, kinds, (name, only))
        assert ctx.find_rows_serial() == 0


def test_zero_segment_cell_is_the_key_cell(ctx, oracle):
    """for unique keys the 0-segment value cell is the [key] cell of the record's object (sj_find_device)"""
    recs, nd = ndjson_records("update-center")
    keys = sorted({k for r in recs for k in r})
    res = ctx.parse_find_members(nd, [], [[]] * 4, [fo.INT64, fo.STRING, fj.JSON, fo.ELEMENT])
    rc, N, R, index, cols = res
    assert rc == 0 and N == len(recs)
    by_key = {}
    for k in keys:
        rc, rows, c = ctx.parse_find(nd, [[k.encode()]] * 4, [fo.INT64, fo.STRING, fj.JSON, fo.ELEMENT])
        by_key[k] = c
    offs = _np(index.rec_offsets)
    for r in range(N):
        for q in range(int(offs[r]), int(offs[r + 1])):
            k = index.key(q).decode()
            for p in range(4):
                a, b = cols[p], by_key[k][p]
                assert (a.status[q], a.tag[q], a.index[q], a.value[q]) == (b.status[r], b.tag[r], b.index[r], b.value[r]), (r, k, p)
                if p in (1, 2):
                    assert bytes(a.data[a.offsets[q]:a.offsets[q + 1]]) == bytes(b.data[b.offsets[r]:b.offsets[r + 1]])


def test_fuzz_seeds(ctx, oracle):
    n = 0
    for name, data in fuzz_corpus("corpus", max_size=1 << 14):
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson)
            if rc:
                continue
            keys = harvest(data, 6)[:-3]
            for rp in ([], keys[0] if keys else [b"a"]):
                paths = harvest(data, 8) + [[]]
                kinds = [ALL[i % len(ALL)] for i in range(len(paths))]
                w = want(tape, strs, data[off:off + ln], rp, paths, kinds)
                check_members(ctx.parse_find_members(data, rp, paths, kinds, ndjson=ndjson), w, kinds, (name, ndjson, rp))
                n += 1
    assert n > 40


def test_own_tape_equals_foreign_and_deserialized(ctx):
    """the same output for the context's own tape and a copy passed as foreign; a Deserialize'd tape against the port;
    the launch count of this configuration is pinned"""
    import simdjson_b200 as sj
    import torch
    doc = load_fixture("citm_catalog")
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
    paths, kinds = [[b"name"], [b"subTopicIds"], []], [fo.STRING, fl.ARRAY_INT64, fj.JSON]
    l0 = ctx.launches()
    own = ctx.find_members_device(tape, strs, msg, [b"events"], paths, kinds)
    l1 = ctx.launches()
    fgn = ctx.find_members_device(tape.clone(), strs, msg, [b"events"], paths, kinds)
    l2 = ctx.launches()
    assert own[:3] == fgn[:3] == (0, 1, 184)
    for a, b in zip(list(own[3]) + [x for c in own[4] for x in c if x is not None],
                    list(fgn[3]) + [x for c in fgn[4] for x in c if x is not None]):
        assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
    t = tape.cpu().numpy().view(np.uint64)
    w = want(t, strs.cpu().numpy().tobytes(), doc, [b"events"], paths, kinds)
    check_members(own, w, kinds, "own")
    print("launches", l1 - l0, l2 - l1)
    # the sizes call: the member rows (KR1 .. KR7 with KO1, KO2 and the key lengths' scan: 28), KF3, KF4 + 2 scans (4),
    # and for the list and JSON paths their passes; the second call adds KR8, KO4 and KF5 and the cells' writers; a
    # foreign tape adds KM1, KC1a, KC1b and their scans (7) to each
    assert (l2 - l1) - (l1 - l0) == 2 * 7
    base = ctx.launches()
    ctx.find_members_device(tape, strs, msg, [b"events"], [[b"name"]], [fo.STRING])
    assert ctx.launches() - base == (28 + 4) + (28 + 4 + 3)
    back = sj.Serializer(ctx).Deserialize(sj.Serializer(ctx).Serialize(sj.Parse(doc, ctx=ctx)))
    t, s, m = np.asarray(back.Tape, dtype=np.uint64), bytes(back.Strings), bytes(back.Message)
    foreign(ctx, t, s, m, [b"events"], paths, kinds, "deserialize")


def _tape_of(records):
    """rec() per record, laid end to end, links moved to each record's place"""
    words, at = [], 0
    for members, link in records:
        for w in rec(members, link):
            if (w >> 56) in b"r{[}]":
                w += at
            words.append(w)
        at = len(words)
    return np.array(words, dtype=np.uint64)


@pytest.mark.parametrize("q", QUIRKS, ids=[q[0] for q in QUIRKS])
def test_quirk_tapes(ctx, q):
    """each quirk tape of tests/test_find_members_cpu.py, alone and behind a record that passes; the records that need
    the one-thread walk take it, the others do not"""
    name, members, only, link, w = q
    paths, kinds = [[], [], [b"a"]], [fo.INT64, fj.JSON, fo.BOOL]
    for recs in ([(members, link)], [(K("a") + [word("t")], None), (members, link)]):
        tape = _tape_of(recs)
        foreign(ctx, tape, STRS, b"", [], paths, kinds, name, only, fo.roots(tape))
        assert (ctx.find_rows_serial() > 0) == (name in WALKED), name


def _edge_tape(s):
    """one record { "a": [t x s], "b": 1, "c": "d", "e": t } : key "b" at virtual word 5 + s of the object words"""
    arr = [word("[", 6 + s)] + [word("t")] * s + [word("]", 4)]
    return np.array(rec(K("a") + arr + K("b") + [word("l"), 1] + K("c") + [word('"', S | 3), 1] + K("e") + [word("t")]),
                    dtype=np.uint64)


@pytest.mark.parametrize("edge", [4096, 4096 * 1024])
def test_keys_and_values_around_tile_and_group_edges(ctx, edge):
    """keys, their length words and values at -3 .. +3 of a tile edge and of the first group edge (1 024 tiles)"""
    paths, kinds = [[], [], [b"a"]], [fo.INT64, fo.STRING, fo.ELEMENT]
    for s in range(edge - 9, edge - 2):
        tape = _edge_tape(s)
        foreign(ctx, tape, STRS, b"", [], paths, kinds, (edge, s), (b"b", b"e") if s % 2 else (), [0])
        assert ctx.find_rows_serial() == 0


def _rec_np(members, at):
    """rec() of a numpy array of members at tape index `at`"""
    n = 2 + len(members)
    return np.concatenate([np.array([word("r", at + n + 2), word("{", at + n + 1)], dtype=np.uint64),
                           np.asarray(members, dtype=np.uint64), np.array([word("}", at + 1), word("r", at)], dtype=np.uint64)])


def test_small_objects_beside_a_huge_one(ctx):
    """objects of 0, 1 and 2 members beside one of 2^22 + 3 members, as four records of one foreign tape"""
    big = (1 << 22) + 3
    keys = np.arange(big, dtype=np.uint64) % np.uint64(8)
    body = np.empty(3 * big, dtype=np.uint64)
    body[0::3] = np.uint64(ord('"') << 56) | np.uint64(S) | keys
    body[1::3] = 1
    body[2::3] = np.uint64(ord("t") << 56)
    parts, starts = [], []
    for m in ([], K("a") + [word("t")], body, K("b") + [word("l"), 4] + K("c") + [word("f")]):
        starts.append(sum(len(x) for x in parts))
        parts.append(_rec_np(m, starts[-1]))
    tape = np.concatenate(parts)
    rc, N, R, index, cols = ctx.find_members_device(_dev(tape, np.int64), _dev(STRS), None, [], [[]], [fo.BOOL])
    assert (rc, N, R) == (0, 4, big + 3)
    assert _np(index.rec_offsets).tolist() == [0, 0, 1, 1 + big, 3 + big]
    assert _np(index.rec_status).tolist() == [0] * 4
    assert np.array_equal(_np(index.row_index)[1:1 + big], starts[2] + 4 + 3 * np.arange(big))
    ko, kd = _np(index.key_offsets), _np(index.key_data)
    assert ko[-1] == R and bytes(kd[1:1 + big]) == bytes((keys + np.uint64(ord("a"))).astype(np.uint8))
    assert bytes(kd[:1]) + bytes(kd[1 + big:]) == b"abc"
    # BOOL of each value: the 't's are true; the last record's 'l' is CONVERT and its 'f' false
    assert np.all(_np(cols[0].value)[:R - 2] == 1) and np.all(_np(cols[0].status)[:R - 2] == 0)
    assert _np(cols[0].status)[R - 2:].tolist() == [fo.CONVERT, fo.OK] and _np(cols[0].value)[R - 2:].tolist() == [0, 0]
    assert ctx.find_rows_serial() == 0


def test_half_gib_document(ctx):
    """{"plugins": {...}} of update-center's plugins with unique keys, repeated to 0.5 GiB: every member a row, its key
    and its ["version"] cell against the generator, no record walked by one thread"""
    plugins = list(json.loads(load_fixture("update-center"))["plugins"].items())
    parts, keys, versions, total, i = [], [], [], 0, 0
    while total < (512 << 20):
        for k, v in plugins:
            key = "%s~%d" % (k, i)
            p = json.dumps(key).encode() + b":" + json.dumps(v, separators=(",", ":")).encode()
            parts.append(p)
            keys.append(key.encode())
            versions.append(v.get("version") if isinstance(v, dict) else None)
            total += len(p) + 1
        i += 1
    doc = b'{"plugins":{' + b",".join(parts) + b"}}"
    rc, N, R, index, cols = ctx.parse_find_members(doc, [b"plugins"], [[b"version"]], [fo.STRING], ndjson=False)
    assert (rc, N, R) == (0, 1, len(keys))
    assert ctx.find_rows_serial() == 0
    ko, kd = index.key_offsets, index.key_data.tobytes()
    assert ko[-1] == len(kd) and [kd[ko[r]:ko[r + 1]] for r in range(R)] == keys
    c = cols[0]
    got = [bytes(c.data[c.offsets[r]:c.offsets[r + 1]]) if c.status[r] == fo.OK else None for r in range(R)]
    assert got == [v.encode() if isinstance(v, str) else None for v in versions]


def test_array_rows_after_member_rows(ctx):
    """a member-rows call leaves nothing that an array-rows call reads: on the same context, a path of 0 segments on
    array rows stays NOT_FOUND after a member-rows call wrote key heads"""
    nd = b"\n".join([b'{"a":{"x":"xy","y":2},"b":[1,"s",{"x":3}]}', b'{"a":{"z":true},"b":[]}'])
    paths, kinds = [[], [b"x"]], [fo.ELEMENT, fo.INT64]
    assert ctx.parse_find_members(nd, [b"a"], paths, kinds)[:3] == (0, 2, 3)
    rc, N, R, index, cols = ctx.parse_find_rows(nd, [b"b"], paths, kinds)
    assert (rc, N, R) == (0, 2, 3)
    assert cols[0].status.tolist() == [fo.NOT_FOUND] * 3 and cols[0].index.tolist() == [-1] * 3
    assert cols[1].status.tolist() == [fo.NOT_OBJECT, fo.NOT_OBJECT, fo.OK] and int(cols[1].value[2]) == 3


def test_empty_and_rootless_tapes_ask_for_sizes(ctx):
    import simdjson_b200 as sj
    cp, _k = sj._find_paths([[b"a"]], [fo.INT64])
    rp, _r = sj._find_paths([[b"a"], []], [fo.ELEMENT] * 2)
    for t in (None, _dev(np.array([word("n"), word("t"), word("l"), 5], dtype=np.uint64), np.int64)):
        n = [C.c_size_t(7) for _ in range(5)]
        tp, tl = (t.data_ptr(), t.numel()) if t is not None else (None, 0)
        assert ctx.L.sj_find_members_device(ctx.h, None, 0, tp, tl, None, 0, rp, C.pointer(rp[1]), cp,
                                            1, None, None, None, None, *(C.byref(x) for x in n)) == 0
        assert [x.value for x in n] == [0] * 5
    rc, N, R, index, cols = ctx.find_members_device(t, None, None, [b"a"], [[b"a"]], [fo.INT64])
    assert (rc, N, R) == (0, 0, 0) and _np(index.rec_offsets).tolist() == [0] and _np(index.key_offsets).tolist() == [0]


def test_capacity_and_arguments(ctx):
    """sizes exact and nothing written on SJ_ERR_CAPACITY with each of the five caps one short in turn; SJ_ERR_ARGUMENT
    for only_keys of more than 32 keys or of a kind other than ELEMENT"""
    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    nd = b"\n".join([b'{"a":{"x":"xy","y":[1,2]},"b":1}', b'{"a":{}}', b'{"b":1}', b'{"a":{"zz":[3],"x":"q"}}'])
    paths, kinds = [[], []], [fo.STRING, fl.ARRAY_INT64]
    rc, tape, strs, (off, ln) = ctx.parse(nd, ndjson=True)
    assert rc == 0
    t, s, m = _dev(tape, np.int64), _dev(strs), _dev(nd[off:off + ln])
    rc, N, R, index, cols = ctx.find_members_device(t, s, m, [b"a"], paths, kinds)
    assert (rc, N, R) == (0, 4, 4)
    sizes = (4, 4, 3, 3, 5)  # records, rows, string bytes, elements, key bytes
    cpaths, _k = sj._find_paths(paths, kinds)
    full = sj._find_cols(sj._torch_empty(t.device), 2, 1, 1, 4, 3, 3, 4, 5)

    def call(rec_cap, row_cap, str_cap, elem_cap, key_cap, only=((), fo.ELEMENT)):
        rpath, _r = sj._find_paths([[b"a"], list(only[0])], [fo.ELEMENT, only[1]])
        out = [torch.full_like(x, 0x5A) if x.dtype == torch.uint8 else torch.full_like(x, 0x5A5A) for x in full]
        o = _lib.FindOut(*(x.data_ptr() for x in out[:6]), row_cap, str_cap)
        lo = _lib.FindListsOut(out[6].data_ptr(), out[7].data_ptr(), elem_cap)
        ro = _lib.FindRowsOut(*(x.data_ptr() for x in out[8:12]), rec_cap)
        ko = _lib.FindKeysOut(out[12].data_ptr(), out[13].data_ptr(), key_cap)
        n = [C.c_size_t(0) for _ in range(5)]
        rc = ctx.L.sj_find_members_device(ctx.h, m.data_ptr(), m.numel(), t.data_ptr(), t.numel(), s.data_ptr(), s.numel(),
                                          rpath, C.pointer(rpath[1]), cpaths, 2, C.byref(o), C.byref(lo),
                                          C.byref(ro), C.byref(ko), *(C.byref(x) for x in n))
        torch.cuda.synchronize()
        return rc, tuple(x.value for x in n), out
    rc, n, out = call(*sizes)
    assert (rc, n) == (0, sizes)
    assert bytes(out[13][:5].cpu().numpy()) == b"xyzzx" and out[12].cpu().tolist() == [0, 1, 2, 4, 5]
    for k in range(5):
        caps = list(sizes)
        caps[k] -= 1
        rc, n, out = call(*caps)
        assert (rc, n) == (_lib.ERR_CAPACITY, sizes), k
        assert all(bool((x.view(torch.uint8) == 0x5A).all()) for x in out if x.dtype == torch.uint8), k
    assert call(*sizes, only=([b"k%d" % i for i in range(33)], fo.ELEMENT))[0] == _lib.ERR_ARGUMENT
    assert call(*sizes, only=([b"x"], fo.STRING))[0] == _lib.ERR_ARGUMENT
    assert call(*sizes, only=([b"x"] * 32, fo.ELEMENT))[:2] == (0, (4, 2, 3, 0, 2))
