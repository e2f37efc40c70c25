"""GPU tests of the device find (find.cuh): ForEach + FindElement + the accessors, cell for cell against the Python port
(tests/find_oracle.py) on fixtures, fuzz seeds and foreign tapes (builder, Deserialize output with nops, randomly
corrupted words), plus the capacity contract, the argument limits, the launch count and a size-independent check on a
512 MiB K0 batch."""
import ctypes as C
import json
import random

import numpy as np
import pytest

from tests import find_oracle as fo
from tests.tape_builder import TapeBuilder
from tests.util import TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu
KINDS = [fo.ELEMENT, fo.INT64, fo.UINT64, fo.FLOAT64, fo.BOOL, fo.STRING]


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


def _harvest(doc, limit=60):
    """key paths of a JSON document down to depth 4 through objects only, plus missing, empty-key and
    non-object-intermediate paths"""
    out = []

    def walk(v, path):
        if not isinstance(v, dict) or len(path) >= 4:
            return
        for k, x in v.items():
            p = path + [k.encode("utf-8", "surrogatepass")]
            out.append(p)
            if not isinstance(x, dict):
                out.append(p + [b"x"])  # through a value that is not an object
            walk(x, p)

    try:
        v = json.loads(doc)
    except Exception:
        v = None
    walk(v if isinstance(v, dict) else {}, [])
    random.Random(len(doc)).shuffle(out)
    return out[:limit] + [[b"\x00missing"], [b""], [b"", b""], []]


def _check(cols, rows, want, kinds, what):
    assert rows == len(want[0]) if want else True, what
    for p, k in enumerate(kinds):
        c = cols[p]
        st, tag, idx = (np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in (c.status, c.tag, c.index))
        val = c.value.view(torch_int64()).cpu().numpy() if hasattr(c.value, "cpu") else c.value
        val = np.asarray(val).view(np.uint64)
        if k == fo.STRING:
            off = np.asarray(c.offsets.cpu() if hasattr(c.offsets, "cpu") else c.offsets)
            data = (c.data.cpu().numpy() if hasattr(c.data, "cpu") else c.data).tobytes()
        for r, w in enumerate(want[p]):
            got = (int(st[r]), int(tag[r]), int(idx[r]))
            assert got == (w.status, w.tag, w.index), (what, p, r, got, w)
            if k == fo.STRING:
                assert data[off[r]:off[r + 1]] == w.value, (what, p, r)
                assert int(val[r]) == len(w.value), (what, p, r)
            else:
                assert int(val[r]) == w.value, (what, p, r, int(val[r]), w)


def torch_int64():
    import torch
    return torch.int64


def _device_vs_port(ctx, tape, strs, msg, paths, kinds, what):
    rc, rows, cols = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), paths, kinds)
    assert rc == 0, (what, rc)
    want = fo.find(tape, strs, msg, paths, kinds)
    assert rows == len(fo.roots(tape)), what
    _check(cols, rows, want, kinds, what)


def _batches(paths):
    ks = [KINDS[i % len(KINDS)] for i in range(len(paths))]
    for i in range(0, len(paths), 64):
        yield paths[i:i + 64], ks[i:i + 64]


@pytest.mark.parametrize("name", TAPE_FILES)
@pytest.mark.parametrize("copy", [True, False])
def test_fixtures(ctx, oracle_native, name, copy):
    """every fixture: the context's own tape (sj_parse_find) and the oracle's tape as a foreign one (sj_find_device)"""
    doc = load_fixture(name)
    rc, tape, strs, (off, ln) = oracle_native.parse(doc, copy_strings=copy)
    assert rc == 0
    msg = doc[off:off + ln]
    for paths, kinds in _batches(_harvest(doc)):
        want = fo.find(tape, strs, msg, paths, kinds, fo.foreach_roots(tape))
        rc, rows, cols = ctx.parse_find(doc, paths, kinds, ndjson=False, copy_strings=copy)
        assert rc == 0
        _check(cols, rows, want, kinds, name)
        _device_vs_port(ctx, tape, strs, msg, paths, kinds, name)


def test_tricky_ndjson_every_kind(ctx, oracle):
    nd, recs = tricky_ndjson()
    paths = [[b"Make"], [b"a"], [b"a", b"Make"], [b"Make", b"Make"], [b"M\x61ke"], [b""], [b"t"], [b"f"], [b"n"], [b"d"],
             [b"l"], [b"u"], [b"x"], [b"nope"]]
    for copy in (True, False):
        rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
        for k in KINDS:
            ks = [k] * len(paths)
            rc, rows, cols = ctx.parse_find(nd, paths, ks, copy_strings=copy)
            assert rc == 0 and rows == len(recs)
            _check(cols, rows, fo.find(tape, strs, nd[off:off + ln], paths, ks, fo.foreach_roots(tape)), ks, "tricky")


def test_fuzz_seeds(ctx, oracle):
    n = 0
    for name, data in fuzz_corpus("corpus", max_size=1 << 14):
        for ndjson in (False, True):
            rc, tape, strs, (off, ln) = oracle.parse(data, ndjson=ndjson)
            if rc:
                continue
            paths = _harvest(data, 20)
            kinds = [KINDS[i % 6] for i in range(len(paths))]
            rc, rows, cols = ctx.parse_find(data, paths, kinds, ndjson=ndjson)
            assert rc == 0, name
            _check(cols, rows, fo.find(tape, strs, data[off:off + ln], paths, kinds, fo.foreach_roots(tape)), kinds, name)
            n += 1
    assert n > 20


def _records(k):
    b = TapeBuilder()
    for i in range(k):
        b.open("r"); b.open("{")
        b.string(b"k"); b.number("l", i)
        b.string(b"s"); b.string(b"v%d" % i, copy=i % 2 == 0)
        b.string(b"o"); b.open("{"); b.string(b"d"); b.number("d", struct_f(i + 0.5)); b.close()
        b.close(); b.close()
    return b.build()


def struct_f(x):
    return fo._f64_bits(x)


def test_foreign_tapes(ctx):
    """builder tapes, Deserialize output with nops, and randomly corrupted words: equal cells, rows in tape order"""
    from tests import serialize_oracle as so
    paths = [[b"k"], [b"s"], [b"o", b"d"], [b"o"], [b"s", b"x"], [b"k"]]
    kinds = [fo.INT64, fo.STRING, fo.FLOAT64, fo.ELEMENT, fo.UINT64, fo.STRING]
    tape, strs, msg = _records(300)
    _device_vs_port(ctx, tape, strs, msg, paths, kinds, "builder")
    t2, s2, m2 = so.deserialize(so.serialize(tape, strs, msg))
    t2 = np.array(t2, dtype=np.uint64)
    _device_vs_port(ctx, t2, s2, m2, paths, kinds, "deserialized")
    holes = t2.copy()
    for i in fo.roots(t2)[::3]:
        holes[i + 2:i + 6] = [ord("N") << 56 | 4, ord("N") << 56 | 3, ord("N") << 56 | 2, ord("N") << 56 | 1]
    _device_vs_port(ctx, holes, s2, m2, paths, kinds, "nops")
    rng = random.Random(7)
    nd, _ = tricky_ndjson()
    pk = load_fixture("parking-citations")
    from oracle.pyoracle import Oracle
    o = Oracle("scalar")
    for src, ps in ((nd, [[b"Make"], [b"a", b"Make"], [b"x"], [b""]]), (pk, [[b"Make"], [b"Fine"], [b"Ticket"]])):
        rc, tape, strs, (off, ln) = o.parse(src, ndjson=True)
        msg = src[off:off + ln]
        for trial in range(40):
            t = tape.copy()
            for _ in range(rng.choice([1, 3, 20])):
                i = rng.randrange(t.size)
                r = rng.random()
                tag = rng.choice(b'rN{}[]"ludtfn\x00') if r < 0.7 else rng.randrange(256)
                v = rng.choice([0, 1, 2, i, i + 1, i + 2, t.size, t.size + 1, rng.randrange(1 << 56), (1 << 56) - 1])
                t[i] = (tag << 56) | (v & fo.VAL) if r < 0.9 else rng.randrange(1 << 64)
            ks = [KINDS[(trial + j) % 6] for j in range(len(ps))]
            _device_vs_port(ctx, t, strs, msg, ps, ks, "corrupt %d" % trial)


def test_own_tape_equals_foreign(ctx):
    """on the context's own tape the rows are stage 2's root list; the same tape as a foreign one gives equal columns"""
    import torch
    nd = b"\n".join(load_fixture("parking-citations").strip().split(b"\n")[:700])
    L = ctx.L
    d_msg = torch.full((len(nd) + 4096,), 0x20, dtype=torch.uint8, device="cuda")
    d_msg[:len(nd)].copy_(torch.frombuffer(bytearray(nd), dtype=torch.uint8))
    tcap, scap = C.c_size_t(0), C.c_size_t(0)
    L.sj_bounds(len(nd), C.byref(tcap), C.byref(scap))
    d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    assert L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(nd), 3, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                             d_str.data_ptr(), d_str.numel(), C.byref(sl)) == 0
    paths, kinds = [[b"Make"], [b"Ticket"], [b"Fine"], [b"nope"]], [fo.STRING, fo.STRING, fo.ELEMENT, fo.INT64]
    tape, strs, msg = d_tape[:tl.value], d_str[:sl.value], d_msg[:len(nd)]
    l0 = ctx.launches()
    rc, rows, own = ctx.find_device(tape, strs, msg, paths, kinds)
    l1 = ctx.launches()
    rc2, rows2, foreign = ctx.find_device(tape.clone(), strs, msg, paths, kinds)
    l2 = ctx.launches()
    assert rc == rc2 == 0 and rows == rows2 == 700
    # find_device without `out` asks for the sizes first: two calls each
    assert (l1 - l0, l2 - l1) == (4 + 5, (7 + 4) + (7 + 5))
    for a, b in zip(own, foreign):
        for x, y in zip(a, b):
            assert (x is None and y is None) or torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8))
    t = tape.cpu().numpy().view(np.uint64)
    want = fo.find(t, strs.cpu().numpy().tobytes(), nd, paths, kinds, fo.foreach_roots(t))
    _check(own, rows, want, kinds, "own")


@pytest.mark.parametrize("copy", [True, False])
def test_foreign_rows_skip_value_words_that_look_like_roots(ctx, oracle, copy):
    """numbers whose value word starts with the byte 'r' on a foreign tape: the rows are ForEach's, as on the context's
    own tape of the same text"""
    import torch
    from tests.test_find_cpu import ROOT_LOOKALIKES
    nd = b"\n".join([ROOT_LOOKALIKES] * 300)
    rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
    msg = nd[off:off + ln]
    rows_want = fo.foreach_roots(tape)
    assert len(rows_want) == 1500
    paths, kinds = [[b"b"], [b"a"], [b"a", b"c"]], [fo.STRING, fo.INT64, fo.UINT64]
    want = fo.find(tape, strs, msg, paths, kinds, rows_want)
    rc, rows, foreign = ctx.find_device(_dev(tape, np.int64), _dev(strs), _dev(msg), paths, kinds)
    assert rc == 0 and rows == 1500
    _check(foreign, rows, want, kinds, "foreign")
    rc, rows, own = ctx.parse_find(nd, paths, kinds, copy_strings=copy)
    assert rc == 0 and rows == 1500
    _check(own, rows, want, kinds, "own")
    # countWhere counts the same roots
    assert ctx.parse_count_where(nd, b"b", b"z", copy_strings=copy) == (0, 1500, 300)
    roots, matches = C.c_uint64(0), C.c_uint64(0)
    d_tape, d_strs, d_msg = _dev(tape, np.int64), _dev(strs + b"\0"), _dev(msg + b"\0")
    assert ctx.L.sj_count_where_device(ctx.h, d_msg.data_ptr(), d_tape.data_ptr(), len(tape), d_strs.data_ptr(), b"b", 1,
                                       b"z", 1, C.byref(roots), C.byref(matches)) == 0
    assert (roots.value, matches.value) == (1500, 300) == oracle.count_where(tape, strs, msg, b"b", b"z")


def test_no_rows_still_writes_the_first_offset(ctx):
    import torch
    from simdjson_b200 import _find_paths, _lib
    cp, keep = _find_paths([[b"k"], [b"s"]], [fo.STRING, fo.STRING])
    tape = torch.tensor([ord("n") << 56], dtype=torch.int64, device="cuda")  # no root at all
    offs = torch.full((2, 4), -7, dtype=torch.int64, device="cuda")
    st = torch.full((2, 3), 9, dtype=torch.uint8, device="cuda")
    v = torch.full((2, 3), 9, dtype=torch.int64, device="cuda")
    out = _lib.FindOut(st.data_ptr(), st.data_ptr(), v.data_ptr(), v.data_ptr(), offs.data_ptr(), None, 3, 0)
    rows, nb = C.c_size_t(9), C.c_size_t(9)
    for n in (1, 0):
        offs.fill_(-7)
        assert ctx.L.sj_find_device(ctx.h, None, 0, tape.data_ptr(), n, None, 0, cp, 2, C.byref(out), C.byref(rows),
                                    C.byref(nb)) == 0
        assert (rows.value, nb.value) == (0, 0)
        assert offs[:, 0].tolist() == [0, 0] and offs[:, 1:].eq(-7).all()
    import simdjson_b200 as sj
    rc, r, cols = ctx.find_device(tape, None, None, [[b"k"]], [fo.STRING])
    assert rc == 0 and r == 0 and cols[0].offsets.tolist() == [0]


def test_capacity_writes_nothing(ctx):
    import torch
    tape, strs, msg = _records(50)
    paths, kinds = [[b"s"], [b"k"]], [fo.STRING, fo.INT64]
    args = (_dev(tape, np.int64), _dev(strs), _dev(msg))
    rc, rows, cols = ctx.find_device(*args, paths, kinds)
    nbytes = int(cols[0].offsets[-1])
    assert rc == 0 and rows == 50 and nbytes == sum(len(b"v%d" % i) for i in range(50))
    for row_cap, str_cap in ((49, nbytes), (50, nbytes - 1), (0, 0)):
        out = (torch.full((2, row_cap), 0xAB, dtype=torch.uint8, device="cuda"),
               torch.full((2, row_cap), 0xAB, dtype=torch.uint8, device="cuda"),
               torch.full((2, row_cap), -7, dtype=torch.int64, device="cuda"),
               torch.full((2, row_cap), -7, dtype=torch.int64, device="cuda"),
               torch.full((1, row_cap + 1), -7, dtype=torch.int64, device="cuda"),
               torch.full((max(str_cap, 1),), 0xAB, dtype=torch.uint8, device="cuda"))
        before = [t.clone() for t in out]
        rc, r, c = ctx.find_device(*args, paths, kinds, out=out)
        assert rc == 4 and r == 50 and c is None
        assert all(torch.equal(a, b) for a, b in zip(out, before))
    s, b = C.c_size_t(0), C.c_size_t(0)
    from simdjson_b200 import _find_paths
    cp, keep = _find_paths(paths, kinds)
    assert ctx.L.sj_find_device(ctx.h, args[2].data_ptr(), args[2].numel(), args[0].data_ptr(), args[0].numel(),
                                args[1].data_ptr(), args[1].numel(), cp, 2, None, C.byref(s), C.byref(b)) == 4
    assert (s.value, b.value) == (50, nbytes)


def test_argument_limits(ctx):
    import torch
    tape, strs, msg = _records(3)
    args = (_dev(tape, np.int64), _dev(strs), _dev(msg))
    ok = ctx.find_device(*args, [[b"k"]] * 64, [fo.INT64] * 64)
    assert ok[0] == 0 and ok[1] == 3
    assert ctx.find_device(*args, [[b"k"] * 32], [fo.INT64])[0] == 0
    assert ctx.find_device(*args, [[b"k" * 16384]], [fo.INT64])[0] == 0
    for paths, kinds in (([], []), ([[b"k"]] * 65, [fo.INT64] * 65), ([[b"k"] * 33], [fo.INT64]),
                         ([[b"k" * 16385]], [fo.INT64]), ([[b"k" * 8192], [b"k" * 8193]], [0, 0]), ([[b"k"]], [6])):
        assert ctx.find_device(*args, paths, kinds)[0] == 6, (len(paths), kinds)


def test_k0_batch_at_scale(ctx):
    """a 512 MiB K0 batch: row g's Ticket is %010d % g; Fine and Make are those of template line g mod 1000"""
    import torch
    L = ctx.L
    pk = load_fixture("parking-citations").strip()
    lines = pk.split(b"\n")
    mib = 512
    n_rec = (mib << 20) // (len(pk) // len(lines) + 1)
    d_msg = torch.full(((mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device="cuda")
    glen = C.c_size_t(0)
    assert L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d_msg.data_ptr(), d_msg.numel() - (1 << 16), C.byref(glen)) == 0
    n = glen.value
    tcap, scap = C.c_size_t(0), C.c_size_t(0)
    L.sj_bounds(n, C.byref(tcap), C.byref(scap))
    d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    assert L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, 3, d_tape.data_ptr(), d_tape.numel(), C.byref(tl), d_str.data_ptr(),
                             d_str.numel(), C.byref(sl)) == 0
    paths, kinds = [[b"Ticket"], [b"Fine"], [b"Make"]], [fo.STRING] * 3
    rc, rows, cols = ctx.find_device(d_tape[:tl.value], d_str[:sl.value], d_msg[:n], paths, kinds)
    assert rc == 0 and rows == n_rec
    for c in cols:
        assert bool((c.status == 0).all())
    tick = cols[0]
    assert bool((tick.offsets[1:] - tick.offsets[:-1] == 10).all())
    got = tick.data[:10 * n_rec].cpu().numpy().tobytes()
    assert got == b"".join(b"%010d" % (g % 10**10) for g in range(n_rec))
    tmpl = [json.loads(l) for l in lines]
    for c, key in ((cols[1], "Fine"), (cols[2], "Make")):
        vals = [tmpl[g % 1000][key].encode() for g in range(1000)]
        lens = torch.tensor([len(v) for v in vals], dtype=torch.int64, device="cuda")
        g = torch.arange(n_rec, device="cuda") % 1000
        assert torch.equal(c.offsets[1:] - c.offsets[:-1], lens[g])
        whole = c.data[int(c.offsets[0]):int(c.offsets[-1])].cpu().numpy().tobytes()
        reps, rest = divmod(n_rec, 1000)
        assert whole == b"".join(vals) * reps + b"".join(vals[:rest])
