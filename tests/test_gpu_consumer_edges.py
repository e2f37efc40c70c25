"""The device tape consumers at their edges, against plain sequential references: the root finder (KM1, KC1a, KC1b) on
tapes with roots, look-alike value words, parity runs, keys and values at E - 2 .. E + 1 of every tile and group edge
E; countWhere (KC2) at its lane, warp and block edges on the own and the foreign tape; KF3's staged segments at the
find's path limits; KF5's string scan across a group of tiles and its row stride; every accessor conversion; the own
tape's root list against KC1 on messages with record boundaries at stage 2's edges; and the root list after a
Deserialize into the tape a parse left.  The expectations come from tests/consumer_edge_tapes.py, which
tests/test_consumer_edge_tapes_cpu.py checks against tests/find_oracle.py and the C oracle."""
import ctypes as C

import numpy as np
import pytest

from tests import consumer_edge_tapes as ce
from tests import find_oracle as fo

pytestmark = pytest.mark.gpu
FLAG_NDJSON, FLAG_COPY = 1, 2
WS = b" \t\r\n"


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
    return d_tape, d_strs, d_msg


def _count(ctx, d_tape, n, d_strs, d_msg, key, value):
    roots, matches = C.c_uint64(0), C.c_uint64(0)
    sp = d_strs.data_ptr() if d_strs is not None else None
    mp = d_msg.data_ptr() if d_msg is not None else None
    rc = ctx.L.sj_count_where_device(ctx.h, mp, d_tape.data_ptr(), n, sp, key, len(key), value, len(value),
                                     C.byref(roots), C.byref(matches))
    assert rc == 0
    return roots.value, matches.value


def _host(cols):
    """columns as numpy: [(status, tag, index, value bits as int64, offsets or None)], and the string bytes"""
    import torch
    out, data = [], None
    for c in cols:
        out.append((c.status.cpu().numpy(), c.tag.cpu().numpy(), c.index.cpu().numpy(),
                    c.value.contiguous().view(torch.int64).cpu().numpy(),
                    None if c.offsets is None else c.offsets.cpu().numpy()))
        if c.data is not None:
            data = c.data.cpu().numpy().tobytes()
    return out, data


def _check_cells(cols, want, kinds, rows, what):
    """the device columns against expected Cells on the rows `rows` (positions in the columns)"""
    host, data = _host(cols)
    for p, k in enumerate(kinds):
        st, tag, idx, val, off = host[p]
        for r in rows:
            w = want[p][r]
            got = (int(st[r]), int(tag[r]), int(idx[r]))
            assert got == (w.status, w.tag, w.index), (what, p, r, got, w)
            if k == ce.STRING:
                assert data[off[r]:off[r + 1]] == w.value and int(val[r]) == len(w.value), (what, p, r)
            else:
                assert int(val[r]) & ce.M64 == w.value, (what, p, r, hex(int(val[r]) & ce.M64), w)


# ---- the root finder -----------------------------------------------------------------------------------------------
def _run_edge_tape(ctx, et):
    paths, kinds = [p for p, _ in ce.EDGE_PATHS], [k for _, k in ce.EDGE_PATHS]
    d_tape, d_strs, d_msg = _upload(et.tape, et.strings, et.message)
    rc, rows, cols = ctx.find_device(d_tape, d_strs, d_msg, paths, kinds)
    assert rc == 0 and rows == len(et.rows), (et.name, rows, len(et.rows))
    # the rows: ELEMENT of "k" is the head right behind `r {"k"`, on every row
    idx = cols[0].index.cpu().numpy()
    assert np.array_equal(idx, et.rows + 4), et.name
    assert bool((cols[0].status == ce.OK).all())
    _check_cells(cols, et.cells, kinds, range(rows), et.name)
    for (key, value), n in et.count_where.items():
        assert _count(ctx, d_tape, len(et.tape), d_strs, d_msg, key, value) == (len(et.rows), n), (et.name, key)


def test_root_finder_small_tapes(ctx):
    for et in ce.edge_tapes(large=False):
        _run_edge_tape(ctx, et)


@pytest.mark.parametrize("family", ce.FAMILIES)
def test_root_finder_tile_and_group_edges(ctx, family):
    for o in ce.OFFSETS:
        _run_edge_tape(ctx, ce.edge_tape(family, o))


# ---- countWhere ----------------------------------------------------------------------------------------------------
class _Parse:
    """sj_parse_device into buffers reused across messages; the message is followed by spaces in its buffer"""

    def __init__(self, ctx, cap):
        import torch
        tcap, scap = C.c_size_t(0), C.c_size_t(0)
        ctx.L.sj_bounds(cap, C.byref(tcap), C.byref(scap))
        self.ctx = ctx
        self.msg = torch.full((cap + 4096,), 0x20, dtype=torch.uint8, device="cuda")
        self.tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
        self.strs = torch.empty(max(scap.value, 1), dtype=torch.uint8, device="cuda")

    def __call__(self, msg, ndjson=True, copy=True):
        """parse the trimmed window `msg` (sj_parse_device does not trim)"""
        import torch
        assert len(msg) + 4096 <= self.msg.numel() and msg == msg.strip(WS)
        self.msg[:len(msg) + 64].fill_(0x20)
        self.msg[:len(msg)].copy_(torch.frombuffer(bytearray(msg), dtype=torch.uint8))
        tl, sl = C.c_size_t(0), C.c_size_t(0)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY if copy else 0)
        rc = self.ctx.L.sj_parse_device(self.ctx.h, self.msg.data_ptr(), len(msg), flags, self.tape.data_ptr(),
                                        self.tape.numel(), C.byref(tl), self.strs.data_ptr(), self.strs.numel(), C.byref(sl))
        assert rc == 0
        return self.tape[:tl.value], self.strs[:sl.value], self.msg[:len(msg)]


def _own_and_foreign_counts(ctx, tape, strs, msg, key, value):
    """countWhere on the tape the parse left (stage 2's root list: one launch) and on a copy (KC1's roots)"""
    l0 = ctx.launches()
    own = _count(ctx, tape, tape.numel(), strs, msg, key, value)
    own_launches = ctx.launches() - l0
    foreign = _count(ctx, tape.clone(), tape.numel(), strs, msg, key, value)
    assert own_launches == (1 if own[0] else 0)
    return own, foreign


@pytest.mark.parametrize("copy", [True, False])
def test_count_where_lanes_warps_blocks(ctx, copy):
    """matches in no lane, every lane, lane 0, lane 31 and every other lane, at root counts around a warp, KC2's block
    and a tile; key and value lengths 0 .. 70, the keys in Strings.B or in the message"""
    cases = ce.cw_cases()
    big = max(len(ce.cw_message(n, "all", kl, vl)[0]) for n, _, kl, vl in cases if n == max(ce.CW_COUNTS))
    parse = _Parse(ctx, big + 4096)
    for n, pat, kl, vl in cases:
        msg, key, value, hits = ce.cw_message(n, pat, kl, vl)
        tape, strs, m = parse(msg, copy=copy)
        own, foreign = _own_and_foreign_counts(ctx, tape, strs, m, key, value)
        assert own == foreign == (n, len(hits)), (n, pat, kl, vl, own, foreign)
        if n <= ce.KC2_BLOCK + 1 and pat == "alternate":
            t = tape.cpu().numpy().view(np.uint64)
            cells = fo.find(t, strs.cpu().numpy().tobytes(), m.cpu().numpy().tobytes(), [[key]], [fo.STRING],
                            fo.foreach_roots(t))[0]
            assert sum(c.status == fo.OK and c.value == value for c in cells) == len(hits)


@pytest.mark.parametrize("pattern", ["lane0", "alternate"])
def test_count_where_past_a_group_of_tiles(ctx, pattern):
    msg, matches, words = ce.cw_group_message(pattern)
    assert words > ce.G
    parse = _Parse(ctx, len(msg))
    tape, strs, m = parse(msg)
    assert tape.numel() == words
    own, foreign = _own_and_foreign_counts(ctx, tape, strs, m, b"a", b"b")
    assert own == foreign == (1_100_000, matches)


# ---- KF3 -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", ce.KF3_ROWS)
def test_kf3_staged_segments(ctx, rows):
    """64 paths of 16 KiB segment bytes, 32-segment and empty paths, at rows where KF3's blocks hold one path, two, or
    many: every cell against fo.find (on the first rows of each template; the others are those rows moved)"""
    paths, kinds = ce.kf3_paths()
    tape, strs, msg, slots = ce.kf3_tape(rows)
    nt = min(rows, ce.KF3_TEMPLATES)
    first = fo.find(tape, strs, msg, paths, kinds, slots[:nt])
    want = [[None] * rows for _ in paths]
    for p in range(len(paths)):
        for r in range(rows):
            c = first[p][r % ce.KF3_TEMPLATES]
            shift = int(slots[r] - slots[r % ce.KF3_TEMPLATES])
            want[p][r] = ce.Cell(c.status, c.tag, c.index + shift if c.index >= 0 else -1, c.value)
    rc, n, cols = ctx.find_device(*_upload(tape, strs, msg), paths, kinds)
    assert rc == 0 and n == rows
    _check_cells(cols, want, kinds, range(rows), "kf3 rows=%d" % rows)


# ---- KF5 -----------------------------------------------------------------------------------------------------------
def test_kf5_mixed_lengths_and_row_stride(ctx):
    import torch
    tape, strs, msg, paths, kinds, want = ce.kf5_mixed()
    rows = len(want[0])
    d = _upload(tape, strs, msg)
    rc, n, cols = ctx.find_device(*d, paths, kinds)
    assert rc == 0 and n == rows
    strings = [p for p, k in enumerate(kinds) if k == ce.STRING]
    for s, p in enumerate(strings):
        lens = np.array([len(x) for x in want[s]])
        off = cols[p].offsets.cpu().numpy()
        assert np.array_equal(np.diff(off), lens) and bool((cols[p].status == ce.OK).all() or s == 2)
        assert cols[p].data[int(off[0]):int(off[-1])].cpu().numpy().tobytes() == b"".join(want[s])
    nb = int(cols[strings[-1]].offsets[-1])
    # the same into buffers with room behind the rows and the bytes: the stride is row_cap, nothing else is written
    cap = rows + 37
    P, S = len(paths), len(strings)
    out = (torch.full((P, cap), 0xA5, dtype=torch.uint8, device="cuda"), torch.full((P, cap), 0xA5, dtype=torch.uint8, device="cuda"),
           torch.full((P, cap), -7, dtype=torch.int64, device="cuda"), torch.full((P, cap), -7, dtype=torch.int64, device="cuda"),
           torch.full((S, cap + 1), -7, dtype=torch.int64, device="cuda"), torch.full((nb + 4096,), 0xA5, dtype=torch.uint8, device="cuda"))
    rc, n2, cols2 = ctx.find_device(*d, paths, kinds, out=out)
    assert rc == 0 and n2 == rows
    for a, b in zip(cols, cols2):
        for x, y in zip(a[:5], b[:5]):
            assert (x is None and y is None) or torch.equal(x.contiguous().view(torch.uint8), y.contiguous().view(torch.uint8))
    assert bool((out[0][:, rows:] == 0xA5).all() and (out[1][:, rows:] == 0xA5).all())
    assert bool((out[2][:, rows:] == -7).all() and (out[3][:, rows:] == -7).all() and (out[4][:, rows + 1:] == -7).all())
    assert torch.equal(out[5][:nb], cols[0].data[:nb]) and bool((out[5][nb:] == 0xA5).all())


def test_kf5_string_cells_past_a_group(ctx):
    """64 STRING paths x (G / 64 + 1) rows: the string offsets scan crosses a group of tiles"""
    import torch
    tape, strs, paths, slots, offs, lens = ce.kf5_group()
    rows, P = len(slots), len(paths)
    assert rows * P > ce.G
    rc, n, cols = ctx.find_device(*_upload(tape, strs, b""), paths, [ce.STRING] * P)
    assert rc == 0 and n == rows
    nk = len(ce.KF5_GROUP_KEYS)
    key = np.arange(P) % nk
    all_lens = lens[key].reshape(-1).astype(np.int64)           # path-major, the order of the scan
    want_off = np.concatenate([[0], np.cumsum(all_lens)])
    head = torch.from_numpy(slots + 4).cuda()
    for p in range(P):
        k = int(key[p])
        off = cols[p].offsets.cpu().numpy()
        assert np.array_equal(off, want_off[p * rows:(p + 1) * rows + 1]), p
        assert bool((cols[p].status == ce.OK).all()) and torch.equal(cols[p].index, head + 4 * k)
    data = cols[0].data[:int(want_off[-1])].cpu().numpy().tobytes()
    assert data == ce.gather(strs, np.concatenate([offs[k] for k in key]), all_lens)


# ---- conversions ---------------------------------------------------------------------------------------------------
def test_conversions_exact(ctx):
    et, specs = ce.conversion_tape()
    rc, rows, cols = ctx.find_device(*_upload(et.tape, et.strings, et.message), [[b"k"]] * len(ce.KINDS), list(ce.KINDS))
    assert rc == 0 and rows == len(specs)
    _check_cells(cols, et.cells, ce.KINDS, range(rows), "conversions")


# ---- own tape against foreign tape ---------------------------------------------------------------------------------
def _sample_messages():
    from tests import stage2_edge_docs as sd
    nd_items = {n for n, _, _ in sd.ND_ITEMS}
    docs = [d for d in sd.placed_docs(True, group=False) if d.ok and d.name.split(":")[1].split("@")[0] in nd_items]
    out = [(d.name, d.msg, True) for d in docs[::30]]
    out += [(d.name, d.msg, d.ndjson) for d in sd.record_docs()]
    out += [(d.name, d.msg, d.ndjson) for d in list(sd.leading_space_docs())[1::16]]
    out += list(ce.boundary_messages())
    return out


@pytest.mark.parametrize("impl", [0, 1])
def test_own_rows_equal_foreign_rows(ctx, oracle, impl):
    """find and countWhere on the tape a parse left (stage 2's root list) and on its copy (KC1): the same columns,
    byte for byte, and the same counts, in both stage-2 implementations with copy_strings on and off"""
    import torch
    msgs = _sample_messages()
    parse = _Parse(ctx, max(len(m) for _, m, _ in msgs) + 64)
    paths, kinds = [[b"k"], [b"z"], [b"k"], [b"r"]], [ce.STRING, ce.ELEMENT, ce.INT64, ce.ELEMENT]
    ctx.set_stage2_impl(impl)
    try:
        for name, msg, nd in msgs:
            msg = msg.strip(WS)
            orc, otape, ostrs, (off, ln) = oracle.parse(msg, ndjson=nd)
            want_roots = oracle.count_where(otape, ostrs, msg[off:off + ln], b"k", b"a")
            for copy in (True, False):
                tape, strs, m = parse(msg, ndjson=nd, copy=copy)
                rc, rows, own = ctx.find_device(tape, strs, m, paths, kinds)
                rc2, rows2, foreign = ctx.find_device(tape.clone(), strs, m, paths, kinds)
                assert rc == rc2 == 0 and rows == rows2 == want_roots[0], (name, copy, rows, rows2, want_roots)
                for a, b in zip(own, foreign):
                    for x, y in zip(a[:5], b[:5]):
                        assert (x is None and y is None) or torch.equal(x.contiguous().view(torch.uint8),
                                                                        y.contiguous().view(torch.uint8)), (name, copy)
                    if a.data is not None:
                        nb = int(a.offsets[-1])
                        assert torch.equal(a.data[:nb], b.data[:nb])
                own_c, foreign_c = _own_and_foreign_counts(ctx, tape, strs, m, b"k", b"a")
                assert own_c == foreign_c == want_roots, (name, copy)
    finally:
        ctx.set_stage2_impl(0)


# ---- the root list after a Deserialize -----------------------------------------------------------------------------
def test_deserialize_into_the_parse_tape_drops_its_root_list(ctx, oracle):
    """parse A into T, Deserialize a stream of B (same tape length, other roots) into T: find and countWhere on T see
    B's rows, not the root list the parse of A left"""
    import torch
    from tests import serialize_oracle as so
    a, b = b'{"a":"x"}\n{"a":"y"}', b'{"a":"x","b":"y","c":1}'
    rc, tb, sb, (off, ln) = oracle.parse(b, ndjson=False)
    ra, ta, _, _ = oracle.parse(a, ndjson=True)
    assert rc == ra == 0 and len(ta) == len(tb) == 16
    src = so.serialize(tb, sb, b[off:off + ln])
    tb = np.asarray(so.device_result(src)[0], dtype=np.uint64)   # Deserialize's tape of B: its strings in the message
    stream = torch.from_numpy(np.frombuffer(src, dtype=np.uint8).copy()).cuda()
    parse = _Parse(ctx, 4096)
    paths, kinds = [[b"a"], [b"b"], [b"c"]], [ce.STRING, ce.STRING, ce.INT64]
    for copy in (True, False):
        tape, _, _ = parse(a, copy=copy)
        assert tape.numel() == 16
        strs = torch.empty(64, dtype=torch.uint8, device="cuda")
        msg = torch.empty(64, dtype=torch.uint8, device="cuda")
        rc, sizes, views = ctx.deserialize_device(stream, tape=parse.tape, strings=strs, message=msg)
        assert rc == 0 and sizes[0] == 16
        assert torch.equal(parse.tape[:16].cpu(), torch.from_numpy(tb.view(np.int64)))
        rc, rows, cols = ctx.find_device(parse.tape[:16], views[1], views[2], paths, kinds)
        assert rc == 0 and rows == 1, (copy, rows)
        assert cols[0].index.tolist() == [4] and cols[2].value.tolist() == [1]
        o = cols[1].offsets.tolist()
        assert cols[1].data[o[0]:o[1]].cpu().numpy().tobytes() == b"y"
        assert _count(ctx, parse.tape, 16, views[1], views[2], b"b", b"y") == (1, 1)
