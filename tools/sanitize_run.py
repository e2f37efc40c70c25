"""Small end-to-end workload for `compute-sanitizer` (memcheck / racecheck / synccheck / initcheck): every kernel of
the path on inputs small enough for the tool's 10-100x slowdown, each result still checked against the oracle.
usage: compute-sanitizer --tool racecheck python tools/sanitize_run.py [quick]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
import numpy as np

import simdjson_b200 as sj
from oracle.pyoracle import Oracle
from tests.util import load_fixture, tricky_ndjson

quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
ctx = sj.Context(0)          # streaming stage 2 (default with copy_strings)
ctx_legacy = sj.Context(0)   # per-structural stage 2
ctx_legacy.set_stage2_impl(1)
o = Oracle("native")
n = 0


def same(msg, ndjson=False, copy=True):
    global n
    rc_o, tape_o, str_o, win_o = o.parse(msg, ndjson=ndjson, copy_strings=copy)
    for cx in (ctx, ctx_legacy):
        rc_g, tape_g, str_g, win_g = cx.parse(msg, ndjson=ndjson, copy_strings=copy)
        assert rc_g == rc_o and win_g == win_o, (rc_g, rc_o)
        if rc_o == 0:
            assert np.array_equal(tape_g, tape_o) and str_g == str_o
    ok_g, d_g = ctx.find_structural_indices(msg, ndjson)
    ok_o, d_o = o.find_structural_indices(msg, ndjson)
    assert ok_g == ok_o and (not ok_o or np.array_equal(d_g, d_o))
    n += 1


docs = ["twitter", "twitterescaped", "numbers", "apache_builds", "github_events"] if not quick else ["github_events"]
for name in docs:
    d = load_fixture(name).strip()
    same(d)
    same(d, copy=False)
pk = load_fixture("parking-citations").strip()
same(pk[:120000 if quick else len(pk)].rsplit(b"\n", 1)[0], ndjson=True)
nd, _ = tricky_ndjson()
same(nd, ndjson=True)
assert ctx.parse_count_where(nd, b"Make", b"HOND")[0] == 0
# the tape consumers' device entry points (tape.cuh) on the context's own tape (stage 2's root list) and on a copy of it
# (a foreign tape: KM1 + KC1a / KC1b)
import ctypes as C

import torch

from tests import find_oracle as fo
from tests.marshal_oracle import marshal
from tests.serialize_oracle import serialize

small = b"\n".join(pk.split(b"\n")[:40])
rc_o, tape_o, str_o, (off_o, len_o) = o.parse(small, ndjson=True)
d_msg = torch.full((len(small) + 4096,), 0x20, dtype=torch.uint8, device="cuda")
d_msg[:len(small)].copy_(torch.frombuffer(bytearray(small), dtype=torch.uint8))
tcap, scap, tl, sl = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
ctx.L.sj_bounds(len(small), C.byref(tcap), C.byref(scap))
d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
assert ctx.L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(small), 3, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                             d_str.data_ptr(), d_str.numel(), C.byref(sl)) == 0
own, strs, msg = d_tape[:tl.value], d_str[:sl.value], d_msg[:len(small)]
paths, kinds = [[b"Make"], [b"Fine"]], [fo.STRING, fo.ELEMENT]
win = small[off_o:off_o + len_o]
want_text, want_stream = marshal(tape_o, str_o, win), serialize(tape_o, str_o, win)
for tape in (own, own.clone()):
    rc, rows, cols = ctx.find_device(tape, strs, msg, paths, kinds)
    assert rc == 0 and rows == 40, (rc, rows)
    rc, _, text = ctx.marshal_device(tape, strs, msg)
    assert rc == 0 and text.cpu().numpy().tobytes() == want_text
    rc, _, stream = ctx.serialize_device(tape, strs, msg)
    assert rc == 0 and stream.cpu().numpy().tobytes() == want_stream
    rc, sizes, (t2, s2, m2) = ctx.deserialize_device(stream)
    assert rc == 0 and ctx.marshal_device(t2[:sizes[0]], s2[:sizes[1]], m2[:sizes[2]])[2].cpu().numpy().tobytes() == want_text
    n += 1
# the find's array rows (find_rows.cuh): KR1 .. KR8 and KF3 from elements, on the context's own tape and on the same
# tape passed as foreign, with a nop among the elements so that one record takes the one-thread walk
from tests import find_rows_oracle as fr

rdoc = b'{"a":[{"s":"x","n":[1,2]},3,{"s":"yz"},[1]]}\n{"a":[]}\n{"b":1}\n[{"s":"q"},true]'
rc_o, tape_r, str_r, (off_r, len_r) = o.parse(rdoc, ndjson=True)
rpaths, rkinds = [[b"s"], [b"n"], [b"s"]], [fo.STRING, 9, 7]
for rp in ([b"a"], []):
    want_r = fr.find_rows(tape_r, str_r, rdoc[off_r:off_r + len_r], rp, rpaths, rkinds)
    rc, N, R, index, _ = ctx.parse_find_rows(rdoc, rp, rpaths, rkinds)
    assert rc == 0 and index.row_index.tolist() == want_r[3], (rp, index.row_index, want_r[3])
    t_r = torch.from_numpy(tape_r.view(np.int64).copy()).cuda()
    s_r = torch.frombuffer(bytearray(str_r), dtype=torch.uint8).cuda()
    m_r = torch.frombuffer(bytearray(rdoc[off_r:off_r + len_r]), dtype=torch.uint8).cuda()
    rc, N, R, index, _ = ctx.find_rows_device(t_r, s_r, m_r, rp, rpaths, rkinds)
    assert rc == 0 and index.row_index.cpu().tolist() == want_r[3]
nop = tape_r.copy()
k = int(fr.find_rows(tape_r, str_r, b"", [b"a"], [], [])[3][1])  # the head of the element 3
nop[k], nop[k + 1] = (ord("N") << 56) | 1, 0  # a nop over the number: its record is walked by one thread
rc, N, R, index, _ = ctx.find_rows_device(torch.from_numpy(nop.view(np.int64).copy()).cuda(), s_r, m_r, [b"a"], rpaths, rkinds)
assert rc == 0 and ctx.find_rows_serial() == 1
# the find's member rows (KO1 .. KO4 with the array rows' passes), on the own tape and a foreign copy, with only_keys
# and with a nop between a key and its value so that one record takes the one-thread walk
from tests import find_members_oracle as fmo

for rp, only in (([b"a"], []), ([], [b"a", b"b"])):
    want_m = fmo.find_members(tape_r, str_r, rdoc[off_r:off_r + len_r], rp, [[]], [7], only)
    rc, N, R, index, _ = ctx.parse_find_members(rdoc, rp, [[]], [7], only)
    assert rc == 0 and index.row_index.tolist() == want_m[3], (rp, index.row_index, want_m[3])
    rc, N, R, index, _ = ctx.find_members_device(t_r, s_r, m_r, rp, [[]], [7], only)
    assert rc == 0 and index.row_index.cpu().tolist() == want_m[3]
mdoc = b'{"a":{"k":1,"s":"x"},"b":2}'
rc_o, tape_m, str_m, (off_m, len_m) = o.parse(mdoc)
nop = np.insert(tape_m, 7, np.uint64(ord("N") << 56))  # a nop between "k" and its value (skip 0)
scope = np.isin(nop >> np.uint64(56), [ord(c) for c in "r{}"]) & ((nop & np.uint64((1 << 56) - 1)) >= 7)
nop[scope] += np.uint64(1)
rc, N, R, index, _ = ctx.find_members_device(torch.from_numpy(nop.view(np.int64).copy()).cuda(),
                                             torch.frombuffer(bytearray(str_m), dtype=torch.uint8).cuda(),
                                             torch.frombuffer(bytearray(mdoc[off_m:off_m + len_m]), dtype=torch.uint8).cuda(),
                                             [b"a"], [[]], [1])
assert rc == 0 and R == 2 and ctx.find_rows_serial() == 1
# the S2 blocks of CompressFast (s2.cuh): KC1 / KC2 and KX1 / KX2 around the same calls
from tests import s2_oracle
ctx.set_compress_mode(1)
rc, _, stream = ctx.serialize_device(own, strs, msg)
assert rc == 0 and s2_oracle.inflate(stream.cpu().numpy().tobytes()) == want_stream
rc, sizes, (t2, s2, m2) = ctx.deserialize_device(stream)
assert rc == 0 and ctx.marshal_device(t2[:sizes[0]], s2[:sizes[1]], m2[:sizes[2]])[2].cpu().numpy().tobytes() == want_text
ctx.set_compress_mode(0)
# carries across slab / tile edges, long strings (warp-cooperative paths), dense brackets, number-heavy
g = (__import__("ctypes").c_uint32 * 4)()
ctx.L.sj_test_geometry(g)
slab, tile = int(g[2]), int(g[3])
for edge in (slab, tile):
    for run in (1, 33, 64):
        same(b'["' + b"x" * (edge - 2 - run // 2) + b"\\" * run + b'"q\\\\", "tail",true , 12]')
same(b'{"k":"' + b"s" * (tile + 77) + b'","t":[1,2,{"u":null}]}')
same(b'["' + b"\\u30c6\\u30b9\\ud83d\\ude00\\n" * 300 + b'","' + b"abc" * 200 + b'"]')
same(b"[" + b"[1," * 3000 + b"1" + b"]" * 3000 + b"]")
same(b"[" + b",".join(b"%d.%de%d" % (i, i * 7919 % 100000, i % 30 - 15) for i in range(4000)) + b"]")
same(b'{"a":tru}')
same(b'["abc\\q"]')
# the sharded ParseND with the exchange kernel over peer memory (exchange.cuh): two host threads = two ranks on this GPU
import threading

from simdjson_b200.parallel import ShardedParse, split_at_newlines, trimmed_window

stream = pk[:60000].rsplit(b"\n", 1)[0] + b'\n{"esc":"a\\u00e9\\n","n":[1,2.5,-3],"t":true}'
rc_o, tape_o, str_o, (off_o, len_o) = o.parse(stream, ndjson=True, copy_strings=True)
wins = [trimmed_window(stream, a, b) for a, b in split_at_newlines(stream, 2)]
cx = [sj.Context(0), sj.Context(0)]
for r, c in enumerate(cx):
    assert c.L.sj_exchange_create(c.h, r, 2, 1, None) == 0
    assert c.L.sj_exchange_set_timeout_ms(c.h, 120000) == 0
locs = (C.c_void_p * 2)(*[c.L.sj_exchange_local(c.h) for c in cx])
res = [None, None]


def rank(r):
    c = cx[r]
    a, b = wins[r]
    assert c.L.sj_exchange_connect_ptrs(c.h, locs) == 0
    assert c.L.sj_exchange_set_gap(c.h, wins[1][0] - b if r == 0 else 0) == 0
    dev = torch.device("cuda:0")
    d_msg = torch.full((b - a + 256,), 0x20, dtype=torch.uint8, device=dev)
    d_msg[: b - a] = torch.frombuffer(bytearray(stream[a:b]), dtype=torch.uint8).to(dev)
    torch.cuda.synchronize()
    sp = ShardedParse(c)
    rc, tot = sp.count(d_msg.data_ptr(), b - a, True)
    assert rc == 0, rc
    d_tape = torch.empty(tot[1] + 8, dtype=torch.int64, device=dev)
    d_str = torch.empty(tot[2] + 64, dtype=torch.uint8, device=dev)
    assert sp.emit(0, 0, 0, d_tape.data_ptr(), d_tape.numel(), d_str.data_ptr(), d_str.numel(), c.L.sj_exchange_bases(c.h)) == 0
    res[r] = (d_tape[: tot[1]].cpu().numpy().view(np.uint64), d_str[: tot[2]].cpu().numpy().tobytes())


ts = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
for t in ts:
    t.start()
for t in ts:
    t.join()
assert res[0] is not None and res[1] is not None
assert np.array_equal(np.concatenate([res[0][0], res[1][0]]), tape_o) and res[0][1] + res[1][1] == str_o
n += 1
print("sanitize_run ok: %d documents, %d kernel launches" % (n, ctx.launches()))
