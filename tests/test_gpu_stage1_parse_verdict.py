"""Stage 1's verdict in parse mode (K1 with PARSE: the stage 1 of every copy_strings parse through the streaming stage 2)
at its lane, step, slab, tile and grid-round edges, against the oracle's.

The documents come from tests/stage1_verdict_docs.py (their intentions are checked by test_stage1_verdict_docs_cpu.py):
control characters inside and just outside strings opened near the byte or a slab, tile or grid round in front of it,
unterminated strings and backslash runs at the message's end, the last structural far from the end, invalid escapes
with and without a control character in an earlier or later tile, and the accepted twins of all of them.  Every
document goes through the streaming parse; the ones below one tile also through the per-structural stage 2 (copy off,
and copy on with implementation 1, in the first NDJSON mode of the family), whose stage 1 is K1's index mode: the two
modes must not disagree.  The grid round is
the library's own (sj_test_stage1_ctas), so the round edges sit where this device puts them.

sj_parse_device may read up to round_up(len, 16) and is handed buffers readable well past it: a hostile pattern of
quotes, backslashes, brackets and control characters behind `len` must change nothing, at every residue of len mod 16."""
import ctypes as C
import time
import zlib

import numpy as np
import pytest

import tests.stage1_verdict_docs as V
from tests.test_stage1_verdict_docs_cpu import RC

pytestmark = pytest.mark.gpu

HOSTILE = b'"\\{[\x01\n'          # behind the message, at every phase
TAPE_CAP = 1 << 20                # tape words for sj_parse_device (the documents have few structurals)


@pytest.fixture(scope="module")
def ctxs():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    out = {}
    for impl in (0, 1):
        c = sj.Context(0)
        c.set_stage2_impl(impl)
        out[impl] = c
    yield out
    for c in out.values():
        c.close()


@pytest.fixture(scope="module")
def grid_round(ctxs):
    ctas = C.c_uint32(0)
    assert ctxs[0].L.sj_test_stage1_ctas(ctxs[0].h, C.byref(ctas)) == 0
    assert 1 <= ctas.value <= 1024, ctas.value
    print("stage 1 grid: %d CTAs, grid round %d bytes" % (ctas.value, ctas.value * V.TILE))
    return ctas.value * V.TILE


@pytest.fixture(scope="module")
def canvas(grid_round):
    return V.canvas(grid_round)


def _internal(ctx):
    w = C.c_uint32(0xFFFFFFFF)
    assert ctx.L.sj_test_stage2_internal(ctx.h, C.byref(w)) == 0
    return w.value


def _same(got, want, what):
    rc_g, tape_g, str_g, win_g = got
    rc_o, tape_o, str_o, win_o = want
    assert rc_g == rc_o, (what, rc_g, rc_o)
    if rc_o == 0:
        assert win_g == win_o, what
        if not np.array_equal(tape_g, tape_o):
            bad = int(np.nonzero(tape_g != tape_o)[0][0]) if len(tape_g) == len(tape_o) else -1
            raise AssertionError("%s: tape differs at %d" % (what, bad))
        assert str_g == str_o, what


def _modes(d):
    """every mode the family applies in; past one tile one of them, in turn, to keep the file's time"""
    if len(d.msg) <= V.TILE:
        return d.modes
    return [d.modes[zlib.crc32(d.name.encode()) % len(d.modes)]]


@pytest.mark.parametrize("gen", ["inside_outside_docs", "unterminated_docs", "last_structural_docs", "escape_docs"])
def test_parse_mode_verdict(ctxs, oracle_native, grid_round, canvas, gen):
    t0, n, per = time.time(), 0, {}
    for d in getattr(V, gen)(grid_round, canvas):
        for nd in _modes(d):
            want = oracle_native.parse(d.msg, ndjson=nd, copy_strings=True)
            assert want[0] == RC[d.verdicts[nd]], (d.name, nd, want[0])
            _same(ctxs[0].parse(d.msg, ndjson=nd, copy_strings=True), want, (d.name, nd, "parse mode"))
            if want[0] == 0:
                assert _internal(ctxs[0]) == 0, d.name
            if len(d.msg) <= V.TILE and nd == d.modes[0]:   # index mode (the per-structural stage 2): the same verdict
                assert ctxs[0].parse(d.msg, ndjson=nd, copy_strings=False)[0] == want[0], (d.name, nd, "copy off")
                _same(ctxs[1].parse(d.msg, ndjson=nd, copy_strings=True), want, (d.name, nd, "impl 1"))
            n += 1
        key = (d.family, d.edge[0])
        per[key] = per.get(key, 0) + 1
    print("%s: %d parses in %.1f s; documents per (family, edge): %s" % (gen, n, time.time() - t0, sorted(per.items())))
    assert n > 300


# ---- a hostile tail behind the message (sj_parse_device) ----------------------------------------------------------------
class _Device:
    """one message buffer (the message at a 16-byte aligned offset, `HOSTILE` behind it), tape and Strings.B"""

    def __init__(self, cap):
        import torch
        self.torch = torch
        dev = torch.device("cuda:0")
        self.base = 256
        self.buf = torch.empty(cap + self.base + 8192, dtype=torch.uint8, device=dev)
        self.tape = torch.empty(TAPE_CAP, dtype=torch.int64, device=dev)
        self.str = torch.empty(cap + 64, dtype=torch.uint8, device=dev)
        self.pattern = np.frombuffer(HOSTILE * (4096 // len(HOSTILE) + 2), dtype=np.uint8)

    def load(self, msg, phase):
        n = len(msg)
        host = np.concatenate([msg, self.pattern[phase:phase + 4096]])
        self.buf[self.base:self.base + n + 4096].copy_(self.torch.from_numpy(host))
        assert (self.buf.data_ptr() + self.base) % 16 == 0

    def parse(self, ctx, n, nd):
        from simdjson_b200 import _lib
        flags = _lib.FLAG_COPY_STRINGS | (_lib.FLAG_NDJSON if nd else 0)
        tl, sl = C.c_size_t(0), C.c_size_t(0)
        rc = ctx.L.sj_parse_device(ctx.h, self.buf.data_ptr() + self.base, n, flags, self.tape.data_ptr(), TAPE_CAP,
                                   C.byref(tl), self.str.data_ptr(), self.str.numel(), C.byref(sl))
        self.torch.cuda.synchronize()
        assert rc != _lib.ERR_CAPACITY, (n, tl.value, sl.value)
        if rc != 0:
            return rc, None, None, (0, n)
        tape = self.tape[:tl.value].cpu().numpy().view(np.uint64)
        return rc, tape, self.str[:sl.value].cpu().numpy().tobytes(), (0, n)


def _tail_check(ctxs, oracle, dev, msg, modes, phase, what):
    dev.load(msg, phase)
    for nd in modes:
        want = oracle.parse(msg, ndjson=nd, copy_strings=True)
        assert want[3] == (0, len(msg)), what            # nothing to trim: the device parse sees the same window
        for impl in (0, 1):
            _same(dev.parse(ctxs[impl], len(msg), nd), want, (what, nd, impl, phase))


def test_hostile_tail_documents(ctxs, oracle_native, grid_round, canvas):
    """a sample of every family at every edge kind (offsets -1 and 0; every fourth document of a family and edge kind,
    every sixth at the round edges, every sixteenth at the block edges) through sj_parse_device, with the pattern behind
    it at a phase that turns with the document"""
    dev = _Device(len(canvas.a))
    n, kinds, seen = 0, set(), {}
    try:
        for i, d in enumerate(V.all_docs(grid_round, canvas)):
            kind, E = d.edge
            if kind != "end" and d.pos - E not in (-1, 0):
                continue
            k = seen[(d.family, kind)] = seen.get((d.family, kind), -1) + 1
            if k % (16 if kind == "block" else 6 if kind == "round" else 4):
                continue
            _tail_check(ctxs, oracle_native, dev, d.msg, _modes(d), i % len(HOSTILE), d.name)
            kinds.add((d.family, kind))
            n += 1
    finally:
        del dev
    print("hostile tail: %d documents" % n)
    assert {(f, k) for f in V.FAMILIES for k in V.EDGE_KINDS} <= kinds, sorted(kinds)


def test_hostile_tail_every_residue(ctxs, oracle_native):
    """len at every residue mod 16 around a slab and a tile edge: an array closed at len - 1, a string that ends there,
    and one left open; every phase of the pattern, so the bytes up to round_up(len, 16) hold a quote, a backslash and
    a control character in turn"""
    dev = _Device(2 * V.TILE)
    n = 0
    try:
        for E in (V.SLAB, V.TILE):
            for ln in range(E - 8, E + 8):
                shapes = []
                m = np.full(ln, 0x20, dtype=np.uint8)
                m[:4] = np.frombuffer(b"[1,2", dtype=np.uint8)
                m[-1] = ord("]")
                shapes.append(m)
                m = np.full(ln, ord("a"), dtype=np.uint8)
                m[:2] = np.frombuffer(b'["', dtype=np.uint8)
                m[-2:] = np.frombuffer(b'"]', dtype=np.uint8)
                shapes.append(m)
                m = m.copy()
                m[-2:] = ord("a")
                shapes.append(m)
                for m in shapes:
                    for phase in range(len(HOSTILE)):
                        _tail_check(ctxs, oracle_native, dev, m, (False, True), phase, ("residue", ln, phase))
                        n += 1
    finally:
        del dev
    assert n == 2 * 16 * 3 * len(HOSTILE)
