"""K2r's staged tape and its in-step links on the device, through the C ABI, against the oracle.

K2r stages a step's tape words in shared memory at the destination's 32-byte phase and copies them out in whole sectors
(a step that does not fit stores directly); bracket pairs and NDJSON records with both ends in one staged step are
linked there and skipped by K2e / K2f.  The inputs are the ones of the emulation's test_s2s_tape_staging_cpu.py, here
with the tape at 8 and 24 bytes past a 32-byte boundary, plus the sharded emit whose slices start at nonzero tape bases.
Every case also requires K2r's internal-error word to be 0."""
import ctypes as C

import numpy as np
import pytest

from tests.test_s2s_tape_staging_cpu import STEP, SLAB, _pad_to, capacity_targets, words_steps
from tests.util import load_fixture

pytestmark = pytest.mark.gpu


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


def _device_parse(ctx, msg, ndjson, offset):
    """sj_parse_device with d_tape `offset` bytes past a 32-byte boundary: (rc, tape, strings)"""
    import torch
    from simdjson_b200 import _lib
    dev = torch.device("cuda:0")
    n = len(msg)
    d_msg = torch.full((n + 256,), 0x20, dtype=torch.uint8, device=dev)
    if n:
        d_msg[:n] = torch.frombuffer(bytearray(msg), dtype=torch.uint8).to(dev)
    cap = 2 * n + 64
    raw = torch.zeros(cap + 8, dtype=torch.int64, device=dev)
    skip = ((offset - raw.data_ptr()) % 32) // 8
    d_tape = raw[skip:]
    assert d_tape.data_ptr() % 32 == offset
    d_str = torch.zeros(n + 64, dtype=torch.uint8, device=dev)
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    flags = (_lib.FLAG_NDJSON if ndjson else 0) | _lib.FLAG_COPY_STRINGS
    rc = ctx.L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), cap, C.byref(tl), d_str.data_ptr(), d_str.numel(),
                               C.byref(sl))
    torch.cuda.synchronize()
    return rc, d_tape[: tl.value].cpu().numpy().view(np.uint64), d_str[: sl.value].cpu().numpy().tobytes()


def _check(ctx, oracle, msg, ndjson=False, offsets=(8, 24)):
    rc_o, tape_o, str_o, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=True)
    win = bytes(msg[off:off + ln])
    for o in offsets:
        rc, tape, strs = _device_parse(ctx, win, ndjson, o)
        assert _internal(ctx) == 0, ("stage 1's and K2r's slab counts differ", o)
        assert (rc == 0) == (rc_o == 0), (rc, rc_o, o, bytes(msg[:60]))
        if rc_o == 0:
            assert len(tape) == len(tape_o)
            if not np.array_equal(tape, tape_o):
                bad = int(np.nonzero(tape != tape_o)[0][0])
                raise AssertionError("offset %d: tape differs at %d: %016x vs oracle %016x" % (o, bad, int(tape[bad]), int(tape_o[bad])))
            assert strs == str_o
    return rc_o


def test_step_words_around_the_staging_capacity(ctx, oracle_native):
    assert _check(ctx, oracle_native, words_steps(capacity_targets()), offsets=(0, 8, 16, 24)) == 0
    parts = [b"["]
    for s, w in enumerate(capacity_targets()):
        body = b"[]," * (w // 2) + (b"true," if w % 2 else b"")
        used = 1 if s == 0 else 0
        parts.append(body + b" " * (STEP - used - len(body)))
    assert _check(ctx, oracle_native, b"".join(parts) + b"0]", offsets=(0, 8, 16, 24)) == 0


def test_fixtures_at_unaligned_tape(ctx, oracle_native):
    for name in ("twitter", "canada", "citm_catalog", "github_events"):
        assert _check(ctx, oracle_native, load_fixture(name)) == 0
    pk = load_fixture("parking-citations").strip()
    assert _check(ctx, oracle_native, b"\n".join([pk] * 3), True) == 0


@pytest.mark.parametrize("edge", [STEP, SLAB, SLAB + STEP])
def test_bracket_pairs_inside_and_across_edges(ctx, oracle_native, edge):
    for d in range(-3, 4):
        _check(ctx, oracle_native, _pad_to(b'[{"a":[1,2]},[', edge + d) + b'3],{"b":{}}, [[]' + b" " * 40 + b"]]")
        _check(ctx, oracle_native, _pad_to(b'[{"k":[', edge - 2 + d) + b']}, {"m":[]}]')
    mid = b'{"x":[1,[2,[3]]]},' * ((2 * STEP) // 18 + 5)
    assert _check(ctx, oracle_native, _pad_to(b"[[", edge - 10) + mid + b"4]]") == 0
    assert _check(ctx, oracle_native, _pad_to(b"[", edge - 50) + b"[" * 200 + b"]" * 200 + b"]") == 0
    assert _check(ctx, oracle_native, _pad_to(b'{"o":{', edge - 30) + b",".join(b'"k%d":[%d]' % (i, i) for i in range(150)) + b"}}") == 0


def test_first_and_last_step(ctx, oracle_native):
    for n in (2, 10, STEP - 1, STEP, STEP + 1, SLAB + 1):
        _check(ctx, oracle_native, b"[" + b" " * max(0, n - 2) + b"]")
        _check(ctx, oracle_native, b"{}" + b"\n" * n + b"[1]", True)


@pytest.mark.parametrize("edge", [0, STEP, SLAB])
def test_invalid_brackets_fail_as_before(ctx, oracle_native, edge):
    for b in (b'[1,{"a":2]]', b'{"a":[1,2}', b'[1]]', b'{"a":1}}', b'[[[[1', b'{"a":{"b":[', b'[{]}', b'[1,{]', b'{[]}'):
        doc = _pad_to(b"[", edge) + b + b"]" if edge else b
        assert _check(ctx, oracle_native, doc, offsets=(8,)) != 0
        _check(ctx, oracle_native, b'{"a":1}\n' + b + b'\n{"b":2}', True, offsets=(8,))


def test_records_at_step_edges(ctx, oracle_native):
    rec = b'{"k":"v"}'
    for edge in (STEP, SLAB):
        for d in range(-2, 3):
            lead = _pad_to(b'{"a":"', edge - 2 + d) + b'"}'
            _check(ctx, oracle_native, lead + b"\n" + b"\n".join([rec] * 30), True)
            _check(ctx, oracle_native, lead + b" \n\n \n" + rec + b"\n\n\n" + b"\n".join([b"[]"] * 500) + b"\n", True)
    for doc in (b"1\n2\n", b"{}\n" * 3000, b"[1]\n" * 1000, b"{}\n\n\n\n" * 900 + b"[]", b'{"a":[1,{"b":2}]}\n' * 600):
        _check(ctx, oracle_native, doc, True)


@pytest.mark.parametrize("copy", [True, False])
def test_sharded_emit_at_nonzero_tape_base(ctx, oracle_native, copy):
    """two shards written into ONE tape buffer end to end, so the second starts at a nonzero tape base and at whatever
    32-byte phase the first one's length leaves"""
    import torch
    import simdjson_b200 as sj
    from simdjson_b200.parallel import ShardedParse, split_at_newlines, trimmed_window
    pk = load_fixture("parking-citations").strip()
    stream = b"\n".join([pk] * 3) + b"\n\n" + b'{"n":[1,[2,{}]],"t":true}\n' * 200 + pk[:20000].rsplit(b"\n", 1)[0]
    rc, tape_o, str_o, (off_o, _) = oracle_native.parse(stream, ndjson=True, copy_strings=copy)
    assert rc == 0
    dev = torch.device("cuda:0")
    shards = []
    for a, b in split_at_newlines(stream, 2):
        a, b = trimmed_window(stream, a, b)
        c = sj.Context(0)
        d_msg = torch.full((b - a + 256,), 0x20, dtype=torch.uint8, device=dev)
        d_msg[: b - a] = torch.frombuffer(bytearray(stream[a:b]), dtype=torch.uint8).to(dev)
        shards.append((c, ShardedParse(c), d_msg, a, b))
    for lead in (1, 3):  # the whole tape 8 / 24 bytes past a 32-byte boundary
        ranks = []
        for c, sp, d_msg, a, b in shards:  # (an emit consumes its count)
            rc, tot = sp.count(d_msg.data_ptr(), b - a, copy)
            assert rc == 0
            ranks.append((c, sp, d_msg, a, tot))
        words = sum(t[4][1] for t in ranks)
        raw = torch.zeros(words + 8, dtype=torch.int64, device=dev)
        skip = ((8 * lead - raw.data_ptr()) % 32) // 8
        d_tape = raw[skip:]
        d_str = torch.zeros(sum(t[4][2] for t in ranks) + 64, dtype=torch.uint8, device=dev)
        tb = sb = 0
        for c, sp, d_msg, a, tot in ranks:
            assert sp.emit(a - off_o, tb, sb, d_tape.data_ptr() + 8 * tb, tot[1], d_str.data_ptr() + sb, tot[2] + 64) == 0
            tb += tot[1]
            sb += tot[2]
        torch.cuda.synchronize()
        got = d_tape[:words].cpu().numpy().view(np.uint64)
        assert len(got) == len(tape_o)
        assert np.array_equal(got, tape_o), int(np.nonzero(got != tape_o)[0][0])
        assert d_str[:sb].cpu().numpy().tobytes() == str_o
    for c, *_ in shards:
        c.close()
