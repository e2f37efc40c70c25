"""GPU parity tests for the device-side tape consumers (consume.cuh, SURVEY.md 8(f)):
countWhere / countObjects (ndjson_test.go:421-474, Object.FindKey parsed_object.go:97-140) evaluated on
the tape in HBM, against the oracle's restatement on the oracle's tape and the reference's golden
(ndjson_test.go:250-266: 1000 roots, Make == HOND 116 times)."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def test_golden_make_hond(ctx):
    g = golden("G18_G19_fixtures")["parking_citations"]
    msg = load_fixture("parking-citations")
    for copy in (True, False):
        assert ctx.parse_count_where(msg, b"Make", b"HOND", copy_strings=copy) == (0, g["roots"], g["make_hond"])
    # a single document is one root
    assert ctx.parse_count_where(b' {"Make":"HOND"} ', b"Make", b"HOND", ndjson=False) == (0, 1, 1)
    assert ctx.parse_count_where(b'[{"Make":"HOND"}]', b"Make", b"HOND", ndjson=False) == (0, 1, 0)


def test_tricky_records_vs_oracle(ctx, oracle):
    nd, recs = tricky_ndjson()
    for copy in (True, False):
        rc, tape, strs, (off, ln) = oracle.parse(nd, ndjson=True, copy_strings=copy)
        assert rc == 0
        for key, value in ((b"Make", b"HOND"), (b"Make", b""), (b"", b""), (b"Make", b"TOYT"), (b"x", b"1"), (b"a", b"")):
            want = oracle.count_where(tape, strs, nd[off:off + ln], key, value)
            assert ctx.parse_count_where(nd, key, value, copy_strings=copy) == (0,) + want, (key, value, copy)


def test_errors_and_empty(ctx):
    assert ctx.parse_count_where(b'{"a":1}\n{"b":\n', b"a", b"1")[0] == 1      # stage-1 failure, like sj_parse
    assert ctx.parse_count_where(b'{"a":1}\n{"b" 2}\n', b"a", b"1")[0] == 2     # stage-2 failure
    assert ctx.parse_count_where(b"  \n ", b"a", b"1")[0] == 1


@pytest.mark.parametrize("copies", [40, 700])
def test_replicated_stream(ctx, oracle_native, copies):
    """size-independent property: k copies of the fixture give k x the golden counts; every fixture key/value
    pair agrees with the oracle's walk of the oracle's tape"""
    pk = load_fixture("parking-citations").strip()
    nd = b"\n".join([pk] * copies)
    assert ctx.parse_count_where(nd, b"Make", b"HOND") == (0, 1000 * copies, 116 * copies)
    if copies <= 40:
        rc, tape, strs, (off, ln) = oracle_native.parse(nd, ndjson=True)
        assert rc == 0
        for key, value in ((b"Color", b"BK"), (b"RP State Plate", b"CA"), (b"Violation code", b"80.69BS"),
                           (b"Ticket number", b"1103341116"), (b"nope", b"x")):
            want = oracle_native.count_where(tape, strs, nd[off:off + ln], key, value)
            assert ctx.parse_count_where(nd, key, value) == (0,) + want, key


def test_foreign_device_tape(ctx, oracle):
    """sj_count_where_device on a tape this context did not build: roots are found on the device (KC1)"""
    import torch
    nd, _ = tricky_ndjson()
    pk = load_fixture("parking-citations").strip()
    for msg, copy in ((nd, True), (nd, False), (pk, True), (b"\n".join([pk] * 9), True)):
        rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=True, copy_strings=copy)
        assert rc == 0
        d_tape = torch.from_numpy(tape.view(np.int64).copy()).cuda()
        d_strs = torch.from_numpy(np.frombuffer(strs + b"\0", dtype=np.uint8).copy()).cuda()
        d_msg = torch.from_numpy(np.frombuffer(msg[off:off + ln] + b"\0", dtype=np.uint8).copy()).cuda()
        torch.cuda.synchronize()
        for key, value in ((b"Make", b"HOND"), (b"Make", b"TOYT"), (b"", b"")):
            roots, matches = C.c_uint64(0), C.c_uint64(0)
            rc = ctx.L.sj_count_where_device(ctx.h, d_msg.data_ptr(), d_tape.data_ptr(), len(tape), d_strs.data_ptr(), key,
                                             len(key), value, len(value), C.byref(roots), C.byref(matches))
            assert rc == 0
            assert (roots.value, matches.value) == oracle.count_where(tape, strs, msg[off:off + ln], key, value)
    launches = ctx.launches()
    assert launches > 0


def test_gen_ndjson_kernel(ctx):
    """K0 gen_ndjson (SURVEY.md 8d, S3): record g = template line g mod 1000 with Ticket := g, zero padded, joined by
    newlines -- byte for byte what this Python restatement builds, for a window that starts far into the stream"""
    import ctypes as C
    import torch
    pk = load_fixture("parking-citations").strip()
    lines = pk.split(b"\n")
    assert len(lines) == 1000
    for first, n in ((0, 2500), (1_234_567_000, 3001), (9_999_999_000, 1000 + 17)):
        want = b"\n".join(l[:11] + b"%010d" % ((first + i) % 10**10) + l[21:] for i, l in ((i, lines[(first + i) % 1000]) for i in range(n)))
        d_out = torch.zeros(len(want) + 64, dtype=torch.uint8, device="cuda:0")
        glen = C.c_size_t(0)
        rc = ctx.L.sj_gen_ndjson_device(ctx.h, pk, len(pk), first, n, d_out.data_ptr(), d_out.numel(), C.byref(glen))
        assert rc == 0 and glen.value == len(want), (rc, glen.value, len(want))
        got = d_out[: glen.value].cpu().numpy().tobytes()
        assert got == want
    # and the generated stream parses
    rc, roots, matches = ctx.parse_count_where(got, b"Make", b"HOND")
    assert rc == 0 and roots == 1017
