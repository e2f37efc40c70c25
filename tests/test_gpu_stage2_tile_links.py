"""K2t on the device (csrc/s2s_tile.h: K2t-min + K2t-link), through the C ABI, against the oracle: the documents of
stage2_tile_docs.py -- bracket counts at the tile edges, pairs across them, partners several tiles back, nesting deeper
than a tile, NDJSON records over tile edges with and without K2r's in-step links, broken input at the edges -- with the
tape at two 32-byte phases, and the sharded emit of two ranks with tile edges inside each shard.  Tape and Strings.B
must equal the oracle's bit for bit, the return code must be the oracle's, and K2r's internal-error word 0."""
import numpy as np
import pytest

from tests import stage2_tile_docs as TD
from tests.test_gpu_tape_staging import _device_parse, _internal

pytestmark = pytest.mark.gpu

DOCS = TD.all_docs()


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("d", DOCS, ids=[d.name for d in DOCS])
def test_tile_edges(ctx, oracle_native, d):
    rc_o, tape_o, str_o, (off, ln) = oracle_native.parse(d.msg, ndjson=d.ndjson, copy_strings=True)
    if "ok" in d.want:
        assert (rc_o == 0) == d.want["ok"], d.name
    win = bytes(d.msg[off:off + ln])
    for o in (8, 24):
        rc, tape, strs = _device_parse(ctx, win, d.ndjson, o)
        assert _internal(ctx) == 0, (d.name, o)
        assert rc == rc_o, (d.name, o, rc, rc_o)
        if rc_o == 0:
            assert len(tape) == len(tape_o), d.name
            if not np.array_equal(tape, tape_o):
                bad = int(np.nonzero(tape != tape_o)[0][0])
                raise AssertionError("%s offset %d: tape differs at %d: %016x vs oracle %016x" % (d.name, o, bad, int(tape[bad]), int(tape_o[bad])))
            assert strs == str_o, d.name


def test_sharded_emit_with_tile_edges_in_each_shard(ctx, oracle_native):
    """two ranks, each shard over several K2t tiles (records short and longer than a step, one over several tiles),
    written into ONE tape at nonzero bases"""
    import torch
    import simdjson_b200 as sj
    from simdjson_b200.parallel import ShardedParse, split_at_newlines, trimmed_window
    nd = {d.name: d.msg for d in TD.ndjson_docs()}
    stream = nd["nd-mixed"] + b"\n" + nd["nd-long"] + b"\n" + nd["nd-record-over-tiles"] + b"\n" + nd["nd-short-lead3"]
    rc, tape_o, str_o, (off_o, _) = oracle_native.parse(stream, ndjson=True, copy_strings=True)
    assert rc == 0
    dev = torch.device("cuda:0")
    ranks = []
    for a, b in split_at_newlines(stream, 2):
        a, b = trimmed_window(stream, a, b)
        assert TD._count(stream[a:b]) > 2 * TD.T
        c = sj.Context(0)
        d_msg = torch.full((b - a + 256,), 0x20, dtype=torch.uint8, device=dev)
        d_msg[: b - a] = torch.frombuffer(bytearray(stream[a:b]), dtype=torch.uint8).to(dev)
        sp = ShardedParse(c)
        rc, tot = sp.count(d_msg.data_ptr(), b - a, True)
        assert rc == 0
        ranks.append((c, sp, d_msg, a, tot))
    words = sum(t[4][1] for t in ranks)
    d_tape = torch.zeros(words + 8, dtype=torch.int64, device=dev)
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
    for c, *_ in ranks:
        c.close()
