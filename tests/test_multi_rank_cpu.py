"""World-size-2 gloo test of the N > 1 path's host logic (CPU only): newline-aligned
sharding, the 3-integer all_gather, and tape rebasing.  Shards are parsed with the CPU oracle
here (no GPU needed); on GPUs the same code runs over NCCL in bench.py."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, copy, outdir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
    import torch.distributed as dist
    from oracle.pyoracle import Oracle
    from simdjson_b200.parallel import exchange_totals, rebase_shard_tape, split_at_newlines
    from tests.util import load_fixture
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    stream = load_fixture("parking-citations").strip()
    a, b = split_at_newlines(stream, world)[rank]
    o = Oracle("native")
    rc, tape, strings, (off, ln) = o.parse(stream[a:b], ndjson=True, copy_strings=copy)
    assert rc == 0
    base, totals = exchange_totals((b - a, len(tape), len(strings)))
    assert base[0] == a and len(totals) == world
    reb = rebase_shard_tape(tape, base[1], base[2], a + off)
    # tape consumers over a sharded stream: per-shard countWhere, one all_reduce of two integers
    from simdjson_b200.parallel import reduce_counts
    roots, matches = o.count_where(tape, strings, stream[a + off:a + off + ln], b"Make", b"HOND")
    assert reduce_counts((roots, matches)) == (1000, 116)  # ndjson_test.go:263
    np.save(os.path.join(outdir, "tape%d.npy" % rank), reb)
    with open(os.path.join(outdir, "str%d.bin" % rank), "wb") as f:
        f.write(strings)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("copy", [True, False])
def test_two_rank_sharded_parse_equals_whole(tmp_path, oracle_native, copy):
    import torch.multiprocessing as mp
    from tests.util import load_fixture
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, copy, str(tmp_path)), nprocs=world, join=True)
    stream = load_fixture("parking-citations").strip()
    rc, tape, strings, _ = oracle_native.parse(stream, ndjson=True, copy_strings=copy)
    assert rc == 0
    got = np.concatenate([np.load(tmp_path / ("tape%d.npy" % r)) for r in range(world)])
    gstr = b"".join(open(tmp_path / ("str%d.bin" % r), "rb").read() for r in range(world))
    assert np.array_equal(got, tape)
    assert gstr == strings


def test_stream_chunker_is_newline_aligned():
    """host logic of ParseNDStream (simdjson_amd64.go:157-174): chunks end at a record boundary"""
    import io
    sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
    from simdjson_b200.stream import _chunks
    recs = [b'{"i":%d,"pad":"%s"}' % (i, b"x" * (i % 97)) for i in range(5000)]
    stream = b"\n".join(recs)
    for size in (100, 1000, 4096, 1 << 20):
        parts = list(_chunks(io.BytesIO(stream), size))
        assert b"".join(parts) == stream
        assert all(p.endswith(b"\n") for p in parts[:-1])
    assert list(_chunks(io.BytesIO(b""), 10)) == []


def test_split_at_newlines_covers_and_aligns():
    sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
    from simdjson_b200.parallel import split_at_newlines
    buf = b"\n".join(b'{"i":%d}' % i for i in range(1000))
    for world in (1, 2, 3, 4, 8):
        parts = split_at_newlines(buf, world)
        assert parts[0][0] == 0 and parts[-1][1] == len(buf)
        for (a, b), (c, d) in zip(parts, parts[1:]):
            assert b == c and (b == len(buf) or buf[b - 1:b] == b"\n")


def test_bench_reference_arm_prints_the_contract_line():
    """bench.py --impl reference (the CPU arm the GPU line is compared with) runs without a GPU and prints one
    JSON line with the contract's keys"""
    import json
    import subprocess
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in line, k
    assert line["impl"] == "reference" and line["value"] > 0 and line["unit"] == "GB/s"
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["d2h_bytes_per_step"] == 0
