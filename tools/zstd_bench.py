#!/usr/bin/env python3
"""Time the device Serializer in every compress mode -- CompressNone, CompressFast (S2 blocks, s2.cuh), CompressDefault
(zstd tags, S2 message and values) and CompressBest (zstd blocks, zstd.cuh) -- in the same run, and print one JSON
line per workload and mode.

Workloads: k0 (the parking-citations-shaped NDJSON batch sj_gen_ndjson_device generates, as in bench.py), twitter
("[" + twitter.json x K + "]") and canada ("[" + canada.json x K + "]").  Per workload the tape is parsed into HBM once;
per mode: sj_serialize_device and sj_deserialize_device of its stream (CUDA events around back-to-back calls after
warm-up), the stream's bytes, its size against the CompressNone stream, and the tags block against the same bytes
compressed by pyarrow's `zstd` at level 3 on the CPU (one frame).  Before timing, every compressed stream must
deserialize to the same tape and message as the NONE stream.  The card's name and power limit are read in the same run.

    python tools/zstd_bench.py [--mib 512] [--calls 5] [--warmup 2] [--only k0,twitter,canada] [--modes 0,1,2,3]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "simdjson-go_b200"), os.path.join(ROOT, "tools")]

from marshal_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=512)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="k0,twitter,canada")
    ap.add_argument("--modes", default="0,1,2,3")
    args = ap.parse_args()

    import pyarrow as pa
    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    from tests import s2_oracle as s2
    from tests.util import load_fixture

    assert sj.SupportedCPU(), "no sm_90 device: this benchmark measures the GPU only"
    name, plimit = card()
    dev = torch.device("cuda", 0)
    ctx = sj.Context(0)
    L = ctx.L
    ms = C.c_float(0)
    zstd3 = pa.Codec("zstd", compression_level=3)
    names = {0: "none", 1: "fast", 2: "default", 3: "best"}
    modes = [int(m) for m in args.modes.split(",")]

    def timed(fn, calls):
        L.sj_ctx_sync(ctx.h)
        L.sj_event_record(ctx.h, 0)
        for _ in range(calls):
            fn()
        L.sj_event_record(ctx.h, 1)
        L.sj_event_elapsed_ms(ctx.h, C.byref(ms))
        return ms.value / calls

    for wl in args.only.split(","):
        if wl == "k0":
            pk = load_fixture("parking-citations").strip()
            n_rec = (args.mib << 20) // (len(pk) // len(pk.split(b"\n")) + 1)
            d_msg = torch.full(((args.mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device=dev)
            glen = C.c_size_t(0)
            rc = L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d_msg.data_ptr(), d_msg.numel() - (1 << 16), C.byref(glen))
            assert rc == 0, rc
            n, flags = glen.value, _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS
            desc = "K0 gen_ndjson: %d parking-citations-shaped records, ParseND" % n_rec
        else:
            one = load_fixture(wl)
            k = max(1, (args.mib << 20) // (len(one) + 1))
            host_msg = b"[" + b",".join([one] * k) + b"]"
            n, flags = len(host_msg), _lib.FLAG_COPY_STRINGS
            d_msg = torch.full((n + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
            d_msg[:n].copy_(torch.frombuffer(bytearray(host_msg), dtype=torch.uint8))
            del host_msg
            desc = "'[' + %s.json x %d + ']', one document" % (wl, k)
        tcap, scap = C.c_size_t(0), C.c_size_t(0)
        L.sj_bounds(n, C.byref(tcap), C.byref(scap))
        tl, sl = C.c_size_t(0), C.c_size_t(0)
        d_tape = torch.empty(tcap.value, dtype=torch.int64, device=dev)
        d_str = torch.empty(max(scap.value, 1), dtype=torch.uint8, device=dev)
        rc = L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                               d_str.data_ptr(), d_str.numel(), C.byref(sl))
        assert rc == 0, rc
        tape, strs, msg = d_tape[:tl.value], d_str[:sl.value], d_msg[:n]

        none_blocks = None
        none_len = None
        for mode in [0] + [m for m in modes if m]:
            ctx.set_compress_mode(mode)
            rc, slen, stream = ctx.serialize_device(tape, strs, msg)
            assert rc == 0, rc
            rc, sizes, (t2, s2b, m2) = ctx.deserialize_device(stream)
            assert rc == 0 and sizes[0] == tape.numel()
            if mode == sj.CompressNone:
                none_result = (t2.clone(), m2.clone())
            else:
                assert torch.equal(t2, none_result[0]) and torch.equal(m2, none_result[1]), "round trip differs from NONE"
            olen, a, b_, c_ = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)

            def ser():
                assert L.sj_serialize_device(ctx.h, msg.data_ptr(), n, tape.data_ptr(), tape.numel(), strs.data_ptr(),
                                             strs.numel(), stream.data_ptr(), stream.numel(), C.byref(olen)) == 0

            def deser():
                assert L.sj_deserialize_device(ctx.h, stream.data_ptr(), slen, t2.data_ptr(), t2.numel(), C.byref(a),
                                               s2b.data_ptr() if s2b.numel() else None, s2b.numel(), C.byref(b_),
                                               m2.data_ptr(), m2.numel(), C.byref(c_)) == 0

            res = {}
            for key, fn in (("serialize", ser), ("deserialize", deser)):
                for _ in range(args.warmup):
                    fn()
                l0 = ctx.launches()
                res[key] = (timed(fn, args.calls), (ctx.launches() - l0) / args.calls)
            host = stream.cpu().numpy().tobytes()
            _, _, blocks = s2._blocks(host)
            row = {"workload": wl, "input": desc, "mode": names[mode], "input_bytes": n,
                   "stream_bytes": slen, "block_bytes": [len(d) for _, _, d in blocks[1:]],
                   "serialize_ms": round(res["serialize"][0], 3), "serialize_launches": res["serialize"][1],
                   "deserialize_ms": round(res["deserialize"][0], 3), "deserialize_launches": res["deserialize"][1]}
            if mode == sj.CompressNone:
                none_blocks, none_len = [d for _, _, d in blocks[1:]], slen
                tags3 = len(zstd3.compress(none_blocks[1], asbytes=True)) if none_blocks[1] else 0
            else:
                row.update({"ratio_vs_none": round(slen / none_len, 4), "tags_block_bytes": len(blocks[2][2]),
                            "pyarrow_zstd3_tags_bytes": tags3,
                            "tags_ratio_vs_pyarrow_zstd3": round(len(blocks[2][2]) / tags3, 4) if tags3 else None})
            row.update({"timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
                        "card": name, "power_limit_w": plimit})
            print(json.dumps(row), flush=True)
            del stream, t2, s2b, m2, host
        del none_result
        ctx.set_compress_mode(sj.CompressNone)
        del d_msg, d_tape, d_str
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
