#!/usr/bin/env python3
"""Time the device Serializer with uncompressed blocks (CompressNone) and with S2 blocks (CompressFast, s2.cuh) in the
same run, and print one JSON line per workload and mode.

Workloads: k0 (the parking-citations-shaped NDJSON batch sj_gen_ndjson_device generates, as in bench.py), twitter
("[" + twitter.json x K + "]") and canada ("[" + canada.json x K + "]").  Per workload the tape is parsed into HBM once;
per mode: sj_serialize_device and sj_deserialize_device of its stream (CUDA events around back-to-back calls after
warm-up), the stream's bytes, its size against the CompressNone stream, and -- FAST only -- against the same blocks
compressed by pyarrow's `snappy` on the CPU with the same 64 KiB chunking.  Before timing, the FAST stream must
deserialize to the same tape and message as the NONE stream.  The card's name and power limit are read in the same run.

    python tools/s2_bench.py [--mib 512] [--calls 5] [--warmup 2] [--only k0,twitter,canada]
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
    snappy = pa.Codec("snappy")

    def timed(fn, calls):
        L.sj_ctx_sync(ctx.h)
        L.sj_event_record(ctx.h, 0)
        for _ in range(calls):
            fn()
        L.sj_event_record(ctx.h, 1)
        L.sj_event_elapsed_ms(ctx.h, C.byref(ms))
        return ms.value / calls

    def snappy_len(data):
        if not data:
            return 0
        return len(s2.IDENT) + sum(8 + min(len(snappy.compress(data[a:a + s2.CHUNK], asbytes=True)), len(data[a:a + s2.CHUNK]))
                                   for a in range(0, len(data), s2.CHUNK))

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
        for mode in (sj.CompressNone, sj.CompressFast):
            ctx.set_compress_mode(mode)
            rc, slen, stream = ctx.serialize_device(tape, strs, msg)
            assert rc == 0, rc
            rc, sizes, (t2, s2b, m2) = ctx.deserialize_device(stream)
            assert rc == 0 and sizes[0] == tape.numel()
            if mode == sj.CompressNone:
                none_result = (t2.clone(), m2.clone())
            else:
                assert torch.equal(t2, none_result[0]) and torch.equal(m2, none_result[1]), "FAST round trip differs from NONE"
                del none_result
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
            row = {"workload": wl, "input": desc, "mode": "fast" if mode else "none", "input_bytes": n,
                   "stream_bytes": slen, "block_bytes": [len(d) for _, _, d in blocks[1:]],
                   "serialize_ms": round(res["serialize"][0], 3), "serialize_launches": res["serialize"][1],
                   "deserialize_ms": round(res["deserialize"][0], 3), "deserialize_launches": res["deserialize"][1]}
            if mode == sj.CompressNone:
                none_blocks, none_len = [d for _, _, d in blocks[1:]], slen
            else:
                ref = [snappy_len(d) for d in none_blocks]
                row.update({"ratio_vs_none": round(slen / none_len, 4), "pyarrow_snappy_block_bytes": ref,
                            "block_ratio_vs_pyarrow_snappy": [round(len(d) / r, 4) if r else None for (_, _, d), r in zip(blocks[1:], ref)]})
            row.update({"timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
                        "chunk_bytes": s2.CHUNK, "card": name, "power_limit_w": plimit})
            print(json.dumps(row), flush=True)
            del stream, t2, s2b, m2, host
        ctx.set_compress_mode(sj.CompressNone)
        del d_msg, d_tape, d_str
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
