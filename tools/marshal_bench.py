#!/usr/bin/env python3
"""Time MarshalJSON on the device (marshal.cuh) and print one JSON line per workload.

Workloads:
  ndjson   the parking-citations-shaped NDJSON batch K0 (sj_gen_ndjson_device) generates, as in bench.py's stream leg
  twitter  "[" + twitter.json x K + "]": one root, string-heavy
  canada   "[" + canada.json x K + "]": one root, float-heavy

Per workload: marshal time (CUDA events around back-to-back sj_marshal_device calls on a tape parsed into HBM, after
warm-up), the parse time of the same input the same way, output bytes, input GB/s, the algorithmic bytes of one call
over its time as a fraction of the H100 SXM data sheet's 3.35 TB/s, kernel launches per call, and the host-to-host rate
of sj_parse_marshal beside sj_parse's (host buffers both).  Every output is checked before it is timed: the text of the
replicated input must be the replicated text of one copy.  The card's name and power limit are read in the same run.

    python tools/marshal_bench.py [--mib 512] [--calls 10] [--warmup 3] [--only ndjson,twitter,canada]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "simdjson-go_b200")]

import numpy as np  # noqa: E402

HBM_PEAK_GBS = 3350.0  # H100 SXM data sheet (700 W)


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    name, limit = [x.strip() for x in out.split(",")]
    return name, float(limit)


def algorithmic_bytes(tape_words, strings_len, out_bytes):
    """Bytes one call has to move, from the pass structure of marshal.cuh: the tape is read by KM1..KM5; KM2 writes a
    32-bit depth per word that s2_min32, s2_ansv, KM3, KM4 and KM5 read; s2_ansv writes a 32-bit parent per word that
    KM3, KM4 and KM5 read; KM3 writes one bit per word that KM4 and KM5 read; KM4 and KM5 read the string bytes; KM5
    writes the text.  Scan and per-tile arrays (below 0.1 % of these) are left out."""
    n = tape_words
    tape = 5 * 8 * n
    scratch = 4 * n * (1 + 5) + 4 * n * (1 + 3) + (n / 8) * 3
    return tape + scratch + 2 * strings_len + out_bytes, {"tape_read": tape, "scratch": int(scratch),
                                                          "strings_read": 2 * strings_len, "output_written": out_bytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=512)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="ndjson,twitter,canada")
    args = ap.parse_args()

    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    from tests.util import load_fixture

    assert sj.SupportedCPU(), "no sm_90 device: this benchmark measures the GPU only"
    name, plimit = card()
    dev = torch.device("cuda", 0)
    ctx = sj.Context(0)
    L = ctx.L
    ms = C.c_float(0)

    def timed(fn, calls):
        L.sj_ctx_sync(ctx.h)
        L.sj_event_record(ctx.h, 0)
        for _ in range(calls):
            fn()
        L.sj_event_record(ctx.h, 1)
        L.sj_event_elapsed_ms(ctx.h, C.byref(ms))
        return ms.value / 1e3 / calls

    for wl in args.only.split(","):
        # ---- input and its expected text ----
        if wl == "ndjson":
            pk = load_fixture("parking-citations").strip()
            lines = pk.split(b"\n")
            n_rec = (args.mib << 20) // (len(pk) // len(lines) + 1)
            d_msg = torch.full(((args.mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device=dev)
            torch.cuda.synchronize()
            glen = C.c_size_t(0)
            rc = L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d_msg.data_ptr(), d_msg.numel() - (1 << 16), C.byref(glen))
            assert rc == 0, rc
            n = glen.value
            host_msg = d_msg[:n].cpu().numpy().tobytes()
            # record g = template line g mod 1000 with its 10 ticket digits at [11, 21) := g; the text keeps them there
            rc, tm = ctx.parse_marshal(pk, ndjson=True)
            mlines = tm.split(b"\n")
            assert rc == 0 and all(m[11:21] == l[11:21] for m, l in zip(mlines, lines))
            want = b"\n".join(mlines[g % 1000][:11] + b"%010d" % g + mlines[g % 1000][21:] for g in range(n_rec))
            flags = _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS
            desc = "K0 gen_ndjson: %d parking-citations-shaped records, ParseND, copy_strings" % n_rec
        else:
            one = load_fixture(wl)
            k = max(1, (args.mib << 20) // (len(one) + 1))
            host_msg = b"[" + b",".join([one] * k) + b"]"
            n = len(host_msg)
            d_msg = torch.full((n + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
            d_msg[:n].copy_(torch.frombuffer(bytearray(host_msg), dtype=torch.uint8))
            rc, m1 = ctx.parse_marshal(one)
            assert rc == 0
            want = b"[" + b",".join([m1] * k) + b"]"
            flags = _lib.FLAG_COPY_STRINGS
            desc = "'[' + %s.json x %d + ']', one document, copy_strings" % (wl, k)
        torch.cuda.synchronize()

        # ---- parse into HBM (timed too: the marshal's yardstick) ----
        tcap, scap = C.c_size_t(0), C.c_size_t(0)
        L.sj_bounds(n, C.byref(tcap), C.byref(scap))
        tl, sl = C.c_size_t(0), C.c_size_t(0)
        d_tape = torch.empty(tcap.value, dtype=torch.int64, device=dev)
        d_str = torch.empty(scap.value, dtype=torch.uint8, device=dev)

        def parse():
            r = L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                                  d_str.data_ptr(), d_str.numel(), C.byref(sl))
            assert r == 0, r

        for _ in range(args.warmup):
            parse()
        t_parse = timed(parse, args.calls)
        tape_words, strings_len = tl.value, sl.value

        # ---- marshal: checked, then timed ----
        d_out = torch.empty(len(want) + 64, dtype=torch.uint8, device=dev)
        olen = C.c_size_t(0)

        def marshal():
            r = L.sj_marshal_device(ctx.h, d_msg.data_ptr(), n, d_tape.data_ptr(), tape_words, d_str.data_ptr(), strings_len,
                                    d_out.data_ptr(), d_out.numel(), C.byref(olen))
            assert r == 0, r

        marshal()
        assert olen.value == len(want) and d_out[:olen.value].cpu().numpy().tobytes() == want, "marshal output differs"
        for _ in range(args.warmup):
            marshal()
        l0 = ctx.launches()
        t_m = timed(marshal, args.calls)
        launches = (ctx.launches() - l0) / args.calls
        alg, parts = algorithmic_bytes(tape_words, strings_len, len(want))

        # ---- host to host: sj_parse_marshal beside sj_parse ----
        h_in = torch.frombuffer(bytearray(host_msg), dtype=torch.uint8).pin_memory()
        h_out = torch.empty(len(want) + 64, dtype=torch.uint8).pin_memory()
        h_tape = torch.empty(tape_words + 64, dtype=torch.int64).pin_memory()
        h_str = torch.empty(strings_len + 64, dtype=torch.uint8).pin_memory()
        mo_, ml_ = C.c_size_t(0), C.c_size_t(0)

        def host_marshal():
            r = L.sj_parse_marshal(ctx.h, h_in.data_ptr(), n, flags, h_out.data_ptr(), h_out.numel(), C.byref(olen))
            assert r == 0 and olen.value == len(want), r

        def host_parse():
            r = L.sj_parse(ctx.h, h_in.data_ptr(), n, flags, h_tape.data_ptr(), h_tape.numel(), C.byref(tl), h_str.data_ptr(),
                           h_str.numel(), C.byref(sl), C.byref(mo_), C.byref(ml_))
            assert r == 0, r

        host_marshal()
        assert h_out[:len(want)].numpy().tobytes() == want, "sj_parse_marshal output differs"
        rates = {}
        for key, fn in (("parse_marshal", host_marshal), ("parse", host_parse)):
            fn()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            rates[key] = n / ((time.perf_counter() - t0) / args.calls) / 1e9

        print(json.dumps({
            "workload": wl, "input": desc, "input_bytes": n, "tape_words": tape_words, "strings_bytes": strings_len,
            "output_bytes": len(want), "output_per_input_byte": round(len(want) / n, 4),
            "marshal_ms": round(t_m * 1e3, 3), "marshal_input_gbs": round(n / t_m / 1e9, 2),
            "parse_ms": round(t_parse * 1e3, 3), "parse_input_gbs": round(n / t_parse / 1e9, 2),
            "algorithmic_bytes": int(alg), "algorithmic_parts": parts, "algorithmic_gbs": round(alg / t_m / 1e9, 1),
            "hbm_frac": round(alg / t_m / 1e9 / HBM_PEAK_GBS, 4), "hbm_peak": "H100 SXM data sheet 3.35 TB/s (700 W)",
            "launches_per_call": launches,
            "parse_marshal_host_gbs": round(rates["parse_marshal"], 3), "parse_host_e2e_gbs": round(rates["parse"], 3),
            "timer": "CUDA events around %d back-to-back calls after %d warm-up calls; host rates: wall clock, one context"
                     % (args.calls, args.warmup),
            "card": name, "power_limit_w": plimit}), flush=True)
        del d_msg, d_tape, d_str, d_out, h_in, h_out, h_tape, h_str, want, host_msg
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
