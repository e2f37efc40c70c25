#!/usr/bin/env python3
"""Time the device Serializer (serialize.cuh) and print one JSON line per workload.

Workloads:
  ndjson   the parking-citations-shaped NDJSON batch K0 (sj_gen_ndjson_device) generates, as in bench.py's stream leg
  twitter  "[" + twitter.json x K + "]": one root, string-heavy

Per workload, with the tape parsed into HBM: the time of sj_serialize_device and of sj_deserialize_device on its stream
(CUDA events around back-to-back calls after warm-up), input GB/s, the algorithmic bytes of one call over its time as a
fraction of the H100 SXM data sheet's 3.35 TB/s, kernel launches per call, the stream's size beside tape + Strings.B,
and the host-to-host rate of sj_parse_serialize beside sj_parse's.  Before anything is timed, the deserialized tape is
marshalled on the device and must give the parsed tape's text.  The card's name and power limit are read in the same run.

    python tools/serialize_bench.py [--mib 512] [--calls 10] [--warmup 3] [--only ndjson,twitter]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "simdjson-go_b200"), os.path.join(ROOT, "tools")]

from marshal_bench import HBM_PEAK_GBS, card  # noqa: E402


def serialize_bytes(n, strings_read, distinct, out):
    """KM1, KS1, KS2 and KS7 read the tape; KS3 / KS4 read every string twice (hash, compare) and its representative
    once; KS6 copies the distinct strings; the stream is written once.  Per-string scratch (spos, rep, slot, moff: 20
    bytes per string, each written once and read about twice) is counted; tile arrays are left out."""
    strings = out["strings"]
    return 4 * 8 * n + 3 * strings_read + 2 * distinct + out["stream"] + 3 * 20 * strings


def deserialize_bytes(tags, vals, n, msg):
    """KD1 .. KD4 read the tags; KD3 and KD4 read the values; KD2 writes a byte per tape word that KD3 reads; KD4 writes
    the tape; the message block is copied."""
    return 4 * tags + 2 * vals + 2 * n + 8 * n + 2 * msg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=512)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="ndjson,twitter")
    args = ap.parse_args()

    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _lib
    from tests.serialize_oracle import header
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
            flags = _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS
            desc = "K0 gen_ndjson: %d parking-citations-shaped records, ParseND, copy_strings" % n_rec
        else:
            one = load_fixture(wl)
            k = max(1, (args.mib << 20) // (len(one) + 1))
            host_msg = b"[" + b",".join([one] * k) + b"]"
            n = len(host_msg)
            d_msg = torch.full((n + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
            d_msg[:n].copy_(torch.frombuffer(bytearray(host_msg), dtype=torch.uint8))
            flags = _lib.FLAG_COPY_STRINGS
            desc = "'[' + %s.json x %d + ']', one document, copy_strings" % (wl, k)
        torch.cuda.synchronize()

        tcap, scap = C.c_size_t(0), C.c_size_t(0)
        L.sj_bounds(n, C.byref(tcap), C.byref(scap))
        tl, sl = C.c_size_t(0), C.c_size_t(0)
        d_tape = torch.empty(tcap.value, dtype=torch.int64, device=dev)
        d_str = torch.empty(scap.value, dtype=torch.uint8, device=dev)
        rc = L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                               d_str.data_ptr(), d_str.numel(), C.byref(sl))
        assert rc == 0, rc
        tape_words, strings_len = tl.value, sl.value
        tape, strs, msg = d_tape[:tape_words], d_str[:strings_len], d_msg[:n]

        # ---- check: serialize -> deserialize -> marshal gives the parsed tape's text ----
        rc, slen, stream = ctx.serialize_device(tape, strs, msg)
        assert rc == 0, rc
        rc, sizes, (t2, s2, m2) = ctx.deserialize_device(stream)
        assert rc == 0, rc
        rc, _, text = ctx.marshal_device(tape, strs, msg)
        rc2, _, text2 = ctx.marshal_device(t2, s2, m2)
        assert rc == rc2 == 0 and torch.equal(text, text2), "round trip differs"
        del text, text2
        hdr = header(stream.cpu().numpy().tobytes())
        n_tags, n_vals, distinct = len(hdr[3]), len(hdr[4]), len(hdr[2])
        n_strings = int((torch.frombuffer(bytearray(hdr[3]), dtype=torch.uint8) == ord('"')).sum())
        olen = C.c_size_t(0)
        t_out, t_sl, t_ml = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)

        def ser():
            r = L.sj_serialize_device(ctx.h, msg.data_ptr(), n, tape.data_ptr(), tape_words, strs.data_ptr(), strings_len,
                                      stream.data_ptr(), stream.numel(), C.byref(olen))
            assert r == 0, r

        def deser():
            r = L.sj_deserialize_device(ctx.h, stream.data_ptr(), slen, t2.data_ptr(), t2.numel(), C.byref(t_out), None, 0,
                                        C.byref(t_sl), m2.data_ptr(), m2.numel(), C.byref(t_ml))
            assert r == 0, r

        res = {}
        for key, fn in (("serialize", ser), ("deserialize", deser)):
            for _ in range(args.warmup):
                fn()
            l0 = ctx.launches()
            t = timed(fn, args.calls)
            res[key] = (t, (ctx.launches() - l0) / args.calls)
        # the bytes of every string: the length field of each '"' in the values block (a sequence of 8-byte fields)
        import numpy as np
        tags = np.frombuffer(hdr[3], dtype=np.uint8)
        fields = np.where((tags == ord('"')) | (tags == ord("e")), 2, np.where(np.isin(tags, list(b"lud{[r")), 1, 0))
        first = np.cumsum(fields) - fields
        string_bytes = int(np.frombuffer(hdr[4], dtype=np.uint64)[first[tags == ord('"')] + 1].sum())
        alg_s = serialize_bytes(tape_words, string_bytes, distinct, {"stream": slen, "strings": n_strings})
        alg_d = deserialize_bytes(n_tags, n_vals, tape_words, distinct)

        # ---- host to host: sj_parse_serialize beside sj_parse ----
        h_in = torch.frombuffer(bytearray(host_msg), dtype=torch.uint8).pin_memory()
        h_out = torch.empty(slen + 64, dtype=torch.uint8).pin_memory()
        h_tape = torch.empty(tape_words + 64, dtype=torch.int64).pin_memory()
        h_str = torch.empty(strings_len + 64, dtype=torch.uint8).pin_memory()
        mo_, ml_ = C.c_size_t(0), C.c_size_t(0)

        def host_ser():
            r = L.sj_parse_serialize(ctx.h, h_in.data_ptr(), n, flags, h_out.data_ptr(), h_out.numel(), C.byref(olen))
            assert r == 0 and olen.value == slen, r

        def host_parse():
            r = L.sj_parse(ctx.h, h_in.data_ptr(), n, flags, h_tape.data_ptr(), h_tape.numel(), C.byref(tl), h_str.data_ptr(),
                           h_str.numel(), C.byref(sl), C.byref(mo_), C.byref(ml_))
            assert r == 0, r

        rates = {}
        for key, fn in (("parse_serialize", host_ser), ("parse", host_parse)):
            fn()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            rates[key] = n / ((time.perf_counter() - t0) / args.calls) / 1e9

        ts, ls = res["serialize"]
        td, ld = res["deserialize"]
        print(json.dumps({
            "workload": wl, "input": desc, "input_bytes": n, "tape_words": tape_words, "strings_bytes": strings_len,
            "stream_bytes": slen, "tape_plus_strings_bytes": 8 * tape_words + strings_len, "strings": n_strings,
            "distinct_string_bytes": distinct, "tags": n_tags, "values_bytes": n_vals,
            "serialize_ms": round(ts * 1e3, 3), "serialize_input_gbs": round(n / ts / 1e9, 2),
            "serialize_algorithmic_bytes": int(alg_s), "serialize_hbm_frac": round(alg_s / ts / 1e9 / HBM_PEAK_GBS, 4),
            "serialize_launches_per_call": ls,
            "deserialize_ms": round(td * 1e3, 3), "deserialize_stream_gbs": round(slen / td / 1e9, 2),
            "deserialize_algorithmic_bytes": int(alg_d), "deserialize_hbm_frac": round(alg_d / td / 1e9 / HBM_PEAK_GBS, 4),
            "deserialize_launches_per_call": ld, "hbm_peak": "H100 SXM data sheet 3.35 TB/s (700 W)",
            "parse_serialize_host_gbs": round(rates["parse_serialize"], 3), "parse_host_e2e_gbs": round(rates["parse"], 3),
            "timer": "CUDA events around %d back-to-back calls after %d warm-up calls; host rates: wall clock, one context"
                     % (args.calls, args.warmup),
            "card": name, "power_limit_w": plimit}), flush=True)
        del d_msg, d_tape, d_str, stream, t2, s2, m2, h_in, h_out, h_tape, h_str, host_msg
        torch.cuda.empty_cache()
    ctx.close()


if __name__ == "__main__":
    main()
