"""Device find (sj_find_device) on the K0 batch: parking-citations-shaped NDJSON generated on the device (sj_gen_ndjson_device),
ParseND'd into HBM, then ForEach + FindElement with 1, 4 and 16 paths (every key of the record is a STRING path; the
16-path set is the first 16 keys).  Prints one JSON line per path count:
  find_ms            sj_find_device, CUDA events around --calls back-to-back calls after --warmup calls
  parse_ms           sj_parse_device of the same input, timed the same way
  launches_per_call  kernels per sj_find_device call (the context's counter)
  min_bytes          the least the algorithm moves: the tape read once, the string bytes read and written, and the
                     columns written (18 bytes per cell, 8 per STRING offset); min_gbs = min_bytes / find time
  host rates         sj_parse_find, sj_parse and sj_parse_count_where host to host, wall clock, GB/s of input
Then one JSON line per JSON-cell workload (SJ_FIND_KIND_JSON), each beside sj_marshal_device of the same tape:
  K0 batch          ["Fine"] and ["Make"] as JSON against the same paths as STRING
  twitter NDJSON    twitter.json's statuses one per line, repeated to --mib: ["user"], ["entities"], and both
  one cell          {"a": [twitter.json x K]} at --mib: the one cell of ["a"]
  json_ms / string_ms / marshal_ms, launches per call, and min_bytes (the tape words the cells cover read once, the
  text written, the columns) over json_ms as a fraction of 3.35 TB/s
Then one JSON line per list workload (list kinds, sj_find_lists_device):
  one array         {"a": [about 4.5e7 numbers k / 4]} at --mib: ARRAY_FLOAT64 of ["a"], beside sj_marshal_device
  K0 lists          the K0 batch with "ll": [two floats] and "tags": [two strings] in every record: ["ll"] as
                    ARRAY_FLOAT64, ["tags"] as ARRAY_STRING, and both, beside ["Make"] as STRING
  list_ms, launches per call, elements and bytes out, and min_bytes (the array words read once, the elements, bytes
  and columns written) over list_ms as a fraction of 3.35 TB/s
Then one JSON line per array-rows workload (sj_find_rows_device: every record's array at a row path, one row per
element):
  statuses          {"statuses": [twitter's statuses x k]} at --mib, row path ["statuses"]: ["user","screen_name"]
                    STRING, ["retweet_count"] INT64, ["id"] UINT64, ["entities"] JSON, each alone and all four; beside
                    sj_marshal_device and ["statuses"] as one JSON cell (sj_find_lists_device) of the same tape
  github_events     github_events' 30 events repeated into one root array at --mib, row path []: ["type"] STRING,
                    ["payload"] JSON, each alone and both; beside sj_marshal_device
  hashtags          twitter's statuses one per line at --mib, row path ["entities","hashtags"]: ["text"] STRING,
                    ["indices"] ARRAY_INT64, each alone and both; beside sj_marshal_device
  rows_ms, launches per call, records, rows, bytes and elements out, records walked by one thread, and min_bytes
  (the array words read once, the record and row columns, the cells, bytes and elements written) over rows_ms as a
  fraction of 3.35 TB/s
Then one JSON line per member-rows workload (sj_find_members_device: every record's object at a row path, one row per
member, with its key):
  plugins           {"plugins": {...}}: update-center's plugins with their keys made unique, repeated to --mib, row path
                    ["plugins"]: ["version"] STRING, ["url"] STRING, [] JSON (the member's value), each alone and all
  events            citm_catalog's events, the same way: ["name"] STRING, [] JSON, each alone and both
  K0 explode        the K0 batch at --mib, row path [] (every key of every record): [] STRING_CVT with every key, and
                    with two only_keys
  members_ms, launches per call, records, rows, key bytes, bytes out, records walked by one thread, the object words,
  and min_bytes (the object words read once, the record, row and key columns, the cells and bytes written) over
  members_ms as a fraction of 3.35 TB/s, beside sj_marshal_device of the same tape
The card's name and power limit are read in the same run.
usage: python tools/find_bench.py [--mib 512] [--calls 10] [--warmup 3] [--lists-only | --rows-only | --members-only]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, limit = [x.strip() for x in out.split(",")]
    return name, float(limit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=512)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--lists-only", action="store_true", help="only the list workloads")
    ap.add_argument("--rows-only", action="store_true", help="only the array-rows workloads")
    ap.add_argument("--members-only", action="store_true", help="only the member-rows workloads")
    args = ap.parse_args()

    import numpy as np
    import torch
    import simdjson_b200 as sj
    from simdjson_b200 import _find_paths, _lib
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

    pk = load_fixture("parking-citations").strip()
    if args.lists_only:
        return list_rows(args, ctx, L, dev, timed, name, plimit, pk)
    if args.rows_only:
        return array_rows(args, ctx, L, dev, timed, name, plimit)
    if args.members_only:
        return member_rows(args, ctx, L, dev, timed, name, plimit, pk)
    lines = pk.split(b"\n")
    keys = [k.encode() for k in json.loads(lines[0])]
    n_rec = (args.mib << 20) // (len(pk) // len(lines) + 1)
    d_msg = torch.full(((args.mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device=dev)
    glen = C.c_size_t(0)
    assert L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d_msg.data_ptr(), d_msg.numel() - (1 << 16), C.byref(glen)) == 0
    n = glen.value
    flags = _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS
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
    host_msg = d_msg[:n].cpu().numpy().tobytes()
    h_in = torch.frombuffer(bytearray(host_msg), dtype=torch.uint8).pin_memory()

    for k in (1, 4, 16):
        paths, kinds = [[key] for key in keys[:k]], [_lib.FIND_KIND_STRING] * k
        cp, keep = _find_paths(paths, kinds)
        rows, nbytes = C.c_size_t(0), C.c_size_t(0)
        rcap = n_rec + 1
        out_t = (torch.empty((k, rcap), dtype=torch.uint8, device=dev), torch.empty((k, rcap), dtype=torch.uint8, device=dev),
                 torch.empty((k, rcap), dtype=torch.int64, device=dev), torch.empty((k, rcap), dtype=torch.int64, device=dev),
                 torch.empty((k, rcap + 1), dtype=torch.int64, device=dev), torch.empty(n, dtype=torch.uint8, device=dev))
        out = _lib.FindOut(*(t.data_ptr() for t in out_t), rcap, n)

        def find():
            # the tape the context just built: rows come from stage 2's root list
            r = L.sj_find_device(ctx.h, d_msg.data_ptr(), n, d_tape.data_ptr(), tape_words, d_str.data_ptr(), strings_len,
                                 cp, k, C.byref(out), C.byref(rows), C.byref(nbytes))
            assert r == 0 and rows.value == n_rec, (r, rows.value)

        parse()  # the host calls of the previous path count parsed into the context's own buffers
        for _ in range(args.warmup):
            find()
        assert bool((out_t[0][:, :n_rec] == 0).all()), "a cell is not OK"
        l0 = ctx.launches()
        t_find = timed(find, args.calls)
        launches = (ctx.launches() - l0) / args.calls
        cells = k * n_rec
        min_bytes = tape_words * 8 + 2 * nbytes.value + 18 * cells + 8 * (cells + k)

        # host to host
        h_cols = (np.empty((k, rcap), np.uint8), np.empty((k, rcap), np.uint8), np.empty((k, rcap), np.int64),
                  np.empty((k, rcap), np.uint64), np.empty((k, rcap + 1), np.int64), np.empty(n, np.uint8))
        for a in h_cols:
            a.fill(0)
        h_out = _lib.FindOut(*(a.ctypes.data for a in h_cols), rcap, n)
        h_tape = torch.empty(tape_words + 64, dtype=torch.int64).pin_memory()
        h_str = torch.empty(strings_len + 64, dtype=torch.uint8).pin_memory()
        mo_, ml_ = C.c_size_t(0), C.c_size_t(0)
        roots, matches = C.c_uint64(0), C.c_uint64(0)

        def host_find():
            r = L.sj_parse_find(ctx.h, h_in.data_ptr(), n, flags, cp, k, C.byref(h_out), C.byref(rows), C.byref(nbytes))
            assert r == 0, r

        def host_parse():
            r = L.sj_parse(ctx.h, h_in.data_ptr(), n, flags, h_tape.data_ptr(), h_tape.numel(), C.byref(tl), h_str.data_ptr(),
                           h_str.numel(), C.byref(sl), C.byref(mo_), C.byref(ml_))
            assert r == 0, r

        def host_count():
            r = L.sj_parse_count_where(ctx.h, h_in.data_ptr(), n, flags, b"Make", 4, b"HOND", 4, C.byref(roots), C.byref(matches))
            assert r == 0, r

        rates = {}
        for key, fn in (("parse_find", host_find), ("parse", host_parse), ("parse_count_where", host_count)):
            fn()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            rates[key] = n / ((time.perf_counter() - t0) / args.calls) / 1e9

        print(json.dumps({
            "input": "K0 gen_ndjson: %d parking-citations-shaped records, ParseND, copy_strings" % n_rec, "input_bytes": n,
            "tape_words": tape_words, "paths": k, "kind": "STRING", "rows": n_rec, "string_bytes_out": nbytes.value,
            "find_ms": round(t_find * 1e3, 3), "parse_ms": round(t_parse * 1e3, 3),
            "launches_per_call": launches, "min_bytes": int(min_bytes), "min_gbs": round(min_bytes / t_find / 1e9, 1),
            "parse_find_host_gbs": round(rates["parse_find"], 3), "parse_host_e2e_gbs": round(rates["parse"], 3),
            "parse_count_where_host_gbs": round(rates["parse_count_where"], 3),
            "timer": "CUDA events around %d back-to-back calls after %d warm-up calls; host rates: wall clock, one context"
                     % (args.calls, args.warmup),
            "card": name, "power_limit_w": plimit}), flush=True)
        del out_t, h_cols, h_tape, h_str
        torch.cuda.empty_cache()

    def find_call(d_m, mlen, d_t, tw, d_s, slen, paths, kinds):
        """a timed sj_find_device over a device tape into exact-size columns: (seconds, launches, rows, bytes, covered words)"""
        cp, keep = _find_paths(paths, kinds)
        rows, nbytes = C.c_size_t(0), C.c_size_t(0)
        args_ = (ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, cp, len(paths))
        assert L.sj_find_device(*args_, None, C.byref(rows), C.byref(nbytes)) in (0, _lib.ERR_CAPACITY)
        R, k, ns = rows.value, len(paths), sum(x in (_lib.FIND_KIND_STRING, _lib.FIND_KIND_JSON) for x in kinds)
        out_t = (torch.empty((k, R), dtype=torch.uint8, device=dev), torch.empty((k, R), dtype=torch.uint8, device=dev),
                 torch.empty((k, R), dtype=torch.int64, device=dev), torch.empty((k, R), dtype=torch.int64, device=dev),
                 torch.empty((ns, R + 1), dtype=torch.int64, device=dev), torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev))
        out = _lib.FindOut(*(t.data_ptr() for t in out_t), R, nbytes.value)

        def call():
            assert L.sj_find_device(*args_, C.byref(out), C.byref(rows), C.byref(nbytes)) == 0

        for _ in range(args.warmup):
            call()
        assert bool((out_t[0] == 0).all()), "a cell is not OK"
        l0 = ctx.launches()
        t = timed(call, args.calls)
        launches = (ctx.launches() - l0) / args.calls
        covered = 0
        for p, kind in enumerate(kinds):
            if kind == _lib.FIND_KIND_JSON:  # the element's words: head index to the next element's, from the tags
                tags = (d_t[out_t[2][p]].view(torch.int64) >> 56) & 0xff
                val = d_t[out_t[2][p]] & ((1 << 56) - 1)
                scalar = torch.where((tags == ord('"')) | (tags == ord("l")) | (tags == ord("u")) | (tags == ord("d")), 2, 1)
                covered += int(torch.where((tags == ord("{")) | (tags == ord("[")), val - out_t[2][p], scalar).sum())
        return t, launches, R, nbytes.value, covered

    def marshal_call(d_m, mlen, d_t, tw, d_s, slen):
        n_out = C.c_size_t(0)
        assert L.sj_marshal_device(ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, None, 0, C.byref(n_out)) == _lib.ERR_CAPACITY
        o = torch.empty(n_out.value, dtype=torch.uint8, device=dev)

        def call():
            assert L.sj_marshal_device(ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, o.data_ptr(), o.numel(),
                                       C.byref(n_out)) == 0

        for _ in range(args.warmup):
            call()
        l0 = ctx.launches()
        t = timed(call, args.calls)
        return t, (ctx.launches() - l0) / args.calls, n_out.value

    def json_rows(label, d_m, mlen, flags_, path_sets):
        nonlocal d_tape, d_str
        tl_, sl_ = C.c_size_t(0), C.c_size_t(0)
        L.sj_bounds(mlen, C.byref(tl_), C.byref(sl_))
        if tl_.value > d_tape.numel() or sl_.value > d_str.numel():
            d_tape, d_str = None, None
            torch.cuda.empty_cache()
            d_tape = torch.empty(tl_.value, dtype=torch.int64, device=dev)
            d_str = torch.empty(sl_.value, dtype=torch.uint8, device=dev)
        assert L.sj_parse_device(ctx.h, d_m.data_ptr(), mlen, flags_, d_tape.data_ptr(), d_tape.numel(), C.byref(tl_),
                                 d_str.data_ptr(), d_str.numel(), C.byref(sl_)) == 0
        tw, slen = tl_.value, sl_.value
        t_m, l_m, n_m = marshal_call(d_m, mlen, d_tape, tw, d_str, slen)
        for paths in path_sets:
            k = len(paths)
            t_j, l_j, R, nb, covered = find_call(d_m, mlen, d_tape, tw, d_str, slen, paths, [_lib.FIND_KIND_JSON] * k)
            row = {"input": label, "input_bytes": mlen, "tape_words": tw, "paths": [p[0].decode() for p in paths], "rows": R,
                   "json_bytes_out": nb, "covered_words": covered, "json_ms": round(t_j * 1e3, 3), "launches_per_call": l_j}
            if label.startswith("K0"):
                t_s, l_s, _, nb_s, _ = find_call(d_m, mlen, d_tape, tw, d_str, slen, paths, [_lib.FIND_KIND_STRING] * k)
                row.update({"string_ms": round(t_s * 1e3, 3), "string_launches_per_call": l_s, "string_bytes_out": nb_s})
            min_bytes = covered * 8 + nb + 18 * R * k + 8 * (R + 1) * k
            row.update({"marshal_ms": round(t_m * 1e3, 3), "marshal_launches_per_call": l_m, "marshal_bytes_out": n_m,
                        "min_bytes": int(min_bytes), "min_gbs": round(min_bytes / t_j / 1e9, 1),
                        "frac_of_3.35TBs": round(min_bytes / t_j / 3.35e12, 4),
                        "timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
                        "card": name, "power_limit_w": plimit})
            print(json.dumps(row), flush=True)

    # K0 batch: the message generated above
    json_rows("K0 gen_ndjson: %d parking-citations-shaped records, ParseND, copy_strings" % n_rec, d_msg, n, flags,
              [[[b"Fine"]], [[b"Make"]]])
    # twitter statuses as NDJSON
    tw_doc = json.loads(load_fixture("twitter"))
    block = b"\n".join(json.dumps(x, ensure_ascii=False, separators=(",", ":")).encode() for x in tw_doc["statuses"])
    nd = b"\n".join([block] * ((args.mib << 20) // (len(block) + 1)))
    d_nd = torch.full((len(nd) + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
    d_nd[:len(nd)] = torch.frombuffer(bytearray(nd), dtype=torch.uint8).to(dev)
    json_rows("twitter statuses NDJSON, ParseND, copy_strings", d_nd, len(nd), flags,
              [[[b"user"]], [[b"entities"]], [[b"user"], [b"entities"]]])
    del d_nd
    # one cell of about --mib
    tw = load_fixture("twitter").strip()
    one = b'{"a":[' + b",".join([tw] * ((args.mib << 20) // (len(tw) + 1))) + b"]}"
    d_one = torch.full((len(one) + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
    d_one[:len(one)] = torch.frombuffer(bytearray(one), dtype=torch.uint8).to(dev)
    json_rows("{\"a\": [twitter.json x K]}, Parse, copy_strings", d_one, len(one), _lib.FLAG_COPY_STRINGS, [[[b"a"]]])
    ctx.close()


def dev_tools(args, ctx, L, dev, timed):
    """(to_dev, parsed, call_timed, marshal_ms): a message in HBM, its tape, a timed call with its launches, and
    sj_marshal_device of a tape timed the same way"""
    import torch

    def to_dev(b):
        d = torch.full((len(b) + (1 << 16),), 0x20, dtype=torch.uint8, device=dev)
        d[:len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
        return d

    def parsed(d_m, mlen, flags_):
        tl_, sl_ = C.c_size_t(0), C.c_size_t(0)
        L.sj_bounds(mlen, C.byref(tl_), C.byref(sl_))
        d_t = torch.empty(tl_.value, dtype=torch.int64, device=dev)
        d_s = torch.empty(max(sl_.value, 1), dtype=torch.uint8, device=dev)
        assert L.sj_parse_device(ctx.h, d_m.data_ptr(), mlen, flags_, d_t.data_ptr(), d_t.numel(), C.byref(tl_),
                                 d_s.data_ptr(), d_s.numel(), C.byref(sl_)) == 0
        return d_t, tl_.value, d_s, sl_.value

    def call_timed(fn):
        for _ in range(args.warmup):
            fn()
        l0 = ctx.launches()
        t = timed(fn, args.calls)
        return t, (ctx.launches() - l0) / args.calls

    def marshal_ms(d_m, mlen, d_t, tw, d_s, slen):
        n_out = C.c_size_t(0)
        L.sj_marshal_device(ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, None, 0, C.byref(n_out))
        o = torch.empty(n_out.value, dtype=torch.uint8, device=dev)
        t, _ = call_timed(lambda: L.sj_marshal_device(ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen,
                                                      o.data_ptr(), o.numel(), C.byref(n_out)))
        return t

    return to_dev, parsed, call_timed, marshal_ms


def list_rows(args, ctx, L, dev, timed, name, plimit, pk):
    import numpy as np
    import torch
    from simdjson_b200 import _find_paths, _lib

    to_dev, parsed, call_timed, marshal_ms = dev_tools(args, ctx, L, dev, timed)

    def lists_call(d_m, mlen, d_t, tw, d_s, slen, paths, kinds):
        cp, keep = _find_paths(paths, kinds)
        rows, nb, ne = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        a = (ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, cp, len(paths))
        lists = any(k in _lib.FIND_LIST_KINDS for k in kinds)
        if lists:
            assert L.sj_find_lists_device(*a, None, None, C.byref(rows), C.byref(nb), C.byref(ne)) in (0, _lib.ERR_CAPACITY)
        else:
            assert L.sj_find_device(*a, None, C.byref(rows), C.byref(nb)) in (0, _lib.ERR_CAPACITY)
        R, k = rows.value, len(paths)
        ns, nl = sum(x in _lib.FIND_VAR_KINDS for x in kinds), sum(x in _lib.FIND_LIST_KINDS for x in kinds)
        o = [torch.empty((k, R), dtype=torch.uint8, device=dev), torch.empty((k, R), dtype=torch.uint8, device=dev),
             torch.empty((k, R), dtype=torch.int64, device=dev), torch.empty((k, R), dtype=torch.int64, device=dev),
             torch.empty((ns, R + 1), dtype=torch.int64, device=dev), torch.empty(max(nb.value, 1), dtype=torch.uint8, device=dev),
             torch.empty((nl, R + 1), dtype=torch.int64, device=dev), torch.empty(max(ne.value, 1), dtype=torch.int64, device=dev)]
        out = _lib.FindOut(*(t.data_ptr() for t in o[:6]), R, nb.value)
        lo = _lib.FindListsOut(o[6].data_ptr(), o[7].data_ptr(), ne.value)

        def call():
            if lists:
                assert L.sj_find_lists_device(*a, C.byref(out), C.byref(lo), C.byref(rows), C.byref(nb), C.byref(ne)) == 0
            else:
                assert L.sj_find_device(*a, C.byref(out), C.byref(rows), C.byref(nb)) == 0

        t, launches = call_timed(call)
        assert bool((o[0] == 0).all()), "a cell is not OK"
        covered = 0
        for p, kind in enumerate(kinds):
            if kind in _lib.FIND_LIST_KINDS:
                covered += int(((d_t[o[2][p]] & ((1 << 56) - 1)) - o[2][p]).sum())
        return t, launches, R, nb.value, ne.value, covered

    def row(label, mlen, tw, paths, kinds, res, extra):
        t, launches, R, nb, ne, covered = res
        min_bytes = covered * 8 + nb + 8 * ne + 18 * R * len(paths) + 8 * (R + 1) * len(paths)
        r = {"input": label, "input_bytes": mlen, "tape_words": tw, "paths": [p[0].decode() for p in paths],
             "kinds": list(kinds), "rows": R, "elements_out": ne, "bytes_out": nb, "covered_words": covered,
             "list_ms": round(t * 1e3, 3), "launches_per_call": launches, "min_bytes": int(min_bytes),
             "min_gbs": round(min_bytes / t / 1e9, 1), "frac_of_3.35TBs": round(min_bytes / t / 3.35e12, 4),
             "timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
             "card": name, "power_limit_w": plimit}
        r.update(extra)
        print(json.dumps(r), flush=True)

    # one array of --mib
    rng = np.random.default_rng(2024)
    x = rng.integers(0, 1 << 26, int((args.mib << 20) / 11.9)) / 4.0
    one = b'{"a":[' + ",".join(map(repr, x.tolist())).encode() + b"]}"
    d_one = to_dev(one)
    d_t, tw, d_s, slen = parsed(d_one, len(one), _lib.FLAG_COPY_STRINGS)
    res = lists_call(d_one, len(one), d_t, tw, d_s, slen, [[b"a"]], [_lib.FIND_KIND_ARRAY_FLOAT64])
    row('{"a": [%d numbers]}, Parse, copy_strings' % x.size, len(one), tw, [[b"a"]], [_lib.FIND_KIND_ARRAY_FLOAT64], res,
        {"marshal_ms": round(marshal_ms(d_one, len(one), d_t, tw, d_s, slen) * 1e3, 3)})
    del d_one, d_t, d_s
    torch.cuda.empty_cache()

    # the K0 batch with a short float array and a string list in every record
    recs = [json.loads(line) for line in pk.split(b"\n")]
    for i, r in enumerate(recs):
        r["ll"] = [34.0 + i / 64.0, -118.25 - i / 128.0]
        r["tags"] = ["k%d" % (i % 7), "zone-%d" % (i % 13)]
    tpl = b"\n".join(json.dumps(r, separators=(",", ":")).encode() for r in recs)
    n_rec = (args.mib << 20) // (len(tpl) // len(recs) + 1)
    d_msg = torch.full(((args.mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device=dev)
    glen = C.c_size_t(0)
    assert L.sj_gen_ndjson_device(ctx.h, tpl, len(tpl), 0, n_rec, d_msg.data_ptr(), d_msg.numel() - (1 << 16), C.byref(glen)) == 0
    n = glen.value
    d_t, tw, d_s, slen = parsed(d_msg, n, _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS)
    label = "K0 gen_ndjson with ll / tags: %d records, ParseND, copy_strings" % n_rec
    t_s = lists_call(d_msg, n, d_t, tw, d_s, slen, [[b"Make"]], [_lib.FIND_KIND_STRING])[0]
    for paths, kinds in (([[b"ll"]], [_lib.FIND_KIND_ARRAY_FLOAT64]), ([[b"tags"]], [_lib.FIND_KIND_ARRAY_STRING]),
                         ([[b"ll"], [b"tags"]], [_lib.FIND_KIND_ARRAY_FLOAT64, _lib.FIND_KIND_ARRAY_STRING])):
        res = lists_call(d_msg, n, d_t, tw, d_s, slen, paths, kinds)
        row(label, n, tw, paths, kinds, res, {"make_string_ms": round(t_s * 1e3, 3)})
    ctx.close()


def array_rows(args, ctx, L, dev, timed, name, plimit):
    import torch
    from simdjson_b200 import _find_paths, _lib
    from tests.util import load_fixture

    to_dev, parsed, call_timed, marshal_ms = dev_tools(args, ctx, L, dev, timed)
    i64, u8 = torch.int64, torch.uint8

    def rows_call(d_m, mlen, d_t, tw, d_s, slen, row_path, paths, kinds):
        cp, keep = _find_paths(paths, kinds)
        rp, rkeep = _find_paths([row_path], [_lib.FIND_KIND_ELEMENT])
        n = [C.c_size_t(0) for _ in range(4)]  # records, rows, bytes, elements
        a = (ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, rp, cp, len(paths))
        assert L.sj_find_rows_device(*a, None, None, None, *(C.byref(x) for x in n)) in (0, _lib.ERR_CAPACITY)
        N, R, nb, ne = (x.value for x in n)
        k = len(paths)
        ns, nl = sum(x in _lib.FIND_VAR_KINDS for x in kinds), sum(x in _lib.FIND_LIST_KINDS for x in kinds)
        o = [torch.empty((k, R), dtype=u8, device=dev), torch.empty((k, R), dtype=u8, device=dev),
             torch.empty((k, R), dtype=i64, device=dev), torch.empty((k, R), dtype=i64, device=dev),
             torch.empty((ns, R + 1), dtype=i64, device=dev), torch.empty(max(nb, 1), dtype=u8, device=dev),
             torch.empty((nl, R + 1), dtype=i64, device=dev), torch.empty(max(ne, 1), dtype=i64, device=dev),
             torch.empty(max(N, 1), dtype=u8, device=dev), torch.empty(N + 1, dtype=i64, device=dev),
             torch.empty(max(R, 1), dtype=u8, device=dev), torch.empty(max(R, 1), dtype=i64, device=dev)]
        out = _lib.FindOut(*(t.data_ptr() for t in o[:6]), R, nb)
        lo = _lib.FindListsOut(o[6].data_ptr(), o[7].data_ptr(), ne)
        ro = _lib.FindRowsOut(*(t.data_ptr() for t in o[8:12]), N)

        def call():
            assert L.sj_find_rows_device(*a, C.byref(out), C.byref(lo), C.byref(ro), *(C.byref(x) for x in n)) == 0

        t, launches = call_timed(call)
        serial = C.c_uint64(0)
        L.sj_test_find_rows_serial(ctx.h, C.byref(serial))
        ok = int((o[8][:N] == 0).sum())  # records with an array
        # the array words: each record's [head, end), its '[' one word in front of its first row
        first = o[9][:N][o[9][1:N + 1] > o[9][:N]]
        heads = o[11][first] - 1
        covered = int(((d_t[heads] & ((1 << 56) - 1)) - heads).sum())
        return t, launches, N, R, nb, ne, covered, serial.value, ok

    def line(label, mlen, tw, row_path, paths, kinds, res, extra):
        t, launches, N, R, nb, ne, covered, serial, ok = res
        ns = sum(x in _lib.FIND_VAR_KINDS for x in kinds)
        min_bytes = covered * 8 + 9 * N + 8 + 9 * R + 18 * R * len(paths) + 8 * (R + 1) * ns + nb + 8 * ne
        r = {"input": label, "input_bytes": mlen, "tape_words": tw, "row_path": [x.decode() for x in row_path],
             "paths": [".".join(x.decode() for x in p) for p in paths], "kinds": list(kinds), "records": N, "records_ok": ok, "rows": R,
             "bytes_out": nb, "elements_out": ne, "serial_records": serial, "covered_words": covered,
             "rows_ms": round(t * 1e3, 3), "launches_per_call": launches, "min_bytes": int(min_bytes),
             "min_gbs": round(min_bytes / t / 1e9, 1), "frac_of_3.35TBs": round(min_bytes / t / 3.35e12, 4),
             "timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
             "card": name, "power_limit_w": plimit}
        r.update(extra)
        print(json.dumps(r), flush=True)

    def one_json_cell_ms(d_m, mlen, d_t, tw, d_s, slen, path):
        cp, keep = _find_paths([path], [_lib.FIND_KIND_JSON])
        rows, nb, ne = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        a = (ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, cp, 1)
        assert L.sj_find_lists_device(*a, None, None, C.byref(rows), C.byref(nb), C.byref(ne)) in (0, _lib.ERR_CAPACITY)
        R = rows.value
        o = [torch.empty((1, R), dtype=u8, device=dev), torch.empty((1, R), dtype=u8, device=dev),
             torch.empty((1, R), dtype=i64, device=dev), torch.empty((1, R), dtype=i64, device=dev),
             torch.empty((1, R + 1), dtype=i64, device=dev), torch.empty(max(nb.value, 1), dtype=u8, device=dev)]
        out = _lib.FindOut(*(t.data_ptr() for t in o), R, nb.value)
        t, _ = call_timed(lambda: L.sj_find_lists_device(*a, C.byref(out), None, C.byref(rows), C.byref(nb), C.byref(ne)))
        assert bool((o[0] == 0).all())
        return t

    def workload(label, doc, flags, row_path, path_sets, json_cell=None):
        d_m = to_dev(doc)
        d_t, tw, d_s, slen = parsed(d_m, len(doc), flags)
        extra = {"marshal_ms": round(marshal_ms(d_m, len(doc), d_t, tw, d_s, slen) * 1e3, 3)}
        if json_cell:
            extra["one_json_cell_ms"] = round(one_json_cell_ms(d_m, len(doc), d_t, tw, d_s, slen, json_cell) * 1e3, 3)
        for paths, kinds in path_sets:
            res = rows_call(d_m, len(doc), d_t, tw, d_s, slen, row_path, paths, kinds)
            line(label, len(doc), tw, row_path, paths, kinds, res, extra)
        del d_m, d_t, d_s
        torch.cuda.empty_cache()

    def sets(pk):
        return [([p], [k]) for p, k in pk] + [([p for p, _ in pk], [k for _, k in pk])]

    size = args.mib << 20
    tw_doc = json.loads(load_fixture("twitter"))
    statuses = [json.dumps(x, separators=(",", ":")).encode() for x in tw_doc["statuses"]]
    body = b",".join(statuses)
    doc = b'{"statuses":[' + b",".join([body] * max(1, size // (len(body) + 1))) + b"]}"
    workload("{\"statuses\": [twitter statuses x k]}, Parse, copy_strings", doc, _lib.FLAG_COPY_STRINGS, [b"statuses"],
             sets([([b"user", b"screen_name"], _lib.FIND_KIND_STRING), ([b"retweet_count"], _lib.FIND_KIND_INT64),
                   ([b"id"], _lib.FIND_KIND_UINT64), ([b"entities"], _lib.FIND_KIND_JSON)]), json_cell=[b"statuses"])
    events = load_fixture("github_events").strip()
    body = events[1:-1].strip()
    doc = b"[" + b",".join([body] * max(1, size // (len(body) + 1))) + b"]"
    workload("github_events repeated into one root array, Parse, copy_strings", doc, _lib.FLAG_COPY_STRINGS, [],
             sets([([b"type"], _lib.FIND_KIND_STRING), ([b"payload"], _lib.FIND_KIND_JSON)]))
    lines = b"\n".join(statuses)
    doc = b"\n".join([lines] * max(1, size // (len(lines) + 1)))
    workload("twitter statuses as NDJSON, ParseND, copy_strings", doc, _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS,
             [b"entities", b"hashtags"], sets([([b"text"], _lib.FIND_KIND_STRING), ([b"indices"], _lib.FIND_KIND_ARRAY_INT64)]))
    ctx.close()



def member_rows(args, ctx, L, dev, timed, name, plimit, pk):
    import torch
    from simdjson_b200 import _find_paths, _lib
    from tests.util import load_fixture

    to_dev, parsed, call_timed, marshal_ms = dev_tools(args, ctx, L, dev, timed)
    i64, u8 = torch.int64, torch.uint8

    def members_call(d_m, mlen, d_t, tw, d_s, slen, row_path, only, paths, kinds):
        cp, keep = _find_paths(paths, kinds)
        rp, rkeep = _find_paths([row_path, only], [_lib.FIND_KIND_ELEMENT] * 2)
        n = [C.c_size_t(0) for _ in range(5)]  # records, rows, bytes, elements, key bytes
        a = (ctx.h, d_m.data_ptr(), mlen, d_t.data_ptr(), tw, d_s.data_ptr(), slen, rp, C.pointer(rp[1]),
             cp, len(paths))
        assert L.sj_find_members_device(*a, None, None, None, None, *(C.byref(x) for x in n)) in (0, _lib.ERR_CAPACITY)
        N, R, nb, ne, nk = (x.value for x in n)
        k = len(paths)
        ns = sum(x in _lib.FIND_VAR_KINDS for x in kinds)
        o = [torch.empty((k, R), dtype=u8, device=dev), torch.empty((k, R), dtype=u8, device=dev),
             torch.empty((k, R), dtype=i64, device=dev), torch.empty((k, R), dtype=i64, device=dev),
             torch.empty((ns, R + 1), dtype=i64, device=dev), torch.empty(max(nb, 1), dtype=u8, device=dev),
             torch.empty((0, R + 1), dtype=i64, device=dev), torch.empty(1, dtype=i64, device=dev),
             torch.empty(max(N, 1), dtype=u8, device=dev), torch.empty(N + 1, dtype=i64, device=dev),
             torch.empty(max(R, 1), dtype=u8, device=dev), torch.empty(max(R, 1), dtype=i64, device=dev),
             torch.empty(R + 1, dtype=i64, device=dev), torch.empty(max(nk, 1), dtype=u8, device=dev)]
        out = _lib.FindOut(*(t.data_ptr() for t in o[:6]), R, nb)
        lo = _lib.FindListsOut(o[6].data_ptr(), o[7].data_ptr(), 0)
        ro = _lib.FindRowsOut(*(t.data_ptr() for t in o[8:12]), N)
        ko = _lib.FindKeysOut(o[12].data_ptr(), o[13].data_ptr(), nk)

        def call():
            assert L.sj_find_members_device(*a, C.byref(out), C.byref(lo), C.byref(ro), C.byref(ko), *(C.byref(x) for x in n)) == 0

        t, launches = call_timed(call)
        serial = C.c_uint64(0)
        L.sj_test_find_rows_serial(ctx.h, C.byref(serial))
        ok = int((o[8][:N] == 0).sum())
        return t, launches, N, R, nb, nk, serial.value, ok

    def line(label, mlen, tw, words, row_path, only, paths, kinds, res, extra):
        t, launches, N, R, nb, nk, serial, ok = res
        ns = sum(x in _lib.FIND_VAR_KINDS for x in kinds)
        min_bytes = words * 8 + 9 * N + 8 + 9 * R + 8 * (R + 1) + nk + 18 * R * len(paths) + 8 * (R + 1) * ns + nb
        r = {"input": label, "input_bytes": mlen, "tape_words": tw, "object_words": words,
             "row_path": [x.decode() for x in row_path], "only_keys": [x.decode() for x in only],
             "paths": [".".join(x.decode() for x in p) for p in paths], "kinds": list(kinds), "records": N, "records_ok": ok,
             "rows": R, "key_bytes": nk, "bytes_out": nb, "serial_records": serial, "members_ms": round(t * 1e3, 3),
             "launches_per_call": launches, "min_bytes": int(min_bytes), "min_gbs": round(min_bytes / t / 1e9, 1),
             "frac_of_3.35TBs": round(min_bytes / t / 3.35e12, 4),
             "timer": "CUDA events around %d back-to-back calls after %d warm-up calls" % (args.calls, args.warmup),
             "card": name, "power_limit_w": plimit}
        r.update(extra)
        print(json.dumps(r), flush=True)

    def workload(label, d_m, mlen, flags, row_path, words, runs):
        d_t, tw, d_s, slen = parsed(d_m, mlen, flags)
        extra = {"marshal_ms": round(marshal_ms(d_m, mlen, d_t, tw, d_s, slen) * 1e3, 3)}
        for only, paths, kinds in runs:
            res = members_call(d_m, mlen, d_t, tw, d_s, slen, row_path, only, paths, kinds)
            line(label, mlen, tw, words(tw), row_path, only, paths, kinds, res, extra)
        del d_t, d_s
        torch.cuda.empty_cache()

    def sets(pk_):
        return [((), [p], [k]) for p, k in pk_] + [((), [p for p, _ in pk_], [k for _, k in pk_])]

    def one_map(fixture, key):
        """{key: {...}} of the fixture's map at `key`, its members repeated with unique keys to --mib"""
        members = list(json.loads(load_fixture(fixture))[key].items())
        one = [(k, json.dumps(v, separators=(",", ":")).encode()) for k, v in members]
        size, parts, i, total = args.mib << 20, [], 0, 0
        while total < size:
            for k, v in one:
                p = json.dumps("%s~%d" % (k, i)).encode() + b":" + v
                parts.append(p)
                total += len(p) + 1
            i += 1
        return b'{"' + key.encode() + b'":{' + b",".join(parts) + b"}}"

    for fixture, key, runs in (("update-center", "plugins", sets([([b"version"], _lib.FIND_KIND_STRING),
                                                                   ([b"url"], _lib.FIND_KIND_STRING), ([], _lib.FIND_KIND_JSON)])),
                               ("citm_catalog", "events", sets([([b"name"], _lib.FIND_KIND_STRING), ([], _lib.FIND_KIND_JSON)]))):
        doc = one_map(fixture, key)
        d_m = to_dev(doc)
        workload("{\"%s\": %s's %s with unique keys x k}, Parse, copy_strings" % (key, fixture, key), d_m, len(doc),
                 _lib.FLAG_COPY_STRINGS, [key.encode()], lambda tw: tw - 6, runs)
        del d_m
    lines = pk.split(b"\n")
    keys = [k.encode() for k in json.loads(lines[0])]
    n_rec = (args.mib << 20) // (len(pk) // len(lines) + 1)
    d_m = torch.full(((args.mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device=dev)
    glen = C.c_size_t(0)
    assert L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d_m.data_ptr(), d_m.numel() - (1 << 16), C.byref(glen)) == 0
    workload("K0 batch (parking citations), ParseND, copy_strings", d_m, glen.value, _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS,
             [], lambda tw: tw - 2 * n_rec, [((), [[]], [_lib.FIND_KIND_STRING_CVT]),
                                             ((keys[1], keys[5]), [[]], [_lib.FIND_KIND_STRING_CVT])])
    ctx.close()


if __name__ == "__main__":
    main()
