#!/usr/bin/env python3
"""Per-kernel split of one device-resident parse step (bench.py's `value` workload).

Builds bench.py's NDJSON batch (make_batch), warms sj_parse_device up, then profiles --steps steps with
torch.profiler (CUDA activities) and prints, per kernel, the microseconds per step and the share of the step,
plus the idle gaps between consecutive kernels on the device.  The card's name and power limit are printed with
the numbers.  Tracing slows the host, so the step time here is the sum of kernel time plus gaps, not bench.py's
figure; take end-to-end numbers from bench.py.

  python tools/parse_breakdown.py [--batch-mib 512] [--steps 10] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


def short(name):
    """kernel name without its argument list (template arguments stay: they tell the instantiations apart)"""
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return name[:i]
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-mib", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", metavar="OUT", help="also write the table as JSON")
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import simdjson_b200 as sj
    from bench import make_batch
    from simdjson_b200 import _lib

    if not torch.cuda.is_available():
        raise SystemExit("parse_breakdown.py: no CUDA device")
    dev = torch.device("cuda", 0)
    ctx = sj.Context(0)
    L = ctx.L
    batch = make_batch(args.batch_mib << 20)
    n = len(batch)
    flags = _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS
    d_msg = torch.empty(n + (1 << 16), dtype=torch.uint8, device=dev)
    d_msg[:n].copy_(torch.frombuffer(bytearray(batch), dtype=torch.uint8))
    d_msg[n:] = 0x20
    rc, tape_h, strings_h, _ = ctx.parse(np.frombuffer(batch, dtype=np.uint8), ndjson=True, copy_strings=True)
    assert rc == 0, rc
    d_tape = torch.empty(len(tape_h) + 64, dtype=torch.int64, device=dev)
    d_strings = torch.empty(len(strings_h) + 64, dtype=torch.uint8, device=dev)
    tl, sl = C.c_size_t(0), C.c_size_t(0)

    def step():
        r = L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                              d_strings.data_ptr(), d_strings.numel(), C.byref(sl))
        assert r == 0, r

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    ev = [e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    ev.sort(key=lambda e: float(e["ts"]))
    per = {}
    order = []
    gap = 0.0
    for i, e in enumerate(ev):
        name = short(e["name"]) if e["cat"] == "kernel" else e["cat"]
        if name not in per:
            per[name] = [0.0, 0]
            order.append(name)
        per[name][0] += float(e["dur"])
        per[name][1] += 1
        if i:
            prev = ev[i - 1]
            gap += max(0.0, float(e["ts"]) - (float(prev["ts"]) + float(prev["dur"])))
    busy = sum(v[0] for v in per.values())
    span = (float(ev[-1]["ts"]) + float(ev[-1]["dur"]) - float(ev[0]["ts"])) if ev else 0.0
    S = args.steps
    gpu = card()
    print("card: %s" % gpu)
    print("batch: %d bytes, %d tape words, %d Strings.B bytes; %d profiled steps" % (n, len(tape_h), len(strings_h), S))
    print("%-72s %6s %10s %7s" % ("kernel / copy", "calls", "us/step", "share"))
    rows = []
    for name in order:
        t, c = per[name]
        rows.append({"name": name, "calls_per_step": c / S, "us_per_step": t / S, "share": t / span if span else 0.0})
        print("%-72s %6.1f %10.1f %6.1f%%" % (name[:72], c / S, t / S, 100.0 * t / span if span else 0.0))
    print("%-72s %6s %10.1f %6.1f%%" % ("gaps between device activities", "", gap / S, 100.0 * gap / span if span else 0.0))
    print("%-72s %6s %10.1f" % ("device busy", "", busy / S))
    print("%-72s %6s %10.1f   (first activity to last, traced: the host is slowed by the profiler)" % ("step", "", span / S))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": gpu, "batch_bytes": n, "steps": S, "rows": rows, "gap_us_per_step": gap / S,
                       "busy_us_per_step": busy / S, "step_us": span / S}, f, indent=1)


if __name__ == "__main__":
    main()
