#!/usr/bin/env python3
"""Where K1's parse mode (stage1_flatten_kernel<ndjson, ., PARSE=true>) spends its cycles, by section of a worker
iteration.

Builds the library with -DSJ_K1_PROBE into its own directory (never over libsimdjson_b200.so): each worker warp then
stamps clock64() at the section boundaries of its slab loop (stage1.cuh) and adds its sums into a device array when it
leaves the loop.  The tool runs bench.py's batch (make_batch) device-resident a few times and prints, per section, warp
cycles per 6 KiB slab and the share of the sum.  The stamps (and the __syncwarp in front of each) cost cycles of their
own, so the total is not K1's time: read the table for shares, take times from parse_breakdown.py and bench.py.  The
card's name and power limit are printed with the numbers.

  python tools/k1_probe.py [--batch-mib 512] [--steps 5] [--lib PREBUILT.so] [--json OUT]
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

SECTIONS = ["carries (peek, record carry)", "TMA wait", "phase A classify", "pass 2 (escapes, quote parity)",
            "scan-warp waits (bar_S, bar_Q)", "phase B classify", "phase B escapes", "step_events", "slab counts (agg)",
            "SlabAgg store, slab totals, bar_R"]
SLAB_BYTES = 6144


def build_probe(out_dir):
    """nvcc of the product sources with SJ_K1_PROBE defined, into out_dir"""
    from __graft_entry__ import CSRC, NVCC_FLAGS
    lib = os.path.join(out_dir, "libsimdjson_b200_k1_probe.so")
    nvcc = os.environ.get("NVCC", "nvcc")
    subprocess.check_call([nvcc] + NVCC_FLAGS + ["-DSJ_K1_PROBE", "-o", lib, os.path.join(CSRC, "sj_api.cu")], cwd=ROOT)
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-mib", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", help="a probe build made earlier (default: build one into a temporary directory)")
    ap.add_argument("--json", metavar="OUT", help="also write the table as JSON")
    args = ap.parse_args()

    with tempfile.TemporaryDirectory() as td:
        lib = args.lib or build_probe(td)
        os.environ["SJ_B200_LIB"] = lib  # read when simdjson_b200._lib is imported
        run(args, lib)


def run(args, lib):
    import numpy as np
    import torch

    import simdjson_b200 as sj
    from bench import make_batch
    from simdjson_b200 import _lib
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from parse_breakdown import card

    if not torch.cuda.is_available():
        raise SystemExit("k1_probe.py: no CUDA device")
    ctx = sj.Context(0)
    L = ctx.L
    if not hasattr(L, "sj_k1_probe_take"):
        raise SystemExit("k1_probe.py: %s is not a probe build (no sj_k1_probe_take)" % lib)
    L.sj_k1_probe_take.restype = C.c_int
    L.sj_k1_probe_take.argtypes = [C.c_void_p, C.c_void_p]
    dev = torch.device("cuda", 0)
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
    acc = (C.c_ulonglong * len(SECTIONS))()

    def step():
        r = L.sj_parse_device(ctx.h, d_msg.data_ptr(), n, flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                              d_strings.data_ptr(), d_strings.numel(), C.byref(sl))
        assert r == 0, r

    for _ in range(args.warmup):
        step()
    assert L.sj_k1_probe_take(ctx.h, acc) == 0
    for _ in range(args.steps):
        step()
    assert L.sj_k1_probe_take(ctx.h, acc) == 0
    slabs = args.steps * ((n + SLAB_BYTES - 1) // SLAB_BYTES)
    cyc = [acc[i] / slabs for i in range(len(SECTIONS))]
    tot = sum(cyc)
    gpu = card()
    print("card: %s" % gpu)
    print("batch: %d bytes, %d slabs of 6 KiB per parse; %d probed parses" % (n, slabs // args.steps, args.steps))
    print("%-36s %14s %7s" % ("K1 parse-mode section", "cycles/slab", "share"))
    for name, c in zip(SECTIONS, cyc):
        print("%-36s %14.0f %6.1f%%" % (name, c, 100.0 * c / tot if tot else 0.0))
    print("%-36s %14.0f   (probed: the stamps add cycles of their own)" % ("sum", tot))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": gpu, "batch_bytes": n, "parses": args.steps,
                       "rows": [{"section": s, "cycles_per_slab": c} for s, c in zip(SECTIONS, cyc)]}, f, indent=1)


if __name__ == "__main__":
    main()
