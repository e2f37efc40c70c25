"""Quick device-resident stage-1 timing (development aid; bench.py is the contract).
usage: quick_stage1_bench.py [fixture] [MiB] [lib.so ...]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "simdjson-go_b200"))
import torch

from tests.util import load_fixture

name = sys.argv[1] if len(sys.argv) > 1 else "twitter"
target = int(float(sys.argv[2]) * (1 << 20)) if len(sys.argv) > 2 else 1 << 30
libs = sys.argv[3:] or [os.path.join(ROOT, "simdjson-go_b200", "libsimdjson_b200.so")]
doc = load_fixture(name).strip()
k = max(1, target // (len(doc) + 1))
msg = b"[" + b",".join([doc] * k) + b"]"
n = len(msg)
print("input %s x%d = %d bytes" % (name, k, n))
dev = torch.device("cuda:0")
d_msg = torch.empty(n + 65536, dtype=torch.uint8, device=dev)
d_msg[:n] = torch.frombuffer(bytearray(msg), dtype=torch.uint8).to(dev)
d_msg[n:] = 0x20
cap = n // 4 + 1024
d_out = torch.empty(cap, dtype=torch.int32, device=dev)


class Info(C.Structure):
    _fields_ = [("n_idx", C.c_uint64), ("error", C.c_uint32), ("ends_in_string", C.c_uint32), ("last_pos", C.c_uint32),
                ("overflow", C.c_uint32)]


for lib in libs:
    L = C.CDLL(lib)
    vp = C.c_void_p
    L.sj_ctx_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.sj_stage1_device.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_int, vp, C.c_size_t, C.POINTER(Info)]
    L.sj_stage1_launch.argtypes = [vp, vp, C.c_size_t, C.c_int, C.c_int, vp, C.c_size_t]
    L.sj_ctx_sync.argtypes = [vp]
    L.sj_event_record.argtypes = [vp, C.c_int]
    L.sj_event_elapsed_ms.argtypes = [vp, C.POINTER(C.c_float)]
    h = vp()
    assert L.sj_ctx_create(0, C.byref(h)) == 0
    info = Info()
    rc = L.sj_stage1_device(h, d_msg.data_ptr(), n, 0, 0, d_out.data_ptr(), cap, C.byref(info))
    print(os.path.basename(lib), "rc", rc, "n_idx", info.n_idx, "err", info.error, "instr", info.ends_in_string)
    for deltas in (0, 1):
        for it in range(3):
            L.sj_stage1_launch(h, d_msg.data_ptr(), n, 0, deltas, d_out.data_ptr(), cap)
        L.sj_ctx_sync(h)
        reps = 10
        L.sj_event_record(h, 0)
        for it in range(reps):
            L.sj_stage1_launch(h, d_msg.data_ptr(), n, 0, deltas, d_out.data_ptr(), cap)
        L.sj_event_record(h, 1)
        ms = C.c_float(0)
        L.sj_event_elapsed_ms(h, C.byref(ms))
        t = ms.value / reps / 1e3
        alg = n + 4 * info.n_idx
        print("  deltas=%d: %.3f ms  input %.1f GB/s  algorithmic %.1f GB/s" % (deltas, t * 1e3, n / t / 1e9, alg / t / 1e9))
