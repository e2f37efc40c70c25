"""Host emulation of the streaming stage 2 (tests/emu/s2s_emu.cpp): build + ctypes driver.  Test infrastructure."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_SRC = os.path.join(_DIR, "s2s_emu.cpp")
_FLAGS = os.environ.get("S2S_EMU_FLAGS", "").split()  # e.g. -DS2S_EMU_REVERSE: the lanes run in descending order
_LIB = os.path.join(_DIR, "libs2semu%s.so" % ("_" + "_".join(f.strip("-").replace("=", "") for f in _FLAGS) if _FLAGS else ""))
_CSRC = os.path.join(os.path.dirname(_DIR), "..", "simdjson-go_b200", "csrc")
_lib = None


def build(force=False):
    deps = [_SRC] + [os.path.join(_CSRC, f) for f in ("bits.h", "s2s_core.h", "s2s_slab.h")]
    if force or not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Wno-unknown-pragmas"] + _FLAGS + ["-o", _LIB, _SRC])


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB)
        _lib.s2s_emu_parse.restype = C.c_int
        _lib.s2s_emu_parse.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                       C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                       C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_long)]
    return _lib


def emu_parse(oracle, msg, ndjson=False):
    """parseMessage with stage 2 run by the emulated streaming kernels (copy_strings = true).
    Returns (rc, tape, strings) like Oracle.parse; stage 1 and parse_number come from the oracle."""
    msg = bytes(msg)
    a, b = oracle.trim_space(msg)
    win = msg[a:b]
    n = len(win)
    if n == 0:
        return 1, None, None
    ok, deltas = oracle.find_structural_indices(win, ndjson)
    if not ok:
        return 1, None, None
    pos = (np.cumsum(deltas.astype(np.int64)) - 1).astype(np.uint32)
    buf = np.full(((n + 15) // 16) * 16 + 64, 0x20, dtype=np.uint8)
    buf[:n] = np.frombuffer(win, dtype=np.uint8)
    tape = np.zeros(2 * len(pos) + 16, dtype=np.uint64)
    strings = np.zeros(n + 64, dtype=np.uint8)
    npos = np.zeros(len(pos) + 8, dtype=np.uint32)
    nslot = np.zeros(len(pos) + 8, dtype=np.uint32)
    tl, sl, nn, coll = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_long(0)
    rc = lib().s2s_emu_parse(buf.ctypes.data, n, int(ndjson), pos.ctypes.data, len(pos), tape.ctypes.data, tape.size, C.byref(tl),
                             strings.ctypes.data, strings.size, C.byref(sl), npos.ctypes.data, nslot.ctypes.data, npos.size,
                             C.byref(nn), C.byref(coll))
    assert rc in (0, 2), rc
    v = C.c_uint64(0)
    bad = False
    for i in range(nn.value):
        p = int(npos[i])
        tag = oracle.lib.sjo_parse_number(buf.ctypes.data + p, n - p, C.byref(v))
        if tag == 0:
            bad = True
        tape[nslot[i]] = tag
        tape[nslot[i] + 1] = v.value
    if rc != 0 or bad:
        return 2, None, None
    return 0, tape[:tl.value].copy(), strings[:sl.value].tobytes()


def same_as_oracle(oracle, msg, ndjson=False):
    rc_e, tape_e, str_e = emu_parse(oracle, msg, ndjson)
    rc_o, tape_o, str_o, _ = oracle.parse(msg, ndjson=ndjson, copy_strings=True)
    assert rc_e == rc_o, (rc_e, rc_o, bytes(msg[:100]))
    if rc_o == 0:
        assert len(tape_e) == len(tape_o), (len(tape_e), len(tape_o))
        if not np.array_equal(tape_e, tape_o):
            bad = int(np.nonzero(tape_e != tape_o)[0][0])
            raise AssertionError("tape differs at %d of %d: emu %016x oracle %016x" % (bad, len(tape_o), int(tape_e[bad]), int(tape_o[bad])))
        if str_e != str_o:
            k = next(i for i in range(min(len(str_e), len(str_o))) if str_e[i] != str_o[i]) if len(str_e) == len(str_o) else -1
            raise AssertionError("strings differ (len %d vs %d) at %d: %r vs %r" % (len(str_e), len(str_o), k, str_e[max(0, k - 20):k + 20], str_o[max(0, k - 20):k + 20]))
    return rc_e
