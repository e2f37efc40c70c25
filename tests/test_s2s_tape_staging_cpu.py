"""K2r's staged tape and its in-step links, run by the host emulation of the streaming stage 2 and compared bit for bit
with the oracle.

K2r stages a step's tape words in shared memory at the destination's 32-byte phase and copies them out in whole
sectors; a step whose words do not fit (640 words minus that phase) stores them directly.  Bracket pairs and NDJSON
records whose two ends lie in one staged step are linked there, and K2e / K2f skip exactly those.  The driver here
(tests/emu/s2s_link_emu.cpp: the emulation of s2s_emu.cpp with K2r's root-word links switched on, as the device parse
runs it) puts the staging capacity, the tape's alignment, bracket pairs across step and slab edges, invalid documents
and record boundaries at step edges through the same templates the kernels compile."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

STEP, SLAB = 2048, 6144
CAP = 640  # K2r's tape-staging words (S2S_TSTAGE_WORDS)

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_SRC = os.path.join(_DIR, "s2s_link_emu.cpp")
_FLAGS = os.environ.get("S2S_EMU_FLAGS", "").split()  # e.g. -DS2S_EMU_REVERSE: the lanes run in descending order
_LIB = os.path.join(_DIR, "libs2slinkemu%s.so" % ("_" + "_".join(f.strip("-").replace("=", "") for f in _FLAGS) if _FLAGS else ""))
_CSRC = os.path.join(os.path.dirname(_DIR), "..", "simdjson-go_b200", "csrc")
_lib = None


def _linked_lib():
    global _lib
    if _lib is None:
        deps = [_SRC, os.path.join(_DIR, "s2s_emu.cpp")] + [os.path.join(_CSRC, f) for f in ("bits.h", "s2s_core.h", "s2s_slab.h")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Wno-unknown-pragmas"] + _FLAGS +
                                  ["-o", _LIB, _SRC])
        _lib = C.CDLL(_LIB)
        _lib.s2s_emu_parse_linked.restype = C.c_int
        _lib.s2s_emu_parse_linked.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                              C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                              C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
    return _lib


def _emu_at_phase(oracle, msg, ndjson, phase):
    """the emulated parse with the tape placed `phase` words past a 32-byte boundary:
    (rc, tape, strings, (closes, records) K2r has linked)"""
    msg = bytes(msg)
    a, b = oracle.trim_space(msg)
    win = msg[a:b]
    n = len(win)
    ok, deltas = oracle.find_structural_indices(win, ndjson) if n else (False, None)
    if not ok:
        return 1, None, None, (0, 0)  # (stage 1 rejects it)
    pos = (np.cumsum(deltas.astype(np.int64)) - 1).astype(np.uint32)
    buf = np.full(((n + 15) // 16) * 16 + 64, 0x20, dtype=np.uint8)
    buf[:n] = np.frombuffer(win, dtype=np.uint8)
    raw = np.zeros(2 * len(pos) + 32, dtype=np.uint64)
    skip = ((-raw.ctypes.data // 8) + phase) % 4  # words up to the wanted phase
    tape = raw[skip:]
    assert (tape.ctypes.data // 8) % 4 == phase
    strings = np.zeros(n + 64, dtype=np.uint8)
    npos = np.zeros(len(pos) + 8, dtype=np.uint32)
    nslot = np.zeros(len(pos) + 8, dtype=np.uint32)
    linked = np.zeros(2, dtype=np.uint64)
    tl, sl, nn = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    rc = _linked_lib().s2s_emu_parse_linked(buf.ctypes.data, n, int(ndjson), pos.ctypes.data, len(pos), tape.ctypes.data,
                                            tape.size, C.byref(tl), strings.ctypes.data, strings.size, C.byref(sl),
                                            npos.ctypes.data, nslot.ctypes.data, npos.size, C.byref(nn), linked.ctypes.data)
    assert rc in (0, 2), rc
    lk = (int(linked[0]), int(linked[1]))
    v = C.c_uint64(0)
    for i in range(nn.value):
        p = int(npos[i])
        tag = oracle.lib.sjo_parse_number(buf.ctypes.data + p, n - p, C.byref(v))
        if tag == 0:
            return 2, None, None, lk
        tape[nslot[i]] = tag
        tape[nslot[i] + 1] = v.value
    if rc != 0:
        return 2, None, None, lk
    return 0, tape[:tl.value].copy(), strings[:sl.value].tobytes(), lk


def _same_at_phase(oracle, msg, ndjson=False, phase=0):
    """rc, after the tape and the strings are checked against the oracle; _same_at_phase.linked: what K2r linked"""
    rc_e, tape_e, str_e, lk = _emu_at_phase(oracle, msg, ndjson, phase)
    rc_o, tape_o, str_o, _ = oracle.parse(msg, ndjson=ndjson, copy_strings=True)
    assert rc_e == rc_o, (rc_e, rc_o, phase)
    if rc_o == 0:
        assert len(tape_e) == len(tape_o)
        if not np.array_equal(tape_e, tape_o):
            bad = int(np.nonzero(tape_e != tape_o)[0][0])
            raise AssertionError("phase %d: tape differs at %d: emu %016x oracle %016x" % (phase, bad, int(tape_e[bad]), int(tape_o[bad])))
        assert str_e == str_o
    _same_at_phase.linked = lk
    return rc_e



def words_steps(targets):
    """an array whose 2 KiB step s holds exactly targets[s] tape words (the '[' and the root words aside): numbers
    (two words), one atom when the count is odd, blanks up to the step's end"""
    parts = []
    for s, w in enumerate(targets):
        body = b"1," * (w // 2) + (b"true," if w % 2 else b"")
        head = b"[" if s == 0 else b""
        assert len(head) + len(body) <= STEP
        parts.append(head + body + b" " * (STEP - len(head) - len(body)))
    return b"".join(parts) + b"0]"


def capacity_targets():
    # just below, at and just above the capacity for every phase (the first step also carries the '['), back to back,
    # with slab edges between steps 2 / 3 and 5 / 6
    return [CAP - 5, CAP - 3, CAP - 2, CAP - 1, CAP, CAP + 1, CAP + 2, 200, CAP - 4, CAP + 3, CAP - 1, 0, CAP]


@pytest.mark.parametrize("phase", [0, 1, 2, 3])
def test_step_words_around_the_staging_capacity(oracle_native, phase):
    doc = words_steps(capacity_targets())
    assert _same_at_phase(oracle_native, doc, False, phase) == 0
    # the same counts made of brackets (one word each) and strings, so the staged path also carries links
    for unit, words in ((b"[],", 2), (b'{"":[]},', 5), (b'"ab",', 2)):
        parts = [b"["]
        for s, w in enumerate(capacity_targets()):
            k = w // words
            body = unit * k + b"1," * ((w - k * words) // 2) + (b"true," if (w - k * words) % 2 else b"")
            used = len(parts[0]) if s == 0 else 0
            assert used + len(body) <= STEP
            parts.append(body + b" " * (STEP - used - len(body)))
        assert _same_at_phase(oracle_native, b"".join(parts) + b"0]", False, phase) == 0


@pytest.mark.parametrize("phase", [1, 3])
def test_fixtures_at_unaligned_tape(oracle_native, phase):
    from tests.util import load_fixture
    for name in ("twitter", "canada", "citm_catalog"):
        assert _same_at_phase(oracle_native, load_fixture(name), False, phase) == 0
    pk = load_fixture("parking-citations").strip()
    assert _same_at_phase(oracle_native, pk, True, phase) == 0
    closes, records = _same_at_phase.linked
    assert closes > 0 and records > 0, (closes, records)  # both kinds of in-step link ran


def _pad_to(prefix, at):
    assert len(prefix) <= at
    return prefix + b" " * (at - len(prefix))


@pytest.mark.parametrize("edge", [STEP, SLAB, SLAB + STEP])
def test_bracket_pairs_inside_and_across_edges(oracle_native, edge):
    for d in range(-3, 4):
        # a pair across the edge, a pair that ends right at it, one that starts right behind it
        doc = _pad_to(b'[{"a":[1,2]},[', edge + d) + b'3],{"b":{}}, [[]' + b" " * 40 + b"]]"
        _same_at_phase(oracle_native, doc)
        doc = _pad_to(b'[{"k":[', edge - 2 + d) + b']}, {"m":[]}]'
        _same_at_phase(oracle_native, doc)
    # open in step s, close in step s + 2, with pairs in the steps between
    mid = b'{"x":[1,[2,[3]]]},' * ((2 * STEP) // 18 + 5)
    assert _same_at_phase(oracle_native, _pad_to(b"[[", edge - 10) + mid + b"4]]") == 0
    # nesting deeper than the in-step search and wide objects, where the partner is far in front
    assert _same_at_phase(oracle_native, _pad_to(b"[", edge - 50) + b"[" * 200 + b"]" * 200 + b"]") == 0
    assert _same_at_phase(oracle_native, _pad_to(b'{"o":{', edge - 30) + b",".join(b'"k%d":[%d]' % (i, i) for i in range(150)) + b"}}") == 0


def test_first_and_last_step(oracle_native):
    for n in (1, 2, 10, STEP - 2, STEP - 1, STEP, STEP + 1, SLAB - 1, SLAB + 1):
        doc = b"[" + b" " * max(0, n - 2) + b"]"
        _same_at_phase(oracle_native, doc)
        _same_at_phase(oracle_native, b"{}" + b"\n" * n + b"[1]", True)
    _same_at_phase(oracle_native, b"{}")
    _same_at_phase(oracle_native, b"[[]]")


@pytest.mark.parametrize("edge", [0, STEP, SLAB])
def test_invalid_brackets_fail_as_before(oracle_native, edge):
    bad = [b'[1,{"a":2]]', b'{"a":[1,2}', b'[1]]', b'{"a":1}}', b']', b'[[[[1', b'{"a":{"b":[', b'[{]}', b'[1,{]', b'{[]}']
    for b in bad:
        doc = _pad_to(b"[", edge) + b + b"]" if edge else b
        rc = _same_at_phase(oracle_native, doc)
        assert rc != 0, doc[-40:]
        _same_at_phase(oracle_native, b'{"a":1}\n' + b + b'\n{"b":2}', True)


@pytest.mark.parametrize("phase", [0, 3])
def test_records_at_step_edges(oracle_native, phase):
    rec = b'{"k":"v"}'
    for edge in (STEP, SLAB, 2 * STEP):
        for d in range(-2, 3):
            # a record that ends at the step's last event / starts at its first
            lead = _pad_to(b'{"a":"', edge - 2 + d) + b'"}'
            doc = lead + b"\n" + b"\n".join([rec] * 30)
            _same_at_phase(oracle_native, doc, True, phase)
            doc = lead + b" \n\n \n" + rec + b"\n\n\n" + b"\n".join([b"[]"] * 500) + b"\n"
            _same_at_phase(oracle_native, doc, True, phase)
    # one-word records, tiny records (more than the in-step list holds), blank-line runs
    for doc in (b"1\n2\n", b"1\n2\n3", b"{}\n" * 3000, b"[1]\n" * 1000, b"{}\n\n\n\n" * 900 + b"[]",
                b"\n".join([b"[" + b"1," * 30 + b"2]"] * 400), b'{"a":[1,{"b":2}]}\n' * 600):
        _same_at_phase(oracle_native, doc, True, phase)
