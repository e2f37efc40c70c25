"""CPU checks of MarshalJSON: the oracle's walk (tests/marshal_oracle.py) reproduces the reference's expected texts, and the
formatter the marshal kernels run (csrc/fmt.h, compiled with g++ through tests/emu/fmt_shim.cpp) agrees with the oracle
on every kind of double, integer and byte."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from tests import fmt_values as fv
from tests import marshal_oracle as mo
from tests.util import SMALL_FILES, TAPE_FILES, golden, load_fixture, unhex

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_SRC = os.path.join(_DIR, "fmt_shim.cpp")
_LIB = os.path.join(_DIR, "libfmtshim.so")
_CSRC = os.path.join(os.path.dirname(_DIR), "..", "simdjson-go_b200", "csrc")


@pytest.fixture(scope="module")
def shim():
    deps = [_SRC] + [os.path.join(_CSRC, f) for f in ("bits.h", "fmt.h", "pow10_table.inc")]
    if not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wall", "-o", _LIB, _SRC])
    L = C.CDLL(_LIB)
    L.fmt_shim_doubles.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fmt_shim_ints.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    L.fmt_shim_escape.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    L.fmt_shim_escape.restype = C.c_size_t
    L.fmt_shim_pow10_g.argtypes = [C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return L


def _texts(out, lens):
    return [out[32 * i:32 * i + int(n)].tobytes() for i, n in enumerate(lens)]


def _check_doubles(shim, bits):
    bits = np.ascontiguousarray(np.unique(np.asarray(bits, dtype=np.uint64)))
    out = np.zeros(32 * len(bits), dtype=np.uint8)
    lens = np.zeros(len(bits), dtype=np.uint32)
    shim.fmt_shim_doubles(bits.ctypes.data, len(bits), out.ctypes.data, lens.ctypes.data)
    assert not (lens == 0xFFFFFFFF).any(), "measured and written lengths differ"
    for b, got in zip(bits.tolist(), _texts(out, lens)):
        want = mo.format_float(struct.unpack("<d", struct.pack("<Q", b))[0])
        assert got == want, (hex(b), got, want)
    return len(bits)


def _oracle_tape(oracle, msg, ndjson, copy):
    rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
    assert rc == 0
    return tape, strs, msg[off:off + ln]


def _golden_cases():
    g = golden("G16_G17_documents")
    for tc in g["parse_nd"]:
        if tc["want"] is not None:
            yield tc["name"], unhex(tc["js"]), True, unhex(tc["want"])
    for tc in g["pass_cases"]:
        if tc["want"] is not None:
            yield tc["name"], unhex(tc["js"]), False, unhex(tc["want"])


def test_oracle_reproduces_the_golden_texts(oracle):
    cases = list(_golden_cases())
    assert len(cases) == 19
    for name, js, ndjson, want in cases:
        for copy in (True, False):
            tape, strs, msg = _oracle_tape(oracle, js, ndjson, copy)
            assert mo.marshal(tape, strs, msg) == want, (name, copy)


def test_pow10_table_rows(shim):
    """g(q) = floor(10^q * 2^(127 - floor(log2 10^q))) + 1 for every q Schubfach asks for, by exact integer arithmetic"""
    hi, lo = C.c_uint64(0), C.c_uint64(0)
    for q in range(-292, 325):
        if q >= 0:
            e = (10 ** q).bit_length() - 1  # floor(log2 10^q)
            want = 10 ** q << (127 - e) if e <= 127 else 10 ** q >> (e - 127)
        else:
            e = -(10 ** -q).bit_length()  # 10^-q is no power of two
            want = (1 << (127 - e)) // 10 ** -q
        assert want.bit_length() == 128, q
        shim.fmt_shim_pow10_g(q, C.byref(hi), C.byref(lo))
        assert (hi.value << 64 | lo.value) == want + 1, q


def test_doubles_in_the_fixture_tapes(shim, oracle):
    n = 0
    for name in TAPE_FILES + SMALL_FILES + ["parking-citations"]:
        tape, _, _ = _oracle_tape(oracle, load_fixture(name), name == "parking-citations", True)
        tags = tape >> np.uint64(56)
        idx = np.nonzero(tags == ord("d"))[0]
        if len(idx):
            n += _check_doubles(shim, tape[idx + 1])
    assert n > 100000


def test_powers_of_two_and_their_neighbours(shim):
    assert _check_doubles(shim, fv.powers_of_two()) > 4000


def test_notation_boundaries_and_integers(shim):
    _check_doubles(shim, np.concatenate([fv.notation_edges(), fv.integers_near_2_53(), fv.powers_of_ten()]))


def test_a_million_random_bit_patterns(shim):
    assert len(fv.random_bits()) >= 1_000_000
    _check_doubles(shim, fv.random_bits())
    _check_doubles(shim, fv.printf_g())


def test_integers(shim):
    v = np.array(fv.INTEGERS, dtype=np.uint64)
    for signed in (0, 1):
        out = np.zeros(32 * len(v), dtype=np.uint8)
        lens = np.zeros(len(v), dtype=np.uint32)
        shim.fmt_shim_ints(v.ctypes.data, len(v), signed, out.ctypes.data, lens.ctypes.data)
        for x, got in zip(fv.INTEGERS, _texts(out, lens)):
            want = b"%d" % (x - (1 << 64) if signed and x >> 63 else x)
            assert got == want, (x, signed, got)


def test_escapes(shim):
    src = bytes(range(256)) + b'a"b\\c\x7f\xff\xc3\xa9'
    out = np.zeros(6 * len(src), dtype=np.uint8)
    n = shim.fmt_shim_escape(src, len(src), out.ctypes.data)
    assert out[:n].tobytes() == mo.escape(src)
    assert mo.escape(b'\x00\x1f"\\\b\f\n\r\t\x7f\x80') == b'\\u0000\\u001f\\"\\\\\\b\\f\\n\\r\\t\x7f\x80'


def test_oracle_rejects_malformed_tapes(oracle):
    tape, strs, msg = _oracle_tape(oracle, b'{"a":[1,2.5,"x"],"b":{}}', False, True)
    assert mo.marshal(tape, strs, msg) == b'{"a":[1,2.5,"x"],"b":{}}'
    bad = tape.copy()
    bad[2] = (ord("t") << 56)  # key replaced by an atom
    with pytest.raises(mo.MalformedTape):
        mo.marshal(bad, strs, msg)
    bad = tape.copy()
    bad[1] = (ord("{") << 56) | 3  # link of the object broken
    with pytest.raises(mo.MalformedTape):
        mo.marshal(bad, strs, msg)
