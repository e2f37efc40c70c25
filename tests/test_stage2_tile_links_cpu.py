"""K2t (csrc/s2s_tile.h), the streaming stage 2's scope matching, links, grammar verdict and root words, in the host
emulation of the streaming stage 2 (tests/emu/s2s_tile_emu.cpp: K2r on the fiber warp, then K2t's tiles one after the
other) against the oracle, on the documents of stage2_tile_docs.py: bracket counts at the tile edges, pairs across
them, partners several tiles back, nesting deeper than a tile, NDJSON records over tile edges with and without K2r's
in-step links, and broken input at the edges.

Every document runs twice: with K2r writing the root words of the records inside one step (as the device parse runs
it), and without, so that K2t writes every root word."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import stage2_tile_docs as TD

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_SRC = os.path.join(_DIR, "s2s_tile_emu.cpp")
_FLAGS = os.environ.get("S2S_EMU_FLAGS", "").split()  # e.g. -DS2S_EMU_REVERSE: the lanes run in descending order
_LIB = os.path.join(_DIR, "libs2stileemu%s.so" % ("_" + "_".join(f.strip("-").replace("=", "") for f in _FLAGS) if _FLAGS else ""))
_CSRC = os.path.join(os.path.dirname(_DIR), "..", "simdjson-go_b200", "csrc")
_lib = None

DOCS = TD.all_docs()


def _tiled_lib():
    global _lib
    if _lib is None:
        deps = [_SRC, os.path.join(_DIR, "s2s_emu.cpp")] + [os.path.join(_CSRC, f) for f in ("bits.h", "s2s_core.h", "s2s_slab.h", "s2s_tile.h")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Wno-unknown-pragmas"] + _FLAGS +
                                  ["-o", _LIB, _SRC])
        _lib = C.CDLL(_LIB)
        _lib.s2s_emu_parse_tiled.restype = C.c_int
        _lib.s2s_emu_parse_tiled.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                             C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                             C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_int]
    return _lib


def _emu_tiled(oracle, msg, ndjson, k2r_links):
    """parseMessage with stage 2 run by the emulated K2r + K2t: (rc, tape, strings); stage 1 and the numbers from the
    oracle"""
    a, b = oracle.trim_space(msg)
    win = msg[a:b]
    n = len(win)
    ok, deltas = oracle.find_structural_indices(win, ndjson) if n else (False, None)
    if not ok:
        return 1, None, None
    pos = (np.cumsum(deltas.astype(np.int64)) - 1).astype(np.uint32)
    buf = np.full(((n + 15) // 16) * 16 + 64, 0x20, dtype=np.uint8)
    buf[:n] = np.frombuffer(win, dtype=np.uint8)
    tape = np.zeros(2 * len(pos) + 32, dtype=np.uint64)
    strings = np.zeros(n + 64, dtype=np.uint8)
    npos = np.zeros(len(pos) + 8, dtype=np.uint32)
    nslot = np.zeros(len(pos) + 8, dtype=np.uint32)
    tl, sl, nn = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    rc = _tiled_lib().s2s_emu_parse_tiled(buf.ctypes.data, n, int(ndjson), pos.ctypes.data, len(pos), tape.ctypes.data, tape.size,
                                          C.byref(tl), strings.ctypes.data, strings.size, C.byref(sl), npos.ctypes.data,
                                          nslot.ctypes.data, npos.size, C.byref(nn), int(k2r_links))
    assert rc in (0, 2), rc
    v = C.c_uint64(0)
    for i in range(nn.value):
        p = int(npos[i])
        tag = oracle.lib.sjo_parse_number(buf.ctypes.data + p, n - p, C.byref(v))
        if tag == 0:
            return 2, None, None
        tape[nslot[i]] = tag
        tape[nslot[i] + 1] = v.value
    if rc != 0:
        return 2, None, None
    return 0, tape[:tl.value].copy(), strings[:sl.value].tobytes()


@pytest.mark.parametrize("k2r_links", [True, False], ids=["k2r-links", "k2t-all-roots"])
@pytest.mark.parametrize("d", DOCS, ids=[d.name for d in DOCS])
def test_tile_edges_emulated(oracle_native, d, k2r_links):
    rc_o, tape_o, str_o, _ = oracle_native.parse(d.msg, ndjson=d.ndjson, copy_strings=True)
    if "ok" in d.want:
        assert (rc_o == 0) == d.want["ok"], d.name
    rc, tape, strs = _emu_tiled(oracle_native, d.msg, d.ndjson, k2r_links)
    assert rc == rc_o, (d.name, rc, rc_o)
    if rc_o == 0:
        assert len(tape) == len(tape_o), d.name
        if not np.array_equal(tape, tape_o):
            bad = int(np.nonzero(tape != tape_o)[0][0])
            raise AssertionError("%s: tape differs at %d: %016x vs oracle %016x" % (d.name, bad, int(tape[bad]), int(tape_o[bad])))
        assert strs == str_o, d.name


def test_fixtures_and_fuzz_sample_emulated(oracle_native):
    """the emulated K2t on the reference's fixtures and a sample of its fuzz seeds, as documents and as NDJSON"""
    from tests.util import fuzz_corpus, load_fixture
    docs = [(load_fixture(n), nd) for n, nd in (("twitter", False), ("canada", False), ("citm_catalog", False),
                                                 ("parking-citations", True))]
    docs += [(data, nd) for _, data in fuzz_corpus("corpus", limit=400) for nd in (False, True)]
    for msg, nd in docs:
        rc_o, tape_o, str_o, _ = oracle_native.parse(msg, ndjson=nd, copy_strings=True)
        rc, tape, strs = _emu_tiled(oracle_native, msg, nd, True)
        assert rc == rc_o, (rc, rc_o, bytes(msg[:60]))
        if rc_o == 0:
            assert np.array_equal(tape, tape_o) and strs == str_o, bytes(msg[:60])


def test_docs_hit_their_geometry():
    """the counts the documents claim, and every tile-edge placement present"""
    names = {d.name for d in DOCS}
    for n in (0, 1, TD.T - 1, TD.T, TD.T + 1, 2 * TD.T - 1, 2 * TD.T + 1, 3 * TD.T - 1, 3 * TD.T + 1):
        assert "nb%d" % n in names
    for d in DOCS:
        if "brackets" in d.want:
            assert TD._count(d.msg) == d.want["brackets"], d.name
    edge = [d for d in DOCS if "edge_pair" in d.want]
    assert edge
    for d in edge:  # (their strings hold no brackets)
        b = bytes(c for c in d.msg if c in b"[]{}")
        assert b[TD.T - 1:TD.T + 1] in (b"[]", b"{}"), d.name
    for d in (d for d in DOCS if "edge_close" in d.want):
        assert bytes(c for c in d.msg if c in b"[]{}")[TD.T - 1:TD.T + 1] in (b"]]", b"]}"), d.name
