"""The per-structural stage 2 (stage2.cuh: K2a..K2h) at its own thread, warp, tile and group edges, bit for bit against the
oracle.  It runs every parse with copy_strings off and every parse of a context set to stage-2 implementation 1, so both
configurations of CONFIGS go through it: (copy off, implementation 0) and (copy on, implementation 1), the latter with
the escape-free copies and the Strings.B offsets that only copy on produces.

The documents come from tests/stage2_edge_docs.py (checked against the oracle's stage 1 by test_stage2_edge_docs_cpu.py).
Beyond the tape: the launch counts show the dense number kernels and K2d's minimum levels run exactly where they should,
and sj_parse_device keeps its capacity contract (SJ_ERR_CAPACITY, the exact sizes, nothing written)."""
import ctypes as C

import numpy as np
import pytest

import tests.stage2_edge_docs as E
from tests.util import fuzz_corpus

pytestmark = pytest.mark.gpu

CONFIGS = [(False, 0), (True, 1)]     # (copy_strings, stage-2 implementation)
CFG_IDS = ["nocopy-impl0", "copy-impl1"]


@pytest.fixture(scope="module")
def ctxs():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    out = {}
    for copy, impl in CONFIGS:
        c = sj.Context(0)
        c.set_stage2_impl(impl)
        out[(copy, impl)] = c
    yield out
    for c in out.values():
        c.close()


def _same_parse(ctx, oracle, msg, ndjson=False, copy=True):
    rc_g, tape_g, str_g, win_g = ctx.parse(msg, ndjson=ndjson, copy_strings=copy)
    rc_o, tape_o, str_o, win_o = oracle.parse(msg, ndjson=ndjson, copy_strings=copy)
    assert rc_g == rc_o, (rc_g, rc_o, bytes(msg[:80]))
    assert win_g == win_o
    if rc_o == 0:
        assert len(tape_g) == len(tape_o)
        if not np.array_equal(tape_g, tape_o):
            bad = int(np.nonzero(tape_g != tape_o)[0][0])
            raise AssertionError("tape differs at %d: gpu %016x oracle %016x" % (bad, int(tape_g[bad]), int(tape_o[bad])))
        assert str_g == str_o
    return rc_g


def _run(ctx, oracle, docs, copy):
    n = 0
    for d in docs:
        try:
            rc = _same_parse(ctx, oracle, d.msg, ndjson=d.ndjson, copy=copy)
        except AssertionError as e:
            raise AssertionError("%s: %s" % (d.name, e)) from None
        assert (rc == 0) == d.ok, (d.name, rc)
        n += 1
    return n


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("nd", [False, True], ids=["document", "ndjson"])
def test_placed_items(ctxs, oracle_native, cfg, nd):
    """every item kind with its first structural at every index E-5..E+4 of every edge (E-2..E+1 at the group edge)"""
    n = _run(ctxs[cfg], oracle_native, E.placed_docs(nd), cfg[0])
    print("%s %s: %d documents" % (cfg, "ndjson" if nd else "document", n))
    assert n > 9000


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("gen", ["string_docs", "edge_string_docs", "leading_space_docs", "bracket_docs", "density_docs",
                                 "record_docs"])
def test_shaped_documents(ctxs, oracle_native, cfg, gen):
    n = _run(ctxs[cfg], oracle_native, getattr(E, gen)(), cfg[0])
    print("%s %s: %d documents" % (cfg, gen, n))


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_emulation_edge_suite(ctxs, oracle_native, cfg):
    """the streaming kernels' edge suite (tests/test_s2s_emulation.py) through the per-structural kernels: escapes and
    strings straddling block / step / slab edges, invalid escapes, grammar soup, NDJSON corner cases, goldens"""
    import tests.test_s2s_emulation as emu
    orig = emu.same_as_oracle
    calls = [0]

    def via_gpu(oracle, msg, ndjson=False):
        calls[0] += 1
        return _same_parse(ctxs[cfg], oracle, msg, ndjson=ndjson, copy=cfg[0])

    emu.same_as_oracle = via_gpu
    try:
        emu.test_escapes_across_every_edge(oracle_native)
        emu.test_invalid_escapes_and_strings(oracle_native)
        emu.test_strings_across_edges(oracle_native)
        emu.test_structure_and_grammar(oracle_native)
        emu.test_ndjson(oracle_native)
        emu.test_golden_documents(oracle_native)
    finally:
        emu.same_as_oracle = orig
    assert calls[0] > 2500


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("which,expect", [("corpus", 8000), ("go-corpus", 300)])
def test_fuzz_corpus(ctxs, oracle_native, cfg, which, expect):
    """every fuzz seed as a single document and as NDJSON"""
    n = 0
    for _, data in fuzz_corpus(which):
        for nd in (False, True):
            _same_parse(ctxs[cfg], oracle_native, data, ndjson=nd, copy=cfg[0])
        n += 1
    assert n > expect, n


def _launches(ctx, msg, copy):
    ctx.parse(msg, copy_strings=copy)     # (a first parse may grow the index buffer: stage 1 then runs twice)
    l0 = ctx.launches()
    rc = ctx.parse(msg, copy_strings=copy)[0]
    return rc, ctx.launches() - l0


def _base_launches(nb):
    """a per-structural parse: stage 1 (2), K2a + the two K2b scans (3), K2c (1), K2e + K2f (2), and with brackets K2d's
    s2_ansv and s2_scope (2) -- everything but the dense number kernels and K2d's s2_min32 levels"""
    return 2 + 3 + 1 + 2 + (2 if nb else 0)


def _brackets(oracle, msg):
    ok, deltas = oracle.find_structural_indices(msg)
    assert ok
    chars = np.frombuffer(msg, dtype=np.uint8)[np.cumsum(deltas.astype(np.int64)) - 1]
    return int(np.isin(chars, np.frombuffer(b"[]{}", dtype=np.uint8)).sum())


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_dense_number_kernels_launch_on_their_side_of_the_threshold(ctxs, oracle_native, cfg):
    """n_num << S2_DENSE_NUMBERS_SHIFT = n - 1: numbers stay in K2c; = n and n + 1: K2g and K2h run (2 launches)"""
    seen = set()
    for d in E.density_docs():
        rc, got = _launches(ctxs[cfg], d.msg, cfg[0])
        assert rc == 0, d.name
        nb = _brackets(oracle_native, d.msg)
        extra = got - _base_launches(nb) - E.min32_levels(nb)
        assert extra == (2 if d.want["dense"] else 0), (d.name, got, extra)
        seen.add(d.want["dense"])
        assert _same_parse(ctxs[cfg], oracle_native, d.msg, copy=cfg[0]) == 0
    assert seen == {True, False}


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_scope_matching_levels(ctxs, oracle_native, cfg):
    """32^k - 1, 32^k and 32^k + 1 brackets: K2d builds one s2_min32 level per factor of 32 above 32 brackets"""
    levels = set()
    for d in E.bracket_docs():
        rc, got = _launches(ctxs[cfg], d.msg, cfg[0])
        assert (rc == 0) == d.ok, d.name
        nb = d.want["brackets"]
        assert got - _base_launches(nb) == E.min32_levels(nb), (d.name, got)
        levels.add(E.min32_levels(nb))
    assert levels == {0, 1, 2, 3}


def _capacity_docs():
    rec = b'{"k":"a\\nb","s":"plain text","u":"\\u00e9\\ud83d\\ude00","n":[1,-2.5,true,null],"o":{"x":"' + b"y" * 70 + b'"}}'
    yield b"[" + b",".join([rec] * 40) + b"]", False
    yield b"\n".join([rec] * 40), True
    yield b'["' + b"q" * 5000 + b'\\t"]', False


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_capacity_contract(ctxs, oracle_native, cfg):
    """sj_parse_device with one word of tape or one byte of Strings.B too few: SJ_ERR_CAPACITY, the exact required sizes,
    and the caller's buffers untouched; with exactly the required sizes: the oracle's tape and strings, and nothing
    written past them"""
    import torch
    from simdjson_b200 import _lib
    ctx = ctxs[cfg]
    copy = cfg[0]
    dev = torch.device("cuda:0")
    TCAN, SCAN = 0x5A5A5A5A5A5A5A5A, 0xA5
    for msg, nd in _capacity_docs():
        rc, tape_o, str_o, _ = oracle_native.parse(msg, ndjson=nd, copy_strings=copy)
        assert rc == 0
        TL, SL = len(tape_o), len(str_o)
        assert SL > 0
        d_msg = torch.full((len(msg) + 256,), 0x20, dtype=torch.uint8, device=dev)
        d_msg[:len(msg)] = torch.frombuffer(bytearray(msg), dtype=torch.uint8).to(dev)
        flags = (_lib.FLAG_NDJSON if nd else 0) | (_lib.FLAG_COPY_STRINGS if copy else 0)
        for tcap, scap in ((TL - 1, SL + 64), (TL + 64, SL - 1), (TL, SL)):
            d_tape = torch.full((tcap + 64,), TCAN, dtype=torch.int64, device=dev)
            d_str = torch.full((scap + 64,), SCAN, dtype=torch.uint8, device=dev)
            tl, sl = C.c_size_t(0), C.c_size_t(0)
            rc = ctx.L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(msg), flags, d_tape.data_ptr(), tcap, C.byref(tl),
                                       d_str.data_ptr(), scap, C.byref(sl))
            torch.cuda.synchronize()
            tape = d_tape.cpu().numpy().view(np.uint64)
            strs = d_str.cpu().numpy()
            assert (tl.value, sl.value) == (TL, SL), (nd, tcap, scap, tl.value, sl.value)
            if (tcap, scap) != (TL, SL):
                assert rc == _lib.ERR_CAPACITY, (nd, tcap, scap, rc)
                assert (tape == TCAN).all() and (strs == SCAN).all(), (nd, tcap, scap)
            else:
                assert rc == 0
                assert np.array_equal(tape[:TL], tape_o) and strs[:SL].tobytes() == str_o
                assert (tape[TL:] == TCAN).all() and (strs[SL:] == SCAN).all()
