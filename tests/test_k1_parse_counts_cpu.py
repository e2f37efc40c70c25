"""Stage 1's parse mode counts each slab for stage 2 from one classification per block, and runs the slab's collectives
once per slab (agg_lane_add / agg_warp_finish, s2s_slab.h).  Checked on the CPU:

- the classes it rebuilds from its structurals and two extra planes (parse_planes, s2s_core.h) against classify_block2,
  for every byte value at every position of a block;
- the emulator's counting pass, which runs the same helpers, on slabs whose last quote or last three structurals lie in
  each of the slab's steps, and with steps that hold no structural or no quote.  The emulated K2r checks every slab's
  counts against its own and the tape against the oracle, so a miscount fails the parse."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu_util
from tests.emu_util import same_as_oracle

SLAB, STEP = 6144, 2048


def _shim():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
    L = emu_util._build_shim(os.path.join(d, "parse_planes_shim.cpp"), os.path.join(d, "libparseplanesshim.so"),
                             ("bits.h", "s2s_core.h"))
    L.parse_planes_check.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
    L.parse_planes_check.restype = None
    return L


@pytest.mark.parametrize("filler", [0x20, ord("a"), ord("0"), ord(","), ord("{"), 0x0A, 0xC3])
def test_parse_planes_every_byte_every_position(filler):
    blocks = np.full((256 * 64, 64), filler, dtype=np.uint8)
    for v in range(256):
        for i in range(64):
            blocks[64 * v + i, i] = v
    out = np.zeros((len(blocks), 10), dtype=np.uint64)
    _shim().parse_planes_check(blocks.ctypes.data, len(blocks), out.ctypes.data)
    names = ["open", "close", "cc", "numc", "atomc"]
    for k, name in enumerate(names):
        bad = np.nonzero(out[:, k] != out[:, 5 + k])[0]
        assert len(bad) == 0, "%s differs for byte 0x%02x at position %d" % (name, bad[0] // 64, bad[0] % 64)
    # the planes see every class at all: the check above is not vacuous
    assert all(out[:, k].any() for k in range(5))


def _quote_docs():
    """the slab's last real quote at each step of slab 0 and slab 1, followed by bytes with or without structurals"""
    for slab in (0, 1):
        for off in (5, 63, 64, 2000, STEP - 1, STEP, STEP + 1, 3000, 2 * STEP - 1, 2 * STEP, 5000, SLAB - 2, SLAB - 1):
            pos = slab * SLAB + off
            head = b'["' + b"a" * (pos - 2) + b'"'  # the string's closing quote at pos
            assert head[pos:pos + 1] == b'"'
            fill = SLAB * (slab + 1) + 100 - len(head)
            yield head + b"," + b" " * fill + b'"tail"]'            # no structural, no quote behind it
            yield head + b",1" * (fill // 2) + b',"tail"]'          # structurals, no quote behind it
            yield head + b',"' + b"b" * fill + b'"]'                 # a string open across the slab edge
            yield head + b',"' + b"b\\n" * (fill // 3) + b'"]'       # ... with escapes that drop bytes


def _last_docs():
    """the slab's last three structurals spread over its steps: one or two of them in the last step with any"""
    spots = [(100, 200, 300), (STEP - 3, STEP + 5, STEP + 9), (STEP - 2, STEP - 1, 2 * STEP + 7), (50, STEP + 50, 2 * STEP + 50),
             (2 * STEP - 1, 2 * STEP, SLAB - 1), (10, 20, SLAB - 1), (SLAB - 3, SLAB - 2, SLAB - 1)]
    for a, b, c in spots:
        doc = bytearray(b" " * (SLAB + 50))
        doc[0:1] = b"["
        doc[a:a + 1], doc[b:b + 1], doc[c:c + 1] = b"1", b",", b"2"
        # the next token is behind the slab: [1 ,2 ,3]  -- K2r of the next slab starts from these three
        yield bytes(doc) + b",3]"
        doc[a:a + 1], doc[b:b + 1], doc[c:c + 1] = b"[", b"]", b","  # brackets: [ [ ] ,3]
        yield bytes(doc) + b"3]"
        # the slab ends inside a string: its opening quote is the last structural, the two in front of it count
        doc[a:a + 1], doc[b:b + 1] = b"1", b","
        doc[c:] = b'"' + b"x" * (len(doc) - c - 1)
        yield bytes(doc) + b'"]'


@pytest.mark.parametrize("ndjson", [False, True])
def test_counting_pass_last_quote_in_every_step(oracle_native, ndjson):
    n = 0
    for doc in _quote_docs():
        same_as_oracle(oracle_native, doc, ndjson)
        same_as_oracle(oracle_native, doc + b"\n" + doc, ndjson)
        n += 1
    assert n == 2 * 13 * 4


@pytest.mark.parametrize("ndjson", [False, True])
def test_counting_pass_last_structurals_across_steps(oracle_native, ndjson):
    for doc in _last_docs():
        same_as_oracle(oracle_native, doc, ndjson)
        same_as_oracle(oracle_native, doc + b"\n" + doc + b"\n" + doc, ndjson)
