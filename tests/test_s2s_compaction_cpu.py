"""K2r's Strings.B compaction and tape slots at their edges, run by the 32-fiber warp emulation (tests/emu/s2s_emu.cpp)
and compared bit for bit with the oracle.

The compaction stores every staging word once, by the lane that holds its first byte; a lane that keeps 0-3 bytes can
share a word with the lanes around it, so runs of such lanes are laid out here in every combination, at every 16-byte
phase of the destination (`shift`: the string bytes in front of the step, mod 16).  The emission loops fold the record
starts into the two-word events where no record starts on a number; records that start with each kind of value sit at
lane (64-byte) and half (32-byte) edges."""
import itertools

import numpy as np
import pytest

from tests.emu_util import same_as_oracle

BLOCK = 64


def _block(keep):
    """one 64-byte block of an array's body that adds `keep` bytes to Strings.B (None: whitespace only)"""
    if keep is None:
        return b" " * BLOCK
    assert keep <= BLOCK - 3
    return (b'"' + b"k" * keep + b'",').ljust(BLOCK, b" ")


def _array(phase, keeps):
    """an array whose first block puts `phase` string bytes in front of the rest, then one block per entry of keeps"""
    head = (b'["' + b"p" * phase + b'",').ljust(BLOCK, b" ")
    return head + b"".join(_block(k) for k in keeps) + b'"end"]'


@pytest.mark.parametrize("phase", range(16))
def test_seam_words_every_combination(oracle_native, phase):
    """three consecutive lanes that keep 0, 1, 2 or 3 bytes or none at all, in every combination"""
    keeps = [k for combo in itertools.product([None, 0, 1, 2, 3], repeat=3) for k in combo]
    assert same_as_oracle(oracle_native, _array(phase, keeps)) == 0


@pytest.mark.parametrize("phase", range(16))
def test_seam_words_random_runs(oracle_native, phase):
    """long runs of lanes that keep few bytes, mixed with lanes that fill whole words"""
    rng = np.random.default_rng(phase)
    choices = [None, 0, 1, 2, 3, 4, 5, 7, 8, 13, 30, 61]
    keeps = [choices[i] for i in rng.integers(0, len(choices), 400)]
    keeps += [1] * 40 + [0, 1] * 20 + [None, 3] * 20
    assert same_as_oracle(oracle_native, _array(phase, keeps)) == 0


@pytest.mark.parametrize("phase", range(16))
def test_steps_all_kept_and_none_kept(oracle_native, phase):
    """steps inside one long string (every byte kept), then steps without a string byte"""
    doc = b'["' + b"p" * phase + b'","' + bytes(b"abcdefghij"[i % 10] for i in range(3 * 6144 + 77)) + b'",' + b"1," * 5000 + b"2]"
    assert same_as_oracle(oracle_native, doc) == 0
    doc = b"[" + b" " * (4096 + phase) + b'"' + b"x" * (2048 * 3) + b'"]'
    assert same_as_oracle(oracle_native, doc) == 0


def _records(kinds, pads):
    return b"\n".join(b" " * p + k for k, p in zip(kinds, pads))


@pytest.mark.parametrize("phase", range(0, 16, 5))
def test_record_starts_at_lane_and_half_edges(oracle_native, phase):
    """NDJSON records that start with a bracket, at every offset of a 64-byte block (so on both halves' edges),
    behind string bytes of every phase"""
    recs = [b'{"a":"' + b"s" * phase + b'"}', b'["x",1,true]', b'{"k":[null,"v"]}', b"[[],{}]", b'["a"]']
    kinds, pads = [], []
    for off in range(BLOCK + 2):
        for r in recs:
            kinds.append(r)
            pads.append(off)
    assert same_as_oracle(oracle_native, _records(kinds, pads), True) == 0


@pytest.mark.parametrize("first", [b"1", b"-2.5e3", b"true", b"null", b"false", b'"s"', b"{}", b"[7]"])
def test_records_that_start_with_each_kind_of_value(oracle_native, first):
    """a record that starts with a number, an atom, a string or a bracket (the first three are rejected at the top
    level; the verdict must match) at lane and half edges, between records that start with brackets"""
    for off in (0, 1, 30, 31, 32, 33, 62, 63):
        lead = b'{"a":"b"}\n' * 3
        pad = (off - len(lead)) % BLOCK
        doc = lead + b" " * pad + first + b'\n{"c":1}\n[2,"d"]'
        same_as_oracle(oracle_native, doc, True)
        # the same record inside a longer stream, behind a string byte phase of 1..3
        doc = b'{"x":"' + b"y" * (off % 4) + b'"}\n' + b" " * off + first + b"\n" + b'["e"]\n' * 40
        same_as_oracle(oracle_native, doc, True)
