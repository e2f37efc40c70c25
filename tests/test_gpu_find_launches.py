"""GPU test of the device find's kernel launches per call for one mix of every cell family: a STRING, a JSON, a numeric
list (ARRAY_FLOAT64) and a string list (ARRAY_STRING) path in one call, over the roots and over array rows.  The counts
are the per-call formulas in the headers of sj_find.inl and sj_find_rows.inl."""
import ctypes as C

import pytest

from tests import find_json_oracle as fj
from tests import find_lists_oracle as fl
from tests import find_oracle as fo

pytestmark = pytest.mark.gpu

RECORD = b'{"s":"x","j":{"a":1},"f":[1.5,2],"t":["p","q"]}'
PATHS = [[b"s"], [b"j"], [b"f"], [b"t"]]
KINDS = [fo.STRING, fj.JSON, fl.ARRAY_FLOAT64, fl.ARRAY_STRING]

# one call that writes the columns (sj_find.inl): KF3 (1); KJ0's reduce, two scans and prefix (4); the JSON path's
# KJ1 + 2 scans, KJ2, K2d, KM3 + 2 scans, KJ4 + 2 scans and KJ5 (12 + a_j, a_j = 0: its 3 cells of 6 words are at most
# 32 words); the numeric list's KL2 and KL4 (2); the string list's KJ1 + 2 scans, KL2, KL3 + 2 scans and KL4 (8); the
# element counts' reduce, two scans and prefix (4); KF4 + 2 scans (3); KF5 (1), KJ6 (1), KL5 (1), KL6 for each list
# path and KL7 for the string list (3).  A call that only asks for the sizes stops in front of KF5.
MEASURE = 1 + 4 + 12 + 2 + 8 + 4 + 3
EMIT = 1 + 1 + 1 + 3
FOREIGN = 7  # KM1, KC1a and KC1b with their scans: the roots of a tape the context did not parse
# array rows (sj_find_rows.inl), with array words: KR1 and the records' word scan (5), KJ1 + 2 scans, KR2, KR3 + 2
# scans and KR4 (8), KR5 and the row counts' scan (5), KR6 and KR7 (2) in front of the find's passes over the rows, and
# KR8 (1) in front of KF5
ROWS = 5 + 8 + 5 + 2
KR8 = 1


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _own_tape(ctx, msg, flags):
    """msg parsed into HBM by sj_parse_device: the context's own tape, strings and message as tensors"""
    import torch
    d_msg = torch.full((len(msg) + 4096,), 0x20, dtype=torch.uint8, device="cuda")
    d_msg[:len(msg)].copy_(torch.frombuffer(bytearray(msg), dtype=torch.uint8))
    tcap, scap = C.c_size_t(0), C.c_size_t(0)
    ctx.L.sj_bounds(len(msg), C.byref(tcap), C.byref(scap))
    d_tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    d_str = torch.empty(scap.value, dtype=torch.uint8, device="cuda")
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    assert ctx.L.sj_parse_device(ctx.h, d_msg.data_ptr(), len(msg), flags, d_tape.data_ptr(), d_tape.numel(), C.byref(tl),
                                 d_str.data_ptr(), d_str.numel(), C.byref(sl)) == 0
    return d_tape[:tl.value], d_str[:sl.value], d_msg[:len(msg)]


def test_mixed_paths_launches(ctx):
    """find_device without `out` asks for the sizes, then writes the columns: two calls"""
    tape, strs, msg = _own_tape(ctx, b"\n".join([RECORD] * 3), 3)
    l0 = ctx.launches()
    rc, rows, cols = ctx.find_device(tape, strs, msg, PATHS, KINDS)
    l1 = ctx.launches()
    rc2, rows2, _ = ctx.find_device(tape.clone(), strs, msg, PATHS, KINDS)
    l2 = ctx.launches()
    assert (rc, rows, rc2, rows2) == (0, 3, 0, 3)
    assert [int(c.status.max()) for c in cols] == [fo.OK] * 4
    assert (l1 - l0, l2 - l1) == (2 * MEASURE + EMIT, 2 * (FOREIGN + MEASURE) + EMIT)


def test_mixed_paths_under_a_row_path_launches(ctx):
    """the same mix over the elements of every record's array at a row path: two calls each"""
    tape, strs, msg = _own_tape(ctx, b'{"rows":[' + b",".join([RECORD] * 3) + b"]}", 2)
    l0 = ctx.launches()
    rc, records, rows, index, cols = ctx.find_rows_device(tape, strs, msg, [b"rows"], PATHS, KINDS)
    l1 = ctx.launches()
    rc2, records2, rows2, _, _ = ctx.find_rows_device(tape.clone(), strs, msg, [b"rows"], PATHS, KINDS)
    l2 = ctx.launches()
    assert (rc, records, rows, rc2, records2, rows2) == (0, 1, 3, 0, 1, 3)
    assert [int(c.status.max()) for c in cols] == [fo.OK] * 4
    assert (l1 - l0, l2 - l1) == (2 * (ROWS + MEASURE) + KR8 + EMIT, 2 * (FOREIGN + ROWS + MEASURE) + KR8 + EMIT)
