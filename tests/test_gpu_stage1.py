"""GPU parity tests for stage 1 + flatten (kernel K1) through the C ABI.

The CUDA path is compared with the CPU oracle bit for bit, and replays the same
reference goldens (G1..G10) the oracle is pinned on.
"""
import numpy as np
import pytest

from tests.util import SMALL_FILES, TAPE_FILES, golden, load_fixture, unhex

pytestmark = pytest.mark.gpu
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


# ---- reference goldens through the device code ---------------------------------------
def test_g1_finalize_structurals(ctx):
    for i, tc in enumerate(golden("G1_finalize_structurals")):
        got = ctx.finalize_structurals(tc["structurals"], tc["whitespace"], tc["quote_mask"], tc["quote_bits"], 0)
        assert got == (tc["expected_strls"], tc["expected_pseudo"]), i


def test_g2_newline_delimiters(ctx):
    g = golden("G2_newline_delimiters")
    nd = unhex(g["input"])
    for k, off in enumerate(range(0, len(nd) - 64, 64)):
        assert ctx.find_newline_delimiters(nd[off:off + 64], 0) == g["want"][k]
    q = bytearray(unhex(g["quoted_case"]["input"]))
    for p in g["quoted_case"]["newline_at"]:
        q[p] = 0x0A
    qm, _, _, _ = ctx.find_quote_mask_and_bits(bytes(q), 0, 0)
    assert ctx.find_newline_delimiters(bytes(q), qm) == g["quoted_case"]["want"]
    # and fused: the ndjson structural mask contains exactly the unquoted newline
    assert ctx._one(bytes(q), prev_pseudo=1, ndjson=1)[6] & (1 << 50)
    assert not ctx._one(bytes(q), prev_pseudo=1, ndjson=1)[6] & (1 << 10)


def test_g3_odd_backslash(ctx):
    for i, tc in enumerate(golden("G3_odd_backslash")):
        got = ctx.find_odd_backslash_sequences(unhex(tc["input"]), tc["prev_ends_odd"])
        assert got == (tc["expected"], tc["ends_odd_backslash"]), i
    for i in range(1, 129):
        t = b" " * (i - 1) + b'\\"' + b" " * (62 + 64)
        lo, c = ctx.find_odd_backslash_sequences(t[:64], 0)
        hi, c = ctx.find_odd_backslash_sequences(t[64:128], c)
        assert (lo, hi) == ((1 << i, 0) if i < 64 else (0, (1 << (i - 64)) & M64)), i


def test_g4_quote_mask_and_bits(ctx):
    g = golden("G4_quote_mask")
    for i, tc in enumerate(g["cases"]):
        # odd_ends in the table is 0 or 1: bit 0 set <=> the block before ended in an odd run
        got = ctx.find_quote_mask_and_bits(unhex(tc["input"]), tc["odd_ends"], 0)
        assert got == (tc["expected"], tc["quote_bits"], tc["piiq"], tc["error_mask"]), i
    for i, tc in enumerate(g["piiq_cases"]):
        assert ctx.find_quote_mask_and_bits(unhex(tc["input"]), 0, tc["piiq_in"])[2] == tc["piiq_out"], i


def test_g5_whitespace_and_structurals(ctx):
    for i, tc in enumerate(golden("G5_whitespace_structurals")):
        assert ctx.find_whitespace_and_structurals(unhex(tc["input"])[:64]) == (tc["ws"], tc["structurals"]), i


def test_g9_flatten_bits(ctx):
    for i, tc in enumerate(golden("G9_flatten_bits")):
        assert ctx.flatten_bits(tc["masks"])[0] == tc["expected"], i


def test_g10_demo_json_positions(ctx):
    g = golden("G10_stage1_marks")
    ok, deltas = ctx.find_structural_indices(unhex(g["demo_json"]))
    assert ok
    assert (np.cumsum(deltas.astype(np.int64)) - 1).tolist() == g["positions"]


def test_g7_tail_padding(ctx):
    msg = unhex(golden("G7_tail_padding")["msg"])
    for l in range(len(msg), 0, -1):
        ok, deltas = ctx.find_structural_indices(msg[:l])
        assert len(deltas) == l and int(deltas.astype(np.int64).sum()) - 1 == l - 1  # (':' last => not ok, by design)


def test_g8_twitter_count(ctx):
    g = golden("G8_twitter_loop")
    msg = load_fixture("twitter")
    ok, deltas = ctx.find_structural_indices(msg)
    assert ok and len(deltas) == g["count"]
    pos = len(msg) - 1
    for j, ch in enumerate(g["reversed_tail"]):
        assert msg[pos:pos + 1].decode() == ch
        pos -= int(deltas[len(deltas) - 1 - j])


# ---- differential tests against the oracle ---------------------------------------------
ALPHABET = np.frombuffer(b'{}[]:,"\\\\\\ \t\n\r ab019.-etrufalsn\x00\x1f\x7f\x80\xc3\xa9/', dtype=np.uint8)


def test_block_masks_random_vs_oracle(ctx, oracle):
    rng = np.random.default_rng(1234)
    n = 4096
    blocks = ALPHABET[rng.integers(0, len(ALPHABET), size=(n, 64))]
    blocks[:64] = ord("\\")  # all-backslash blocks
    blocks[64:128, :32] = ord("\\")
    carries = np.zeros((n, 4), dtype=np.uint64)
    carries[:, 0] = rng.integers(0, 2, n)
    carries[:, 1] = np.where(rng.integers(0, 2, n) == 1, np.uint64(M64), np.uint64(0))
    carries[:, 2] = rng.integers(0, 2, n)
    carries[:, 3] = rng.integers(0, 2, n)
    got = ctx.block_masks(blocks, carries)
    for i in range(n):
        blk = blocks[i].tobytes()
        po, pi, pp, nd = (int(x) for x in carries[i])
        oe, oc = oracle.find_odd_backslash_sequences(blk, po)
        qm, qb, pi2, em = oracle.find_quote_mask_and_bits(blk, oe, pi)
        ws, st = oracle.find_whitespace_and_structurals(blk)
        fin, pp2 = oracle.finalize_structurals(st, ws, qm, qb, pp)
        nl = oracle.find_newline_delimiters(blk, 0)
        if nd:
            fin |= nl & ~qm & M64
        want = [oe, qm, qb, em, ws, st, fin, nl, oc, pi2, pp2]
        assert [int(x) for x in got[i][:11]] == want, i


def _check(ctx, oracle, msg, ndjson):
    ok_g, d_g = ctx.find_structural_indices(msg, ndjson)
    ok_o, d_o = oracle.find_structural_indices(msg, ndjson)
    assert ok_g == ok_o
    if ok_o:
        assert len(d_g) == len(d_o)
        assert np.array_equal(d_g, d_o)
    else:
        # the reference stops handing chunks to stage 2 at the failing chunk
        # (stage1_find_marks_amd64.go:115-129 break before the channel send): prefix only
        assert len(d_g) >= len(d_o)
        assert np.array_equal(d_g[:len(d_o)], d_o)


@pytest.mark.parametrize("name", TAPE_FILES + SMALL_FILES + ["parking-citations"])
def test_fixture_deltas_vs_oracle(ctx, oracle_native, name):
    msg = load_fixture(name).strip()
    _check(ctx, oracle_native, msg, False)
    _check(ctx, oracle_native, msg, True)


def test_small_and_boundary_sizes(ctx, oracle_native):
    tw = load_fixture("twitter")
    for n in list(range(1, 70)) + [127, 128, 129, 2047, 2048, 2049, 8191, 8192, 8193, 16384, 16385, 98304, 98305, 200001]:
        _check(ctx, oracle_native, tw[:n], False)
    for doc in (b"{}", b"[]", b"[", b'"', b'"\\', b"\\", b" ", b"a", b'{"a":1}', b'["\\""]'):
        _check(ctx, oracle_native, doc, False)


def _geometry(ctx):
    import ctypes as C
    g = (C.c_uint32 * 4)()
    ctx.L.sj_test_geometry(g)
    return tuple(int(x) for x in g)  # block, step, slab, tile


def test_carries_across_slabs(ctx, oracle_native):
    """Backslash runs, escaped / unescaped quotes and pseudo-structural predecessors straddling every kind of edge of
    the stage-1 kernel: 64-byte block, 2 KiB step, slab (one warp's share of a tile: the odd-backslash and
    pseudo-predecessor carries are recovered from the 32 bytes in front of it, runs of 32 and more walk further back)
    and tile (the in-string state crosses it through look-back chain 1).  The edges come from the kernel's own
    constants (sj_test_geometry), so a change of geometry moves the test with it.
    find_subroutines_amd64_test.go:153-198 sweeps the same carry over a 128-byte window."""
    block, step, slab, tile = _geometry(ctx)
    assert (block, step) == (64, 2048) and tile % slab == 0 and slab % step == 0
    rng = np.random.default_rng(7)
    edges = [block, step, slab, 2 * slab, 5 * slab, tile - slab, tile, tile + slab, 2 * tile, 3 * tile + 2 * slab]
    runs = [1, 2, 3, 4, 5, 30, 31, 32, 33, 34, 35, 62, 63, 64, 65, 66, 95, 96, 97, 127, 128, 129, 200]
    n = 0
    for edge in edges:
        for run in runs:
            # `a` backslashes of the run sit in front of the edge, run - a behind it
            for a in sorted({0, 1, 2, run // 2, run - 2, run - 1, run} & set(range(0, run + 1))):
                pre = edge - 2 - a
                if pre < 0:
                    continue
                body = b'["' + b"x" * pre + b"\\" * run + b'"q\\\\", "tail",true , 12]'
                assert body[edge - a:edge - a + run] == b"\\" * run and (edge - a == 0 or body[edge - a - 1:edge - a] != b"\\")
                _check(ctx, oracle_native, body, False)
                n += 1
    assert n > 1000
    # a quote exactly at the last byte in front of an edge / the first byte behind it, behind k backslashes
    # (k >= 32 forces the walk of backslash_run_before for the quote's own escape state too)
    for edge in (slab, 3 * slab, tile, 2 * tile + slab):
        for k in (0, 1, 2, 3, 30, 31, 32, 33, 64, 65):
            for at in (edge - 1, edge):  # position of the quote
                pad = at - 2 - k
                _check(ctx, oracle_native, b'["' + b"y" * pad + b"\\" * k + b'","z"]', False)
                _check(ctx, oracle_native, b'["' + b"y" * pad + b"\\" * k + b'"  ,  "z"  ]', False)
    # pseudo-structural predecessor across an edge: the byte in front of the edge is whitespace / a structural /
    # a quote / an ordinary character, the byte behind it starts (or does not start) an atom
    for edge in (step, slab, tile, tile + 4 * slab):
        for last in (b" ", b",", b"[", b'"', b"x", b"\n", b":"):
            for first in (b"t", b"1", b"[", b'"', b" ", b"n"):
                head = b"[" + b"1," * ((edge - 8) // 2)
                head = head + b" " * (edge - 1 - len(head)) + last
                assert len(head) == edge
                _check(ctx, oracle_native, head + first + b'rue,"k" ]', False)
                _check(ctx, oracle_native, head + first + b'rue,"k" ]', True)
    # an open string across one and several tiles (chain 1 carries "in string" over tiles that hold no quote at all)
    for span in (tile // 2, tile, 3 * tile + 5):
        _check(ctx, oracle_native, b'{"k":"' + b"s" * span + b'","t":[1,2,{"u":null}]}', False)
        _check(ctx, oracle_native, b'{"k":"' + b"s" * span + b'\\","t":[1,2,{"u":null}]}', False)  # escaped closing quote: ends in string
    # random soup: every structural / escape class, sizes that leave partial slabs and partial tiles
    for n in (5000, slab, 20000, 70000, tile + 1, 300007):
        buf = ALPHABET[rng.integers(0, len(ALPHABET), size=n)].tobytes()
        _check(ctx, oracle_native, buf, False)
        _check(ctx, oracle_native, buf, True)


def test_large_replicated_input(ctx, oracle_native):
    """many slabs in flight on every SM: 64 MiB of twitter-shaped data, bit-exact deltas"""
    tw = load_fixture("twitter")
    k = 100
    msg = b"[" + b",".join([tw] * k) + b"]"
    _check(ctx, oracle_native, np.frombuffer(msg, dtype=np.uint8), False)


def test_ndjson_newlines(ctx, oracle_native):
    pk = load_fixture("parking-citations").strip()
    _check(ctx, oracle_native, b"\n".join([pk] * 40), True)
    _check(ctx, oracle_native, b'{"a":"x\ny"}\n\n{"b":2}', True)  # raw newline inside a string => stage-1 error


def test_control_char_error(ctx, oracle_native):
    for c in (0, 1, 9, 10, 13, 31):
        _check(ctx, oracle_native, b'{"a":"x' + bytes([c]) + b'y"}', False)
        _check(ctx, oracle_native, b'{"a" ' + bytes([c]) + b' :"xy"}', False)


def test_dense_structurals(ctx, oracle_native):
    """more than one structural per 4 bytes: the flatten's staging area (slab / 4 entries) overflows,
    so the mid-slab flush and the straight-to-global path are exercised (positions and deltas)"""
    docs = [
        b"[" * 150000 + b"]" * 150000,                      # every byte structural
        b"[" + b"[1," * 60000 + b"1" + b"]" * 60000 + b"]",  # 2 of 3 bytes
        b"[" + b",".join([b"[]"] * 90000) + b"]",             # all structural, no values
        b"[" + b",".join([b'{"a":[1,2],"b":{}}'] * 20000) + b"]",
        b"[" + b"1," * 30000 + b"[" * 5000 + b"]" * 5000 + b"," + b'"x"' * 1 + b"]",  # sparse then dense then sparse
    ]
    for d in docs:
        _check(ctx, oracle_native, d, False)
        _check(ctx, oracle_native, d, True)
