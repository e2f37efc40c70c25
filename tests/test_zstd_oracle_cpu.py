"""CPU tests of tests/zstd_oracle.py, the zstd restatement the device decoder is checked against: XXH64, every golden
.zst fixture, pyarrow's zstd output at several levels and in streaming frames, constructed frames from the oracle's own
writer (every literal and table mode, treeless and repeat-mode blocks, the literal-length-0 offset shift, skippable and
concatenated frames), one rejection per acceptance rule, and the mode-aware stream oracle."""
import glob
import os
import random

import pytest

from tests import s2_oracle as s2
from tests import serialize_oracle as so
from tests import zstd_oracle as zo
from tests.util import load_fixture

pa = pytest.importorskip("pyarrow")
ZSTD = pa.Codec("zstd")
DATA = os.path.join(os.path.dirname(__file__), "golden", "data")


def _pa(frame, n):
    return ZSTD.decompress(frame, decompressed_size=n, asbytes=True)


def test_xxh64_check_values():
    assert zo.xxh64(b"") == 0xEF46DB3751D8E999
    assert zo.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert zo.xxh64(b"abc") == 0x44BC2CF5AD770999
    assert zo.xxh64(b"Nobody inspects the spammish repetition") == 0xFBCEA83C8A378BF1


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(DATA, "*.zst"))),
                         ids=os.path.basename)
def test_golden_fixtures(path):
    b = open(path, "rb").read()
    got = zo.decode(b)
    assert _pa(b, len(got)) == got


@pytest.mark.parametrize("level", [1, 3, 9, 19])
def test_pyarrow_levels(level):
    rnd = random.Random(level)
    c = pa.Codec("zstd", compression_level=level)
    for d in (load_fixture("twitter"), load_fixture("citm_catalog")[:200000], bytes(rnd.randrange(256) for _ in range(70000)),
              b"ab" * 100000, b"", b"x"):
        assert zo.decode(c.compress(d, asbytes=True)) == d


def test_pyarrow_streaming_frames():
    for d in (load_fixture("twitter"), load_fixture("canada")[:300000]):
        bo = pa.BufferOutputStream()
        with pa.CompressedOutputStream(bo, "zstd") as s:
            s.write(d)
        f = bo.getvalue().to_pybytes()
        assert (f[4] & 0x20) == 0  # a window descriptor, no single segment
        assert zo.decode(f) == d


# ---- constructed frames ---------------------------------------------------------------------------------------------
W = [4, 3, 2, 1, 1, 0, 0, 0]  # direct weights of symbols 0 .. 7 (8's, 5, is implied); literals drawn from them
FSE_LL = ([12, 8, 4, 3, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, -1] + [0] * 19, 5)


def _lits(n, seed):
    rnd = random.Random(seed)
    return bytes(rnd.choice([0, 1, 2, 3, 4, 8]) for _ in range(n))


def _exec(lit, seqs, rep=None):
    """the bytes a block with these literals and (ll, ml, offset_value) sequences decodes to, on `out`"""
    out = bytearray()
    rep = rep or [1, 4, 8]
    li = 0
    for ll, ml, ofv in seqs:
        out += lit[li:li + ll]
        li += ll
        o = zo.apply_offset(rep, ll, ofv)
        for _ in range(ml):
            out.append(out[-o])
    out += lit[li:]
    return bytes(out), rep


def constructed_frames():
    """(name, frame, decoded bytes) of frames from the oracle's writer"""
    out = []
    lit = _lits(300, 1)
    seqs = [(10, 50, 3 + 4), (0, 60, 1), (7, 40, 3 + 9), (3, 80, 2), (0, 40, 2), (2, 30, 1)]
    content, _ = _exec(lit, seqs)
    for kind, lname in ((0, "raw"), (1, "rle"), (2, "huf1"), (4, "huf4")):
        L = lit if kind != 1 else bytes([lit[0]]) * 300
        c, _ = _exec(L, seqs)
        ls = zo.literals_section(L, min(kind, 2), W if kind >= 2 else None, streams=4 if kind == 4 else 1)
        body = ls + zo.encode_sequences(seqs)
        out.append(("lit-" + lname, zo.frame_bytes([zo.block(body, 2, True)], c, checksum=True), c))
    # treeless: block 2 reuses block 1's table; repeat-mode tables; RLE and FSE table modes
    lit2 = _lits(200, 2)
    s1 = [(5, 4, 3 + 2), (5, 4, 3 + 2)]
    s2_ = [(6, 5, 3 + 3), (1, 4, 1)]
    b1 = zo.literals_section(lit, 2, W) + zo.encode_sequences(s1, (2, 1, 0), [FSE_LL, None, None])
    b2 = zo.literals_section(lit2, 3, W) + zo.encode_sequences(s2_, (3, 0, 3), [FSE_LL, None, zo.ML_DEFAULT])
    c1, rep = _exec(lit, s1)
    c2, _ = _exec(lit2, s2_, rep)
    # the second block's matches reach back into the first: execute on the joined output
    full = bytearray(c1)
    li, r = 0, list(rep)
    for ll, ml, ofv in s2_:
        full += lit2[li:li + ll]
        li += ll
        o = zo.apply_offset(r, ll, ofv)
        for _ in range(ml):
            full.append(full[-o])
    full += lit2[li:]
    full = bytes(full)
    out.append(("treeless-repeat", zo.frame_bytes([zo.block(b1), zo.block(b2, 2, True)], full), full))
    # the literal-length-0 shift: offset_value 1 is rep2, 2 rep3, 3 rep1 - 1
    lit3 = b"abcdefgh" * 4
    for name, sq in (("ll0-rep2", [(10, 50, 3 + 4), (0, 60, 1)]), ("ll0-rep3", [(8, 40, 3 + 6), (1, 30, 3 + 2), (0, 50, 2)]),
                     ("ll0-rep1-minus-1", [(8, 50, 3 + 6), (0, 60, 3)])):
        c3, _ = _exec(lit3, sq)
        body = zo.literals_section(lit3, 0) + zo.encode_sequences(sq)
        out.append((name, zo.frame_bytes([zo.block(body, 2, True)], c3), c3))
    # raw and RLE blocks, an empty sequences section, a streaming-shaped header, skippable and concatenated frames
    e = zo.block(zo.literals_section(b"hello", 0) + b"\0")
    f = zo.frame_bytes([zo.block(b"raw!", 0), zo.block(b"", 1, size=7) + b"z"[:0] if False else zo.block(b"z", 1, size=7), e,
                        zo.block(b"", 0, True)], b"raw!" + b"z" * 7 + b"hello", window_log=20)
    out.append(("raw-rle-empty-seq", f, b"raw!" + b"z" * 7 + b"hello"))
    # a raw block larger than the window: RFC 8878 limits it, libzstd (and this decoder) accept it
    wide = bytes(range(256)) * 8
    out.append(("raw-over-window", zo.frame_bytes([zo.block(wide, 0, True)], wide, window_log=10, fcs=False), wide))
    out.append(("no-fcs", zo.frame_bytes([zo.block(b"abc", 0, True)], b"abc", window_log=10, fcs=False), b"abc"))
    cat = zo.skippable(b"skip me", 3) + out[0][1] + zo.skippable(b"") + out[-1][1]
    out.append(("skippable-concatenated", cat, out[0][2] + b"abc"))
    big = load_fixture("twitter")[:100000]
    out.append(("pyarrow-concatenated", ZSTD.compress(big, asbytes=True) + ZSTD.compress(big[:777], asbytes=True), big + big[:777]))
    return out


@pytest.mark.parametrize("name,frame,want", constructed_frames(), ids=lambda x: x if isinstance(x, str) else "")
def test_constructed_frames(name, frame, want):
    assert zo.decode(frame) == want
    assert _pa(frame, len(want)) == want


def rejected_frames():
    """(name, frame, the block size it is read as) of frames the oracle rejects"""
    good = zo.frame_bytes([zo.block(b"abc", 0, True)], b"abc")
    out = []

    def flip(at, v, name):
        m = bytearray(good)
        m[at] = v
        out.append((name, bytes(m), 3))
    flip(0, 0x29, "magic")
    flip(4, good[4] | 8, "reserved-bit")
    out.append(("dictionary-id", zo.MAGIC.to_bytes(4, "little") + bytes([0x21, 5, 3]) + zo.block(b"abc", 0, True), 3))
    out.append(("fcs-mismatch", zo.frame_bytes([zo.block(b"abc", 0, True)], b"abcd"), 3))
    out.append(("checksum", zo.frame_bytes([zo.block(b"abc", 0, True)], b"abc", checksum=True)[:-1] + b"\0", 3))
    out.append(("reserved-block-type", zo.frame_bytes([((3 << 3) | 6 | 1).to_bytes(3, "little") + b"abc"], b"abc"), 3))
    big = zo.literals_section(b"a" * 1995, 0) + b"\0"
    out.append(("block-over-window", zo.frame_bytes([zo.block(big, 2, True)], b"a" * 1995, window_log=10, fcs=False), 1995))
    out.append(("treeless-first", zo.frame_bytes([zo.block(zo.literals_section(b"\0\1", 3, W) + b"\0", 2, True)], b"\0\1"), 2))
    out.append(("repeat-first", zo.frame_bytes([zo.block(zo.literals_section(b"ab", 0) + zo.encode_sequences(
        [(2, 3, 1 + 3)], (3, 0, 0), [zo.LL_DEFAULT, None, None]), 2, True)], b"ababa"), 5))
    out.append(("offset-before-frame", zo.frame_bytes([zo.block(zo.literals_section(b"ab", 0) + zo.encode_sequences(
        [(2, 3, 3 + 3)]), 2, True)], b"ab???"), 5))
    body = zo.literals_section(b"ab", 0) + zo.encode_sequences([(2, 3, 1 + 3)])
    out.append(("bitstream-not-exact", zo.frame_bytes([zo.block(body + b"\1", 2, True)], b"ababa"), 5))
    out.append(("lit-lengths-past-literals", zo.frame_bytes([zo.block(zo.literals_section(b"ab", 0) + zo.encode_sequences(
        [(3, 3, 1 + 3)]), 2, True)], b"ababab"), 6))
    out.append(("bytes-behind-empty-sequences", zo.frame_bytes([zo.block(zo.literals_section(b"ab", 0) + b"\0\0", 2, True)], b"ab"), 2))
    lit3 = b"abcdefgh" * 4
    sq = [(1, 50, 1), (0, 60, 3)]  # rep1 = 1, then rep1 - 1 = 0
    out.append(("rep1-minus-1-zero", zo.frame_bytes([zo.block(zo.literals_section(lit3, 0) + zo.encode_sequences(sq), 2, True)],
                                                    b"?" * 143), 143))
    late = zo.literals_section(b"ab", 0) + zo.encode_sequences([(2, 300, 3 + 1), (0, 50, 3 + 5000)])
    out.append(("late-offset-before-frame", zo.frame_bytes([zo.block(late, 2, True)], b"?" * 352), 352))
    rle = zo.literals_section(b"r" * 100000, 1) + b"\0"
    out.append(("literals-over-size", zo.frame_bytes([zo.block(rle, 2, True)], b"r" * 1000), 1000))
    out.append(("size-past-blocks", good, 1 << 40))
    out.append(("truncated", good[:-1], 3))
    out.append(("trailing-garbage", good + b"\1", 3))
    out.append(("skippable-cut", zo.skippable(b"abcdef")[:-1], 0))
    out.append(("wrong-size", good, 4))
    return out


@pytest.mark.parametrize("name,frame,n", rejected_frames(), ids=lambda x: x if isinstance(x, str) else "")
def test_rejections(name, frame, n):
    with pytest.raises(zo.ZstdError):
        zo.read_block(frame, n)
    # where libzstd has the same rule, pyarrow rejects the frame too
    if name not in ("wrong-size", "skippable-cut", "repeat-first", "trailing-garbage", "size-past-blocks",
                    "literals-over-size"):
        with pytest.raises(Exception):
            got = _pa(frame, n)
            assert len(got) == n


def test_stream_oracle_modes():
    """the mode-aware stream oracle inflates S2 and zstd blocks; serialize_oracle and s2_oracle keep their verdicts"""
    from tests.tape_builder import TapeBuilder
    b = TapeBuilder()
    b.open("r")
    b.open("{")
    for i in range(300):
        b.string(b"key%d" % (i % 7))
        b.number("l", i * 3)
    b.close()
    b.close()
    tape_stream = so.serialize(*b.build())
    v, ts, blocks = s2._blocks(tape_stream)
    best = s2._assemble(v, ts, [blocks[0]] + [(raw, 2, ZSTD.compress(d, asbytes=True) if d else b"") for raw, _, d in blocks[1:]])
    assert zo.inflate(best) == tape_stream
    assert zo.device_result(best, 3) == so.device_result(tape_stream)
    with pytest.raises(so.Unsupported):
        zo.device_result(best, 1)
    with pytest.raises(so.Unsupported):
        s2.inflate(best)

