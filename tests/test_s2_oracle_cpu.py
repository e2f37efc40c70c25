"""CPU checks of the S2 oracle (tests/s2_oracle.py) that the device S2 codec is held to: CRC-32C against its check values,
the Snappy subset against an independent codec (pyarrow's `snappy`), every element code on purpose, and one rejection
per rule of the format."""
import random

import pytest

from tests import s2_oracle as s2
from tests.serialize_oracle import Rejected, Unsupported, uvarint
from tests.util import SMALL_FILES, TAPE_FILES, load_fixture

pa = pytest.importorskip("pyarrow")
SNAPPY = pa.Codec("snappy")


def _crc_sequential(data):
    r = s2.M32
    for b in data:
        r = s2._TL[(r ^ b) & 0xFF] ^ (r >> 8)
    return ~r & s2.M32


def test_crc32c_check_values():
    assert s2.crc32c(b"123456789") == 0xE3069283
    assert s2.crc32c(bytes(32)) == 0x8A9136AA
    assert s2.crc32c(b"") == 0
    c = 0xE3069283
    assert s2.masked_crc(b"123456789") == (((c >> 15) | (c << 17)) + 0xA282EAD8) & s2.M32


def test_crc32c_bulk_matches_the_sequential_loop():
    """the slices joined by shifts equal the byte loop, at every length around the slice count"""
    rnd = random.Random(5)
    for n in (0, 1, 1023, 1024 * 8 - 1, 1024 * 8, 1024 * 8 + 1, 70001, 200000):
        d = bytes(rnd.getrandbits(8) for _ in range(n))
        assert s2.crc32c(d) == _crc_sequential(d), n


def _samples():
    rnd = random.Random(1)
    yield "random", bytes(rnd.getrandbits(8) for _ in range(50000))
    yield "runs", b"".join(bytes([rnd.randrange(4)]) * rnd.randrange(1, 300) for _ in range(500))
    for name in SMALL_FILES + ["canada", "twitter", "update-center"]:
        yield name, load_fixture(name)[:300000]


@pytest.mark.parametrize("name,data", list(_samples()), ids=lambda x: x if isinstance(x, str) else "")
def test_oracle_decodes_pyarrow_snappy(name, data):
    for at in range(0, len(data), 65536):
        d = data[at:at + 65536]
        assert s2.decode_block(SNAPPY.compress(d, asbytes=True)) == d


@pytest.mark.parametrize("name,data", list(_samples()), ids=lambda x: x if isinstance(x, str) else "")
def test_pyarrow_decodes_the_oracle_encoder(name, data):
    st = s2.stream(data)
    assert s2.read(st, len(data)) == data
    at = 0
    for t, body in s2.chunks(st)[1:]:
        n = s2.decoded_len(body[4:]) if t == 0 else len(body) - 4
        d = SNAPPY.decompress(body[4:], decompressed_size=n, asbytes=True) if t == 0 else body[4:]
        assert d == data[at:at + n] and s2.masked_crc(d) == int.from_bytes(body[:4], "little")
        at += n
    assert at == len(data)


def _execute(ops):
    """the output of a list of ('lit', bytes) / ('copy', offset, length) byte by byte: the meaning of the elements,
    independent of the decoder"""
    out = bytearray()
    for op in ops:
        if op[0] == "lit":
            out += op[1]
        else:
            for _ in range(op[2]):
                out.append(out[-op[1]])
    return bytes(out)


def _every_code():
    """(elements, ops, snappy_subset) covering each literal length class, copy1 / copy2 / copy4 at their extreme offsets
    and lengths, overlapping copies at offsets 1 .. 33 and repeats of each length code"""
    rnd = random.Random(2)
    base = bytes(rnd.getrandbits(8) for _ in range(70000))
    cases = []
    for n in (1, 2, 59, 60, 61, 256, 257, 65536, 65537):
        cases.append(([s2.lit(base[:n])], [("lit", base[:n])], True))
    for nb in (1, 2, 3, 4):
        cases.append(([s2.lit_form(base[:200], nb)], [("lit", base[:200])], True))
    head = [s2.lit(base[:66000])]
    hops = [("lit", base[:66000])]
    for off, n in ((1, 4), (1, 11), (2047, 4), (2047, 11), (256, 7)):
        cases.append((head + [s2.copy1(off, n)], hops + [("copy", off, n)], True))
    for off, n in ((1, 1), (1, 64), (65535, 1), (65535, 64), (300, 33)):
        cases.append((head + [s2.copy2(off, n)], hops + [("copy", off, n)], True))
    for off, n in ((1, 1), (65999, 64), (65536, 1), (66000, 64)):
        cases.append((head + [s2.copy4(off, n)], hops + [("copy", off, n)], True))
    for off in range(1, 34):  # overlapping copies: the run repeats the last `off` bytes
        cases.append(([s2.lit(base[:off]), s2.copy2(off, 64), s2.copy1(off, 11) if off < 2048 else s2.copy2(off, 11)],
                      [("lit", base[:off]), ("copy", off, 64), ("copy", off, 11)], True))
    for n in (4, 5, 6, 7, 8, 9, 263, 264, 65539, 65540, 65541, 70000, 300000):  # repeats of each length code
        cases.append(([s2.lit(base[:40]), s2.copy2(7, 5), s2.repeat(n)], [("lit", base[:40]), ("copy", 7, 5), ("copy", 7, n)],
                      False))
    return cases


def test_every_code_round_trips():
    seen = set()
    for elements, ops, snappy in _every_code():
        want = _execute(ops)
        body = s2.block(len(want), *elements)
        assert s2.decode_block(body) == want
        if snappy:
            assert SNAPPY.decompress(body, decompressed_size=len(want), asbytes=True) == want
        for e in elements:
            seen.add((e[0] & 3, e[0] >> 2 if e[0] & 3 == 0 and e[0] >> 2 >= 60 else e[0] >> 2 & 7 if e[0] & 3 == 1 and e[1] == 0 else None))
        st = s2.IDENT + s2.compressed(want, body)
        assert s2.read(st, len(want)) == want
    assert {(0, 60), (0, 61), (0, 62), (0, 63)} <= seen
    assert {(1, k) for k in range(8)} <= seen
    assert {(2, None), (3, None)} <= seen


def _rejected(st, want):
    with pytest.raises(Rejected):
        s2.read(st, want)


def test_rejection_matrix():
    d = b"abcdefgh" * 40
    good = s2.compressed(d)
    crc = s2.masked_crc(d).to_bytes(4, "little")
    n = len(d)
    assert s2.read(s2.IDENT + good, n) == d
    # block rules
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.repeat(n))), n)                        # repeat with no offset
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.copy2(0, 8))), n)                      # copy offset 0
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]), s2.copy2(9, 8))), n)       # offset past the output
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))[:-1]), n)                  # literal past the body
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))[:2] + b"\xf0"), n)         # length bytes past the body
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(4, s2.lit(d[:8]))), 4)                       # literal past n
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(8, s2.lit(d[:4]), s2.copy2(4, 8))), 8)       # copy past n
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))), 8)                       # ends short of n
    _rejected(s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]), b"\x01")), 8)              # copy1 past the body
    _rejected(s2.IDENT + s2.chunk(0, crc + b"\xff" * 11), 8)                                     # length overflows
    # stream rules
    _rejected(good, n)                                                                           # no identifier first
    _rejected(s2.chunk(0x80, b"") + s2.IDENT + good, n)                                          # skippable first
    _rejected(s2.chunk(0xFF, b"S2sTwX") + good, n)                                               # bad identifier
    _rejected(s2.chunk(0xFF, b"S2sTwO!") + good, n)                                              # identifier length
    _rejected(s2.IDENT + s2.chunk(0, crc[:3]), n)                                                # compressed shorter than 4
    _rejected(s2.IDENT + s2.chunk(1, crc[:3]), n)                                                # stored shorter than 4
    big = bytes(s2.MAX_DECODED + 1)
    _rejected(s2.IDENT + s2.chunk(0, crc + uvarint(len(big)) + s2.lit(b"\0") + s2.repeat(4)), len(big))  # > 4 MiB
    _rejected(s2.IDENT + s2.chunk(1, s2.masked_crc(big).to_bytes(4, "little") + big), len(big))          # stored > 4 MiB
    sn = bytes(65537)
    _rejected(s2.SNAPPY_IDENT + s2.stored(sn), len(sn))                                           # > 64 KiB after sNaPpY
    assert s2.read(s2.SNAPPY_IDENT + s2.stored(sn[:65536]), 65536) == sn[:65536]
    assert s2.read(s2.SNAPPY_IDENT + s2.IDENT + s2.stored(sn), len(sn)) == sn                     # S2 again
    _rejected(s2.IDENT + s2.chunk(0, (int.from_bytes(crc, "little") ^ 1).to_bytes(4, "little") + good[8:]), n)  # CRC
    _rejected(s2.IDENT + s2.stored(d)[:4] + crc[::-1] + d, n)                                     # stored CRC
    for t in (0x02, 0x7F):
        _rejected(s2.IDENT + s2.chunk(t, b"") + good, n)                                          # reserved unskippable
    _rejected(s2.IDENT + good[:-1], n)                                                            # chunk past the block
    _rejected(s2.IDENT + good, n + 1)                                                             # out of chunks
    _rejected(s2.IDENT + good + b"\x00\x00", n + 1)                                               # header cut short
    _rejected(b"", 1)
    # what is accepted
    for t in (0x80, 0x99, 0xFE):
        assert s2.read(s2.IDENT + s2.chunk(t, b"anything") + good, n) == d                        # skippable
    assert s2.read(s2.IDENT + s2.IDENT + good, n) == d                                            # identifier repeats
    assert s2.read(s2.IDENT + good + b"trailing garbage", n) == d                                 # nothing behind is read
    assert s2.read(s2.IDENT + good + s2.chunk(0x05, b""), n) == d
    assert s2.read(s2.IDENT + good, 10) == d[:10]                                                 # a chunk past the size
    _rejected(s2.IDENT + s2.chunk(0, crc + good[8:-1] + b"!"), 10)                               # ... is still checked in full
    assert s2.read(b"garbage", 0) == b""                                                          # size 0 reads nothing
    assert s2.read(s2.IDENT + s2.chunk(0, s2.masked_crc(b"").to_bytes(4, "little") + b"\0") + good, n) == d  # empty chunk


def test_inflate_and_compress_whole_streams():
    """compress() of an uncompressed stream gives S2 message, tags and values blocks whose inflation is the stream; a
    zstd block stays unsupported, the uncompressed-size-0 S2 block reads nothing"""
    from tests import serialize_oracle as so
    from tests.tape_builder import TapeBuilder
    b = TapeBuilder()
    b.open("r")
    b.open("{")
    for i in range(300):
        b.string(b"key%d" % (i % 7))
        b.number("l", i)
    b.close()
    b.close()
    tape, strs, msg = b.build()
    src = so.serialize(tape, strs, msg)
    for cs in (s2.CHUNK, 1000, 1 << 20):
        fast = s2.compress(src, cs)
        assert fast != src and s2.inflate(fast) == src
        assert s2.device_result(fast) == so.device_result(src)
    empty = so.serialize([], b"", b"")
    assert s2.inflate(s2.compress(empty)) == empty
    for typ, exc in ((1, None), (2, Unsupported)):
        body = uvarint(0) + b"\0\0" + uvarint(0) + uvarint(2) + bytes([typ]) + b"x" + (uvarint(0) + b"\0") * 2
        st = b"\3" + uvarint(len(body)) + body
        if exc:
            with pytest.raises(exc):
                s2.inflate(st)
        else:
            assert s2.device_result(st) == ([], b"", b"")
