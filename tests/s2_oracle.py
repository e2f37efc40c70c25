"""The S2 stream of the Serializer's CompressFast blocks (parsed_serialize.go:791-833 encBlock, :697-756 decBlock),
restated as plain sequential Python.  Test infrastructure: the expected output of the device decoder (s2.cuh KX1 / KX2),
a checker of what the device encoder (KC1 / KC2) writes, and builders of streams with every code and chunk type.

The S2 sources are not part of this project.  The rules below restate the published Snappy / S2 framing and block
formats together with the chunk loop of s2.Reader; the Snappy subset of the block format is also checked against an
independent decoder (pyarrow's `snappy` codec), the S2 repeat code and the reader's rules rest on this restatement:

Block (a chunk's body behind its CRC): uvarint(decoded length n), then elements.
  tag & 3 == 0  literal: length (tag >> 2) + 1 below 60; 60 .. 63: 1 .. 4 little-endian length bytes follow, + 1
  tag & 3 == 1  copy, 1-byte offset: length 4 + ((tag >> 2) & 7), offset (tag >> 5) << 8 | next byte.  Offset 0 is an
                S2 repeat of the last offset, its length code: 0 .. 4 -> 4 .. 8; 5 -> 1 byte + 8; 6 -> u16 + 260;
                7 -> u24 + 65540
  tag & 3 == 2  copy, 2-byte LE offset; tag & 3 == 3  copy, 4-byte LE offset: length (tag >> 2) + 1
  rejected: a copy whose offset is 0 (a repeat with no earlier offset) or beyond the bytes produced, anything that runs
  past the body or past n, output that does not end at exactly n.
Stream: chunks of a type byte and a 3-byte LE length.  The first chunk is the identifier 0xff, length 6, "S2sTwO" or
  "sNaPpY" (then a chunk that decodes to more than 64 KiB is rejected); it may repeat.  0x00 compressed (4-byte CRC +
  block), 0x01 stored (4-byte CRC + bytes): rejected when shorter than 4, decoding to more than 4 MiB or with a CRC that
  does not match.  0x80 .. 0xfe are skipped, 0x02 .. 0x7f rejected.  Chunks are read in order until the block's
  uncompressed size is filled; a chunk that is only partly needed is still decoded and checked in full, nothing behind
  it is read.  Running out of chunks first is rejected; a block of size 0 reads nothing.
CRC: CRC-32C (Castagnoli), masked as ((c >> 15) | (c << 17)) + 0xa282ead8.
"""
import numpy as np

from tests import serialize_oracle as so
from tests.serialize_oracle import Rejected, Unsupported, uvarint

M32 = 0xFFFFFFFF
POLY = 0x82F63B78
IDENT = b"\xff\x06\x00\x00S2sTwO"
SNAPPY_IDENT = b"\xff\x06\x00\x00sNaPpY"
MAX_DECODED = 4 << 20
SNAPPY_MAX_DECODED = 65536
CHUNK = 65536  # what the device encoder cuts its input into


# ---- CRC-32C --------------------------------------------------------------------------------------------------------
def _table():
    t = []
    for i in range(256):
        r = i
        for _ in range(8):
            r = (r >> 1) ^ (POLY if r & 1 else 0)
        t.append(r)
    return np.array(t, dtype=np.uint32)


_T = _table()
_TL = [int(x) for x in _T]


def _mul(a, b):
    """a * b mod P, reflected (bit 31 is x^0)"""
    p = 0
    for i in range(32):
        if a & (0x80000000 >> i):
            p ^= b
        b = (b >> 1) ^ (POLY if b & 1 else 0)
    return p


def _shift(r, n):
    """register r carried over n zero bytes: r * x^(8n)"""
    x = 0x00800000  # x^8
    while n:
        if n & 1:
            r = _mul(x, r)
        x = _mul(x, x)
        n >>= 1
    return r


def _raw(data):
    """the CRC register over data from 0 (no final xor): slices run side by side in numpy and are joined by shifts"""
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    r, done = 0, 0
    S = 1024
    L = len(a) // S
    if L >= 8:
        m = a[:S * L].reshape(S, L)
        regs = np.zeros(S, dtype=np.uint32)
        for j in range(L):
            regs = _T[(regs ^ m[:, j]) & 0xFF] ^ (regs >> np.uint32(8))
        xL = _shift(0x80000000, L)
        for v in regs.tolist():
            r = _mul(xL, r) ^ v
        done = S * L
    for b in a[done:].tolist():
        r = _TL[(r ^ b) & 0xFF] ^ (r >> 8)
    return r


def crc32c(data):
    return ~(_raw(data) ^ _shift(M32, len(data))) & M32


def masked_crc(data):
    c = crc32c(data)
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & M32


# ---- block elements -------------------------------------------------------------------------------------------------
def lit(data):
    """a literal element: the shortest length form"""
    x = len(data) - 1
    if x < 60:
        return bytes([x << 2]) + bytes(data)
    nb = (x.bit_length() + 7) // 8
    return bytes([(59 + nb) << 2]) + x.to_bytes(nb, "little") + bytes(data)


def lit_form(data, nb):
    """a literal with its length in nb = 1 .. 4 extra bytes (60 .. 63), whatever it is"""
    return bytes([(59 + nb) << 2]) + (len(data) - 1).to_bytes(nb, "little") + bytes(data)


def copy1(off, n):
    assert 4 <= n <= 11 and 1 <= off < 2048
    return bytes([1 | (n - 4) << 2 | (off >> 8) << 5, off & 0xFF])


def copy2(off, n):
    assert 1 <= n <= 64 and off < 65536
    return bytes([2 | (n - 1) << 2]) + off.to_bytes(2, "little")


def copy4(off, n):
    assert 1 <= n <= 64 and off < 1 << 32
    return bytes([3 | (n - 1) << 2]) + off.to_bytes(4, "little")


def repeat(n):
    """an S2 repeat of the last offset, n bytes, by the shortest length code"""
    if 4 <= n <= 8:
        return bytes([1 | (n - 4) << 2, 0])
    if n - 8 < 256:
        return bytes([1 | 5 << 2, 0, n - 8])
    if n - 260 < 65536:
        return bytes([1 | 6 << 2, 0]) + (n - 260).to_bytes(2, "little")
    assert n - 65540 < 1 << 24
    return bytes([1 | 7 << 2, 0]) + (n - 65540).to_bytes(3, "little")


def block(n, *elements):
    return uvarint(n) + b"".join(elements)


def _uvarint_at(b, at):
    x = s = 0
    for i in range(10):
        if at >= len(b):
            raise Rejected("block: EOF in the length")
        c = b[at]
        at += 1
        if c < 0x80:
            if i == 9 and c > 1:
                raise Rejected("block: length overflows")
            return x | c << s, at
        x |= (c & 0x7F) << s
        s += 7
    raise Rejected("block: length overflows")


def decoded_len(body):
    return _uvarint_at(body, 0)[0]


def decode_block(body):
    """the bytes of an S2 block (Snappy's and the repeat code)"""
    body = bytes(body)
    n, at = _uvarint_at(body, 0)
    out = bytearray()
    last = 0
    while at < len(body):
        tag = body[at]
        kind = tag & 3
        if kind == 0:
            x = tag >> 2
            at += 1
            if x >= 60:
                nb = x - 59
                if nb > len(body) - at:
                    raise Rejected("literal length past the body")
                x = int.from_bytes(body[at:at + nb], "little")
                at += nb
            L = x + 1
            if L > len(body) - at or L > n - len(out):
                raise Rejected("literal past the body or past n")
            out += body[at:at + L]
            at += L
            continue
        if kind == 1:
            if len(body) - at < 2:
                raise Rejected("copy1 past the body")
            off = (tag >> 5) << 8 | body[at + 1]
            L = 4 + ((tag >> 2) & 7)
            at += 2
            if off == 0:
                code = (tag >> 2) & 7
                if code >= 5:
                    nb = code - 4
                    if nb > len(body) - at:
                        raise Rejected("repeat length past the body")
                    L = int.from_bytes(body[at:at + nb], "little") + (8, 260, 65540)[code - 5]
                    at += nb
                off = last
        elif kind == 2:
            if len(body) - at < 3:
                raise Rejected("copy2 past the body")
            off = int.from_bytes(body[at + 1:at + 3], "little")
            L = (tag >> 2) + 1
            at += 3
        else:
            if len(body) - at < 5:
                raise Rejected("copy4 past the body")
            off = int.from_bytes(body[at + 1:at + 5], "little")
            L = (tag >> 2) + 1
            at += 5
        if off == 0 or off > len(out) or L > n - len(out):
            raise Rejected("copy offset 0 / beyond the output / past n")
        last = off
        if off >= L:
            out += out[len(out) - off:len(out) - off + L]
        else:
            pat = bytes(out[len(out) - off:])
            out += (pat * (L // off + 1))[:L]
    if len(out) != n:
        raise Rejected("block does not end at n")
    return bytes(out)


def encode_block(data):
    """a Snappy-subset block of data: greedy matches from the last position of each 4-byte value, copies as Snappy's
    emitCopy writes them"""
    data = bytes(data)
    out = bytearray(uvarint(len(data)))
    last = {}
    emit = s = 0
    while s + 4 <= len(data):
        v = data[s:s + 4]
        c = last.get(v)
        last[v] = s
        if c is None or s - c >= 65536:
            s += 1
            continue
        L = 4
        while s + L < len(data) and data[c + L] == data[s + L]:
            L += 1
        if emit < s:
            out += lit(data[emit:s])
        off = s - c
        n = L
        while n > 0:
            l = 64 if n >= 68 else 60 if n > 64 else n
            out += copy1(off, l) if l < 12 and off < 2048 else copy2(off, l)
            n -= l
        s += L
        emit = s
    if emit < len(data):
        out += lit(data[emit:])
    return bytes(out)


# ---- chunks and streams ---------------------------------------------------------------------------------------------
def chunk(typ, body):
    return bytes([typ]) + len(body).to_bytes(3, "little") + bytes(body)


def compressed(data, body=None):
    """a 0x00 chunk of data (its block `body`, by default encode_block's)"""
    return chunk(0, masked_crc(data).to_bytes(4, "little") + (encode_block(data) if body is None else body))


def stored(data):
    return chunk(1, masked_crc(data).to_bytes(4, "little") + bytes(data))


def stream(data, chunk_size=CHUNK, ident=IDENT):
    """an S2 stream of data as a writer with this chunk size writes it: compressed chunks, stored when not shorter"""
    out = bytearray(ident if data else b"")
    for at in range(0, len(data), chunk_size):
        d = data[at:at + chunk_size]
        b = encode_block(d)
        out += compressed(d, b) if len(b) < len(d) else stored(d)
    return bytes(out)


def chunks(b):
    """[(type, body)] of a stream, without checks beyond the framing"""
    out, p = [], 0
    while p < len(b):
        t, L = b[p], int.from_bytes(b[p + 1:p + 4], "little")
        out.append((t, bytes(b[p + 4:p + 4 + L])))
        p += 4 + L
    assert p == len(b), "chunk runs past the stream"
    return out


def read(b, want):
    """what s2.Reader gives for io.ReadFull of `want` bytes from the stream b"""
    b = bytes(b)
    out = bytearray()
    p, first, snappy = 0, True, False
    while len(out) < want:
        if len(b) - p < 4:
            raise Rejected("out of chunks")
        t, L = b[p], int.from_bytes(b[p + 1:p + 4], "little")
        p += 4
        if L > len(b) - p:
            raise Rejected("chunk past the block")
        body = b[p:p + L]
        p += L
        if first and t != 0xFF:
            raise Rejected("no stream identifier")
        first = False
        if t == 0xFF:
            if body not in (b"S2sTwO", b"sNaPpY"):
                raise Rejected("bad stream identifier")
            snappy = body == b"sNaPpY"
        elif t in (0, 1):
            if L < 4:
                raise Rejected("chunk shorter than its CRC")
            n = decoded_len(body[4:]) if t == 0 else L - 4
            if n > (SNAPPY_MAX_DECODED if snappy else MAX_DECODED):
                raise Rejected("chunk decodes to too much")
            data = decode_block(body[4:]) if t == 0 else body[4:]
            if masked_crc(data) != int.from_bytes(body[:4], "little"):
                raise Rejected("CRC mismatch")
            out += data
        elif t < 0x80:
            raise Rejected("reserved unskippable chunk")
    return bytes(out[:want])


# ---- whole serialized streams ---------------------------------------------------------------------------------------
def _blocks(src):
    """version, tape words and [(raw, type or None, data)] of the four blocks of a stream whose header Deserialize
    reads (so.header's checks first)"""
    so.header(src)
    r = so._Reader(bytes(src))
    v = r.byte()
    r.uvarint()
    ts = r.uvarint()
    out = []
    for _ in range(4):
        raw, size = r.uvarint(), r.uvarint()
        if size == 0:
            out.append((raw, None, b""))
            continue
        typ = r.byte()
        out.append((raw, typ, r.b[r.at:r.at + size - 1]))
        r.at += size - 1
    return v, ts, out


def _assemble(v, ts, blocks):
    body = uvarint(ts)
    for raw, typ, data in blocks:
        body += uvarint(raw) + (uvarint(len(data) + 1) + bytes([typ]) + data if typ is not None else b"\0")
    return bytes([v]) + uvarint(len(body)) + body


def inflate(src):
    """the stream with every S2 block replaced by its inflated bytes as an uncompressed block; Rejected for a header
    Deserialize rejects or an S2 block that breaks a rule, Unsupported for a zstd block"""
    v, ts, blocks = _blocks(src)
    if any(t == 2 for _, t, _ in blocks):
        raise Unsupported("zstd block")
    return _assemble(v, ts, [(raw, 0, read(d, raw)) if t == 1 else (raw, t, d) for raw, t, d in blocks])


def compress(src, chunk_size=CHUNK, ident=IDENT):
    """an uncompressed stream's message, tags and values blocks as S2 blocks (CompressFast): each non-empty block an S2
    stream (stream()), an empty one no bytes behind its type byte"""
    v, ts, blocks = _blocks(src)
    out = [blocks[0]] + [(raw, 1, stream(d, chunk_size, ident)) for raw, t, d in blocks[1:]]
    return _assemble(v, ts, out)


def device_result(src):
    """what the device deserializer in CompressFast mode gives: serialize_oracle.device_result of the inflated stream"""
    return so.device_result(inflate(src))
