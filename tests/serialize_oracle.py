"""Serializer.Serialize / Deserialize (parsed_serialize.go:200-695) with uncompressed blocks, restated as plain sequential
Python.  Test infrastructure: the expected output of the device serializer (serialize.cuh) and the rule for which
streams the device deserializer accepts.

serialize() deduplicates strings exactly, keeping the first occurrence (the project's rule).  dedup="ref" emulates the
reference's 16 K-bucket table under a seeded hash, dedup="none" writes every string: both give streams the reference
itself could write.  deserialize() runs the reference's reconstruction on a zeroed tape and raises Rejected for each of
its error returns and for what would panic in Go (an index out of range, a make() of an impossible size)."""
import hashlib
import struct

TAG = 56
VAL = (1 << 56) - 1
STRINGBUFBIT = 1 << 55
M64 = (1 << 64) - 1
EMPTY_STREAM_LEN = 14


class MalformedTape(ValueError):
    pass


class Rejected(ValueError):
    pass


class Unsupported(Rejected):
    """an S2 or zstd block: the device returns SJ_ERR_UNSUPPORTED"""


def uvarint(x):
    out = bytearray()
    while x >= 0x80:
        out.append((x & 0x7F) | 0x80)
        x >>= 7
    out.append(x)
    return bytes(out)


def _string_bytes(tape, i, strings, message):
    if i + 1 >= len(tape):
        raise MalformedTape("string head as the last word")
    v = int(tape[i]) & VAL
    n = int(tape[i + 1])
    buf, off = (strings, v & (STRINGBUFBIT - 1)) if v & STRINGBUFBIT else (message, v)
    if off > len(buf) or n > len(buf) - off:
        raise MalformedTape("string range outside its buffer at %d" % i)
    return bytes(buf[off:off + n])


def serialize(tape, strings=b"", message=b"", dedup="exact", seed=0):
    """the v3 stream with CompressNone blocks"""
    tape = [int(w) for w in tape]
    n = len(tape)
    tags, vals, msg = bytearray(), bytearray(), bytearray()
    seen = {}          # exact: bytes -> offset
    table = [0] * (1 << 14)  # ref: bucket -> offset + 1
    i = 0
    while i < n:
        w = tape[i]
        t = w >> TAG
        v = w & VAL
        if t == ord('"'):
            sb = _string_bytes(tape, i, strings, message)
            if dedup == "exact":
                if sb not in seen:
                    seen[sb] = len(msg)
                    msg += sb
                off = seen[sb]
            elif dedup == "ref":
                h = int.from_bytes(hashlib.blake2b(sb, digest_size=8, key=struct.pack("<Q", seed)).digest(), "little") & 0x3FFF
                o = table[h] - 1
                if o >= 0 and o + len(sb) <= len(msg) and bytes(msg[o:o + len(sb)]) == sb:
                    off = o
                else:
                    off = len(msg)
                    msg += sb
                    table[h] = off + 1
            else:
                off = len(msg)
                msg += sb
            vals += struct.pack("<QQ", off, len(sb))
            i += 1
        elif t in (ord("l"), ord("u"), ord("d")):
            if i + 1 >= n:
                raise MalformedTape("number head as the last word")
            if t == ord("d") and v:
                t = ord("e")
                vals += struct.pack("<Q", w)
            vals += struct.pack("<Q", tape[i + 1])
            i += 1
        elif t in (ord("{"), ord("["), ord("r")):
            vals += struct.pack("<Q", (v - i) & M64)
        elif t not in (ord("}"), ord("]"), ord("n"), ord("t"), ord("f"), ord("N"), 0):
            raise MalformedTape("unknown tag %d at %d" % (t, i))
        tags.append(t)
        i += 1
    blocks = b""
    for raw in (msg, tags, vals):
        blocks += uvarint(len(raw)) + uvarint(len(raw) + 1) + b"\0" + bytes(raw)
    body = uvarint(n) + b"\0\0" + blocks
    return b"\3" + uvarint(len(body)) + body


# ---- Deserialize ---------------------------------------------------------------------------------------------------
class _Reader:
    def __init__(self, b):
        self.b, self.at = b, 0

    def left(self):
        return len(self.b) - self.at

    def byte(self):
        if self.at >= len(self.b):
            raise Rejected("EOF")
        self.at += 1
        return self.b[self.at - 1]

    def uvarint(self):
        x = s = 0
        for i in range(10):
            if self.at >= len(self.b):
                raise Rejected("EOF in a varint")
            c = self.b[self.at]
            self.at += 1
            if c < 0x80:
                if i == 9 and c > 1:
                    raise Rejected("varint overflows")
                return x | c << s
            x |= (c & 0x7F) << s
            s += 7
        raise Rejected("varint overflows")


MAX_WORDS = 0x7FFFFFFF  # beyond this the device returns SJ_ERR_TOO_LARGE (and Go's make() needs more memory than test hosts have)


def header(src):
    """(tape words, Strings.B, message, tags, values, unsupported): the blocks as Deserialize reads them (:466-579)"""
    r = _Reader(bytes(src))
    if r.byte() > 3:
        raise Rejected("unknown version")
    c = r.uvarint()
    if (c - (1 << 64) if c >> 63 else c) > r.left():  # Go compares int(c)
        raise Rejected("stream too short")
    ts = r.uvarint()
    unsupported = False
    blocks = []
    for _ in range(4):  # Strings.B, message, tags, values: raw size, then decBlock (:697-756)
        raw = r.uvarint()
        size = r.uvarint()
        if size > r.left():
            raise Rejected("block size extends beyond input")
        if size == 0 and raw == 0:
            blocks.append(b"")
            continue
        if size < 1:
            raise Rejected("block size too small")
        typ = r.byte()
        data = r.b[r.at:r.at + size - 1]
        r.at += size - 1
        if typ in (1, 2):
            unsupported = True
            blocks.append(None)
        elif typ != 0 or len(data) != raw:
            raise Rejected("unknown compression type or short uncompressed block")
        else:
            blocks.append(data)
    return ts, blocks[0], blocks[1], blocks[2], blocks[3], unsupported


def deserialize(src):
    """(tape as a list of ints, Strings.B, message), as Deserialize writes them on a zeroed tape; Unsupported for
    S2 / zstd blocks, Rejected for any error return or panic"""
    ts, strings, message, tags, values, unsupported = header(src)
    if unsupported:
        raise Unsupported("S2 or zstd block")
    if ts > MAX_WORDS:
        raise Rejected("tape too large")
    tape = [0] * ts
    off = vo = nskips = 0

    def get(k):
        nonlocal vo
        if len(values) - vo < k:
            raise Rejected("no values left")
        v = struct.unpack_from("<%dQ" % (k // 8), values, vo)
        vo += k
        return v

    def put(i, w):
        if not 0 <= i < ts:
            raise Rejected("panic: index out of range")
        tape[i] = w & M64

    for t in tags:
        if off == ts:
            raise Rejected("tags extended beyond tape")
        tw = t << TAG
        if nskips and t != ord("N"):
            for k in range(nskips):
                put(off, (ord("N") << TAG) | (nskips - k))
                off += 1
            nskips = 0
        if t == ord("N"):
            nskips += 1
        elif t == ord('"'):
            o, ln = get(16)
            put(off, tw | o)
            put(off + 1, ln)
            off += 2
        elif t in (ord("d"), ord("l"), ord("u")):
            (x,) = get(8)
            put(off, tw)
            put(off + 1, x)
            off += 2
        elif t == ord("e"):
            a, b = get(16)
            put(off, a)
            put(off + 1, b)
            off += 2
        elif t in (ord("n"), ord("t"), ord("f"), 0):
            put(off, tw)
            off += 1
        elif t in (ord("{"), ord("[")):
            (x,) = get(8)
            val = (x + off) & M64
            if val > ts:
                raise Rejected("open extends beyond tape")
            put(off, tw | val)
            put(val - 1, ((ord("}") if t == ord("{") else ord("]")) << TAG) | off)
            off += 1
        elif t == ord("r"):
            (x,) = get(8)
            val = (x + off) & M64
            if val > ts:
                raise Rejected("root extends beyond tape")
            put(off, tw | val)
            off += 1
        elif t in (ord("}"), ord("]")):
            if tape[off] >> TAG != t:
                raise Rejected("start tag did not match")
            off += 1
        else:
            raise Rejected("unknown tag")
    for k in range(nskips):
        put(off, (ord("N") << TAG) | (nskips - k))
        off += 1
    if off != ts:
        raise Rejected("tags did not fill tape")
    if vo != len(values):
        raise Rejected("values did not fill tape")
    return tape, bytes(strings), bytes(message)


def opens_name_their_closes(src):
    """predicate (b): every '{' / '[' names a later word that starts its matching close tag, and no close is named twice
    (for a stream deserialize() accepts)"""
    ts, _, _, tags, values, _ = header(src)
    pos, at, vo = {}, 0, 0
    for t in tags:
        pos[at] = t
        at += 2 if t in b'"lude' else 1
    at = vo = 0
    named = set()
    for t in tags:
        if t in b"{[":
            val = (struct.unpack_from("<Q", values, vo)[0] + at) & M64
            c = val - 1
            if not (at < c < ts and pos.get(c) == (ord("}") if t == ord("{") else ord("]")) and c not in named):
                return False
            named.add(c)
        vo += {ord('"'): 16, ord("e"): 16, ord("l"): 8, ord("u"): 8, ord("d"): 8, ord("{"): 8, ord("["): 8, ord("r"): 8}.get(t, 0)
        at += 2 if t in b'"lude' else 1
    return True


def device_result(src):
    """what the device deserializer gives: (tape, Strings.B, message); raises Unsupported / Rejected"""
    out = deserialize(src)
    if not opens_name_their_closes(src):
        raise Rejected("an open does not name a later matching close of its own")
    return out
