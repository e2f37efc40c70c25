"""GPU tests of the device Serializer in CompressFast mode (s2.cuh): S2 message, tags and values blocks written by KC1 /
KC2 and read back by KX1 / KX2, against the S2 restatement in tests/s2_oracle.py, pyarrow's `snappy` codec and the
CompressNone stream of the same context."""
import random

import numpy as np
import pytest

from tests import s2_oracle as s2
from tests import serialize_oracle as so
from tests.tape_builder import TapeBuilder
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, load_fixture

pytestmark = pytest.mark.gpu

OK, ERR_CAPACITY, ERR_TOO_LARGE, ERR_ARGUMENT, ERR_UNSUPPORTED = 0, 4, 5, 6, 12
pa = pytest.importorskip("pyarrow")
SNAPPY = pa.Codec("snappy")


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    c.set_compress_mode(sj.CompressFast)
    yield c
    c.close()


def _u8(b):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(b) + b"\0", dtype=np.uint8).copy()).cuda()[:len(b)]


def _none(ctx, fn):
    """fn() with the context in CompressNone mode"""
    ctx.set_compress_mode(0)
    try:
        return fn()
    finally:
        ctx.set_compress_mode(1)


def _check_s2_blocks(fast):
    """every S2 block of a stream the device wrote: the identifier, then chunks of at most 64 KiB that pyarrow decodes
    (compressed) or that are not shorter compressed (stored), each with its CRC"""
    _, _, blocks = s2._blocks(fast)
    assert blocks[0] == (0, None, b"")
    for raw, typ, data in blocks[1:]:
        assert typ == 1
        if raw == 0:
            assert data == b""
            continue
        cs = s2.chunks(data)
        assert cs[0] == (0xFF, b"S2sTwO") and all(t in (0, 1) for t, _ in cs[1:])
        assert len(cs) - 1 == (raw + s2.CHUNK - 1) // s2.CHUNK
        for t, body in cs[1:]:
            n = s2.decoded_len(body[4:]) if t == 0 else len(body) - 4
            assert n == min(s2.CHUNK, raw) or (t, body) == cs[-1]
            d = SNAPPY.decompress(body[4:], decompressed_size=n, asbytes=True) if t == 0 else body[4:]
            assert s2.masked_crc(d) == int.from_bytes(body[:4], "little")
            raw -= n


# ---- codec hooks ----------------------------------------------------------------------------------------------------
def _codec_inputs():
    rnd = random.Random(3)
    yield "empty", b""
    yield "one", b"x"
    yield "random", bytes(rnd.getrandbits(8) for _ in range(200000))
    yield "runs", b"".join(bytes([rnd.randrange(3)]) * rnd.randrange(1, 2000) for _ in range(300))
    for n in (3, 4, 31, 32, 33, 65535, 65536, 65537, 3 * 65536 + 5):
        yield "size%d" % n, (b"abcdefghij%d" % rnd.randrange(10)) * (n // 11) + b"z" * (n % 11)
    for name in SMALL_FILES + ["twitter", "canada", "citm_catalog"]:
        yield name, load_fixture(name)


@pytest.mark.parametrize("name,data", list(_codec_inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_encoder(ctx, name, data):
    rc, n, out = ctx.s2_encode(_u8(data))
    assert rc == OK
    st = out.cpu().numpy().tobytes()
    assert s2.read(st, len(data)) == data  # framing and CRCs, by the oracle
    at = 0
    for t, body in s2.chunks(st)[1:]:
        k = min(s2.CHUNK, len(data) - at)
        d = SNAPPY.decompress(body[4:], decompressed_size=k, asbytes=True) if t == 0 else body[4:]
        assert t in (0, 1) and d == data[at:at + k]
        at += k
    assert at == len(data)
    assert ctx.s2_encode(_u8(data))[2].cpu().numpy().tobytes() == st  # deterministic
    assert ctx.s2_decode(_u8(st), len(data))[1].cpu().numpy().tobytes() == data
    if n:
        import torch
        small = torch.full((n + 8,), 0xA5, dtype=torch.uint8, device="cuda")
        rc, n2, _ = ctx.s2_encode(_u8(data), small[:n - 1])
        assert (rc, n2) == (ERR_CAPACITY, n) and bool((small == 0xA5).all())


def _rle_block(d):
    """an S2 block of d with repeats: each run of 9 or more equal bytes as a literal byte, a copy at offset 1 and
    repeats of that offset"""
    a = np.frombuffer(d, dtype=np.uint8)
    starts = np.flatnonzero(np.concatenate(([True], a[1:] != a[:-1])))
    ends = np.append(starts[1:], len(a))
    els, lit_from = [], 0
    for i, j in zip(starts.tolist(), ends.tolist()):
        if j - i < 9:
            continue
        if lit_from < i:
            els.append(s2.lit(d[lit_from:i]))
        els += [s2.lit(d[i:i + 1]), s2.copy2(1, 4)]
        rest = j - i - 5
        while rest:
            k = min(rest, 65540 + (1 << 24) - 1)
            if 0 < rest - k < 4:
                k -= 4
            els.append(s2.repeat(k))
            rest -= k
        lit_from = j
    if lit_from < len(d):
        els.append(s2.lit(d[lit_from:]))
    return s2.block(len(d), *els)


def _chunked(d, cs, make):
    out = bytearray(s2.IDENT)
    for at in range(0, len(d), cs):
        out += make(d[at:at + cs])
    return bytes(out)


def _decoder_streams():
    rnd = random.Random(4)
    rand = bytes(rnd.getrandbits(8) for _ in range(300000))
    runs = b"".join(bytes([rnd.randrange(4)]) * rnd.randrange(1, 100000) for _ in range(200))
    tw = load_fixture("twitter")
    yield "pyarrow", _chunked(tw, 65536, lambda d: s2.compressed(d, SNAPPY.compress(d, asbytes=True))), len(tw)
    yield "pyarrow-4MiB", _chunked(runs, 4 << 20, lambda d: s2.compressed(d, SNAPPY.compress(d, asbytes=True))), len(runs)
    yield "repeats", _chunked(runs, 1 << 20, lambda d: s2.compressed(d, _rle_block(d))), len(runs)
    far = rand[:200000] + bytes(rnd.getrandbits(8) for _ in range(3 << 20))
    fb = s2.block(len(far) + 64 + 300, s2.lit(far), s2.copy4(len(far), 64), s2.repeat(300))
    want = far + far[:64] + (far[64:] + far)[:300]
    yield "far-copy", s2.IDENT + s2.compressed(want, fb), len(want)
    yield "stored", _chunked(rand, 1 << 20, s2.stored), len(rand)
    mixed = s2.IDENT + s2.chunk(0xFE, bytes(100)) + s2.stored(tw[:1000]) + s2.chunk(0x99, b"index") + s2.IDENT
    mixed += s2.chunk(0x80, b"") + s2.compressed(tw[1000:70000]) + s2.SNAPPY_IDENT + s2.stored(tw[70000:130000])
    yield "mixed", mixed + b"trailing garbage", 130000
    yield "partial", s2.IDENT + s2.compressed(tw[:50000]) + s2.chunk(0x02, b""), 20000
    yield "1MiB", s2.stream(tw[:600000] * 2, 1 << 20), 1200000
    for k in (131, 132, 133, 263, 264, 265):  # one and two waves of the SMs' warps
        d = (tw * 2)[:k * 1000]
        yield "chunks%d" % k, _chunked(d, 1000, lambda x: s2.compressed(x) if x[0] % 2 else s2.stored(x)), len(d)


@pytest.mark.parametrize("name,st,want", list(_decoder_streams()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_decoder_equals_oracle(ctx, name, st, want):
    exp = s2.read(st, want)
    rc, out = ctx.s2_decode(_u8(st), want)
    assert rc == OK and out.cpu().numpy().tobytes() == exp


def _rejections():
    d = b"abcdefgh" * 40
    good = s2.compressed(d)
    crc = s2.masked_crc(d).to_bytes(4, "little")
    n = len(d)
    big = bytes(s2.MAX_DECODED + 1)
    yield "repeat-no-offset", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.repeat(n))), n
    yield "offset0", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.copy2(0, 8))), n
    yield "offset-past", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]), s2.copy2(9, 8))), n
    yield "literal-past-body", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))[:-1]), n
    yield "length-past-body", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))[:2] + b"\xf0"), n
    yield "literal-past-n", s2.IDENT + s2.chunk(0, crc + s2.block(4, s2.lit(d[:8]))), 4
    yield "copy-past-n", s2.IDENT + s2.chunk(0, crc + s2.block(8, s2.lit(d[:4]), s2.copy2(4, 8))), 8
    yield "short-of-n", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]))), 8
    yield "copy1-past-body", s2.IDENT + s2.chunk(0, crc + s2.block(n, s2.lit(d[:8]), b"\x01")), 8
    yield "varint-overflow", s2.IDENT + s2.chunk(0, crc + b"\xff" * 11), 8
    yield "no-identifier", good, n
    yield "skippable-first", s2.chunk(0x80, b"") + s2.IDENT + good, n
    yield "bad-identifier", s2.chunk(0xFF, b"S2sTwX") + good, n
    yield "identifier-length", s2.chunk(0xFF, b"S2sTwO!") + good, n
    yield "compressed-short", s2.IDENT + s2.chunk(0, crc[:3]), n
    yield "stored-short", s2.IDENT + s2.chunk(1, crc[:3]), n
    yield "over-4MiB", s2.IDENT + s2.chunk(0, crc + s2.uvarint(len(big)) + s2.lit(b"\0") + s2.repeat(4)), len(big)
    yield "stored-over-4MiB", s2.IDENT + s2.chunk(1, s2.masked_crc(big).to_bytes(4, "little") + big), len(big)
    yield "snappy-over-64KiB", s2.SNAPPY_IDENT + s2.stored(bytes(65537)), 65537
    yield "crc", s2.IDENT + s2.chunk(0, (int.from_bytes(crc, "little") ^ 1).to_bytes(4, "little") + good[8:]), n
    yield "stored-crc", s2.IDENT + s2.stored(d)[:4] + crc[::-1] + d, n
    yield "reserved-02", s2.IDENT + s2.chunk(0x02, b"") + good, n
    yield "reserved-7f", s2.IDENT + s2.chunk(0x7F, b"") + good, n
    yield "chunk-past-block", s2.IDENT + good[:-1], n
    yield "out-of-chunks", s2.IDENT + good, n + 1
    yield "header-cut", s2.IDENT + good + b"\x00\x00", n + 1
    yield "partial-chunk-checked", s2.IDENT + s2.chunk(0, crc + good[8:-1] + b"!"), 10


@pytest.mark.parametrize("name,st,want", list(_rejections()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_decoder_rejects(ctx, name, st, want):
    import torch
    with pytest.raises(so.Rejected):
        s2.read(st, want)
    canary = torch.full((want + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, _ = ctx.s2_decode(_u8(st), want, canary[:want])
    assert rc == ERR_ARGUMENT and bool((canary == 0xA5).all())


# ---- Serialize ------------------------------------------------------------------------------------------------------
def _docs():
    for name in SMALL_FILES + TAPE_FILES:
        yield name, load_fixture(name), False
    yield "parking-citations", load_fixture("parking-citations"), True


@pytest.mark.parametrize("name,msg,nd", list(_docs()), ids=lambda x: x if isinstance(x, str) else "")
def test_serialize_fast_fixtures(ctx, name, msg, nd):
    """the stream inflates to the CompressNone stream; it is the same from both stage-2 implementations, both
    copy_strings modes and two calls; the device reads it back as the oracle does"""
    rc, fast = ctx.parse_serialize(msg, ndjson=nd)
    assert rc == OK
    _check_s2_blocks(fast)
    none = _none(ctx, lambda: ctx.parse_serialize(msg, ndjson=nd))[1]
    assert s2.inflate(fast) == none
    for impl in (0, 1):
        ctx.set_stage2_impl(impl)
        for copy in (True, False):
            assert ctx.parse_serialize(msg, ndjson=nd, copy_strings=copy) == (OK, fast)
    ctx.set_stage2_impl(0)
    want = so.device_result(none)
    rc, sizes, views = ctx.deserialize_device(_u8(fast))
    assert rc == OK
    got = ([int(x) & so.M64 for x in views[0].cpu().numpy()], views[1].cpu().numpy().tobytes(), views[2].cpu().numpy().tobytes())
    assert got == want


@pytest.mark.parametrize("which", ["corpus", "go-corpus"])
def test_serialize_fast_fuzz_seeds(ctx, which):
    n = 0
    for name, data in fuzz_corpus(which):
        for nd in (False, True):
            rc, fast = ctx.parse_serialize(data, ndjson=nd)
            rc2, none = _none(ctx, lambda: ctx.parse_serialize(data, ndjson=nd))
            assert rc == rc2, name
            if rc == OK:
                assert s2.inflate(fast) == none, name
                n += 1
    assert n > 100


def _serialize_tape(ctx, tape, strs=b"", msg=b"", out=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(tape, dtype=np.uint64)).view(np.int64).copy()).cuda()
    return ctx.serialize_device(t, _u8(strs) if strs else None, _u8(msg) if msg else None, out)


def _edge_tapes():
    C = s2.CHUNK
    for k in (1, C - 3, C - 2, C - 1, 5 * C + 7):  # tags block of k + 2 bytes: 1 .. one chunk +- 1, many chunks
        b = TapeBuilder(raw=True)
        b.open("r")
        b.atoms("n" * k)
        b.close()
        yield "tags%d" % (k + 2), b.build()
    for k in (0, C // 8 - 3, C // 8 - 2, C // 8 - 1, 3 * C // 8):  # values block of 8 k + 16 bytes
        b = TapeBuilder(raw=True)
        b.open("r")
        for i in range(k):
            b.number("l", i * 0x9E3779B97F4A7C15 & ((1 << 63) - 1))
        b.close()
        yield "values%d" % (8 * k + 16), b.build()
    rnd = random.Random(6)
    for n in (1, C - 1, C, C + 1, 4 * C + 3):  # message block of n bytes: one string
        b = TapeBuilder(raw=True)
        b.open("r")
        b.string(bytes(rnd.randrange(32, 127) for _ in range(n)))
        b.close()
        yield "message%d" % n, b.build()
    yield "empty", ([], b"", b"")


@pytest.mark.parametrize("name,t", list(_edge_tapes()), ids=lambda x: x if isinstance(x, str) else "")
def test_serialize_fast_edges(ctx, name, t):
    import torch
    tape, strs, msg = t
    rc, n, out = _serialize_tape(ctx, tape, strs, msg)
    assert rc == OK
    fast = out.cpu().numpy().tobytes()
    _check_s2_blocks(fast)
    none = so.serialize(tape, strs, msg)
    assert _none(ctx, lambda: _serialize_tape(ctx, tape, strs, msg))[2].cpu().numpy().tobytes() == none
    assert s2.inflate(fast) == none
    assert _serialize_tape(ctx, tape, strs, msg)[2].cpu().numpy().tobytes() == fast
    # the capacity contract: exact length, nothing written
    buf = torch.full((n + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, n2, _ = _serialize_tape(ctx, tape, strs, msg, buf[:n - 1])
    assert (rc, n2) == (ERR_CAPACITY, n) and bool((buf == 0xA5).all())
    rc, sizes, views = ctx.deserialize_device(out)
    assert rc == OK and [int(x) & so.M64 for x in views[0].cpu().numpy()] == so.device_result(none)[0]


# ---- Deserialize ----------------------------------------------------------------------------------------------------
def _expect(ctx, src):
    try:
        want, verdict = s2.device_result(src), OK
    except so.Unsupported:
        want, verdict = None, ERR_UNSUPPORTED
    except so.Rejected as e:
        want, verdict = None, ERR_TOO_LARGE if "too large" in str(e) else ERR_ARGUMENT
    rc, sizes, views = ctx.deserialize_device(_u8(src))
    assert rc == verdict
    if rc == OK:
        got = ([int(x) & so.M64 for x in views[0].cpu().numpy()], views[1].cpu().numpy().tobytes(), views[2].cpu().numpy().tobytes())
        assert got == want
    return rc


def _stored_stream(d, cs):
    return _chunked(d, cs, s2.stored) if d else b""


def test_deserialize_reference_shaped(ctx):
    """CompressFast streams as the reference writes them: 1 MiB chunks, repeats, stored chunks, and each block's
    framing mixed"""
    for name in ("twitter", "canada", "citm_catalog"):
        none = _none(ctx, lambda: ctx.parse_serialize(load_fixture(name)))[1]
        v, ts, blocks = s2._blocks(none)
        for make in (lambda d: s2.stream(d, 1 << 20), lambda d: _chunked(d, 1 << 20, lambda x: s2.compressed(x, _rle_block(x))) if d else b"",
                     lambda d: _stored_stream(d, 100000)):
            src = s2._assemble(v, ts, [blocks[0]] + [(raw, 1, make(d)) for raw, _, d in blocks[1:]])
            assert _expect(ctx, src) == OK
        # only some blocks compressed
        src = s2._assemble(v, ts, [blocks[0], blocks[1], (blocks[2][0], 1, s2.stream(blocks[2][2])), blocks[3]])
        assert _expect(ctx, src) == OK


def test_deserialize_type1_size0_and_zstd(ctx):
    """a block of uncompressed size 0 with type 1 reads nothing (accepted, like the reference); zstd stays unsupported"""
    for v, want in ((1, OK), (2, ERR_UNSUPPORTED)):
        for blk in range(3):
            typs = [0, 0, 0]
            typs[blk] = v
            body = so.uvarint(0) + b"\0\0" + b"".join(so.uvarint(0) + so.uvarint(1) + bytes([t]) for t in typs)
            st = b"\3" + so.uvarint(len(body)) + body
            assert _expect(ctx, st) == want
            body = so.uvarint(0) + b"\0\0" + b"".join(so.uvarint(0) + (so.uvarint(2) + bytes([t]) + b"?" if t else b"\0")
                                                       for t in typs)
            st = b"\3" + so.uvarint(len(body)) + body
            assert _expect(ctx, st) == want


def test_deserialize_fast_mutations(ctx):
    """bytes of an S2 stream changed at random: the device's verdict and result are the oracle's"""
    b = TapeBuilder()
    b.open("r")
    b.open("{")
    for i in range(400):
        b.string(b"key%d" % (i % 9))
        b.number("l", i * 7)
    b.close()
    b.close()
    tape, strs, msg = b.build()
    rc, n, out = _serialize_tape(ctx, tape, strs, msg)
    src = out.cpu().numpy().tobytes()
    rnd = random.Random(12)
    verdicts = {}
    for _ in range(300):
        m = bytearray(src)
        for _ in range(rnd.randrange(1, 4)):
            m[rnd.randrange(len(m))] = rnd.randrange(256)
        rc = _expect(ctx, bytes(m))
        verdicts[rc] = verdicts.get(rc, 0) + 1
    assert verdicts.get(ERR_ARGUMENT, 0) > 100, verdicts


# ---- large inputs and compression ratio -----------------------------------------------------------------------------
def _k0(ctx, mib):
    import torch
    from simdjson_b200 import _lib
    import ctypes as C
    pk = load_fixture("parking-citations").strip()
    n_rec = (mib << 20) // (len(pk) // len(pk.split(b"\n")) + 1)
    d = torch.full(((mib << 20) + (4 << 20),), 0x20, dtype=torch.uint8, device="cuda")
    n = C.c_size_t(0)
    rc = ctx.L.sj_gen_ndjson_device(ctx.h, pk, len(pk), 0, n_rec, d.data_ptr(), d.numel() - (1 << 16), C.byref(n))
    assert rc == OK
    return d, n.value, _lib.FLAG_NDJSON | _lib.FLAG_COPY_STRINGS


def _twitter(mib):
    import torch
    from simdjson_b200 import _lib
    one = load_fixture("twitter")
    k = max(1, (mib << 20) // (len(one) + 1))
    msg = b"[" + b",".join([one] * k) + b"]"
    d = torch.full((len(msg) + (1 << 16),), 0x20, dtype=torch.uint8, device="cuda")
    d[:len(msg)].copy_(torch.frombuffer(bytearray(msg), dtype=torch.uint8))
    return d, len(msg), _lib.FLAG_COPY_STRINGS


def _parse_device(ctx, d, n, flags):
    import torch
    import ctypes as C
    tcap, scap = C.c_size_t(0), C.c_size_t(0)
    ctx.L.sj_bounds(n, C.byref(tcap), C.byref(scap))
    tape = torch.empty(tcap.value, dtype=torch.int64, device="cuda")
    strs = torch.empty(max(scap.value, 1), dtype=torch.uint8, device="cuda")
    tl, sl = C.c_size_t(0), C.c_size_t(0)
    rc = ctx.L.sj_parse_device(ctx.h, d.data_ptr(), n, flags, tape.data_ptr(), tape.numel(), C.byref(tl), strs.data_ptr(),
                               strs.numel(), C.byref(sl))
    assert rc == OK
    return tape[:tl.value], strs[:sl.value], d[:n]


@pytest.mark.parametrize("which", ["k0", "twitter"])
def test_large_round_trip(ctx, which):
    """a 512 MiB K0 batch and a 0.5 GiB twitter document: serialize -> deserialize on the device, and marshal / find of
    the result equal the parse's"""
    import torch
    d, n, flags = _k0(ctx, 512) if which == "k0" else _twitter(512)
    tape, strs, msg = _parse_device(ctx, d, n, flags)
    rc, slen, stream = ctx.serialize_device(tape, strs, msg)
    assert rc == OK
    rc, none_len, none = _none(ctx, lambda: ctx.serialize_device(tape, strs, msg))
    assert rc == OK and slen < none_len
    rc, sizes, (t2, s2_, m2) = ctx.deserialize_device(stream)
    assert rc == OK and sizes[0] == tape.numel()
    rc, _, (t3, s3, m3) = _none(ctx, lambda: ctx.deserialize_device(none))
    assert rc == OK and torch.equal(t2, t3) and torch.equal(s2_, s3) and torch.equal(m2, m3)
    del none, t3, s3, m3
    rc, _, text = ctx.marshal_device(tape, strs, msg)
    rc2, _, text2 = ctx.marshal_device(t2, s2_, m2)
    assert rc == rc2 == OK and torch.equal(text, text2)
    del text, text2
    path = [[b"Ticket"]] if which == "k0" else [[b"search_metadata", b"count"]]
    kinds = [5] if which == "k0" else [1]
    r1 = ctx.find_device(tape, strs, msg, path, kinds)
    r2 = ctx.find_device(t2, s2_, m2, path, kinds)
    assert r1[0] == r2[0] == OK and r1[1] == r2[1] > 0
    for a, b in zip(r1[2][0], r2[2][0]):
        if a is not None:
            assert torch.equal(a, b)


def _snappy_len(data):
    """an S2 stream of data with pyarrow's snappy on the same chunking"""
    if not data:
        return 0
    return len(s2.IDENT) + sum(8 + min(len(SNAPPY.compress(data[at:at + s2.CHUNK], asbytes=True)), len(data[at:at + s2.CHUNK]))
                              for at in range(0, len(data), s2.CHUNK))


@pytest.mark.parametrize("which", ["k0", "twitter", "canada"])
def test_compression_ratio(ctx, which):
    """each S2 block is at most 1.25x the size of pyarrow's snappy on the same chunking"""
    if which == "k0":
        d, n, flags = _k0(ctx, 64)
        msg = d[:n].cpu().numpy().tobytes()
        nd = True
    else:
        msg, nd = load_fixture(which), False
    rc, fast = ctx.parse_serialize(msg, ndjson=nd)
    none = _none(ctx, lambda: ctx.parse_serialize(msg, ndjson=nd))[1]
    _, _, fb = s2._blocks(fast)
    _, _, nb = s2._blocks(none)
    for (raw, _, ours), (_, _, plain) in zip(fb[1:], nb[1:]):
        ref = _snappy_len(plain)
        assert len(ours) <= 1.25 * ref + 16, (which, raw, len(ours), ref)
