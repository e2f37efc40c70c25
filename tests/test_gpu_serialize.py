"""GPU tests of the device Serializer (serialize.cuh): Serializer.Serialize / Deserialize (parsed_serialize.go:200-695)
with uncompressed blocks, against the sequential restatement in tests/serialize_oracle.py."""
import random
import re
import struct

import numpy as np
import pytest

from tests import marshal_oracle as mo
from tests import serialize_oracle as so
from tests.tape_builder import STRINGBUFBIT, TapeBuilder, word
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, load_fixture, tricky_ndjson

pytestmark = pytest.mark.gpu

OK, ERR_CAPACITY, ERR_TOO_LARGE, ERR_ARGUMENT, ERR_UNSUPPORTED = 0, 4, 5, 6, 12


def _const(name):
    import os
    src = open(os.path.join(os.path.dirname(__file__), "..", "simdjson-go_b200", "csrc", "serialize.cuh")).read()
    return int(re.search(r"constexpr uint64_t %s = (\d+);" % name, src).group(1))


SZ_TILE, DZ_TILE = _const("SZ_TILE"), _const("DZ_TILE")


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _u8(b):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(b) + b"\0", dtype=np.uint8).copy()).cuda()[:len(b)]


def _upload(tape, strs, msg):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(np.asarray(tape, dtype=np.uint64)).view(np.int64).copy()).cuda()
    return t, _u8(strs), _u8(msg)


def _serialize_device(ctx, tape, strs=b"", msg=b""):
    rc, n, out = ctx.serialize_device(*_upload(tape, strs, msg))
    return rc, (out.cpu().numpy().tobytes() if rc == OK else None)


def _deserialize_device(ctx, src):
    """(rc, (tape list, strings, message)) with a canary behind every output buffer"""
    import torch
    rc, sizes, _ = ctx.deserialize_device(_u8(src))
    if rc not in (OK, ERR_CAPACITY):
        # still check that nothing is written: buffers of a plausible size, all canary
        bufs = (torch.full((64,), 0x5A5A, dtype=torch.int64, device="cuda"), torch.full((64,), 0xA5, dtype=torch.uint8, device="cuda"),
                torch.full((64,), 0xA5, dtype=torch.uint8, device="cuda"))
        rc2, _, _ = ctx.deserialize_device(_u8(src), bufs[0], bufs[1], bufs[2])
        assert rc2 == rc
        assert bool((bufs[0] == 0x5A5A).all()) and bool((bufs[1] == 0xA5).all()) and bool((bufs[2] == 0xA5).all())
        return rc, None
    tl, sl, ml = sizes
    tape = torch.full((tl + 8,), 0x5A5A, dtype=torch.int64, device="cuda")
    strs = torch.full((sl + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    msg = torch.full((ml + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, sizes2, views = ctx.deserialize_device(_u8(src), tape[:tl], strs[:sl], msg[:ml])
    assert rc == OK and sizes2 == sizes
    assert bool((tape[tl:] == 0x5A5A).all()) and bool((strs[sl:] == 0xA5).all()) and bool((msg[ml:] == 0xA5).all())
    return rc, ([int(x) & so.M64 for x in views[0].cpu().numpy()], views[1].cpu().numpy().tobytes(), views[2].cpu().numpy().tobytes())


def _expect_deserialize(ctx, src):
    try:
        want = so.device_result(src)
    except so.Unsupported:
        want = ERR_UNSUPPORTED
    except so.Rejected:
        want = ERR_ARGUMENT
    rc, got = _deserialize_device(ctx, src)
    if isinstance(want, int):
        assert rc == want, (rc, want, src[:64].hex())
    else:
        assert rc == OK and got == want, src[:64].hex()


def _round_trip(ctx, tape, strs, msg):
    """serialize_device -> deserialize_device -> marshal_device equals the marshal of the original"""
    d = _upload(tape, strs, msg)
    rc, n, stream = ctx.serialize_device(*d)
    assert rc == OK
    rc, sizes, (t2, s2, m2) = ctx.deserialize_device(stream)
    assert rc == OK
    rc, n, text = ctx.marshal_device(t2, s2, m2)
    assert rc == OK
    return stream.cpu().numpy().tobytes(), text.cpu().numpy().tobytes()


@pytest.mark.parametrize("impl", [0, 1])
def test_fixtures_vs_oracle(ctx, oracle_native, impl):
    ctx.set_stage2_impl(impl)
    try:
        for name in TAPE_FILES + SMALL_FILES + ["parking-citations"]:
            msg = load_fixture(name)
            nd = name == "parking-citations"
            streams = set()
            for copy in (True, False):
                rc, tape, strs, (off, ln) = oracle_native.parse(msg, ndjson=nd, copy_strings=copy)
                assert rc == 0
                want = so.serialize(tape, strs, msg[off:off + ln])
                streams.add(want)
                assert ctx.parse_serialize(msg, ndjson=nd, copy_strings=copy) == (OK, want), (name, copy)
                if impl == 0:
                    assert _serialize_device(ctx, tape, strs, msg[off:off + ln]) == (OK, want), (name, copy)
                    stream, text = _round_trip(ctx, tape, strs, msg[off:off + ln])
                    assert text == mo.marshal(tape, strs, msg[off:off + ln]), name
                    _expect_deserialize(ctx, stream)
            assert len(streams) == 1, name  # the stream does not depend on copy_strings
    finally:
        ctx.set_stage2_impl(0)


def test_parking_citations_pinned(ctx):
    rc, s = ctx.parse_serialize(load_fixture("parking-citations"), ndjson=True)
    assert rc == OK and len(s) == 709472


@pytest.mark.parametrize("which,expect", [("corpus", 8000), ("go-corpus", 300)])
def test_fuzz_seeds(ctx, oracle_native, which, expect):
    n = parsed = 0
    for name, data in fuzz_corpus(which):
        n += 1
        rc, tape, strs, (off, ln) = oracle_native.parse(data)
        if rc != 0:
            continue
        parsed += 1
        m = data[off:off + ln]
        want = so.serialize(tape, strs, m)
        assert ctx.parse_serialize(data) == (OK, want), name
        stream, text = _round_trip(ctx, tape, strs, m)
        assert stream == want and text == mo.marshal(tape, strs, m), name
    assert n > expect and parsed > 0


def test_foreign_tapes(ctx):
    """Nop runs, tag-0 words and flagged floats, which no parse writes"""
    b = TapeBuilder(raw=True)
    b.open("r")
    b.open("[")
    b.number("d", 0x3FF8000000000000, flags=5)
    b.words([word("N", 3), word("N", 2), word("N", 1)])
    b.string(b"abc")
    b.words([0, word("N", 1)])
    b.string(b"abc", copy=False)
    b.number("l", -1)
    b.number("u", 1 << 63)
    b.atoms("tfn")
    b.close(2)
    b.words([word("N", 2), word("N", 1)])
    tape, strs, msg = b.build()
    want = so.serialize(tape, strs, msg)
    assert _serialize_device(ctx, tape, strs, msg) == (OK, want)
    _expect_deserialize(ctx, want)
    rc, got = _deserialize_device(ctx, want)
    assert got[0][2] == int(tape[2])  # the flagged float's whole tag word
    for dedup in ("ref", "none"):
        _expect_deserialize(ctx, so.serialize(tape, strs, msg, dedup=dedup, seed=7))
    import torch
    assert ctx.serialize_device(torch.zeros(0, dtype=torch.int64, device="cuda"))[:2] == (OK, so.EMPTY_STREAM_LEN)


def test_deserialize_reference_streams(ctx, oracle):
    """streams the reference could write: its lossy dedup, no dedup, a Strings.B block, trailing bytes, versions 0-3"""
    for name, nd in (("twitter", False), ("parking-citations", True), ("citm_catalog", False)):
        msg = load_fixture(name)
        rc, tape, strs, (off, ln) = oracle.parse(msg, ndjson=nd)
        m = msg[off:off + ln]
        for dedup, seed in (("exact", 0), ("ref", 1), ("ref", 2), ("none", 0)):
            s = so.serialize(tape, strs, m, dedup=dedup, seed=seed)
            _expect_deserialize(ctx, s)
        s = so.serialize(tape, strs, m)
        _expect_deserialize(ctx, s + b"trailing bytes")
        for v in range(5):
            _expect_deserialize(ctx, bytes([v]) + s[1:])
    # a non-empty Strings.B block: tape strings point into it
    body = so.uvarint(4) + so.uvarint(3) + so.uvarint(4) + b"\0abc"
    body += so.uvarint(0) + so.uvarint(1) + b"\0"
    tags = b'r"r'
    body += so.uvarint(3) + so.uvarint(4) + b"\0" + tags
    vals = struct.pack("<QQQQ", 4, STRINGBUFBIT | 0, 3, (-3) & so.M64)
    body += so.uvarint(len(vals)) + so.uvarint(len(vals) + 1) + b"\0" + vals
    s = b"\3" + so.uvarint(len(body)) + body
    assert so.device_result(s)[1] == b"abc"
    _expect_deserialize(ctx, s)


def test_dedup(ctx):
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    rnd = random.Random(5)
    for ln in list(range(0, 131)) + [5000]:
        base = bytes(rnd.randrange(256) for _ in range(ln))
        variants = [base]
        for at in {0, ln // 2, ln - 1} if ln else ():
            v = bytearray(base)
            v[at] ^= 1
            variants.append(bytes(v))
        variants += [base + b"x", base[:-1]]
        for v in variants + variants[::-1]:
            b.string(v, copy=rnd.random() < 0.5)
    b.close(2)
    tape, strs, msg = b.build()
    want = so.serialize(tape, strs, msg)
    assert _serialize_device(ctx, tape, strs, msg) == (OK, want)
    try:
        for bits in (1, 2, 8):
            ctx.set_string_hash_bits(bits)
            assert _serialize_device(ctx, tape, strs, msg) == (OK, want), bits
        ctx.set_string_hash_bits(2)
        for name in ("twitter", "citm_catalog"):
            rc, s = ctx.parse_serialize(load_fixture(name))
            ctx.set_string_hash_bits(0)
            assert ctx.parse_serialize(load_fixture(name)) == (rc, s)
            ctx.set_string_hash_bits(2)
    finally:
        ctx.set_string_hash_bits(0)
    _expect_deserialize(ctx, want)


def test_twitter_and_twitterescaped_equal(ctx):
    a = ctx.parse_serialize(load_fixture("twitter"))
    assert a[0] == OK and ctx.parse_serialize(load_fixture("twitterescaped")) == a


def _edge_tapes(tile):
    """items placed at E-3 .. E+2 for the first tile and group edges E"""
    for e in (tile, 2 * tile, 1024 * tile):
        group = e == 1024 * tile  # (4 M words: fewer cases, the oracle walks each in Python)
        for d in range(-1, 2) if group else range(-3, 3):
            for kind in ("string", "float", "nops") if group else ("string", "number", "float", "open", "close", "nops"):
                b = TapeBuilder(raw=True)
                b.open("r")
                b.open("[")
                b.pad_to(e + d - (1 if kind == "close" else 0))
                if kind == "string":
                    b.string(b"edge")
                elif kind == "number":
                    b.number("l", 7)
                elif kind == "float":
                    b.number("d", 0x400921FB54442D18, flags=1)
                elif kind == "open":
                    b.open("{")
                    b.close()
                elif kind == "close":
                    b.open("[")
                    b.close()
                else:
                    b.words([word("N", 3), word("N", 2), word("N", 1)])
                b.string(b"edge", copy=False)
                b.close(2)
                yield (e, d, kind), b.build()


def test_tile_and_group_edges(ctx):
    seen = set()
    for tile in (SZ_TILE, DZ_TILE):
        for key, (tape, strs, msg) in _edge_tapes(tile):
            if (key, len(tape)) in seen:
                continue
            seen.add((key, len(tape)))
            want = so.serialize(tape, strs, msg)
            assert _serialize_device(ctx, tape, strs, msg) == (OK, want), key
            rc, got = _deserialize_device(ctx, want)
            assert rc == OK and got == so.deserialize(want), key


def _mutations(s, rnd, k):
    for _ in range(k):
        b = bytearray(s)
        op = rnd.randrange(4)
        if op == 0:
            b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
        elif op == 1:
            b[rnd.randrange(len(b))] = rnd.choice(b'"lude{}[]rntfN\0x\1\2\3')
        elif op == 2:
            del b[rnd.randrange(len(b)):]
        else:
            at = rnd.randrange(len(b))
            b[at:at] = bytes([rnd.randrange(256)])
        yield bytes(b)


def test_malformed_streams(ctx):
    """every mutated stream: the oracle's verdict (or its tape), with canaries behind the output buffers"""
    b = TapeBuilder(raw=True)
    b.open("r")
    b.open("{")
    b.string(b"k")
    b.open("[")
    b.number("d", 0x3FF0000000000000, flags=2)
    b.words([word("N", 2), word("N", 1)])
    b.atoms("tf")
    b.close()
    b.close()
    b.close()
    tape, strs, msg = b.build()
    s = so.serialize(tape, strs, msg)
    rnd = random.Random(11)
    verdicts = {}
    for m in _mutations(s, rnd, 600):
        try:
            so.device_result(m)
            verdicts["ok"] = verdicts.get("ok", 0) + 1
        except so.Unsupported:
            verdicts["unsupported"] = verdicts.get("unsupported", 0) + 1
        except so.Rejected:
            verdicts["rejected"] = verdicts.get("rejected", 0) + 1
        _expect_deserialize(ctx, m)
    assert verdicts.get("rejected", 0) > 100, verdicts
    # S2 / zstd block types in every block
    for v in (1, 2):
        for blk in range(3):
            typs = [0, 0, 0]
            typs[blk] = v
            body = so.uvarint(0) + b"\0\0" + b"".join(so.uvarint(0) + so.uvarint(1) + bytes([t]) for t in typs)
            st = b"\3" + so.uvarint(len(body)) + body
            with pytest.raises(so.Unsupported):
                so.device_result(st)
            assert _deserialize_device(ctx, st)[0] == ERR_UNSUPPORTED
    # an open that names a close twice / word -1 / the second word of a string
    for name, tg, vals in (("twice", b"r[[]]r", [6, 4, 3, (-5) & so.M64]), ("word -1", b"r[]r", [4, (-1) & so.M64, (-3) & so.M64]),
                           ("value word", b'r["]r', [6, 3, 0, 1, (-5) & so.M64])):
        tws = sum(2 if c in b'"lude' else 1 for c in tg)
        v = struct.pack("<%dQ" % len(vals), *vals)
        body = so.uvarint(tws) + b"\0\0" + so.uvarint(0) + so.uvarint(1) + b"\0"
        body += so.uvarint(len(tg)) + so.uvarint(len(tg) + 1) + b"\0" + tg + so.uvarint(len(v)) + so.uvarint(len(v) + 1) + b"\0" + v
        st = b"\3" + so.uvarint(len(body)) + body
        _expect_deserialize(ctx, st)
        assert _deserialize_device(ctx, st)[0] == ERR_ARGUMENT, name


def test_malformed_tapes(ctx):
    b = TapeBuilder()
    b.open("r")
    b.open("[")
    b.string(b"abc")
    b.number("l", 1)
    b.close(2)
    tape, strs, msg = b.build()
    cases = {"unknown tag": {4: word("x")}, "string past Strings.B": {3: 100},
             "offset + length wraps": {2: word('"', STRINGBUFBIT | 1), 3: (1 << 64) - 1}, "string in an empty message": {2: word('"', 0)}}
    for name, change in cases.items():
        bad = tape.copy()
        for k, v in change.items():
            bad[k] = v
        with pytest.raises(so.MalformedTape):
            so.serialize(bad, strs, msg)
        assert _serialize_device(ctx, bad, strs, msg)[0] == ERR_ARGUMENT, name
    for last in ('"', "l", "u", "d"):
        bad = np.concatenate([tape, np.array([word(last)], dtype=np.uint64)])
        assert _serialize_device(ctx, bad, strs, msg)[0] == ERR_ARGUMENT, last


def test_capacity_and_limits(ctx, oracle):
    import torch
    msg = load_fixture("twitter")
    rc, tape, strs, (off, ln) = oracle.parse(msg)
    want = so.serialize(tape, strs, msg[off:off + ln])
    d = _upload(tape, strs, msg[off:off + ln])
    buf = torch.full((len(want) + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, n, _ = ctx.serialize_device(*d, out=buf[:len(want) - 1])
    assert (rc, n) == (ERR_CAPACITY, len(want)) and bool((buf == 0xA5).all())
    rc, n, out = ctx.serialize_device(*d, out=buf[:len(want)])
    assert (rc, n) == (OK, len(want)) and out.cpu().numpy().tobytes() == want and bool((buf[len(want):] == 0xA5).all())
    src = _u8(want)
    none = torch.empty(0, dtype=torch.uint8, device="cuda")
    rc, sizes, _ = ctx.deserialize_device(src, torch.empty(0, dtype=torch.int64, device="cuda"), none, none)
    assert (rc, sizes) == (ERR_CAPACITY, (len(tape), 0, len(so.header(want)[2])))
    t = torch.full((len(tape) + 4,), 7, dtype=torch.int64, device="cuda")
    mm = torch.full((sizes[2] + 4,), 7, dtype=torch.uint8, device="cuda")
    rc, sizes2, _ = ctx.deserialize_device(src, t[:len(tape) - 1], None, mm[:sizes[2]])
    assert (rc, sizes2) == (ERR_CAPACITY, sizes) and bool((t == 7).all()) and bool((mm == 7).all())
    big = b"\3" + so.uvarint(20) + so.uvarint(1 << 31) + b"\0\0" + b"\0\1\0" * 3 + b"\0" * 8
    assert ctx.deserialize_device(_u8(big))[0] == ERR_TOO_LARGE


def test_serializer_api(oracle):
    import simdjson_b200 as sj
    msg = load_fixture("citm_catalog")
    pj = sj.Parse(msg)
    s = sj.Serializer().Serialize(pj)
    rc, tape, strs, (off, ln) = oracle.parse(msg)
    assert s == so.serialize(tape, strs, msg[off:off + ln])
    pj2 = sj.Serializer().Deserialize(s)
    assert pj2.Iter().MarshalJSON() == pj.Iter().MarshalJSON()


def test_scale_replicated_ndjson(ctx):
    pk = load_fixture("parking-citations").strip()
    rc, one = ctx.parse_serialize(pk, ndjson=True)
    assert rc == OK
    k = (512 << 20) // len(pk)
    big = b"\n".join([pk] * k)
    rc, got = ctx.parse_serialize(big, ndjson=True)
    assert rc == OK
    h1, hk = so.header(one), so.header(got)
    assert hk[0] == k * h1[0] and hk[2] == h1[2]
    assert hk[3] == h1[3] * k
    # values: string offsets and lengths repeat (same dedup), root links repeat (relative)
    assert hk[4] == h1[4] * k
    _check_device_round_trip(ctx, big, True)


def test_scale_single_document(ctx):
    tw = load_fixture("twitter")
    rc, one = ctx.parse_serialize(tw)
    assert rc == OK
    k = 850
    big = b"[" + b",".join([tw] * k) + b"]"
    rc, got = ctx.parse_serialize(big)
    assert rc == OK
    h1, hk = so.header(one), so.header(got)
    assert hk[2] == h1[2]
    t1 = h1[3][1:-1]  # one document's tags without its root words
    assert hk[3] == b"r[" + t1 * k + b"]r"
    _check_device_round_trip(ctx, big, False)


def _check_device_round_trip(ctx, big, nd):
    """parse -> serialize -> deserialize -> marshal equals the marshal of the parse, all in HBM"""
    rc, text = ctx.parse_marshal(big, ndjson=nd)
    assert rc == OK
    rc, s = ctx.parse_serialize(big, ndjson=nd)
    assert rc == OK
    rc, sizes, (t, st, m) = ctx.deserialize_device(_u8(s))
    assert rc == OK
    rc, n, out = ctx.marshal_device(t, st, m)
    assert rc == OK and out.cpu().numpy().tobytes() == text
