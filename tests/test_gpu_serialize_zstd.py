"""GPU tests of the device Serializer in CompressDefault / CompressBest mode (zstd.cuh): zstd blocks written by KZ1 and
read back by KX1 / KZ2 .. KZ8, against the zstd restatement in tests/zstd_oracle.py, pyarrow's `zstd` codec and the
CompressNone stream of the same context."""
import random

import numpy as np
import pytest

from tests import s2_oracle as s2
from tests import serialize_oracle as so
from tests import zstd_oracle as zo
from tests.tape_builder import TapeBuilder
from tests.test_zstd_oracle_cpu import constructed_frames, rejected_frames
from tests.util import SMALL_FILES, TAPE_FILES, fuzz_corpus, load_fixture

pytestmark = pytest.mark.gpu

OK, ERR_CAPACITY, ERR_TOO_LARGE, ERR_ARGUMENT, ERR_UNSUPPORTED = 0, 4, 5, 6, 12
NONE, FAST, DEFAULT, BEST = 0, 1, 2, 3
pa = pytest.importorskip("pyarrow")
ZSTD = pa.Codec("zstd")


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


def _in_mode(ctx, mode, fn):
    before = ctx.compress_mode
    ctx.set_compress_mode(mode)
    try:
        return fn()
    finally:
        ctx.set_compress_mode(before)


def _pa_decode(frame, n):
    return ZSTD.decompress(frame, decompressed_size=n, asbytes=True) if n else b""


# ---- the codec alone ------------------------------------------------------------------------------------------------
def _decoder_inputs():
    import glob
    import os
    here = os.path.join(os.path.dirname(__file__), "golden", "data")
    for path in sorted(glob.glob(os.path.join(here, "*.zst"))):
        if "fuzz-corpus" in path:
            continue  # test_device_decoder_fuzz_corpus: 280 MB decoded, pyarrow's output is its reference
        yield os.path.basename(path), open(path, "rb").read()
    tw = load_fixture("twitter")
    for lvl in (1, 3, 9, 19):
        yield "twitter-l%d" % lvl, pa.Codec("zstd", compression_level=lvl).compress(tw, asbytes=True)
        yield "canada-l%d" % lvl, pa.Codec("zstd", compression_level=lvl).compress(load_fixture("canada"), asbytes=True)
    bo = pa.BufferOutputStream()
    with pa.CompressedOutputStream(bo, "zstd") as s:
        s.write(tw)
    yield "twitter-streaming", bo.getvalue().to_pybytes()
    for name, frame, _ in constructed_frames():
        yield "constructed-" + name, frame


@pytest.mark.parametrize("name,frame", list(_decoder_inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_decoder_equals_pyarrow(ctx, name, frame):
    want = zo.decode(frame)
    if not name.startswith("constructed-"):
        assert _pa_decode(frame, len(want)) == want
    rc, got = ctx.zstd_decode(_u8(frame), len(want))
    assert rc == OK
    assert got.cpu().numpy().tobytes() == want
    # one byte more or less than the frames hold
    assert ctx.zstd_decode(_u8(frame), len(want) + 1)[0] == ERR_ARGUMENT
    if want:
        assert ctx.zstd_decode(_u8(frame), len(want) - 1)[0] == ERR_ARGUMENT


def test_device_decoder_fuzz_corpus(ctx):
    """the one foreign streaming frame with a 4 MiB window and 280 MB of output: matches reach back across many blocks"""
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "data", "fuzz-corpus.tar.zst")
    frame = open(path, "rb").read()
    want = pa.CompressedInputStream(pa.OSFile(path), "zstd").read()
    assert (frame[4] & 0x20) == 0 and len(want) > 200 << 20
    rc, got = ctx.zstd_decode(_u8(frame), len(want))
    assert rc == OK
    assert got.cpu().numpy().tobytes() == want
    assert ctx.zstd_decode(_u8(frame), len(want) - 1)[0] == ERR_ARGUMENT


@pytest.mark.parametrize("name,frame,n", list(rejected_frames()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_decoder_rejects(ctx, name, frame, n):
    import torch
    out = torch.empty(16 if n > 1 << 30 else max(n, 1), dtype=torch.uint8, device="cuda")  # (written only when accepted)
    assert ctx.zstd_decode(_u8(frame), n, out)[0] == ERR_ARGUMENT


def test_device_decoder_rejects_after_large(ctx):
    """a block rejected halfway through its matches, right after a large decode left the context's scratch full of
    earlier positions: the verdict is SJ_ERR_ARGUMENT, and the next frame still decodes"""
    big = load_fixture("canada") * 8
    ok = pa.Codec("zstd", compression_level=3).compress(big, asbytes=True)
    bad = dict((name, (f, n)) for name, f, n in rejected_frames())
    for _ in range(2):
        rc, got = ctx.zstd_decode(_u8(ok), len(big))
        assert rc == OK and got.cpu().numpy().tobytes() == big
        for name in ("late-offset-before-frame", "offset-before-frame", "rep1-minus-1-zero", "literals-over-size"):
            f, n = bad[name]
            assert ctx.zstd_decode(_u8(f), n)[0] == ERR_ARGUMENT, name
        small = load_fixture("twitter")
        rc, got = ctx.zstd_decode(_u8(ZSTD.compress(small, asbytes=True)), len(small))
        assert rc == OK and got.cpu().numpy().tobytes() == small


def test_device_decoder_mutations(ctx):
    """small frames changed or cut at random: the device's verdict and bytes are the oracle's"""
    rnd = random.Random(3)
    srcs = [pa.Codec("zstd", compression_level=l).compress(load_fixture("payload-medium"), asbytes=True) for l in (1, 19)]
    srcs += [f for _, f, _ in constructed_frames()]
    counts = {}
    for i in range(600):
        src = srcs[i % len(srcs)]
        m = bytearray(src)
        if i % 5 == 0:
            m = m[:rnd.randrange(len(m))]
        else:
            for _ in range(rnd.randrange(1, 3)):
                m[rnd.randrange(len(m))] = rnd.randrange(256)
        want_n = len(zo.decode(src))
        try:
            want = zo.read_block(bytes(m), want_n)
        except zo.ZstdError:
            want = None
        rc, got = ctx.zstd_decode(_u8(bytes(m)), want_n)
        assert rc == (OK if want is not None else ERR_ARGUMENT), (i, rc)
        if want is not None:
            assert got.cpu().numpy().tobytes() == want
        counts[rc] = counts.get(rc, 0) + 1
    assert counts.get(ERR_ARGUMENT, 0) > 200 and counts.get(OK, 0) > 10, counts


def _encoder_inputs():
    C = 128 << 10
    rnd = random.Random(9)
    for name in ("twitter", "canada", "citm_catalog", "payload-small"):
        yield name, load_fixture(name)
    yield "empty", b""
    yield "one", b"x"
    for n in (C - 1, C, C + 1, 64 << 10, (64 << 10) + 1):
        yield "edge%d" % n, (load_fixture("twitter") * 2)[:n]
    yield "random", bytes(rnd.randrange(256) for _ in range(300000))
    yield "runs", b"a" * 500000 + b"b" * 70000
    yield "many-blocks", load_fixture("canada") * 3


@pytest.mark.parametrize("name,data", list(_encoder_inputs()), ids=lambda x: x if isinstance(x, str) else "")
def test_device_encoder(ctx, name, data):
    import torch
    rc, n, out = ctx.zstd_encode(_u8(data))
    assert rc == OK
    frame = out.cpu().numpy().tobytes()
    if not data:
        assert frame == b""
        return
    assert _pa_decode(frame, len(data)) == data
    assert zo.decode(frame) == data
    assert ctx.zstd_encode(_u8(data))[2].cpu().numpy().tobytes() == frame  # deterministic
    rc, got = ctx.zstd_decode(out, len(data))
    assert rc == OK and got.cpu().numpy().tobytes() == data
    # the capacity contract
    buf = torch.full((n + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, n2, _ = ctx.zstd_encode(_u8(data), buf[:n - 1])
    assert (rc, n2) == (ERR_CAPACITY, n) and bool((buf == 0xA5).all())
    rc, n3, _ = ctx.zstd_encode(_u8(data), buf[:n])
    assert (rc, n3) == (OK, n) and buf[:n].cpu().numpy().tobytes() == frame and bool((buf[n:] == 0xA5).all())
    if name == "random":  # stored: every block raw
        assert len(frame) <= len(data) + 16 + 3 * ((len(data) >> 16) + 1)
    if name in ("twitter", "runs", "many-blocks"):
        assert len(frame) < len(data) // 2


# ---- Serialize ------------------------------------------------------------------------------------------------------
def _check_blocks(stream, mode):
    """block types as the reference's mode; each zstd block is one frame pyarrow decodes; the stream inflated"""
    _, _, blocks = s2._blocks(stream)
    assert blocks[0][1] in (None, 0)
    for (raw, typ, data), want in zip(blocks[1:], zo.MODE_TYPES[mode]):
        assert typ == want
        if typ == 2:
            assert _pa_decode(data, raw) == zo.read_block(data, raw)
    return zo.inflate(stream)


def _docs():
    for name in SMALL_FILES + TAPE_FILES:
        yield name, load_fixture(name), False
    yield "parking-citations", load_fixture("parking-citations"), True


@pytest.mark.parametrize("mode", [DEFAULT, BEST])
@pytest.mark.parametrize("name,msg,nd", list(_docs()), ids=lambda x: x if isinstance(x, str) else "")
def test_serialize_fixtures(ctx, name, msg, nd, mode):
    rc, packed = _in_mode(ctx, mode, lambda: ctx.parse_serialize(msg, ndjson=nd))
    assert rc == OK
    none = _in_mode(ctx, NONE, lambda: ctx.parse_serialize(msg, ndjson=nd))[1]
    assert _check_blocks(packed, mode) == none
    assert _in_mode(ctx, mode, lambda: ctx.parse_serialize(msg, ndjson=nd)) == (OK, packed)
    want = so.device_result(none)
    rc, sizes, views = _in_mode(ctx, mode, lambda: ctx.deserialize_device(_u8(packed)))
    assert rc == OK
    got = ([int(x) & so.M64 for x in views[0].cpu().numpy()], views[1].cpu().numpy().tobytes(), views[2].cpu().numpy().tobytes())
    assert got == want
    # NONE and FAST do not read zstd blocks
    for m in (NONE, FAST):
        assert _in_mode(ctx, m, lambda: ctx.deserialize_device(_u8(packed)))[0] == ERR_UNSUPPORTED


@pytest.mark.parametrize("which", ["corpus", "go-corpus"])
def test_serialize_fuzz_seeds(ctx, which):
    n = 0
    for name, data in fuzz_corpus(which):
        for mode in (DEFAULT, BEST):
            rc, packed = _in_mode(ctx, mode, lambda: ctx.parse_serialize(data, ndjson=False))
            rc2, none = _in_mode(ctx, NONE, lambda: ctx.parse_serialize(data, ndjson=False))
            assert rc == rc2, name
            if rc == OK:
                assert _check_blocks(packed, mode) == none, name
                rc, sizes, views = _in_mode(ctx, mode, lambda: ctx.deserialize_device(_u8(packed)))
                assert rc == OK, name
                assert views[2].cpu().numpy().tobytes() == so.device_result(none)[2], name
                n += 1
    assert n > 100


def _edge_tapes():
    for k in (1, (64 << 10) - 3, (128 << 10) - 2, (128 << 10) - 1, (128 << 10), 5 * (64 << 10) + 7):
        b = TapeBuilder(raw=True)
        b.open("r")
        b.atoms("n" * k)
        b.close()
        yield "tags%d" % (k + 2), b.build()
    yield "empty", ([], b"", b"")


@pytest.mark.parametrize("mode", [DEFAULT, BEST])
@pytest.mark.parametrize("name,t", list(_edge_tapes()), ids=lambda x: x if isinstance(x, str) else "")
def test_serialize_edges(ctx, name, t, mode):
    import torch
    tape, strs, msg = t
    tt = torch.from_numpy(np.ascontiguousarray(np.asarray(tape, dtype=np.uint64)).view(np.int64).copy()).cuda()

    def ser(out=None):
        return ctx.serialize_device(tt, _u8(strs) if strs else None, _u8(msg) if msg else None, out)
    rc, n, out = _in_mode(ctx, mode, ser)
    assert rc == OK
    packed = out.cpu().numpy().tobytes()
    none = so.serialize(tape, strs, msg)
    assert _check_blocks(packed, mode) == none
    buf = torch.full((n + 8,), 0xA5, dtype=torch.uint8, device="cuda")
    rc, n2, _ = _in_mode(ctx, mode, lambda: ser(buf[:n - 1]))
    assert (rc, n2) == (ERR_CAPACITY, n) and bool((buf == 0xA5).all())
    rc, sizes, views = _in_mode(ctx, mode, lambda: ctx.deserialize_device(out))
    assert rc == OK and [int(x) & so.M64 for x in views[0].cpu().numpy()] == so.device_result(none)[0]


# ---- Deserialize of foreign streams ---------------------------------------------------------------------------------
def _expect(ctx, src, mode):
    try:
        want, verdict = zo.device_result(src, mode), OK
    except so.Unsupported:
        want, verdict = None, ERR_UNSUPPORTED
    except so.Rejected as e:
        want, verdict = None, ERR_TOO_LARGE if "too large" in str(e) else ERR_ARGUMENT
    rc, sizes, views = _in_mode(ctx, mode, lambda: ctx.deserialize_device(_u8(src)))
    assert rc == verdict
    if rc == OK:
        got = ([int(x) & so.M64 for x in views[0].cpu().numpy()], views[1].cpu().numpy().tobytes(), views[2].cpu().numpy().tobytes())
        assert got == want
    return rc


def _streaming(d):
    bo = pa.BufferOutputStream()
    with pa.CompressedOutputStream(bo, "zstd") as s:
        s.write(d)
    return bo.getvalue().to_pybytes()


def test_deserialize_foreign_mixes(ctx):
    """every mix of types 0, 1 and 2 over the message, tags and values blocks, the zstd ones pyarrow frames (one-shot
    and streaming): accepted exactly when the inflated stream is, and read back to the same buffers"""
    import itertools
    for name in ("twitter", "citm_catalog"):
        none = _in_mode(ctx, NONE, lambda: ctx.parse_serialize(load_fixture(name)))[1]
        v, ts, blocks = s2._blocks(none)
        for types in itertools.product((0, 1, 2), repeat=3):
            for zmake in (lambda d: ZSTD.compress(d, asbytes=True) if d else b"", lambda d: _streaming(d) if d else b""):
                enc = {0: lambda d: d, 1: s2.stream, 2: zmake}
                src = s2._assemble(v, ts, [blocks[0]] + [(raw, t, enc[t](d)) for (raw, _, d), t in zip(blocks[1:], types)])
                for mode in (DEFAULT, BEST):
                    assert _expect(ctx, src, mode) == OK
                if 2 in types:
                    assert _in_mode(ctx, FAST, lambda: ctx.deserialize_device(_u8(src)))[0] == ERR_UNSUPPORTED


def test_deserialize_mutations(ctx):
    """bytes of a CompressBest stream changed at random: the device's verdict and result are the oracle's"""
    src = _in_mode(ctx, BEST, lambda: ctx.parse_serialize(load_fixture("payload-medium")))[1]
    rnd = random.Random(12)
    verdicts = {}
    for _ in range(300):
        m = bytearray(src)
        for _ in range(rnd.randrange(1, 4)):
            m[rnd.randrange(len(m))] = rnd.randrange(256)
        rc = _expect(ctx, bytes(m), BEST)
        verdicts[rc] = verdicts.get(rc, 0) + 1
    assert verdicts.get(ERR_ARGUMENT, 0) > 100, verdicts


# ---- large inputs ---------------------------------------------------------------------------------------------------
def _canada(mib):
    import torch
    from simdjson_b200 import _lib
    one = load_fixture("canada")
    k = max(1, (mib << 20) // (len(one) + 1))
    msg = b"[" + b",".join([one] * k) + b"]"
    d = torch.full((len(msg) + (1 << 16),), 0x20, dtype=torch.uint8, device="cuda")
    d[:len(msg)].copy_(torch.frombuffer(bytearray(msg), dtype=torch.uint8))
    return d, len(msg), _lib.FLAG_COPY_STRINGS


@pytest.mark.parametrize("mode", [DEFAULT, BEST])
@pytest.mark.parametrize("which", ["k0", "twitter", "canada"])
def test_large_round_trip(ctx, which, mode):
    """512 MiB inputs: serialize -> deserialize on the device equals the CompressNone round trip"""
    import torch
    from tests.test_gpu_serialize_s2 import _k0, _parse_device, _twitter
    d, n, flags = _k0(ctx, 512) if which == "k0" else _twitter(512) if which == "twitter" else _canada(512)
    tape, strs, msg = _parse_device(ctx, d, n, flags)
    rc, slen, stream = _in_mode(ctx, mode, lambda: ctx.serialize_device(tape, strs, msg))
    assert rc == OK
    rc, none_len, none = _in_mode(ctx, NONE, lambda: ctx.serialize_device(tape, strs, msg))
    assert rc == OK and slen < none_len
    rc, sizes, (t2, s2_, m2) = _in_mode(ctx, mode, lambda: ctx.deserialize_device(stream))
    assert rc == OK and sizes[0] == tape.numel()
    rc, _, (t3, s3, m3) = _in_mode(ctx, NONE, lambda: ctx.deserialize_device(none))
    assert rc == OK and torch.equal(t2, t3) and torch.equal(s2_, s3) and torch.equal(m2, m3)
