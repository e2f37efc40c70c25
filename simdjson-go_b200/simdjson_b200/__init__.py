"""simdjson_b200 -- host-side mirror of the reference's parse API over the C ABI.

Names follow the reference (minio/simdjson-go): SupportedCPU (simdjson_amd64.go:37),
Parse (:66), ParseND (:82), ParsedJson{Message, Tape, Strings} (parsed_json.go:64-71),
WithCopyStrings (options.go:13).  All byte work happens in the sm_90a kernels behind
libsimdjson_b200.so; this module only marshals buffers.  No CPU fallback.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (ERR_CAPACITY, ERR_STAGE1, ERR_STAGE2, ERR_UNSUPPORTED, FLAG_COPY_STRINGS, FLAG_NDJSON, OK, SjError,
                   Stage1Info)

JSONVALUEMASK = 0xFF_FFFF_FFFF_FFFF  # parsed_json.go:26
JSONTAGOFFSET = 56
STRINGBUFBIT = 0x80_0000_0000_0000   # parsed_json.go:29
M64 = (1 << 64) - 1


def SupportedCPU():
    """simdjson_amd64.go:37 -- here: is an sm_90 device usable?"""
    return bool(_lib.load().sj_supported())


def _addr(a):
    return a.ctypes.data


def _as_u8(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b, dtype=np.uint8)
    return np.frombuffer(bytes(b), dtype=np.uint8)


class Context:
    """One CUDA stream + reusable device scratch (sj_ctx)."""

    def __init__(self, device=-1):
        self.L = _lib.load()
        h = C.c_void_p()
        rc = self.L.sj_ctx_create(device, C.byref(h))
        if rc != OK:
            raise SjError(rc)
        self.h = h

    def set_stage2_impl(self, impl):
        """0 = streaming stage-2 kernels whenever copy_strings is on (default), 1 = per-structural kernels always"""
        rc = self.L.sj_ctx_set_stage2_impl(self.h, int(impl))
        if rc != OK:
            raise SjError(rc)

    def close(self):
        if getattr(self, "h", None):
            self.L.sj_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- stage 1 ---------------------------------------------------------------
    def find_structural_indices(self, msg, ndjson=False):
        """findStructuralIndices (stage1_find_marks_amd64.go:41): (ok, uint32 deltas)."""
        m = _as_u8(msg)
        cap = m.size + 64
        out = np.empty(cap, dtype=np.uint32)
        n = C.c_size_t(0)
        rc = self.L.sj_find_structural_indices(self.h, _addr(m) if m.size else None, m.size, int(ndjson), _addr(out), cap,
                                               C.byref(n))
        if rc not in (OK, ERR_STAGE1):
            raise SjError(rc)
        return rc == OK, out[:n.value].copy()

    # ---- whole parse -----------------------------------------------------------
    def parse(self, msg, ndjson=False, copy_strings=True):
        """parseMessage (parse_json_amd64.go:52): (rc, tape, strings bytes, (msg_off, msg_len))."""
        m = _as_u8(msg)
        tcap, scap = C.c_size_t(0), C.c_size_t(0)
        self.L.sj_bounds(m.size, C.byref(tcap), C.byref(scap))
        tape = np.empty(tcap.value, dtype=np.uint64)
        strings = np.empty(scap.value, dtype=np.uint8)
        tl, sl, mo, ml = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        rc = self.L.sj_parse(self.h, _addr(m) if m.size else None, m.size, flags, _addr(tape), tape.size, C.byref(tl),
                             _addr(strings), strings.size, C.byref(sl), C.byref(mo), C.byref(ml))
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, None, None, (mo.value, ml.value)
        if rc != OK:
            raise SjError(rc)
        return rc, tape[:tl.value].copy(), strings[:sl.value].tobytes(), (mo.value, ml.value)

    # ---- device-side tape consumers ------------------------------------------
    def parse_count_where(self, msg, key, value, ndjson=True, copy_strings=True):
        """parseMessage + countWhere(key, value) (parse_json_amd64_test.go:134-157) with the tape left in
        HBM: (rc, roots, matches).  roots = countObjects (ndjson_test.go:461)."""
        m = _as_u8(msg)
        key, value = bytes(key), bytes(value)
        roots, matches = C.c_uint64(0), C.c_uint64(0)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        rc = self.L.sj_parse_count_where(self.h, _addr(m) if m.size else None, m.size, flags, key, len(key), value,
                                         len(value), C.byref(roots), C.byref(matches))
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, 0, 0
        if rc != OK:
            raise SjError(rc)
        return rc, roots.value, matches.value

    def parse_marshal(self, msg, ndjson=False, copy_strings=True):
        """parseMessage + Iter.MarshalJSON (parsed_json.go:394) with the tape left in HBM: (rc, JSON text bytes).  Only
        the text is copied back; on a parse error the text is b""."""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        n = C.c_size_t(0)
        cap = m.size + 64  # compact text is rarely longer than its input; else once more at the exact size
        for _ in range(2):
            out = np.empty(max(cap, 1), dtype=np.uint8)
            rc = self.L.sj_parse_marshal(self.h, _addr(m) if m.size else None, m.size, flags, _addr(out), cap, C.byref(n))
            if rc != ERR_CAPACITY:
                break
            cap = n.value
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, b""
        if rc != OK:
            raise SjError(rc)
        return rc, out[:n.value].tobytes()

    def marshal_device(self, tape, strings=None, message=None, out=None):
        """Iter.MarshalJSON of a tape already on this context's device: `tape` (int64 / uint64 torch tensor), `strings`
        (Strings.B) and `message` (uint8 tensors, or None when empty).  Writes into `out` (uint8 tensor) or a new tensor.
        Returns (rc, length of the text, the uint8 tensor view holding it); rc is SJ_ERR_CAPACITY when `out` is too small
        (the length is still exact) and SJ_ERR_ARGUMENT for a malformed tape."""
        import torch

        def ptr_len(t):
            return (t.data_ptr(), t.numel()) if t is not None and t.numel() else (None, 0)

        sp, sl = ptr_len(strings)
        mp, ml = ptr_len(message)
        n = C.c_size_t(0)
        if out is None:
            rc = self.L.sj_marshal_device(self.h, mp, ml, tape.data_ptr(), tape.numel(), sp, sl, None, 0, C.byref(n))
            if rc not in (OK, ERR_CAPACITY):
                return rc, n.value, None
            out = torch.empty(max(n.value, 1), dtype=torch.uint8, device=tape.device)
        op, cap = out.data_ptr(), out.numel()
        rc = self.L.sj_marshal_device(self.h, mp, ml, tape.data_ptr(), tape.numel(), sp, sl, op, cap, C.byref(n))
        return rc, n.value, out[:n.value]

    # ---- Serializer (parsed_serialize.go), uncompressed blocks ------------------
    def parse_serialize(self, msg, ndjson=False, copy_strings=True):
        """parseMessage + Serializer.Serialize (parsed_serialize.go:200) with the tape left in HBM: (rc, stream bytes).
        Only the stream is copied back; on a parse error it is b""."""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        n = C.c_size_t(0)
        cap = 2 * m.size + 64  # tags + values are about 1.5x the input at most for typical JSON; else once more at the exact size
        for _ in range(2):
            out = np.empty(max(cap, 1), dtype=np.uint8)
            rc = self.L.sj_parse_serialize(self.h, _addr(m) if m.size else None, m.size, flags, _addr(out), cap, C.byref(n))
            if rc != ERR_CAPACITY:
                break
            cap = n.value
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, b""
        if rc != OK:
            raise SjError(rc)
        return rc, out[:n.value].tobytes()

    def serialize_device(self, tape, strings=None, message=None, out=None):
        """Serializer.Serialize of a tape already on this context's device, arguments as marshal_device.  Returns (rc,
        length of the stream, the uint8 tensor view holding it); SJ_ERR_CAPACITY when `out` is too small (the length is
        still exact), SJ_ERR_ARGUMENT for a tape the reference's Serialize panics on."""
        import torch
        sp, sl = _ptr_len(strings)
        mp, ml = _ptr_len(message)
        tp, tl = _ptr_len(tape)
        n = C.c_size_t(0)
        if out is None:
            rc = self.L.sj_serialize_device(self.h, mp, ml, tp, tl, sp, sl, None, 0, C.byref(n))
            if rc not in (OK, ERR_CAPACITY):
                return rc, n.value, None
            out = torch.empty(max(n.value, 1), dtype=torch.uint8, device=tape.device)
        rc = self.L.sj_serialize_device(self.h, mp, ml, tp, tl, sp, sl, out.data_ptr(), out.numel(), C.byref(n))
        return rc, n.value, out[:n.value]

    def deserialize_device(self, stream, tape=None, strings=None, message=None):
        """Serializer.Deserialize (parsed_serialize.go:466) of a stream (uint8 tensor) on this context's device.  Writes
        into `tape` (int64 tensor), `strings` and `message` (uint8 tensors), or new tensors when all three are None.
        Returns (rc, (tape words, strings bytes, message bytes), (tape, strings, message) views).  rc is SJ_ERR_CAPACITY
        when a buffer is too small (the sizes are still exact), SJ_ERR_UNSUPPORTED for S2 / zstd blocks and
        SJ_ERR_ARGUMENT for a stream the device does not accept."""
        import torch
        ip, il = _ptr_len(stream)
        tl, sl, ml = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        dev = stream.device
        if tape is None and strings is None and message is None:
            rc = self.L.sj_deserialize_device(self.h, ip, il, None, 0, C.byref(tl), None, 0, C.byref(sl), None, 0, C.byref(ml))
            if rc not in (OK, ERR_CAPACITY):
                return rc, (tl.value, sl.value, ml.value), None
            tape = torch.empty(max(tl.value, 1), dtype=torch.int64, device=dev)
            strings = torch.empty(max(sl.value, 1), dtype=torch.uint8, device=dev)
            message = torch.empty(max(ml.value, 1), dtype=torch.uint8, device=dev)

        def buf(t):
            return (t.data_ptr(), t.numel()) if t is not None else (None, 0)

        (tp, tc), (sp, sc), (mp, mc) = buf(tape), buf(strings), buf(message)
        rc = self.L.sj_deserialize_device(self.h, ip, il, tp, tc, C.byref(tl), sp, sc, C.byref(sl), mp, mc, C.byref(ml))
        sizes = (tl.value, sl.value, ml.value)
        if rc != OK:
            return rc, sizes, None
        return rc, sizes, (tape[:sizes[0]], strings[:sizes[1]], message[:sizes[2]])

    def set_string_hash_bits(self, bits):
        """test hook: keep only `bits` bits of the serializer's string hash (0 = all), to force collisions"""
        rc = self.L.sj_test_set_string_hash_bits(self.h, int(bits))
        if rc != OK:
            raise SjError(rc)

    # ---- unit-test hooks (same method names as oracle.pyoracle.Oracle) -----------
    def block_masks(self, blocks, carries):
        """blocks: (n,64) uint8; carries: (n,4) uint64 -> (n,12) uint64 (see simdjson_b200.h)."""
        b = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, 64)
        c = np.ascontiguousarray(carries, dtype=np.uint64).reshape(-1, 4)
        out = np.empty((b.shape[0], 12), dtype=np.uint64)
        rc = self.L.sj_test_block_masks(self.h, _addr(b), b.shape[0], _addr(c), _addr(out))
        if rc != OK:
            raise SjError(rc)
        return out

    def _one(self, in64, prev_odd=0, prev_inside=0, prev_pseudo=0, ndjson=0):
        blk = np.frombuffer(bytes(in64)[:64].ljust(64, b" "), dtype=np.uint8)
        return [int(x) for x in self.block_masks(blk, np.array([prev_odd, prev_inside, prev_pseudo, ndjson],
                                                                dtype=np.uint64))[0]]

    def find_odd_backslash_sequences(self, in64, prev):
        o = self._one(in64, prev_odd=prev)
        return o[0], o[8]

    def find_quote_mask_and_bits(self, in64, odd_ends, prev_inside, error_mask=0):
        # the hook derives odd_ends itself; callers replaying the goldens pass the carry
        # that produces the same odd_ends (bit 0 <=> previous block ended in an odd run)
        o = self._one(in64, prev_odd=odd_ends & 1, prev_inside=prev_inside)
        return o[1], o[2], o[9], error_mask | o[3]

    def find_whitespace_and_structurals(self, in64):
        o = self._one(in64)
        return o[4], o[5]

    def finalize_structurals(self, structurals, whitespace, quote_mask, quote_bits, prev_pseudo):
        a = np.array([structurals, whitespace, quote_mask, quote_bits, prev_pseudo], dtype=np.uint64)
        out = np.empty(2, dtype=np.uint64)
        rc = self.L.sj_test_finalize(self.h, _addr(a), 1, _addr(out))
        if rc != OK:
            raise SjError(rc)
        return int(out[0]), int(out[1])

    def find_newline_delimiters(self, in64, quote_mask):
        return self._one(in64, ndjson=1)[7] & ~quote_mask & M64

    def find_structural_bits(self, in64, prev_odd, prev_inside, error_mask, prev_pseudo):
        o = self._one(in64, prev_odd, prev_inside, prev_pseudo)
        return o[6], o[8], o[9], error_mask | o[3], o[10]

    def flatten_bits(self, masks, carried=0, position=M64):
        assert carried == 0 and position == M64
        m = np.array(masks, dtype=np.uint64)
        cap = 64 * len(masks) + 8
        out = np.empty(cap, dtype=np.uint32)
        n = C.c_size_t(0)
        rc = self.L.sj_test_flatten_bits(self.h, _addr(m), m.size, _addr(out), cap, C.byref(n))
        if rc != OK:
            raise SjError(rc)
        return [int(x) for x in out[:n.value]], None, None

    def parse_strings(self, items, max_sizes=None):
        """items: list of byte strings each starting AT its opening quote.
        Returns list of (ok, src_len, dst_len, unescaped bytes)."""
        offs = np.zeros(len(items) + 1, dtype=np.uint64)
        for i, it in enumerate(items):
            offs[i + 1] = offs[i] + len(it)
        buf = np.frombuffer(b"".join(items) + b"\0" * 64, dtype=np.uint8)
        ms = np.array(max_sizes if max_sizes is not None else [len(it) for it in items], dtype=np.uint64)
        n = len(items)
        ok = np.zeros(n, dtype=np.uint8)
        sl = np.zeros(n, dtype=np.uint64)
        dl = np.zeros(n, dtype=np.uint64)
        dst = np.zeros(buf.size + 64, dtype=np.uint8)
        rc = self.L.sj_test_parse_strings(self.h, _addr(buf), _addr(offs), n, _addr(ms), _addr(ok), _addr(sl), _addr(dl),
                                          _addr(dst))
        if rc != OK:
            raise SjError(rc)
        res = []
        for i in range(n):
            o = int(offs[i])
            res.append((bool(ok[i]), int(sl[i]), int(dl[i]), dst[o:o + int(dl[i])].tobytes() if ok[i] else b""))
        return res

    def parse_numbers(self, items):
        """items: list of byte strings (number text + delimiter).  Returns list of (tag word, value)."""
        offs = np.zeros(len(items) + 1, dtype=np.uint64)
        for i, it in enumerate(items):
            offs[i + 1] = offs[i] + len(it)
        buf = np.frombuffer(b"".join(items) + b"\0" * 64, dtype=np.uint8)
        n = len(items)
        tag = np.zeros(n, dtype=np.uint64)
        val = np.zeros(n, dtype=np.uint64)
        rc = self.L.sj_test_parse_numbers(self.h, _addr(buf), _addr(offs), n, _addr(tag), _addr(val))
        if rc != OK:
            raise SjError(rc)
        return [(int(tag[i]), int(val[i])) for i in range(n)]

    def launches(self):
        n = C.c_uint64(0)
        self.L.sj_kernel_launches(self.h, C.byref(n))
        return n.value


def _ptr_len(t):
    return (t.data_ptr(), t.numel()) if t is not None and t.numel() else (None, 0)


_default_ctx = None


def default_context():
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context()
    return _default_ctx


class ParsedJson:
    """parsed_json.go:64-71: Message (trimmed input), Tape []uint64, Strings.B []byte."""

    def __init__(self, message, tape, strings):
        self.Message = message
        self.Tape = tape
        self.Strings = strings

    def Iter(self):
        from .iter import Iter
        return Iter(self)


class ParseError(ValueError):
    pass


def _parse(b, ndjson, copy_strings, ctx):
    ctx = ctx or default_context()
    rc, tape, strings, (off, ln) = ctx.parse(b, ndjson=ndjson, copy_strings=copy_strings)
    if rc == ERR_STAGE1:
        raise ParseError("Failed to find all structural indices for stage 1")  # parse_json_amd64.go:93
    if rc == ERR_STAGE2:
        raise ParseError("Bad parsing while executing stage 2")  # parse_json_amd64.go:81
    return ParsedJson(bytes(b)[off:off + ln], tape, strings)


def Parse(b, reuse=None, copy_strings=True, ctx=None):
    """simdjson_amd64.go:66 Parse(b, reuse, WithCopyStrings(copy_strings))."""
    return _parse(b, False, copy_strings, ctx)


def ParseND(b, reuse=None, copy_strings=True, ctx=None):
    """simdjson_amd64.go:82 ParseND: newline-delimited JSON."""
    return _parse(b, True, copy_strings, ctx)


class Serializer:
    """parsed_serialize.go:44 Serializer, on the default context's device.  Blocks are always uncompressed
    (CompressNone), and strings are deduplicated exactly (first occurrence), so the stream does not depend on
    copy_strings; the reference's Deserialize reads it."""

    def __init__(self, ctx=None):
        self.ctx = ctx

    def Serialize(self, pj):
        """the v3 stream of pj (a ParsedJson) as bytes"""
        import torch
        ctx = self.ctx or default_context()
        tape = torch.from_numpy(np.ascontiguousarray(pj.Tape, dtype=np.uint64).view(np.int64)).cuda()
        strs = torch.from_numpy(np.frombuffer(bytes(pj.Strings), dtype=np.uint8).copy()).cuda()
        msg = torch.from_numpy(np.frombuffer(bytes(pj.Message), dtype=np.uint8).copy()).cuda()
        rc, n, out = ctx.serialize_device(tape, strs, msg)
        if rc != OK:
            raise SjError(rc)
        return out.cpu().numpy().tobytes()

    def Deserialize(self, src):
        """a ParsedJson from a v3 stream with uncompressed blocks (SJ_ERR_UNSUPPORTED for S2 / zstd blocks)"""
        import torch
        ctx = self.ctx or default_context()
        d = torch.from_numpy(np.frombuffer(bytes(src), dtype=np.uint8).copy()).cuda()
        rc, sizes, bufs = ctx.deserialize_device(d)
        if rc != OK:
            raise SjError(rc)
        tape, strs, msg = (b.cpu().numpy() for b in bufs)
        return ParsedJson(msg.tobytes(), tape.view(np.uint64).copy(), strs.tobytes())
