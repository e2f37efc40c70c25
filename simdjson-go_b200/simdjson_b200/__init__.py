"""simdjson_b200 -- host-side mirror of the reference's parse API over the C ABI.

Names follow the reference (minio/simdjson-go): SupportedCPU (simdjson_amd64.go:37),
Parse (:66), ParseND (:82), ParsedJson{Message, Tape, Strings} (parsed_json.go:64-71),
WithCopyStrings (options.go:13).  All byte work happens in the sm_90a kernels behind
libsimdjson_b200.so; this module only marshals buffers.  No CPU fallback.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import (COMPRESS_BEST, COMPRESS_DEFAULT, COMPRESS_FAST, COMPRESS_NONE, ERR_CAPACITY, ERR_STAGE1, ERR_STAGE2,
                   ERR_UNSUPPORTED, FIND_CONVERT, FIND_CORRUPT, FIND_KIND_BOOL,
                   FIND_KIND_ARRAY_FLOAT64, FIND_KIND_ARRAY_INT64, FIND_KIND_ARRAY_STRING, FIND_KIND_ARRAY_STRING_CVT,
                   FIND_KIND_ARRAY_UINT64, FIND_KIND_ELEMENT, FIND_KIND_FLOAT64, FIND_KIND_INT64, FIND_KIND_JSON,
                   FIND_KIND_STRING, FIND_KIND_STRING_CVT, FIND_KIND_UINT64, FIND_LIST_KINDS, FIND_VAR_KINDS,
                   FIND_NOT_FOUND, FIND_NOT_OBJECT, FIND_OK, FLAG_COPY_STRINGS, FLAG_NDJSON, OK, SjError, Stage1Info)

JSONVALUEMASK = 0xFF_FFFF_FFFF_FFFF  # parsed_json.go:26
JSONTAGOFFSET = 56
STRINGBUFBIT = 0x80_0000_0000_0000   # parsed_json.go:29
M64 = (1 << 64) - 1

# parsed_serialize.go:79-91 CompressMode.  Fast writes S2 blocks; Default zstd tags and S2 message and values; Best zstd
# blocks throughout.
CompressNone, CompressFast, CompressDefault, CompressBest = COMPRESS_NONE, COMPRESS_FAST, COMPRESS_DEFAULT, COMPRESS_BEST


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
        self.compress_mode = CompressNone

    def set_compress_mode(self, mode):
        """Serializer.CompressMode of this context's serialize / deserialize calls: CompressNone (default, uncompressed
        blocks), CompressFast (S2 blocks), CompressDefault (zstd tags, S2 message and values) or CompressBest (zstd
        blocks).  Deserialize reads S2 blocks in every mode but CompressNone, and zstd blocks in CompressDefault /
        CompressBest only (SJ_ERR_UNSUPPORTED in the others)."""
        rc = self.L.sj_ctx_set_compress_mode(self.h, int(mode))
        if rc != OK:
            raise SjError(rc)
        self.compress_mode = int(mode)

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

    def parse_find(self, msg, paths, kinds, ndjson=True, copy_strings=True):
        """parseMessage + ForEach(FindElement(path...) + the accessor of each kind) (ndjson_test.go:294-315) with the tape
        left in HBM: (rc, rows, columns).  `paths` is a list of key paths (each a list of byte strings), `kinds` the
        FIND_KIND_* of each.  columns[p] is a FindColumn of numpy arrays (status, tag, index, value, offsets, data):
        `value` is int64 / uint64 / float64 by kind (int64 for ELEMENT, BOOL, STRING and JSON, where it is the length); a
        STRING or JSON column's row r is data[offsets[r]:offsets[r + 1]] (JSON: the element's MarshalJSON text).  Only the columns are copied back; on a parse error
        rows is 0 and columns is None.  A list kind's column is a ListColumn: row r's elements are
        elems[list_offsets[r]:list_offsets[r + 1]] (float64 / int64 / uint64; for string lists each element's byte
        length, with the bytes in data as for STRING).  Without list kinds the call is sj_parse_find."""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        cpaths, keep = _find_paths(paths, kinds)
        n_str, n_list = _find_counts(kinds)
        rows, nbytes, nelems = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        # rows: one per record (records are separated by newlines) or the one document; strings: at most the input per
        # STRING path, guessed at its size -- else once more at the exact sizes
        caps = (int(np.count_nonzero(m == 10)) + 1 if ndjson else 1, m.size + 64, m.size // 2 + 1 if n_list else 0)

        def call(out, lout, rout):
            if n_list:
                return self.L.sj_parse_find_lists(self.h, _addr(m) if m.size else None, m.size, flags, cpaths, len(paths), out,
                                                  lout, C.byref(rows), C.byref(nbytes), C.byref(nelems))
            return self.L.sj_parse_find(self.h, _addr(m) if m.size else None, m.size, flags, cpaths, len(paths), out,
                                        C.byref(rows), C.byref(nbytes))
        rc, cols = _find_host(call, len(paths), n_str, n_list, caps, lambda: (rows.value, nbytes.value, nelems.value))
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, 0, None
        if rc != OK:
            raise SjError(rc)
        return rc, rows.value, _find_columns(cols, rows.value, kinds, lambda a, dt: a.view(dt))

    def parse_find_rows(self, msg, row_path, paths, kinds, ndjson=True, copy_strings=True):
        """parseMessage, then Array.ForEach over every record's array at `row_path` (a key path; [] takes a record that
        is itself an array), each element one row of parse_find's columns (FindElement(path...) from the element's Iter
        + the accessor of each kind, list kinds included): (rc, records, rows, RowIndex, columns).  RowIndex holds
        rec_status and rec_offsets per record (record k's rows are rec_offsets[k]:rec_offsets[k + 1]) and row_tag and
        row_index per row (the element head's tag and tape index).  Only the columns are copied back; on a parse error
        records and rows are 0 and RowIndex and columns are None."""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        cpaths, keep = _find_paths(paths, kinds)
        rpath, rkeep = _find_paths([row_path], [FIND_KIND_ELEMENT])
        n_str, n_list = _find_counts(kinds)
        records, rows, nbytes, nelems = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)

        def call(out, lout, rout):
            return self.L.sj_parse_find_rows(self.h, _addr(m) if m.size else None, m.size, flags, rpath, cpaths, len(paths),
                                             out, lout, rout, C.byref(records), C.byref(rows), C.byref(nbytes), C.byref(nelems))
        # the sizes first (no outputs), then the call at the exact sizes
        rc, cols = _find_host(call, len(paths), n_str, n_list, (0, 0, 0, 0),
                              lambda: (rows.value, nbytes.value, nelems.value, records.value))
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, 0, 0, None, None
        if rc != OK:
            raise SjError(rc)
        R, n = records.value, rows.value
        index = RowIndex(cols[8][:R], cols[9][:R + 1], cols[10][:n], cols[11][:n])
        return rc, R, n, index, _find_columns(cols, n, kinds, lambda a, dt: a.view(dt))

    def find_rows_device(self, tape, strings, message, row_path, paths, kinds, out=None):
        """Array.ForEach over every record's array at `row_path` on a tape already on this context's device (torch
        tensors as for find_device): (rc, records, rows, RowIndex, columns) as parse_find_rows, of tensor views.  `out`
        (optional) is find_device's tuple with L list paths' two tensors always present (list_offsets [L, R + 1], elems
        [E]), then rec_status u8 [N], rec_offsets i64 [N + 1], row_tag u8 [R], row_index i64 [R]; without it the tensors
        are allocated at the exact sizes.  rc is SJ_ERR_CAPACITY when `out` is too small (the sizes are still exact)."""
        cpaths, keep = _find_paths(paths, kinds)
        rpath, rkeep = _find_paths([row_path], [FIND_KIND_ELEMENT])
        n_str, n_list = _find_counts(kinds)
        sp, sl = _ptr_len(strings)
        mp, ml = _ptr_len(message)
        tp, tl = _ptr_len(tape)
        records, rows, nbytes, nelems = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)

        def call(o, lo, ro):
            return self.L.sj_find_rows_device(self.h, mp, ml, tp, tl, sp, sl, rpath, cpaths, len(paths), o, lo, ro,
                                              C.byref(records), C.byref(rows), C.byref(nbytes), C.byref(nelems))
        if out is None:
            rc = call(None, None, None)
            if rc not in (OK, ERR_CAPACITY):
                return rc, records.value, rows.value, None, None
            out = _find_cols(_torch_empty(tape.device), len(paths), n_str, n_list, rows.value, nbytes.value, nelems.value,
                             records.value)
        if len(out) != 12:
            raise ValueError("find_rows_device: out needs 12 tensors")
        row_cap = out[0].shape[1]
        shapes = [(len(paths), row_cap)] * 4 + [(n_str, row_cap + 1), None, (n_list, row_cap + 1)]
        for t, shape in zip(out, shapes):
            if (shape is not None and tuple(t.shape) != shape) or not t.is_contiguous():
                raise ValueError("find_rows_device: out tensors must be contiguous with shapes %s" % shape)
        rec_cap = out[9].numel() - 1
        if out[8].numel() < rec_cap or out[10].numel() < row_cap or out[11].numel() < row_cap:
            raise ValueError("find_rows_device: record and row columns smaller than their caps")
        o, lo, ro = _find_outs(out, _data_ptr, row_cap, out[5].numel(), out[7].numel(), rec_cap)
        rc = call(C.byref(o), C.byref(lo), C.byref(ro))
        N, R = records.value, rows.value
        if rc != OK:
            return rc, N, R, None, None
        index = RowIndex(out[8][:N], out[9][:N + 1], out[10][:R], out[11][:R])
        return rc, N, R, index, _find_columns(out, R, kinds, _torch_view)

    def parse_find_members(self, msg, row_path, paths, kinds, only_keys=None, ndjson=True, copy_strings=True):
        """parseMessage, then Object.ForEach(fn, onlyKeys) over every record's object at `row_path` (a key path; [] takes
        the record itself, so every key of every NDJSON record), each member fn receives one row of parse_find's
        columns: (rc, records, rows, MemberIndex, columns).  A path of >= 1 segment is FindElement(path...) from the
        member's Iter; a path of 0 segments is the member's value itself.  `only_keys` (a list of byte strings, None or
        [] for every key) is onlyKeys.  MemberIndex is RowIndex (row_tag / row_index of each member's value head) with
        each row's key: key(r), or key_data[key_offsets[r]:key_offsets[r + 1]].  A record whose ForEach returned an
        error is SJ_FIND_CORRUPT and keeps the rows in front of the error.  On a parse error records and rows are 0
        and MemberIndex and columns are None."""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        cpaths, keep = _find_paths(paths, kinds)
        rpath, rkeep = _find_paths([row_path, only_keys or []], [FIND_KIND_ELEMENT] * 2)
        n_str, n_list = _find_counts(kinds)
        records, rows, nbytes, nelems, nkeys = (C.c_size_t(0) for _ in range(5))

        def call(out, lout, rout, kout):
            return self.L.sj_parse_find_members(self.h, _addr(m) if m.size else None, m.size, flags, rpath,
                                                C.pointer(rpath[1]), cpaths, len(paths), out, lout,
                                                rout, kout, C.byref(records), C.byref(rows), C.byref(nbytes),
                                                C.byref(nelems), C.byref(nkeys))
        # the sizes first (no outputs), then the call at the exact sizes
        rc, cols = _find_host(call, len(paths), n_str, n_list, (0, 0, 0, 0, 0),
                              lambda: (rows.value, nbytes.value, nelems.value, records.value, nkeys.value))
        if rc in (ERR_STAGE1, ERR_STAGE2):
            return rc, 0, 0, None, None
        if rc != OK:
            raise SjError(rc)
        R, n = records.value, rows.value
        index = MemberIndex(cols[8][:R], cols[9][:R + 1], cols[10][:n], cols[11][:n], cols[12][:n + 1], cols[13][:nkeys.value])
        return rc, R, n, index, _find_columns(cols, n, kinds, lambda a, dt: a.view(dt))

    def find_members_device(self, tape, strings, message, row_path, paths, kinds, only_keys=None, out=None):
        """Object.ForEach over every record's object at `row_path` on a tape already on this context's device (torch
        tensors as for find_device): (rc, records, rows, MemberIndex, columns) as parse_find_members, of tensor views.
        `out` (optional) is find_rows_device's 12 tensors, then key_offsets i64 [R + 1] and key_bytes u8 [K]; without
        it the tensors are allocated at the exact sizes.  rc is SJ_ERR_CAPACITY when `out` is too small (the sizes are
        still exact)."""
        cpaths, keep = _find_paths(paths, kinds)
        rpath, rkeep = _find_paths([row_path, only_keys or []], [FIND_KIND_ELEMENT] * 2)
        n_str, n_list = _find_counts(kinds)
        sp, sl = _ptr_len(strings)
        mp, ml = _ptr_len(message)
        tp, tl = _ptr_len(tape)
        records, rows, nbytes, nelems, nkeys = (C.c_size_t(0) for _ in range(5))

        def call(o, lo, ro, ko):
            return self.L.sj_find_members_device(self.h, mp, ml, tp, tl, sp, sl, rpath, C.pointer(rpath[1]),
                                                 cpaths, len(paths), o, lo, ro, ko, C.byref(records), C.byref(rows),
                                                 C.byref(nbytes), C.byref(nelems), C.byref(nkeys))
        if out is None:
            rc = call(None, None, None, None)
            if rc not in (OK, ERR_CAPACITY):
                return rc, records.value, rows.value, None, None
            out = _find_cols(_torch_empty(tape.device), len(paths), n_str, n_list, rows.value, nbytes.value, nelems.value,
                             records.value, nkeys.value)
        if len(out) != 14:
            raise ValueError("find_members_device: out needs 14 tensors")
        row_cap = out[0].shape[1]
        shapes = [(len(paths), row_cap)] * 4 + [(n_str, row_cap + 1), None, (n_list, row_cap + 1)]
        for t, shape in zip(out, shapes):
            if (shape is not None and tuple(t.shape) != shape) or not t.is_contiguous():
                raise ValueError("find_members_device: out tensors must be contiguous with shapes %s" % shape)
        rec_cap = out[9].numel() - 1
        if out[8].numel() < rec_cap or out[10].numel() < row_cap or out[11].numel() < row_cap or out[12].numel() != row_cap + 1:
            raise ValueError("find_members_device: record, row and key columns do not match their caps")
        o, lo, ro, ko = _find_outs(out, _data_ptr, row_cap, out[5].numel(), out[7].numel(), rec_cap, out[13].numel())
        rc = call(C.byref(o), C.byref(lo), C.byref(ro), C.byref(ko))
        N, R = records.value, rows.value
        if rc != OK:
            return rc, N, R, None, None
        index = MemberIndex(out[8][:N], out[9][:N + 1], out[10][:R], out[11][:R], out[12][:R + 1], out[13][:nkeys.value])
        return rc, N, R, index, _find_columns(out, R, kinds, _torch_view)

    def find_rows_serial(self):
        """test hook: the records of the last array-rows or member-rows call whose rows one thread walked
        (sj_test_find_rows_serial)"""
        n = C.c_uint64(0)
        if self.L.sj_test_find_rows_serial(self.h, C.byref(n)) != OK:
            raise SjError(ERR_ARGUMENT)
        return n.value

    def find_device(self, tape, strings, message, paths, kinds, out=None):
        """ForEach + FindElement + accessors over a tape already on this context's device (torch tensors as for
        marshal_device).  `out` (optional) is a tuple of tensors (status u8 [P, R], tag u8 [P, R], index i64 [P, R],
        value i64 [P, R], str_offsets i64 [S, R + 1], str_bytes u8 [B]) for P paths, S of them with a byte column
        (STRING, JSON, STRING_CVT, ARRAY_STRING, ARRAY_STRING_CVT), R >= rows, and with L list paths two more
        (list_offsets i64 [L, R + 1], elems i64 [E]); without it they are allocated at the exact sizes.  Returns (rc, rows,
        columns): columns[p] is a FindColumn (a ListColumn for a list kind) of tensor views (value viewed as float64 for
        FLOAT64 and uint64 for UINT64, elems as float64 / int64 / uint64 by list kind), or None unless rc is OK.  rc is
        SJ_ERR_CAPACITY when `out` is too small (rows and the byte total are still exact, in `rows` and nothing written).
        Without list kinds the call is sj_find_device."""
        cpaths, keep = _find_paths(paths, kinds)
        n_str, n_list = _find_counts(kinds)
        sp, sl = _ptr_len(strings)
        mp, ml = _ptr_len(message)
        tp, tl = _ptr_len(tape)
        rows, nbytes, nelems = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)

        def call(o, lo):
            if n_list:
                return self.L.sj_find_lists_device(self.h, mp, ml, tp, tl, sp, sl, cpaths, len(paths), o, lo, C.byref(rows),
                                                   C.byref(nbytes), C.byref(nelems))
            return self.L.sj_find_device(self.h, mp, ml, tp, tl, sp, sl, cpaths, len(paths), o, C.byref(rows), C.byref(nbytes))
        if out is None:
            rc = call(None, None)
            if rc not in (OK, ERR_CAPACITY):
                return rc, rows.value, None
            out = _find_cols(_torch_empty(tape.device), len(paths), n_str, n_list, rows.value, nbytes.value,
                             nelems.value)[:8 if n_list else 6]
        row_cap = out[0].shape[1]
        shapes = [(len(paths), row_cap)] * 4 + [(n_str, row_cap + 1)] + ([(n_list, row_cap + 1)] if n_list else [])
        for t, shape in zip(out[:5] + out[6:7], shapes):
            if tuple(t.shape) != shape or not t.is_contiguous():
                raise ValueError("find_device: out tensors must be contiguous with shapes %s" % shape)
        if len(out) != (8 if n_list else 6):
            raise ValueError("find_device: out needs %d tensors" % (8 if n_list else 6))
        o, lo, _ = _find_outs(out, _data_ptr, row_cap, out[5].numel(), out[7].numel() if n_list else 0)
        rc = call(C.byref(o), C.byref(lo) if n_list else None)
        if rc != OK:
            return rc, rows.value, None
        return rc, rows.value, _find_columns(out, rows.value, kinds, _torch_view)

    def parse_marshal(self, msg, ndjson=False, copy_strings=True):
        """parseMessage + Iter.MarshalJSON (parsed_json.go:394) with the tape left in HBM: (rc, JSON text bytes).  Only
        the text is copied back; on a parse error the text is b""."""
        # compact text is rarely longer than its input
        return self._parse_to_bytes(self.L.sj_parse_marshal, msg, ndjson, copy_strings, lambda size: size + 64)

    def _parse_to_bytes(self, fn, msg, ndjson, copy_strings, guess):
        """fn (sj_parse_marshal / sj_parse_serialize) into a buffer of guess(input bytes), else once more at the exact
        size: (rc, output bytes), b"" on a parse error"""
        m = _as_u8(msg)
        flags = (FLAG_NDJSON if ndjson else 0) | (FLAG_COPY_STRINGS if copy_strings else 0)
        n = C.c_size_t(0)
        cap = guess(m.size)
        for _ in range(2):
            out = np.empty(max(cap, 1), dtype=np.uint8)
            rc = fn(self.h, _addr(m) if m.size else None, m.size, flags, _addr(out), cap, C.byref(n))
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
        sp, sl = _ptr_len(strings)
        mp, ml = _ptr_len(message)
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
        # tags + values are about 1.5x the input at most for typical JSON
        return self._parse_to_bytes(self.L.sj_parse_serialize, msg, ndjson, copy_strings, lambda size: 2 * size + 64)

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
        when a buffer is too small (the sizes are still exact), SJ_ERR_UNSUPPORTED for S2 blocks in CompressNone mode
        and zstd blocks in CompressNone / CompressFast mode, and SJ_ERR_ARGUMENT for a stream the device does not
        accept."""
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

    def s2_encode(self, data, out=None):
        """test hook: one S2 stream (identifier and chunks) of `data` (uint8 tensor on this context's device), written by
        the device encoder into `out` or a new tensor: (rc, length, the view holding it); SJ_ERR_CAPACITY when `out` is
        too small (the length is still exact)"""
        import torch
        ip, il = _ptr_len(data)
        n = C.c_size_t(0)
        if out is None:
            rc = self.L.sj_test_s2_encode(self.h, ip, il, None, 0, C.byref(n))
            if rc not in (OK, ERR_CAPACITY):
                return rc, n.value, None
            out = torch.empty(max(n.value, 1), dtype=torch.uint8, device=data.device)
        rc = self.L.sj_test_s2_encode(self.h, ip, il, out.data_ptr(), out.numel(), C.byref(n))
        return rc, n.value, out[:n.value]

    def s2_decode(self, stream, want, out=None):
        """test hook: the S2 stream `stream` (uint8 tensor) read as a block of `want` uncompressed bytes by the device
        decoder, into `out` or a new tensor: (rc, the view of its `want` bytes or None)"""
        import torch
        ip, il = _ptr_len(stream)
        if out is None:
            out = torch.empty(max(want, 1), dtype=torch.uint8, device=stream.device)
        got = C.c_size_t(0)
        rc = self.L.sj_test_s2_decode(self.h, ip, il, out.data_ptr(), want, C.byref(got))
        return rc, (out[:got.value] if rc == OK else None)

    def zstd_encode(self, data, out=None):
        """test hook: one zstd frame (single segment, content size, no checksum; nothing for empty data) of `data` (uint8
        tensor on this context's device), written by the device encoder into `out` or a new tensor: (rc, length, the
        view holding it); SJ_ERR_CAPACITY when `out` is too small (the length is still exact)"""
        import torch
        ip, il = _ptr_len(data)
        n = C.c_size_t(0)
        if out is None:
            rc = self.L.sj_test_zstd_encode(self.h, ip, il, None, 0, C.byref(n))
            if rc not in (OK, ERR_CAPACITY):
                return rc, n.value, None
            out = torch.empty(max(n.value, 1), dtype=torch.uint8, device=data.device)
        rc = self.L.sj_test_zstd_encode(self.h, ip, il, out.data_ptr(), out.numel(), C.byref(n))
        return rc, n.value, out[:n.value]

    def zstd_decode(self, stream, want, out=None):
        """test hook: the zstd frames `stream` (uint8 tensor) read as a block of `want` uncompressed bytes by the device
        decoder, into `out` or a new tensor: (rc, the view of its `want` bytes or None)"""
        import torch
        ip, il = _ptr_len(stream)
        if out is None:
            out = torch.empty(max(want, 1), dtype=torch.uint8, device=stream.device)
        got = C.c_size_t(0)
        rc = self.L.sj_test_zstd_decode(self.h, ip, il, out.data_ptr(), want, C.byref(got))
        return rc, (out[:got.value] if rc == OK else None)

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


class FindColumn(tuple):
    """one path's column: status, tag, index, value per row; offsets / data for the byte columns (else None)"""
    __slots__ = ()
    _fields = ("status", "tag", "index", "value", "offsets", "data")

    def __new__(cls, *a):
        return tuple.__new__(cls, a)

    status = property(lambda s: s[0])
    tag = property(lambda s: s[1])
    index = property(lambda s: s[2])
    value = property(lambda s: s[3])
    offsets = property(lambda s: s[4])
    data = property(lambda s: s[5])


class ListColumn(FindColumn):
    """a list path's column: FindColumn's fields, then list_offsets (row r's elements are
    elems[list_offsets[r]:list_offsets[r + 1]]) and elems (float64 / int64 / uint64 values, or for string lists each
    element's byte length, its bytes back to back in data[offsets[r]:offsets[r + 1]])"""
    __slots__ = ()
    _fields = FindColumn._fields + ("list_offsets", "elems")

    list_offsets = property(lambda s: s[6])
    elems = property(lambda s: s[7])

    def strings(self, r):
        """row r of a string list as a list of bytes (numpy columns)"""
        lens = np.asarray(self.elems[self.list_offsets[r]:self.list_offsets[r + 1]])
        at = int(self.offsets[r])
        out = []
        for n in lens.tolist():
            out.append(bytes(np.asarray(self.data[at:at + n])))
            at += n
        return out


class RowIndex(tuple):
    """the records and rows of a find over array rows: rec_status and rec_offsets per record (record k's rows are
    rec_offsets[k]:rec_offsets[k + 1]), row_tag and row_index per row (its element head's tag byte and tape index)"""
    __slots__ = ()
    _fields = ("rec_status", "rec_offsets", "row_tag", "row_index")

    def __new__(cls, *a):
        return tuple.__new__(cls, a)

    rec_status = property(lambda s: s[0])
    rec_offsets = property(lambda s: s[1])
    row_tag = property(lambda s: s[2])
    row_index = property(lambda s: s[3])


class MemberIndex(RowIndex):
    """the records and rows of a find over member rows: RowIndex's fields (row_tag and row_index of each member's value
    head), then key_offsets and key_data: row r's key is key_data[key_offsets[r]:key_offsets[r + 1]]"""
    __slots__ = ()
    _fields = RowIndex._fields + ("key_offsets", "key_data")

    key_offsets = property(lambda s: s[4])
    key_data = property(lambda s: s[5])

    def key(self, r):
        """row r's key as bytes"""
        a, b = int(self.key_offsets[r]), int(self.key_offsets[r + 1])
        d = self.key_data[a:b]
        return bytes(d.cpu().numpy() if hasattr(d, "cpu") else d)


def _find_paths(paths, kinds):
    """the sj_find_path array (and the buffers it points into)"""
    if len(paths) != len(kinds):
        raise ValueError("one kind per path")
    arr = (_lib.FindPath * max(len(paths), 1))()
    keep = []
    for i, (path, kind) in enumerate(zip(paths, kinds)):
        segs = [bytes(s) for s in path]
        blob = C.create_string_buffer(b"".join(segs) or b"\0")
        lens = (C.c_uint32 * max(len(segs), 1))(*[len(s) for s in segs])
        keep += [blob, lens]
        arr[i] = _lib.FindPath(C.cast(blob, C.c_void_p), lens, len(segs), int(kind))
    return arr, keep


def _find_counts(kinds):
    """the paths with a byte column and the list paths"""
    return sum(k in FIND_VAR_KINDS for k in kinds), sum(k in FIND_LIST_KINDS for k in kinds)


def _find_cols(empty, n_paths, n_str, n_list, row_cap, str_cap, elem_cap, rec_cap=None, key_cap=None):
    """a find's columns at the given capacities, each empty(shape, numpy dtype): status, tag, index, value [paths, row_cap],
    str_offsets [n_str, row_cap + 1], str_bytes [str_cap], list_offsets [n_list, row_cap + 1], elems [elem_cap]; with
    rec_cap the array rows' rec_status [rec_cap], rec_offsets [rec_cap + 1], row_tag and row_index [row_cap] behind them,
    and with key_cap the member rows' key_offsets [row_cap + 1] and key_bytes [key_cap] behind those"""
    P = n_paths
    cols = (empty((P, row_cap), np.uint8), empty((P, row_cap), np.uint8), empty((P, row_cap), np.int64),
            empty((P, row_cap), np.uint64), empty((n_str, row_cap + 1), np.int64), empty(max(str_cap, 1), np.uint8),
            empty((n_list, row_cap + 1), np.int64), empty(max(elem_cap, 1), np.uint64))
    if rec_cap is not None:
        cols += (empty(max(rec_cap, 1), np.uint8), empty(rec_cap + 1, np.int64), empty(max(row_cap, 1), np.uint8),
                 empty(max(row_cap, 1), np.int64))
    if key_cap is not None:
        cols += (empty(row_cap + 1, np.int64), empty(max(key_cap, 1), np.uint8))
    return cols


def _find_outs(cols, ptr, row_cap, str_cap, elem_cap, rec_cap=None, key_cap=None):
    """the sj_find_out, sj_find_lists_out (None for 6 columns) and sj_find_rows_out (None without rec_cap) over
    _find_cols' columns, ptr(column) their addresses; with key_cap the sj_find_keys_out behind them"""
    out = _lib.FindOut(*(ptr(a) for a in cols[:6]), row_cap, str_cap)
    lout = _lib.FindListsOut(ptr(cols[6]), ptr(cols[7]), elem_cap) if len(cols) > 6 else None
    rout = _lib.FindRowsOut(*(ptr(a) for a in cols[8:12]), rec_cap) if rec_cap is not None else None
    if key_cap is None:
        return out, lout, rout
    return out, lout, rout, _lib.FindKeysOut(ptr(cols[12]), ptr(cols[13]), key_cap)


def _find_host(call, n_paths, n_str, n_list, caps, sizes):
    """call(out, lists, rows_out[, keys_out]) into numpy columns at caps = (row_cap, str_cap, elem_cap[, rec_cap[,
    key_cap]]), and once more at the exact sizes() when that returns ERR_CAPACITY: (rc, columns)"""
    for _ in range(2):
        cols = _find_cols(np.empty, n_paths, n_str, n_list, *caps)
        outs = _find_outs(cols, _addr, *caps)
        rc = call(*(C.byref(o) if o is not None else None for o in outs))
        if rc != ERR_CAPACITY:
            break
        caps = sizes()
    return rc, cols


def _data_ptr(t):
    return t.data_ptr()


def _torch_empty(dev):
    """empty(shape, numpy dtype) for _find_cols: torch tensors on dev (int64 for the uint64 columns)"""
    import torch
    dt = {np.uint8: torch.uint8, np.int64: torch.int64, np.uint64: torch.int64}
    return lambda shape, d: torch.empty(shape, dtype=dt[d], device=dev)


def _torch_view(a, dt):
    import torch
    return a.view({np.float64: torch.float64, np.uint64: torch.uint64, np.int64: torch.int64}[dt])


def _find_columns(out, rows, kinds, view):
    status, tag, index, value, offs, data = out[:6]
    cols, s, l = [], 0, 0
    for p, k in enumerate(kinds):
        dt = np.float64 if k == FIND_KIND_FLOAT64 else np.uint64 if k == FIND_KIND_UINT64 else np.int64
        o = d = None
        if k in FIND_VAR_KINDS:
            o, d, s = offs[s, :rows + 1], data, s + 1
        c = (status[p, :rows], tag[p, :rows], index[p, :rows], view(value[p, :rows], dt), o, d)
        if k in FIND_LIST_KINDS:
            lo = out[6][l, :rows + 1]
            n = int(lo[rows]) if rows else 0
            et = {FIND_KIND_ARRAY_FLOAT64: np.float64, FIND_KIND_ARRAY_UINT64: np.uint64}.get(k, np.int64)
            cols.append(ListColumn(*c, lo, view(out[7][:n], et)))
            l += 1
        else:
            cols.append(FindColumn(*c))
    return cols


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
    """parsed_serialize.go:44 Serializer, on the default context's device.  Blocks are uncompressed (CompressNone) unless
    CompressMode asks for S2 (CompressFast), zstd tags with S2 message and values (CompressDefault) or zstd blocks
    (CompressBest), and strings are deduplicated exactly (first occurrence), so the stream
    does not depend on copy_strings; the reference's Deserialize reads it."""

    def __init__(self, ctx=None):
        self.ctx = ctx
        self.mode = CompressNone

    def CompressMode(self, c):
        """parsed_serialize.go:93 CompressMode: CompressNone, CompressFast, CompressDefault or CompressBest"""
        if c not in (CompressNone, CompressFast, CompressDefault, CompressBest):
            raise ValueError("unknown compression mode")
        self.mode = c

    def _call(self, fn):
        """fn(ctx) with the context in this Serializer's compress mode, restored afterwards"""
        ctx = self.ctx or default_context()
        before = ctx.compress_mode
        ctx.set_compress_mode(self.mode)
        try:
            return fn(ctx)
        finally:
            ctx.set_compress_mode(before)

    def Serialize(self, pj):
        """the v3 stream of pj (a ParsedJson) as bytes"""
        return self._call(lambda ctx: self._serialize(ctx, pj))

    def _serialize(self, ctx, pj):
        import torch
        tape = torch.from_numpy(np.ascontiguousarray(pj.Tape, dtype=np.uint64).view(np.int64)).cuda()
        strs = torch.from_numpy(np.frombuffer(bytes(pj.Strings), dtype=np.uint8).copy()).cuda()
        msg = torch.from_numpy(np.frombuffer(bytes(pj.Message), dtype=np.uint8).copy()).cuda()
        rc, n, out = ctx.serialize_device(tape, strs, msg)
        if rc != OK:
            raise SjError(rc)
        return out.cpu().numpy().tobytes()

    def Deserialize(self, src):
        """a ParsedJson from a v3 stream with uncompressed blocks, S2 blocks outside CompressNone mode and zstd blocks in
        CompressDefault / CompressBest mode (SJ_ERR_UNSUPPORTED for the others)"""
        return self._call(lambda ctx: self._deserialize(ctx, src))

    def _deserialize(self, ctx, src):
        import torch
        d = torch.from_numpy(np.frombuffer(bytes(src), dtype=np.uint8).copy()).cuda()
        rc, sizes, bufs = ctx.deserialize_device(d)
        if rc != OK:
            raise SjError(rc)
        tape, strs, msg = (b.cpu().numpy() for b in bufs)
        return ParsedJson(msg.tobytes(), tape.view(np.uint64).copy(), strs.tobytes())
