"""GPU tests of what the device find's cell kinds share (find.cuh, find_json.cuh, find_list.cuh, find_rows.cuh,
sj_find*.inl), at the edges where one merged copy serves several callers:
  - fd_number: the exact conversion table under the scalar kinds of array rows, the numeric lists ([v] and
    [ok, v, ok], Uint's float bound 2^63 there and 2^64 for Iter.Uint), behind a nop, on builder tapes and a parsed
    message;
  - fd_cell_text: StringCvt's text of every number of the table, the 24-byte extremes and notation edges from the
    scalar writer (KF5), the parallel list writer (KL6), the one-thread list walk (KL7) and array rows, across the
    byte scan's first tile edge, each double's text read back to its bits with repr's shortest digits;
  - fj_lower_stop: two stopping heads of one row in the same warp call, on every lane and round, beside a neighbour
    row's stop on the lane in front, for numeric lists, string lists and array rows; the second stop ends the walk
    without an error, so a cell that stopped there would read differently;
  - scan_counts: each of its callers with a count array past entry 2^22 (one group of 1 024 tiles).
Expected values come from the ports (find_oracle, find_lists_oracle, find_rows_oracle, find_json_oracle), which
tests/test_find_edge_tapes_cpu.py holds to an exact spec, and for the large workloads from their generators' formulas."""
import math

import numpy as np
import pytest

from tests import find_edge_tapes as fe
from tests import find_json_oracle as fj
from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import find_rows_oracle as fr
from tests.test_gpu_find_lists import _dev, _foreign, _np, check, want_cells
from tests.test_gpu_find_rows import check_rows, foreign, want

pytestmark = pytest.mark.gpu
SPECS = fe.conversion_specs()
NUM_LISTS = [fl.ARRAY_FLOAT64, fl.ARRAY_INT64, fl.ARRAY_UINT64, fl.ARRAY_STRING_CVT]
SCALARS = [fo.FLOAT64, fo.INT64, fo.UINT64, fl.STRING_CVT]


@pytest.fixture(scope="module")
def ctx():
    import simdjson_b200 as sj
    if not sj.SupportedCPU():
        pytest.skip("no sm_90 device (the CUDA path has no CPU fallback)")
    c = sj.Context(0)
    yield c
    c.close()


def _up(t, s, m):
    return _dev(t, np.int64), _dev(s), _dev(m)


# ---- §1 conversions --------------------------------------------------------------------------------------------------
def test_conversions_in_list_cells(ctx):
    """[v] and [ok, v, ok] of every value under AsFloat / AsInteger / AsUint64 / AsStringCvt on the parallel passes;
    the numeric lists also against the exact spec"""
    t, s, m = fe.list_tape(SPECS)
    _foreign(ctx, t, s, m, [[b"k"]] * 4, NUM_LISTS, "lists")
    rc, rows, cols = ctx.find_device(*_up(t, s, m), [[b"k"]] * 3, NUM_LISTS[:3])
    forms = [f for sp in SPECS for f in fe.list_forms(sp)]
    assert rc == 0 and rows == len(forms)
    for c, kind in zip(cols, NUM_LISTS[:3]):
        st, lo, el = _np(c.status), _np(c.list_offsets), _np(c.elems).view(np.uint64)
        for r, form in enumerate(forms):
            want_st, want_el = fe.spec_list(form, kind)
            assert (int(st[r]), el[lo[r]:lo[r + 1]].tolist()) == (want_st, want_el), (kind, form)


def test_conversions_behind_a_nop(ctx):
    """a nop in front of the value: the numeric lists are CONVERT there, a StringCvt list finishes in one thread"""
    t, s, m = fe.list_tape(SPECS, nop=True)
    _foreign(ctx, t, s, m, [[b"k"]] * 5, NUM_LISTS + [fl.ARRAY_STRING], "nop")
    rc, rows, cols = ctx.find_device(*_up(t, s, m), [[b"k"]] * 3, NUM_LISTS[:3])
    assert rc == 0 and all((_np(c.status) == fo.CONVERT).all() for c in cols)


def test_conversions_in_array_rows(ctx):
    t, s, m = fe.rows_tape(SPECS)
    foreign(ctx, t, s, m, [b"r"], [[b"k"]] * 4, SCALARS, "rows")
    t, s, m = fe.rows_tape(SPECS, lists=True)
    foreign(ctx, t, s, m, [b"r"], [[b"k"]] * 4, NUM_LISTS, "row lists")


def test_conversions_in_a_parsed_message(ctx, oracle):
    """the table's JSON-expressible values through parse_find and parse_find_rows, against the ports on the oracle's
    tape of the same message"""
    msg = fe.conversion_message(SPECS)
    rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
    assert rc == 0
    m = msg[off:off + ln]
    paths, kinds = [[b"k"]] * 4 + [[b"l"]] * 4 + [[b"m"]] * 4, SCALARS + NUM_LISTS + NUM_LISTS
    rc, rows, cols = ctx.parse_find(msg, paths, kinds)
    assert rc == 0
    check(cols, rows, want_cells(t, s, m, paths, kinds), kinds, "parsed")
    rkinds = SCALARS + NUM_LISTS
    rpaths = [[b"k"]] * len(rkinds)
    check_rows(ctx.parse_find_rows(msg, [b"r"], rpaths, rkinds), want(t, s, m, [b"r"], rpaths, rkinds), rkinds, "parsed rows")


# ---- §2 StringCvt text -----------------------------------------------------------------------------------------------
def _texts_ok(specs, texts):
    """each finite double's text reads back to its bits with repr's shortest digits"""
    n = 0
    for sp, b in zip(specs, texts):
        if sp[0] != "d" or b is None:
            continue
        x = fe.f64(sp[1])
        assert fe.f64_bits(float(b)) == sp[1] and fe.shortest_digits(b.decode()) == fe.shortest_digits(repr(x)), (sp, b)
        n += 1
    assert n > 50


def _col_texts(c, rows):
    off, data, st = _np(c.offsets), _np(c.data).tobytes(), _np(c.status)
    return [data[off[r]:off[r + 1]] if st[r] == fo.OK else None for r in range(rows)]


def test_string_cvt_text_at_every_writer(ctx):
    specs = fe.text_specs()
    (t, s, m), pad = fe.text_scalar_tape(specs)
    _foreign(ctx, t, s, m, [[b"k"]], [fl.STRING_CVT], "scalar text")
    rc, rows, (c,) = ctx.find_device(*_up(t, s, m), [[b"k"]], [fl.STRING_CVT])
    got = _col_texts(c, rows)[pad:]
    assert rc == 0 and all((g is None) == (sp[0] == "d" and not math.isfinite(fe.f64(sp[1]))) for sp, g in zip(specs, got))
    _texts_ok(specs, got)
    for nop in (False, True):
        t, s, m = fe.text_list_tape(specs, nop)
        _foreign(ctx, t, s, m, [[b"k"]], [fl.ARRAY_STRING_CVT], ("list text", nop))
    (t, s, m), pad = fe.text_rows_tape(specs)
    res = foreign(ctx, t, s, m, [b"r"], [[b"k"]], [fl.STRING_CVT], "row text")
    _texts_ok(specs, _col_texts(res[4][0], res[2])[pad:])


# ---- §3 stop words ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", list(fe.STOP_FAMILIES))
def test_two_stops_of_one_row_in_one_warp_call(ctx, family):
    """the first stop wins whichever lane, round and call the second one, and a neighbour row's stop, meet it on"""
    _stops(ctx, family, False)


@pytest.mark.parametrize("family", list(fe.STOP_FAMILIES))
def test_second_stops_alone(ctx, family):
    """the same tapes with the first stops disarmed: every case row stops on its second, which reads differently"""
    _stops(ctx, family, True)


def _stops(ctx, family, disarm):
    kinds = fe.STOP_FAMILIES[family][0]
    t, s, m, placed = fe.stop_tape(family, disarm=disarm)
    assert len(placed) > 1000
    if family == "rows":
        foreign(ctx, t, s, m, [b"a"], [[b"k"]], [fo.ELEMENT], (family, disarm))
        assert ctx.find_rows_serial() == 0
    else:
        _foreign(ctx, t, s, m, [[b"a"]] * len(kinds), list(kinds), (family, disarm))


# ---- §4 count scans past a group -------------------------------------------------------------------------------------
def _edge_rows(n, k=10_000):
    return list(range(min(k, n))) + list(range(max(k, n - k), n))


def test_json_cells_past_a_count_group(ctx, oracle):
    """64 JSON paths x 65 537 records: the word counts' scan (KJ0) and the text scan cross entry 2^22"""
    n = fe.SCAN_RECORDS
    msg = fe.json_scan_message(n)
    P = fe.SCAN_PATHS
    rc, rows, cols = ctx.parse_find(msg, [[b"a"]] * P, [fj.JSON] * P)
    assert rc == 0 and rows == n
    r = np.arange(n)
    k = fe.json_scan_kind(r)
    texts = fe.json_scan_texts(r)
    lens = np.char.str_len(texts).astype(np.int64)
    T = int(lens.sum())
    data = "".join(texts.tolist()).encode()
    assert len(data) == T
    for p, c in enumerate(cols):
        assert np.array_equal(_np(c.status), np.where(k == 5, fo.NOT_FOUND, fo.OK)), p
        assert np.array_equal(_np(c.value), lens), p
        assert np.array_equal(_np(c.offsets), p * T + np.concatenate([[0], np.cumsum(lens)])), p
    assert _np(cols[0].data).tobytes() == data * P
    # the first and last rows cell for cell against the port
    rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
    roots = fo.foreach_roots(t)
    sel = _edge_rows(n)
    w = want_cells(t, s, msg[off:off + ln], [[b"a"]], [fj.JSON], rows=[roots[i] for i in sel])[0]
    for p in (0, P // 2, P - 1):
        c = cols[p]
        st, tag, idx, off_, d = _np(c.status), _np(c.tag), _np(c.index), _np(c.offsets), _np(c.data)
        for j, i in enumerate(sel):
            s_, t_, i_, v_, _, b_ = w[j]
            assert (int(st[i]), int(tag[i]), int(idx[i]), d[off_[i]:off_[i + 1]].tobytes()) == (s_, t_, i_, b_), (p, i)


def test_list_cells_past_a_count_group(ctx, oracle):
    """64 list paths x 65 537 records of 0..4 ints or strings: the element counts' scan crosses entry 2^22, and so do
    the element pool and the byte column"""
    n, P = fe.SCAN_RECORDS, fe.SCAN_PATHS
    msg = fe.list_scan_message(n)
    kinds = fe.list_scan_kinds()
    rc, rows, cols = ctx.parse_find(msg, [[b"a"]] * P, kinds)
    assert rc == 0 and rows == n
    at_e = at_s = 0
    pool, text = [], []
    exp = {k: fe.list_scan_expected(k, n) for k in set(kinds)}
    for p, (c, kind) in enumerate(zip(cols, kinds)):
        st, cnt, el, tx = exp[kind]
        assert np.array_equal(_np(c.status), st), p
        assert np.array_equal(_np(c.value), cnt), p
        assert np.array_equal(_np(c.list_offsets), at_e + np.concatenate([[0], np.cumsum(cnt)])), p
        at_e += int(cnt.sum())
        pool.append(el)
        if tx is not None:
            b = np.char.str_len(tx).astype(np.int64)
            per_row = np.bincount(np.repeat(np.arange(n), cnt), weights=b, minlength=n).astype(np.int64)
            assert np.array_equal(_np(c.offsets), at_s + np.concatenate([[0], np.cumsum(per_row)])), p
            at_s += int(per_row.sum())
            text.append("".join(tx.tolist()))
    assert at_e > fe.GROUP and at_s > fe.GROUP
    got, exp_pool = _np(cols[-1].elems).view(np.uint64), np.concatenate(pool)  # (a column's elems end at its own)
    bad = np.nonzero(got != exp_pool)[0]
    starts = np.cumsum([0] + [len(x) for x in pool])
    assert bad.size == 0, (bad.size, [(int(i), int(np.searchsorted(starts, i, "right") - 1), int(got[i]), int(exp_pool[i]))
                                      for i in bad[:8]], bad[-3:].tolist())
    assert _np(cols[fl.STRING_LISTS[0] - fl.ARRAY_FLOAT64].data).tobytes() == "".join(text).encode()
    # the first and last rows cell for cell against the port, one path of each kind
    rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
    roots = fo.foreach_roots(t)
    sel = _edge_rows(n)
    for p in range(len(fe.LIST_SCAN_KINDS)):
        kind = kinds[P - 1 - p]
        w = want_cells(t, s, msg[off:off + ln], [[b"a"]], [kind], rows=[roots[i] for i in sel])[0]
        c = cols[P - 1 - p]
        st, tag, idx, lo, el = _np(c.status), _np(c.tag), _np(c.index), _np(c.list_offsets), _np(c.elems).view(np.uint64)
        for j, i in enumerate(sel):
            s_, t_, i_, v_, e_, b_ = w[j]
            assert (int(st[i]), int(tag[i]), int(idx[i]), el[lo[i]:lo[i + 1]].tolist()) == (s_, t_, i_, e_), (kind, i)


def test_array_rows_past_a_count_group(ctx, oracle):
    """2^22 + 3 records {"a":[{"k":[...]},...]}: the per-record scans (array words, element counts) and, under a list
    path, the per-row element counts' scan cross entry 2^22"""
    R = fe.ROW_RECORDS
    msg = fe.rows_scan_message()
    rc, N, n, index, (c,) = ctx.parse_find_rows(msg, [b"a"], [[b"k"]], [fl.ARRAY_INT64])
    cnt = fe.row_scan_shape(np.arange(R))
    assert rc == 0 and N == R and n == int(cnt.sum()) > fe.GROUP
    assert (_np(index.rec_status) == fo.OK).all()
    assert np.array_equal(_np(index.rec_offsets), np.concatenate([[0], np.cumsum(cnt)]))
    assert (_np(index.row_tag) == ord("{")).all()
    q = np.arange(n)
    m = fe.row_scan_inner(q)
    assert (_np(c.status) == fo.OK).all() and np.array_equal(_np(c.value), m)
    assert np.array_equal(_np(c.list_offsets), np.concatenate([[0], np.cumsum(m)]))
    qq = np.repeat(q, m)
    jj = np.arange(int(m.sum())) - np.repeat(np.cumsum(m) - m, m)
    assert np.array_equal(_np(c.elems), (qq + jj) % 10)
    # the first and last records (over 10 000 rows each) against the port on the oracle's tape of just them
    ridx = _np(index.row_index)
    cst, ctag, cidx, lo, el = _np(c.status), _np(c.tag), _np(c.index), _np(c.list_offsets), _np(c.elems)
    for first, last in ((0, 8500), (R - 8500, R)):
        sub = fe.rows_scan_message(first, last)
        rc, t, s, (off, ln) = oracle.parse(sub, ndjson=True)
        st, offs, tags, idx, cells = fr.find_rows(t, s, sub[off:off + ln], [b"a"], [[b"k"]], [fl.ARRAY_INT64])
        a = int(cnt[:first].sum())
        assert len(idx) > 10_000
        shift = int(ridx[a]) - idx[0]
        assert (ridx[a:a + len(idx)] - shift).tolist() == idx
        assert np.diff(_np(index.rec_offsets)[first:last + 1]).tolist() == np.diff(offs).tolist()
        for j, (s_, t_, i_, v_, e_, b_) in enumerate(cells[0]):
            i = a + j
            assert (int(cst[i]), int(ctag[i]), int(cidx[i]) - shift, el[lo[i]:lo[i + 1]].tolist()) == (s_, t_, i_, e_), i

