"""CPU checks of tests/find_edge_tapes.py: its exact conversion spec equals the ports (find_oracle, find_lists_oracle,
find_rows_oracle) on every value and kind, StringCvt's text of every double reads back to its bits with repr's
shortest digits, and every generator lands where it claims -- stop words on their lane, round, warp call and tile,
text on the byte scan's tile edge, count arrays past a group -- walked in Python on the generators' tapes or small
instances of them."""
import math

import numpy as np
import pytest

from tests import find_edge_tapes as fe
from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import find_json_oracle as fj
from tests import find_rows_oracle as fr

SPECS = fe.conversion_specs()
NUMS = [s for s in SPECS if s[0] in ("d", "l", "u")]


def test_spec_equals_scalar_and_row_ports():
    """Iter.Int / Uint / Float on every value, on root rows and on array rows"""
    t, s, m = fe.rows_tape(SPECS)
    rec = fr.find_rows(t, s, m, [b"r"], [[b"k"]] * 3, [fo.FLOAT64, fo.INT64, fo.UINT64])
    assert len(rec[2]) == len(SPECS)
    for p, kind in enumerate((fo.FLOAT64, fo.INT64, fo.UINT64)):
        for sp, cell in zip(SPECS, rec[4][p]):
            ok, v = fe.spec_number(sp[0], sp[1], kind) if sp in NUMS else (False, 0)
            assert (cell[0], cell[3]) == ((fo.OK, v) if ok else (fo.CONVERT, 0)), (sp, kind, cell)


def test_spec_equals_list_ports():
    """AsFloat / AsInteger / AsUint64 of [v] and [ok, v, ok]; behind a nop every numeric list is CONVERT and a
    StringCvt list reads as without it"""
    t, s, m = fe.list_tape(SPECS)
    tn, sn, mn = fe.list_tape(SPECS, nop=True)
    rows, rows_n = fo.roots(t), fo.roots(tn)
    forms = [f for sp in SPECS for f in fe.list_forms(sp)]
    assert len(rows) == len(rows_n) == len(forms)
    for kind in fe.NUMERIC.values():
        for r, rn, form in zip(rows, rows_n, forms):
            c, e, _ = fl.list_cell(t, s, m, int(r), [b"k"], kind)
            st, want = fe.spec_list(form, kind)
            assert (c.status, e) == (st, want), (form, kind, c, e)
            cn, _, _ = fl.list_cell(tn, sn, mn, int(rn), [b"k"], kind)
            assert cn.status == fo.CONVERT, (form, kind)
    for r, rn, form in zip(rows, rows_n, forms):
        a = fl.list_cell(t, s, m, int(r), [b"k"], fl.ARRAY_STRING_CVT)
        b = fl.list_cell(tn, sn, mn, int(rn), [b"k"], fl.ARRAY_STRING_CVT)
        assert (a[0].status, a[0].value, a[1], a[2]) == (b[0].status, b[0].value, b[1], b[2]), form


def test_spec_pins_the_quirks():
    """the values the merged accessor is most likely to get wrong, spelled out"""
    two63, two64 = fe.f64_bits(2.0 ** 63), fe.f64_bits(2.0 ** 64)
    nan, neg0 = 0x7FF8000000000000, fe.f64_bits(-0.0)
    assert fe.spec_number("d", two63, fl.ARRAY_UINT64) == (True, 1 << 63)
    assert fe.spec_number("d", fe.f64_bits(math.nextafter(2.0 ** 63, math.inf)), fl.ARRAY_UINT64) == (False, 0)
    assert fe.spec_number("d", fe.f64_bits(math.nextafter(2.0 ** 63, math.inf)), fo.UINT64)[0]
    assert fe.spec_number("d", two64, fo.UINT64) == (True, 1 << 63)
    assert fe.spec_number("d", two64, fl.ARRAY_UINT64) == (False, 0)
    for k in (fo.INT64, fl.ARRAY_INT64, fo.UINT64, fl.ARRAY_UINT64):
        assert fe.spec_number("d", nan, k) == (True, 1 << 63)
    assert fe.spec_number("d", neg0, fl.ARRAY_UINT64) == (True, 0)
    assert fe.spec_number("d", fe.f64_bits(-(2.0 ** 63)), fl.ARRAY_INT64) == (True, 1 << 63)
    assert fe.spec_number("d", two63, fo.INT64) == (True, 1 << 63)
    assert fe.spec_number("l", 2 ** 53 + 1, fo.FLOAT64) == (True, fe.f64_bits(2.0 ** 53))
    assert fe.spec_number("l", 2 ** 53 + 3, fl.ARRAY_FLOAT64) == (True, fe.f64_bits(2.0 ** 53 + 4))


def _text_ok(bits, text):
    x = fe.f64(bits)
    assert fe.f64_bits(float(text)) == bits, (hex(bits), text)
    assert fe.shortest_digits(text.decode()) == fe.shortest_digits(repr(x)), (hex(bits), text)


def test_text_of_every_double():
    """the port's StringCvt text of every double of text_specs(): its bits read back, repr's shortest digits; Inf
    and NaN are CONVERT"""
    specs = fe.text_specs()
    t, s, m = fe.rows_tape(specs)
    rec = fr.find_rows(t, s, m, [b"r"], [[b"k"]], [fl.STRING_CVT])
    n = 0
    for sp, cell in zip(specs, rec[4][0]):
        if sp[0] != "d":
            continue
        x = fe.f64(sp[1])
        if math.isinf(x) or math.isnan(x):
            assert cell[0] == fo.CONVERT, sp
            continue
        assert cell[0] == fo.OK
        _text_ok(sp[1], cell[5])
        n += 1
    assert n > 50
    assert max(len(c[5]) for c in rec[4][0]) == 24


def test_text_tapes_cross_the_byte_scan_tile_edge():
    specs = fe.text_specs()
    (t, s, m), pad = fe.text_scalar_tape(specs)
    assert pad < fe.TILE < pad + len(specs) and len(fo.roots(t)) == pad + len(specs)
    for nop in (False, True):
        t, s, m = fe.text_list_tape(specs, nop)
        heads, V = fe.virtual_cells(t, s, (b"k",))
        first = fe.TILE - sum(fe.ce.Records.width(x) for x in specs) // 2   # the first spec's virtual word
        assert V[0] == 0 and first < fe.TILE < V[1]
        assert (int(t[heads[0] + first]) >> 56) == ord(specs[0][0])
    (t, s, m), pad = fe.text_rows_tape(specs)
    rec = fr.find_rows(t, s, m, [b"r"], [[b"k"]], [fo.ELEMENT])
    assert len(rec[2]) == pad + len(specs) > fe.TILE > pad


def _stop_output(family, t, s, m, kinds, root):
    """what the port reads for one case row: every list kind's cell, or the record's rows"""
    if family == "rows":
        st, offs, tags, idx, _ = fr.find_rows(t, s, m, [b"a"], [[b"k"]], [fo.ELEMENT], records=[root])
        return st, idx
    return [(c.astuple(), e, b) for c, e, b in (fl.list_cell(t, s, m, root, [b"a"], k) for k in kinds)]


@pytest.mark.parametrize("family", list(fe.STOP_FAMILIES))
def test_stop_words_land_in_one_warp_call(family):
    """every case row: its first stop on word A, its second on B and its neighbour's ']' on N, where stop_tape()
    says; every (lane, round) of a warp holds a first stop, pairs on one call's round with A on a lower lane are many,
    and so are neighbours in A's call; the port stops on A, and reads the row differently when it stops on B (the
    disarmed tape)"""
    kinds, _, first, second = fe.STOP_FAMILIES[family]
    t, s, m, placed = fe.stop_tape(family)
    td, sd, md, placed_d = fe.stop_tape(family, disarm=True)
    assert placed_d == placed and len(td) == len(t)
    heads, V = fe.virtual_cells(t, s)
    tags1 = {ord(x[0]) for x in first}
    tags2 = {ord(x[0]) for x in second}
    same_call = neighbours = 0
    seen = set()
    roots = fo.foreach_roots(t)
    for row, A, B, N in placed:
        h = heads[row]
        assert V[row] < A < B < V[row + 1] and V[row] == N + 1 and V[row - 1] < N, (row, A, B, N)
        assert int(t[h + A - V[row]]) >> 56 in tags1 and int(t[h + B - V[row]]) >> 56 in tags2, (row, A, B)
        assert int(td[h + A - V[row]]) >> 56 not in tags1 and int(td[h + B - V[row]]) >> 56 in tags2, (row, A, B)
        assert int(t[h - 7]) >> 56 == ord("]"), row     # the neighbour's ']', then } r, and r { "a" in front of h
        pa, pb, pn = fe.place(A), fe.place(B), fe.place(N)
        seen.add(pa[2:])
        if pa[:2] == pb[:2] and pa[3] == pb[3]:
            assert pa[2] < pb[2]
            same_call += 1
        if pa[:2] == pn[:2] and pa[3] == pn[3] and pn[2] + 1 == pa[2]:
            neighbours += 1
        else:
            assert A % fe.WARP < 4, (row, A, N)                             # only then is N in the window in front
    assert len(seen) == fe.LANES * fe.ROUNDS, family
    assert same_call > 150, (family, same_call)
    assert neighbours > 900, (family, neighbours)
    assert any(fe.place(A)[0] != fe.place(B)[0] for _, A, B, _ in placed), family
    for row, A, B, N in placed[::3]:
        r = int(roots[row])
        armed, disarmed = _stop_output(family, t, s, m, kinds, r), _stop_output(family, td, sd, md, kinds, r)
        assert armed != disarmed, (family, row)
        if family == "rows":  # the rows in front of A
            st, idx = armed
            at = heads[row] + A - V[row]
            assert st == [fo.OK] and idx and idx[-1] < at and idx[-1] + (2 if t[idx[-1]] >> 56 == ord("l") else 1) == at
        else:
            assert all(c[0][0] == fo.CONVERT for c in armed) and all(c[0][0] == fo.OK for c in disarmed), (family, row)


def test_scan_generators(oracle):
    """small instances parsed by the oracle equal the formulas; the full sizes cross 2^22 entries"""
    n = 60
    msg = fe.json_scan_message(n)
    rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
    assert rc == 0
    texts = fe.json_scan_texts(np.arange(n))
    for r, root in enumerate(fo.foreach_roots(t)):
        c = fj.json_cell(t, s, msg[off:off + ln], int(root), [b"a"])
        assert c.value == texts[r].encode(), r
    msg = fe.list_scan_message(n)
    rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
    for kind in fe.LIST_SCAN_KINDS:
        st, cnt, el, tx = fe.list_scan_expected(kind, n)
        at = 0
        for r, root in enumerate(fo.foreach_roots(t)):
            c, e, b = fl.list_cell(t, s, msg[off:off + ln], int(root), [b"a"], kind)
            assert (c.status, len(e)) == (st[r], cnt[r]), (kind, r)
            assert e == el[at:at + cnt[r]].tolist(), (kind, r)
            if tx is not None:
                assert b == "".join(tx[at:at + cnt[r]].tolist()).encode()
            at += cnt[r]
    for first, last in ((0, 40), (fe.ROW_RECORDS - 30, fe.ROW_RECORDS)):
        msg = fe.rows_scan_message(first, last)
        rc, t, s, (off, ln) = oracle.parse(msg, ndjson=True)
        assert rc == 0
        st, offs, tags, idx, cells = fr.find_rows(t, s, msg[off:off + ln], [b"a"], [[b"k"]], [fl.ARRAY_INT64])
        assert np.array_equal(np.diff(offs), fe.row_scan_shape(np.arange(first, last)))
        q0 = int(fe.row_scan_shape(np.arange(first)).sum())
        q = np.arange(q0, q0 + len(idx))
        assert [c[3] for c in cells[0]] == fe.row_scan_inner(q).tolist()
        assert [c[4] for c in cells[0]] == [[(int(x) + j) % 10 for j in range(int(k))] for x, k in zip(q, fe.row_scan_inner(q))]
    # the full sizes: every count array crosses entry 2^22
    assert fe.SCAN_PATHS * fe.SCAN_RECORDS > fe.GROUP
    pool = sum(int(fe.list_scan_expected(k)[1].sum()) for k in fe.list_scan_kinds())
    nbytes = sum(int(fe.list_scan_expected(k)[2].sum()) for k in fe.list_scan_kinds() if k in fl.STRING_LISTS)
    assert pool > fe.GROUP and nbytes > fe.GROUP, (pool, nbytes)
    assert fe.ROW_RECORDS > fe.GROUP and int(fe.row_scan_shape(np.arange(fe.ROW_RECORDS)).sum()) > fe.GROUP
