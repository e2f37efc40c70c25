"""Inputs that put the device find's shared pieces at their edges: the one number accessor (fd_number) and text writer
(fd_cell_text) under every cell kind that calls them, the warp-aggregated stop (fj_lower_stop) at every lane and round
of one warp call, and the one count-array scan (scan_counts) past a group of its count array.  Test infrastructure:
generators, the exact conversion spec they are checked against, and the places their words land on.

The word passes of the list cells and array rows run over a path's virtual words (the cells laid end to end): a tile
is TAPE_TILE = 4 096 words, thread t of a tile takes the TAPE_ROUNDS = 4 consecutive words from 4t on, and word j of
every lane of a warp is one call of fj_lower_stop.  So one warp call covers a window of 32 x 4 = 128 words, and two
words of a window meet in the same call exactly when they sit on the same round (offset mod 4)."""
import math
import struct
from fractions import Fraction

import numpy as np

from tests import consumer_edge_tapes as ce
from tests import find_lists_oracle as fl
from tests import find_oracle as fo
from tests import fmt_values
from tests.tape_builder import TapeBuilder, word

TILE, ROUNDS, LANES = 4096, 4, 32
WARP = LANES * ROUNDS               # the virtual words of one warp call
GROUP = TILE * 1024                 # a count-array group: 1 024 tiles
M64 = (1 << 64) - 1
NUMERIC = {fo.FLOAT64: fl.ARRAY_FLOAT64, fo.INT64: fl.ARRAY_INT64, fo.UINT64: fl.ARRAY_UINT64}


def place(v):
    """(tile, warp in the tile, lane, round) of virtual word v"""
    t = v % TILE
    return v // TILE, t // WARP, (t // ROUNDS) % LANES, v % ROUNDS


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


# ---- the exact spec --------------------------------------------------------------------------------------------------
def spec_number(tag, p, kind):
    """(ok, value bits) of Float / Int / Uint (kinds FLOAT64 / INT64 / UINT64) or AsFloat / AsInteger / AsUint64 (the
    ARRAY_ kinds) of the number (tag, p), from the Go source with Python ints only:
      Int and AsInteger pass -2^63 <= x <= 2^63 (and NaN); the value is x truncated toward zero, 1<<63 for 2^63 and NaN
      Uint passes 0 <= x <= 2^64, AsUint64 0 <= x <= 2^63 (both: -0.0 and NaN too); amd64's float64ToUint64 is the
        truncation below 2^64 and 1<<63 for 2^64 and NaN
      int64 / uint64 -> float64 round to nearest, ties to even (Python's float(int))"""
    signed = p - (1 << 64) if p >> 63 else p
    if kind in (fo.FLOAT64, fl.ARRAY_FLOAT64):
        return True, p if tag == "d" else f64_bits(float(signed if tag == "l" else p))
    to_int = kind in (fo.INT64, fl.ARRAY_INT64)
    if tag in "lu":
        x = signed if tag == "l" else p
        ok = x < 1 << 63 if to_int else x >= 0
        return ok, (x & M64) if ok else 0
    x = f64(p)
    if math.isnan(x):
        return True, 1 << 63
    if math.isinf(x):
        return False, 0
    lo, hi = (-(1 << 63), 1 << 63) if to_int else (0, 1 << 64 if kind == fo.UINT64 else 1 << 63)
    if not lo <= Fraction(x) <= hi:
        return False, 0
    t = int(x)
    if t == (1 << 64) or (to_int and t == 1 << 63):
        return True, 1 << 63
    return True, t & M64


def spec_list(items, kind):
    """(status, elements) of a numeric list of item specs under kind: the first item that fails decides"""
    out = []
    for it in items:
        if it[0] not in ("d", "l", "u"):
            return fo.CONVERT, []
        ok, v = spec_number(it[0], it[1], kind)
        if not ok:
            return fo.CONVERT, []
        out.append(v)
    return fo.OK, out


def shortest_digits(s):
    """the significant digits of a decimal numeral: no sign, point, exponent, leading or trailing zeros"""
    m = s.lower().split("e")[0].lstrip("-").replace(".", "")
    return m.strip("0") or "0"


# ---- §1: conversions in every numeric and text walk ------------------------------------------------------------------
OK_ITEM = ("l", 7)
NOP = [word("N", 1), word("n")]     # a nop that skips the one word behind it


def conversion_specs():
    return ce.conversion_values() + ce.CONVERSION_OTHERS


def list_forms(spec):
    """the arrays each spec is read in: [v] and [ok, v, ok]"""
    return [[spec], [OK_ITEM, spec, OK_ITEM]]


def _put_items(b, items, nop_before=None):
    for it in items:
        if nop_before is not None and it is nop_before:
            b.words(NOP)
        ce.put_value(b, it)


def list_tape(specs, nop=False):
    """one record {"k":[...]} per form of list_forms() of every spec; with nop, a nop in front of the spec's item"""
    b = TapeBuilder(raw=True)
    for sp in specs:
        for form in list_forms(sp):
            b.open("r"); b.open("{"); b.string(b"k"); b.open("[")
            _put_items(b, form, sp if nop else None)
            b.close(3)
    return b.build()


def rows_tape(specs, lists=False, per_record=17):
    """records {"r":[{"k":v0},{"k":v1},...]} (lists: {"r":[{"k":[v0]},{"k":[ok, v1, ok]},...]}), per_record
    elements each"""
    b = TapeBuilder()
    for at in range(0, len(specs), per_record):
        b.open("r"); b.open("{"); b.string(b"r"); b.open("[")
        for i, sp in enumerate(specs[at:at + per_record]):
            b.open("{"); b.string(b"k")
            if lists:
                b.open("[")
                _put_items(b, list_forms(sp)[i % 2])
                b.close()
            else:
                ce.put_value(b, sp)
            b.close()
        b.close(3)
    return b.build()


def json_text(spec):
    """the JSON text of a number or atom spec, or None (Inf and NaN, which JSON cannot express, strings and arrays)"""
    tag = spec[0]
    if tag == "d":
        x = f64(spec[1])
        return None if math.isinf(x) or math.isnan(x) else repr(x)
    if tag == "l":
        return str(spec[1] - (1 << 64) if spec[1] >> 63 else spec[1])
    if tag == "u":
        return str(spec[1])
    return {"t": "true", "f": "false", "n": "null", "{": '{"a":true}'}.get(tag)


def conversion_message(specs):
    """NDJSON, one record per expressible spec v: {"k":v,"l":[v],"m":[7,v,7],"r":[{"k":v},{"k":[v]}]}"""
    lines = []
    for sp in specs:
        v = json_text(sp)
        if v is not None:
            lines.append('{"k":%s,"l":[%s],"m":[7,%s,7],"r":[{"k":%s},{"k":[%s]}]}' % (v, v, v, v, v))
    return "\n".join(lines).encode()


# ---- §2: StringCvt text at every writer ------------------------------------------------------------------------------
def text_specs():
    """the conversion table's numbers, the 24-byte extremes, int64's minimum, uint64's maximum and a slice of
    fmt_values.notation_edges()"""
    out = list(ce.conversion_values())
    out += [("d", f64_bits(-1.7976931348623157e308)), ("d", f64_bits(-2.2250738585072014e-308)),
            ("l", (-(1 << 63)) & M64), ("u", M64)]
    out += [("d", int(x)) for x in fmt_values.notation_edges()[::3]]
    return out


def text_scalar_tape(specs):
    """records {"k":v}: pad rows (small ints) so that the specs' rows straddle row 4 096, the first tile edge of the
    STRING_CVT column's byte scan"""
    pad = TILE - len(specs) // 2
    b = TapeBuilder()
    for sp in [("l", i % 1000) for i in range(pad)] + list(specs):
        b.open("r"); b.open("{"); b.string(b"k")
        ce.put_value(b, sp)
        b.close(2)
    return b.build(), pad


def text_list_tape(specs, nop=False):
    """two records {"k":[pad..., specs...]}: one-word pads (true) so that the specs straddle virtual word 4 096 (the
    byte scan's first tile edge), then the specs reversed; with nop a nop leads each array (one thread writes it)"""
    b = TapeBuilder(raw=True)
    words = sum(ce.Records.width(s) for s in specs)
    for k, items in enumerate((list(specs), list(specs)[::-1])):
        b.open("r"); b.open("{"); b.string(b"k"); b.open("[")
        if nop:
            b.words(NOP)
        if k == 0:
            b.atoms(("t", TILE - 1 - words // 2 - (len(NOP) if nop else 0)))
        _put_items(b, items)
        b.close(3)
    return b.build()


def text_rows_tape(specs):
    """one record {"r":[{"k":pad}..., {"k":v}...]}: its rows straddle row 4 096"""
    pad = TILE - len(specs) // 2
    return rows_tape([("l", i % 1000) for i in range(pad)] + list(specs), per_record=10 ** 9), pad


# ---- §3: stop words inside one warp call -----------------------------------------------------------------------------
# per family: the list kinds it is read under, its filler items by word count, the items a row's first stop is made
# of (CONVERT for the lists) and those of its second stop.  A second stop ends the walk with no error (OK, with the
# elements in front of it) or, for array rows, after more rows, so a cell that stopped on it instead of on the first
# would read differently.  Numeric lists read heads at odd offsets only (2-word fillers), so a family without a 1-word
# filler shifts a cell's parity with a padding row [t] of 3 words.
STOP_FAMILIES = {
    "numeric": ((fl.ARRAY_FLOAT64, fl.ARRAY_INT64, fl.ARRAY_UINT64), {2: ("l", 3)},
                [('"', b"s", True)], [("]",)]),
    "string": ((fl.ARRAY_STRING,), {2: ('"', b"ab", True)},
               [("l", 5), ("[", 0)], [("x",), ("]",)]),
    "string_cvt": ((fl.ARRAY_STRING_CVT,), {1: ("t",), 2: ('"', b"ab", True)},
                   [("[", 0), ("{",), ("d", 0x7FF8000000000000)], [("x",), ("]",)]),
    "rows": ((), {1: ("t",), 2: ("l", 3)}, [("x",)], [("y",)]),
}


def _fill(gap, fills):
    """filler items of exactly `gap` words, or None"""
    if gap < 0 or (gap % 2 and 1 not in fills):
        return None
    return [fills[2]] * (gap // 2) + ([fills[1]] if gap % 2 else [])


RAW_ITEMS = ("x", "y", "]")


def _width(it):
    return 1 if it[0] in RAW_ITEMS else ce.Records.width(it)


def _put(b, it):
    if it[0] in RAW_ITEMS:
        b.words([word(it[0])])      # unknown tags and a stray ']' end every walk with no error
    else:
        ce.put_value(b, it)


def stop_cases():
    """(a, b, tile_end): the first stop on offset a of a warp window, the second on offset b of it (b >= 128: a later
    window), the window the last of its tile when tile_end.  b takes every value up to 140 for a in (0, 1, 62, 125,
    127), and a sample of the same round and of others for every other a"""
    out = []
    for a in range(WARP):
        if a in (0, 1, 62, 125, 127):
            bs = range(a + 1, a + 141)
        else:  # its neighbours, its round on later lanes, and its round on a lane of the next window
            bs = {a + 1, a + 2, a + 3, a + 4, a + 8, a + 20, a + 44, a + 128 - 4 * (a % 3)}
        out += [(a, b, False) for b in sorted(bs)]
    out += [(a, b, True) for a in (3, 64, 120, 127) for b in (a + 4, 128 + (a % 4), 131 + 4 * 8, a + 129)]
    return out


def stop_tape(family, cases=None, disarm=False):
    """one record {"a":[...]} per case whose first stop lands on virtual word A = W + a of a warp window W and whose
    second stop on B = W + b, each behind a neighbour row of fillers whose own stop (its ']') lands on N = A - 4: A's
    round on the lane in front of A's, in A's warp call whenever a >= 4.  Cases a family cannot place (a gap its
    fillers cannot fill) are dropped.  disarm: the same tape with every first stop replaced by fillers of its width,
    so the case rows stop on B.  Returns (tape, strings, message, placed) with placed = [(row, A, B, N)] for the case
    rows."""
    kinds, fills, first, second = STOP_FAMILIES[family]
    cases = stop_cases() if cases is None else cases
    b = TapeBuilder(raw=True)
    v, row, placed = 0, 0, []

    def cell(items):
        nonlocal v, row
        b.open("r"); b.open("{"); b.string(b"a"); b.open("[")
        for it in items:
            _put(b, it)
        b.close(3)
        v += 2 + sum(_width(it) for it in items)
        row += 1

    for a, bb, tile_end in cases:
        picks = [(s1, _fill(bb - a - _width(s1), fills), s2) for s1 in first for s2 in second]
        picks = [p for p in picks if p[1] is not None]
        if not picks:
            continue
        s1, mid, s2 = picks[(a + bb) % len(picks)]
        for _ in range(2):
            W = (v + 5 - a + WARP - 1) // WARP * WARP                  # the first window with A >= v + 5
            if tile_end:
                W = max(W, (W // TILE + 1) * TILE - WARP)
            A, B, N = W + a, W + bb, W + a - 4
            nb = _fill(N - v - 1, fills)
            if nb is not None:
                cell(nb)                                               # the neighbour: '[' at v, ']' at N
                placed.append((row, A, B, N))
                head = _fill(_width(s1), fills) if disarm else [s1]
                cell(_fill(2, fills) + head + mid + [s2] + [fills[min(fills)]])   # '[' at N + 1
                break
            cell([("t",)])                                             # 3 words: the next cell's parity flips
    t, s, m = b.build()
    return t, s, m, placed


def virtual_cells(tape, strings, path=(b"a",)):
    """(row heads, V): every root's array at `path` as the word passes lay it out (the '[' of row r at virtual word
    V[r], V[-1] the total); rows without an array add no words"""
    heads, V = [], [0]
    for r in fo.foreach_roots(tape):
        c = fo.find_cell(tape, strings, b"", int(r), list(path), fo.ELEMENT)
        ok = c.status == fo.OK and c.tag == ord("[")
        heads.append(c.index if ok else -1)
        V.append(V[-1] + ((int(tape[c.index]) & fo.VAL) - c.index if ok else 0))
    return heads, V


# ---- §4: every scan_counts caller past a count-array group ----------------------------------------------------------
SCAN_PATHS = 64                     # FD_MAX_PATHS
SCAN_RECORDS = GROUP // SCAN_PATHS + 1                 # 65 537: 64 paths' cells cross entry 2^22
ROW_RECORDS = GROUP + 3
LIST_SCAN_KINDS = (fl.ARRAY_FLOAT64, fl.ARRAY_INT64, fl.ARRAY_UINT64, fl.ARRAY_STRING, fl.ARRAY_STRING_CVT)


def json_scan_kind(r):
    """the value of record r of json_scan_message: 0 null, 1 the int r, 2 [], 3 [r % 10,1], 4 {"b":true}, 5 no "a"
    """
    return (r * 5 + r // 3) % 6


def json_scan_texts(r):
    """the MarshalJSON text of every record's "a" (b"" where it has none), vectorised over the int array r"""
    k = json_scan_kind(r)
    ints = np.char.mod("%d", r)
    pair = np.char.add(np.char.add("[", np.char.mod("%d", r % 10)), ",1]")
    t = np.where(k == 0, "null", np.where(k == 1, ints, np.where(k == 2, "[]", np.where(k == 3, pair, np.where(
        k == 4, '{"b":true}', "")))))
    return t


def json_scan_message(n=SCAN_RECORDS):
    r = np.arange(n)
    k = json_scan_kind(r)
    t = json_scan_texts(r)
    lines = np.where(k == 5, np.char.add(np.char.add('{"z":', t), "0}"), np.char.add(np.char.add('{"a":', t), "}"))
    return "\n".join(lines.tolist()).encode()


def list_scan_shape(r):
    """record r of list_scan_message: (element count 0..4, strings instead of ints) vectorised"""
    return (r * 3 + r // 5) % 5, r % 7 == 3


def list_scan_values(r, j):
    return (r * 31 + j * 7) % 100000


def list_scan_message(n=SCAN_RECORDS):
    r = np.arange(n)
    cnt, strs = list_scan_shape(r)
    lines = []
    for i in range(n):
        vs = [list_scan_values(i, j) for j in range(cnt[i])]
        body = ",".join(('"s%d"' % x) if strs[i] else str(x) for x in vs)
        lines.append('{"a":[%s]}' % body)
    return "\n".join(lines).encode()


def list_scan_kinds():
    return [LIST_SCAN_KINDS[p % len(LIST_SCAN_KINDS)] for p in range(SCAN_PATHS)]


def list_scan_expected(kind, n=SCAN_RECORDS):
    """(status, element counts, elements, text per row) of one path of list_scan_message, vectorised (text only for
    the string lists)"""
    r = np.arange(n)
    cnt, strs = list_scan_shape(r)
    ok = np.ones(n, dtype=bool)
    if kind in (fl.ARRAY_FLOAT64, fl.ARRAY_INT64, fl.ARRAY_UINT64):
        ok = ~strs | (cnt == 0)
    elif kind == fl.ARRAY_STRING:
        ok = strs | (cnt == 0)
    c = np.where(ok, cnt, 0)
    rr = np.repeat(r, c)
    jj = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
    vals = list_scan_values(rr, jj)
    is_s = np.repeat(strs, c)
    texts = None
    if kind == fl.ARRAY_FLOAT64:
        el = vals.astype(np.float64).view(np.uint64)
    elif kind in (fl.ARRAY_INT64, fl.ARRAY_UINT64):
        el = vals.astype(np.uint64)
    else:
        t = np.char.mod("%d", vals)
        t = np.where(is_s, np.char.add("s", t), t)
        el = np.char.str_len(t).astype(np.uint64)
        texts = t
    return np.where(ok, fo.OK, fo.CONVERT), c, el, texts


def row_scan_shape(r):
    """record r of rows_scan_message: its element count 0..3"""
    return (r * 3 + r // 5) % 4


def row_scan_inner(q):
    """row q (an element {"k":[...]}) of rows_scan_message: its list's length 0..2; its values are (q + j) % 10"""
    return (q * 5 + q // 3) % 3


def rows_scan_message(first=0, last=ROW_RECORDS):
    """NDJSON records first .. last - 1 of {"a":[{"k":[...]},...]}: row_scan_shape elements, row_scan_inner values"""
    r = np.arange(first, last)
    n = row_scan_shape(r)
    all_n = row_scan_shape(np.arange(ROW_RECORDS)) if first else None
    q0 = int(all_n[:first].sum()) if first else 0
    m = row_scan_inner(np.arange(q0, q0 + int(n.sum())))
    q = np.arange(q0, q0 + m.size)
    elem = {}
    for mm in range(3):
        for d in range(10):
            elem[(mm, d)] = '{"k":[%s]}' % ",".join(str((d + j) % 10) for j in range(mm))
    et = [elem[(int(a), int(b))] for a, b in zip(m.tolist(), (q % 10).tolist())]
    out, at = [], 0
    for c in n.tolist():
        out.append('{"a":[' + ",".join(et[at:at + c]) + "]}")
        at += c
    return "\n".join(out).encode()
