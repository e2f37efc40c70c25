"""The edge documents of tests/stage2_edge_docs.py are what they claim to be: checked against the CPU oracle's stage 1
(the index the per-structural stage 2 is built on) and its parse.  Without this the GPU tests that run them could drift
off their edges, after a change of geometry or of a generator, and still pass."""
import numpy as np
import pytest

import tests.stage2_edge_docs as E

# what the generator must keep producing: deleting one of these kinds fails test_every_kind_is_generated
ITEM_KINDS = {"number", "uint", "true", "false", "null", "obj", "arr", "pair", "kv_num", "kv_str", "kv_arr", "key_colon",
              "str", "str_esc", "str_surrogate", "bad_escape", "bad_atom", "bad_atom2", "bad_number", "bad_number2",
              "mismatched"}
ND_ITEM_KINDS = {"record", "blank1", "blank2", "blank3", "blank_ws"}
STRING_KINDS = {"plain0", "plain1", "plain31", "plain32", "plain33", "plain63", "plain64", "plain65", "plain300"}
EDGE_STRING_KINDS = {"first", "last", "none", "other_first", "other_last"}


def _edges():
    """the structural indices every item must be placed at, derived here from the constants on their own"""
    es = list(range(E.S2_ITEMS, 32 * E.S2_ITEMS + 1, E.S2_ITEMS)) + [32, E.S2_THREADS * E.S2_ITEMS, 2 * E.S2_THREADS * E.S2_ITEMS]
    want = {a for e in es for a in range(e - 5, e + 5) if a >= 0}
    g = 1024 * E.S2_THREADS * E.S2_ITEMS
    return want, set(range(g - 2, g + 2))


def _index(oracle, doc):
    a, b = oracle.trim_space(doc.msg)
    win = doc.msg[a:b]
    ok, deltas = oracle.find_structural_indices(win, doc.ndjson)
    assert ok, doc.name
    return a, win, (np.cumsum(deltas.astype(np.int64)) - 1)


def _check(oracle, doc, stats):
    a, win, pos = _index(oracle, doc)
    if doc.at is not None:
        assert doc.at < len(pos) and int(pos[doc.at]) == doc.byte - a, (doc.name, doc.at, len(pos))
    rc, tape, _, _ = oracle.parse(doc.msg, ndjson=doc.ndjson, copy_strings=False)
    assert (rc == 0) == doc.ok, (doc.name, rc)
    w = doc.want
    chars = np.frombuffer(win, dtype=np.uint8)[pos]
    n_num = int(((chars == ord("-")) | ((chars >= ord("0")) & (chars <= ord("9")))).sum())
    dense = n_num != 0 and (n_num << E.S2_DENSE_NUMBERS_SHIFT) >= len(pos)
    if "filler" in w:
        stats.setdefault(doc.name.split("@")[0], set()).add(dense)
    ps = int(pos[doc.at]) if doc.at is not None else None
    if "dl" in w:
        ok, sl, dl = oracle.parse_string_validate_only(win[ps:], int(pos[doc.at + 1]) - ps)
        assert ok and (sl, dl) == (w["sl"], w["dl"]), (doc.name, sl, dl)
    if "per_window" in w:
        body = win[ps + 1:ps + 1 + w["sl"]]
        counts = [body[i:i + 32].count(b"\\") for i in range(0, len(body) - 31, 32)]
        assert counts and counts[0] == w["per_window"] and all(1 <= c <= 5 for c in counts), (doc.name, counts)
    if "gap" in w:
        assert int(pos[doc.at + 1]) - ps == w["gap"], doc.name
    if "body" in w:
        s, e = w["body"]
        edge = w["edge"]
        assert ps == s - 1 and win[e:e + 1] == b'"' and int(pos[doc.at + 1]) > e and s < edge <= e - 1, doc.name
        if edge % E.BS_WORD == 0:
            assert (s // E.BS_BLOCK) // 32 != (e // E.BS_BLOCK) // 32, doc.name      # the block range spans two map words
        bs = np.nonzero(np.frombuffer(win, dtype=np.uint8) == ord("\\"))[0]
        blocks = sorted({int(i) // E.BS_BLOCK for i in bs} & set(range(s // E.BS_BLOCK, e // E.BS_BLOCK + 1)))
        in_body = [int(i) for i in bs if s <= i < e]
        want = {"first": [s // E.BS_BLOCK], "last": [e // E.BS_BLOCK], "none": [], "other_first": [s // E.BS_BLOCK],
                "other_last": [e // E.BS_BLOCK]}[w["bs"]]
        assert blocks == want, (doc.name, blocks)
        assert bool(in_body) == (w["bs"] in ("first", "last")), doc.name
    if "brackets" in w:
        assert int(np.isin(chars, np.frombuffer(b"[]{}", dtype=np.uint8)).sum()) == w["brackets"], doc.name
    if "n" in w:
        assert (len(pos), n_num, dense) == (w["n"], w["numbers"], w["dense"]), (doc.name, len(pos), n_num)
    if "records" in w:
        assert int((tape >> np.uint64(56) == ord("r")).sum()) // 2 == w["records"], doc.name
    return doc


def test_placed_items_sit_on_their_edges(oracle_native):
    stats, seen = {}, {}
    for nd in (False, True):
        for doc in E.placed_docs(nd, group=False):
            _check(oracle_native, doc, stats)
            kind = doc.name.split(":")[1].split("@")[0]
            seen.setdefault((kind, nd), set()).add(doc.at)
    want, _ = _edges()
    for kind in ITEM_KINDS:
        for nd in (False, True):
            got = seen.get((kind, nd), set())
            assert want - {0} <= got, (kind, nd, sorted(want - got)[:8])
    for kind in ND_ITEM_KINDS:
        assert want - {0, 2} <= seen.get((kind, True), set()), kind
    # `0,` fillers make the document number-heavy (K2g / K2h), `true,` / `null,` keep numbers inline in K2c
    assert stats["place:number"] == {True, False} and stats["place:uint"] == {True, False}


def test_placed_items_at_the_group_edge(oracle_native):
    _, want = _edges()
    seen = {}
    for nd in (False, True):
        for doc in E.placed_docs(nd):
            if doc.at < min(want):
                continue
            _check(oracle_native, doc, {})
            seen.setdefault(doc.name.split(":")[1].split("@")[0], set()).add(doc.at)
    assert set(seen) == ITEM_KINDS | ND_ITEM_KINDS
    assert all(v == want for v in seen.values()), seen


@pytest.mark.parametrize("gen", ["string_docs", "edge_string_docs", "leading_space_docs", "bracket_docs", "density_docs",
                                 "record_docs"])
def test_shaped_documents(oracle_native, gen):
    docs = [_check(oracle_native, d, {}) for d in getattr(E, gen)()]
    names = {d.name for d in docs}
    if gen == "string_docs":
        assert {k for k in STRING_KINDS if "str:%s/obj" % k in names and "str:%s/arr" % k in names} == STRING_KINDS
        assert {d.want["dl"] for d in docs if "per_window" in d.want} == {E.S2_COOP_MIN - 1, E.S2_COOP_MIN, E.S2_COOP_MIN + 1}
        f = E.S2_FAST_MIN_BACKSLASHES
        assert {f - 1, f, f + 1} <= {d.want["per_window"] for d in docs if "per_window" in d.want}
        assert {d.want["gap"] for d in docs if "gap" in d.want} == {E.S2_COOP_MIN - 1, E.S2_COOP_MIN, E.S2_COOP_MIN + 1}
    if gen == "edge_string_docs":
        for edge in (E.BS_BLOCK, E.BS_WORD):
            assert {d.want["bs"] for d in docs if d.want["edge"] == edge} == EDGE_STRING_KINDS, edge
    if gen == "leading_space_docs":
        assert {d.byte for d in docs} == set(range(1, 64))
    if gen == "bracket_docs":
        assert {d.want["brackets"] for d in docs} >= {32 ** k + j for k in (1, 2, 3) for j in (-1, 0, 1)}
        assert {d.want["brackets"] for d in docs if d.name.startswith("nest")} == {2046, 2048, 2050, 6000}
    if gen == "density_docs":
        assert {d.want["n"] - (d.want["numbers"] << E.S2_DENSE_NUMBERS_SHIFT) for d in docs} == {-1, 0, 1}
        assert max(d.want["n"] for d in docs) > 1024 * E.S2_TILE       # one of them crosses a K2b group
    if gen == "record_docs":
        assert {d.want["records"] for d in docs} == {255, 256, 257, 511, 512, 513}
