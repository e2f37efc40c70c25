"""The verdict documents of tests/stage1_verdict_docs.py are what they claim to be, checked with the CPU oracle alone:
the intended verdict is the oracle's, in every NDJSON mode the family applies in; the placed byte sits at its offset on
its side of its edge; the quote state in front of it, and where its string opened, are the intended ones; every family
reaches every edge kind.  Without this the GPU test that runs them could drift off its edges and still pass."""
import numpy as np
import pytest

import tests.stage1_verdict_docs as V

RC = {"OK": 0, "STAGE1": 1, "STAGE2": 2}
GEOMETRY = {"block": V.BLOCK, "step": V.STEP, "slab": V.SLAB, "tile": V.TILE}


def _structurals(oracle, msg, nd):
    _, deltas = oracle.find_structural_indices(msg, nd)
    return np.cumsum(deltas.astype(np.int64)) - 1


def _quote_state(oracle, d):
    """(inside, structural positions) at the placed byte: the byte is replaced by a comma, which is a structural
    exactly when it lies outside every string (the index is the oracle's; for an unterminated string it still runs to
    the end)"""
    m = d.msg.copy()
    m[d.pos] = ord(",")
    pos = _structurals(oracle, m, False)
    return d.pos not in set(pos.tolist()), pos


def _check(oracle, d, R):
    msg = d.msg
    for nd, v in d.verdicts.items():
        rc = oracle.parse(msg, ndjson=nd, copy_strings=True)[0]
        assert rc == RC[v], (d.name, nd, rc, v)
    assert msg[0] not in V.WS and msg[-1] not in V.WS, d.name          # nothing for the host's trim to move
    kind, E = d.edge
    if kind != "end":
        assert d.pos - E in V.OFFSETS, d.name
        if kind == "round":
            assert E in (R, R + V.TILE, 2 * R), d.name
        elif kind == "tile":                    # (T + slab: the first slab edge behind a look-back)
            assert E in (V.TILE, V.TILE + V.SLAB, 2 * V.TILE), d.name
        else:
            unit = GEOMETRY[kind]
            outer = {"block": V.STEP, "step": V.SLAB, "slab": V.TILE, "tile": R}[kind]
            assert E % unit == 0 and E % outer != 0, d.name
    if d.want.get("last") and d.family in "de":
        assert d.pos == len(msg) - 1, d.name                              # the placed byte is the message's last
    if d.want.get("last") and "escape" in d.want:
        assert d.pos + len(d.want["escape"]) == len(msg), d.name
    if "byte" in d.want and d.family != "g":
        assert msg[d.pos] == d.want["byte"], d.name
    if d.family in "abcg" and "escape" not in d.want:
        inside, pos = _quote_state(oracle, d)
        assert inside == d.inside, (d.name, inside)
        # the string the byte is in, or ends just in front of, opened at d.open: a structural quote, and nothing
        # structural between it and the byte but the `,` / `]` a spot puts right in front of the byte
        assert msg[d.open] == ord('"') and d.open in set(pos.tolist()), d.name
        between = pos[(pos > d.open) & (pos < d.pos)]
        assert all(between == d.pos - 1) and (len(between) == 0 or not d.inside), (d.name, between[:4])
        v = d.want.get("open_variant", "")
        if v.startswith("prev"):
            assert d.open < V._starts(d.pos, R)[v] <= d.pos, d.name      # the string crosses the slab / tile / round start
    if d.family == "d":
        # the message ends inside the string that opened at d.open, unless an even run closed it: behind the message
        # (its raw newline made 'a'), `,]` leaves stage 1 unterminated, or puts a structural comma at len(msg)
        m = np.concatenate([np.where(msg == 0x0A, np.uint8(ord("a")), msg), np.frombuffer(b",]", dtype=np.uint8)])
        ok, deltas = oracle.find_structural_indices(m, False)
        ends_inside = not ok
        assert ends_inside or len(msg) in set((np.cumsum(deltas.astype(np.int64)) - 1).tolist()), d.name
        assert msg[d.open] == ord('"') and ends_inside == (d.want.get("run", 1) % 2 == 1), d.name
    if d.family == "e":
        # the message's last structural: the one in front of a `]` put behind it (which makes stage 1 accept)
        pos = _structurals(oracle, np.append(msg, np.uint8(ord("]"))), False)
        assert pos[-1] == len(msg) and int(pos[-2]) == d.want["last_structural"], (d.name, pos[-3:])
    if d.family in "fg" and "escape" in d.want:
        assert msg[d.pos] == (ord("x") if d.family == "g" else ord("\\")), d.name


@pytest.mark.parametrize("ctas", [132, 114])
def test_documents_keep_their_intentions(oracle_native, ctas):
    R = ctas * V.TILE
    seen, n = {}, 0
    for d in V.all_docs(R):
        _check(oracle_native, d, R)
        seen.setdefault(d.family, set()).add(d.edge[0])
        n += 1
    # every family reaches every edge kind (family e also has documents of one structural)
    for fam in V.FAMILIES:
        assert set(V.EDGE_KINDS) <= seen.get(fam, set()), (fam, seen.get(fam))
    assert "end" in seen["e"]
    assert n > 5000, n


def test_every_variant_is_generated():
    """the bytes, openings, spots, runs and escapes the generators promise, each at every edge kind"""
    R = 132 * V.TILE
    got = {}
    for d in V.all_docs(R):
        kind = d.edge[0]
        w = d.want
        if d.family == "a":
            got.setdefault(("a-byte", w["byte"]), set()).add(kind)
            got.setdefault(("a-open", w["open_variant"]), set()).add(kind)
        elif d.family in "bc":
            got.setdefault((d.family + "-spot", w["spot"]), set()).add(kind)
            got.setdefault((d.family + "-byte", w["byte"]), set()).add(kind)
            got.setdefault((d.family + "-open", w["open_variant"]), set()).add(kind)
        elif d.family == "d" and "run" in w:
            got.setdefault(("d-run", w["run"], w["close"]), set()).add(kind)
        elif d.family == "f":
            got.setdefault(("f", w["escape"], w["extra"]), set()).add(kind)
    every = set(V.EDGE_KINDS)
    for x in V.CTRL6:
        assert got[("a-byte", x)] == every, x
    assert {k[1] for k in got if k[0] == "a-byte"} == set(range(0x20))
    for v in ("near", "esc1", "esc33"):
        assert got[("a-open", v)] == every, v
    for v in ("prev_slab", "prev_tile", "prev_round"):
        assert ("round" in got[("a-open", v)] and "round" in got[("b-open", v)]), v
    assert got[("a-open", "prev_slab")] >= {"block", "step", "slab", "tile"}
    assert got[("b-open", "esc2")] == every
    for s in V.SPOTS_OUT:
        assert got[("b-spot", s)] == every and got[("c-spot", s)] == every, s
    for x in V.CTRL6:
        assert got[("b-byte", x)] == every, x
    for x in V.NONCTRL:
        assert got[("c-byte", x)] == every, x
    for run in (1, 2, 33, 64):
        for close in (False, True):
            assert got[("d-run", run, close)] == every, (run, close)
    for esc in V.ESCAPES:
        assert got[("f", esc, "")] == every, esc
    for extra in ("early", "late"):
        assert got[("f", b"\\uZZZZ", extra)] == every, extra
