"""Documents placed against the tiles of K2t (simdjson-go_b200/csrc/s2s_tile.h), the streaming stage 2's scope matching:
one CTA per S2T_TILE brackets, a search that leaves its tile climbs the minima of the depths.

Their geometry is counted in brackets: every document says where its brackets fall relative to the tile edges, and
`want` holds what must hold of it (the oracle gives the tape and the verdict).  K2r links a pair itself when both ends
lie in one 2 KiB step of the message, so the cases that matter here come with long strings between the two ends as well."""
import collections

T = 2048          # S2T_TILE: brackets per K2t tile
STEP = 2048       # K2r's step: a pair inside one is linked by K2r, not by K2t

Doc = collections.namedtuple("Doc", "name msg ndjson want")


def _gap(n=STEP + 100):
    """a string longer than a step: the brackets around it lie in different steps"""
    return b'"' + b"x" * n + b'"'


def _flat(pairs):
    """'[' + pairs x '[]' + ']': 2 * pairs + 2 brackets, pair j at brackets (2j + 1, 2j + 2) -- one pair straddles every
    odd tile edge"""
    return b"[" + b"[]," * (pairs - 1) + (b"[]" if pairs else b"") + b"]"


def _count(msg):
    return sum(msg.count(c) for c in (b"[", b"]", b"{", b"}"))


def count_docs():
    """0, 1, T - 1, T, T + 1, k T +- 1 brackets: even counts balanced, odd ones with the outer '[' left open"""
    out = [Doc("nb0", b'"no brackets"', False, {"brackets": 0, "ok": False}),
           Doc("nb0-nd", b"1\n2\n", True, {"brackets": 0, "ok": False})]
    for nb in (1, 2, 3, T - 2, T - 1, T, T + 1, T + 2, 2 * T - 1, 2 * T, 2 * T + 1, 3 * T - 1, 3 * T + 1):
        if nb % 2 == 0:
            out.append(Doc("nb%d" % nb, _flat((nb - 2) // 2), False, {"brackets": nb, "ok": True}))
            out.append(Doc("nb%d-nd" % nb, b"\n".join([b"{}"] * (nb // 2)), True, {"brackets": nb, "ok": True}))
        else:
            out.append(Doc("nb%d" % nb, b"[" + (b"[]," * ((nb - 3) // 2) + b"[]" if nb > 1 else b""), False,
                           {"brackets": nb, "ok": False}))
    for d in out:
        assert _count(d.msg) == d.want["brackets"], d.name
    return out


def edge_docs():
    """pairs and containers at and across the tile edges, with and without K2r's in-step link"""
    out = []
    # the open is the last bracket of tile 0, the close the first of tile 1; with a step between them K2r leaves them to K2t
    for gap in (b"", _gap()):
        m = b"[" + b"[]," * (T // 2 - 1) + b"[" + gap + b"]]"
        out.append(Doc("pair-across-edge" + ("-gap" if gap else ""), m, False, {"edge_pair": T - 1}))
        m = b"[" + b"{}," * (T // 2 - 1) + b'{"k":' + (gap or b"1") + b"}]"
        out.append(Doc("obj-across-edge" + ("-gap" if gap else ""), m, False, {"edge_pair": T - 1}))
    # a partner several tiles back: one '[', >= 3T brackets of balanced pairs inside it, then ']'
    out.append(Doc("partner-3-tiles-back", _flat(3 * T // 2 + 7), False, {"span_tiles": 3}))
    out.append(Doc("partner-4-tiles-back-obj", b'{"a":' + _flat(2 * T) + b',"b":' + _gap() + b"}", False, {"span_tiles": 4}))
    # nesting deeper than a tile
    out.append(Doc("deep-5000", b"[" * 5000 + b"]" * 5000, False, {"depth": 5000}))
    out.append(Doc("deep-5000-obj", b'{"a":' * 2500 + b"[" * 2500 + b"1" + b"]" * 2500 + b"}" * 2500, False, {"depth": 5000}))
    out.append(Doc("deep-9000-mixed", (b'[{"a":' * 4500) + b"true" + (b"}]" * 4500), False, {"depth": 9000}))
    # every bracket of the later tiles has its smaller-depth partner only in tile 0
    out.append(Doc("parent-in-tile-0", b"[" + b"{}," * (3 * T // 2) + b"{}]", False, {"parent": 0}))
    out.append(Doc("parent-in-tile-0-obj", b'{"a":[' + b"[]," * (2 * T) + b'[]],"b":{}}', False, {"parent": 1}))
    # a rising and falling saw across many tiles: par far back inside a tile and on every level of the minima
    saw = b"".join(b"[" * d + b"1" + b"]" * d + b"," for d in range(1, 200)) + b"2"
    out.append(Doc("saw", b"[" + saw + b"]", False, {}))
    return out


def ndjson_docs():
    """records straddling tile edges, short ones (K2r links them) and ones longer than a step (K2t links them)"""
    out = []
    short = b'{"a":[1,{"b":[]}],"c":{}}'  # 8 brackets
    for lead in range(0, 8, 3):
        pre = b"\n".join([b"[]"] * lead) + (b"\n" if lead else b"")
        out.append(Doc("nd-short-lead%d" % lead, pre + b"\n".join([short] * (3 * T // 8 + 5)), True, {}))
    long_ = b'{"a":[1,{"b":[]}],"s":' + _gap() + b',"c":{"d":[[]]}}'  # 10 brackets, longer than a step
    out.append(Doc("nd-long", b"\n".join([long_] * (T // 10 + 9)), True, {}))
    mixed = b"\n".join((long_ if i % 7 == 3 else short) for i in range(2 * T // 8 + 40))
    out.append(Doc("nd-mixed", mixed, True, {}))
    # one record spanning several tiles, the records around it short
    big = b'{"x":' + _flat(T + 3) + b',"s":' + _gap() + b"}"
    out.append(Doc("nd-record-over-tiles", b"\n".join([short] * 600 + [big] + [short] * 600), True, {}))
    return out


def bad_docs():
    """unbalanced and mismatched input at the tile edges: they fail as the oracle fails"""
    out = []
    head = b"[" + b"[]," * (T // 2 - 1)  # brackets 0 .. T - 2
    out.append(Doc("mismatch-at-edge", head + b"{]}]", False, {"ok": False}))          # '{' = T - 1, ']' = T
    out.append(Doc("mismatch-at-edge-gap", head + b"{" + _gap() + b"]}]", False, {"ok": False}))
    # ']' = T - 1 closes the root, the extra close is bracket T
    out.append(Doc("extra-close-first-of-tile", head[:-1] + b"]}", False, {"ok": False}))
    out.append(Doc("extra-close-first-of-tile-2", head[:-1] + b"]]" + b"[]" * 10, False, {"ok": False}))
    # bracket T - 1 closes an array inside an object; segment T (",1]") is legal only in an array: the tile of bracket T
    # finds the object through two searches into tile 0
    mid = b'[{"a":[' + b"[]," * ((T - 4) // 2 - 1) + b"[]"
    out.append(Doc("object-context-across-edge", mid + b"],1]]", False, {"ok": False, "edge_close": T - 1}))
    out.append(Doc("object-context-across-edge-ok", mid + b'],"b":1}]', False, {"ok": True, "edge_close": T - 1}))
    out.append(Doc("unclosed-last-tile", _flat(T + 100)[:-1] + b",[", False, {"ok": False}))
    out.append(Doc("unclosed-last-tile-gap", b"[" + _flat(T)[:-1] + b"," + _gap() + b"]", False, {"ok": False}))
    out.append(Doc("swap-across-tiles", b"{" + b'"a":' + _flat(T) + b"]", False, {"ok": False}))
    nd = b"\n".join([b'{"a":[1]}'] * (T // 4 + 3))
    out.append(Doc("nd-extra-close", nd + b"}\n" + nd, True, {"ok": False}))
    out.append(Doc("nd-unclosed", nd + b"\n{" + b"[]," * (T // 2) + b"[]", True, {"ok": False}))
    out.append(Doc("nd-mismatch-at-edge", b"\n".join([b"[]"] * (T // 2 - 1)) + b"\n{]\n" + b"\n".join([b"{}"] * 100), True,
                   {"ok": False}))
    return out


def all_docs():
    return count_docs() + edge_docs() + ndjson_docs() + bad_docs()
