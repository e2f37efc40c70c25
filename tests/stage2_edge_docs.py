"""Documents that put JSON items on the edges of the per-structural stage 2 (stage2.cuh), the kernels every parse with
copy_strings off, and every parse of a context set to stage-2 implementation 1, runs.

Their geometry is counted in structurals, not bytes: K2a / K2e take S2_ITEMS structurals per thread (a warp covers
32 * S2_ITEMS), K2c one per thread with a prefix per 32 structurals, K2b scans tiles of S2_TILE structurals in groups of
1 024 tiles.  `place` puts an item's first structural at a chosen index of stage 1's index; the other generators build
strings at K1's backslash-map block and word edges, bracket counts at the levels of K2d's minimum tree, and number
densities on either side of the threshold for the dense number kernels (K2g / K2h).

Every document carries what it is meant to test (`Doc`); tests/test_stage2_edge_docs_cpu.py checks those intentions
against the CPU oracle's stage 1 and parse, and tests/test_gpu_stage2_structural_edges.py runs the documents through
the kernels.  The constants are read from the headers, so a change of geometry moves the documents with it."""
import json
import os
import re
from dataclasses import dataclass, field

_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "simdjson-go_b200", "csrc")


def _const(header, name):
    with open(os.path.join(_CSRC, header)) as f:
        src = f.read()
    return int(re.search(r"constexpr\s+\w+\s+%s\s*=\s*(\d+)\s*;" % name, src).group(1))


S2_THREADS = _const("stage2_common.cuh", "S2_THREADS")
S2_ITEMS = _const("stage2.cuh", "S2_ITEMS")
S2_COOP_MIN = _const("stage2.cuh", "S2_COOP_MIN")
S2_DENSE_NUMBERS_SHIFT = _const("stage2.cuh", "S2_DENSE_NUMBERS_SHIFT")
S2_FAST_MIN_BACKSLASHES = _const("stage2.cuh", "S2_FAST_MIN_BACKSLASHES")
S2_TILE = S2_THREADS * S2_ITEMS                 # structurals per K2a / K2e block = one K2b tile
S2_WARP = 32 * S2_ITEMS                         # structurals per K2a / K2e warp
S2_GROUP = 1024 * S2_TILE                       # K2b: scan_groups_kernel runs 1 024 tiles per block
BS_BLOCK = 64                                   # K1's backslash map: one bit per 64-byte block ...
BS_WORD = 32 * BS_BLOCK                         # ... one u32 word per 2 KiB step

FILLERS = (b"0,", b"true,", b"null,")           # two structurals each; `0,` makes the document number-heavy


@dataclass
class Doc:
    name: str
    msg: bytes
    ndjson: bool
    ok: bool                        # the oracle (and so the kernels) must accept it
    at: int = None                  # stage 1's index of the trimmed message has ...
    byte: int = None                # ... this byte offset of `msg` at index `at`
    want: dict = field(default_factory=dict)    # further intentions, see test_stage2_edge_docs_cpu.py


# ---- items placed at a structural index -------------------------------------------------------------------------------
# (name, text, accepted, may be a root / sits in a flat record) -- `text`'s first byte is its first structural
ITEMS = [
    ("number", b"-12.5e-3", True), ("uint", b"18446744073709551615", True),
    ("true", b"true", True), ("false", b"false", True), ("null", b"null", True),
    ("obj", b"{}", True), ("arr", b"[]", True), ("pair", b"[{}]", True),
    ("kv_num", b'{"k":0}', True), ("kv_str", b'{"k":"v"}', True), ("kv_arr", b'{"k":[]}', True),
    ("key_colon", b'{"a":null,"bb":true}', True),
    ("str", b'"abc"', True), ("str_esc", b'"a\\"b\\\\c\\n"', True), ("str_surrogate", b'"\\ud83d\\ude00x"', True),
    ("bad_escape", b'"\\q"', False), ("bad_atom", b"tru", False), ("bad_atom2", b"nulL", False),
    ("bad_number", b"-", False), ("bad_number2", b"01", False), ("mismatched", b"[}", False),
]
CONTAINERS = {"obj", "arr", "pair", "kv_num", "kv_str", "kv_arr", "key_colon", "mismatched"}
# NDJSON only: a record boundary, and runs of 1-3 blank lines, inside the item (the prefix's record stays open)
ND_ITEMS = [("record", b"0]\n[0", True)] + [("blank%d" % r, b"0]" + b"\n" * (r + 1) + b"[0", True) for r in (1, 2, 3)] + \
           [("blank_ws", b"0]\n \n\t\n[0", True)]
ND_TAIL = b'\n{"z":[1]}'


def place(item, at, filler, ndjson):
    """(msg, byte offset of the item) with the item's first structural at index `at` of stage 1's index.  Odd `at`:
    `[` + fillers; even: `[[` + fillers (single document) or `{}` NEWLINE `[` + fillers (NDJSON: a flat record, so that
    an item holding a record boundary closes it); `at` 0: the item is the (first) root.  None where that cannot be."""
    name, text, _ = item
    flat = name in {n for n, _, _ in ND_ITEMS}
    if at == 0:
        if name not in CONTAINERS:
            return None
        pre, post = b"", b""
    elif at % 2:
        pre, post = b"[" + filler * ((at - 1) // 2), b"]"
    elif ndjson and at >= 4:
        pre, post = b"{}\n[" + filler * ((at - 4) // 2), b"]"
    elif not flat:
        pre, post = b"[[" + filler * ((at - 2) // 2), b"]]"
    else:
        return None
    return pre + text + post + (ND_TAIL if ndjson else b""), len(pre)


def edges():
    """(edge, offsets): every multiple of S2_ITEMS inside a K2a warp, the warp, K2c's 32, the tile, the second tile
    (a non-zero tile prefix) and the group; offsets E-5..E+4, narrower at the group edge (2 MB documents)"""
    out = [(e, range(e - 5, e + 5)) for e in range(S2_ITEMS, S2_WARP + 1, S2_ITEMS)]
    if not any(e == 32 for e, _ in out):
        out.append((32, range(27, 37)))
    out += [(S2_TILE, range(S2_TILE - 5, S2_TILE + 5)), (2 * S2_TILE, range(2 * S2_TILE - 5, 2 * S2_TILE + 5)),
            (S2_GROUP, range(S2_GROUP - 2, S2_GROUP + 2))]
    return out


def placed_docs(ndjson, group=True):
    """every item at every index of `edges()` (each index once), with every filler below the group edge and one
    filler per index (in turn) at it"""
    ats = set()
    for e, offs in edges():
        if e == S2_GROUP and not group:
            continue
        ats.update(a for a in offs if a >= 0)
    items = ITEMS + (ND_ITEMS if ndjson else [])
    for at in sorted(ats):
        fillers = FILLERS if at < S2_GROUP - 5 else (FILLERS[at % len(FILLERS)],)
        for filler in fillers:
            for item in items:
                r = place(item, at, filler, ndjson)
                if r is None:
                    continue
                msg, off = r
                yield Doc("place:%s@%d/%s%s" % (item[0], at, filler[:-1].decode(), "/nd" if ndjson else ""), msg, ndjson,
                          item[2], at, off, {"filler": filler})


# ---- strings -----------------------------------------------------------------------------------------------------------
def _unescaped_len(body):
    return len(json.loads(b'"' + body + b'"').encode("utf-8", "surrogatepass"))


def _escaped_body(dl, per_window, esc):
    """a string body whose unescaped length is `dl`, with `per_window` escapes `esc` in every 32 source bytes"""
    src, n, step = bytearray(), 0, 32 // per_window
    esc_dl = _unescaped_len(esc)
    while n < dl:
        w = len(src) % 32
        if w % step == 0 and w + len(esc) <= 32 and (w // step) < per_window and n + esc_dl <= dl:
            src += esc
            n += esc_dl
        else:
            src += b"a"
            n += 1
    return bytes(src)


def _string_forms(name, s, want, ok=True):
    """a string (with its quotes) as key and value of a one-member object, and among other values of an array"""
    yield Doc(name + "/obj", b'{' + s + b':' + s + b'}', False, ok, 1, 1, dict(want))
    yield Doc(name + "/arr", b'[0,' + s + b',null]', False, ok, 3, 3, dict(want))


def string_docs():
    for ln in (0, 1, 31, 32, 33, 63, 64, 65, 300):
        yield from _string_forms("str:plain%d" % ln, b'"' + b"s" * ln + b'"', {"dl": ln, "sl": ln})
    for dl in (S2_COOP_MIN - 1, S2_COOP_MIN, S2_COOP_MIN + 1):
        # backslashes per 32 source bytes below, at and above K2c's S2_FAST_MIN_BACKSLASHES
        for per in range(max(1, S2_FAST_MIN_BACKSLASHES - 2), S2_FAST_MIN_BACKSLASHES + 3):
            for esc in (b"\\n", b"\\u00e9", b'\\"'):
                body = _escaped_body(dl, per, esc)
                yield from _string_forms("str:esc%d/%dper32/%s" % (dl, per, esc[1:2].decode()), b'"' + body + b'"',
                                         {"dl": dl, "sl": len(body), "per_window": per})
    # next_pos - ps (the measure's bound, whitespace behind the string included) just below, at and above S2_COOP_MIN
    for gap in (S2_COOP_MIN - 1, S2_COOP_MIN, S2_COOP_MIN + 1):
        for body in (b"a\\nb", b"xyz", b"\\u00e9" * 3, b""):
            s = b'"' + body + b'"'
            for ws in (b" ", b"\n", b"\t", b"\r"):
                pad = ws * (gap - len(s))
                yield Doc("str:gap%d/%s/%r" % (gap, body.decode(), ws), b'[' + s + pad + b',1]', False, True, 1, 1,
                          {"gap": gap})
                yield Doc("str:gapkey%d/%s/%r" % (gap, body.decode(), ws), b'{' + s + pad + b':1}', False, True, 1, 1,
                          {"gap": gap})


def edge_string_docs():
    """strings whose body crosses a 64-byte block edge or a 2 KiB word edge of K1's backslash map; the backslash sits
    in the body's first block only, its last block only, nowhere, or in another string that shares the first or the
    last block (a false positive: the measure must take the slow path and still agree)"""
    for edge in (BS_BLOCK, 10 * BS_BLOCK, BS_WORD, 2 * BS_WORD):
        for a in (1, 2, 40, 63):            # body bytes in front of the edge
            for b in (1, 2, 40, 63):        # body bytes behind it
                for where in ("first", "last", "none", "other_first", "other_last"):
                    s = edge - a                    # first body byte; the opening quote is at s - 1
                    e = edge + b                    # closing quote
                    body = bytearray(b"x" * (a + b))
                    if where == "first":
                        body[0:2] = b"\\n"
                    elif where == "last":
                        if e % BS_BLOCK < 2:
                            continue
                        body[-2:] = b"\\n"
                    decoy_front = where == "other_first"
                    if decoy_front and s % BS_BLOCK < 6:
                        continue
                    if where == "other_last" and e % BS_BLOCK > BS_BLOCK - 5:
                        continue
                    front = b'"\\n",' if decoy_front else b""
                    head = b"[" + b" " * (s - 2 - len(front)) + front
                    if len(head) < 1 or s - 1 - len(front) < 1:
                        continue
                    tail = (b',"\\n"' if where == "other_last" else b"") + b",1]"
                    msg = head + b'"' + bytes(body) + b'"' + tail
                    assert msg[s - 1:s] == b'"' and msg[e:e + 1] == b'"'
                    yield Doc("str:edge%d/%d+%d/%s" % (edge, a, b, where), msg, False, True, 3 if decoy_front else 1, s - 1,
                              {"body": (s, e), "edge": edge, "bs": where})


def leading_space_docs():
    """1-63 spaces in front of documents: the trimmed window (and, with copy off, the tape's message offsets) moves
    against the blocks of the untrimmed input"""
    bases = [b'{"k":"' + b"v" * 70 + b'","e":"a\\nb","n":[1,2.5,"x"]}',
             b'["' + b"w" * 2100 + b'","\\u00e9' + b"z" * 40 + b'"]']
    for i, base in enumerate(bases):
        for k in range(1, 64):
            yield Doc("lead:%d/%d" % (i, k), b" " * k + base, False, True, 0, k, {})
            yield Doc("lead_nd:%d/%d" % (i, k), b" " * k + base + b"\n" + base + b"\n", True, True, 0, k, {})


# ---- brackets and numbers ----------------------------------------------------------------------------------------------
def min32_levels(nb):
    """s2_min32 launches of K2d for nb brackets: one per level of 32-wide minima above the brackets themselves"""
    lv = 0
    while nb > 32:
        nb = (nb + 31) // 32
        lv += 1
    return lv


def bracket_docs():
    for depth in (1023, 1024, 1025, 3000):
        yield Doc("nest:%d" % depth, b"[" * depth + b"]" * depth, False, True, 0, 0, {"brackets": 2 * depth})
    for k in (1, 2, 3):
        for nb in (32 ** k - 1, 32 ** k, 32 ** k + 1):
            pairs = (nb + 1) // 2 - 1                       # `[` + pairs * `[]` + `]`: 2 + 2 * pairs brackets
            msg = b"[" + b",".join([b"[]"] * pairs) + b"]"
            if nb % 2:                                      # an odd count cannot balance: drop the last close
                msg = msg[:-1]
            yield Doc("flat:%d" % nb, msg, False, nb % 2 == 0, 0, 0, {"brackets": nb})


def density_docs():
    """n_num << S2_DENSE_NUMBERS_SHIFT equal to n - 1, n and n + 1 (n: stage 1's structural count): `[` v values `]`
    has 2 v + 1 structurals; one `[]` among the values makes it 2 v + 2"""
    for n_num in (1, 3, 64, 1000, 70000):
        for delta in (-1, 0, 1):
            n = (n_num << S2_DENSE_NUMBERS_SHIFT) - delta
            vals = [b"-1.5", b"7", b"123456789", b"0.25e3"] * (n_num // 4 + 1)
            vals = vals[:n_num]
            if n % 2:
                v = (n - 1) // 2
                rest = [b"true"] * (v - n_num)
            else:
                v = (n - 2) // 2
                rest = [b"[]"] + [b"null"] * (v - n_num - 1)
            vals = [x for pair in zip(vals, rest) for x in pair] + vals[len(rest):] + rest[len(vals):]
            yield Doc("dense:%d%+d" % (n_num, delta), b"[" + b",".join(vals) + b"]", False, True, 0, 0,
                      {"n": n, "numbers": n_num, "dense": delta >= 0})


def record_docs():
    """NDJSON record counts around K2f's 256 records per block"""
    for nrec in (255, 256, 257, 511, 512, 513):
        yield Doc("records:%d" % nrec, b"\n".join(b'{"r":%d}' % i for i in range(nrec)), True, True, 0, 0, {"records": nrec})
        yield Doc("records_blank:%d" % nrec, b"\n\n".join(b"[%d]" % i for i in range(nrec)) + b"\n", True, True, 0, 0,
                  {"records": nrec})


def all_docs(group=True):
    """every document above: placed items single-document and NDJSON, then the string, bracket, density and record
    documents"""
    yield from placed_docs(False, group)
    yield from placed_docs(True, group)
    yield from string_docs()
    yield from edge_string_docs()
    yield from leading_space_docs()
    yield from bracket_docs()
    yield from density_docs()
    yield from record_docs()
