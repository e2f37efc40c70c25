"""Documents that put stage 1's verdict on the edges of K1's parse mode (stage1.cuh, stage1_flatten_kernel with PARSE),
the stage 1 of every parse through the streaming stage 2 (copy_strings on, stage-2 implementation 0).

K1 works in 64-byte blocks (one lane each), 2 KiB steps (one warp pass), slabs of S1_STEPS steps (one warp), tiles of
S1_WARPS slabs (one CTA, one look-back) and grid rounds of `ctas` tiles (the cooperative grid deals tiles round-robin).
Its verdict -- a control character inside a string, a message that ends inside a string, the last structural's byte,
and the invalid escapes its counts find for stage 2 -- depends on carries across every one of those edges, so each
document places one byte at offsets E-2 .. E+1 of an edge E:

  a  a control character inside a string                               STAGE1
  b  a control character just outside a string                         STAGE2 (OK for JSON whitespace)
  c  0x20, 0x7F, 0x80, 0xFF inside and outside a string                 OK inside; STAGE2 outside, but for the space
  d  the message ends inside a string, at the edge                     STAGE1 (OK where an even backslash run closes it)
  e  the last structural far from the end, or `]` / `}` at the edge    STAGE1 / OK
  f  an invalid escape at the edge, alone or with a control character   STAGE2 / STAGE1 (stage 1 wins)
     inside a string in an earlier or a later tile
  g  the twin of an a, b, c or f document with the offending byte made harmless ('x' inside a string, a space or a
     newline outside, the escape's backslash made 'x'): accepted, so the tape and Strings.B are compared

The string that holds (or, in b, ends just in front of) the placed byte opens near it, in the slab, tile or grid round
in front of its own, or ends in a backslash run of 1, 2 or 33 in front of a quote next to the byte (an odd run escapes
the quote: the byte stays inside; an even one closes the string: the byte is outside).

The large documents (past two grid rounds) are written into one canvas of spaces and undone after use, so a generator
yields a view that is valid until it is advanced.  tests/test_stage1_verdict_docs_cpu.py checks every intention against
the CPU oracle; tests/test_gpu_stage1_parse_verdict.py runs the documents through the kernels.  The geometry is read
from the headers, so a change of geometry moves the documents with it."""
import os
import re
from dataclasses import dataclass, field

import numpy as np

_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "simdjson-go_b200", "csrc")


def _constants():
    """the integer constexprs of s2s_core.h and stage1.cuh, evaluated in order (S1_STEPS is S2S_STEPS, S1_SLAB_BYTES a
    product of two others, ...)"""
    env = {}
    for header in ("s2s_core.h", "stage1.cuh"):
        with open(os.path.join(_CSRC, header)) as f:
            src = f.read()
        for m in re.finditer(r"constexpr\s+(?:int|unsigned|uint32_t|size_t)\s+(\w+)\s*=\s*([^;]+);", src):
            expr = re.sub(r"\((?:int|unsigned|uint32_t|size_t|uint64_t)\)", "", m.group(2))
            try:
                env[m.group(1)] = int(eval(expr, {"__builtins__": {}}, dict(env)))
            except (NameError, SyntaxError, TypeError):
                pass
    return env


_C = _constants()
STEP = _C["S1_STEP_BYTES"]          # one warp pass: 32 lanes x 64 bytes
SLAB = _C["S1_SLAB_BYTES"]          # one warp's slab
TILE = _C["S1_TILE_BYTES"]          # one CTA's tile = one look-back
BLOCK = 64
assert STEP == 32 * BLOCK and SLAB == _C["S1_STEPS"] * STEP and TILE == _C["S1_WARPS"] * SLAB

CTRL6 = (0x00, 0x01, 0x09, 0x0A, 0x0D, 0x1F)     # at every edge
NONCTRL = (0x20, 0x7F, 0x80, 0xFF)
WS = (0x09, 0x0A, 0x0D, 0x20)
OPENS = ("near", "prev_slab", "prev_tile", "prev_round", "esc1", "esc2", "esc33")
SPOTS_OUT = ("after_close", "before_open", "key_colon", "between")
FAMILIES = "abcdefg"
EDGE_KINDS = ("block", "step", "slab", "tile", "round")


def edges(R):
    """(kind, E): every block edge inside the middle step of the second slab (lanes 0..31 at bits 63 / 0), the two step
    edges of the second slab, the first, second and last slab edge of the first tile, T, T + slab, 2T, and R, R + T, 2R
    for a grid round of R bytes"""
    base = SLAB + STEP
    out = [("block", base + BLOCK * k) for k in range(1, STEP // BLOCK)]
    out += [("step", SLAB + STEP * k) for k in range(1, SLAB // STEP)]
    out += [("slab", SLAB), ("slab", 2 * SLAB), ("slab", TILE - SLAB)]
    out += [("tile", TILE), ("tile", TILE + SLAB), ("tile", 2 * TILE)]
    out += [("round", R), ("round", R + TILE), ("round", 2 * R)]
    return out


OFFSETS = (-2, -1, 0, 1)


def _offsets(kind, fam):
    """every offset, but at the grid-round edges (documents of 12-25 MiB) only the byte on either side of the edge for
    the families other than a and b"""
    return OFFSETS if kind != "round" or fam in "ab" else (-1, 0)


@dataclass
class Doc:
    name: str
    family: str
    msg: np.ndarray                 # uint8 view of the canvas: valid until the generator is advanced
    pos: int                        # the placed byte
    edge: tuple                     # (kind, E); kind "end" for the documents that have no edge of their own
    verdicts: dict                  # {ndjson: "OK" | "STAGE1" | "STAGE2"} for the modes the family applies in
    inside: bool = None             # the placed byte lies inside a string
    open: int = None                # the opening quote of that string (a, b, c, d)
    want: dict = field(default_factory=dict)

    @property
    def modes(self):
        return sorted(self.verdicts)


class Canvas:
    """a buffer of spaces that documents are written into and undone from"""

    def __init__(self, cap):
        self.a = np.full(cap, 0x20, dtype=np.uint8)
        self.dirty = []

    def fill(self, lo, hi, c):
        if hi > lo:
            self.a[lo:hi] = c
            self.dirty.append((lo, hi))

    def put(self, off, b):
        if isinstance(b, int):
            b = bytes([b])
        self.a[off:off + len(b)] = np.frombuffer(b, dtype=np.uint8)
        self.dirty.append((off, off + len(b)))

    def reset(self):
        for lo, hi in self.dirty:
            self.a[lo:hi] = 0x20
        self.dirty.clear()


def _starts(pos, R):
    return {"prev_slab": pos // SLAB * SLAB, "prev_tile": pos // TILE * TILE, "prev_round": pos // R * R}


def _open_at(v, pos, R, c):
    """the opening quote of the string in front of the placed byte for opening variant `v`; `c` is where the string's
    last quote (closing, or escaped with an odd run) sits; None where the variant cannot be"""
    if v == "near":
        o = c - 2
    elif v.startswith("esc"):
        o = c - int(v[3:]) - 6
    else:
        o = _starts(pos, R)[v] - 40
    return o if o >= 2 else None


def _string(cv, o, c, run):
    """`"` at o, body of 'a', a run of `run` backslashes in front of a quote at c (no quote at c for run None)"""
    cv.put(o, b'"')
    if run is None:
        cv.fill(o + 1, c, ord("a"))
        return
    cv.fill(o + 1, c - run, ord("a"))
    cv.fill(c - run, c, ord("\\"))
    cv.put(c, b'"')


def _out_verdict(x, spot, nd):
    if spot == "between":
        return "OK" if (nd and x == 0x0A) else "STAGE2"
    if x in WS:
        return "STAGE2" if (nd and x == 0x0A) else "OK"
    return "STAGE2"


def _in_out_doc(cv, fam, x, v, spot, pos, R, twin):
    """one a / b / c document (or its twin): the byte x at pos inside (spot None) or outside a string that opens per
    variant v.  Returns (doc fields) or None where the variant cannot be placed."""
    run = int(v[3:]) if v.startswith("esc") else None
    inside = spot is None
    if inside and run is not None and run % 2 == 0:
        return None                                   # an even run closes the string: that is an outside document
    if not inside and run is not None and run % 2 == 1:
        return None
    if inside:
        c = pos - 1 if run is not None else pos       # the (escaped) quote in front of the byte, or the byte itself
        o = _open_at(v, pos, R, c)
        if o is None:
            return None
        cv.put(0, b"[")
        _string(cv, o, c, run)
        tail = b'aa"]'
        verdict = {nd: ("OK" if twin else ("STAGE1" if x < 0x20 else "OK")) for nd in (False, True)}
        harmless = ord("x")
    else:
        c = pos - 1 if spot == "after_close" or spot == "key_colon" else pos - 2
        o = _open_at(v, pos, R, c)
        if o is None:
            return None
        cv.put(0, b"{" if spot == "key_colon" else b"[")
        _string(cv, o, c, run if run is not None else 0)
        if spot == "before_open":
            cv.put(pos - 1, b",")
        elif spot == "between":
            cv.put(pos - 1, b"]")
        tail = {"after_close": b"]", "before_open": b'"b"]', "key_colon": b":1}", "between": b"[0]"}[spot]
        harmless = 0x0A if spot == "between" else 0x20
        modes = (True,) if spot == "between" else (False, True)
        verdict = {nd: _out_verdict(harmless if twin else x, spot, nd) for nd in modes}
    cv.put(pos, harmless if twin else x)
    cv.put(pos + 1, tail)
    return pos + 1 + len(tail), verdict, inside, o


def _rot(seq, i):
    return seq[i % len(seq)]


def _combos(kind, E, R, opens, fam):
    """(offset, variant) pairs of one edge, each placeable variant at each offset"""
    for o in _offsets(kind, fam):
        pos = E + o
        for v in opens:
            if v.startswith("prev") and _starts(pos, R)[v] < 64:
                continue
            yield pos, v


def inside_outside_docs(R, cv, families="abc"):
    """families a, b, c and their twins (g).  Every combination of offset and opening variant at every edge gets one
    byte (and for b / c one spot) in rotation, so each edge sees each byte; the first slab edge and the step edges get
    every control character 0x00..0x1F with the `near` opening."""
    cv.reset()                          # (whatever a consumer that stopped early left behind)
    for ei, (kind, E) in enumerate(edges(R)):
        for fam in families:
            items = []
            for i, (pos, v) in enumerate(_combos(kind, E, R, OPENS, fam)):
                if fam == "a":
                    if v == "esc2":
                        continue
                    items.append((pos, v, _rot(CTRL6, i + ei), None))
                elif fam == "b":
                    if v in ("esc1", "esc33"):
                        continue
                    items.append((pos, v, _rot(CTRL6, i + ei), _rot(SPOTS_OUT, i // 2 + ei)))
                else:
                    inside = i % 2 == 0
                    if v in (("esc2",) if inside else ("esc1", "esc33")):
                        continue
                    items.append((pos, v, _rot(NONCTRL, i // 2 + ei), None if inside else _rot(SPOTS_OUT, i // 4 + ei)))
            if fam == "a" and (kind == "step" or E == SLAB):
                items += [(E + o, "near", x, None) for o in OFFSETS for x in range(0x20) if x not in CTRL6]
            for j, (pos, v, x, spot) in enumerate(items):
                # twins: every combination below one tile, every other one at the tile and round edges
                twins = (False, True) if fam != "c" and (kind not in ("tile", "round") or j % 2) else (False,)
                for twin in twins:
                    r = _in_out_doc(cv, fam, x, v, spot, pos, R, twin)
                    if r is None:
                        cv.reset()
                        continue
                    n, verdict, inside, o = r
                    name = "%s:%s/%s/%02x@%s%+d" % ("g" if twin else fam, v, spot or "in", x, kind, pos - E)
                    yield Doc(name, "g" if twin else fam, cv.a[:n], pos, (kind, E), verdict, inside, o,
                              {"of": fam, "byte": x, "spot": spot or "in", "open_variant": v})
                    cv.reset()


def unterminated_docs(R, cv):
    """family d: the message's last byte at the edge, inside a string -- opened near it, a tile or a grid round in
    front; ending in a quote behind a run of 1, 2, 31, 32, 33 or 64 backslashes (alone: STAGE1 either way; with `]`
    behind it: accepted exactly when the run is even); in NDJSON, a raw newline inside the string at a slab edge"""
    cv.reset()                          # (whatever a consumer that stopped early left behind)
    for ei, (kind, E) in enumerate(edges(R)):
        if kind == "block":                 # (three of the six runs at each block edge, in turn)
            runs = (1, 2, 33) if ei % 2 else (31, 32, 64)
        elif kind in ("tile", "round"):
            runs = (1, 2, 33, 64)
        else:
            runs = (1, 2, 31, 32, 33, 64)
        for o in _offsets(kind, "d"):
            pos = E + o
            for v in ("near", "prev_tile", "prev_round"):
                op = _open_at(v, pos, R, pos)
                if op is None or (v != "near" and _starts(pos, R)[v] < 64):
                    continue
                cv.put(0, b"[")
                _string(cv, op, pos + 1, None)
                yield Doc("d:%s@%s%+d" % (v, kind, pos - E), "d", cv.a[:pos + 1], pos, (kind, E),
                          {False: "STAGE1", True: "STAGE1"}, True, op, {"last": True})
                cv.reset()
            for run in (runs if kind not in ("tile", "round") or o in (-1, 0) else ()):
                for close in (False, True):
                    q = pos - 1 if close else pos         # the quote; with `]` behind it that is the last byte
                    op = q - run - 4
                    if op < 2:
                        continue
                    cv.put(0, b"[")
                    _string(cv, op, q, run)
                    n = q + 1
                    if close:
                        cv.put(q + 1, b"]")
                        n += 1
                    ok = close and run % 2 == 0
                    yield Doc("d:run%d%s@%s%+d" % (run, "_close" if close else "", kind, pos - E), "d", cv.a[:n], pos,
                              (kind, E), {False: "OK" if ok else "STAGE1", True: "OK" if ok else "STAGE1"},
                              True, op, {"last": True, "run": run, "close": close})
                    cv.reset()
            if kind in ("slab", "tile", "round") and o == -1:
                # NDJSON: a raw newline inside a string that crosses the slab edge, the message ending 40 bytes on
                op = pos - 30
                cv.put(0, b"[")
                _string(cv, op, pos + 41, None)
                cv.put(pos, b"\n")
                yield Doc("d:nd_newline@%s%+d" % (kind, pos - E), "d", cv.a[:pos + 41], pos, (kind, E),
                          {True: "STAGE1"}, True, op, {"last": False, "byte": 0x0A})
                cv.reset()


def last_structural_docs(R, cv):
    """family e: `[1,2]` / `{"a":1}` and a run of 'x' up to the edge (the last structural is the run's first byte:
    STAGE1); the same documents with spaces up to `]` / `}` at the edge (every tile between holds no structural: OK);
    documents of one structural"""
    cv.reset()                          # (whatever a consumer that stopped early left behind)
    for kind, E in edges(R):
        for o in _offsets(kind, "e"):
            pos = E + o
            heads = ((b"[1,2", b"]"), (b'{"a":1', b"}"))
            if kind in ("tile", "round"):   # (one of the two in turn)
                heads = heads[o % 2:][:1]
            for head, close in heads:
                cv.put(0, head + close)
                cv.fill(len(head) + 1, pos + 1, ord("x"))
                yield Doc("e:xrun%s@%s%+d" % (close.decode(), kind, pos - E), "e", cv.a[:pos + 1], pos, (kind, E),
                          {False: "STAGE1", True: "STAGE1"}, False, None, {"last": True, "last_structural": len(head) + 1})
                cv.reset()
                cv.put(0, head)
                cv.put(pos, close)
                yield Doc("e:close%s@%s%+d" % (close.decode(), kind, pos - E), "e", cv.a[:pos + 1], pos, (kind, E),
                          {False: "OK", True: "OK"}, False, None, {"last": True, "last_structural": pos})
                cv.reset()
    for one, v in ((b"]", "STAGE2"), (b"}", "STAGE2"), (b"[", "STAGE1"), (b"1", "STAGE1"), (b'"a"', "STAGE1")):
        cv.put(0, one)
        yield Doc("e:one/%s" % one.decode(), "e", cv.a[:len(one)], 0, ("end", len(one)), {False: v, True: v}, False,
                  None, {"last_structural": 0})
        cv.reset()


ESCAPES = (b"\\uZZZZ", b"\\x", b'\\u12"]')


def escape_docs(R, cv):
    """family f: an invalid escape with its backslash at the edge (an escape whose head lies in the slab in front
    reaches K1's head_info); the truncated `\\u12` ends the message.  With o = -1 also a string holding 0x01 at the
    start of the message and one a tile behind the escape: stage 1's verdict wins.  Twins (g): the backslash made 'x'."""
    cv.reset()                          # (whatever a consumer that stopped early left behind)
    for kind, E in edges(R):
        for o in _offsets(kind, "f"):
            pos = E + o
            for k, esc in enumerate(ESCAPES):
                v = ("near", "prev_slab", "prev_tile")[(o + k) % 3]
                if _starts(pos, R).get(v, 64) < 64:
                    v = "near"
                extras = ["", "early", "late"] if o == -1 else [""]
                for extra in extras + ["twin"]:
                    op = _open_at(v, pos, R, pos)
                    if op is None or (extra == "early" and op < 8):
                        continue
                    cv.put(0, b"[")
                    if extra == "early":
                        cv.put(1, b'"\x01",')
                    _string(cv, op, pos, None)
                    cv.put(pos, b"x" if extra == "twin" else b"\\")
                    cv.put(pos + 1, esc[1:])
                    n = pos + len(esc)
                    if not esc.endswith(b"]"):
                        cv.put(n, b'a"')
                        n += 2
                        if extra == "late":
                            cv.put(n, b",")
                            cv.put(n + TILE, b'"\x01"')
                            n += TILE + 3
                        cv.put(n, b"]")
                        n += 1
                    elif extra == "late":
                        continue
                    if extra == "twin":
                        verdict, fam = "OK", "g"
                    else:
                        verdict, fam = ("STAGE1" if extra else "STAGE2"), "f"
                    yield Doc("%s:%s%s/%s@%s%+d" % (fam, esc[:3].decode().replace("\\", "bs"), "/" + extra if extra else "",
                                                    v, kind, pos - E), fam, cv.a[:n], pos, (kind, E),
                              {False: verdict, True: verdict}, True, op,
                              {"of": "f", "escape": esc, "extra": extra, "last": esc.endswith(b"]")})
                    cv.reset()


def canvas(R):
    return Canvas(2 * R + 2 * TILE + 4096)


def all_docs(R, cv=None):
    cv = cv or canvas(R)
    yield from inside_outside_docs(R, cv)
    yield from unterminated_docs(R, cv)
    yield from last_structural_docs(R, cv)
    yield from escape_docs(R, cv)
