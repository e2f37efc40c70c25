"""Tapes and messages that put the work of the device tape consumers on their edges: the root finder (tape.cuh: KM1's
head scan, KC1a / KC1b), countWhere (consume.cuh: KC2) and the find (find.cuh: KF3 fd_walk, KF5 fd_emit).

Every generator records what it intends -- the slot of every root, the cell every path must give on every row, the
edge and offset of every feature -- so that tests/test_consumer_edge_tapes_cpu.py can check those intentions against
the sequential ports (tests/find_oracle.py, the C oracle's count_where) and tests/test_gpu_consumer_edges.py can check
the device against the intentions.  The expected cells are computed here without find_oracle.py: the accessors'
conversions below are restated from Go's definitions with Python integers and fractions.

Geometry is read from the headers, so a change of tile, block or limit moves the tapes with it:
  T = TAPE_THREADS * TAPE_ROUNDS words per tile of the word-parallel passes, G = GROUP_TILES tiles per group of the
  two-level tile scan, KC2_BLOCK roots per countWhere block, FD_THREADS cells per KF3 block, FD_SHORT the longest string
  KF5 copies per thread, and the find's path limits."""
import fractions
import math
import os
import re
import struct
from dataclasses import dataclass, field

import numpy as np

from tests.tape_builder import STRINGBUFBIT, TapeBuilder, word

_ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")


def _src(path):
    with open(os.path.join(_ROOT, path)) as f:
        return f.read()


def _match(path, pattern):
    return int(re.search(pattern, _src(path)).group(1))


TAPE_THREADS = _match("simdjson-go_b200/csrc/tape.cuh", r"constexpr int TAPE_THREADS = (\d+);")
TAPE_ROUNDS = _match("simdjson-go_b200/csrc/tape.cuh", r"constexpr int TAPE_ROUNDS = (\d+);")
FD_THREADS = _match("simdjson-go_b200/csrc/find.cuh", r"constexpr int FD_THREADS = (\d+);")
FD_SHORT = _match("simdjson-go_b200/csrc/find.cuh", r"constexpr uint64_t FD_SHORT = (\d+);")
KC2_BLOCK = _match("simdjson-go_b200/csrc/sj_consume.inl", r"tc_count_where_kernel<<<blocks, (\d+),")
assert KC2_BLOCK == _match("simdjson-go_b200/csrc/consume.cuh", r"__launch_bounds__\((\d+)\) tc_count_where_kernel")
GROUP_TILES = _match("simdjson-go_b200/csrc/sj_tape.inl", r"ngroups = \(ntiles \+ \d+\) / (\d+);")
FD_MAX_PATHS = _match("simdjson-go_b200/csrc/sj_find.inl", r"FD_MAX_PATHS = (\d+)")
FD_MAX_SEGS = _match("simdjson-go_b200/csrc/sj_find.inl", r"FD_MAX_SEGS = (\d+)")
FD_MAX_SEG_BYTES = _match("simdjson-go_b200/csrc/sj_find.inl", r"FD_MAX_SEG_BYTES = (\d+)")
T = TAPE_THREADS * TAPE_ROUNDS      # words per tile (KM1, KC1a, KC1b) and string cells per tile (KF4, KF5)
G = GROUP_TILES * T                 # words per group of tiles: one block of the first scan level

# cell statuses and path kinds (simdjson_b200.h)
_H = _src("include/simdjson_b200.h")
OK, NOT_FOUND, NOT_OBJECT, CONVERT, CORRUPT = (int(re.search(r"#define SJ_FIND_%s (\d+)" % s, _H).group(1))
                                               for s in ("OK", "NOT_FOUND", "NOT_OBJECT", "CONVERT", "CORRUPT"))
ELEMENT, INT64, UINT64, FLOAT64, BOOL, STRING = (int(re.search(r"#define SJ_FIND_KIND_%s (\d+)" % s, _H).group(1))
                                                 for s in ("ELEMENT", "INT64", "UINT64", "FLOAT64", "BOOL", "STRING"))
KINDS = (ELEMENT, INT64, UINT64, FLOAT64, BOOL, STRING)
M64 = (1 << 64) - 1
VAL = (1 << 56) - 1


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def bits_f64(b):
    return struct.unpack("<d", struct.pack("<Q", b & M64))[0]


# ---- the accessors, restated ---------------------------------------------------------------------------------------
def _trunc_amd64(x):
    """int64(x) as Go lowers it on amd64 (CVTTSD2SQ): the value truncated toward zero, and the 'integer indefinite'
    0x8000000000000000 for NaN and for everything outside [-2^63, 2^63)"""
    if x != x or x in (math.inf, -math.inf):
        return 1 << 63
    q = fractions.Fraction(x)
    t = q.numerator // q.denominator if q >= 0 else -((-q.numerator) // q.denominator)
    return t & M64 if -(1 << 63) <= t < (1 << 63) else 1 << 63


def convert(tag, payload, kind):
    """(status, value) of the accessor `kind` on an element with tag `tag` (a str) and, for numbers, the raw payload
    word, for strings the bytes.  Int / Uint / Float / Bool / StringBytes of parsed_json.go; the float-to-integer
    conversions are amd64's: a comparison with NaN is false, float64(MaxInt64) is 2^63, uint64(v) is
    v < 2^63 ? int64(v) : int64(v - 2^63) | 1 << 63."""
    if kind == ELEMENT:
        return OK, 0
    if kind == BOOL:
        return (OK, int(tag == "t")) if tag in "tf" and tag else (CONVERT, 0)
    if kind == STRING:
        return (OK, bytes(payload)) if tag == '"' else (CONVERT, b"")
    if tag not in ("l", "u", "d"):
        return CONVERT, 0
    p = int(payload) & M64
    signed = p - (1 << 64) if p >> 63 else p
    if kind == FLOAT64:
        if tag == "d":
            return OK, p
        return OK, f64_bits(float(signed if tag == "l" else p))   # int -> float64 rounds to nearest, ties to even
    d = bits_f64(p)
    if kind == INT64:
        if tag == "d":
            if d > 2.0 ** 63 or d < -2.0 ** 63:
                return CONVERT, 0
            return OK, _trunc_amd64(d)
        if tag == "u" and p >= 1 << 63:
            return CONVERT, 0
        return OK, p
    if tag == "d":  # UINT64
        if d > 2.0 ** 64 or d < 0:
            return CONVERT, 0
        if d < 2.0 ** 63:
            return OK, _trunc_amd64(d)
        return OK, _trunc_amd64(d - 2.0 ** 63) | (1 << 63)
    if tag == "l" and p >> 63:
        return CONVERT, 0
    return OK, p


@dataclass
class Cell:
    status: int
    tag: int = 0
    index: int = -1
    value: object = 0

    def astuple(self):
        return self.status, self.tag, self.index, self.value


def missing(kind):
    return Cell(NOT_FOUND, 0, -1, b"" if kind == STRING else 0)


def found(spec, head, kind):
    """the cell of a path whose element is `spec` (see put_value) with its head word at `head`"""
    tag = spec[0][0]
    st, v = convert(tag, spec[1] if tag in 'lud"' else 0, kind)
    return Cell(st, ord(tag), head, v)


def put_value(b, spec):
    """one value on TapeBuilder b: ("n",), ("t",), ("f",), (tag, payload) for l / u / d, ('"', bytes, copy), ("[", m)
    an array of m nulls, ("[d", payloads, pad) an array of `pad` nulls and then doubles, ("{",) the object {"a":true}"""
    tag = spec[0]
    if tag in ("l", "u", "d"):
        b.number(tag, spec[1])
    elif tag == '"':
        b.string(spec[1], copy=spec[2] if len(spec) > 2 else True)
    elif tag in ("[", "[d"):
        b.open("[")
        pad = spec[1] if tag == "[" else spec[2]
        if pad:
            b.atoms(("n", pad))
        if tag == "[d":
            b.numbers("d", spec[1])
        b.close()
    elif tag == "{":
        b.open("{")
        b.string(b"a")
        b.atom("t")
        b.close()
    else:
        b.atom(tag)


# ---- records on a tape ---------------------------------------------------------------------------------------------
@dataclass
class Feature:
    family: str
    edge: str            # edge kind ("T", "2T", ... "2G")
    E: int               # the edge: a word index
    offset: int          # the feature word is E + offset
    at: int              # = E + offset
    window: tuple        # [ws, we): whole records around it behind a head word ws
    detail: str = ""


@dataclass
class EdgeTape:
    name: str
    tape: np.ndarray
    strings: bytes
    message: bytes
    rows: np.ndarray                 # the slot of every root, in tape order
    cells: list                      # cells[p][r]: Cell of path p on row r
    features: list = field(default_factory=list)
    count_where: dict = field(default_factory=dict)   # (key, value) -> matches


class Records:
    """records `r { "k" <kval> ["v" <vval>] } r` (value specs as put_value) written with TapeBuilder; every record's
    slot, its values and its cell for each of `paths` are kept"""

    def __init__(self, paths):
        self.b = TapeBuilder()
        self.paths = paths
        self.rows = []
        self.cells = [[] for _ in paths]
        self.values = []     # {b"k": kval, b"v": vval} per row

    @property
    def n(self):
        return self.b.n

    @staticmethod
    def width(spec):
        tag = spec[0]
        return {"[": lambda: spec[1] + 2, "[d": lambda: 2 * len(spec[1]) + spec[2] + 2, "{": lambda: 5}.get(
            tag, lambda: 2 if tag in 'lud"' else 1)()

    def record(self, kval, vval=None):
        """one record at the current word; returns its slot"""
        s, b = self.n, self.b
        b.open("r")
        b.open("{")
        b.string(b"k")
        put_value(b, kval)
        heads = {b"k": s + 4}
        if vval is not None:
            b.string(b"v")
            heads[b"v"] = self.n
            put_value(b, vval)
        b.close(2)
        assert self.n - s == 6 + self.width(kval) + (0 if vval is None else 2 + self.width(vval))
        vals = {b"k": kval, b"v": vval}
        self.rows.append(s)
        self.values.append(vals)
        for p, (path, kind) in enumerate(self.paths):
            key = path[0] if len(path) == 1 else None
            self.cells[p].append(found(vals[key], heads[key], kind) if vals.get(key) is not None else missing(kind))
        return s

    def fill_to(self, at):
        """records up to word `at`: one holding an array of nulls, or one `"k":null` record for a gap of 7"""
        d = at - self.n
        assert d == 0 or d >= 7, (self.n, at)
        if d == 7:
            self.record(("n",))
        elif d:
            self.record(("[", d - 8))

    def matches(self, key, value):
        """countWhere(key, value) of the records: those whose `key` holds the string `value`"""
        return sum(1 for v in self.values if v.get(key) is not None and v[key][0] == '"' and v[key][1] == value)


# which cells every edge tape reports: the row check (ELEMENT of "k": its index is slot + 4) and the accessors on the
# feature values
EDGE_PATHS = [([b"k"], ELEMENT), ([b"k"], INT64), ([b"k"], UINT64), ([b"k"], FLOAT64), ([b"k"], BOOL), ([b"k"], STRING),
              ([b"v"], ELEMENT), ([b"v"], STRING), ([b"v"], INT64)]
EDGE_NEEDLES = [(b"v", b"x"), (b"k", b"rrrrr"), (b"k", b"")]
EDGE_KINDS = ("T", "2T", "1023T", "G", "G+T", "2G")
EDGES = dict(zip(EDGE_KINDS, (T, 2 * T, 1023 * T, G, G + T, 2 * G)))
SMALL_EDGES = ("T", "2T")
OFFSETS = (-2, -1, 0, 1)
FAMILIES = ("root_open", "root_close", "lookalike_num", "lookalike_str", "parity", "key_straddle", "value_straddle")

LOOK_R = 0x72FF_FFFF_FFFF_FFF0     # top byte 'r', value bits far past any slot: a root open if read as a head
RUN_D = 0x6400_0000_0000_0000      # top byte 'd': doubles near 2.5e173, whose value words carry a value tag too
X = ('"', b"x", True)


def _feature_records(rs, fam, F, i):
    """the records of family `fam` around the feature word F (i: the edge's number); returns (ws, detail)"""
    if fam == "root_open":          # a root opens at F
        rs.fill_to(F - 7)
        ws = rs.record(("n",))
        rs.record(("n",), X)
        rs.record(("l", 5))
        return ws, "open"
    if fam == "root_close":         # a root's closing 'r' at F, the next root opens at F + 1
        rs.fill_to(F - 6 - 8)
        ws = rs.record(("d", f64_bits(1.5)))
        rs.record(("n",))
        rs.record(("t",), X)
        return ws, "close"
    if fam == "lookalike_num":      # a number's head at F - 1, its value word at F starts with 'r' and points forward
        tag = "lud"[i % 3]
        rs.fill_to(F - 5 - 7)
        ws = rs.record(("n",))
        rs.record((tag, LOOK_R | i), X)
        rs.record(("f",), X)
        return ws, tag
    if fam == "lookalike_str":      # a string's head at F - 1, its length word at F
        rs.fill_to(F - 5 - 7)
        ws = rs.record(("n",))
        rs.record(('"', b"rrrrr", i % 2 == 0), X)
        rs.record(("n",))
        return ws, "string"
    if fam == "parity":             # a run of words that all carry a value tag ends with an 'r' value word at F
        s = rs.n
        pad = (F - s - 6) % 2       # the array opens at s + 4; nulls in front of its doubles fix the parity
        k = (F - s - 6 - pad) // 2 + 1
        run = RUN_D | np.arange(k, dtype=np.uint64)
        run[-1] = LOOK_R | i
        rs.record(("[d", run, pad))
        ws = F - 1 - 2 * min(k - 1, 64)   # the head of a double inside the run
        rs.record(("n",), X)
        rs.record(("u", 7))
        return ws, "run of %d" % k
    if fam == "key_straddle":       # the key "v" of a path: its head at F - 1, its length at F
        rs.fill_to(F - 6 - 7)
        ws = rs.record(("n",))
        rs.record(("n",), ("u", 1 << 63 | i) if i % 2 else X)
        rs.record(("n",), X)
        return ws, "key"
    if fam == "value_straddle":     # the value of "v": its head at F - 1, its payload (or length) at F
        v = [X, ("u", LOOK_R), ("d", f64_bits(-0.5)), ("l", (1 << 64) - 3)][i % 4]
        rs.fill_to(F - 8 - 7)
        ws = rs.record(("n",))
        rs.record(("n",), v)
        rs.record(("n",), X)
        return ws, "value " + v[0]
    raise ValueError(fam)


def edge_tape(fam, offset, edges=EDGE_KINDS):
    """one tape with the feature of family `fam` at E + offset for every edge E of `edges`"""
    rs = Records(EDGE_PATHS)
    feats = []
    for i, kind in enumerate(edges):
        E = EDGES[kind]
        ws, detail = _feature_records(rs, fam, E + offset, i)
        feats.append(Feature(fam, kind, E, offset, E + offset, (ws, rs.n), detail))
    rs.fill_to(rs.n + 40)
    rs.record(("n",), X)
    tape, strs, msg = rs.b.build()
    return EdgeTape("%s%+d/%s" % (fam, offset, "large" if len(edges) > 2 else "small"), tape, strs, msg,
                    np.array(rs.rows, dtype=np.int64), rs.cells, feats,
                    {(k, v): rs.matches(k, v) for k, v in EDGE_NEEDLES})


def edge_tapes(large):
    """every family at every offset: the small tapes carry the edges T and 2T (whole-tape checks on the CPU), the
    large ones all of EDGE_KINDS (a tape of 2G words and more)"""
    for fam in FAMILIES:
        for o in OFFSETS:
            yield edge_tape(fam, o, EDGE_KINDS if large else SMALL_EDGES)


def window(tape, ws, we):
    """tape[ws:we] as a tape of its own: the links of its heads ({ [ } ] r) moved down by ws, value words untouched.
    ws must be a head word.  The rows of the window, plus ws, are the tape's rows inside [ws, we)."""
    w = np.array(tape[ws:we], dtype=np.uint64)
    tags = (w >> np.uint64(56)).astype(np.int64)
    value = np.isin(tags, [ord(c) for c in '"lud'])
    head = np.ones(w.size, dtype=bool)
    h = True
    for i, v in enumerate(value.tolist()):
        head[i] = h
        h = not (h and v)
    link = head & np.isin(tags, [ord(c) for c in "{[}]r"])
    low = w & np.uint64(VAL)
    moved = np.where(low >= np.uint64(ws), low - np.uint64(ws), np.uint64(0))
    w[link] = (w[link] & ~np.uint64(VAL)) | moved[link]
    return w


# ---- the conversion table ------------------------------------------------------------------------------------------
def _next_up(x):
    return math.nextafter(x, math.inf)


def _next_down(x):
    return math.nextafter(x, -math.inf)


def conversion_values():
    """(tag, payload) of every element the conversion table holds"""
    ds = [0.0, -0.0, 5e-324, -5e-324, 0.5, -0.5, -1 + 2.0 ** -53, 2.0 ** 53 - 1, 2.0 ** 53, 2.0 ** 53 + 2, 1.5, -1.5, 1e300, -1e300]
    for e in (2.0 ** 63, -(2.0 ** 63), 2.0 ** 64):
        ds += [_next_down(e), e, _next_up(e)]
    out = [("d", f64_bits(x)) for x in ds]
    out += [("d", 0x7FF0000000000000), ("d", 0xFFF0000000000000),           # +-Inf
            ("d", 0x7FF8000000000000), ("d", 0x7FF0000000000001),           # quiet, signalling NaN
            ("d", 0xFFF8000000000000), ("d", 0xFFF0000000000001),           # negative NaNs
            ("d", LOOK_R)]
    ints = [2 ** 53 + k for k in (1, 2, 3)] + [2 ** 62 + 2 ** 9 + k for k in (-1, 0, 1)] + [2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1,
                                                                                             0, 1, LOOK_R]
    for tag in "lu":
        out += [(tag, x) for x in ints]
        out += [(tag, (-(2 ** 53 + k)) & M64) for k in (1, 2, 3)]
        out += [(tag, (-(2 ** 62 + 2 ** 9 + k)) & M64) for k in (-1, 0, 1)]
    return out


CONVERSION_OTHERS = [("t",), ("f",), ("n",), ('"', b"1", True), ('"', b"", False), ('"', b"-0.5", True), ("[", 0),
                     ("[", 2), ("{",)]


def conversion_tape():
    """one record `{"k": <element>}` per entry of the table and per other tag, read by every kind: (EdgeTape, the
    element of every row)"""
    rs = Records([([b"k"], k) for k in KINDS])
    specs = conversion_values() + CONVERSION_OTHERS
    for sp in specs:
        rs.record(sp)
    tape, strs, msg = rs.b.build()
    return EdgeTape("conversions", tape, strs, msg, np.array(rs.rows, dtype=np.int64), rs.cells), specs


# ---- countWhere messages -------------------------------------------------------------------------------------------
CW_COUNTS = (1, 31, 32, 33, KC2_BLOCK - 1, KC2_BLOCK, KC2_BLOCK + 1, T - 1, T, T + 1)
CW_LENS = (0, 1, 31, 32, 33, 70)
PATTERNS = {
    "none": lambda i: False,
    "all": lambda i: True,
    "lane0": lambda i: i % 32 == 0,
    "lane31": lambda i: i % 32 == 31,
    "alternate": lambda i: i % 2 == 0,
}


def _letters(n, base):
    return bytes(base + j % 26 for j in range(n))


def cw_needles(klen, vlen):
    return _letters(klen, 97), _letters(vlen, 65)


def cw_message(n, pattern, klen, vlen):
    """n NDJSON records; record i has `key` = `value` as its first member of that name exactly when pattern(i).  The
    others miss in one of five ways: another value, another key, a number, the key twice with the match second, the
    match one level down.  Returns (message, key, value, matching rows)."""
    key, value = cw_needles(klen, vlen)
    other = value[:-1] + bytes([value[-1] ^ 1]) if value else b"x"
    ks, vs, os_ = key.decode(), value.decode(), other.decode()
    lines, hits = [], []
    for i in range(n):
        if PATTERNS[pattern](i):
            hits.append(i)
            lines.append(['{"%s":"%s"}', '{"z%s":0,"%s":"%s","q":[1]}', '{"%s":"%s","%s":"%s"}'][i % 3]
                         % ((ks, vs), (ks, ks, vs), (ks, vs, ks, os_))[i % 3])
        else:
            lines.append(['{"%s":"%s"}' % (ks, os_), '{"%sq":"%s"}' % (ks, vs), '{"%s":1}' % ks,
                          '{"%s":"%s","%s":"%s"}' % (ks, os_, ks, vs), '{"o":{"%s":"%s"}}' % (ks, vs)][i % 5])
    return "\n".join(lines).encode(), key, value, hits


def cw_cases():
    """(n, pattern, klen, vlen): every count with every pattern, the key and value lengths turning through CW_LENS"""
    out = []
    for ni, n in enumerate(CW_COUNTS):
        for pi, pat in enumerate(PATTERNS):
            out.append((n, pat, CW_LENS[(ni + pi) % len(CW_LENS)], CW_LENS[(ni + 2 * pi + 1) % len(CW_LENS)]))
    for kl in CW_LENS:
        for vl in CW_LENS:
            out.append((33, "alternate", kl, vl))
    return out


def cw_group_message(pattern, n=1_100_000):
    """n records of `{}` and `{"a":"b"}` (the match, where pattern(i)): a tape of more than G words"""
    hit = np.array([PATTERNS[pattern](i) for i in range(64)], dtype=bool)[np.arange(n) % 64]
    parts = np.where(hit, '{"a":"b"}', "{}")
    return "\n".join(parts.tolist()).encode(), int(hit.sum()), int((np.where(hit, 8, 4)).sum())


# ---- KF3: 64 paths, 16 KiB of segment bytes ------------------------------------------------------------------------
KF3_ROWS = (1, 2, FD_THREADS - 1, FD_THREADS, FD_THREADS + 1, 2 * FD_THREADS - 1, 2 * FD_THREADS, 2 * FD_THREADS + 1)
KF3_TEMPLATES = 4


def kf3_paths():
    """FD_MAX_PATHS paths: one of no segment, one of FD_MAX_SEGS 8-byte segments, one of FD_MAX_SEGS 1-byte segments,
    and long keys of one length that differ in their last four bytes only; FD_MAX_SEG_BYTES segment bytes in all"""
    n_long = FD_MAX_PATHS - 3
    deep8 = [b"s%07d" % j for j in range(FD_MAX_SEGS)]
    deep1 = [b"a"] * FD_MAX_SEGS
    rest = FD_MAX_SEG_BYTES - 8 * FD_MAX_SEGS - FD_MAX_SEGS
    L = rest // n_long
    longs = [[b"K" * (L - 4) + b"%04d" % p] for p in range(n_long)]
    longs[-1] = [b"K" * (rest - L * (n_long - 1) - 4) + b"%04d" % (n_long - 1)]
    paths = longs[:20] + [deep8] + longs[20:40] + [[]] + longs[40:] + [deep1]
    kinds = [KINDS[p % len(KINDS)] for p in range(len(paths))]
    assert len(paths) == FD_MAX_PATHS and sum(len(s) for p in paths for s in p) == FD_MAX_SEG_BYTES
    return paths, kinds


def _kf3_value(p, t):
    return [("l", p * 1000 + t), ("d", f64_bits(p + t / 8)), ('"', b"v%d.%d" % (p, t), (p + t) % 2 == 0), ("t",),
            ("u", (1 << 63) + p), ("f",)][(p + t) % 6]


def kf3_tape(rows):
    """rows records of KF3_TEMPLATES kinds in turn: template t holds every long key but those of paths p with
    (p + t) % 5 == 0, the 8-byte chain to depth 32 - 3t, and the 1-byte chain to depth 32 (t even) or with a number at
    depth 16 (t odd).  Returns (tape, strings, message, slots)."""
    paths, _ = kf3_paths()
    b = TapeBuilder()
    slots = []
    for r in range(rows):
        t = r % KF3_TEMPLATES
        slots.append(b.n)
        b.open("r")
        b.open("{")
        for p, path in enumerate(paths):
            if len(path) == 1 and (p + t) % 5:
                b.string(path[0])
                put_value(b, _kf3_value(p, t))
            elif len(path) == FD_MAX_SEGS and path[0] == b"s0000000":
                depth = FD_MAX_SEGS - 3 * t
                for s in path[:depth]:
                    b.string(s)
                    b.open("{")
                b.string(b"end")
                b.number("l", t)
                b.close(depth)
            elif len(path) == FD_MAX_SEGS:
                depth = FD_MAX_SEGS if t % 2 == 0 else 16
                for s in path[:depth - 1]:
                    b.string(s)
                    b.open("{")
                b.string(path[depth - 1])
                b.number("l", 100 + t)
                b.close(depth - 1)
        b.close(2)
    tape, strs, msg = b.build()
    return tape, strs, msg, np.array(slots, dtype=np.int64)


# ---- KF5: string columns -------------------------------------------------------------------------------------------
KF5_LENS = (0, 1, FD_SHORT - 1, FD_SHORT, FD_SHORT + 1, 2 * FD_SHORT, 4095)


def kf5_mixed(rows=1000):
    """records {"s": S, "t": S2} whose string lengths run through KF5_LENS (7 against a warp of 32, so every warp mixes
    them), S in Strings.B and S2 in the message on alternate rows.  Returns (tape, strings, message, paths, kinds,
    expected STRING columns: one list of bytes per STRING path)."""
    b = TapeBuilder()
    cols = {b"s": [], b"t": []}
    for r in range(rows):
        b.open("r")
        b.open("{")
        for key, ln, copy in ((b"s", KF5_LENS[r % 7], True), (b"t", KF5_LENS[(3 * r + 1) % 7], r % 2 == 0)):
            s = bytes((r * 7 + key[0] + j) % 251 + 1 for j in range(ln))
            b.string(key)
            b.string(s, copy=copy)
            cols[key].append(s)
        b.close(2)
    tape, strs, msg = b.build()
    paths = [[b"s"], [b"t"], [b"s"], [b"x"], [b"t"]]
    kinds = [STRING, STRING, ELEMENT, STRING, INT64]
    want = [cols[b"s"], cols[b"t"], [b""] * rows]
    return tape, strs, msg, paths, kinds, want


KF5_GROUP_KEYS = (b"a", b"b", b"c", b"d")


def kf5_group(rows=G // FD_MAX_PATHS + 1):
    """FD_MAX_PATHS STRING paths over `rows` records of four string members: rows * FD_MAX_PATHS string cells, one
    group of tiles and more.  Built with numpy.  The value of key k on row r is pool[off:off + ln] in Strings.B with
    off = (13 r + 101 k) % 4000, ln = (r + k) % 4.  Returns (tape, strings, paths, slots, offs, lens) with offs / lens
    [4, rows]."""
    nk = len(KF5_GROUP_KEYS)
    pool = (np.arange(4096) % 251 + 1).astype(np.uint8).tobytes()
    strings = pool + b"".join(KF5_GROUP_KEYS)
    koff = [len(pool) + i for i in range(nk)]
    r = np.arange(rows, dtype=np.uint64)
    per = 2 + 4 * nk + 2
    w = np.empty((rows, per), dtype=np.uint64)
    slot = r * np.uint64(per)
    w[:, 0] = np.uint64(word("r")) | (slot + np.uint64(per))
    w[:, 1] = np.uint64(word("{")) | (slot + np.uint64(per - 1))
    offs = np.empty((nk, rows), dtype=np.uint64)
    lens = np.empty((nk, rows), dtype=np.uint64)
    for k in range(nk):
        offs[k] = (r * np.uint64(13) + np.uint64(101 * k)) % np.uint64(4000)
        lens[k] = (r + np.uint64(k)) % np.uint64(4)
        c = 2 + 4 * k
        w[:, c] = np.uint64(word('"', STRINGBUFBIT | koff[k]))
        w[:, c + 1] = 1
        w[:, c + 2] = np.uint64(word('"', STRINGBUFBIT)) | offs[k]
        w[:, c + 3] = lens[k]
    w[:, per - 2] = np.uint64(word("}")) | (slot + np.uint64(1))
    w[:, per - 1] = np.uint64(word("r")) | slot
    paths = [[KF5_GROUP_KEYS[p % nk]] for p in range(FD_MAX_PATHS)]
    return w.reshape(-1), strings, paths, slot.astype(np.int64), offs, lens


def gather(pool, offs, lens):
    """the bytes pool[offs[i]:offs[i] + lens[i]] for every i, joined"""
    offs = np.asarray(offs, dtype=np.int64).reshape(-1)
    lens = np.asarray(lens, dtype=np.int64).reshape(-1)
    start = np.repeat(offs - (np.cumsum(lens) - lens), lens)
    idx = start + np.arange(int(lens.sum()))
    return np.frombuffer(pool, dtype=np.uint8)[idx].tobytes()


# ---- record boundaries at stage 2's edges --------------------------------------------------------------------------
def boundary_messages():
    """NDJSON messages whose first record ends (its newline, or a run of blank lines) at byte E - 2 .. E + 1 of the
    streaming stage 2's step, slab and tile (read from stage 1's headers), plus blank lines at the start and the end,
    and a single document.  Yields (name, message, ndjson)."""
    from tests.stage1_verdict_docs import SLAB, STEP, TILE
    tail = b'\n{"z":[1],"k":"a"}\n[2]\n{"k":3}'
    for ename, E in (("step", STEP), ("slab", SLAB), ("2slab", 2 * SLAB), ("tile", TILE), ("tile+slab", TILE + SLAB),
                     ("2tile", 2 * TILE)):
        for o in OFFSETS:
            for sep in (b"\n", b"\n\n", b"\n \n\t\n"):
                head = b'{"k":"'
                pad = E + o - len(head) - 2
                msg = head + b"p" * pad + b'"}' + sep + tail
                assert msg[E + o:E + o + 1] == b"\n"
                yield "%s%+d/%d" % (ename, o, len(sep)), msg, True
    yield "blank_ends", b"\n\n" + b'{"k":"a"}\n\n\n{"k":"b"}\n' + b"\n" * 5, True
    yield "single", b' {"k":"a","z":[1,{"k":2}]} ', False
    yield "single_nd", b'{"k":"a"}', True
