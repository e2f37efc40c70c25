#!/usr/bin/env python3
"""Extract the reference's golden vectors into JSON fixtures.

Run it where a checkout of minio/simdjson-go is at hand; the tests only read its output:

    python tests/golden/make_golden.py <path of the simdjson-go checkout>

It parses the table-driven test literals out of the reference's Go test files
with a small Go-literal evaluator (raw/interpreted strings, rune and integer
literals, composite literals with positional or keyed fields, a handful of
conversions) and writes tests/golden/*.json. Byte strings are stored as hex so
that control characters and invalid UTF-8 survive. It also copies the
reference's compressed data fixtures (testdata/*.zst: public JSON corpora, data
not source) to tests/golden/data/, so the tests need nothing outside this repository.

Golden-vector ids (G1..G20) follow SURVEY.md appendix D.
"""
import json
import os
import re
import shutil
import sys

REF = sys.argv[1] if __name__ == "__main__" and len(sys.argv) > 1 else "simdjson-go"
OUT = os.path.dirname(os.path.abspath(__file__))


# --------------------------------------------------------------------------
# Go tokenizer
# --------------------------------------------------------------------------
class Tok:
    def __init__(self, kind, val, pos):
        self.kind, self.val, self.pos = kind, val, pos

    def __repr__(self):
        return "Tok(%s,%r)" % (self.kind, self.val)


_SIMPLE_ESC = {"n": 10, "t": 9, "r": 13, "\\": 92, '"': 34, "'": 39, "a": 7, "b": 8, "f": 12, "v": 11}


def _unescape(body):
    """Interpreted Go string/rune body -> bytes."""
    out = bytearray()
    i = 0
    while i < len(body):
        c = body[i]
        if c != "\\":
            out += c.encode("utf-8")
            i += 1
            continue
        e = body[i + 1]
        if e in _SIMPLE_ESC:
            out.append(_SIMPLE_ESC[e])
            i += 2
        elif e == "x":
            out.append(int(body[i + 2:i + 4], 16))
            i += 4
        elif e == "u":
            out += chr(int(body[i + 2:i + 6], 16)).encode("utf-8", "surrogatepass")
            i += 6
        elif e == "U":
            out += chr(int(body[i + 2:i + 10], 16)).encode("utf-8")
            i += 10
        elif e in "01234567":
            out.append(int(body[i + 1:i + 4], 8))
            i += 4
        else:
            raise ValueError("bad escape \\" + e)
    return bytes(out)


def tokenize(src, start=0, end=None):
    toks = []
    i = start
    n = len(src) if end is None else end
    while i < n:
        c = src[i]
        if c in " \t\r\n":
            i += 1
        elif src.startswith("//", i):
            j = src.find("\n", i)
            i = n if j < 0 else j
        elif src.startswith("/*", i):
            i = src.index("*/", i) + 2
        elif c == "`":
            j = src.index("`", i + 1)
            toks.append(Tok("str", src[i + 1:j].replace("\r", "").encode("utf-8"), i))
            i = j + 1
        elif c == '"':
            j = i + 1
            while src[j] != '"':
                j += 2 if src[j] == "\\" else 1
            toks.append(Tok("str", _unescape(src[i + 1:j]), i))
            i = j + 1
        elif c == "'":
            j = i + 1
            while src[j] != "'":
                j += 2 if src[j] == "\\" else 1
            b = _unescape(src[i + 1:j])
            toks.append(Tok("num", ord(b.decode("utf-8")), i))
            i = j + 1
        elif c.isdigit() or (c == "." and src[i + 1].isdigit()):
            m = re.compile(r"0[xX][0-9a-fA-F_]+|0[bB][01_]+|[0-9][0-9_]*(\.[0-9]*)?([eE][+-]?[0-9]+)?|\.[0-9]+([eE][+-]?[0-9]+)?").match(src, i)
            t = m.group(0).replace("_", "")
            if t[:2].lower() == "0x":
                v = int(t, 16)
            elif t[:2].lower() == "0b":
                v = int(t[2:], 2)
            elif re.fullmatch(r"[0-9]+", t):
                v = int(t, 10)  # (no octal literals occur in the tables)
            else:
                v = float(t)
            toks.append(Tok("num", v, i))
            i = m.end()
        elif c.isalpha() or c == "_":
            m = re.compile(r"[A-Za-z_][A-Za-z0-9_]*").match(src, i)
            toks.append(Tok("id", m.group(0), i))
            i = m.end()
        else:
            for op in ("<<", ">>", "&^", "{", "}", "(", ")", "[", "]", ",", ":", "+", "-", "*", "/", "^", "|", "&", ".", "=", ";", "!", "<", ">", "%"):
                if src.startswith(op, i):
                    toks.append(Tok("op", op, i))
                    i += len(op)
                    break
            else:
                raise ValueError("unexpected char %r at %d" % (c, i))
    return toks


# --------------------------------------------------------------------------
# Go literal-expression evaluator
# --------------------------------------------------------------------------
class Err:
    """Stands for a Go error value in a table (only nil / non-nil matters)."""

    def __init__(self, name):
        self.name = name


class Parser:
    def __init__(self, toks, env):
        self.t, self.i, self.env = toks, 0, env

    def peek(self, k=0):
        return self.t[self.i + k] if self.i + k < len(self.t) else Tok("eof", None, -1)

    def next(self):
        tok = self.peek()
        self.i += 1
        return tok

    def accept(self, kind, val=None):
        tok = self.peek()
        if tok.kind == kind and (val is None or tok.val == val):
            self.i += 1
            return True
        return False

    def expect(self, kind, val=None):
        tok = self.next()
        if tok.kind != kind or (val is not None and tok.val != val):
            raise ValueError("expected %s %r, got %r at %d" % (kind, val, tok, tok.pos))
        return tok

    # -- types ----------------------------------------------------------------
    def skip_type(self):
        """Skip a Go type expression: []T, [N]T, struct{...}, *T, pkg.T, T."""
        if self.accept("op", "["):
            while not self.accept("op", "]"):
                self.next()
            return self.skip_type()
        if self.accept("op", "*"):
            return self.skip_type()
        tok = self.expect("id")
        if tok.val == "struct":
            self.expect("op", "{")
            depth = 1
            while depth:
                t = self.next()
                if t.kind == "op" and t.val == "{":
                    depth += 1
                elif t.kind == "op" and t.val == "}":
                    depth -= 1
            return
        if tok.val == "func":
            raise ValueError("func types unsupported")
        while self.accept("op", "."):
            self.expect("id")

    # -- expressions ----------------------------------------------------------
    PREC = {"|": 1, "^": 1, "+": 1, "-": 1, "*": 2, "/": 2, "<<": 2, ">>": 2, "&": 2, "&^": 2, "%": 2}

    def expr(self, minprec=1):
        lhs = self.unary()
        while True:
            tok = self.peek()
            if tok.kind != "op" or tok.val not in self.PREC or self.PREC[tok.val] < minprec:
                return lhs
            self.next()
            rhs = self.expr(self.PREC[tok.val] + 1)
            lhs = self.binop(tok.val, lhs, rhs)

    @staticmethod
    def binop(op, a, b):
        if op == "+":
            return a + b
        if op == "-":
            return a - b
        if op == "*":
            return a * b
        if op == "/":
            return a // b if isinstance(a, int) and isinstance(b, int) else a / b
        if op == "<<":
            return a << b
        if op == ">>":
            return a >> b
        if op == "|":
            return a | b
        if op == "&":
            return a & b
        if op == "^":
            return a ^ b
        if op == "%":
            return a % b
        raise ValueError(op)

    def unary(self):
        if self.accept("op", "-"):
            return -self.unary()
        if self.accept("op", "+"):
            return self.unary()
        if self.accept("op", "^"):
            return ~self.unary() & ((1 << 64) - 1)  # every ^x in the tables is a uint64
        if self.accept("op", "&"):
            return self.unary()
        return self.primary()

    def composite(self):
        """'{' elem, ... '}' -> list (positional) or dict (keyed)."""
        self.expect("op", "{")
        items, keyed = [], {}
        while not self.accept("op", "}"):
            if self.peek().kind == "op" and self.peek().val == "{":
                v = self.composite()
                items.append(v)
            elif self.peek().kind == "id" and self.peek(1).kind == "op" and self.peek(1).val == ":":
                k = self.next().val
                self.next()
                keyed[k] = self.composite() if (self.peek().kind == "op" and self.peek().val == "{") else self.expr()
            else:
                items.append(self.expr())
            self.accept("op", ",")
        if keyed and items:
            raise ValueError("mixed keyed/positional literal")
        return keyed if keyed else items

    def args(self):
        self.expect("op", "(")
        out = []
        while not self.accept("op", ")"):
            out.append(self.expr())
            self.accept("op", ",")
        return out

    def primary(self):
        tok = self.peek()
        if tok.kind in ("str", "num"):
            self.next()
            return tok.val
        if tok.kind == "op" and tok.val == "(":
            self.next()
            v = self.expr()
            self.expect("op", ")")
            return v
        if tok.kind == "op" and tok.val == "[":
            # []T{...} composite or []byte(expr) conversion
            self.skip_type()
            if self.peek().kind == "op" and self.peek().val == "{":
                v = self.composite()
                return v
            a = self.args()
            return self.conv_bytes(a[0])
        if tok.kind == "id":
            name = self.next().val
            while self.accept("op", "."):
                name += "." + self.expect("id").val
            if self.peek().kind == "op" and self.peek().val == "(":
                a = self.args()
                return self.call(name, a)
            if self.peek().kind == "op" and self.peek().val == "{" and name in self.env.get("__types__", ()):
                return self.composite()
            if name == "struct":
                self.i -= 1
                self.skip_type()
                return self.composite()
            if name in ("true", "false"):
                return name == "true"
            if name == "nil":
                return None
            if name in self.env:
                return self.env[name]
            if name.startswith("strconv.Err"):
                return Err(name)
            raise ValueError("unknown identifier %s at %d" % (name, tok.pos))
        raise ValueError("unexpected token %r" % tok)

    @staticmethod
    def conv_bytes(v):
        if isinstance(v, bytes):
            return v
        if isinstance(v, list):
            return bytes(v)
        raise ValueError("cannot convert %r to []byte" % (v,))

    def call(self, name, a):
        if name in ("uint64", "uint32", "uint8", "byte", "uint", "uint16"):
            bits = {"uint64": 64, "uint32": 32, "uint8": 8, "byte": 8, "uint": 64, "uint16": 16}[name]
            v = a[0]
            if isinstance(v, tuple) and v[0] == "not":
                v = ~v[1]
            return v & ((1 << bits) - 1)
        if name in ("int64", "int", "int32"):
            return a[0]
        if name == "float64":
            return float(a[0])
        if name == "string":
            if isinstance(a[0], int):  # string(byte(x)) / string(rune): UTF-8 of the code point
                return chr(a[0]).encode("utf-8")
            return self.conv_bytes(a[0])
        if name == "strings.Repeat":
            return a[0] * a[1]
        if name == "errors.New":
            return Err("errors.New")
        if name.endswith(".Flags"):
            return a and a[0] or self.env.get(name[:-6], 0)
        raise ValueError("unknown call %s" % name)


def find_literal(src, anchor, env, which=0):
    """Evaluate the composite literal that follows the `which`-th occurrence of
    `anchor` (a regex matching up to just before the type expression)."""
    ms = list(re.finditer(anchor, src))
    m = ms[which]
    toks = tokenize(src, m.end())
    p = Parser(toks, env)
    p.skip_type()
    return p.composite()


def hx(b):
    return b.hex()


def read(name):
    with open(os.path.join(REF, name), encoding="utf-8") as f:
        return f.read()


def main():
    env = {"__types__": ()}
    pj_test = read("parsed_json_test.go")
    nd_test = read("ndjson_test.go")
    m = re.search(r"const demo_json = ", pj_test)
    demo_json = Parser(tokenize(pj_test, m.end(), m.end() + 2000), env).expr()
    m = re.search(r"const demo_ndjson = ", nd_test)
    demo_ndjson = Parser(tokenize(nd_test, m.end(), m.end() + 2000), env).expr()
    env["demo_json"], env["demo_ndjson"] = demo_json, demo_ndjson
    env["nul"] = 0

    G = {}
    sub = read("find_subroutines_amd64_test.go")

    # G1 finalize_structurals
    rows = find_literal(sub, r"func TestFinalizeStructurals[\s\S]*?testCases := ", env)
    G["G1_finalize_structurals"] = [dict(zip(("structurals", "whitespace", "quote_mask", "quote_bits", "expected_strls", "expected_pseudo"), r)) for r in rows]

    # G2 newline delimiters
    want = find_literal(sub, r"func testFindNewlineDelimiters[\s\S]*?want := ", env)
    G["G2_newline_delimiters"] = {"input": hx(demo_ndjson), "want": want,
                                   "quoted_case": {"input": hx(b'  "-------------------------------------"                       '),
                                                   "newline_at": [10, 50], "want": 1 << 50}}

    # G3 odd backslash sequences
    rows = find_literal(sub, r"func testFindOddBackslashSequences[\s\S]*?testCases := ", env)
    G["G3_odd_backslash"] = [dict(prev_ends_odd=r[0], input=hx(r[1]), expected=r[2], ends_odd_backslash=r[3]) for r in rows]

    # G4 quote mask and bits
    rows = find_literal(sub, r"func testFindQuoteMaskAndBits[\s\S]*?testCases := ", env)
    rows2 = find_literal(sub, r"testCasesPIIQ := ", env)
    G["G4_quote_mask"] = {
        "cases": [dict(odd_ends=r[0], input=hx(r[1]), expected=r[2], quote_bits=r[3], piiq=r[4], error_mask=r[5]) for r in rows],
        "piiq_cases": [dict(piiq_in=r[0], input=hx(r[1]), piiq_out=r[2]) for r in rows2],
    }

    # G5 whitespace and structurals
    rows = find_literal(sub, r"func testFindWhitespaceAndStructurals[\s\S]*?testCases := ", env)
    G["G5_whitespace_structurals"] = [dict(input=hx(r[0]), ws=r[1], structurals=r[2]) for r in rows]

    # G6 fused == composed inputs
    rows = find_literal(sub, r"func testFindStructuralBits\(t[\s\S]*?testCases := ", env)
    G["G6_fused_inputs"] = [hx(r[0]) for r in rows]

    # G7 tail padding (procedural in the reference; record the parameters)
    G["G7_tail_padding"] = {"msg": hx(b":" * 64)}

    # G8 twitter loop
    m = re.search(r'expectedStructuralsReversed = `([^`]*)`\s*const expectedLength = (\d+)', sub)
    G["G8_twitter_loop"] = {"reversed_tail": m.group(1), "count": int(m.group(2))}

    # G9 flatten_bits_incremental
    rows = find_literal(sub, r"func TestFlattenBitsIncremental[\s\S]*?testCases := ", env)
    G["G9_flatten_bits"] = [dict(masks=r[0], expected=r[1]) for r in rows]

    # G10 stage-1 marks of demo_json + structural positions
    s1 = read("stage1_find_marks_amd64_test.go")
    rows = find_literal(s1, r"func TestStage1FindMarks[\s\S]*?testCases := ", env)
    parsed = find_literal(s1, r"func TestFindStructuralIndices[\s\S]*?parsed := ", env)
    positions = [len(p) - len(p.lstrip(b" ")) for p in parsed]
    G["G10_stage1_marks"] = {
        "demo_json": hx(demo_json),
        "masks_msb_first_reversed": dict(zip(("quoted", "structurals", "whitespace", "structurals_finalized"), [r.decode() for r in rows[0]])),
        "positions": positions,
    }

    # G11 stage-2 tapes
    s2 = read("stage2_build_tape_amd64_test.go")
    env2 = dict(env)
    for mm in re.finditer(r"var (floatHexRepresentation\d) uint64 = (0x[0-9a-f]+)", s2):
        env2[mm.group(1)] = int(mm.group(2), 16)
    rows = find_literal(s2, r"func TestStage2BuildTape[\s\S]*?testCases := ", env2)
    G["G11_tapes"] = [dict(input=hx(r[0]), tape=[(c << 56) | v for c, v in r[1]]) for r in rows]

    # G12 demo_ndjson tape
    rows = find_literal(nd_test, r"func verifyDemoNdjson[\s\S]*?testCases := ", env)
    G["G12_ndjson_tape"] = {"input": hx(demo_ndjson), "tape": [(c << 56) | v for c, v in rows[0][0]]}

    # G13 atoms
    atoms = {}
    for name in ("True", "False", "Null"):
        rows = find_literal(s2, r"func TestIsValid%sAtom[\s\S]*?testCases := " % name, env)
        atoms[name.lower()] = [dict(input=hx(r[0]), expected=r[1]) for r in rows]
    G["G13_atoms"] = atoms

    # G14 strings
    ps = read("parse_string_test.go")
    rows = find_literal(ps, r"var tests = ", env)
    G["G14_strings"] = [dict(name=r["name"].decode(), str=hx(r["str"]), success=r.get("success", False),
                             want=hx(Parser.conv_bytes(r["want"])) if r.get("want") is not None else None) for r in rows]

    # G15 numbers
    pjt = read("parse_json_amd64_test.go")
    envn = dict(env)
    envn.update({"TagInteger": "l", "TagUint": "u", "TagFloat": "d", "TagEnd": "", "FloatOverflowedInteger": 1,
                 "__types__": ()})
    rows = find_literal(pjt, r"func TestParseNumber[\s\S]*?testCases := ", envn)
    num = {"parse_number": [dict(input=r["input"].decode(), tag=r["wantTag"], d=repr(float(r.get("expectedD", 0.0))),
                                 i=r.get("expectedI", 0), u=r.get("expectedU", 0), flags=r.get("flags", 0)) for r in rows]}
    rows = find_literal(pjt, r"var parseInt64Tests = ", envn)
    num["parse_int64"] = [dict(input=r[0].decode(), out=r[1], tag=r[2]) for r in rows]
    rows = find_literal(pjt, r"var atoftests = ", envn)
    num["atof"] = [dict(input=r[0].decode(), out=r[1].decode(), err=r[2] is not None) for r in rows]
    pn = read("parse_number_test.go")
    rows = find_literal(pn, r"func TestNumberIsValid[\s\S]*?validTests := ", envn)
    num["valid"] = [r.decode() for r in rows]
    rows = find_literal(pn, r"invalidTests := ", envn)
    num["invalid"] = [r.decode() for r in rows]
    G["G15_numbers"] = num

    # G16/G17 documents
    sj = read("simdjson_amd64_test.go")
    docs = {}
    for key, anchor in (("parse_nd", r"func TestParseND[\s\S]*?tests := "),
                        ("fail_cases", r"func TestParseFailCases[\s\S]*?tests := "),
                        ("pass_cases", r"func TestParsePassCases[\s\S]*?tests := ")):
        rows = find_literal(sj, anchor, env)
        docs[key] = [dict(name=r["name"].decode(), js=hx(r["js"]), want=hx(r["want"]) if r.get("want") is not None else None,
                          want_err=bool(r.get("wantErr", False))) for r in rows]
    rows = find_literal(pjt, r"ndjson_emptylines := ", env)
    docs["ndjson_emptylines"] = [hx(r) for r in rows]
    G["G16_G17_documents"] = docs

    # G18/G19 fixture-level facts
    rows = find_literal(pj_test, r"var testCases = ", env)
    G["G18_G19_fixtures"] = {"parking_citations": {"roots": 1000, "make_hond": 116},
                             "verify_tape_files": [r["name"].decode() for r in rows]}

    for k, v in G.items():
        with open(os.path.join(OUT, k + ".json"), "w") as f:
            json.dump(v, f, indent=1)
        print("wrote", k, "(%d entries)" % (len(v) if hasattr(v, "__len__") else 1))

    # data fixtures
    os.makedirs(os.path.join(OUT, "data"), exist_ok=True)
    for fn in sorted(os.listdir(os.path.join(REF, "testdata"))):
        if fn.endswith(".zst"):
            shutil.copyfile(os.path.join(REF, "testdata", fn), os.path.join(OUT, "data", fn))
    for fn in ("corpus.tar.zst", "go-corpus.tar.zst"):
        shutil.copyfile(os.path.join(REF, "testdata", "fuzz", fn), os.path.join(OUT, "data", "fuzz-" + fn))
    shutil.copyfile(os.path.join(REF, "examples", "parking-citations.json"), os.path.join(OUT, "data", "examples-parking-citations.json"))
    print("copied data fixtures")


if __name__ == "__main__":
    sys.exit(main())
