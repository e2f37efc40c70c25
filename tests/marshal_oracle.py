"""Iter.MarshalJSON (parsed_json.go:394-556) restated as a plain sequential walk of a tape.  Test infrastructure: the
expected output of the device marshal (marshal.cuh) and of its formatter (fmt.h).

Roots are joined by one newline; members are "key":value separated by commas; strings are escaped like escapeBytes
(parsed_json.go:1171-1238); floats are laid out like appendFloat (parsed_json.go:1250-1272) from the shortest
round-trip digits, which Python's repr gives."""
import math
import struct

TAG = 56
VAL = (1 << 56) - 1
STRINGBUFBIT = 1 << 55


class MalformedTape(ValueError):
    pass


def escape(b):
    out = bytearray()
    for c in bytes(b):
        if c == 0x22:
            out += b'\\"'
        elif c == 0x5C:
            out += b"\\\\"
        elif c < 0x20:
            out += {8: b"\\b", 12: b"\\f", 10: b"\\n", 13: b"\\r", 9: b"\\t"}.get(c, b"\\u00%02x" % c)
        else:
            out.append(c)
    return bytes(out)


def format_float(x):
    """appendFloat: fixed notation for 1e-6 <= |x| < 1e21 and 0, else d[.ddd]e(+|-)N with no leading exponent zeros."""
    if math.isnan(x) or math.isinf(x):
        raise MalformedTape("INF or NaN number found")
    sign = "-" if math.copysign(1.0, x) < 0 else ""
    ax = abs(x)
    if ax == 0:
        return (sign + "0").encode()
    r = repr(ax)
    mant, _, exp = r.partition("e")
    ip, _, fp = mant.partition(".")
    digits = (ip + fp).lstrip("0")
    point = len(digits) + int(exp or 0) - len(fp)  # value = 0.digits * 10^point
    digits = digits.rstrip("0")
    if 1e-6 <= ax < 1e21:
        if point <= 0:
            s = "0." + "0" * (-point) + digits
        elif point < len(digits):
            s = digits[:point] + "." + digits[point:]
        else:
            s = digits + "0" * (point - len(digits))
    else:
        s = digits[0] + ("." + digits[1:] if len(digits) > 1 else "") + "e%+d" % (point - 1)
    return (sign + s).encode()


def _string(tape, i, strings, message):
    w = int(tape[i]) & VAL
    if i + 1 >= len(tape):
        raise MalformedTape("string without length word at %d" % i)
    n = int(tape[i + 1])
    buf, off = (strings, w - STRINGBUFBIT) if w & STRINGBUFBIT else (message, w)
    if off + n > len(buf):
        raise MalformedTape("string range outside its buffer at %d" % i)
    return bytes(buf[off:off + n])


def marshal(tape, strings=b"", message=b""):
    """The whole tape as compact JSON text, one line per root."""
    out = bytearray()
    n = len(tape)
    stack = []  # [kind, direct children so far, open index]
    i = 0
    while i < n:
        w = int(tape[i])
        t, v = chr(w >> TAG), w & VAL
        top = stack[-1] if stack else None
        if t in "}]" or (t == "r" and v <= i):
            want = {"}": "{", "]": "[", "r": "r"}[t]
            if top is None or top[0] != want or v != top[2] or (int(tape[top[2]]) & VAL) != i + 1:
                raise MalformedTape("close %r at %d does not match its open" % (t, i))
            if t == "}" and top[1] % 2:
                raise MalformedTape("object closed after a key at %d" % i)
            stack.pop()
            if t == "r":
                if i + 1 < n:
                    out += b"\n"
            else:
                out += t.encode()
            i += 1
            continue
        if t == "r":
            if stack:
                raise MalformedTape("root inside a value at %d" % i)
            stack.append(["r", 0, i])
            i += 1
            continue
        if top is None:
            raise MalformedTape("value outside a root at %d" % i)
        if top[0] in "{[":
            if top[1]:
                out += b":" if top[0] == "{" and top[1] % 2 else b","
            if top[0] == "{" and top[1] % 2 == 0 and t != '"':
                raise MalformedTape("object key at %d is not a string" % i)
        top[1] += 1
        if t == '"':
            out += b'"' + escape(_string(tape, i, strings, message)) + b'"'
            i += 2
        elif t in "lud":
            if i + 1 >= n:
                raise MalformedTape("number without value word at %d" % i)
            p = int(tape[i + 1])
            if t == "l":
                out += b"%d" % (p - (1 << 64) if p >> 63 else p)
            elif t == "u":
                out += b"%d" % p
            else:
                out += format_float(struct.unpack("<d", struct.pack("<Q", p))[0])
            i += 2
        elif t in "tfn":
            out += {"t": b"true", "f": b"false", "n": b"null"}[t]
            i += 1
        elif t in "{[":
            out += t.encode()
            stack.append([t, 0, i])
            i += 1
        else:
            raise MalformedTape("unknown tag %r at %d" % (t, i))
    if stack:
        raise MalformedTape("containers left open at the end of the tape")
    return bytes(out)
