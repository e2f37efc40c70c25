"""Minimal tape reader (the reference's Iter, parsed_json.go:95-1040, is a pure host-side
consumer of the {Message, Tape, Strings} triple and is out of scope for the GPU path; this
small mirror exists so callers and tests can read values off a tape produced on the device).
"""
import struct

TAG = 56
VAL = (1 << 56) - 1
STRINGBUFBIT = 1 << 55


class Iter:
    def __init__(self, pj):
        self.pj = pj
        self.tape = pj.Tape
        self.off = 0

    def _string(self, i):
        w = int(self.tape[i]) & VAL
        ln = int(self.tape[i + 1])
        if w & STRINGBUFBIT:  # parsed_json.go:107-120
            o = w - STRINGBUFBIT
            return self.pj.Strings[o:o + ln]
        return self.pj.Message[w:w + ln]

    def _value(self, i):
        w = int(self.tape[i])
        t = chr(w >> TAG)
        if t == '"':
            return self._string(i).decode("utf-8", "surrogatepass"), i + 2
        if t == "l":
            return struct.unpack("<q", struct.pack("<Q", int(self.tape[i + 1])))[0], i + 2
        if t == "u":
            return int(self.tape[i + 1]), i + 2
        if t == "d":
            return struct.unpack("<d", struct.pack("<Q", int(self.tape[i + 1])))[0], i + 2
        if t in "tfn":
            return {"t": True, "f": False, "n": None}[t], i + 1
        if t == "[":
            out, j = [], i + 1
            end = (w & VAL) - 1
            while j < end:
                v, j = self._value(j)
                out.append(v)
            return out, end + 1
        if t == "{":
            out, j = {}, i + 1
            end = (w & VAL) - 1
            while j < end:
                k, j = self._value(j)
                v, j = self._value(j)
                out[k] = v
            return out, end + 1
        raise ValueError("unexpected tape tag %r at %d" % (t, i))

    def roots(self):
        """Yield the value under every root (one per NDJSON record)."""
        i = 0
        n = len(self.tape)
        while i < n:
            w = int(self.tape[i])
            assert chr(w >> TAG) == "r"
            v, j = self._value(i + 1)
            yield v
            i = (w & VAL)

    def Interface(self):
        """Iter.Interface(): the first root as Python objects."""
        for v in self.roots():
            return v
        return None

    def MarshalJSON(self, ctx=None):
        """Iter.MarshalJSON of a fresh Iter (parsed_json.go:394): the whole tape as compact JSON, one line per root.
        The triple is uploaded and marshalled on the device (marshal.cuh) of `ctx` (default: the default context)."""
        import numpy as np
        import torch

        from . import default_context
        from ._lib import ERR_ARGUMENT, OK, SjError
        ctx = ctx or default_context()
        dev = torch.device("cuda", torch.cuda.current_device())

        def up(a):
            a = np.ascontiguousarray(a)
            return torch.from_numpy(a.copy()).to(dev) if a.size else None

        tape = up(np.asarray(self.tape, dtype=np.uint64).view(np.int64))
        if tape is None:
            return b""
        strings = up(np.frombuffer(bytes(self.pj.Strings), dtype=np.uint8))
        message = up(np.frombuffer(bytes(self.pj.Message), dtype=np.uint8))
        torch.cuda.synchronize(dev)  # the library runs on its own stream
        rc, n, out = ctx.marshal_device(tape, strings, message)
        if rc == ERR_ARGUMENT:
            raise ValueError("malformed tape")
        if rc != OK:
            raise SjError(rc)
        return out.cpu().numpy().tobytes()

    def count_where(self, key, value):
        """ndjson_test.go:421 countWhere: records whose top-level `key` equals `value`."""
        return sum(1 for r in self.roots() if isinstance(r, dict) and r.get(key) == value)
