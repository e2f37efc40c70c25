"""Tapes written directly, with no parse.  Test infrastructure, like tests/marshal_oracle.py: it lets a test put any tape
item at any word index, at sizes no fixture reaches, and write the malformed tapes a parser never produces.

The layout is the parser's (parsed_json.go): a word is tag << 56 | value.  An open `{` `[` `r` holds one past the index
of its close, a close holds the index of its open.  A string is `"` | offset, then its length; the offset points into
Strings.B when STRINGBUFBIT is set and into the message otherwise.  `l` `u` `d` are followed by a raw 64-bit payload
word.  `t` `f` `n` are one word.

Items are emitted in order.  Runs of millions of words (fillers, numbers, nesting) are written with numpy.  In grammar
mode the builder refuses what JSON cannot express (a non-string key, an object closed behind a key, a value outside a
root); `raw=True` skips those checks, and `words()` appends anything."""
import numpy as np

TAG = 56
VAL = (1 << 56) - 1
STRINGBUFBIT = 1 << 55
M64 = (1 << 64) - 1
_CLOSE = {ord("{"): ord("}"), ord("["): ord("]"), ord("r"): ord("r")}


def word(tag, v=0):
    return (ord(tag) << TAG) | v


class TapeBuilder:
    def __init__(self, raw=False):
        self.raw = raw
        self._t = np.zeros(1 << 12, dtype=np.uint64)
        self.n = 0
        self.strings = bytearray()
        self.message = bytearray()
        self._keys = {}
        # the containers still open, innermost last: tag, index of the open, items written inside it so far
        self._kind = np.zeros(64, dtype=np.uint64)
        self._open = np.zeros(64, dtype=np.uint64)
        self._items = np.zeros(64, dtype=np.int64)
        self.depth = 0

    # ---- storage -----------------------------------------------------------------------------------------------
    def _grow(self, k):
        if self.n + k > self._t.size:
            t = np.zeros(max(2 * self._t.size, self.n + k), dtype=np.uint64)
            t[:self.n] = self._t[:self.n]
            self._t = t

    def _put(self, words):
        w = np.asarray(words, dtype=np.uint64)
        self._grow(w.size)
        self._t[self.n:self.n + w.size] = w
        self.n += w.size

    def _push(self, kind, at):
        if self.depth + at.size > self._kind.size:
            m = max(2 * self._kind.size, self.depth + at.size)
            for name in ("_kind", "_open", "_items"):
                a = getattr(self, name)
                b = np.zeros(m, dtype=a.dtype)
                b[:self.depth] = a[:self.depth]
                setattr(self, name, b)
        d = self.depth
        self._kind[d:d + at.size] = kind
        self._open[d:d + at.size] = at
        self._items[d:d + at.size] = 0
        self.depth += at.size

    def key_offset(self, key):
        """offset of `key` in Strings.B, written there once"""
        if key not in self._keys:
            self._keys[key] = len(self.strings)
            self.strings += key
        return self._keys[key]

    # ---- grammar -----------------------------------------------------------------------------------------------
    def _items_in_top(self, k, keyed=False):
        """k items written in a run into the innermost container; keyed: they are k / 2 key-value pairs"""
        if not self.raw:
            assert self.depth, "a value outside a root"
            if self._kind[self.depth - 1] == ord("{"):
                assert self._items[self.depth - 1] % 2 == 0 and keyed, "an object member needs a string key"
        if self.depth:
            self._items[self.depth - 1] += k

    def _value(self, is_string=False):
        if not self.raw:
            assert self.depth, "a value outside a root"
            if self._kind[self.depth - 1] == ord("{") and self._items[self.depth - 1] % 2 == 0:
                assert is_string, "an object key must be a string"
        if self.depth:
            self._items[self.depth - 1] += 1

    # ---- items -------------------------------------------------------------------------------------------------
    def open(self, kind):
        """`{`, `[` or a root `r`; its link is filled in by close()"""
        if kind == "r":
            assert self.raw or self.depth == 0, "a root inside a value"
        else:
            self._value()
        self._push(ord(kind), np.array([self.n], dtype=np.uint64))
        self._put([word(kind)])

    def nest(self, kind, depth, key=b"a"):
        """`depth` opens, each the first value of the one before: [[[... or {"a":{"a":...  The innermost is empty."""
        self._value()
        if kind == "[":
            at = np.arange(self.n, self.n + depth, dtype=np.uint64)
            self._put(np.full(depth, word("["), dtype=np.uint64))
            self._push(ord("["), at)
            return
        off = self.key_offset(key)
        w = np.empty((depth, 3), dtype=np.uint64)
        w[:, 0] = word("{")
        w[:, 1] = word('"', STRINGBUFBIT | off)
        w[:, 2] = len(key)
        at = np.arange(self.n, self.n + 3 * depth, 3, dtype=np.uint64)
        self._put(w.reshape(-1)[:-2])
        self._push(ord("{"), at)
        self._items[self.depth - depth:self.depth - 1] = 2

    def close(self, k=1):
        """close the k innermost containers"""
        assert 0 < k <= self.depth
        kind = self._kind[self.depth - k:self.depth][::-1]
        at = self._open[self.depth - k:self.depth][::-1]
        if not self.raw:
            items = self._items[self.depth - k:self.depth][::-1]
            assert not ((kind == ord("{")) & (items % 2 == 1)).any(), "an object closed behind a key"
        pos = np.arange(self.n, self.n + k, dtype=np.uint64)
        close_tag = np.where(kind == ord("{"), ord("}"), np.where(kind == ord("["), ord("]"), ord("r"))).astype(np.uint64)
        self._t[at] |= pos + np.uint64(1)
        self._put((close_tag << np.uint64(TAG)) | at)
        self.depth -= k

    def string(self, s, copy=True):
        """a string in Strings.B (copy) or at the end of the message"""
        self._value(is_string=True)
        s = bytes(s)
        if copy:
            w = word('"', STRINGBUFBIT | len(self.strings))
            self.strings += s
        else:
            w = word('"', len(self.message))
            self.message += s
        self._put([w, len(s)])

    def number(self, tag, payload, flags=0):
        """`l`, `u` or `d` with a raw 64-bit payload; `flags` goes into the head's value bits"""
        assert tag in "lud"
        self._value()
        self._put([word(tag, flags), int(payload) & M64])

    def numbers(self, tag, payloads, key=None):
        """one number per payload; with `key`, each is an object member under that key (stored once)"""
        assert tag in "lud"
        p = np.asarray(payloads, dtype=np.uint64)
        if key is None:
            self._items_in_top(p.size)
            w = np.empty((p.size, 2), dtype=np.uint64)
        else:
            self._items_in_top(2 * p.size, keyed=True)
            w = np.empty((p.size, 4), dtype=np.uint64)
            w[:, 0] = word('"', STRINGBUFBIT | self.key_offset(key))
            w[:, 1] = len(key)
        w[:, -2] = word(tag)
        w[:, -1] = p
        self._put(w.reshape(-1))

    def atom(self, tag):
        assert tag in "tfn"
        self._value()
        self._put([word(tag)])

    def atoms(self, tags):
        """one-word atoms, one per character of `tags` (a str), or `tags` = (tag, count)"""
        if isinstance(tags, tuple):
            tag, k = tags
            w = np.full(k, word(tag), dtype=np.uint64)
        else:
            w = np.frombuffer(tags.encode(), dtype=np.uint8).astype(np.uint64) << np.uint64(TAG)
        self._items_in_top(w.size)
        self._put(w)

    def pad_to(self, index, tag="n"):
        """one-word atoms up to `index`, so the next word lands on it; returns their count"""
        k = index - self.n
        assert k >= 0, (index, self.n)
        if k:
            self.atoms((tag, k))
        return k

    def pad_members_to(self, index, key=b"k"):
        """object members "key":null (3 words) and "key":0 (4 words) up to `index`; returns (count of 3, count of 4)"""
        d = index - self.n
        n4 = d % 3
        n3 = (d - 4 * n4) // 3
        assert n3 >= 0, (index, self.n)
        off = self.key_offset(key)
        self._items_in_top(2 * (n3 + n4), keyed=True)
        w3 = np.empty((n3, 3), dtype=np.uint64)
        w3[:] = [word('"', STRINGBUFBIT | off), len(key), word("n")]
        w4 = np.empty((n4, 4), dtype=np.uint64)
        w4[:] = [word('"', STRINGBUFBIT | off), len(key), word("l"), 0]
        self._put(np.concatenate([w3.reshape(-1), w4.reshape(-1)]))
        return n3, n4

    def words(self, ws):
        """raw words, appended as they are (raw mode only)"""
        assert self.raw
        self._put(ws)

    # ---- result ------------------------------------------------------------------------------------------------
    def build(self):
        """(tape as uint64, Strings.B, message)"""
        assert self.raw or self.depth == 0, "containers left open"
        return self._t[:self.n].copy(), bytes(self.strings), bytes(self.message)
