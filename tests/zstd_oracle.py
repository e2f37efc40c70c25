"""A Python restatement of the zstd decoder (RFC 8878) the device reads the Serializer's zstd blocks with (block type 2,
CompressDefault / CompressBest), its acceptance rules included, XXH64, a small frame writer for constructed frames and a
stream oracle that knows the compress modes.

decode(data) -> bytes, or raises ZstdError.  The rules are the header's (include/simdjson_b200.h): zero or more
frames back to back, zstd or skippable; no dictionary; FCS and checksum checked when present; raw, RLE and compressed
blocks, a compressed block at most min(window, 128 KiB) both ways (raw and RLE blocks are not limited, as in libzstd); every literal and sequence mode, table repeats only
after a table of the same frame; bitstreams ending exactly at their padding; no match reaching in front of the frame.
"""

MAGIC = 0xFD2FB528
BLOCK_MAX = 128 << 10
M64 = (1 << 64) - 1


class ZstdError(ValueError):
    pass


def _need(cond, what):
    if not cond:
        raise ZstdError(what)


# ---------------------------------------------------------------------------------------------------------------------
# XXH64
# ---------------------------------------------------------------------------------------------------------------------
P1, P2, P3, P4, P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _round(acc, v):
    return (_rotl((acc + v * P2) & M64, 31) * P1) & M64


def xxh64(data, seed=0):
    n, i = len(data), 0
    if n >= 32:
        v = [(seed + P1 + P2) & M64, (seed + P2) & M64, seed, (seed - P1) & M64]
        while i + 32 <= n:
            for k in range(4):
                v[k] = _round(v[k], int.from_bytes(data[i + 8 * k:i + 8 * k + 8], "little"))
            i += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M64
        for k in range(4):
            h = ((h ^ _round(0, v[k])) * P1 + P4) & M64
    else:
        h = (seed + P5) & M64
    h = (h + n) & M64
    while i + 8 <= n:
        h = (_rotl(h ^ _round(0, int.from_bytes(data[i:i + 8], "little")), 27) * P1 + P4) & M64
        i += 8
    if i + 4 <= n:
        h = (_rotl(h ^ (int.from_bytes(data[i:i + 4], "little") * P1) & M64, 23) * P2 + P3) & M64
        i += 4
    while i < n:
        h = (_rotl(h ^ (data[i] * P5) & M64, 11) * P1) & M64
        i += 1
    h = ((h ^ (h >> 33)) * P2) & M64
    h = ((h ^ (h >> 29)) * P3) & M64
    return h ^ (h >> 32)


# ---------------------------------------------------------------------------------------------------------------------
# bitstreams read backwards from their padding
# ---------------------------------------------------------------------------------------------------------------------
class BackBits:
    """the bits of s, last byte's highest set bit the padding; read(n) takes the n highest unread bits, zeros past
    the start (then `left` goes negative and the stream cannot end exactly)"""

    def __init__(self, s):
        _need(len(s) > 0 and s[-1] != 0, "bitstream without padding")
        self.v = int.from_bytes(s, "little")
        self.left = 8 * len(s) - (8 - s[-1].bit_length()) - 1

    def read(self, n):
        if n == 0:
            return 0
        self.left -= n
        if self.left >= 0:
            return (self.v >> self.left) & ((1 << n) - 1)
        return ((self.v << -self.left) & ((1 << n) - 1)) if self.left > -n else 0

    def done(self):
        return self.left == 0


# ---------------------------------------------------------------------------------------------------------------------
# FSE tables
# ---------------------------------------------------------------------------------------------------------------------
LL_DEFAULT = ([4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1], 6)
ML_DEFAULT = ([1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
               1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1], 6)
OF_DEFAULT = ([1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1], 5)
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = [i + 3 for i in range(32)] + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                        16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_MAX, ML_MAX, OF_MAX = 35, 52, 31
LL_LOG, ML_LOG, OF_LOG = 9, 9, 8


def fse_table(counts, al):
    """the decoding table of normalized counts at accuracy log al: (symbol, nbits, baseline) per state"""
    size = 1 << al
    sym = [0] * size
    high = size - 1
    nxt = list(counts)
    for s, c in enumerate(counts):
        if c == -1:
            sym[high] = s
            high -= 1
            nxt[s] = 1
    step, pos = (size >> 1) + (size >> 3) + 3, 0
    for s, c in enumerate(counts):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    _need(pos == 0, "FSE spread does not return to 0")
    tab = []
    for u in range(size):
        s = sym[u]
        x = nxt[s]
        nxt[s] += 1
        nb = al - (x.bit_length() - 1)
        tab.append((s, nb, (x << nb) - size))
    return tab


def read_ncount(s, at, end, max_sym, max_log):
    """an FSE table description at s[at:]: (counts, al, bytes)"""
    bits = int.from_bytes(s[at:end], "little")
    nbytes = end - at
    _need(nbytes >= 1, "FSE description cut")
    al = (bits & 15) + 5
    _need(al <= max_log, "FSE accuracy log too large")
    pos = 4
    remaining = (1 << al) + 1
    threshold = 1 << al
    nb = al + 1
    counts = []
    prev0 = False
    while remaining > 1 and len(counts) <= max_sym:
        if prev0:
            n0 = 0
            while True:
                r = (bits >> pos) & 3
                pos += 2
                n0 += r
                if r != 3:
                    break
            _need(len(counts) + n0 <= max_sym + 1, "FSE zero run past the last symbol")
            counts += [0] * n0
            if len(counts) > max_sym:
                break
        mx = (2 * threshold - 1) - remaining
        low = (bits >> pos) & (threshold - 1)
        if low < mx:
            v = low
            pos += nb - 1
        else:
            v = (bits >> pos) & (2 * threshold - 1)
            if v >= threshold:
                v -= mx
            pos += nb
        c = v - 1
        remaining -= -c if c < 0 else c
        counts.append(c)
        prev0 = c == 0
        while remaining < threshold:
            nb -= 1
            threshold >>= 1
    _need(remaining == 1, "FSE counts do not add up")
    _need(len(counts) <= max_sym + 1, "FSE symbol past the last")
    used = (pos + 7) >> 3
    _need(used <= nbytes, "FSE description cut")
    return counts + [0] * (max_sym + 1 - len(counts)), al, used


# ---------------------------------------------------------------------------------------------------------------------
# Huffman
# ---------------------------------------------------------------------------------------------------------------------
def read_huffman(s, at, end):
    """a Huffman tree description at s[at:end]: (table of (symbol, nbits) per maxbits-bit prefix, maxbits, bytes)"""
    _need(at < end, "Huffman description cut")
    h = s[at]
    if h < 128:
        _need(h >= 1 and at + 1 + h <= end, "Huffman FSE weights cut")
        counts, al, used = read_ncount(s, at + 1, at + 1 + h, 255, 6)
        tab = fse_table(counts, al)
        br = BackBits(s[at + 1 + used:at + 1 + h])
        s1, s2 = br.read(al), br.read(al)
        w = []
        while True:
            _need(len(w) < 255, "too many Huffman weights")
            sy, nb, base = tab[s1]
            w.append(sy)
            s1 = base + br.read(nb)
            if br.left < 0:
                w.append(tab[s2][0])
                break
            _need(len(w) < 255, "too many Huffman weights")
            sy, nb, base = tab[s2]
            w.append(sy)
            s2 = base + br.read(nb)
            if br.left < 0:
                w.append(tab[s1][0])
                break
        _need(len(w) <= 255, "too many Huffman weights")
        size = 1 + h
    else:
        n = h - 127
        size = 1 + (n + 1) // 2
        _need(at + size <= end, "Huffman direct weights cut")
        w = []
        for k in range(n):
            b = s[at + 1 + k // 2]
            w.append(b >> 4 if k % 2 == 0 else b & 15)
    _need(all(x <= 11 for x in w), "Huffman weight too large")
    total = sum(1 << (x - 1) for x in w if x)
    _need(total > 0, "no Huffman weights")
    maxbits = total.bit_length()
    left = (1 << maxbits) - total
    _need(left & (left - 1) == 0 and left > 0, "Huffman weights do not complete a tree")
    _need(maxbits <= 11, "Huffman tree too deep")
    w.append(left.bit_length())
    start, pos = {}, 0
    for wt in range(1, maxbits + 1):
        start[wt] = pos
        pos += sum(1 for x in w if x == wt) << (wt - 1)
    tab = [None] * (1 << maxbits)
    for sy, wt in enumerate(w):
        if wt:
            ln = 1 << (wt - 1)
            for k in range(ln):
                tab[start[wt] + k] = (sy, maxbits + 1 - wt)
            start[wt] += ln
    return tab, maxbits, size


def huff_stream(s, tab, maxbits, n):
    br = BackBits(s)
    out = bytearray()
    for _ in range(n):
        saved = br.left
        sy, nb = tab[br.read(maxbits)]
        br.left = saved
        br.read(nb)
        out.append(sy)
    _need(br.done(), "Huffman stream does not end at its padding")
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# blocks
# ---------------------------------------------------------------------------------------------------------------------
class FrameState:
    def __init__(self):
        self.huf = None
        self.tabs = [None, None, None]  # LL, OF, ML
        self.rep = [1, 4, 8]


def literals(s, at, end, st):
    """the literals section at s[at:end]: (literal bytes, where the sequences section starts)"""
    _need(at < end, "literals header cut")
    b0 = s[at]
    t, sf = b0 & 3, (b0 >> 2) & 3
    if t <= 1:
        if sf & 1 == 0:
            n, hl = b0 >> 3, 1
        elif sf == 1:
            _need(at + 2 <= end, "literals header cut")
            n, hl = (b0 >> 4) | (s[at + 1] << 4), 2
        else:
            _need(at + 3 <= end, "literals header cut")
            n, hl = (b0 >> 4) | (s[at + 1] << 4) | (s[at + 2] << 12), 3
        _need(n <= BLOCK_MAX, "literals larger than a block")
        at += hl
        if t == 0:
            _need(at + n <= end, "raw literals cut")
            return bytes(s[at:at + n]), at + n
        _need(at + 1 <= end, "RLE literal cut")
        return bytes([s[at]]) * n, at + 1
    hl = 3 if sf <= 1 else sf + 2
    _need(at + hl <= end, "literals header cut")
    h = int.from_bytes(s[at:at + hl], "little")
    nstreams = 1 if sf == 0 else 4
    sb = 10 if sf <= 1 else 14 if sf == 2 else 18
    n, csize = (h >> 4) & ((1 << sb) - 1), (h >> (4 + sb)) & ((1 << sb) - 1)
    _need(n <= BLOCK_MAX, "literals larger than a block")
    at += hl
    _need(at + csize <= end, "compressed literals cut")
    lend = at + csize
    if t == 2:
        st.huf = read_huffman(s, at, lend)
        at += st.huf[2]
    else:
        _need(st.huf is not None, "treeless literals without an earlier Huffman table")
    tab, maxbits, _ = st.huf
    if nstreams == 1:
        return huff_stream(s[at:lend], tab, maxbits, n), lend
    _need(lend - at >= 6, "jump table cut")
    sz = [s[at] | s[at + 1] << 8, s[at + 2] | s[at + 3] << 8, s[at + 4] | s[at + 5] << 8]
    at += 6
    sz.append(lend - at - sum(sz))
    _need(sz[3] >= 0, "jump table past the literals")
    q = (n + 3) // 4
    ns = [q, q, q, n - 3 * q]
    _need(ns[3] >= 0, "too few literals for four streams")
    out = b""
    for k in range(4):
        out += huff_stream(s[at:at + sz[k]], tab, maxbits, ns[k])
        at += sz[k]
    return out, lend


def sequences(s, at, end, st):
    """the sequences section: a list of (ll, ml, offset_value)"""
    _need(at < end, "sequences header cut")
    b0 = s[at]
    if b0 == 0:
        _need(at + 1 == end, "bytes behind an empty sequences section")
        return []
    if b0 < 128:
        nseq, at = b0, at + 1
    elif b0 < 255:
        _need(at + 2 <= end, "sequences header cut")
        nseq, at = ((b0 - 128) << 8) + s[at + 1], at + 2
    else:
        _need(at + 3 <= end, "sequences header cut")
        nseq, at = s[at + 1] + (s[at + 2] << 8) + 0x7F00, at + 3
    _need(at < end, "sequences modes cut")
    modes = s[at]
    at += 1
    _need(modes & 3 == 0, "reserved sequences mode bits")
    for k, (shift, dflt, mx, ml) in enumerate(((6, LL_DEFAULT, LL_MAX, LL_LOG), (4, OF_DEFAULT, OF_MAX, OF_LOG),
                                                (2, ML_DEFAULT, ML_MAX, ML_LOG))):
        m = (modes >> shift) & 3
        if m == 0:
            st.tabs[k] = (fse_table(*dflt), dflt[1])
        elif m == 1:
            _need(at < end and s[at] <= mx, "RLE symbol")
            st.tabs[k] = ([(s[at], 0, 0)], 0)
            at += 1
        elif m == 2:
            counts, al, used = read_ncount(s, at, end, mx, ml)
            st.tabs[k] = (fse_table(counts, al), al)
            at += used
        else:
            _need(st.tabs[k] is not None, "repeat mode without an earlier table")
    (llt, lla), (oft, ofa), (mlt, mla) = st.tabs
    br = BackBits(s[at:end])
    sl, so, sm = br.read(lla), br.read(ofa), br.read(mla)
    out = []
    for i in range(nseq):
        oc, mc, lc = oft[so][0], mlt[sm][0], llt[sl][0]
        _need(oc <= OF_MAX, "offset code")
        ofv = (1 << oc) + br.read(oc)
        ml = ML_BASE[mc] + br.read(ML_BITS[mc])
        ll = LL_BASE[lc] + br.read(LL_BITS[lc])
        out.append((ll, ml, ofv))
        if i != nseq - 1:
            for tab, k in ((llt, 0), (mlt, 2), (oft, 1)):
                cur = (sl, so, sm)[k]
                nxt = tab[cur][2] + br.read(tab[cur][1])
                if k == 0:
                    sl = nxt
                elif k == 1:
                    so = nxt
                else:
                    sm = nxt
    _need(br.done(), "sequences bitstream does not end at its padding")
    return out


def apply_offset(rep, ll, ofv):
    """the offset of one sequence and the repeat offsets behind it"""
    if ofv > 3:
        o = ofv - 3
        rep[:] = [o, rep[0], rep[1]]
        return o
    k = ofv - 1 + (ll == 0)
    if k == 0:
        return rep[0]
    o = rep[0] - 1 if k == 3 else rep[k]
    _need(o != 0, "repeat offset rep1 - 1 is 0")  # (libzstd rejects it too)
    if k == 1:
        rep[:] = [o, rep[0], rep[2]]
    else:
        rep[:] = [o, rep[0], rep[1]]
    return o


def compressed_block(s, at, end, st, out, fstart, limit):
    lit, at = literals(s, at, end, st)
    seqs = sequences(s, at, end, st)
    bstart, li = len(out), 0
    for ll, ml, ofv in seqs:
        _need(li + ll <= len(lit), "literal lengths past the literals")
        out += lit[li:li + ll]
        li += ll
        o = apply_offset(st.rep, ll, ofv)
        _need(o <= len(out) - fstart, "match in front of the frame")
        _need(len(out) + ml - bstart <= limit, "block decodes past its limit")
        for _ in range(ml):
            out.append(out[-o])
    out += lit[li:]
    _need(len(out) - bstart <= limit, "block decodes past its limit")


def frame(s, at, out):
    """one zstd frame at s[at:] (behind its magic) appended to out: where it ends"""
    _need(at < len(s), "frame header cut")
    fhd = s[at]
    at += 1
    fcs_flag, single, cks, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3
    _need(fhd & 8 == 0, "reserved frame header bit")
    window = None
    if not single:
        _need(at < len(s), "window descriptor cut")
        wd = s[at]
        at += 1
        base = 1 << (10 + (wd >> 3))
        window = base + (base >> 3) * (wd & 7)
    dn = [0, 1, 2, 4][did]
    _need(at + dn <= len(s), "dictionary ID cut")
    _need(int.from_bytes(s[at:at + dn], "little") == 0, "dictionary ID")
    at += dn
    fn = [1 if single else 0, 2, 4, 8][fcs_flag]
    _need(at + fn <= len(s), "frame content size cut")
    fcs = int.from_bytes(s[at:at + fn], "little") + (256 if fn == 2 else 0) if fn else None
    at += fn
    if single:
        window = fcs
    limit = min(window, BLOCK_MAX)
    st = FrameState()
    fstart = len(out)
    while True:
        _need(at + 3 <= len(s), "block header cut")
        bh = int.from_bytes(s[at:at + 3], "little")
        at += 3
        last, bt, bs = bh & 1, (bh >> 1) & 3, bh >> 3
        _need(bt != 3, "reserved block type")
        if bt == 1:
            _need(at + 1 <= len(s), "RLE block cut")
            out += bytes([s[at]]) * bs
            at += 1
        else:
            _need(bt == 0 or bs <= limit, "compressed block larger than its limit")
            _need(at + bs <= len(s), "block cut")
            if bt == 0:
                out += s[at:at + bs]
            else:
                compressed_block(s, at, at + bs, st, out, fstart, limit)
            at += bs
        if last:
            break
    n = len(out) - fstart
    _need(fcs is None or fcs == n, "frame content size")
    if cks:
        _need(at + 4 <= len(s), "checksum cut")
        _need(int.from_bytes(s[at:at + 4], "little") == xxh64(bytes(out[fstart:])) & 0xFFFFFFFF, "checksum")
        at += 4
    return at


def decode(data):
    """every frame of data, back to back"""
    s = bytes(data)
    out, at = bytearray(), 0
    while at < len(s):
        _need(len(s) - at >= 4, "frame magic cut")
        m = int.from_bytes(s[at:at + 4], "little")
        if m & 0xFFFFFFF0 == 0x184D2A50:
            _need(len(s) - at >= 8, "skippable frame cut")
            n = int.from_bytes(s[at + 4:at + 8], "little")
            _need(n <= len(s) - at - 8, "skippable frame cut")
            at += 8 + n
            continue
        _need(m == MAGIC, "frame magic")
        at = frame(s, at + 4, out)
    return bytes(out)


def read_block(data, raw):
    """a zstd block of the stream as Deserialize reads it: its bytes when they decode to exactly `raw` bytes"""
    out = decode(data)
    _need(len(out) == raw, "zstd block decodes to the wrong size")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# a small frame writer for constructed frames
# ---------------------------------------------------------------------------------------------------------------------
class FwdBits:
    """bits written forward, read back by BackBits from the end"""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, x, nb):
        self.v |= (x & ((1 << nb) - 1)) << self.n
        self.n += nb

    def close(self):
        self.put(1, 1)
        return self.v.to_bytes((self.n + 7) // 8, "little")


def fse_encoder(counts, al):
    """for each symbol and next state, the state in front of it: enc[sym][next] (the decoding table run backwards)"""
    tab = fse_table(counts, al)
    enc = {}
    for u, (sy, nb, base) in enumerate(tab):
        for x in range(base, base + (1 << nb)):
            enc.setdefault(sy, {})[x] = u
    return tab, enc


def _code(v, base):
    c = 0
    while c + 1 < len(base) and base[c + 1] <= v:
        c += 1
    return c


def of_code(ofv):
    return ofv.bit_length() - 1


def write_ncount(counts, al):
    """an FSE table description (the inverse of read_ncount)"""
    w = FwdBits()
    w.put(al - 5, 4)
    remaining, threshold, nb = (1 << al) + 1, 1 << al, al + 1
    last = max(i for i, c in enumerate(counts) if c)
    i = 0
    while i <= last:
        c = counts[i]
        v = c + 1
        mx = (2 * threshold - 1) - remaining
        if v < mx:
            w.put(v, nb - 1)
        else:
            w.put(v + mx if v >= threshold else v, nb)
        remaining -= -c if c < 0 else c
        while remaining < threshold:
            nb -= 1
            threshold >>= 1
        i += 1
        if c == 0:
            z = 0
            while i + z <= last and counts[i + z] == 0:
                z += 1
            i += z
            while z >= 3:
                w.put(3, 2)
                z -= 3
            w.put(z, 2)
    return w.v.to_bytes((w.n + 7) // 8, "little")


def encode_sequences(seqs, modes=(0, 0, 0), tables=None):
    """a sequences section of (ll, ml, offset_value): modes per LL, OF, ML of 0 predefined, 1 RLE (the one symbol),
    2 FSE with `tables[k]` = (counts, al) written, 3 repeat with `tables[k]` = (counts, al) of the table it repeats"""
    bases = ((LL_BASE, LL_BITS), None, (ML_BASE, ML_BITS))
    codes = [[_code(ll, LL_BASE) for ll, _, _ in seqs], [of_code(o) for _, _, o in seqs], [_code(ml, ML_BASE) for _, ml, _ in seqs]]
    n = len(seqs)
    hdr = bytes([n]) if n < 128 else bytes([128 + (n >> 8), n & 255]) if n < 0x7F00 else bytes([255, (n - 0x7F00) & 255, (n - 0x7F00) >> 8])
    if n == 0:
        return hdr
    desc = b""
    encs = []
    for k in range(3):
        m = modes[k]
        if m == 1:
            sy = codes[k][0]
            assert all(c == sy for c in codes[k])
            desc += bytes([sy])
            encs.append(([(sy, 0, 0)], {sy: {0: 0}}, 0))
            continue
        if m == 0:
            counts, al = (LL_DEFAULT, OF_DEFAULT, ML_DEFAULT)[k]
        else:
            counts, al = tables[k]
            if m == 2:
                desc += write_ncount(counts, al)
        tab, enc = fse_encoder(counts, al)
        encs.append((tab, enc, al))
    hdr += bytes([(modes[0] << 6) | (modes[1] << 4) | (modes[2] << 2)]) + desc
    w = FwdBits()
    # states from the last sequence back: state[k][i] decodes codes[k][i]
    states = [[0] * n for _ in range(3)]
    for k in range(3):
        tab, enc, al = encs[k]
        states[k][n - 1] = next(u for u, t in enumerate(tab) if t[0] == codes[k][n - 1])
        for i in range(n - 2, -1, -1):
            states[k][i] = enc[codes[k][i]][states[k][i + 1]]
    for i in range(n - 1, -1, -1):
        if i != n - 1:
            for k in (1, 2, 0):  # written in reverse of the reading order LL, ML, OF
                tab, _, _ = encs[k]
                _, nb, base = tab[states[k][i]]
                w.put(states[k][i + 1] - base, nb)
        ll, ml, ofv = seqs[i]
        lc, oc, mc = codes[0][i], codes[1][i], codes[2][i]
        w.put(ll - LL_BASE[lc], LL_BITS[lc])
        w.put(ml - ML_BASE[mc], ML_BITS[mc])
        w.put(ofv - (1 << oc), oc)
    for k in (2, 1, 0):
        w.put(states[k][0], encs[k][2])
    return hdr + w.close()


def huffman_code(weights):
    """(code, nbits) per symbol of a weight list with its last weight implied, as read_huffman assigns them"""
    total = sum(1 << (x - 1) for x in weights if x)
    maxbits = total.bit_length()
    w = list(weights) + [((1 << maxbits) - total).bit_length()]
    start, pos = {}, 0
    for wt in range(1, maxbits + 1):
        start[wt] = pos
        pos += sum(1 for x in w if x == wt) << (wt - 1)
    codes = {}
    for sy, wt in enumerate(w):
        if wt:
            nb = maxbits + 1 - wt
            codes[sy] = (start[wt] >> (maxbits - nb), nb)
            start[wt] += 1 << (wt - 1)
    return codes


def literals_section(lit, kind, weights=None, streams=1):
    """kind 0 raw, 1 RLE, 2 Huffman with `weights` (direct 4-bit form), 3 treeless (the frame's last weights)"""
    n = len(lit)
    if kind in (0, 1):
        if n < 32:
            h = bytes([kind | (n << 3)])
        elif n < 4096:
            h = bytes([kind | 4 | ((n & 15) << 4), n >> 4])
        else:
            h = bytes([kind | 12 | ((n & 15) << 4), (n >> 4) & 255, n >> 12])
        return h + (lit if kind == 0 else lit[:1])
    codes = huffman_code(weights)
    tree = b""
    if kind == 2:
        nw = len(weights)
        tree = bytes([127 + nw]) + bytes(((weights[i] << 4) | (weights[i + 1] if i + 1 < nw else 0)) for i in range(0, nw, 2))
    if streams == 1:
        body = tree + huff_bits(lit, codes)
        sf = 0
    else:
        q = (n + 3) // 4
        parts = [huff_bits(lit[k * q:(k + 1) * q] if k < 3 else lit[3 * q:], codes) for k in range(4)]
        body = tree + b"".join(len(p).to_bytes(2, "little") for p in parts[:3]) + b"".join(parts)
        sf = 1
    assert n < 1024 and len(body) < 1024
    h = kind | (sf << 2) | (n << 4) | (len(body) << 14)
    return h.to_bytes(3, "little") + body


def huff_bits(data, codes):
    """a Huffman stream: the decoder reads the last symbol's code... from the end: symbols written last to first"""
    bits, nbits = 0, 0
    for b in reversed(data):
        c, nb = codes[b]
        bits |= c << nbits
        nbits += nb
    bits |= 1 << nbits
    return bits.to_bytes((nbits + 8) // 8, "little")


def block(body, kind=2, last=False, size=None):
    """a block header (type kind: 0 raw, 1 RLE with size, 2 compressed) and its body"""
    n = size if kind == 1 else len(body)
    return ((n << 3) | (kind << 1) | int(last)).to_bytes(3, "little") + body


def frame_bytes(blocks, content=None, checksum=False, window_log=None, fcs=True):
    """a zstd frame of blocks (block() outputs, the last flagged); content: the decoded bytes (for FCS / checksum)"""
    if window_log is None:
        n = len(content)
        fcs_flag = 0 if n < 256 else 1 if n < 65536 + 256 else 2
        fhd = (fcs_flag << 6) | 0x20 | (4 if checksum else 0)
        v = n - 256 if fcs_flag == 1 else n
        head = bytes([fhd]) + v.to_bytes([1, 2, 4][fcs_flag], "little")
    else:
        fhd = (2 << 6 if fcs else 0) | (4 if checksum else 0)
        head = bytes([fhd, (window_log - 10) << 3]) + (len(content).to_bytes(4, "little") if fcs else b"")
    out = MAGIC.to_bytes(4, "little") + head + b"".join(blocks)
    if checksum:
        out += (xxh64(content) & 0xFFFFFFFF).to_bytes(4, "little")
    return out


def skippable(payload, k=0):
    return (0x184D2A50 + k).to_bytes(4, "little") + len(payload).to_bytes(4, "little") + payload


# ---------------------------------------------------------------------------------------------------------------------
# whole serialized streams, mode-aware (s2_oracle's block walk; its verdicts and serialize_oracle's stay as they are)
# ---------------------------------------------------------------------------------------------------------------------
def inflate(src):
    """the stream with every S2 and zstd block replaced by its inflated bytes as an uncompressed block, as
    CompressDefault / CompressBest read it; s2_oracle.Rejected for a header Deserialize rejects or a compressed block
    that breaks a rule"""
    from tests import s2_oracle as s2
    v, ts, blocks = s2._blocks(src)
    out = []
    for raw, t, d in blocks:
        if t == 1:
            out.append((raw, 0, s2.read(d, raw)))
        elif t == 2:
            try:
                out.append((raw, 0, read_block(d, raw)))
            except ZstdError as e:
                raise s2.Rejected(str(e))
        else:
            out.append((raw, t, d))
    return s2._assemble(v, ts, out)


# block types of the message, tags and values blocks Serialize writes in each compress mode
MODE_TYPES = {0: (0, 0, 0), 1: (1, 1, 1), 2: (1, 2, 1), 3: (2, 2, 2)}


def device_result(src, mode):
    """what the device deserializer gives in compress mode `mode`: s2_oracle's result in NONE / FAST mode, else
    serialize_oracle.device_result of the stream with S2 and zstd blocks inflated"""
    from tests import s2_oracle as s2
    from tests import serialize_oracle as so
    if mode == 1:
        return s2.device_result(src)
    if mode == 0:
        return so.device_result(src)
    return so.device_result(inflate(src))
