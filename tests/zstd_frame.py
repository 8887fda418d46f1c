"""A strict decoder of one zstd frame, written from RFC 8878 (test infrastructure, not part of the product).

It decodes every block type (Raw, RLE, Compressed), every literals type (Raw, RLE, Huffman_Compressed with one or four
streams and FSE-compressed or direct weights, Treeless), every sequence table mode (Predefined, RLE, FSE_Compressed,
Repeat) and repeat offsets, and raises ZstdError on anything a lenient decoder would let pass:
  * reserved bits that are not zero, a dictionary, a content checksum (not supported), or a window smaller than the
    data needs;
  * a block over 128 KiB (or the window), compressed or decompressed;
  * a Frame_Content_Size that differs from the output, and bytes after the frame;
  * bitstreams that are not consumed exactly to their padding bit (the Huffman weights' two-state FSE stream ends by
    its overflow rule, RFC 8878 4.2.1.2);
  * Huffman weights whose sum does not reach a power of two through the implied last weight, codes longer than 11 bits;
  * FSE table descriptions whose counts do not fill the table, or that name symbols past the alphabet;
  * offsets before the start of the output, zero offsets;
  * literal sizes that do not fit the block, four-stream jump tables whose sizes do not add up, sequences that ask for
    more literals than the section holds.
"""

MAGIC = b"\x28\xb5\x2f\xfd"
BLOCK_MAX = 128 << 10


class ZstdError(ValueError):
    pass


def _need(cond, msg):
    if not cond:
        raise ZstdError(msg)


def _highbit(x):
    return x.bit_length() - 1


class _Fwd:
    """forward little-endian bit reader (FSE table descriptions)"""

    def __init__(self, buf):
        self.b, self.pos = buf, 0

    def read(self, n):
        _need(self.pos + n <= 8 * len(self.b), "FSE table description runs past its data")
        v = (int.from_bytes(self.b[self.pos >> 3:(self.pos + n + 7 >> 3) + 1], "little") >> (self.pos & 7)) & ((1 << n) - 1)
        self.pos += n
        return v

    def peek(self, n):
        avail = 8 * len(self.b) - self.pos
        v = int.from_bytes(self.b[self.pos >> 3:(self.pos + n + 7 >> 3) + 1], "little") >> (self.pos & 7)
        return v & ((1 << min(n, avail)) - 1)


class _Back:
    """backward bit reader: from the bit below the padding 1 bit of the last byte towards bit 0"""

    def __init__(self, buf):
        _need(len(buf) >= 1, "empty bitstream")
        _need(buf[-1] != 0, "bitstream without its padding bit")
        self.b = bytes(buf)
        self.pos = 8 * (len(buf) - 1) + _highbit(buf[-1])

    def read(self, n):
        if n == 0:
            return 0
        _need(self.pos >= n, "bitstream read past its start")
        self.pos -= n
        lo = self.pos
        return (int.from_bytes(self.b[lo >> 3:(lo + n + 7 >> 3) + 1], "little") >> (lo & 7)) & ((1 << n) - 1)

    def peek(self, n):
        """the next n bits, zero-filled past the start"""
        if self.pos >= n:
            lo = self.pos - n
            return (int.from_bytes(self.b[lo >> 3:(lo + n + 7 >> 3) + 1], "little") >> (lo & 7)) & ((1 << n) - 1)
        return (int.from_bytes(self.b[:(self.pos + 7 >> 3) + 1], "little") & ((1 << self.pos) - 1)) << (n - self.pos)

    def done(self):
        _need(self.pos == 0, "bitstream not consumed exactly to its padding bit (%d bits left)" % self.pos)


# ---------------------------------------------------------------------------------------------------- FSE
def read_ncount(buf, max_al, max_sym):
    """FSE table description (RFC 8878 4.1.1): (normalised counts, accuracy log, bytes used)"""
    r = _Fwd(buf)
    al = r.read(4) + 5
    _need(al <= max_al, "accuracy log %d over %d" % (al, max_al))
    remaining, norm = (1 << al) + 1, []
    threshold, nbits = 1 << al, al + 1
    while remaining > 1:
        _need(len(norm) <= max_sym, "FSE description names symbols past the alphabet")
        mx = (2 * threshold - 1) - remaining
        low = r.peek(nbits - 1)
        if low < mx:
            count = r.read(nbits - 1)
        else:
            count = r.read(nbits)
            if count >= threshold:
                count -= mx
        count -= 1
        _need(count == -1 or count <= remaining - 1, "FSE counts overfill the table")
        remaining -= abs(count)
        norm.append(count)
        if count == 0:
            while True:
                rep = r.read(2)
                norm.extend([0] * rep)
                if rep < 3:
                    break
        while remaining < threshold:
            nbits -= 1
            threshold >>= 1
    _need(remaining == 1, "FSE counts do not fill the table")
    _need(len(norm) <= max_sym + 1, "FSE description names symbols past the alphabet")
    return norm, al, (r.pos + 7) >> 3


def fse_table(norm, al):
    """decoding table: list of (symbol, nbits, baseline) per state"""
    size = 1 << al
    _need(sum(1 if c == -1 else c for c in norm) == size, "FSE counts do not fill the table")
    sym = [None] * size
    high = size - 1
    for s, c in enumerate(norm):
        if c == -1:
            sym[high] = s
            high -= 1
    pos, step = 0, (size >> 1) + (size >> 3) + 3
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            sym[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    _need(pos == 0, "FSE spread did not return to state 0")
    nxt = [1 if c == -1 else c for c in norm]
    tab = []
    for u in range(size):
        s = sym[u]
        x = nxt[s]
        nxt[s] += 1
        nb = al - _highbit(x)
        tab.append((s, nb, (x << nb) - size))
    return tab


def rle_table(sym):
    return [(sym, 0, 0)]


# ---------------------------------------------------------------------------------------------------- Huffman
def huffman_table(data):
    """Huffman tree description (RFC 8878 4.2.1): ((table, max_bits), bytes used)"""
    _need(len(data) >= 1, "missing Huffman tree description")
    hb = data[0]
    if hb < 128:
        csize = hb
        _need(1 + csize <= len(data), "Huffman weights run past the literals section")
        body = data[1:1 + csize]
        norm, al, used = read_ncount(body, 6, 255)
        tab = fse_table(norm, al)
        r = _Back(body[used:])
        s1, s2 = r.read(al), r.read(al)
        weights = []
        states = [s1, s2]
        k = 0
        while True:  # two interleaved states; stop when an update would read past the start (RFC 8878 4.2.1.2)
            sym, nb, base = tab[states[k]]
            weights.append(sym)
            _need(len(weights) <= 255, "too many Huffman weights")
            if r.pos < nb:
                weights.append(tab[states[1 - k]][0])
                break
            states[k] = base + r.read(nb)
            k = 1 - k
        used_total = 1 + csize
    else:
        n = hb - 127
        used_total = 1 + (n + 1) // 2
        _need(used_total <= len(data), "Huffman weights run past the literals section")
        weights = []
        for i in range(n):
            b = data[1 + i // 2]
            weights.append(b >> 4 if i % 2 == 0 else b & 15)
    _need(all(w <= 11 for w in weights), "Huffman weight over 11")
    total = sum(1 << (w - 1) for w in weights if w)
    _need(total > 0, "Huffman weights all zero")
    max_bits = _highbit(total) + 1
    rest = (1 << max_bits) - total
    _need(rest & (rest - 1) == 0, "Huffman weights do not sum to a power of two")
    _need(max_bits <= 11, "Huffman code longer than 11 bits")
    weights.append(_highbit(rest) + 1)
    _need(len(weights) <= 256, "too many Huffman weights")
    _need(sum(1 for w in weights if w == 1) >= 2 and sum(1 for w in weights if w == 1) % 2 == 0,
          "Huffman tree with an odd number of longest codes")
    table = [None] * (1 << max_bits)
    pos = 0
    for w in range(1, max_bits + 1):
        for s, ws in enumerate(weights):
            if ws == w:
                n = 1 << (w - 1)
                table[pos:pos + n] = [(s, max_bits + 1 - w)] * n
                pos += n
    _need(pos == len(table), "Huffman table not full")
    return (table, max_bits), used_total


def huffman_stream(buf, count, huf):
    table, max_bits = huf
    r = _Back(buf)
    out = bytearray()
    for _ in range(count):
        s, nb = table[r.peek(max_bits)]
        r.read(nb)
        out.append(s)
    r.done()
    return bytes(out)


# ---------------------------------------------------------------------------------------------------- sequences
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384,
                             32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = list(range(3, 35)) + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195,
                                16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
LL_DEFAULT = ([4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1,
               -1, -1, -1, -1], 6)
ML_DEFAULT = ([1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7, 6)
OF_DEFAULT = ([1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5, 5)


class _Frame:
    def __init__(self, window):
        self.out = bytearray()
        self.window = window
        self.rep = [1, 4, 8]
        self.huf = None
        self.tabs = [None, None, None]  # LL, OF, ML (for Repeat mode)


def _literals(d, fr):
    """literals section: (literals, bytes used)"""
    _need(len(d) >= 1, "missing literals section")
    b0 = d[0]
    lt, sf = b0 & 3, (b0 >> 2) & 3
    if lt in (0, 1):
        if sf in (0, 2):
            R, h = b0 >> 3, 1
        elif sf == 1:
            _need(len(d) >= 2, "literals header past the block")
            R, h = (b0 >> 4) + (d[1] << 4), 2
        else:
            _need(len(d) >= 3, "literals header past the block")
            R, h = (b0 >> 4) + (d[1] << 4) + (d[2] << 12), 3
        _need(R <= BLOCK_MAX, "literals over 128 KiB")
        if lt == 0:
            _need(h + R <= len(d), "Raw literals past the block")
            return bytes(d[h:h + R]), h + R
        _need(h + 1 <= len(d), "RLE literal past the block")
        return bytes(d[h:h + 1]) * R, h + 1
    h, bits = {0: (3, 10), 1: (3, 10), 2: (4, 14), 3: (5, 18)}[sf]
    _need(len(d) >= h, "literals header past the block")
    v = int.from_bytes(d[:h], "little")
    R, C = (v >> 4) & ((1 << bits) - 1), v >> (4 + bits)
    _need(R <= BLOCK_MAX, "literals over 128 KiB")
    _need(h + C <= len(d), "compressed literals size past the block")
    body = bytes(d[h:h + C])
    if lt == 2:
        fr.huf, used = huffman_table(body)
        body = body[used:]
    else:
        _need(fr.huf is not None, "Treeless literals without an earlier Huffman table")
    if sf == 0:
        return huffman_stream(body, R, fr.huf), h + C
    _need(len(body) >= 6, "jump table past the literals section")
    s1, s2, s3 = (int.from_bytes(body[i:i + 2], "little") for i in (0, 2, 4))
    s4 = len(body) - 6 - s1 - s2 - s3
    _need(s4 >= 1 and min(s1, s2, s3) >= 1, "jump table sizes do not match the literals section")
    q = (R + 3) // 4
    _need(R - 3 * q >= 0, "too few literals for four streams")
    o, out = 6, b""
    for k, sz in enumerate((s1, s2, s3, s4)):
        out += huffman_stream(body[o:o + sz], q if k < 3 else R - 3 * q, fr.huf)
        o += sz
    return out, h + C


def _table(mode, d, k, default, max_al, max_sym, fr):
    """one sequence table: (FSE decoding table, bytes used)"""
    if mode == 0:
        t = fse_table(*default)
    elif mode == 1:
        _need(k < len(d), "RLE symbol past the block")
        _need(d[k] <= max_sym, "RLE symbol past the alphabet")
        return rle_table(d[k]), 1
    elif mode == 2:
        norm, al, used = read_ncount(d[k:], max_al, max_sym)
        return fse_table(norm, al), used
    else:
        _need(fr is not None, "Repeat mode without an earlier table")
        return fr, 0
    return t, 0


def _sequences(d, lits, fr):
    _need(len(d) >= 1, "missing sequences section")
    b0 = d[0]
    if b0 == 0:
        _need(len(d) == 1, "bytes after an empty sequences section")
        fr.out += lits
        return
    if b0 < 128:
        ns, k = b0, 1
    elif b0 < 255:
        _need(len(d) >= 2, "sequence count past the block")
        ns, k = ((b0 - 128) << 8) + d[1], 2
    else:
        _need(len(d) >= 3, "sequence count past the block")
        ns, k = d[1] + (d[2] << 8) + 0x7F00, 3
    _need(k < len(d), "compression modes past the block")
    modes = d[k]
    _need(modes & 3 == 0, "reserved bits of the compression modes are set")
    k += 1
    tabs = []
    for i, (mode, default, max_al, max_sym) in enumerate(((modes >> 6, LL_DEFAULT, 9, 35),
                                                          ((modes >> 4) & 3, OF_DEFAULT, 8, 31),
                                                          ((modes >> 2) & 3, ML_DEFAULT, 9, 52))):
        t, used = _table(mode, d, k, default, max_al, max_sym, fr.tabs[i])
        tabs.append(t)
        k += used
    fr.tabs = tabs
    ll_t, of_t, ml_t = tabs
    r = _Back(d[k:])
    al = lambda t: _highbit(len(t))  # noqa: E731
    sll, sof, sml = r.read(al(ll_t)), r.read(al(of_t)), r.read(al(ml_t))
    out, lp = fr.out, 0
    for i in range(ns):
        ofc, mlc, llc = of_t[sof][0], ml_t[sml][0], ll_t[sll][0]
        _need(ofc <= 31 and mlc <= 52 and llc <= 35, "sequence code past the alphabet")
        ov = (1 << ofc) + r.read(ofc)
        ml = ML_BASE[mlc] + r.read(ML_BITS[mlc])
        ll = LL_BASE[llc] + r.read(LL_BITS[llc])
        if ov > 3:
            off = ov - 3
            fr.rep = [off, fr.rep[0], fr.rep[1]]
        else:
            idx = ov - 1 if ll else ov
            if idx == 0:
                off = fr.rep[0]
            elif idx == 1:
                off = fr.rep[1]
                fr.rep = [off, fr.rep[0], fr.rep[2]]
            elif idx == 2:
                off = fr.rep[2]
                fr.rep = [off, fr.rep[0], fr.rep[1]]
            else:
                off = fr.rep[0] - 1
                _need(off >= 1, "repeat offset 0")
                fr.rep = [off, fr.rep[0], fr.rep[1]]
        _need(lp + ll <= len(lits), "sequences ask for more literals than the section holds")
        out += lits[lp:lp + ll]
        lp += ll
        _need(1 <= off <= len(out), "offset before the start of the output")
        _need(off <= fr.window, "offset beyond the window")
        if off >= ml:
            out += out[len(out) - off:len(out) - off + ml]
        else:
            for _ in range(ml):
                out.append(out[-off])
        if i + 1 < ns:
            _, nb, base = ll_t[sll]
            sll = base + r.read(nb)
            _, nb, base = ml_t[sml]
            sml = base + r.read(nb)
            _, nb, base = of_t[sof]
            sof = base + r.read(nb)
    r.done()
    out += lits[lp:]


def decode(frame):
    """the content of exactly one zstd frame (bytes), or ZstdError"""
    d = bytes(frame)
    _need(d[:4] == MAGIC, "bad magic")
    _need(len(d) >= 5, "truncated frame header")
    fhd = d[4]
    fcs_flag, single, reserved, checksum, did = fhd >> 6, (fhd >> 5) & 1, (fhd >> 3) & 1, (fhd >> 2) & 1, fhd & 3
    _need(reserved == 0, "reserved bit of the frame header descriptor is set")
    _need(not checksum, "content checksums are not supported")
    p = 5
    window = None
    if not single:
        _need(p < len(d), "truncated frame header")
        wd = d[p]
        base = 1 << (10 + (wd >> 3))
        window = base + (base >> 3) * (wd & 7)
        p += 1
    dsz = [0, 1, 2, 4][did]
    _need(p + dsz <= len(d), "truncated frame header")
    _need(int.from_bytes(d[p:p + dsz], "little") == 0, "dictionaries are not supported")
    p += dsz
    fsz = [1 if single else 0, 2, 4, 8][fcs_flag]
    _need(p + fsz <= len(d), "truncated frame header")
    fcs = int.from_bytes(d[p:p + fsz], "little") + (256 if fsz == 2 else 0) if fsz else None
    p += fsz
    if single:
        window = fcs
    fr = _Frame(window)
    bmax = min(window, BLOCK_MAX)
    while True:
        _need(p + 3 <= len(d), "truncated block header")
        bh = int.from_bytes(d[p:p + 3], "little")
        p += 3
        last, bt, bs = bh & 1, (bh >> 1) & 3, bh >> 3
        _need(bt != 3, "reserved block type")
        if bt == 1:
            _need(bs <= bmax, "block over its maximum size")
            _need(p + 1 <= len(d), "truncated RLE block")
            fr.out += d[p:p + 1] * bs
            p += 1
        else:
            _need(bs <= bmax, "block over its maximum size")
            _need(p + bs <= len(d), "truncated block")
            blk = d[p:p + bs]
            p += bs
            if bt == 0:
                fr.out += blk
            else:
                start = len(fr.out)
                lits, used = _literals(blk, fr)
                _sequences(blk[used:], lits, fr)
                _need(len(fr.out) - start <= bmax, "block decompresses to more than its maximum size")
        if fcs is not None:
            _need(len(fr.out) <= fcs, "output larger than Frame_Content_Size")
        if last:
            break
    _need(p == len(d), "bytes after the frame")
    if fcs is not None:
        _need(len(fr.out) == fcs, "Frame_Content_Size differs from the output")
    return bytes(fr.out)
