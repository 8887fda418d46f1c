"""Inputs of the LZ4 tests: serialised 512 KB groups of the bench shapes (synth + oracle.sls_serialize_logs), edge-case
segments, and the system's liblz4 (not vendored) as the second decoder and the ratio reference."""
import ctypes as C
import random

import numpy as np

from loongcollector_b200 import synth
from oracle import oracle as O

GROUP_BYTES = 512 << 10
SHAPES = ["c2_regex", "c2_split", "c3_java", "c4_csv", "c1_random"]
T0 = 1700000000


def _lines(buf, off, ln, budget):
    out, used = [], 0
    for o, n in zip(off.tolist(), ln.tolist()):
        if used >= budget:
            break
        out.append(bytes(buf[o:o + n]))
        used += n + 1
    return out


def shape_group(name, seed=1):
    """The `Logs` bytes of one group built from GROUP_BYTES of source lines (records for C3) of a shape."""
    if name in ("c2_regex", "c2_split"):
        buf, off, ln = synth.nginx_lines(GROUP_BYTES // 256 + 1, seed=seed)
        lines = _lines(buf, off, ln, GROUP_BYTES)
        if name == "c2_split":
            evs = [(T0 + i, None, [(b"content", x)]) for i, x in enumerate(lines)]
        else:
            keys = [k.encode() for k in synth.NGINX_KEYS]
            m = len(lines)
            st, co, cl = O.regex_parse_batch(O.Regex(synth.NGINX_PATTERN), buf, off[:m], ln[:m], len(keys))
            evs = []
            for i, x in enumerate(lines):
                kv = ([(k, bytes(buf[co[i][j]:co[i][j] + cl[i][j]])) for j, k in enumerate(keys)]
                      if st[i] == 0 else [(b"__raw_log__", x)])
                evs.append((T0 + i, None, kv))
    elif name == "c3_java":
        buf, _, _ = synth.java_stack_records(600, seed=seed)
        raw = bytes(buf)
        recs, i = [], 0
        while len(b"".join(recs)) < GROUP_BYTES:
            j = raw.find(b"\n[", i)
            recs.append(raw[i:j if j >= 0 else len(raw)])
            if j < 0:
                break
            i = j + 1
        evs = [(T0 + i, None, [(b"content", r)]) for i, r in enumerate(recs)]
    elif name == "c4_csv":
        buf, off, ln = synth.csv_lines(GROUP_BYTES // 100, seed=seed)
        evs = [(T0 + i, None, [(b"content", x)]) for i, x in enumerate(_lines(buf, off, ln, GROUP_BYTES))]
    else:
        buf, off, ln = synth.newline_lines(GROUP_BYTES // 512 + 1, seed=seed)
        evs = [(T0 + i, None, [(b"content", x)]) for i, x in enumerate(_lines(buf, off, ln, GROUP_BYTES))]
    return O.sls_serialize_logs(evs, False)[0]


def edge_segments():
    """The edge-case matrix: (name, bytes)."""
    rng = random.Random(7)
    rb = lambda n: bytes(rng.getrandbits(8) for _ in range(n))  # noqa: E731
    segs = [("len%d" % n, rb(n)) for n in range(0, 301)]
    segs += [("text%d" % n, (b"the quick brown fox " * 20)[:n]) for n in range(0, 64)]
    for c in (65536, 2 * 65536):
        for d in (-33, -13, -12, -5, -4, -1, 0, 1, 4, 5, 12, 13, 33):
            segs.append(("chunk%d%+d" % (c, d), (b"abcdefgh" * (c // 4))[:c + d] if d % 2 else rb(c + d)))
    for n in (1, 4, 5, 12, 13, 14, 16, 17, 19, 20, 100, 65535, 65536, 65537, 300000):
        segs.append(("run%d" % n, b"z" * n))
    # a random block repeated at distance 65535 (usable) and at 65536 (must not be used); the zeros between the copies
    # hash to one table entry, so the first copy's positions stay in the table
    blk = rb(300)
    for dist in (65535, 65536):
        segs.append(("dist%d" % dist, blk + bytes(dist - len(blk)) + blk + rb(40)))
    # literal and match lengths at 14/15/16 and 15 + 255k +- 1
    pat = rb(2000)
    # ("lit": the run before the second copy of pat[:8] is 8 + (L - 8) bytes; "match": the match-length field is L)
    for L in (14, 15, 16, 269, 270, 271, 524, 525, 526, 1289):
        segs.append(("lit%d" % L, pat[:8] + rb(L - 8) + pat[:8] + rb(L - 8) + rb(20)))
        segs.append(("match%d" % L, pat[:L + 4] + rb(7) + pat[:L + 4] + rb(20)))
    # matches that cross chunk boundaries: a text that repeats with a period of 10000
    segs.append(("cross", (rb(10000) * 30)[:300007]))
    return segs


_LZ4 = None


def liblz4():
    """The system's liblz4 (ctypes), or None."""
    global _LZ4
    if _LZ4 is None:
        try:
            L = C.CDLL("liblz4.so.1")
        except OSError:
            _LZ4 = False
            return None
        L.LZ4_compress_default.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
        L.LZ4_decompress_safe.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int]
        _LZ4 = L
    return _LZ4 or None


def lz4_compress(data: bytes) -> bytes:
    L = liblz4()
    cap = len(data) + len(data) // 255 + 16
    out = C.create_string_buffer(cap)
    n = L.LZ4_compress_default(data, out, len(data), cap)
    assert n > 0
    return out.raw[:n]


def lz4_decompress(blk: bytes, raw_size: int) -> bytes:
    L = liblz4()
    out = C.create_string_buffer(max(raw_size, 1))
    n = L.LZ4_decompress_safe(blk, out, len(blk), raw_size)
    assert n == raw_size, "liblz4 rejected the block (%d)" % n
    return out.raw[:n]
