"""Inputs and references of the zstd tests: the edge matrix beyond tests/lz4_cases.py's, and the system's libzstd (not
vendored) as the second decoder and the ratio reference."""
import ctypes as C
import random

BLOCK = 128 << 10

_ZSTD = None


def libzstd():
    """The system's libzstd (ctypes), or None."""
    global _ZSTD
    if _ZSTD is None:
        try:
            L = C.CDLL("libzstd.so.1")
        except OSError:
            _ZSTD = False
            return None
        L.ZSTD_compress.restype = C.c_size_t
        L.ZSTD_compress.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int]
        L.ZSTD_decompress.restype = C.c_size_t
        L.ZSTD_decompress.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
        L.ZSTD_isError.argtypes = [C.c_size_t]
        L.ZSTD_getErrorName.restype = C.c_char_p
        L.ZSTD_getErrorName.argtypes = [C.c_size_t]
        L.ZSTD_getFrameContentSize.restype = C.c_ulonglong
        L.ZSTD_getFrameContentSize.argtypes = [C.c_char_p, C.c_size_t]
        L.ZSTD_versionNumber.restype = C.c_uint
        _ZSTD = L
    return _ZSTD or None


def zstd_compress(data: bytes, level=1) -> bytes:
    L = libzstd()
    cap = bound(len(data))
    out = C.create_string_buffer(max(cap, 1))
    n = L.ZSTD_compress(out, cap, data, len(data), level)
    assert not L.ZSTD_isError(n)
    return out.raw[:n]


def zstd_decompress(frame: bytes, raw_size: int) -> bytes:
    """ZSTD_decompress, after checking ZSTD_getFrameContentSize == raw_size"""
    L = libzstd()
    assert L.ZSTD_getFrameContentSize(frame, len(frame)) == raw_size
    out = C.create_string_buffer(max(raw_size, 1))
    n = L.ZSTD_decompress(out, max(raw_size, 1), frame, len(frame))
    assert not L.ZSTD_isError(n), "libzstd rejected the frame: %s" % L.ZSTD_getErrorName(n).decode()
    assert n == raw_size
    return out.raw[:n]


def bound(n):
    """ZSTD_compressBound"""
    return n + (n >> 8) + (((128 << 10) - n) >> 11 if n < (128 << 10) else 0)


def block_segments():
    """Segments around the block size, one-byte runs, skewed wire-like bytes and literal runs across blocks:
    (name, bytes)."""
    rng = random.Random(11)
    text = b"".join(b"k%03d=v%05d;" % (rng.randrange(40), rng.randrange(99999)) for _ in range(60000))
    segs = []
    for m in (1, 2, 3):
        for d in range(-16, 17):
            n = m * BLOCK + d
            segs.append(("block%d%+d" % (m, d), text[:n] if d % 2 else rng.randbytes(n) if m == 1 else text[:n]))
    segs.append(("byte", b"x"))
    segs.append(("run1m", b"q" * (1 << 20)))
    # wire-like bytes: a skewed alphabet with bytes >= 0x80 (varints, tags)
    alpha = bytes(range(0x20, 0x7F)) + bytes(range(0x80, 0x100, 3))
    w = [200 if c < 0x7F else 3 for c in alpha]
    segs.append(("skewed", bytes(rng.choices(alpha, w, k=300000))))
    segs.append(("high", bytes(rng.choices(range(0x80, 0x100), [1 + (i % 7) ** 3 for i in range(128)], k=200000))))
    # a literal run that spans block boundaries between two compressible stretches
    segs.append(("span", text[:100000] + rng.randbytes(200000) + text[:100000]))
    return segs
