"""ctypes wrapper of the TEST-ONLY host build of the zstd frame compressor (tests/emul/lc_zstd_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

BLOCK = 131072  # LC_ZSTD_BLOCK


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_zstd_emul.so")
        srcs = [os.path.join(_HERE, "lc_zstd_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.emul_zstd_compress.restype = C.c_int64
        L.emul_zstd_compress.argtypes = [vp, u64, vp, vp, u32, vp, u64, vp, vp]
        _LIB = L
    return _LIB


def compress(segments, nlanes=32):
    """One zstd frame per segment (a list of bytes), with `nlanes` emulated lanes per batch.  Returns the list of
    frames."""
    lens = np.array([len(s) for s in segments], np.uint32)
    offs = np.zeros(len(segments), np.uint64)
    if len(segments) > 1:
        offs[1:] = np.cumsum(lens[:-1].astype(np.uint64))
    data = np.frombuffer(b"".join(segments) + b"\0", np.uint8)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    n = max(len(segments), 1)
    foff, flen = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    total = int(lib().emul_zstd_compress(p(data), len(segments), p(offs), p(lens), nlanes, None, 0, p(foff), p(flen)))
    out = np.full(total + 64, 0xA5, np.uint8)
    got = int(lib().emul_zstd_compress(p(data), len(segments), p(offs), p(lens), nlanes, p(out), total, p(foff),
                                       p(flen)))
    assert got == total
    assert (out[total:] == 0xA5).all(), "wrote past the end of the output"
    return [bytes(out[int(o):int(o) + int(ln)]) for o, ln in zip(foff[:len(segments)], flen[:len(segments)])]
