"""ctypes wrapper of the TEST-ONLY host build of the split-fed SLS serialiser (tests/emul/lc_split_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_split_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.emul_split_sls.restype = C.c_int64
        L.emul_split_sls.argtypes = [vp, u64, vp, vp, u64, C.c_char_p, u32, C.c_char_p, u32, u64, u32, u32, u64, u32,
                                     vp, u64, vp]
        _LIB = L
    return _LIB


def serialize(src: bytes, off, ln, key: bytes, offset_key, src_pos, time, ns=None, tile=0, nlanes=1, src_align=0,
              out_align=0):
    """The `Logs` bytes of the pieces (off, ln) of src: key -> piece, plus offset_key -> decimal(src_pos + off) when
    offset_key is not None (replacing the piece when it equals key).  src / out start src_align / out_align bytes past
    a 16-byte boundary; the output is written in tiles of `tile` bytes (0 = one tile) by `nlanes` emulated lanes."""
    a = np.zeros(len(src) + 32, np.uint8)
    base = (-a.ctypes.data) % 16 + src_align
    a = a[base:base + len(src)] if len(src) else a[base:base + 1]
    a[:len(src)] = np.frombuffer(src, np.uint8)
    off = np.ascontiguousarray(off, np.uint32)
    ln = np.ascontiguousarray(ln, np.uint32)
    n = off.size
    rec = np.zeros(max(n, 1), np.uint64)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    nsv = 0xFFFFFFFF if ns is None else int(ns)
    args = [p(a), len(src), p(off), p(ln), n, key, len(key), offset_key, len(offset_key or b""), int(src_pos),
            int(time) & 0xFFFFFFFF, nsv, int(tile), int(nlanes)]
    total = int(lib().emul_split_sls(*args, None, 0, p(rec)))
    buf = np.full(total + 64, 0xA5, np.uint8)
    o = (-buf.ctypes.data) % 16 + out_align
    out = buf[o:o + total + 16]
    got = int(lib().emul_split_sls(*args, p(out), total, p(rec)))
    assert got == total
    assert (out[total:] == 0xA5).all(), "wrote past the end of the output"
    return bytes(out[:total])
