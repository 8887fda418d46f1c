"""ctypes wrapper of the TEST-ONLY host build of the JSON parse (tests/emul/lc_json_emul.cpp).  It takes an event
table (ev_len 0xFFFFFFFF = no SourceKey) and returns what lc_json_parse returns, plus the slow-event count."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_json_emul.so")
        srcs = [os.path.join(_HERE, "lc_json_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emul_json_parse.argtypes = [C.c_char_p, u32, vp, vp, vp, u64, u32, vp, vp, vp, u64, vp, vp, u64, vp, vp,
                                      vp]
        L.emul_json_parse.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def parse(source_key, base, off, ln, W=32):
    """(status, first, entries [m, 4], arena bytes, counters, n_slow); raises on an emit-range error"""
    if isinstance(source_key, str):
        source_key = source_key.encode()
    off = np.ascontiguousarray(off, np.uint32)
    ln = np.ascontiguousarray(ln, np.uint32)
    n = off.size
    st, first, cnt = np.zeros(n, np.uint8), np.zeros(n + 1, np.uint64), np.zeros(3, np.uint64)
    m, a, ns = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    b = base if base.size else np.zeros(1, np.uint8)

    def call(ent, ecap, ar, acap):
        return lib().emul_json_parse(source_key, len(source_key), _p(b), _p(off), _p(ln), n, W, _p(st), _p(first),
                                     _p(ent), ecap, _p(m), _p(ar), acap, _p(a), _p(cnt), _p(ns))
    call(np.zeros((1, 4), np.uint32), 0, np.zeros(1, np.uint8), 0)
    ent = np.zeros((max(int(m[0]), 1), 4), np.uint32)
    ar = np.zeros(max(int(a[0]), 1), np.uint8)
    rc = call(ent, int(m[0]), ar, int(a[0]))
    if rc:
        raise RuntimeError("emit pass left its range (%d)" % rc)
    return st, first, ent[:int(m[0])], ar[:int(a[0])].tobytes(), cnt, int(ns[0])
