"""ctypes wrapper of the TEST-ONLY host build of the Apsara parse (tests/emul/lc_apsara_emul.cpp).  It takes the
event tables of tests/emul/timestamp.layout and returns what lc_apsara_parse returns."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_apsara_emul.so")
        srcs = [os.path.join(_HERE, "lc_apsara_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u64, i64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_int32, C.c_uint32
        L.emul_apsara_parse.argtypes = [i32, C.c_char_p, u32, vp, u64, vp, vp, u64, vp, u64, i64, i32, u32, vp, vp,
                                        vp, vp, vp, vp, u64, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def parse(source_key, adjust, base, off, ln, grp, now, discard_interval=-1, W=32):
    """(status, sec, nsec, micro, first, entries [m, 4], counters)"""
    if isinstance(source_key, str):
        source_key = source_key.encode()
    n = off.size
    st, sec, ns, us = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint32), np.zeros(n, np.int64)
    first, cnt, m = np.zeros(n + 1, np.uint64), np.zeros(5, np.uint64), np.zeros(1, np.uint64)
    b = base if base.size else np.zeros(1, np.uint8)
    args = lambda ent, cap: (int(adjust), source_key, len(source_key), _p(b), base.size, _p(off), _p(ln), n,  # noqa
                             _p(grp), grp.size - 1, int(now), int(discard_interval), W, _p(st), _p(sec), _p(ns),
                             _p(us), _p(first), _p(ent), cap, _p(m), _p(cnt))
    ent = np.zeros((1, 4), np.uint32)
    lib().emul_apsara_parse(*args(ent, 0))
    ent = np.zeros((max(int(m[0]), 1), 4), np.uint32)
    lib().emul_apsara_parse(*args(ent, int(m[0])))
    return st, sec, ns, us, first, ent[:int(m[0])], cnt
