"""ctypes wrapper of the TEST-ONLY host build of the timestamp parse (tests/emul/lc_timestamp_emul.cpp), plus the
event-table layout the tests, the GPU calls and the oracles share."""
import ctypes as C
import os
import subprocess
import time

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
NO_KEY = 0xFFFFFFFF


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_timestamp_emul.so")
        srcs = [os.path.join(_HERE, "lc_timestamp_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u64, i64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_int32, C.c_uint32
        L.emul_ts_compile.restype = C.c_int
        L.emul_ts_compile.argtypes = [C.c_char_p, u64, i32, i32, vp, C.c_char_p]
        L.emul_ts_conf_size.restype = u64
        L.emul_ts_parse.argtypes = [vp, vp, vp, vp, u64, vp, u64, i64, vp, i32, u32, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def layout(groups):
    """groups: list of lists of values (bytes, or None for an event without SourceKey).  Returns (base, off, len, grp):
    the values back to back, the last one ending exactly at the end of base."""
    vals = [v for g in groups for v in g]
    off = np.zeros(len(vals), np.uint32)
    ln = np.full(len(vals), NO_KEY, np.uint32)
    parts, pos = [], 0
    for i, v in enumerate(vals):
        if v is not None:
            off[i], ln[i] = pos, len(v)
            parts.append(v)
            pos += len(v)
    grp = np.zeros(len(groups) + 1, np.uint32)
    grp[1:] = np.cumsum([len(g) for g in groups])
    base = np.frombuffer(b"".join(parts), np.uint8) if parts else np.zeros(0, np.uint8)
    return np.ascontiguousarray(base), off, ln, grp


class Compiled:
    def __init__(self, fmt, source_year=-1, adjust=0):
        if isinstance(fmt, str):
            fmt = fmt.encode()
        self.conf = np.zeros(int(lib().emul_ts_conf_size()), np.uint8)
        err = C.create_string_buffer(256)
        self.ok = lib().emul_ts_compile(fmt, len(fmt), source_year, adjust, _p(self.conf), err) == 0
        self.error = err.value.decode()

    def parse(self, base, off, ln, grp, now, discard_interval=43200, W=32):
        n = off.size
        lt = time.localtime(now)
        now_tm = np.array([lt.tm_year - 1900, lt.tm_mon - 1, lt.tm_mday], np.int32)
        st, sec, ns = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint32)
        cnt = np.zeros(5, np.uint64)
        b = base if base.size else np.zeros(1, np.uint8)
        lib().emul_ts_parse(_p(self.conf), _p(b), _p(off), _p(ln), n, _p(grp), grp.size - 1, int(now), _p(now_tm),
                            int(discard_interval), W, _p(sec), _p(ns), _p(st), _p(cnt))
        return st, sec, ns, cnt
