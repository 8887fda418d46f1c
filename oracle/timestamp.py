"""ctypes wrappers of the two CPU oracles of ProcessorParseTimestampNative: the flat C restatement
(oracle/lc_timestamp_oracle.c, built here on first use) and, where oracle/build_ref_strptime.sh could build it, the
reference's own strptime_ns behind oracle/ref_strptime_driver.cpp (oracle/_ref/libref_strptime.so).  Both take the
event tables of tests/emul/timestamp.layout and return (status, sec, nsec, counters)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libref_strptime.so")
_LIBS = {}


def _load(which):
    if which not in _LIBS:
        if which == "ref":
            L = C.CDLL(REF_SO)
            fn = L.ref_ts_process
        else:
            so = os.path.join(_HERE, "liblc_timestamp_oracle.so")
            src = os.path.join(_HERE, "lc_timestamp_oracle.c")
            if not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
                subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-std=c11", "-o", so, src])
            L = C.CDLL(so)
            fn = L.orc_ts_process
        vp = C.c_void_p
        fn.argtypes = [C.c_char_p, C.c_int32, C.c_int32, vp, vp, vp, vp, C.c_uint64, C.c_int64, C.c_int32, vp, vp, vp,
                       vp]
        _LIBS[which] = (L, fn)
    return _LIBS[which][1]


def have_reference():
    return os.path.exists(REF_SO)


def process(fmt, source_year, adjust, base, off, ln, grp, now, discard_interval=43200, which="c"):
    if isinstance(fmt, str):
        fmt = fmt.encode()
    n = off.size
    st, sec, ns = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint32)
    cnt = np.zeros(5, np.uint64)
    b = base if base.size else np.zeros(1, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    _load(which)(fmt, source_year, adjust, p(b), p(off), p(ln), p(grp), grp.size - 1, int(now), int(discard_interval),
                 p(sec), p(ns), p(st), p(cnt))
    return st, sec, ns, cnt
