"""ctypes wrapper of the TEST-ONLY host build of the delimiter-fed SLS serialiser (tests/emul/lc_delim_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_delim_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_delim_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.emul_delim_sls.restype = C.c_int64
        L.emul_delim_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, C.c_uint8, C.c_int, C.c_int,
                                     vp, vp, u32, C.c_char_p, u32, C.c_char_p, u32, C.c_int, C.c_int, C.c_int, vp, vp,
                                     u32, vp, u64, C.c_char_p, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def serialize(buf, ev_off, ev_len, tables, max_fields, sep: bytes, quote: int, treatment: str, keys, source_key,
              renamed_key, keep_fail, keep_succeed, copy_raw, times, nss=None, nlanes=1):
    """tables = (status, nfields, f_off, f_len, f_dq) of the delimiter stage; treatment: extend / keep / discard.
    Returns the `Logs` bytes of the events ProcessorParseDelimiterNative leaves behind (flat events in)."""
    pad = 16
    a = np.zeros(len(buf) + 2 * pad, np.uint8)
    a[pad:pad + len(buf)] = np.frombuffer(bytes(buf), np.uint8)
    off = np.ascontiguousarray(ev_off, np.uint32) + pad
    ln = np.ascontiguousarray(ev_len, np.uint32)
    st = np.ascontiguousarray(tables[0], np.uint8)
    nf, fl, fd = (np.ascontiguousarray(x, np.uint32) for x in (tables[1], tables[3], tables[4]))
    fo = np.ascontiguousarray(tables[2], np.uint32) + np.uint32(pad)
    n = off.size
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x is not None else None  # noqa: E731
    karr = (C.c_char_p * max(len(keys), 1))(*keys)
    kl = np.array([len(k) for k in keys] or [0], np.uint32)
    sp = np.frombuffer(sep, np.uint8)
    t = np.ascontiguousarray(times, np.uint32)
    ns = np.ascontiguousarray(nss, np.uint32) if nss is not None else None
    err = C.create_string_buffer(256)
    args = [p(a), p(off), p(ln), n, p(st), p(nf), p(fo), p(fl),
            p(fd), max_fields, p(sp), len(sep), quote, int(treatment == "extend"),
            int(treatment == "discard"), C.cast(karr, C.c_void_p), p(kl), len(keys), source_key, len(source_key),
            renamed_key, len(renamed_key), int(keep_fail), int(keep_succeed), int(copy_raw), p(t), p(ns), nlanes]
    total = lib().emul_delim_sls(*args, None, 0, err, 256)
    if total == -1:
        raise Refused(err.value.decode())
    out = np.zeros(max(int(total), 1), np.uint8)
    got = lib().emul_delim_sls(*args, p(out), int(total), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total])
