"""ctypes wrapper of the TEST-ONLY host build of the delimiter -> regex -> SLS chain
(tests/emul/lc_delim_regex_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_delim_regex_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_delim_regex_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        cfg = [vp, u32, C.c_uint8, i32, i32, vp, vp, u32, C.c_char_p, u32, C.c_char_p, u32, i32, i32, i32,  # delimiter
               vp, vp, u32, C.c_char_p, u32, C.c_char_p, u32, i32, i32, i32, i32, u32]  # regex stage
        tables = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u32]
        L.emul_delim_regex_tap.restype = C.c_int64
        L.emul_delim_regex_tap.argtypes = tables + cfg + [u32, vp, vp, C.c_char_p, u32]
        L.emul_delim_regex_sls.restype = C.c_int64
        L.emul_delim_regex_sls.argtypes = tables + cfg + [vp, vp, vp, vp, vp, vp, vp, u32, vp, u64, vp, C.c_char_p,
                                                          u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def _p(x):
    return x.ctypes.data_as(C.c_void_p) if x is not None else None


def _keys(keys):
    arr = (C.c_char_p * max(len(keys), 1))(*keys)
    return arr, np.array([len(k) for k in keys] or [0], np.uint32)


def serialize(buf, ev_off, ev_len, dcfg, rcfg, times, nss=None, nlanes=1):
    """dcfg: a tests.delim_sls_cases configuration; rcfg: a tests.regex_sls_cases configuration whose "source" is one of
    dcfg's keys.  Returns (Logs bytes, counters[8], value table (off, len), side bytes) of the chain, the regex stage
    run by the oracle's matcher over the tapped values."""
    pad = 16
    n = len(ev_off)
    side_cap = int(np.asarray(ev_len, np.uint64).sum())
    side_at = (pad + len(buf) + 15) // 16 * 16
    a = np.zeros(side_at + side_cap + 2 * pad, np.uint8)
    a[pad:pad + len(buf)] = np.frombuffer(bytes(buf), np.uint8)
    off = np.ascontiguousarray(ev_off, np.uint32) + pad
    ln = np.ascontiguousarray(ev_len, np.uint32)
    quote = dcfg["quote"] if len(dcfg["sep"]) == 1 else ord('"')
    st, nf, fo, fl, fd = orc.delim_parse_batch(buf, ev_off, ev_len, dcfg["sep"], quote, len(dcfg["keys"]),
                                               dcfg["treatment"] == "extend", dcfg["allow_short"], dcfg["max_fields"])
    fo = np.ascontiguousarray(fo, np.uint32) + np.uint32(pad)
    whole = rcfg["regex"] == "(.*)"
    rx = None if whole else orc.Regex(rcfg["regex"])
    pitch = 0 if whole else rx.ngroups
    dk, dkl = _keys([k.encode() for k in dcfg["keys"]])
    rk, rkl = _keys([k.encode() for k in rcfg["keys"]])
    dsrc, dren = dcfg["source"].encode(), (dcfg["renamed"] or dcfg["source"]).encode()
    rsrc, rren = rcfg["source"].encode(), (rcfg["renamed"] or rcfg["source"]).encode()
    sp = np.frombuffer(dcfg["sep"], np.uint8)
    tables = [_p(a), _p(off), _p(ln), n, _p(st), _p(nf), _p(fo), _p(np.ascontiguousarray(fl, np.uint32)),
              _p(np.ascontiguousarray(fd, np.uint32)), dcfg["max_fields"]]
    cfg = [_p(sp), len(dcfg["sep"]), quote, int(dcfg["treatment"] == "extend"), int(dcfg["treatment"] == "discard"),
           C.cast(dk, C.c_void_p), _p(dkl), len(dcfg["keys"]), dsrc, len(dsrc), dren, len(dren),
           int(dcfg["keep_fail"]), int(dcfg["keep_succeed"]), int(dcfg["copy_raw"]),
           C.cast(rk, C.c_void_p), _p(rkl), len(rcfg["keys"]), rsrc, len(rsrc), rren, len(rren),
           int(rcfg["keep_fail"]), int(rcfg["keep_succeed"]), int(rcfg["copy_raw"]), int(whole), pitch]
    err = C.create_string_buffer(256)
    vo, vl = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    side = lib().emul_delim_regex_tap(*tables, *cfg, side_at, _p(vo), _p(vl), err, 256)
    if side == -1:
        raise Refused(err.value.decode())
    assert 0 <= side <= side_cap
    rs = co = cl = None
    if not whole:
        rs, co, cl = orc.regex_parse_batch(rx, a, vo[:n], vl[:n], len(rcfg["keys"]))
        co = np.ascontiguousarray(co, np.uint32)
        cl = np.ascontiguousarray(cl, np.uint32)
    t = np.ascontiguousarray(times, np.uint32)
    ns = np.ascontiguousarray(nss, np.uint32) if nss is not None else None
    ctr = np.zeros(8, np.uint64)
    rest = [_p(vo), _p(vl), _p(rs), _p(co), _p(cl), _p(t), _p(ns), nlanes]
    total = lib().emul_delim_regex_sls(*tables, *cfg, *rest, None, 0, _p(ctr), err, 256)
    assert total >= 0, total
    out = np.zeros(max(int(total), 1), np.uint8)
    got = lib().emul_delim_regex_sls(*tables, *cfg, *rest, _p(out), int(total), _p(ctr), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total]), ctr, (vo[:n] - pad, vl[:n]), bytes(a[side_at:side_at + side])
