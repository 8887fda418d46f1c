"""ctypes wrapper of the TEST-ONLY host build of the split -> delimiter -> regex -> SLS chain
(tests/emul/lc_split_delim_regex_sls_emul.cpp)."""
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
        so = os.path.join(_HERE, "liblc_split_delim_regex_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_delim_regex_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, i32, cs = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_char_p
        tables = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u32]
        cfg = [vp, u32, C.c_uint8, i32, i32, vp, vp, u32, cs, u32, cs, u32, i32, i32, i32,  # delimiter
               vp, vp, u32, cs, u32, cs, u32, i32, i32, i32, i32, u32,  # regex stage
               cs, u32, u64, u32, u32]  # offset content, time, ns
        L.emul_split_delim_regex_tap.restype = C.c_int64
        L.emul_split_delim_regex_tap.argtypes = tables + cfg + [u64, vp, vp, cs, u32]
        L.emul_split_delim_regex_sls.restype = C.c_int64
        L.emul_split_delim_regex_sls.argtypes = tables + cfg + [vp, vp, vp, vp, vp, u32, vp, u64, vp, cs, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def _p(x):
    return x.ctypes.data_as(C.c_void_p) if x is not None else None


def _keys(keys):
    arr = (C.c_char_p * max(len(keys), 1))(*keys)
    return arr, np.array([len(k) for k in keys] or [0], np.uint32)


def serialize(val, off, ln, tabs, dcfg, rcfg, offset_key, src_pos, time, time_ns, nlanes=1, raw_args=None):
    """The chain over the pieces (off, ln) of val and the delimiter tables tabs = (status, nfields, f_off, f_len, f_dq)
    over them: the tap, the oracle's matcher over the tapped values, then the serialiser.  dcfg: a
    tests.split_delim_sls_cases configuration; rcfg: a tests.regex_sls_cases configuration.  offset_key None = no
    log.file.offset metadata; time_ns None = no Time_ns.  Returns (Logs bytes, counters[8], value table (off, len),
    side bytes).  raw_args: overrides of the C arguments by position, to exercise the refusals."""
    pad = 16
    val = bytes(val)
    n = len(off)
    side_at = (pad + len(val) + 15) // 16 * 16
    a = np.zeros(side_at + len(val) + 2 * pad, np.uint8)
    a[pad:pad + len(val)] = np.frombuffer(val, np.uint8)
    po = np.ascontiguousarray(off, np.uint32) + np.uint32(pad)
    pl = np.ascontiguousarray(ln, np.uint32)
    st = np.ascontiguousarray(tabs[0], np.uint8)
    nf, fl, fd = (np.ascontiguousarray(x, np.uint32) for x in (tabs[1], tabs[3], tabs[4]))
    fo = np.ascontiguousarray(tabs[2], np.uint32) + np.uint32(pad)
    quote = dcfg["quote"] if len(dcfg["sep"]) == 1 else ord('"')
    whole = rcfg["regex"] == "(.*)"
    rx = None if whole else orc.Regex(rcfg["regex"])
    pitch = 0 if whole else rx.ngroups
    dk, dkl = _keys([k.encode() for k in dcfg["keys"]])
    rk, rkl = _keys([k.encode() for k in rcfg["keys"]])
    dsrc, dren = dcfg["source"].encode(), (dcfg["renamed"] or dcfg["source"]).encode()
    rsrc, rren = rcfg["source"].encode(), (rcfg["renamed"] or rcfg["source"]).encode()
    sp = np.frombuffer(dcfg["sep"], np.uint8)
    tables = [_p(a), _p(po), _p(pl), n, _p(st), _p(nf), _p(fo), _p(fl), _p(fd), dcfg["max_fields"]]
    # the pieces' file offsets are relative to the unpadded value
    cfg = [_p(sp), len(dcfg["sep"]), quote, int(dcfg["treatment"] == "extend"), int(dcfg["treatment"] == "discard"),
           C.cast(dk, C.c_void_p), _p(dkl), len(dcfg["keys"]), dsrc, len(dsrc), dren, len(dren),
           int(dcfg["keep_fail"]), int(dcfg["keep_succeed"]), int(dcfg["copy_raw"]),
           C.cast(rk, C.c_void_p), _p(rkl), len(rcfg["keys"]), rsrc, len(rsrc), rren, len(rren),
           int(rcfg["keep_fail"]), int(rcfg["keep_succeed"]), int(rcfg["copy_raw"]), int(whole), pitch,
           offset_key, len(offset_key) if offset_key is not None else 0, (src_pos - pad) % (1 << 64),
           time & 0xFFFFFFFF, 0xFFFFFFFF if time_ns is None else time_ns]
    for k, v in (raw_args or {}).items():
        cfg[k] = v
    err = C.create_string_buffer(256)
    vo, vl = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    side = lib().emul_split_delim_regex_tap(*tables, *cfg, side_at, _p(vo), _p(vl), err, 256)
    if side == -1:
        raise Refused(err.value.decode())
    assert 0 <= side <= len(val)
    rs = co = cl = None
    if not whole:
        rs, co, cl = orc.regex_parse_batch(rx, a, vo[:n], vl[:n], len(rcfg["keys"]))
        co = np.ascontiguousarray(co, np.uint32)
        cl = np.ascontiguousarray(cl, np.uint32)
    ctr = np.zeros(8, np.uint64)
    rest = [_p(vo), _p(vl), _p(rs), _p(co), _p(cl), nlanes]
    total = lib().emul_split_delim_regex_sls(*tables, *cfg, *rest, None, 0, _p(ctr), err, 256)
    assert total >= 0, total
    out = np.zeros(max(int(total), 1), np.uint8)
    got = lib().emul_split_delim_regex_sls(*tables, *cfg, *rest, _p(out), int(total), _p(ctr), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total]), ctr, (vo[:n] - pad, vl[:n]), bytes(a[side_at:side_at + side])
