"""ctypes wrapper of the TEST-ONLY host build of the split -> delimiter -> timestamp chain
(tests/emul/lc_split_delim_timestamp_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess
import time as _time

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_split_delim_timestamp_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_delim_timestamp_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, i32, i64, ci, cs = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_int, C.c_char_p
        L.emul_split_delim_ts_sls.restype = C.c_int64
        L.emul_split_delim_ts_sls.argtypes = [vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, C.c_uint8, ci,
                                              ci, vp, vp, u32, cs, u32, cs, u32, ci, ci, ci, cs, u32, u64, u32, u32,
                                              cs, u32, cs, u64, i32, i32, i64, vp, i32, ci, u32, vp, vp, vp, vp, vp,
                                              u64, vp, cs, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def serialize(val, off, ln, tables, max_fields, sep: bytes, quote: int, treatment: str, keys, source_key,
              renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, tkey, fmt, now,
              discard_interval=-1, enable_ns=False, source_year=-1, adjust=0, nlanes=1):
    """tables = (status, nfields, f_off, f_len, f_dq) of the delimiter stage over the pieces (off, ln) of val;
    treatment: extend / keep / discard; offset_key None = no log.file.offset metadata; time_ns None = no Time_ns.
    Returns (the `Logs` bytes, counters[9], the timestamp stage's status per piece, the tap's (off, len) table over
    val, the value buffer as long as val)."""
    pad = 16
    a = np.zeros(len(val) + 2 * pad, np.uint8)
    a[pad:pad + len(val)] = np.frombuffer(bytes(val), np.uint8)
    off = np.ascontiguousarray(off, np.uint32) + np.uint32(pad)
    ln = np.ascontiguousarray(ln, np.uint32)
    n = off.size
    st = np.ascontiguousarray(tables[0], np.uint8)
    nf, fl, fd = (np.ascontiguousarray(x, np.uint32) for x in (tables[1], tables[3], tables[4]))
    fo = np.ascontiguousarray(tables[2], np.uint32) + np.uint32(pad)
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x is not None else None  # noqa: E731
    karr = (C.c_char_p * max(len(keys), 1))(*keys)
    kl = np.array([len(k) for k in keys] or [0], np.uint32)
    sp = np.frombuffer(sep, np.uint8)
    if isinstance(fmt, str):
        fmt = fmt.encode()
    lt = _time.localtime(now)
    now_tm = np.array([lt.tm_year - 1900, lt.tm_mon - 1, lt.tm_mday], np.int32)
    err = C.create_string_buffer(256)
    voff, vlen = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32)
    vbuf = np.zeros(a.size, np.uint8)
    tst = np.zeros(max(n, 1), np.uint8)
    ctr = np.zeros(9, np.uint64)

    def call(out, cap):
        ctr[:] = 0
        # the pieces' file offsets are relative to the unpadded value
        return lib().emul_split_delim_ts_sls(
            p(a), a.size, p(off), p(ln), n, p(st), p(nf), p(fo), p(fl), p(fd), max_fields, p(sp), len(sep), quote,
            int(treatment == "extend"), int(treatment == "discard"), C.cast(karr, C.c_void_p), p(kl), len(keys),
            source_key, len(source_key), renamed_key, len(renamed_key), int(keep_fail), int(keep_succeed),
            int(copy_raw), offset_key, len(offset_key) if offset_key is not None else 0, (src_pos - pad) % (1 << 64),
            time & 0xFFFFFFFF, 0xFFFFFFFF if time_ns is None else time_ns, tkey, len(tkey), fmt, len(fmt),
            source_year, adjust, int(now), p(now_tm), int(discard_interval), int(bool(enable_ns)), nlanes, p(voff),
            p(vlen), p(vbuf), p(tst), p(out), cap, p(ctr), err, 256)

    total = call(None, 0)
    if total == -1:
        raise Refused(err.value.decode())
    out = np.zeros(max(int(total), 1), np.uint8)
    got = call(out, int(total))
    assert got == total, (got, total)
    vo = voff[:n].astype(np.int64) - pad
    return (bytes(out[:total]), [int(x) for x in ctr], tst[:n].copy(), (vo, vlen[:n].copy()),
            bytes(vbuf[pad:pad + len(val)]))
