"""ctypes wrapper of the TEST-ONLY host build of the split -> delimiter chain's serialiser
(tests/emul/lc_split_delim_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_split_delim_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_delim_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, ci, cs = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_char_p
        L.emul_split_delim_sls.restype = C.c_int64
        L.emul_split_delim_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, C.c_uint8, ci, ci, vp,
                                           vp, u32, cs, u32, cs, u32, ci, ci, ci, cs, u32, u64, u32, u32, u32, vp,
                                           u64, vp, cs, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def serialize(val, off, ln, tables, max_fields, sep: bytes, quote: int, treatment: str, keys, source_key,
              renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, nlanes=1,
              raw_args=None):
    """tables = (status, nfields, f_off, f_len, f_dq) of the delimiter stage over the pieces (off, ln) of val;
    treatment: extend / keep / discard; offset_key None = no log.file.offset metadata; time_ns None = no Time_ns.
    Returns (the `Logs` bytes of the pieces the chain leaves behind, counters[4] = successful, failed, discarded,
    blank).  raw_args: overrides of the C arguments by position, to exercise the refusals."""
    pad = 16
    a = np.zeros(len(val) + 2 * pad, np.uint8)
    a[pad:pad + len(val)] = np.frombuffer(bytes(val), np.uint8)
    off = np.ascontiguousarray(off, np.uint32) + np.uint32(pad)
    ln = np.ascontiguousarray(ln, np.uint32)
    st = np.ascontiguousarray(tables[0], np.uint8)
    nf, fl, fd = (np.ascontiguousarray(x, np.uint32) for x in (tables[1], tables[3], tables[4]))
    fo = np.ascontiguousarray(tables[2], np.uint32) + np.uint32(pad)
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x is not None else None  # noqa: E731
    karr = (C.c_char_p * max(len(keys), 1))(*keys)
    kl = np.array([len(k) for k in keys] or [0], np.uint32)
    sp = np.frombuffer(sep, np.uint8)
    err = C.create_string_buffer(256)
    # the pieces' file offsets are relative to the unpadded value
    args = [p(a), p(off), p(ln), off.size, p(st), p(nf), p(fo), p(fl), p(fd), max_fields, p(sp), len(sep), quote,
            int(treatment == "extend"), int(treatment == "discard"), C.cast(karr, C.c_void_p), p(kl), len(keys),
            source_key, len(source_key), renamed_key, len(renamed_key), int(keep_fail), int(keep_succeed),
            int(copy_raw), offset_key, len(offset_key) if offset_key is not None else 0, (src_pos - pad) % (1 << 64),
            time & 0xFFFFFFFF, 0xFFFFFFFF if time_ns is None else time_ns, nlanes]
    for k, v in (raw_args or {}).items():
        args[k] = v
    ctr = np.zeros(4, np.uint64)
    total = lib().emul_split_delim_sls(*args, None, 0, p(ctr), err, 256)
    if total == -1:
        raise Refused(err.value.decode())
    out = np.zeros(max(int(total), 1), np.uint8)
    ctr[:] = 0
    got = lib().emul_split_delim_sls(*args, p(out), int(total), p(ctr), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total]), [int(x) for x in ctr]
