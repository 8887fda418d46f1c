"""ctypes wrapper of the TEST-ONLY host build of the split -> Apsara chain: the Apsara passes over the pieces and the
row function (tests/emul/lc_split_apsara_sls_emul.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_split_apsara_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_apsara_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, i32, i64, ci, cs = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_int, C.c_char_p
        L.emul_split_apsara_sls.restype = C.c_int64
        L.emul_split_apsara_sls.argtypes = [vp, u64, vp, vp, u64, cs, u32, i32, i64, i32, u32, cs, u32, ci, ci, ci, cs,
                                            u32, u64, u32, u32, ci, u32, vp, u64, vp, cs, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def serialize(val, off, ln, source_key, adjust, now, discard_interval, renamed_key, keep_fail, keep_succeed,
              copy_raw, offset_key, src_pos, time, time_ns, enable_ns, nlanes=1, W=32):
    """The Apsara stage (SourceKey source_key, Timezone adjustment `adjust`, `now`, discard_interval -1 = no history
    discard; W emulated lanes) over the pieces (off, ln) of val with val as their base, then the row function.
    offset_key None = no log.file.offset metadata; time_ns None = no source Time_ns.  Returns (the `Logs` bytes of
    the pieces the chain leaves behind, counters[5] in lc_apsara_parse's order)."""
    a = np.frombuffer(bytes(val) or b"\0", np.uint8)
    off = np.ascontiguousarray(off, np.uint32)
    ln = np.ascontiguousarray(ln, np.uint32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    err = C.create_string_buffer(256)
    args = [p(a), len(val), p(off), p(ln), off.size, source_key, len(source_key), int(adjust), int(now),
            int(discard_interval), W, renamed_key, len(renamed_key), int(keep_fail), int(keep_succeed),
            int(copy_raw), offset_key, len(offset_key) if offset_key is not None else 0, src_pos, time & 0xFFFFFFFF,
            0xFFFFFFFF if time_ns is None else time_ns, int(enable_ns), nlanes]
    ctr = np.zeros(5, np.uint64)
    total = lib().emul_split_apsara_sls(*args, None, 0, p(ctr), err, 256)
    if total == -1:
        raise Refused(err.value.decode())
    out = np.zeros(max(int(total), 1), np.uint8)
    ctr[:] = 0
    got = lib().emul_split_apsara_sls(*args, p(out), int(total), p(ctr), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total]), [int(x) for x in ctr]
