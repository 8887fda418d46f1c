"""ctypes wrapper of the TEST-ONLY host build of the split -> regex -> filter chain's serialiser
(tests/emul/lc_split_regex_filter_sls_emul.cpp).  The boolean match between its tap and its eval runs here, with the
oracle's regex, over exactly the values and digit scratch the tap wrote."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
DIGIT_PITCH = 20
SRC_DIGITS, SRC_ABSENT = 0xFFFFFFFE, 0xFFFFFFFD


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblc_split_regex_filter_sls_emul.so")
        srcs = [os.path.join(_HERE, "lc_split_regex_filter_sls_emul.cpp"),
                os.path.join(_HERE, "..", "..", "loongcollector_b200", "csrc", "lc_exec.cuh")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, srcs[0]])
        L = C.CDLL(so)
        vp, u32, u64, ci, cs = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_char_p
        chain = [vp, vp, u64, vp, vp, vp, u32, vp, vp, u32, cs, u32, cs, u32, ci, ci, ci, ci, cs, u32, u64, u32, u32,
                 u32, vp, vp, u32, vp]
        L.emul_filter_tap.restype = C.c_int
        L.emul_filter_tap.argtypes = chain + [vp, vp, vp, vp, cs, u32]
        L.emul_split_regex_filter_sls.restype = C.c_int64
        L.emul_split_regex_filter_sls.argtypes = [vp] + chain + [vp, u32, vp, u64, vp, cs, u32]
        _LIB = L
    return _LIB


class Refused(ValueError):
    pass


def serialize(val, off, ln, tables, pitch, keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw,
              whole_line, offset_key, src_pos, time, time_ns, leaves, prog, nlanes=1):
    """tables = (status, cap_off, cap_len) of the regex stage over the pieces (off, ln) of val, or None in whole-line
    mode; offset_key None = no log.file.offset metadata; time_ns None = no Time_ns.  leaves: [(key bytes, oracle
    Regex)]; prog: the postfix program (ints, LC_FILTER_* codes).  Returns (the `Logs` bytes of the pieces the chain
    keeps, counters[4] = successful, failed, discarded, removed by the filter)."""
    a = np.frombuffer(bytes(val) or b"\0", np.uint8)
    off = np.ascontiguousarray(off, np.uint32)
    ln = np.ascontiguousarray(ln, np.uint32)
    n = off.size
    p = lambda x: x.ctypes.data_as(C.c_void_p) if x is not None else None  # noqa: E731
    st = co = cl = None
    if tables is not None:
        st = np.ascontiguousarray(tables[0], np.uint8)
        co = np.ascontiguousarray(tables[1], np.uint32)
        cl = np.ascontiguousarray(tables[2], np.uint32)
    karr = (C.c_char_p * max(len(keys), 1))(*keys)
    kl = np.array([len(k) for k in keys] or [0], np.uint32)
    larr = (C.c_char_p * max(len(leaves), 1))(*[k for k, _ in leaves])
    ll = np.array([len(k) for k, _ in leaves] or [0], np.uint32)
    pr = np.array(list(prog) or [0], np.uint32)
    err = C.create_string_buffer(256)
    args = [p(off), p(ln), n, p(st), p(co), p(cl), pitch, C.cast(karr, C.c_void_p), p(kl), len(keys), source_key,
            len(source_key), renamed_key, len(renamed_key), int(keep_fail), int(keep_succeed), int(copy_raw),
            int(whole_line), offset_key, len(offset_key) if offset_key is not None else 0, src_pos,
            time & 0xFFFFFFFF, 0xFFFFFFFF if time_ns is None else time_ns, len(leaves), C.cast(larr, C.c_void_p),
            p(ll), len(prog), p(pr)]
    L = len(leaves)
    src = np.zeros(max(L * n, 1), np.uint32)
    voff = np.zeros(max(L * n, 1), np.uint32)
    vlen = np.zeros(max(L * n, 1), np.uint32)
    dig = np.zeros(max(n * DIGIT_PITCH, 1), np.uint8)
    if lib().emul_filter_tap(*args, p(src), p(voff), p(vlen), p(dig), err, 256) == -1:
        raise Refused(err.value.decode())
    vb, db = bytes(val), dig.tobytes()
    m = np.zeros(max(2 * L * n, 1), np.uint8)
    for lf in range(L):
        rx = leaves[lf][1]
        for i in range(n):
            k = lf * n + i
            s, o, vl = int(src[k]), int(voff[k]), int(vlen[k])
            if s == SRC_ABSENT:
                continue
            if s == SRC_DIGITS:
                m[(L + lf) * n + i] = rx.full_match(db[i * DIGIT_PITCH:i * DIGIT_PITCH + vl]) is not None
            else:
                m[k] = rx.full_match(vb[o:o + vl]) is not None
    ctr = np.zeros(4, np.uint64)
    total = lib().emul_split_regex_filter_sls(p(a), *args, p(m), nlanes, None, 0, p(ctr), err, 256)
    if total == -1:
        raise Refused(err.value.decode())
    out = np.zeros(max(int(total), 1), np.uint8)
    ctr[:] = 0
    got = lib().emul_split_regex_filter_sls(p(a), *args, p(m), nlanes, p(out), int(total), p(ctr), err, 256)
    assert got == total, (got, total)
    return bytes(out[:total]), [int(x) for x in ctr]
