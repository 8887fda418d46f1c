"""CPU oracle of ProcessorParseApsaraNative: a ctypes wrapper of the flat C restatement (oracle/lc_apsara_oracle.c,
built here on first use) over the event tables of tests/emul/timestamp.layout, and a group-level
ProcessorParseApsaraNative on oracle.oracle's Event / Group / CommonParserOptions (ProcessorParseApsaraNative.cpp:
37-241, AddLog 465-473: every field is appended, never de-duplicated)."""
import ctypes as C
import os
import subprocess
import time

import numpy as np

from oracle.oracle import LOG, CommonParserOptions, Group, _b

_HERE = os.path.dirname(os.path.abspath(__file__))
_FN = None
NO_KEY = 0xFFFFFFFF
BASE_KEYS = (b"__LEVEL__", b"__THREAD__", b"__FILE__", b"__LINE__")
OK, NOT_FOUND, EMPTY, FAILED, DISCARDED, OVERWRITTEN = 0, 1, 2, 3, 4, 0x80


def _load():
    global _FN
    if _FN is None:
        so = os.path.join(_HERE, "liblc_apsara_oracle.so")
        srcs = [os.path.join(_HERE, "lc_apsara_oracle.c"), os.path.join(_HERE, "lc_timestamp_oracle.c")]
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-std=c11", "-o", so, srcs[0]])
        fn = C.CDLL(so).orc_apsara_process
        vp, u64, i64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_int32, C.c_uint32
        fn.argtypes = [i32, C.c_char_p, u32, vp, u64, vp, vp, vp, u64, i64, i32, vp, vp, vp, vp, vp, vp, u64, vp, vp]
        _FN = fn
    return _FN


def process(source_key, adjust, base, off, ln, grp, now, discard_interval=-1):
    """(status, sec, nsec, micro, first, entries [m, 4], counters), as lc_apsara_parse returns them"""
    source_key = _b(source_key)
    n = off.size
    st, sec, ns, us = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint32), np.zeros(n, np.int64)
    first, cnt, m = np.zeros(n + 1, np.uint64), np.zeros(5, np.uint64), np.zeros(1, np.uint64)
    b = base if base.size else np.zeros(1, np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731

    def call(ent, cap):
        cnt[:] = 0
        _load()(int(adjust), source_key, len(source_key), p(b), base.size, p(off), p(ln), p(grp), grp.size - 1,
                int(now), int(discard_interval), p(st), p(sec), p(ns), p(us), p(first), p(ent), cap, p(m), p(cnt))
    call(np.zeros((1, 4), np.uint32), 0)
    ent = np.zeros((max(int(m[0]), 1), 4), np.uint32)
    call(ent, int(m[0]))
    return st, sec, ns, us, first, ent[:int(m[0])], cnt


def tz_offset(tz):
    """ParseTimeZoneOffsetSecond (TimeUtil.cpp:372-391): "GMT+hh:mm" -> seconds east, None when not valid"""
    if not isinstance(tz, str) or len(tz) != 9 or tz[:3] != "GMT" or tz[3] not in "+-" or tz[6] != ":" or \
            not (tz[4:6].isdigit() and tz[7:9].isdigit()):
        return None
    sec = int(tz[4:6]) * 3600 + int(tz[7:9]) * 60
    return -sec if tz[3] == "-" else sec


class ProcessorParseApsaraNative:
    name = "processor_parse_apsara_native"

    def __init__(self, cfg, discard_interval=-1):
        """discard_interval: ilogtail_discard_interval with ilogtail_discard_old_data on, -1 with it off"""
        if not isinstance(cfg.get("SourceKey"), str):
            raise ValueError("mandatory string param SourceKey")
        self.source_key = _b(cfg["SourceKey"])
        tz = cfg.get("Timezone", "")
        off = tz_offset(tz) if tz else None
        self.adjust = off - time.localtime().tm_gmtoff if off is not None else 0
        self.common = CommonParserOptions(cfg)
        self.discard_interval = discard_interval
        self.counters = {"discarded": 0, "out_failed": 0, "out_key_not_found": 0, "out_successful": 0,
                         "history_failure": 0}

    def process(self, g: Group, now=None):
        self.process_groups([g], now)

    def process_groups(self, groups, now=None):
        now = int(time.time()) if now is None else now
        vals, grp = [], [0]
        for g in groups:
            for e in g.events:
                vals.append(e.get(self.source_key) if e.type == LOG and e.has(self.source_key) else None)
            grp.append(len(vals))
        parts, off, ln, pos = [], np.zeros(len(vals), np.uint32), np.full(len(vals), NO_KEY, np.uint32), 0
        for i, v in enumerate(vals):
            if v is not None:
                off[i], ln[i] = pos, len(v)
                parts.append(v)
                pos += len(v)
        raw = b"".join(parts)
        base = np.frombuffer(raw, np.uint8) if raw else np.zeros(0, np.uint8)
        st, sec, ns, us, first, ent, cnt = process(self.source_key, self.adjust, base, off, ln,
                                                   np.array(grp, np.uint32), now, self.discard_interval)
        c = self.counters
        i = 0
        for g in groups:
            out = []
            for e in g.events:
                s = int(st[i]) & 7
                if e.type != LOG:
                    c["out_failed"] += 1
                elif s == NOT_FOUND:
                    c["out_key_not_found"] += 1
                elif s == EMPTY:
                    c["out_failed"] += 1
                elif s == DISCARDED:
                    c["history_failure"] += 1
                    c["discarded"] += 1
                    i += 1
                    continue
                elif s == FAILED:
                    c["out_failed"] += 1
                    v = vals[i]
                    e.delete(self.source_key)
                    if self.common.should_add_source(False) and not e.has(self.common.renamed):
                        e.contents.append([self.common.renamed, v, True])
                    if self.common.should_add_legacy_raw(False) and not e.has(self.common.legacy_raw_key):
                        e.contents.append([self.common.legacy_raw_key, v, True])
                    if self.common.should_erase(False, e, g.metadata):
                        c["discarded"] += 1
                        i += 1
                        continue
                else:
                    v = vals[i]
                    e.timestamp, e.ns = int(sec[i]), int(ns[i])
                    for ko, kl, vo, vl in ent[int(first[i]):int(first[i + 1])].tolist():
                        key = BASE_KEYS[ko - 0xFFFFFFF0] if ko >= 0xFFFFFFF0 else raw[ko:ko + kl]
                        e.contents.append([key, raw[vo:vo + vl], True])
                    e.contents.append([b"microtime", b"%d" % int(us[i]), True])
                    if not int(st[i]) & OVERWRITTEN:
                        e.delete(self.source_key)
                    if self.common.should_add_source(True) and not e.has(self.common.renamed):
                        e.contents.append([self.common.renamed, v, True])
                    c["out_successful"] += 1
                out.append(e)
                i += 1
            g.events = out
