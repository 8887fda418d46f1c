"""CPU oracle of ProcessorParseJsonNative: a ctypes wrapper of the flat C restatement (oracle/lc_json_oracle.c, built
here on first use) over an event table (ev_len 0xFFFFFFFF = no SourceKey), and a group-level
ProcessorParseJsonNative on oracle.oracle's Event / Group / CommonParserOptions (ProcessorParseJsonNative.cpp:
ProcessEvent; the members are applied with overwrite as AddLog(key, value, event) does, the source and __raw_log__
without)."""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle.oracle import LOG, CommonParserOptions, Group, _b

_HERE = os.path.dirname(os.path.abspath(__file__))
_FN = None
NO_KEY = 0xFFFFFFFF
ARENA = 0x80000000
OK, NOT_FOUND, EMPTY, FAILED, OVERWRITTEN = 0, 1, 2, 3, 0x80


def _load():
    global _FN
    if _FN is None:
        so = os.path.join(_HERE, "liblc_json_oracle.so")
        src = os.path.join(_HERE, "lc_json_oracle.c")
        if not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
            subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-std=c11", "-o", so, src, "-lm"])
        fn = C.CDLL(so).orc_json_process
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        fn.argtypes = [C.c_char_p, u32, vp, u64, vp, vp, u64, vp, vp, vp, u64, vp, vp, u64, vp, vp]
        _FN = fn
    return _FN


def process(source_key, base, off, ln):
    """(status, first, entries [m, 4], arena bytes, counters), as lc_json_parse returns them"""
    source_key = _b(source_key)
    off = np.ascontiguousarray(off, np.uint32)
    ln = np.ascontiguousarray(ln, np.uint32)
    n = off.size
    st, first, cnt = np.zeros(n, np.uint8), np.zeros(n + 1, np.uint64), np.zeros(3, np.uint64)
    m, a = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    b = base if base.size else np.zeros(1, np.uint8)
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731

    def call(ent, ecap, ar, acap):
        _load()(source_key, len(source_key), p(b), base.size, p(off), p(ln), n, p(st), p(first), p(ent), ecap, p(m),
                p(ar), acap, p(a), p(cnt))
    call(np.zeros((1, 4), np.uint32), 0, np.zeros(1, np.uint8), 0)
    ent = np.zeros((max(int(m[0]), 1), 4), np.uint32)
    ar = np.zeros(max(int(a[0]), 1), np.uint8)
    call(ent, int(m[0]), ar, int(a[0]))
    return st, first, ent[:int(m[0])], ar[:int(a[0])].tobytes(), cnt


def span(raw, arena, o, ln):
    """the bytes an entry offset names"""
    return arena[o & ~ARENA:(o & ~ARENA) + ln] if o & ARENA else raw[o:o + ln]


def table(values):
    """(base u8, off, len) of a list of values (None = no SourceKey), back to back"""
    off = np.zeros(len(values), np.uint32)
    ln = np.full(len(values), NO_KEY, np.uint32)
    parts, pos = [], 0
    for i, v in enumerate(values):
        if v is not None:
            off[i], ln[i] = pos, len(v)
            parts.append(v)
            pos += len(v)
    raw = b"".join(parts)
    return (np.frombuffer(raw, np.uint8) if raw else np.zeros(0, np.uint8)), off, ln


def members(values, source_key=b"content"):
    """per value: None when it does not parse (or has no key / is empty), else its [key, value] list"""
    base, off, ln = table(values)
    raw = base.tobytes()
    st, first, ent, arena, _ = process(source_key, base, off, ln)
    out = []
    for i in range(len(values)):
        if int(st[i]) & 0x7F != OK:
            out.append(None)
            continue
        out.append([(span(raw, arena, ko, kl), span(raw, arena, vo, vl))
                    for ko, kl, vo, vl in ent[int(first[i]):int(first[i + 1])].tolist()])
    return out


class ProcessorParseJsonNative:
    name = "processor_parse_json_native"

    def __init__(self, cfg):
        if not isinstance(cfg.get("SourceKey"), str):
            raise ValueError("mandatory string param SourceKey")
        self.source_key = _b(cfg["SourceKey"])
        self.common = CommonParserOptions(cfg)
        self.counters = {"discarded": 0, "out_failed": 0, "out_key_not_found": 0, "out_successful": 0}

    def process(self, g: Group):
        self.process_groups([g])

    def process_groups(self, groups):
        vals = [e.get(self.source_key) if e.type == LOG and e.has(self.source_key) else None
                for g in groups for e in g.events]
        base, off, ln = table(vals)
        raw = base.tobytes()
        st, first, ent, arena, _ = process(self.source_key, base, off, ln)
        c = self.counters
        i = 0
        for g in groups:
            out = []
            for e in g.events:
                s = int(st[i]) & 0x7F
                v = vals[i]
                if e.type != LOG:
                    c["out_failed"] += 1
                elif s == NOT_FOUND:
                    c["out_key_not_found"] += 1
                else:
                    ok = s == OK
                    if not ok and s == FAILED:
                        c["out_failed"] += 1
                    if ok:
                        for ko, kl, vo, vl in ent[int(first[i]):int(first[i + 1])].tolist():
                            e.set(span(raw, arena, ko, kl), span(raw, arena, vo, vl))
                    if not ok or not int(st[i]) & OVERWRITTEN:
                        e.delete(self.source_key)
                    if self.common.should_add_source(ok) and not e.has(self.common.renamed):
                        e.contents.append([self.common.renamed, v, True])
                    if self.common.should_add_legacy_raw(ok) and not e.has(self.common.legacy_raw_key):
                        e.contents.append([self.common.legacy_raw_key, v, True])
                    if self.common.should_erase(ok, e, g.metadata):
                        c["discarded"] += 1
                        i += 1
                        continue
                    c["out_successful"] += 1
                out.append(e)
                i += 1
            g.events = out
