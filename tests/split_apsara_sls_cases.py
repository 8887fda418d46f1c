"""Shared cases of the split -> Apsara -> SLS tests: the oracle's splitter over one flat source event, then
oracle/apsara.py's ProcessorParseApsaraNative with a fixed `now`, then sls_serialize_logs; the CommonParserOptions
matrix and Apsara lines built to hit the row rule's corners (duplicate keys, keys equal to the chain's own keys, the
time cache across failed and erased pieces, the history discard on both sides of its boundary)."""
import random
import time as _time

from oracle import apsara as oap
from oracle import oracle as orc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"
NOW = 1700000000 + 43200  # 2023-11-15 10:13:20 UTC
DI = 43200                # ilogtail_discard_interval's default
BOUNDARY = NOW - DI       # a time more than DI behind NOW is discarded
ML_START = r"\[\d{4}-.*"  # an Apsara record starts with "[YYYY-"
BIG_EPOCH = 10000000000000  # 14 digits: 10 of seconds, then the fraction


def config(source="content", renamed=None, keep_fail=False, keep_succeed=False, copy_raw=False, tz=None):
    cfg = {"SourceKey": source, "KeepingSourceWhenParseFail": keep_fail,
           "KeepingSourceWhenParseSucceed": keep_succeed, "CopingRawLog": copy_raw}
    if renamed is not None:
        cfg["RenamedSourceKey"] = renamed
    if tz is not None:
        cfg["Timezone"] = tz
    return cfg


def renamed_key(cfg):
    """the effective RenamedSourceKey (SourceKey when unset or empty)"""
    return (cfg.get("RenamedSourceKey") or cfg["SourceKey"]).encode()


def adjust(cfg):
    """mLogTimeZoneOffsetSecond of the configuration in the process's current zone"""
    off = oap.tz_offset(cfg.get("Timezone", ""))
    return off - _time.localtime().tm_gmtoff if off is not None else 0


def flag_configs(renamed=None, source="content"):
    """the 8 CommonParserOptions combinations"""
    return [config(source, renamed, bool(f & 1), bool(f & 2), bool(f & 4)) for f in range(8)]


def ml_config(source="content"):
    return {"SourceKey": source, "StartPattern": ML_START, "UnmatchedContentTreatment": "single_line"}


def oracle_chain(val, split_cfg, acfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True, now=NOW,
                 di=DI):
    """(Logs bytes, Apsara counters [5] in lc_apsara_parse's order, splitter counters or None, piece count)"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    ap = oap.ProcessorParseApsaraNative(acfg, di)
    ap.process(g, now)
    c = ap.counters
    return (sc.wire_of(g.events, enable_ns),
            [c["out_key_not_found"], c["out_failed"], c["history_failure"], c["discarded"], c["out_successful"]],
            sp.counters if multiline else None, npieces)


def date(t, frac=b""):
    """"[YYYY-MM-DD HH:MM:SS<frac>]" of t rendered in UTC (parsed in the process's zone)"""
    return b"[" + _time.strftime("%Y-%m-%d %H:%M:%S", _time.gmtime(t)).encode() + frac + b"]"


def epoch(t, micro=0):
    return b"[%d%06d]" % (t, micro)


def special_lines(source="content", okey=OKEY, renamed="raw"):
    """lines that put the chain's own keys among the fields, once and repeated, around recent times"""
    s, o, r = source.encode(), (okey if okey is not None else b"off"), renamed.encode()
    t = NOW - 100
    return [
        date(t, b".5") + b"\t[INFO]\t[1234]\t[src/a.cpp:12]\tk1:v1\tk2:v2",
        date(t, b".6") + b"\t" + s + b":over\tk:v",
        date(t) + b"\t" + s + b":a\tx:y\t" + s + b":b",
        date(t + 1) + b"\t[WARN]\t" + o + b":o1\t" + o + b":o2",
        date(t + 1) + b"\t__LEVEL__:lv\t__THREAD__:th\t__FILE__:f\t__LINE__:9",
        date(t + 1) + b"\t[ERROR]\t[77]\tmicrotime:m\tmicrotime:n",
        date(t + 2) + b"\t" + r + b":rv\t__raw_log__:rl",
        date(t + 2) + b"\t[DEBUG]\t[5]\t[./x.cc:]\tk1:a\tk1:b\tk1:c",
        epoch(t + 3, 123456) + b"\t[INFO]\tk:v",
        b"[%d]\tk:v" % BIG_EPOCH,
        b"[1700000000]",
        date(t + 3),
        date(t + 3, b",456") + b"\t:\t:x\ty:\t\tz",
        b"",
        b"garbage line",
        b"[",
        b"[x]\tk:v",
        b"[2023-13-01 00:00:00]\tk:v",        # a failed full parse ...
        date(t + 3, b".77") + b"\tk:v",        # ... then a hit on the key of the line before it
        b"[2024-1-1 1:2:3]",                   # a short time string: its key runs into the chunk's next bytes
        b"[2024-1-1 1:2:3]\tk:short",
        date(BOUNDARY - 3600) + b"\told:1",    # discarded at DI
        date(t + 3, b".88") + b"\tafter:discard",
    ]


def random_line(rng, t_lo, t_hi):
    """an Apsara line with a time in [t_lo, t_hi]: a date (fractions ".", ","), an epoch, or a broken time; 0..4 base
    fields; 0..8 key:value fields (keys repeat)"""
    t = rng.randint(t_lo, t_hi)
    kind = rng.random()
    if kind < 0.15:
        head = epoch(t, rng.randrange(10 ** 6))
    elif kind < 0.22:
        head = rng.choice([b"[2024-13-01 00:00:00]", b"2024-01-01", b"[2024-01-01 00:00", b"[", b"[x]", b"x"])
    else:
        head = date(t, rng.choice([b"", b".%d" % rng.randrange(10 ** 6), b",%03d" % rng.randrange(1000),
                                   b".%09d" % rng.randrange(10 ** 9)]))
    base = [b"INFO", b"12345", b"src/x.cpp:%d" % rng.randrange(999), b"ERROR", b"a.b"]
    rng.shuffle(base)
    parts = [head] + [b"[" + f + b"]" for f in base[:rng.randint(0, 4)]]
    for _ in range(rng.randint(0, 8)):
        parts.append(b"k%d:%s" % (rng.randrange(6), bytes(rng.choice(b"abc:[]/. 09") for _ in range(rng.randrange(30)))))
    return b"\t".join(parts)


def random_value(seed, nlines=80, trailing=None, source="content", okey=OKEY, renamed="raw"):
    """random lines around the discard boundary, repeated ones (cache hits), special lines and empty lines"""
    rng = random.Random(seed)
    lines = []
    for _ in range(nlines):
        r = rng.random()
        if r < 0.05:
            lines.append(b"")
        elif r < 0.25 and lines:
            lines.append(rng.choice(lines))  # the same time string again: a cache hit
        elif r < 0.4:
            lines.append(random_line(rng, BOUNDARY - 30, BOUNDARY + 30))
        else:
            lines.append(random_line(rng, NOW - 3000, NOW))
    lines += special_lines(source, okey, renamed)
    rng.shuffle(lines)
    val = b"\n".join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def ml_value(seed, nrec=20):
    """multiline Apsara records: a header line, then stack-trace lines; unmatched lines between some records"""
    rng = random.Random(seed)
    out = []
    for i in range(nrec):
        out.append(random_line(rng, NOW - 3000, NOW) if rng.random() < 0.8 else date(NOW - 5) + b"\t[ERROR]\tboom")
        if not out[-1].startswith(b"[") or out[-1][1:5] != b"%d" % 2023:
            out[-1] = date(NOW - 7, b".%d" % i) + b"\t" + out[-1]
        out += [b"\tat com.example.Frame%d(Frame.java:%d)" % (j, rng.randint(1, 999)) for j in
                range(rng.randint(0, 6))]
        if rng.random() < 0.2:
            out.append(b"unmatched %d" % i)
    return b"\n".join(out) + (b"\n" if rng.random() < 0.5 else b"")
