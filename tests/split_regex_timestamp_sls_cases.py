"""Shared cases of the split -> regex -> timestamp -> SLS tests: the oracle's splitter over one flat source event, its
ProcessorParseRegexNative, a group-level ProcessorParseTimestampNative step over the C oracle of the timestamp parse,
then sls_serialize_logs; and value generators whose time strings hit and miss the second-level cache, fail, and fall
behind the history discard."""
import time as _time

import numpy as np

from oracle import oracle as orc
from oracle import timestamp as ots
from tests import regex_sls_cases as rc
from tests import split_sls_cases as sc
from tests.emul import timestamp as ets

OKEY = b"__file_offset__"
NOW = 1700000000  # 2023-11-14 22:13:20 UTC
NGINX_FMT = "%d/%b/%Y:%H:%M:%S"
F_FMT = "%Y-%m-%dT%H:%M:%S.%f"
PATTERN = r"(\S*) (\w+) (.*)"  # time, level, message; a line without a space fails
KEYS = ["time", "level", "msg"]
_MON = ("Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec")


def render(fmt, t, frac=""):
    """the time t (seconds, UTC) in fmt; frac: the digits of %f"""
    s = _time.gmtime(t)
    if fmt == NGINX_FMT:
        return "%02d/%s/%04d:%02d:%02d:%02d" % (s.tm_mday, _MON[s.tm_mon - 1], s.tm_year, s.tm_hour, s.tm_min,
                                                s.tm_sec)
    if fmt == F_FMT:
        return "%04d-%02d-%02dT%02d:%02d:%02d.%s" % (s.tm_year, s.tm_mon, s.tm_mday, s.tm_hour, s.tm_min, s.tm_sec,
                                                     frac or "5")
    return str(t)  # "%s"


def time_pool(fmt, rng):
    """time strings for fmt: recent ones (kept at discard_interval 43200, several repeated so that the cache hits),
    one a day old and one before 1970 (discarded), garbage and empty ones (failed), and a recent one with a suffix
    (a cache hit on its prefix, also after a failed full parse)"""
    recent = [NOW - rng.randint(0, 3000) for _ in range(4)]
    if fmt == "%s":
        vals = [str(t) for t in recent] + [str(NOW - 86400), "-5", "0", "x12", "", "5000000123", "12345",
                                           "%d999" % recent[0], "%d123456789" % recent[1]]
    else:
        vals = [render(fmt, t, str(rng.randint(0, 999999))) for t in recent]
        vals += [render(fmt, NOW - 86400), render(fmt, -86400 * 400), "garbage", "", vals[0] + "zz", vals[1] + "7"]
    return [v.encode() for v in vals]


def lines_value(rng, fmt, nlines, trailing=None):
    """lines for PATTERN with times from time_pool (about 20 % failing the regex or empty)"""
    pool = time_pool(fmt, rng)
    lines = []
    for _ in range(nlines):
        r = rng.random()
        if r < 0.1:
            lines.append(b"")
        elif r < 0.2:
            lines.append(rng.choice(pool) + b"nospace")
        else:
            lines.append(rng.choice(pool) + b" " + rng.choice([b"INFO", b"WARN", b"E"]) + b" msg %d" % rng.randint(0, 99))
    val = b"\n".join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def timestamp_step(events, tkey, fmt, source_year, adjust, now, discard_interval):
    """ProcessorParseTimestampNative over the events as one group (the C oracle of the parse): sets the times of the
    parsed events, erases the discarded ones; returns (events, counters [5])"""
    vals = [e.get(tkey) if e.type == orc.LOG and e.has(tkey) else None for e in events]
    base, off, ln, grp = ets.layout([vals])
    st, sec, ns, cnt = ots.process(fmt, source_year, adjust, base, off, ln, grp, now, discard_interval)
    kept = []
    for e, s, t, n in zip(events, st, sec, ns):
        if s == 3:
            continue
        if s == 0:
            e.timestamp, e.ns = int(t) & 0xFFFFFFFF, int(n)
        kept.append(e)
    return kept, [int(x) for x in cnt]


def oracle_chain(val, split_cfg, rcfg, tkey, fmt, now, discard_interval, time, ns, pos, offset_key=None,
                 multiline=False, enable_ns=True, source_year=-1, adjust=0):
    """(Logs bytes, counters [8] = the regex stage's three and the timestamp stage's five, splitter counters dict or
    None, piece count) of the oracle chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    rp = orc.ProcessorParseRegexNative(rc.oracle_config(rcfg))
    rp.process(g)
    g.events, tctr = timestamp_step(g.events, tkey, fmt, source_year, adjust, now, discard_interval)
    return (sc.wire_of(g.events, enable_ns), rc.counters_of(rp.counters) + tctr, sp.counters if multiline else None,
            npieces)


def configs():
    """(id, regex cfg, tkey): tkey a regex key, a repeated regex key, SourceKey kept on success, RenamedSourceKey and
    "__raw_log__" on kept failures, a key nobody sets"""
    yield "capture", rc.config(KEYS, regex=PATTERN), b"time"
    yield "capture_keep_fail", rc.config(KEYS, "content", None, True, False, False, regex=PATTERN), b"time"
    yield "repeated", rc.config(["time", "level", "time"], "content", None, True, False, False, regex=PATTERN), b"time"
    yield "repeated2", rc.config(["level", "time", "time"], regex=PATTERN), b"time"
    yield "source_keep_succeed", rc.config(KEYS, "content", None, True, True, False, regex=PATTERN), b"content"
    yield "source_fail_only", rc.config(KEYS, "content", None, True, False, False, regex=PATTERN), b"content"
    yield "renamed", rc.config(KEYS, "content", "raw", True, False, False, regex=PATTERN), b"raw"
    yield "raw_log", rc.config(KEYS, "content", None, True, False, True, regex=PATTERN), b"__raw_log__"
    yield "absent", rc.config(KEYS, "content", None, True, True, True, regex=PATTERN), b"nope"
    yield "key_overwrites_source", rc.config(["content", "level", "msg"], regex=PATTERN), b"content"


def device_args(cfg):
    """the regex stage's keyword arguments of the Engine bindings"""
    return dict(keys=[k.encode() for k in cfg["keys"]], source_key=cfg["source"].encode(),
                renamed_key=rc.renamed_key(cfg), keep_fail=cfg["keep_fail"], keep_succeed=cfg["keep_succeed"],
                copy_raw=cfg["copy_raw"], whole_line=rc.whole_line(cfg))


def tables_of(val, off, ln, cfg):
    """the regex stage's tables over the pieces (None in whole-line mode or without pieces) and the row pitch"""
    if rc.whole_line(cfg) or not off.size:
        return None, 0
    st, co, cl, pitch = rc.parse_tables(np.frombuffer(val, np.uint8), off, ln, cfg)
    return (st, co, cl), pitch
