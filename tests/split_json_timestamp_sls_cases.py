"""Shared cases of the split -> JSON -> timestamp -> SLS tests: the oracle's splitter over one flat source event,
oracle/json_parse.py's ProcessorParseJsonNative, the group-level ProcessorParseTimestampNative step of the split ->
regex -> timestamp tests, then sls_serialize_logs; and JSON lines whose time member is a plain string (a chunk value),
an escaped string (an arena value), an integer or a float (its %f rendering, in the arena), repeated and spelled
escaped, so that the second-level cache hits and misses across chunk and arena values."""
import json
import time as _time

import numpy as np

from oracle import json_parse as ojs
from oracle import oracle as orc
from tests import split_json_sls_cases as jsc
from tests import split_regex_timestamp_sls_cases as tc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"
NOW = tc.NOW
YMD = "%Y-%m-%d %H:%M:%S"
FORMATS = [YMD, "%s"]
config = jsc.config
renamed_key = jsc.renamed_key


def render(fmt, t):
    """the time t (seconds, UTC) in fmt"""
    if fmt == "%s":
        return str(t)
    return _time.strftime(YMD, _time.gmtime(t))


def escaped(s):
    """JSON string text of s with its first character written as a \\u escape (the rendering lands in the arena)"""
    if not s:
        return '""'
    return '"\\u%04x%s"' % (ord(s[0]), json.dumps(s)[2:-1])


def time_pool(fmt, rng):
    """JSON value texts for the time member: recent times (kept at discard_interval 43200, repeated so that the cache
    hits), plain and escaped, one a day old and one before 1970 (discarded), garbage and empty ones (failed), a recent
    one with a suffix (a cache hit on its prefix); for %s also integers, -0 and floats"""
    recent = [NOW - rng.randint(0, 3000) for _ in range(3)]
    vals = []
    for t in recent:
        vals += [json.dumps(render(fmt, t)), escaped(render(fmt, t))]
    vals += [json.dumps(render(fmt, NOW - 86400)), escaped(render(fmt, NOW - 86400)), '"garbage"', '""',
             json.dumps(render(fmt, recent[0]) + "zz"), escaped(render(fmt, recent[1]) + "7"), "12", "true",
             '{"a":1}']
    if fmt == "%s":
        vals += [str(recent[0]), str(recent[2]), "-0", "0", "-5", "%d.25" % recent[1], "%d.5e0" % recent[0],
                 "5000000123", '"x12"']
    else:
        vals += [json.dumps(render(fmt, -86400 * 400))]
    return vals


def lines_value(rng, fmt, nlines, member=b"time", trailing=None):
    """JSON lines with their time under `member` (plain or escaped key, sometimes repeated), mixed with {}, empty
    pieces, failed documents, documents without the member and bare time strings (which fail to parse)"""
    pool = time_pool(fmt, rng)
    k = member.decode()
    lines = []
    for _ in range(nlines):
        r = rng.random()
        v = rng.choice(pool)
        if r < 0.05:
            lines.append(b"")
        elif r < 0.1:
            lines.append(b"{}")
        elif r < 0.17:
            lines.append(b"not json " + v.encode())
        elif r < 0.22:
            lines.append(render(fmt, NOW - rng.randint(0, 3000)).encode())  # a bare time: a failure
        elif r < 0.27:
            lines.append(jsc.doc([('"other"', v)]))
        elif r < 0.4:
            lines.append(jsc.doc([(escaped(k), v), ('"msg"', '"m%d"' % rng.randint(0, 9))]))
        elif r < 0.5:
            lines.append(jsc.doc([(json.dumps(k), '"bad"'), ('"x"', "1"), (escaped(k), v)]))
        elif r < 0.55:
            lines.append(jsc.doc([(escaped(k), v), (json.dumps(k), rng.choice(pool))]))
        else:
            lines.append(jsc.doc([('"lvl"', '"INFO"'), (json.dumps(k), v), ('"msg"', '"m%d"' % rng.randint(0, 99))]))
    val = b"\n".join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def oracle_chain(val, split_cfg, jcfg, tkey, fmt, now, discard_interval, time, ns, pos, offset_key=None,
                 multiline=False, enable_ns=True, source_year=-1, adjust=0):
    """(Logs bytes, counters [8] = the JSON stage's three and the timestamp stage's five, splitter counters or None,
    piece count) of the oracle chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    jp = ojs.ProcessorParseJsonNative(jcfg)
    jp.process(g)
    c = jp.counters
    g.events, tctr = tc.timestamp_step(g.events, tkey, fmt, source_year, adjust, now, discard_interval)
    return (sc.wire_of(g.events, enable_ns), [c["out_successful"], c["out_failed"], c["discarded"]] + tctr,
            sp.counters if multiline else None, npieces)


def configs():
    """(id, JSON cfg, tkey, time member key of the lines)"""
    yield "member", config("content"), b"time", b"time"
    yield "member_keep_fail", config("content", None, True, False, True), b"time", b"time"
    yield "source_overwritten", config("content", None, True), b"content", b"content"
    yield "source_not_overwritten", config("content", None, True, False), b"content", b"time"
    yield "source_keep_succeed", config("content", None, False, True), b"content", b"time"
    yield "renamed_keep_succeed", config("content", "raw", True, True), b"raw", b"time"
    yield "renamed_member", config("content", "raw", False, True), b"raw", b"raw"
    yield "renamed_fail", config("content", "raw", True), b"raw", b"time"
    yield "raw_log", config("content", None, True, False, True), b"__raw_log__", b"time"
    yield "absent", config("content", None, True, True, True), b"nope", b"time"


def tables_of(val, off, ln, jcfg):
    """the JSON stage's tables over the pieces: (status, first, entries [m, 4], arena bytes)"""
    st, first, ent, arena, _ = ojs.process(jcfg["SourceKey"].encode(), np.frombuffer(val, np.uint8), off, ln)
    return st, first, ent, arena
