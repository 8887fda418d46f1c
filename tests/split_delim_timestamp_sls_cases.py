"""Shared cases of the split -> delimiter -> timestamp -> SLS tests: the oracle's splitter over one flat source event,
its ProcessorParseDelimiterNative, the group-level ProcessorParseTimestampNative step of the split -> regex ->
timestamp tests, then sls_serialize_logs; and CSV lines whose time column hits and misses the second-level cache,
fails, falls behind the history discard, is quoted around the separator or holds doubled quotes."""
import time as _time

from oracle import oracle as orc
from tests import delim_sls_cases as dc
from tests import split_delim_sls_cases as sdc
from tests import split_regex_timestamp_sls_cases as tc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"
NOW = tc.NOW
YMD = "%Y-%m-%d %H:%M:%S"
F_FMT = tc.F_FMT  # ends in %f
COMMA_FMT = "%b %d, %Y %H:%M:%S"  # holds the separator: the column is quoted
DQ_FMT = '%Y-%m-%d"%H:%M:%S'  # holds the quote: the column is quoted with it doubled, and parses only collapsed
FORMATS = [YMD, "%s", F_FMT, COMMA_FMT, DQ_FMT]
_MON = ("Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec")
config = sdc.config


def render(fmt, t, frac=""):
    """the time t (seconds, UTC) in fmt; frac: the digits of %f"""
    s = _time.gmtime(t)
    if fmt == YMD:
        return _time.strftime(YMD, s)
    if fmt == COMMA_FMT:
        return "%s %02d, %04d %02d:%02d:%02d" % (_MON[s.tm_mon - 1], s.tm_mday, s.tm_year, s.tm_hour, s.tm_min,
                                                  s.tm_sec)
    if fmt == DQ_FMT:
        return '%04d-%02d-%02d"%02d:%02d:%02d' % (s.tm_year, s.tm_mon, s.tm_mday, s.tm_hour, s.tm_min, s.tm_sec)
    return tc.render(fmt, t, frac)


def time_pool(fmt, rng):
    """time strings for fmt: recent ones (kept at discard_interval 43200, several repeated so that the cache hits),
    one a day old and one before 1970 (discarded), garbage and empty ones (failed), and recent ones with a suffix (a
    cache hit on their prefix, also after a failed full parse)"""
    recent = [NOW - rng.randint(0, 3000) for _ in range(4)]
    if fmt == "%s":
        vals = [str(t) for t in recent] + [str(NOW - 86400), "-5", "0", "x12", "", "5000000123", "%d999" % recent[0],
                                           "%d123456789" % recent[1]]
    else:
        vals = [render(fmt, t, str(rng.randint(0, 999999))) for t in recent]
        vals += [render(fmt, NOW - 86400), render(fmt, -86400 * 400), "garbage", "", vals[0] + "zz", vals[1] + "7"]
    return [v.encode() for v in vals]


def field(v: bytes, sep: bytes, quote: int, rng=None):
    """v as a CSV column: quoted (quotes doubled) when it holds the separator or the quote, or now and then anyway;
    as it is when the row is split without quote handling"""
    if len(sep) != 1 or quote == sep[0]:
        return v
    q = bytes([quote])
    if sep in v or q in v or (rng is not None and rng.random() < 0.2):
        return q + v.replace(q, q + q) + q
    return v


def csv_line(rng, pool, sep, quote, ncols, tcol):
    """one line: the time at column tcol of ncols, with empty, blank, broken, short and wide rows among them"""
    use_quote = len(sep) == 1 and quote != sep[0]
    r = rng.random()
    if r < 0.04:
        return b""
    if r < 0.07:
        return rng.choice([b"   ", b" \r", b"\r"])
    cols = [rng.choice([b"INFO", b"WARN", b"E", b"", b"m%d" % rng.randint(0, 99)]) for _ in range(ncols)]
    cols[tcol] = field(rng.choice(pool), sep, quote, rng)
    if r < 0.12:
        cols = cols[:rng.randint(1, max(tcol, 1))] if tcol else cols[:0]  # short: does not reach the time column
    elif r < 0.17:
        cols += [b"x%d" % k for k in range(rng.randint(1, 4))]  # wide: overflow columns
    line = sep.join(cols)
    if r > 0.93 and use_quote:
        line = (b'"open' + sep + line) if rng.random() < 0.5 else (b'ab"c' + sep + line)  # the state machine fails
    if rng.random() < 0.1:
        line = b" " + line
    return line


def lines_value(rng, fmt, nlines, sep=b",", quote=ord('"'), ncols=3, tcol=0, trailing=None):
    pool = time_pool(fmt, rng)
    val = b"\n".join(csv_line(rng, pool, sep, quote, ncols, tcol) for _ in range(nlines))
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def bare_value(rng, fmt, nlines, sep=b","):
    """lines that are a time string alone, or with one more column (so that short-row and failure rules put the whole
    piece under RenamedSourceKey / "__raw_log__"), with empty and broken lines among them"""
    pool = time_pool(fmt, rng)
    lines = []
    for _ in range(nlines):
        r = rng.random()
        v = rng.choice(pool)
        if r < 0.05:
            lines.append(b"")
        elif r < 0.15:
            lines.append(v + b' "x' + sep + b"y")  # a quote inside a plain column: a failure
        elif r < 0.5:
            lines.append(v + sep + b"INFO")
        else:
            lines.append(v)
    return b"\n".join(lines)


def counters_of(dctr, tctr):
    """the oracle's counters in the order the chain's counters[9] fold to: successful, failed + blank, discarded, then
    the timestamp stage's five"""
    return [dctr["out_successful"], dctr["out_failed"], dctr["discarded"]] + list(tctr)


def fold(ctr):
    """the chain's counters[9] as counters_of orders the oracle's"""
    return sdc.fold(ctr[:4]) + [int(x) for x in ctr[4:]]


def oracle_chain(val, split_cfg, cfg, tkey, fmt, now, discard_interval, time, ns, pos, offset_key=None,
                 multiline=False, enable_ns=True, source_year=-1, adjust=0):
    """(Logs bytes, counters [8] as counters_of, splitter counters dict or None, piece count) of the oracle chain:
    split_delim_sls_cases' splitter and delimiter, then the group-level timestamp step"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    dp = orc.ProcessorParseDelimiterNative(dc.oracle_config(cfg))
    dp.process(g)
    g.events, tctr = tc.timestamp_step(g.events, tkey, fmt, source_year, adjust, now, discard_interval)
    return sc.wire_of(g.events, enable_ns), counters_of(dp.counters, tctr), sp.counters if multiline else None, npieces


def configs():
    """(id, delimiter cfg, tkey, value generator rng, fmt -> value): tkey at a column every row reaches and at one
    short rows do not reach; SourceKey among the keys and not; RenamedSourceKey with keep_succeed; kept failures under
    RenamedSourceKey and "__raw_log__"; "_" in discard mode; an absent key; the three overflow treatments, a
    multi-byte separator and a quote equal to the separator"""
    keys = ["time", "level", "msg"]
    yield ("col0", config(keys), b"time", lambda r, f: lines_value(r, f, 80))
    yield ("col_short", config(["level", "msg", "time"]), b"time", lambda r, f: lines_value(r, f, 80, tcol=2))
    yield ("col_short_keep_succeed", config(["level", "msg", "time"], renamed="time", keep_succeed=True), b"time",
           lambda r, f: lines_value(r, f, 80, tcol=2))
    yield ("source_in_keys", config(["level", "msg", "content"]), b"content",
           lambda r, f: lines_value(r, f, 80, tcol=2))
    yield ("source_not_key", config(keys, keep_fail=True), b"content", lambda r, f: lines_value(r, f, 80))
    yield ("renamed_keep_succeed", config(["level", "msg"], renamed="raw", keep_succeed=True), b"raw",
           lambda r, f: bare_value(r, f, 80))
    yield ("renamed_fail", config(["a", "b"], renamed="raw", keep_fail=True, allow_short=False), b"raw",
           lambda r, f: bare_value(r, f, 80))
    yield ("raw_log_fail", config(["a", "b"], keep_fail=True, copy_raw=True, allow_short=False), b"__raw_log__",
           lambda r, f: bare_value(r, f, 80))
    yield ("underscore_discard", config(["_", "level", "_"], treatment="discard"), b"_",
           lambda r, f: lines_value(r, f, 80))
    yield ("absent", config(keys, keep_fail=True, keep_succeed=True, copy_raw=True), b"nope",
           lambda r, f: lines_value(r, f, 80))
    yield ("keep", config(keys, treatment="keep"), b"time", lambda r, f: lines_value(r, f, 80))
    yield ("discard", config(keys, treatment="discard"), b"time", lambda r, f: lines_value(r, f, 80))
    yield ("multibyte", config(keys, sep=b"|#"), b"time", lambda r, f: lines_value(r, f, 80, sep=b"|#"))
    yield ("quote_is_sep", config(keys, quote=ord(",")), b"time",
           lambda r, f: lines_value(r, f, 80, quote=ord(",")))


def plain_fmt(fmt, cfg):
    """whether fmt's strings can stand in a column of cfg's rows: a separator or a quote inside needs the quote state
    machine"""
    if fmt in (COMMA_FMT, DQ_FMT):
        return len(cfg["sep"]) == 1 and cfg["quote"] != cfg["sep"][0]
    return True


tables = sdc.tables
device_args = sdc.device_args
