"""The reference's ProcessorParseTimestampNative unit-test cases (tests/golden/ref_timestamp.json) turned into event
tables for a given "now" and the process's zone."""
import json
import os
import time

from tests.emul import timestamp as ets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_timestamp.json")))


def tz_seconds(tz):
    """ParseTimeZoneOffsetSecond of "GMT+hh:mm" (the fixtures use only that form)"""
    sec = int(tz[4:6]) * 3600 + int(tz[7:9]) * 60
    return -sec if tz[3] == "-" else sec


def adjust(tz, now):
    """mLogTimeZoneOffsetSecond: SourceTimezone's offset minus the local one at `now`"""
    return tz_seconds(tz) - time.localtime(now).tm_gmtoff if tz else 0


def process_case(c, now):
    """(format, source_year, adjust, groups, expected [(status, sec, nsec)] of the two events, counters)"""
    cfg = c["config"]
    t = now + c["now_shift"]
    v = time.strftime(c["strftime"], time.localtime(t)).encode()
    sy = cfg.get("SourceYear", -1)
    if sy == "now":
        sy = time.localtime(now).tm_year
    adj = adjust(cfg.get("SourceTimezone", ""), now)
    status = {"parsed": 0, "unchanged": 2, "erased": 3}[c["expect"]]
    sec = t - adj if status != 2 else 0
    return cfg["SourceFormat"], sy, adj, [[v, v]], [(status, sec, c["nanosecond"] if status == 0 else 0)] * 2


def parse_layout(c):
    return ets.layout([[v.encode() for v in c["values"]]])


def parse_expect(c, adj):
    """The expected (tv_sec, tv_nsec) of a ParseLogTime case.  The reference's expectations hold in a zone at UTC; a %s
    value is zone-free, so elsewhere the timezone adjustment moves it."""
    if c["format"] != "%s":
        return c["expect"]
    return [[s - adj, n] for s, n in c["expect"]]
