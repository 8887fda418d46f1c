"""GPU tier: the host class ProcessorParseTimestampNative (loongcollector_b200/host) replays the reference's unit-test
cases (tests/golden/ref_timestamp.json) to the reference's expected events and counters, through Process(group) and
through the batched Process(std::vector<PipelineEventGroup>&) that sends every group to the device in one call."""
import random
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import timestamp as ots  # noqa: E402
from tests import timestamp_cases as tc  # noqa: E402
from tests import timestamp_fixtures as fx  # noqa: E402
from tests.emul import timestamp as ets  # noqa: E402

NAME = "processor_parse_timestamp_native"
UNTOUCHED = 12345678901


def _group(values):
    evs = []
    for v in values:
        e = {"contents": {"time": v} if v is not None else {"other": "x"}, "timestamp": UNTOUCHED,
             "timestampNanosecond": 0, "type": 1}
        evs.append(e)
    return {"events": evs}


def _times(group):
    return [(e["timestamp"], e.get("timestampNanosecond", 0)) for e in (group or {}).get("events", [])]


def test_init_cases():
    import loongcollector_b200 as lc
    for c in fx.FIXTURES["init"]:
        if c["ok"]:
            lc.HostProcessor(NAME, c["config"])
        else:
            with pytest.raises(Exception):
                lc.HostProcessor(NAME, c["config"])
    for fmt in ("%c", "%x", "%X"):
        with pytest.raises(Exception, match="SourceFormat"):
            lc.HostProcessor(NAME, {"SourceKey": "time", "SourceFormat": fmt})


@pytest.mark.parametrize("k", range(len(fx.FIXTURES["process"])))
def test_process_cases(k):
    import loongcollector_b200 as lc
    c = fx.FIXTURES["process"][k]
    cfg = dict(c["config"])
    now = int(time.time())
    fmt, sy, adj, groups, want = fx.process_case(c, now)
    if cfg.get("SourceYear") == "now":
        cfg["SourceYear"] = sy
    p = lc.HostProcessor(NAME, cfg)
    out = p.process(_group([v.decode() for v in groups[0]]), True)
    if c["expect"] == "erased":
        assert _times(out) == []
    elif c["expect"] == "unchanged":
        assert _times(out) == [(UNTOUCHED, 0)] * 2
    else:
        assert _times(out) == [(s, n) for _, s, n in want]
    cnt = p.counters()
    assert cnt["discarded"] == c["counters"]["DiscardedEventsTotal"]
    assert cnt["out_failed"] == c["counters"]["OutFailedEventsTotal"]
    assert cnt["history_failure"] == cnt["discarded"]


def test_parse_cases_in_one_call(eng):
    """every ParseLogTime case of one configuration is a group of its own and all of them go through one call: the
    device gives the reference's expected times (lc_timestamp_parse without the history rule, as ParseLogTime has
    none), and the host class, whose Process applies that rule, erases these years-old events and counts them"""
    import loongcollector_b200 as lc
    now = int(time.time())
    by_cfg = {}
    for c in fx.FIXTURES["parse"]:
        by_cfg.setdefault((c["format"], c["timezone"]), []).append(c)
    for (fmt, tz), cases in by_cfg.items():
        adj = fx.adjust(tz, now)
        base, off, ln, grp = ets.layout([[v.encode() for v in c["values"]] for c in cases])
        st, sec, ns, cnt = eng.timestamp_parse(lc.Timestamp(fmt, -1, adj), base, off, ln, grp, now, -1)
        assert (st == 0).all()
        got = [[int(s), int(n)] for s, n in zip(sec, ns)]
        assert got == [e for c in cases for e in fx.parse_expect(c, adj)], fmt
        p = lc.HostProcessor(NAME, {"SourceKey": "time", "SourceFormat": fmt, "SourceTimezone": tz})
        outs = p.process_groups([_group(c["values"]) for c in cases], True)
        assert all(_times(out) == [] for out in outs)
        c = p.counters()
        assert c["history_failure"] == c["discarded"] == off.size and c["out_successful"] == 0


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def test_random_groups_equal_oracle():
    """mixed groups (missing keys, non-log events, damaged values, old times) through one batched call"""
    import loongcollector_b200 as lc
    rng = random.Random(11)
    now = int(time.time())
    fmt = "%Y-%m-%d %H:%M:%S.%f"
    p = lc.HostProcessor(NAME, {"SourceKey": "time", "SourceFormat": fmt})
    groups, vals = [], []
    for _ in range(200):
        g = []
        t = now - rng.choice((0, 0, 100000))
        for _ in range(rng.randint(0, 50)):
            t += rng.random() < 0.3
            v = tc.render(fmt, time.localtime(t), rng)
            r = rng.random()
            v = tc.damage(v, rng).replace(b"\x00", b"?").replace(b"\xff", b"?") if r < 0.15 else v
            g.append(None if r < 0.05 else v)
        vals.append(g)
        groups.append(_group([v.decode() if v is not None else None for v in g]))
    outs = p.process_groups(groups, True)
    base, off, ln, grp = ets.layout(vals)
    st, sec, ns, cnt = ots.process(fmt, -1, 0, base, off, ln, grp, now, 43200, "c")
    i = 0
    for g, out in zip(vals, outs):
        want = []
        for _ in g:
            if st[i] == 0:
                want.append((int(sec[i]), int(ns[i])))
            elif st[i] != 3:
                want.append((UNTOUCHED, 0))
            i += 1
        assert _times(out) == want
    c = p.counters()
    assert [c["out_key_not_found"], c["out_failed"], c["history_failure"], c["discarded"], c["out_successful"]] == \
        [int(x) for x in cnt]
