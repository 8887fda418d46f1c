"""The reference's unit-test cases of ProcessorParseTimestampNative (tests/golden/ref_timestamp.json) replayed through
the C oracle and the host build of the device program, in two zones."""
import os
import time

import numpy as np
import pytest

from oracle import timestamp as ots
from tests import timestamp_fixtures as fx
from tests.emul import timestamp as ets

COUNTER = {"DiscardedEventsTotal": 3, "OutFailedEventsTotal": 1}


@pytest.fixture(params=("UTC", "Asia/Shanghai"))
def zone(request):
    saved = os.environ.get("TZ")
    os.environ["TZ"] = request.param
    time.tzset()
    yield request.param
    if saved is None:
        os.environ.pop("TZ", None)
    else:
        os.environ["TZ"] = saved
    time.tzset()


def _both(fmt, sy, adj, base, off, ln, grp, now, di):
    want = ots.process(fmt, sy, adj, base, off, ln, grp, now, di, "c")
    c = ets.Compiled(fmt, sy, adj)
    assert c.ok, c.error
    for W in (1, 32):
        got = c.parse(base, off, ln, grp, now, di, W)
        assert all(np.array_equal(x, y) for x, y in zip(got, want)), fmt
    return want


@pytest.mark.parametrize("k", range(len(fx.FIXTURES["parse"])))
def test_parse_log_time_cases(zone, k):
    c = fx.FIXTURES["parse"][k]
    now = int(time.time())
    base, off, ln, grp = fx.parse_layout(c)
    adj = fx.adjust(c["timezone"], now)
    st, sec, ns, cnt = _both(c["format"], -1, adj, base, off, ln, grp, now, -1)
    assert st.tolist() == [0] * len(c["values"])
    assert [[int(s), int(n)] for s, n in zip(sec, ns)] == fx.parse_expect(c, adj), c["values"]


@pytest.mark.parametrize("k", range(len(fx.FIXTURES["process"])))
def test_process_cases(zone, k):
    c = fx.FIXTURES["process"][k]
    now = int(time.time())
    fmt, sy, adj, groups, want, counters = *fx.process_case(c, now), c["counters"]
    st, sec, ns, cnt = _both(fmt, sy, adj, *ets.layout(groups), now, 43200)
    assert list(zip(st.tolist(), sec.tolist(), ns.tolist())) == want
    for name, v in counters.items():
        assert int(cnt[COUNTER[name]]) == v, name


def test_init_cases():
    for c in fx.FIXTURES["init"]:
        fmt = c["config"]["SourceFormat"]
        # an empty SourceFormat fails Init before the program is compiled (GetMandatoryStringParam)
        assert (fmt != "" and ets.Compiled(fmt).ok) == c["ok"], c["name"]
