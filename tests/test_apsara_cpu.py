"""CPU tier of the Apsara parse: the oracle (oracle/lc_apsara_oracle.c and oracle.apsara) reproduces every case of the
reference's unit test (tests/golden/ref_apsara.json), and the host build of the device functions
(tests/emul/lc_apsara_emul.cpp) equals the oracle on every output and counter with 1, 3 and 32 lanes."""
import os
import time

import numpy as np
import pytest

from oracle import apsara as oap
from oracle import oracle as orc
from tests import apsara_cases as ac
from tests.emul import apsara as eap
from tests.emul import timestamp as ets

FX = ac.FIXTURES


@pytest.fixture
def zone(request):
    old = os.environ.get("TZ")
    os.environ["TZ"] = request.param if hasattr(request, "param") else "UTC"
    time.tzset()
    yield os.environ["TZ"]
    if old is None:
        del os.environ["TZ"]
    else:
        os.environ["TZ"] = old
    time.tzset()


def _adjust(cfg):
    off = oap.tz_offset(cfg.get("Timezone", ""))
    return off - time.localtime().tm_gmtoff if off is not None else 0


def test_time_sequence(zone):
    cfg = FX["time"]["config"]
    vals = [s["value"].encode() for s in FX["time"]["steps"]]
    base, off, ln, grp = ets.layout([vals])
    st, sec, ns, us, first, ent, cnt = oap.process(cfg["SourceKey"], _adjust(cfg), base, off, ln, grp, 0)
    assert [int(x) for x in sec] == [s["time"] for s in FX["time"]["steps"]]
    assert [int(x) for x in us] == [s["micro"] for s in FX["time"]["steps"]]


def _run_groups(cfg, groups, now=0, interval=-1, split=None):
    p = oap.ProcessorParseApsaraNative(cfg, interval)
    for g in groups:
        if split == "string":
            orc.ProcessorSplitLogStringNative(cfg).process(g)
        elif split == "multiline":
            orc.ProcessorSplitMultilineLogStringNative(cfg).process(g)
    p.process_groups(groups, now)
    return p


def test_lines(zone):
    cfg = FX["lines"]["config"]
    for c in FX["lines"]["cases"]:
        g = orc.Group.from_json(ac.group_json([c["value"].encode()]))
        _run_groups(cfg, [g])
        out = g.to_json()
        if not c["pairs"]:
            assert out is None, c
            continue
        got = out["events"][0]["contents"]
        for k, v in c["pairs"][:c["pinned"]]:
            assert got[k] == v, (c, got)


def _norm(x):
    return orc.Group.from_json(x).to_json() if x is not None else None


@pytest.mark.parametrize("case", FX["process"], ids=lambda c: c["name"])
def test_process_cases(zone, case):
    g = orc.Group.from_json(case["input"])
    p = _run_groups(case["config"], [g], split=case["split"])
    assert g.to_json() == _norm(case["expect"])
    names = {"DiscardedEventsTotal": "discarded", "OutFailedEventsTotal": "out_failed"}
    for k, v in case["counters"].items():
        if k in names:
            assert p.counters[names[k]] == v, (k, p.counters)


def _same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("zone", ac.ZONES, indirect=True)
@pytest.mark.parametrize("tz", ["", "GMT+08:00", "GMT-03:30", "bogus"])
def test_emul_equals_oracle(zone, tz):
    cfg = {"SourceKey": "content", "Timezone": tz}
    adj = _adjust(cfg)
    groups = ac.random_groups(hash((zone, tz)) & 0xFFFF) + [ac.corner_values()]
    base, off, ln, grp = ets.layout(groups)
    now = 1700000000 + 43200
    for interval in (-1, 43200 + 5):
        want = oap.process("content", adj, base, off, ln, grp, now, interval)
        assert int(want[6][4]) > 0
        for W in (1, 3, 32):
            _same(eap.parse("content", adj, base, off, ln, grp, now, interval, W), want)


def test_emul_fixture_values(zone):
    vals = [s["value"].encode() for s in FX["time"]["steps"]] + [c["value"].encode() for c in FX["lines"]["cases"]]
    for groups in ([vals], [[v] for v in vals]):
        base, off, ln, grp = ets.layout(groups)
        want = oap.process("content", 8 * 3600, base, off, ln, grp, 0)
        for W in (1, 3, 32):
            _same(eap.parse("content", 8 * 3600, base, off, ln, grp, 0, -1, W), want)


def test_small_and_large_values(zone):
    groups = [[b"", b"[", b"[2"], [b"[2024-01-02 03:04:05.5]\t" + b"a:b\t" * 20000]]
    base, off, ln, grp = ets.layout(groups)
    assert int(ln.max()) > 65536
    want = oap.process("content", 0, base, off, ln, grp, 0)
    assert want[0].tolist() == [2, 3, 3, 0]
    for W in (1, 3, 32):
        _same(eap.parse("content", 0, base, off, ln, grp, 0, -1, W), want)


def test_cache_after_failed_parses(zone):
    """a failed full parse leaves the cache alone, and a hit needs no full parse of its own"""
    vals = [b"[2024-01-02 03:04:05.1]\tk:v", b"[2024-01-02 03:04:xx]\tk:v", b"[2024-01-02 03:04:05.2]\tk:v",
            b"[2024-01-02         03:04:06]\tk:v", b"[2024-01-02         x55]\tk:v", b"[2024-01-02 03:04:0x9]"]
    base, off, ln, grp = ets.layout([vals])
    st, sec, ns, us, first, ent, cnt = oap.process("content", 0, base, off, ln, grp, 0)
    t = 1704164645  # 2024-01-02 03:04:05 UTC
    local = t - time.localtime(t).tm_gmtoff
    assert st.tolist() == [0, 3, 0, 0, 0, 0]
    assert sec.tolist() == [local, 0, local, local + 1, local + 1, local - 5]
    assert ns.tolist() == [100000000, 0, 200000000, 0, 550000000, 900000000]
    for W in (1, 3, 32):
        _same(eap.parse("content", 0, base, off, ln, grp, 0, -1, W), (st, sec, ns, us, first, ent, cnt))


def test_reference_strptime_cross_check(zone):
    from oracle import timestamp as ots
    if not ots.have_reference():
        pytest.skip("oracle/_ref/libref_strptime.so was not built")
    vals = [v for g in ac.random_groups(7) for v in g if v and v.startswith(b"[") and b"]" in v]
    times = [v[1:v.index(b"]")] for v in vals]
    for fmt, pick in (("%s", lambda t: t[:1] == b"1"), ("%Y-%m-%d %H:%M:%S", lambda t: t[:1] != b"1")):
        sel = [[t] for t in times if pick(t)]
        base, off, ln, grp = ets.layout(sel)
        a = ots.process(fmt, -1, 0, base, off, ln, grp, 0, -1, which="c")
        b = ots.process(fmt, -1, 0, base, off, ln, grp, 0, -1, which="ref")
        _same(a, b)
    # %f: after the seconds' separator, at the time string + 20 (a hit), and at bytes that do not start with a digit
    dates = [t for t in times if t[:1] != b"1"] + [t + b"]" for t in (b"x", b"2024-01-02 03:04:05", b"\x00")]
    sel = [[t[k:]] for t in dates for k in (19, 20, 21)]
    base, off, ln, grp = ets.layout(sel)
    a = ots.process("%f", -1, 0, base, off, ln, grp, 0, -1, which="c")
    b = ots.process("%f", -1, 0, base, off, ln, grp, 0, -1, which="ref")
    _same(a, b)
    assert int((a[2] != 0).sum()) > 0
