"""GPU tier: the host class ProcessorParseApsaraNative (loongcollector_b200/host) replays the reference's unit-test cases
(tests/golden/ref_apsara.json) to the reference's expected events and counters, and equals the oracle's group-level
Process on generated groups, history discards included, through Process(group) and through the batched
Process(std::vector<PipelineEventGroup>&) that sends every group to the device in one call."""
import copy
import os
import time

import pytest

pytestmark = pytest.mark.gpu

from oracle import apsara as oap  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from tests import apsara_cases as ac  # noqa: E402


@pytest.fixture
def utc():
    old = os.environ.get("TZ")
    os.environ["TZ"] = "UTC"
    time.tzset()
    yield
    if old is None:
        os.environ.pop("TZ", None)
    else:
        os.environ["TZ"] = old
    time.tzset()


NAME = "processor_parse_apsara_native"


def _host(cfg):
    import loongcollector_b200 as lc
    p = lc.HostProcessor(NAME, cfg)
    p.set_discard_old_data(False)
    return p


def _norm(x):
    return orc.Group.from_json(x).to_json() if x is not None else None


@pytest.mark.parametrize("case", ac.FIXTURES["process"], ids=lambda c: c["name"])
def test_host_class_fixtures(utc, case):
    import loongcollector_b200 as lc
    g = orc.Group.from_json(case["input"])
    if case["split"]:
        sp = {"string": orc.ProcessorSplitLogStringNative, "multiline": orc.ProcessorSplitMultilineLogStringNative}
        sp[case["split"]](case["config"]).process(g)
    p = _host(case["config"])
    out = p.process(g.to_json() or {"events": []})
    assert _norm(out) == _norm(case["expect"])
    c = p.counters()
    names = {"DiscardedEventsTotal": "discarded", "OutFailedEventsTotal": "out_failed"}
    for k, v in case["counters"].items():
        if k in names:
            assert c[names[k]] == v
    del lc


def test_host_class_lines(utc):
    cfg = ac.FIXTURES["lines"]["config"]
    for c in ac.FIXTURES["lines"]["cases"]:
        out = _host(cfg).process(ac.group_json([c["value"].encode()]))
        if not c["pairs"]:
            assert not (out or {}).get("events")
            continue
        got = out["events"][0]["contents"]
        for k, v in c["pairs"][:c["pinned"]]:
            assert got[k] == v


@pytest.mark.parametrize("cfg", [
    {"SourceKey": "content"},
    {"SourceKey": "content", "Timezone": "GMT+08:00", "KeepingSourceWhenParseFail": True, "CopingRawLog": True},
    {"SourceKey": "content", "KeepingSourceWhenParseSucceed": True, "RenamedSourceKey": "raw"},
    {"SourceKey": "k1", "Timezone": "bogus", "KeepingSourceWhenParseFail": True},
])
def test_host_class_random_groups(utc, cfg):
    now = int(time.time())
    # half the groups are timed well behind the history limit (43200 s behind now), so their events are discarded;
    # every time stays a minute or more away from the limit, so the oracle's now and the call's agree on each event
    groups = [ac.group_json([v.decode("latin-1").encode("utf-8") if v else v for v in g], {"k1": "[x"})
              for t0 in (now - 100, now - 43200 - 200) for g in ac.random_groups(21, 30, t0)]
    groups = [g for g in groups if g["events"]]
    want = [orc.Group.from_json(copy.deepcopy(g)) for g in groups]
    ref = oap.ProcessorParseApsaraNative(cfg, 43200)
    ref.process_groups(want, now)
    p = _host(cfg)
    p.set_discard_old_data(True, 43200)
    got = p.process_groups(groups)
    assert [_norm(x) for x in got] == [w.to_json() for w in want]
    p2 = _host(cfg)
    p2.set_discard_old_data(True, 43200)
    got1 = [p2.process(g) for g in groups]
    assert [_norm(x) for x in got1] == [w.to_json() for w in want]
    for k, v in ref.counters.items():
        assert p.counters()[k] == v and p2.counters()[k] == v
    if cfg["SourceKey"] == "content":
        assert ref.counters["history_failure"] > 0 and ref.counters["out_successful"] > 0
