"""GPU tier: the splitters' SerializeSls / SerializeSlsLz4(group, ProcessorParseApsaraNative&) through
lc_host_chain_serialize_sls: mode 0 (the device path where it applies, else the three host calls) and mode 2 (its LZ4
block) against mode 1 (Process + Process + SLSEventGroupSerializer::Serialize), with both processors' counters, on
generated groups, on the fallbacks, and on the reference's Apsara Process cases with each group's values joined into
one source event."""
import copy
import time

import pytest

from tests import apsara_cases as apc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_apsara_sls_cases as ac  # noqa: E402

pytestmark = pytest.mark.gpu

OKEY = ac.OKEY.decode()
SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": ac.ML_START, "UnmatchedContentTreatment": "single_line"})]


def _procs(split_type, split_cfg, acfg, discard):
    import loongcollector_b200 as lc
    ap = lc.HostProcessor("processor_parse_apsara_native", acfg)
    if discard is not None:
        ap.set_discard_old_data(discard)
    return lc.HostProcessor(split_type, split_cfg), ap


def _group(vals, offset_key=None, extra=None):
    g = {"metadata": {}, "tags": {"__topic__": "t"}, "events": []}
    if offset_key is not None:
        g["metadata"]["log.file.offset"] = offset_key
    for i, v in enumerate(vals):
        ev = {"type": 1, "timestamp": 1700000000 + i, "timestampNanosecond": 17 + i, "fileOffset": 1000 * i,
              "rawSize": len(v), "contents": {"content": v}}
        if extra:
            ev["contents"].update(extra)
        g["events"].append(ev)
    return g


def _counters(p):  # the event counters (wall-time counters end in _ns)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _check_modes(split_type, split_cfg, acfg, group, enable_ns=True, discard=None):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, acfg, discard)
    b = _procs(split_type, split_cfg, acfg, discard)
    got = capi.host_chain_serialize_sls(a[0], a[1], copy.deepcopy(group), enable_ns, 0)
    want = capi.host_chain_serialize_sls(b[0], b[1], copy.deepcopy(group), enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert _counters(a[0]) == _counters(b[0]) and _counters(a[1]) == _counters(b[1])
    c = _procs(split_type, split_cfg, acfg, discard)
    z = capi.host_chain_serialize_sls(c[0], c[1], copy.deepcopy(group), enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    assert _counters(c[0]) == _counters(b[0]) and _counters(c[1]) == _counters(b[1])
    return want, _counters(b[1])


def _recent_value(seed):
    """Apsara lines timed from this test's own clock: an hour back, far from the 12 h discard boundary, plus lines a
    day back (discarded with the rule on)"""
    now = int(time.time())
    val = ac.random_value(seed).replace(b"2023-11-15", b"2023-11-1X")  # the cases' fixed dates: failed parses now
    lines = [ac.date(now - 3600 - k, b".%d" % k) + b"\t[INFO]\t[%d]\tk:v%d" % (k, k) for k in range(20)]
    lines += [ac.epoch(now - 3600 + k, k) + b"\tk:e" for k in range(5)]
    lines += [ac.date(now - 86400 - k) + b"\told:%d" % k for k in range(5)]
    return (val + b"\n" + b"\n".join(lines)).decode("latin1")


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(split_type, split_cfg):
    vals = [_recent_value(s) for s in (1, 2)]
    cfgs = [ac.config("content", "raw", True, True, True), ac.config("content", None, False, False),
            ac.config("content", OKEY, True, True, False), ac.config("content", "__raw_log__", True, False, True)]
    for acfg in cfgs:
        for okey in (None, OKEY, "", "k1"):
            for enable_ns in (True, False):
                _check_modes(split_type, split_cfg, acfg, _group(vals[:1], okey), enable_ns)  # the device path
            _check_modes(split_type, split_cfg, acfg, _group(vals, okey))  # two source events: the host calls
    base = cfgs[0]
    want, ctr = _check_modes(split_type, split_cfg, base, _group(vals[:1], OKEY))
    assert ctr["history_failure"] >= 5 and ctr["out_successful"] >= 20, ctr
    _, ctr = _check_modes(split_type, split_cfg, base, _group(vals[:1], OKEY), discard=False)
    assert ctr["history_failure"] == 0, ctr
    # fallbacks: raw content, another Apsara SourceKey, offset key = SourceKey, a non-flat group, an empty value
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), base, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(base, SourceKey="other"), _group(vals[:1]))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], "content"))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], extra={"x": "y"}))
    _check_modes(split_type, split_cfg, base, _group([""]))
    # errors: empty group, every piece erased
    assert _check_modes(split_type, split_cfg, base, _group([]))[0][2] == "empty event group"
    erased = ac.config("content", None, False, False)
    assert _check_modes(split_type, split_cfg, erased, _group(["x\ny\nz"]))[0][0] is None


def _joined(case):
    vals = [e["contents"].get("content") for e in case["input"]["events"]]
    if any(v is None or "\n" in v for v in vals):
        return None
    g = copy.deepcopy(case["input"])
    g["events"] = [g["events"][0]]
    g["events"][0]["contents"] = {"content": "\n".join(vals)}
    return g


@pytest.mark.parametrize("case", [c for c in apc.FIXTURES["process"] if _joined(c) is not None],
                         ids=lambda c: c["name"])
def test_reference_groups(case):
    """the reference's Apsara Process cases, each group's values joined by \\n into one source event (their 2023
    times: with the history discard off, and on)"""
    cfg = case["config"]
    for okey in (None, OKEY):
        g = _joined(case)
        if okey is not None:
            g.setdefault("metadata", {})["log.file.offset"] = okey
        for discard in (False, True):
            _check_modes("processor_split_string_native", {"SourceKey": cfg["SourceKey"]}, cfg, g, discard=discard)
