"""GPU tier: the splitters' SerializeSls / SerializeSlsLz4(group, ProcessorParseJsonNative&) through
lc_host_chain_serialize_sls: mode 0 (the device path where it applies, else the three host calls) and mode 2 (its LZ4
block) against mode 1 (Process + Process + SLSEventGroupSerializer::Serialize), with both processors' counters, on
generated groups and on every one-source-event input group of the reference's unit test."""
import copy
import random

import pytest

from tests import json_fixtures as jf  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_json_sls_cases as jsc  # noqa: E402

pytestmark = pytest.mark.gpu

OKEY = jsc.OKEY.decode()
SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"\{.*", "UnmatchedContentTreatment": "single_line"})]


def _procs(split_type, split_cfg, jcfg):
    import loongcollector_b200 as lc
    return lc.HostProcessor(split_type, split_cfg), lc.HostProcessor("processor_parse_json_native", jcfg)


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


def _check_modes(split_type, split_cfg, jcfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, jcfg)
    b = _procs(split_type, split_cfg, jcfg)
    got = capi.host_chain_serialize_sls(a[0], a[1], copy.deepcopy(group), enable_ns, 0)
    want = capi.host_chain_serialize_sls(b[0], b[1], copy.deepcopy(group), enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert _counters(a[0]) == _counters(b[0]) and _counters(a[1]) == _counters(b[1])
    c = _procs(split_type, split_cfg, jcfg)
    z = capi.host_chain_serialize_sls(c[0], c[1], copy.deepcopy(group), enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    assert _counters(c[0]) == _counters(b[0]) and _counters(c[1]) == _counters(b[1])
    return want


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(split_type, split_cfg):
    vals = [jsc.random_value(s).decode("latin1") for s in (1, 2, 3)]
    cfgs = [jsc.config("content", "raw", True, True, True), jsc.config("content", None, False, False),
            jsc.config("content", OKEY, True, True, False), jsc.config("content", "__raw_log__", True, False, True)]
    for jcfg in cfgs:
        for okey in (None, OKEY, "", "a"):
            _check_modes(split_type, split_cfg, jcfg, _group(vals[:1], okey))  # the one-chunk LZ4 device path
            _check_modes(split_type, split_cfg, jcfg, _group(vals, okey))      # several source events
    base = cfgs[0]
    # fallbacks: raw content, another JSON SourceKey, offset key = SourceKey, a non-flat group, an empty value
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), base, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(base, SourceKey="other"), _group(vals[:1]))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], "content"))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], extra={"x": "y"}))
    _check_modes(split_type, split_cfg, base, _group([""]))
    # errors: empty group, every piece erased
    assert _check_modes(split_type, split_cfg, base, _group([]))[2] == "empty event group"
    erased = jsc.config("content", None, False, False)
    assert _check_modes(split_type, split_cfg, erased, _group(["x\ny\n\nz"]))[0] is None


@pytest.mark.parametrize("case", [c for c in jf.PROCESS if len(c["input"]["events"]) == 1],
                         ids=lambda c: c["name"])
def test_reference_groups(case):
    """every one-source-event input group of the reference's unit test, TestMultipleLines with its \\0 splitter"""
    cfg = case["config"]
    split_cfg = {"SourceKey": cfg["SourceKey"], "SplitChar": cfg.get("SplitChar", 10)}
    jcfg = {k: v for k, v in cfg.items() if k != "SplitChar"}
    for okey in (None, OKEY):
        g = copy.deepcopy(case["input"])
        if okey is not None:
            g.setdefault("metadata", {})["log.file.offset"] = okey
        _check_modes("processor_split_string_native", split_cfg, jcfg, g)


def test_synth_json_lines_groups():
    from loongcollector_b200 import synth
    buf = synth.json_lines(2000, seed=3, hi=2048)[0]
    val = bytes(buf).decode("latin1")
    rng = random.Random(1)
    for split_type, split_cfg in SPLITTERS:
        jcfg = jsc.config("content", None, bool(rng.getrandbits(1)), bool(rng.getrandbits(1)))
        _check_modes(split_type, split_cfg, jcfg, _group([val], OKEY))
