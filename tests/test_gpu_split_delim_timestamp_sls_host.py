"""GPU tier: the splitters' SerializeSls / SerializeSlsLz4(group, ProcessorParseDelimiterNative&,
ProcessorParseTimestampNative&) through lc_host_chain3_serialize_sls: mode 0 (the device path where it applies, else
the four host calls) and mode 2 (its LZ4 block) against mode 1 (Process x 3 + SLSEventGroupSerializer::Serialize),
with all three processors' counters, including the fallbacks: several source events, EnableRawContent and refused
timestamp keys."""
import random
import time as _time

import pytest

from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_delim_timestamp_sls_cases as dtc  # noqa: E402

pytestmark = pytest.mark.gpu

OKEY = dtc.OKEY.decode()
SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"\d.*", "UnmatchedContentTreatment": "single_line"})]


def _procs(split_type, split_cfg, cfg, tcfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor(split_type, split_cfg),
            lc.HostProcessor("processor_parse_delimiter_native", dc.oracle_config(cfg)),
            lc.HostProcessor("processor_parse_timestamp_native", tcfg))


def _group(vals, offset_key=None, ns=True):
    g = {"metadata": {}, "tags": {"__topic__": "t"}, "events": []}
    if offset_key is not None:
        g["metadata"]["log.file.offset"] = offset_key
    for i, v in enumerate(vals):
        ev = {"type": 1, "timestamp": 1700000000 + i, "fileOffset": 1000 * i, "rawSize": len(v),
              "contents": {"content": v}}
        if ns:
            ev["timestampNanosecond"] = 17 + i
        g["events"].append(ev)
    return g


def _counters(p):  # the event counters (wall-time counters end in _ns)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _check_modes(split_type, split_cfg, cfg, tcfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, cfg, tcfg)
    b = _procs(split_type, split_cfg, cfg, tcfg)
    got = capi.host_chain3_serialize_sls(a[0], a[1], a[2], group, enable_ns, 0)
    want = capi.host_chain3_serialize_sls(b[0], b[1], b[2], group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    for k in range(3):
        assert _counters(a[k]) == _counters(b[k]), k
    c = _procs(split_type, split_cfg, cfg, tcfg)
    z = capi.host_chain3_serialize_sls(c[0], c[1], c[2], group, enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    for k in range(3):
        assert _counters(c[k]) == _counters(b[k]), k
    return want


def _host_lines(rng, n, fmt):
    """CSV lines whose times are far from the discard threshold of the real clock: an hour old (kept), ten days old
    (discarded), garbage (failed), some quoted, and lines that fail to parse, are short or are blank"""
    now = int(_time.time())
    pool = [dtc.render(fmt, now - 3600 - k).encode() for k in range(3)] + \
        [dtc.render(fmt, now - 864000).encode(), b"garbage", b""]
    lines = []
    for i in range(n):
        r = rng.random()
        v = dtc.field(rng.choice(pool), b",", ord('"'), rng)
        if r < 0.05:
            lines.append(b"")
        elif r < 0.1:
            lines.append(b'%d,"open' % i)
        elif r < 0.15:
            lines.append(b"%d" % i)
        else:
            lines.append(b"%d,%s,m%d" % (i, v, rng.randint(0, 9)))
    return b"\n".join(lines).decode("latin1")


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(split_type, split_cfg):
    rng = random.Random(5)
    for fmt in (dtc.YMD, "%s", dtc.COMMA_FMT):
        vals = [_host_lines(rng, 40, fmt) for _ in range(3)]
        tcfg = {"SourceKey": "time", "SourceFormat": fmt}
        for keep_fail in (False, True):
            cfg = dtc.config(["i", "time", "msg"], renamed="raw", keep_fail=keep_fail, copy_raw=True)
            for okey in (None, OKEY):
                for enable_ns in (False, True):
                    for ns in (False, True):
                        _check_modes(split_type, split_cfg, cfg, tcfg, _group(vals[:1], okey, ns=ns), enable_ns)
                # several source events: the host path
                _check_modes(split_type, split_cfg, cfg, tcfg, _group(vals, okey))
    vals = [_host_lines(rng, 40, dtc.YMD)]
    tcfg = {"SourceKey": "time", "SourceFormat": dtc.YMD}
    cfg = dtc.config(["i", "time", "msg"], renamed="raw", keep_fail=True, copy_raw=True)
    for tkey in ("raw", "__raw_log__", "content", "nope"):
        _check_modes(split_type, split_cfg, cfg, dict(tcfg, SourceKey=tkey), _group(vals, OKEY))
    # EnableRawContent: the host path
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), cfg, tcfg, _group(vals))
    # the offset key as tkey, and an overflow-form tkey outside discard mode: refused by the device calls, so the host
    # path runs
    _check_modes(split_type, split_cfg, cfg, dict(tcfg, SourceKey=OKEY), _group(vals, OKEY))
    _check_modes(split_type, split_cfg, cfg, dict(tcfg, SourceKey="__column3__"), _group(vals, OKEY))
    # errors: every event discarded, empty group
    old = "\n".join("%d,%s" % (i, dtc.render(dtc.YMD, int(_time.time()) - 864000)) for i in range(20))
    assert _check_modes(split_type, split_cfg, cfg, tcfg, _group([old]))[2] == "empty event group"
    assert _check_modes(split_type, split_cfg, cfg, tcfg, _group([]))[2] == "empty event group"
