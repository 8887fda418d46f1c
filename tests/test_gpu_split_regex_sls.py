"""GPU tier: the split -> regex -> SLS chain.  lc_sls_serialize_split_regex_dev over the device tables of
lc_split_lines_dev / lc_multiline_split_dev and lc_regex_parse_dev, the four host calls, and the splitters'
SerializeSls(group, regex) against the oracle chain (its splitter, then its ProcessorParseRegexNative, then
sls_serialize_logs) and against Process + Process + Serialize, byte for byte and counter for counter."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402
from tests import split_regex_sls_cases as src  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = src.OKEY
SPLIT = {"SourceKey": "content", "SplitChar": 10}


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _rx(cfg):
    import loongcollector_b200 as lc
    return None if rc.whole_line(cfg) else lc.Regex(cfg["regex"])


def _ml_handles(cfg):
    import loongcollector_b200 as lc
    p = orc.ProcessorSplitMultilineLogStringNative(cfg)
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


def device_chain(eng, val, cfg, okey, pos, time, ns, ml=None):
    """split, regex and serialise on the device into a poisoned buffer with guard bytes; checks the sizing query, the
    capacity refusal and the guard; returns (wire bytes, counters)"""
    import torch

    import loongcollector_b200 as lc
    d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
    if val:
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    cap = max(len(val), 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    if ml is None:
        n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), cap)
    else:
        d_fl = torch.empty(cap, dtype=torch.uint8, device="cuda")
        n, _ = eng.multiline_split_dev(d.data_ptr(), len(val), *ml, d_off.data_ptr(), d_len.data_ptr(),
                                       d_fl.data_ptr(), cap)
    rx = _rx(cfg)
    G = 0 if rx is None else rx.ngroups
    tabs = (None, None, None)
    if rx is not None and n:
        st = torch.empty(n, dtype=torch.uint8, device="cuda")
        co = torch.empty(n * G + 1, dtype=torch.int32, device="cuda")
        cl = torch.empty(n * G + 1, dtype=torch.int32, device="cuda")
        eng.regex_parse_dev(rx, d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, len(cfg["keys"]),
                            st.data_ptr(), co.data_ptr(), cl.data_ptr())
        tabs = (st.data_ptr(), co.data_ptr(), cl.data_ptr())
    args = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n) + tabs + (G,)
    kw = dict(src.device_args(cfg), offset_key=okey, src_pos=pos, time=time, time_ns=ns)
    need, ctr0 = eng.sls_serialize_split_regex_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr]


CASES = list(src.matrix())


@pytest.mark.parametrize("cid,cfg", CASES, ids=[c[0] for c in CASES])
def test_dev_chain_matrix(eng, cid, cfg):
    rng = random.Random(hash(cid) & 0xFFFF)
    val = src.random_lines_value(rng, 60)
    for i, okey in enumerate(src.OFFSET_KEYS[:3] if "offset" not in cid else [OKEY]):
        t, ns = sc.TIMES[i % len(sc.TIMES)]
        pos = sc.POSITIONS[(3 * i + len(cid)) % len(sc.POSITIONS)]
        want, wctr, _, _ = src.oracle_chain(val, SPLIT, cfg, t, ns, pos, okey)
        got, ctr = device_chain(eng, val, cfg, okey, pos, t, ns)
        assert got == want and ctr == wctr, (cid, okey)


@pytest.mark.parametrize("okey", src.OFFSET_KEYS, ids=lambda k: "none" if k is None else k.decode() or "empty")
def test_offset_keys_against_regex_keys(eng, okey):
    rng = random.Random(7)
    val = src.random_lines_value(rng, 80, trailing=True)
    for f in range(8):
        cfg = rc.config(["a", "raw", "c"], "content", "raw" if f & 1 else "__raw_log__", bool(f & 1), bool(f & 2),
                        bool(f & 4))
        want, wctr, _, _ = src.oracle_chain(val, SPLIT, cfg, 1 << 29, 5, 123456789, okey)
        assert device_chain(eng, val, cfg, okey, 123456789, 1 << 29, 5) == (want, wctr)


def test_refusals(eng):
    """an offset key equal to SourceKey is refused by the device-fed and the host-buffer calls"""
    import loongcollector_b200 as lc
    cfg = rc.config(["a", "b", "c"])
    kw = dict(src.device_args(cfg), offset_key=b"content")
    calls = [lambda: eng.split_regex_parse_sls(_rx(cfg), b"a 1 b\n", 10, **kw),
             lambda: eng.split_regex_parse_sls_lz4(_rx(cfg), b"a 1 b\n", 10, **kw),
             lambda: eng.multiline_split_regex_parse_sls(_rx(cfg), b"a 1 b\n", None, None, None, False, **kw),
             lambda: eng.sls_serialize_split_regex_dev(None, 0, None, None, 0, None, None, None, 3, **kw)]
    for call in calls:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


@pytest.mark.parametrize("size", [0, 1, 512 * 1024])
def test_host_calls(eng, size):
    rng = random.Random(size)
    val = src.random_lines_value(rng, max(1, size // 60), long_every=0)[:size] if size else b""
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, True)
    tail = b"\x1a\x05topic"
    for okey in (None, OKEY):
        want, wctr, _, npieces = src.oracle_chain(val, SPLIT, cfg, 1700000000, 42, 4096, okey)
        kw = dict(src.device_args(cfg), offset_key=okey, src_pos=4096, time=1700000000, time_ns=42)
        data, nev, ctr = eng.split_regex_parse_sls(_rx(cfg), val, 10, **kw)
        assert data == want and [int(x) for x in ctr] == wctr and nev == npieces
        block, raw, nev2, ctr2 = eng.split_regex_parse_sls_lz4(_rx(cfg), val, 10, **kw, tail=tail)
        assert raw == len(want) + len(tail) and nev2 == nev and list(ctr2) == list(ctr)
        assert lz4_block.decode(block) == want + tail


def test_long_pieces_among_short_ones(eng):
    rng = random.Random(11)
    val = src.random_lines_value(rng, 40, long_every=9)
    cfg = rc.config(["a", "b", "c"], "content", None, True, False, True)
    want, wctr, _, npieces = src.oracle_chain(val, SPLIT, cfg, 7, None, 10 ** 9, OKEY)
    assert device_chain(eng, val, cfg, OKEY, 10 ** 9, 7, None) == (want, wctr)
    data, nev, ctr = eng.split_regex_parse_sls(_rx(cfg), val, 10, **src.device_args(cfg), offset_key=OKEY,
                                               src_pos=10 ** 9, time=7)
    assert data == want and nev == npieces


def test_c2_nginx_lines(eng):
    from loongcollector_b200 import synth
    buf, _, _ = synth.nginx_lines(20000)
    val = buf.tobytes()
    cfg = rc.config(synth.NGINX_KEYS, "content", None, False, False, False, regex=synth.NGINX_PATTERN)
    want, wctr, _, npieces = src.oracle_chain(val, SPLIT, cfg, 1700000000, None, 1 << 33, OKEY)
    assert device_chain(eng, val, cfg, OKEY, 1 << 33, 1700000000, None) == (want, wctr)
    data, nev, ctr = eng.split_regex_parse_sls(_rx(cfg), val, 10, **src.device_args(cfg), offset_key=OKEY,
                                               src_pos=1 << 33, time=1700000000)
    assert data == want and nev == npieces and [int(x) for x in ctr] == wctr


@pytest.mark.parametrize("discard", [False, True])
def test_c3_java_records(eng, discard):
    from loongcollector_b200 import synth
    buf, _, _ = synth.java_stack_records(2000)
    val = buf.tobytes()
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
            "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    want, wctr, mctr, npieces = src.oracle_chain(val, mcfg, cfg, 1700000000, 9, 77, OKEY, multiline=True)
    h = _ml_handles(mcfg)
    assert device_chain(eng, val, cfg, OKEY, 77, 1700000000, 9, ml=h) == (want, wctr)
    kw = dict(src.device_args(cfg), offset_key=OKEY, src_pos=77, time=1700000000, time_ns=9)
    data, nev, ctr, ml = eng.multiline_split_regex_parse_sls(_rx(cfg), val, *h, **kw)
    assert data == want and nev == npieces and [int(x) for x in ctr] == wctr
    assert int(ml[0]) == mctr["matched_events"] and int(ml[2]) == mctr["unmatched_lines"]
    assert int(ml[1]) - int(ml[2]) == mctr["matched_lines"]
    block, raw, nev2, ctr2, ml2 = eng.multiline_split_regex_parse_sls_lz4(_rx(cfg), val, *h, **kw, tail=b"\x22\x01s")
    assert lz4_block.decode(block) == want + b"\x22\x01s" and list(ml2) == list(ml) and nev2 == nev


# ---- the host classes through lc_host_chain_serialize_sls
def _procs(split_type, split_cfg, rcfg):
    import loongcollector_b200 as lc
    c = dict(rc.oracle_config(rcfg))
    return lc.HostProcessor(split_type, split_cfg), lc.HostProcessor("processor_parse_regex_native", c)


def _group(vals, offset_key=None, raw=False, extra=None):
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


def _counters(p):  # the event counters (the regex class's phase timers are wall time)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _check_modes(split_type, split_cfg, rcfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, rcfg)
    b = _procs(split_type, split_cfg, rcfg)
    got = capi.host_chain_serialize_sls(a[0], a[1], group, enable_ns, 0)
    want = capi.host_chain_serialize_sls(b[0], b[1], group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert _counters(a[0]) == _counters(b[0]) and _counters(a[1]) == _counters(b[1])
    c = _procs(split_type, split_cfg, rcfg)
    z = capi.host_chain_serialize_sls(c[0], c[1], group, enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    assert _counters(c[0]) == _counters(b[0]) and _counters(c[1]) == _counters(b[1])
    return want


SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"\w+ \d+.*", "UnmatchedContentTreatment": "single_line"})]


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(eng, split_type, split_cfg):
    rng = random.Random(5)
    vals = [src.random_lines_value(rng, 30).decode("ascii") for _ in range(3)]
    cfgs = [rc.config(["a", "b", "c"], "content", "raw", True, True, True),
            rc.config(["a", OKEY.decode(), "c"], "content", None, False, True, False),
            rc.config(["content"], "content", None, False, False, False, regex=rc.WHOLE_LINE)]
    for rcfg in cfgs:
        for okey in (None, OKEY.decode(), ""):
            _check_modes(split_type, split_cfg, rcfg, _group(vals[:1], okey))  # the one-chunk LZ4 device path
            _check_modes(split_type, split_cfg, rcfg, _group(vals, okey))      # several source events
    # fallbacks: raw content, another regex SourceKey, offset key = SourceKey, a non-flat group, an empty value
    rcfg = cfgs[0]
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), rcfg, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(rcfg, source="other"), _group(vals[:1]))
    _check_modes(split_type, split_cfg, rcfg, _group(vals[:1], "content"))
    _check_modes(split_type, split_cfg, rcfg, _group(vals[:1], extra={"x": "y"}))
    _check_modes(split_type, split_cfg, rcfg, _group([""]))
    # errors: empty group, all empty logs, size limit
    assert _check_modes(split_type, split_cfg, rcfg, _group([]))[2] == "empty event group"
    erased = rc.config(["a", "b", "c"], "content", None, False, False, False, regex=r"(\d)(\d)(\d)zzz")
    assert _check_modes(split_type, split_cfg, erased, _group(vals[:1]))[2] == "empty event group"
    nokeys = rc.config([], "content", None, False, False, False)
    assert _check_modes(split_type, split_cfg, nokeys, _group(vals[:1]))[2] == "all empty logs"
    big = ("w 1 " + "x" * 1000 + "\n") * 6000
    err = _check_modes(split_type, split_cfg, rcfg, _group([big, big]))[2]
    assert err is not None and err.startswith("log group exceeds size limit")
