"""GPU tier: the split -> regex -> filter -> SLS chain.  lc_sls_serialize_split_regex_filter_dev over the device
tables of lc_split_lines_dev / lc_multiline_split_dev and lc_regex_parse_dev, the four host calls, and the splitters'
SerializeSls(group, regex, filter) against the oracle chain (its splitter, ProcessorParseRegexNative and
ProcessorFilterNative, then sls_serialize_logs) and against Process x 3 + Serialize, byte for byte and counter for
counter."""
import random
import zlib

import pytest

pytestmark = pytest.mark.gpu

from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402
from tests import split_regex_filter_sls_cases as fc  # noqa: E402
from tests import split_regex_sls_cases as src  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = fc.OKEY
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


def _filter(fcfg, prog=None):
    import loongcollector_b200 as lc
    leaves, p = fc.program(fcfg)
    return lc.capi.Filter([(k, lc.Regex(r)) for k, r in leaves], p if prog is None else prog)


def device_chain(eng, val, cfg, filt, okey, pos, time, ns):
    """split, regex, filter and serialise on the device into a poisoned buffer with guard bytes; checks the sizing
    query, the capacity refusal and the guard; returns (wire bytes, counters[4])"""
    import torch

    import loongcollector_b200 as lc
    d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
    if val:
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    cap = max(len(val), 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), cap)
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
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    need, ctr0 = eng.sls_serialize_split_regex_filter_dev(*args, keys, skey, filt, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_regex_filter_dev(*args, keys, skey, filt, **kw, d_out=d_out.data_ptr(),
                                                     out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_regex_filter_dev(*args, keys, skey, filt, **kw, d_out=d_out.data_ptr(),
                                                        out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr]


MATRIX = list(fc.matrix())


@pytest.mark.parametrize("fid", list(fc.FILTERS))
def test_dev_chain_matrix(eng, fid):
    filt = _filter(fc.FILTERS[fid])
    for cid, cfg in MATRIX:
        rng = random.Random(zlib.crc32((cid + fid).encode()))
        val = src.random_lines_value(rng, 50)
        t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + len(fid)) % len(sc.POSITIONS)]
        for okey in (None, OKEY):
            want, wctr, _, _ = fc.oracle_chain(val, SPLIT, cfg, fc.FILTERS[fid], t, ns, pos, okey)
            got, ctr = device_chain(eng, val, cfg, filt, okey, pos, t, ns)
            assert got == want and ctr == wctr, (cid, fid, okey)


@pytest.mark.parametrize("fid", ["rule_regex_key", "rule_offset", "nested", "rule_missing", "bypass"])
@pytest.mark.parametrize("size", [0, 1, 512 * 1024])
def test_host_calls(eng, fid, size):
    rng = random.Random(size)
    val = src.random_lines_value(rng, max(1, size // 60))[:size] if size else b""
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, True)
    filt = _filter(fc.FILTERS[fid])
    tail = b"\x1a\x05topic"
    for okey in (None, OKEY):
        want, wctr, _, npieces = fc.oracle_chain(val, SPLIT, cfg, fc.FILTERS[fid], 1700000000, 42, 4096, okey)
        kw = dict(src.device_args(cfg), offset_key=okey, src_pos=4096, time=1700000000, time_ns=42)
        keys, skey = kw.pop("keys"), kw.pop("source_key")
        data, nev, ctr = eng.split_regex_filter_parse_sls(_rx(cfg), val, 10, keys, skey, filt, **kw)
        assert data == want and [int(x) for x in ctr] == wctr and nev == npieces
        block, raw, nev2, ctr2 = eng.split_regex_filter_parse_sls_lz4(_rx(cfg), val, 10, keys, skey, filt, **kw,
                                                                      tail=tail)
        assert raw == len(want) + len(tail) and nev2 == nev and list(ctr2) == list(ctr)
        assert lz4_block.decode(block) == want + tail
        if fid == "bypass":  # BYPASS: the unfiltered chain's bytes
            plain, _, pctr = eng.split_regex_parse_sls(_rx(cfg), val, 10, keys, skey, **kw)
            assert plain == data and list(pctr) == [int(x) for x in ctr[:3]]


@pytest.mark.parametrize("discard", [False, True])
def test_multiline_host_calls(eng, discard):
    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    buf, _, _ = synth.java_stack_records(2000)
    val = buf.tobytes()
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
            "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    fcfg = {"ConditionExp": {"operator": "and", "operands": [
        {"key": "level", "exp": "ERROR|WARN", "type": "regex"},
        {"operator": "not", "operands": [{"key": OKEY.decode(), "exp": r"\d*[05]", "type": "regex"}]}]}}
    filt = _filter(fcfg)
    want, wctr, mctr, npieces = fc.oracle_chain(val, mcfg, cfg, fcfg, 1700000000, 9, 77, OKEY, multiline=True)
    from oracle import oracle as orc
    p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
    h = tuple(lc.Regex(r.pattern) if r is not None else None for r in (p.start, p.cont, p.end)) + (p.opts.discard,)
    kw = dict(src.device_args(cfg), offset_key=OKEY, src_pos=77, time=1700000000, time_ns=9)
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    data, nev, ctr, ml = eng.multiline_split_regex_filter_parse_sls(_rx(cfg), val, *h, keys, skey, filt, **kw)
    assert data == want and nev == npieces and [int(x) for x in ctr] == wctr
    assert int(ml[0]) == mctr["matched_events"] and int(ml[2]) == mctr["unmatched_lines"]
    block, raw, nev2, ctr2, ml2 = eng.multiline_split_regex_filter_parse_sls_lz4(_rx(cfg), val, *h, keys, skey, filt,
                                                                                 **kw, tail=b"\x22\x01s")
    assert lz4_block.decode(block) == want + b"\x22\x01s" and list(ml2) == list(ml) and list(ctr2) == list(ctr)


def test_long_pieces_and_every_piece_removed(eng):
    rng = random.Random(11)
    val = src.random_lines_value(rng, 40, long_every=9)
    cfg = rc.config(["a", "b", "c"], "content", None, True, False, True)
    for fid in ("rule_source_key", "nested", "rule_missing"):
        filt = _filter(fc.FILTERS[fid])
        want, wctr, _, _ = fc.oracle_chain(val, SPLIT, cfg, fc.FILTERS[fid], 7, None, 10 ** 9, OKEY)
        assert device_chain(eng, val, cfg, filt, OKEY, 10 ** 9, 7, None) == (want, wctr)
    # every piece removed: no bytes; the LZ4 call returns the block of the tail alone
    filt = _filter(fc.FILTERS["rule_missing"])
    kw = dict(src.device_args(cfg), offset_key=OKEY, src_pos=5, time=7)
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    data, nev, ctr = eng.split_regex_filter_parse_sls(_rx(cfg), val, 10, keys, skey, filt, **kw)
    assert data == b"" and nev > 0 and int(ctr[3]) == int(ctr[0])
    block, raw, _, _ = eng.split_regex_filter_parse_sls_lz4(_rx(cfg), val, 10, keys, skey, filt, **kw, tail=b"\x1a\x01t")
    assert raw == 3 and lz4_block.decode(block) == b"\x1a\x01t"


def test_c2_nginx_lines(eng):
    from loongcollector_b200 import synth
    buf, _, _ = synth.nginx_lines(20000)
    val = buf.tobytes()
    cfg = rc.config(synth.NGINX_KEYS, "content", None, False, False, False, regex=synth.NGINX_PATTERN)
    for fcfg in ({"FilterKey": ["status"], "FilterRegex": [r"[45]\d\d"]},
                 {"FilterKey": [synth.NGINX_KEYS[-1]], "FilterRegex": ["no-agent"]}):
        filt = _filter(fcfg)
        want, wctr, _, npieces = fc.oracle_chain(val, SPLIT, cfg, fcfg, 1700000000, None, 1 << 33, OKEY)
        assert device_chain(eng, val, cfg, filt, OKEY, 1 << 33, 1700000000, None) == (want, wctr)
        kw = dict(src.device_args(cfg), offset_key=OKEY, src_pos=1 << 33, time=1700000000)
        keys, skey = kw.pop("keys"), kw.pop("source_key")
        data, nev, ctr = eng.split_regex_filter_parse_sls(_rx(cfg), val, 10, keys, skey, filt, **kw)
        assert data == want and nev == npieces and [int(x) for x in ctr] == wctr


def test_refusals(eng):
    import loongcollector_b200 as lc
    cfg = rc.config(["a", "b", "c"])
    kw = dict(src.device_args(cfg))
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    many = _filter({"FilterKey": ["k%d" % i for i in range(33)], "FilterRegex": [".*"] * 33})
    bad = [many] + [_filter({"FilterKey": ["a"], "FilterRegex": [".*"]}, prog=p)
                    for p in ([fc.AND], [0, 0], [1], [0, 7], [0] * 129)]
    bad.append(lc.capi.Filter([(b"a", None)], [0]))  # a missing leaf regex
    for f in bad:
        for call in (lambda: eng.split_regex_filter_parse_sls(_rx(cfg), b"a 1 b\n", 10, keys, skey, f, **kw),
                     lambda: eng.split_regex_filter_parse_sls_lz4(_rx(cfg), b"a 1 b\n", 10, keys, skey, f, **kw),
                     lambda: eng.multiline_split_regex_filter_parse_sls(_rx(cfg), b"a 1 b\n", None, None, None, False,
                                                                        keys, skey, f, **kw),
                     lambda: eng.sls_serialize_split_regex_filter_dev(None, 0, None, None, 0, None, None, None, 3,
                                                                      keys, skey, f, **kw)):
            with pytest.raises(lc.LcError) as ei:
                call()
            assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


# ---- the host classes through lc_host_chain3_serialize_sls
def _procs(split_type, split_cfg, rcfg, fcfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor(split_type, split_cfg),
            lc.HostProcessor("processor_parse_regex_native", dict(rc.oracle_config(rcfg))),
            lc.HostProcessor("processor_filter_regex_native", fcfg))


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


def _counters(p):  # the event counters (the regex class's phase timers are wall time)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _check_modes(split_type, split_cfg, rcfg, fcfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, rcfg, fcfg)
    b = _procs(split_type, split_cfg, rcfg, fcfg)
    got = capi.host_chain3_serialize_sls(a[0], a[1], a[2], group, enable_ns, 0)
    want = capi.host_chain3_serialize_sls(b[0], b[1], b[2], group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert _counters(a[0]) == _counters(b[0]) and _counters(a[1]) == _counters(b[1])
    c = _procs(split_type, split_cfg, rcfg, fcfg)
    z = capi.host_chain3_serialize_sls(c[0], c[1], c[2], group, enable_ns, 2)
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
    rcfg = rc.config(["a", "b", "c"], "content", "raw", True, True, True)
    for fid in ("bypass", "rule_regex_key", "rule_offset", "include", "nested", "rule_missing"):
        for okey in (None, OKEY.decode()):
            _check_modes(split_type, split_cfg, rcfg, fc.FILTERS[fid], _group(vals[:1], okey))  # one chunk: LZ4
            _check_modes(split_type, split_cfg, rcfg, fc.FILTERS[fid], _group(vals, okey))      # several events
    # fallbacks: DiscardingNonUTF8, raw content, a regex on another key, a non-flat group
    fcfg = fc.FILTERS["nested"]
    _check_modes(split_type, split_cfg, rcfg, dict(fcfg, DiscardingNonUTF8=True), _group(vals[:1], OKEY.decode()))
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), rcfg, fcfg, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(rcfg, source="other"), fcfg, _group(vals[:1]))
    _check_modes(split_type, split_cfg, rcfg, fcfg, _group(vals[:1], extra={"x": "y"}))
    # errors: every event removed by the filter, empty group
    assert _check_modes(split_type, split_cfg, rcfg, fc.FILTERS["rule_missing"], _group(vals))[2] == \
        "empty event group"
    assert _check_modes(split_type, split_cfg, rcfg, fcfg, _group([]))[2] == "empty event group"
