"""GPU tier: the regex -> SLS hand-over.  lc_sls_serialize_regex_dev after lc_regex_parse_dev, lc_regex_parse_sls and
ProcessorParseRegexNative::SerializeSls against the oracle (ProcessorParseRegexNative over flat events +
sls_serialize_logs / sls_serialize_group), byte for byte, with the counters Process moves."""
import json
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import regex_sls_cases as rc  # noqa: E402
from tests.golden_util import input_with_metadata, load_cases  # noqa: E402

POISON, GUARD = 0xA5, 256


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _i32(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).cuda()


def _ptr(t):
    return t.data_ptr() if t is not None else None


def device_serialize(eng, buf, off, ln, cfg, times, nss):
    """regex_parse_dev -> sls_serialize_regex_dev into a poisoned buffer followed by guard bytes; checks the guard, the
    sizing query and the capacity error; returns (wire bytes, counters, status table or None)"""
    import torch

    import loongcollector_b200 as lc
    n = off.size
    keys = [k.encode() for k in cfg["keys"]]
    wl = rc.whole_line(cfg)
    d_buf = torch.from_numpy(np.concatenate([buf, np.zeros(16, np.uint8)])).cuda()
    d_off, d_len = _i32(off), _i32(ln)
    d_st = d_co = d_cl = None
    pitch = 0
    rx = None
    if not wl:
        rx = lc.Regex(cfg["regex"])
        pitch = rx.ngroups
        d_st = torch.full((n,), POISON, dtype=torch.uint8, device="cuda")
        d_co = torch.empty(max(n * pitch, 1), dtype=torch.int32, device="cuda")
        d_cl = torch.empty(max(n * pitch, 1), dtype=torch.int32, device="cuda")
        eng.regex_parse_dev(rx, d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, len(keys),
                            d_st.data_ptr(), d_co.data_ptr(), d_cl.data_ptr())
    d_t = _i32(times)
    d_ns = _i32(nss) if nss is not None else None
    args = (d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, _ptr(d_st), _ptr(d_co), _ptr(d_cl),
            pitch, keys, cfg["source"].encode(), rc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"],
            cfg["copy_raw"], wl)
    kw = dict(d_ev_time=d_t.data_ptr(), d_ev_time_ns=_ptr(d_ns))
    need, ctr0 = eng.sls_serialize_regex_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr], (d_st.cpu().numpy() if d_st is not None else None)


def _host_path(eng, buf, off, ln, cfg, times, nss):
    import loongcollector_b200 as lc
    rx = None if rc.whole_line(cfg) else lc.Regex(cfg["regex"])
    data, c = eng.regex_parse_sls(rx, buf, off, ln, times, [k.encode() for k in cfg["keys"]], cfg["source"].encode(),
                                  rc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"],
                                  rc.whole_line(cfg), ev_time_ns=nss)
    return data, [int(x) for x in c]


def _check(eng, cfg, lines, seed):
    buf, off, ln = rc.arena(lines)
    times, nss = rc.times_for(len(lines), seed)
    for ns in (nss, None):
        want, ctr, _ = rc.oracle_wire(lines, cfg, times, ns, ns is not None)
        got, c, _ = device_serialize(eng, buf, off, ln, cfg, times, ns)
        assert got == want, cfg
        assert c == rc.counters_of(ctr), (cfg, c, ctr)
    want, ctr, _ = rc.oracle_wire(lines, cfg, times, nss, True)
    data, c = _host_path(eng, buf, off, ln, cfg, times, nss)
    assert data == want and c == rc.counters_of(ctr), cfg


MATRIX = [(i, c) for i, c in rc.matrix()] + [(i, c) for i, c in rc.whole_line_matrix()] + \
    [(i, c) for i, c, _ in rc.random_cases(2, 12)]


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_device_tables_to_wire_bytes_match_oracle(eng, case):
    name, cfg = case
    rng = random.Random(sum(name.encode()))
    lines = [rc.random_line(rng) for _ in range(300)] + [b"", b"x 1 ", b" 7 ", b"nomatch"]
    _check(eng, cfg, lines, rng.randint(0, 1 << 30))


def test_pattern_without_groups(eng):
    _check(eng, rc.config([], "content", "raw", True, True, True, regex=r"\d+"), [b"12", b"", b"x", b"007"], 3)


def test_c2_shaped_batch(eng):
    """100 k nginx lines, ten keys, 1 % that do not match"""
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(100_000, seed=12)
    lines = [bytes(buf[o:o + n]) for o, n in zip(off.tolist(), ln.tolist())]
    for extra in ({}, {"keep_fail": True, "renamed": "raw", "copy_raw": True}):
        cfg = rc.config(synth.NGINX_KEYS, regex=synth.NGINX_PATTERN)
        cfg.update(extra)
        times, nss = rc.times_for(len(lines), 9)
        want, ctr, _ = rc.oracle_wire(lines, cfg, times, nss)
        got, c, st = device_serialize(eng, buf, off, ln, cfg, times, nss)
        assert (st != 0).sum() > 100
        assert got == want and c == rc.counters_of(ctr)


def test_every_length_and_alignment(eng):
    rng = random.Random(5)
    buf = bytearray()
    off, ln, lines = [], [], []
    for length in range(0, 301):
        for mis in range(16):
            line = rc.random_line(rng)
            while len(line) < length:
                line += b" 1 " + rc.random_line(rng)
            line = line[:length]
            buf += b"9 " * 8
            buf += b" " * ((mis - len(buf)) % 16)
            off.append(len(buf))
            ln.append(length)
            lines.append(line)
            buf += line
    buf += b" " * 32
    buf = np.frombuffer(bytes(buf), np.uint8)
    off, ln = np.array(off, np.uint32), np.array(ln, np.uint32)
    times, nss = rc.times_for(len(lines), 6)
    for cfg in (rc.config(["a", "content", "c"], "content", None, True, True, True),
                rc.config(["a"], "content", "raw", True, True, False, regex=rc.WHOLE_LINE)):
        want, ctr, _ = rc.oracle_wire(lines, cfg, times, nss)
        got, c, _ = device_serialize(eng, buf, off, ln, cfg, times, nss)
        assert got == want and c == rc.counters_of(ctr)


def test_long_event_among_short_ones(eng):
    """a >= 64 KB line takes the regex stage's follow-up kernel; its captures feed the record like any other"""
    rng = random.Random(8)
    short = [rc.random_line(rng) for _ in range(62)]
    long_ok = b"w 123 " + b"x" * (100 << 10)
    long_bad = b"w x" + b"y" * (70 << 10)
    lines = short[:20] + [long_ok] + short[20:40] + [long_bad] + short[40:]
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, True)
    _check(eng, cfg, lines, 7)


def test_host_buffers_across_pipeline_chunks(eng):
    """> 96 MB of C2 lines: several upload chunks; the bytes equal the device-resident path and the counters equal
    the status table's"""
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(420_000, seed=23)
    assert buf.size > 100 << 20
    cfg = rc.config(synth.NGINX_KEYS, "content", "raw", True, True, True, regex=synth.NGINX_PATTERN)
    times, nss = rc.times_for(off.size, 10)
    ref, c_dev, st = device_serialize(eng, buf, off, ln, cfg, times, nss)
    data, c = _host_path(eng, buf, off, ln, cfg, times, nss)
    assert data == ref and c == c_dev
    assert c == [off.size, int((st == 1).sum()), 0] and c[1] > 0


# ---- host class: SerializeSls == Process + SLSEventGroupSerializer::Serialize on the same in-memory group
def _host_pair(cfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor("processor_parse_regex_native", cfg),
            lc.HostProcessor("processor_parse_regex_native", cfg))


def _check_host(cfg, group, oracle_too=True):
    fast, ref = _host_pair(cfg)
    for ns in (False, True):
        got = fast.serialize_sls(group, ns)
        want = ref.serialize_sls(group, ns, process_then_serialize=True)
        assert got == want, (cfg, ns, got[1], want[1])
        if oracle_too:
            g = orc.Group.from_json(json.loads(json.dumps(group)))
            orc.ProcessorParseRegexNative(cfg).process(g)
            o, oerr = orc.sls_serialize_group(g, ns)
            assert want[0] == o and (want[1] is None) == (oerr is None), (cfg, ns, want[1], oerr)
    # the processor's own counters; the b200_*_ns ones time the phases of the batched Process path
    own = lambda p: {k: v for k, v in p.counters().items() if not k.startswith("b200_")}  # noqa: E731
    assert own(fast) == own(ref)


def test_host_serialize_sls_on_reference_fixtures():
    n = 0
    for case in load_cases("regex"):
        if case["pipeline"][0]["type"] != "processor_parse_regex_native" or len(case["pipeline"]) != 1:
            continue
        _check_host(case["pipeline"][0]["config"], input_with_metadata(case), oracle_too=False)
        n += 1
    assert n >= 7


WHOLE = [c for _, c in rc.whole_line_matrix()]


def test_host_serialize_sls_on_random_groups():
    rng = random.Random(31)
    for k in range(60):
        cfg = rc.random_config(rng) if k % 4 else WHOLE[k % len(WHOLE)]
        evs = []
        for _ in range(rng.choice([0, 1, 5, 40])):
            ev = {"type": 1, "timestamp": rng.choice([5, 1700000000]),
                  "contents": {cfg["source"]: rc.random_line(rng).decode()}}
            if rng.random() < 0.5:
                ev["timestampNanosecond"] = rng.randint(0, 999999999)
            if k % 5 == 4 and rng.random() < 0.3:  # not flat: Process + Serialize
                ev["contents"]["other"] = "x"
            evs.append(ev)
        root = {"events": evs, "tags": {"__topic__": "t", "host.name": "h" * rng.choice([1, 100])}}
        if k % 7 == 6:
            root["metadata"] = {"log.file.offset": "__offset__"}
        _check_host(rc.oracle_config(cfg), root)


def test_host_serialize_sls_size_limit_and_empty_groups():
    cfg = rc.oracle_config(rc.config(["a", "b", "c"]))
    big = {"events": [{"type": 1, "timestamp": 1, "contents": {"content": "w 1 " + "x" * 4096}} for _ in range(3000)]}
    _check_host(cfg, big, oracle_too=True)  # > 10 MB: the size-limit error
    failing = {"events": [{"type": 1, "timestamp": 1, "contents": {"content": "no match"}}]}
    _check_host(cfg, failing)  # every event erased: "empty event group"
    _check_host(cfg, {"events": []})
    whole = rc.oracle_config(rc.config([], "content", regex=rc.WHOLE_LINE))
    _check_host(whole, {"events": [{"type": 1, "timestamp": 1, "contents": {"content": "abc"}}]})  # all empty logs
