"""GPU tier: the split -> regex -> timestamp -> SLS chain.  The device-fed composition (lc_split_lines_dev,
lc_regex_parse_dev, lc_split_regex_timestamp_tap_dev, lc_timestamp_parse_dev with one group,
lc_sls_serialize_split_regex_timestamp_dev), the four host calls and the splitters' SerializeSls(group, regex,
timestamp) against the host build of the chain (tests/emul/split_regex_timestamp_sls.py, itself checked against the
oracle on the CPU tier) and against Process x 3 + Serialize, byte for byte and counter for counter."""
import random
import time as _time
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402
from tests import split_regex_timestamp_sls_cases as tc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_regex_timestamp_sls as emul  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = tc.OKEY
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


def _ts(fmt):
    import loongcollector_b200 as lc
    return lc.Timestamp(fmt)


def emulated(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, off=None, ln=None, tables=None, pitch=0):
    """the host build of the chain over the oracle's split and regex tables (or the given ones)"""
    if off is None:
        off, ln = orc.split_lines(val, 10)
        tables, pitch = tc.tables_of(val, off, ln, cfg)
    a = tc.device_args(cfg)
    return emul.serialize(val, off, ln, tables, pitch, a["keys"], a["source_key"], a["renamed_key"], a["keep_fail"],
                          a["keep_succeed"], a["copy_raw"], a["whole_line"], okey, pos, t, ns, tkey, fmt, now, di,
                          enable_ns)


def device_chain(eng, val, cfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns):
    """split, regex, tap, timestamp passes and serialiser on the device into a poisoned buffer with guard bytes;
    checks the sizing query, the capacity refusal and the guard; returns (wire bytes, counters[8], tap table,
    timestamp status, (off, len, regex tables, pitch) of the device)"""
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
    tabs, host_tabs = (None, None, None), None
    if rx is not None and n:
        st = torch.empty(n, dtype=torch.uint8, device="cuda")
        co = torch.empty(n * G + 1, dtype=torch.int32, device="cuda")
        cl = torch.empty(n * G + 1, dtype=torch.int32, device="cuda")
        eng.regex_parse_dev(rx, d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, len(cfg["keys"]),
                            st.data_ptr(), co.data_ptr(), cl.data_ptr())
        tabs = (st.data_ptr(), co.data_ptr(), cl.data_ptr())
        host_tabs = (st.cpu().numpy(), co[:n * G].cpu().numpy().view(np.uint32),
                     cl[:n * G].cpu().numpy().view(np.uint32))
    args = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n) + tabs + (G,)
    kw = dict(tc.device_args(cfg), offset_key=okey)
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    m = max(n, 1)
    v_off = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    v_len = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    eng.split_regex_timestamp_tap_dev(*args, keys, skey, tkey, v_off.data_ptr(), v_len.data_ptr(), **kw)
    grp = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    sec = torch.empty(m, dtype=torch.int64, device="cuda")
    nsec = torch.empty(m, dtype=torch.int32, device="cuda")
    tst = torch.full((m,), 9, dtype=torch.uint8, device="cuda")
    tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
    eng.timestamp_parse_dev(ts, d.data_ptr(), len(val), v_off.data_ptr(), v_len.data_ptr(), n, grp.data_ptr(), 1, now,
                            di, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(), tcnt.data_ptr())
    tsa = (tst.data_ptr(), sec.data_ptr(), nsec.data_ptr())
    kw.update(src_pos=pos, time=t, time_ns=ns, enable_ns=enable_ns)
    need, ctr0 = eng.sls_serialize_split_regex_timestamp_dev(*args, keys, skey, *tsa, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_regex_timestamp_dev(*args, keys, skey, *tsa, **kw, d_out=d_out.data_ptr(),
                                                        out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_regex_timestamp_dev(*args, keys, skey, *tsa, **kw, d_out=d_out.data_ptr(),
                                                           out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    tap = (v_off[:n].cpu().numpy().view(np.uint32), v_len[:n].cpu().numpy().view(np.uint32))
    dev = (d_off[:n].cpu().numpy().view(np.uint32), d_len[:n].cpu().numpy().view(np.uint32), host_tabs, G)
    return bytes(host[:need]), [int(x) for x in ctr], tap, tst[:n].cpu().numpy(), dev


CONFIGS = list(tc.configs())


@pytest.mark.parametrize("fmt", [tc.NGINX_FMT, tc.F_FMT, "%s"])
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_dev_chain_matrix(eng, case, fmt):
    cid, cfg, tkey = case
    ts = _ts(fmt)
    rng = random.Random(zlib.crc32((cid + fmt).encode()))
    val = tc.lines_value(rng, fmt, 80)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di, enable_ns in ((43200, True), (-1, False)):
            ns_in = ns if enable_ns else None
            want, wctr, wst, wtap = emulated(val, cfg, tkey, fmt, tc.NOW, di, enable_ns, okey, pos, t, ns_in)
            got, ctr, tap, st, _ = device_chain(eng, val, cfg, tkey, ts, tc.NOW, di, enable_ns, okey, pos, t, ns_in)
            assert got == want and ctr == wctr, (cid, fmt, okey, di)
            assert np.array_equal(tap[0], wtap[0]) and np.array_equal(tap[1], wtap[1]) and np.array_equal(st, wst)


def _host(eng, call, val, cfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns, tail=None, ml=None):
    kw = dict(tc.device_args(cfg), offset_key=okey, src_pos=pos, time=t, time_ns=ns, discard_interval=di,
              enable_ns=enable_ns)
    keys, skey = kw.pop("keys"), kw.pop("source_key")
    head = [_rx(cfg), val] + (list(ml) if ml else [10])
    if tail is not None:
        kw["tail"] = tail
    return call(*head, keys, skey, tkey, ts, now, **kw)


@pytest.mark.parametrize("size", [0, 1, 300, 4096, 65536, 512 * 1024])
def test_host_calls(eng, size):
    rng = random.Random(size)
    val = tc.lines_value(rng, tc.NGINX_FMT, max(1, size // 40))[:size] if size else b""
    cfg = rc.config(tc.KEYS, "content", "raw", True, True, True, regex=tc.PATTERN)
    ts = _ts(tc.NGINX_FMT)
    tail = b"\x1a\x05topic"
    for tkey in (b"time", b"raw"):
        for okey in (None, OKEY):
            want, wctr, _, _ = emulated(val, cfg, tkey, tc.NGINX_FMT, tc.NOW, 43200, True, okey, 4096, 1700000000, 42)
            npieces = orc.split_lines(val, 10)[0].size
            data, nev, ctr = _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, tkey, ts, tc.NOW, 43200, True,
                                   okey, 4096, 1700000000, 42)
            assert data == want and [int(x) for x in ctr] == wctr and nev == npieces, (size, tkey, okey)
            block, raw, nev2, ctr2 = _host(eng, eng.split_regex_timestamp_parse_sls_lz4, val, cfg, tkey, ts, tc.NOW,
                                           43200, True, okey, 4096, 1700000000, 42, tail=tail)
            assert raw == len(want) + len(tail) and nev2 == nev and list(ctr2) == list(ctr)
            assert lz4_block.decode(block) == want + tail
            # the device-fed composition agrees
            if size:
                assert device_chain(eng, val, cfg, tkey, ts, tc.NOW, 43200, True, okey, 4096, 1700000000, 42)[:2] == \
                    (want, wctr)


@pytest.mark.parametrize("discard", [False, True])
def test_multiline_host_calls(eng, discard):
    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    from tests import split_regex_sls_cases as src
    buf, _, _ = synth.java_stack_records(2000)
    val = buf.tobytes()
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
            "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    now, di = 1790000000, 86400 * 365 * 3
    want, wctr, mctr, npieces = tc.oracle_chain(val, mcfg, cfg, b"time", tc.F_FMT, now, di, 1700000000, 9, 77, OKEY,
                                                multiline=True)
    p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
    h = tuple(lc.Regex(r.pattern) if r is not None else None for r in (p.start, p.cont, p.end)) + (p.opts.discard,)
    ts = _ts(tc.F_FMT)
    data, nev, ctr, ml = _host(eng, eng.multiline_split_regex_timestamp_parse_sls, val, cfg, b"time", ts, now, di,
                               True, OKEY, 77, 1700000000, 9, ml=h)
    assert data == want and nev == npieces and [int(x) for x in ctr] == wctr
    assert int(ml[0]) == mctr["matched_events"] and int(ml[2]) == mctr["unmatched_lines"]
    block, raw, nev2, ctr2, ml2 = _host(eng, eng.multiline_split_regex_timestamp_parse_sls_lz4, val, cfg, b"time", ts,
                                        now, di, True, OKEY, 77, 1700000000, 9, tail=b"\x22\x01s", ml=h)
    assert lz4_block.decode(block) == want + b"\x22\x01s" and list(ml2) == list(ml) and list(ctr2) == list(ctr)


def test_whole_chunk_discarded(eng):
    old = tc.render(tc.NGINX_FMT, tc.NOW - 86400).encode()
    val = b"\n".join(old + b" INFO %d" % i for i in range(500))
    cfg = rc.config(tc.KEYS, regex=tc.PATTERN)
    ts = _ts(tc.NGINX_FMT)
    data, nev, ctr = _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, b"time", ts, tc.NOW, 43200, False,
                           OKEY, 1, 2, None)
    assert data == b"" and nev == 500 and int(ctr[6]) == 500
    block, raw, _, _ = _host(eng, eng.split_regex_timestamp_parse_sls_lz4, val, cfg, b"time", ts, tc.NOW, 43200,
                             False, OKEY, 1, 2, None, tail=b"\x1a\x01t")
    assert raw == 3 and lz4_block.decode(block) == b"\x1a\x01t"


def test_c2_nginx_64mib(eng):
    """C2's nginx lines with tkey = time: 64 MiB through the host call, against the host build of the chain fed the
    device's own split and regex tables (those are checked against the oracle elsewhere)"""
    from loongcollector_b200 import synth
    buf, _, _ = synth.nginx_lines(262144)
    val = buf.tobytes()
    assert len(val) >= 60 << 20
    cfg = rc.config(synth.NGINX_KEYS, "content", None, False, False, False, regex=synth.NGINX_PATTERN)
    ts = _ts(tc.NGINX_FMT)
    now = 1700000000
    got, ctr, _tap, _st, dev = device_chain(eng, val, cfg, b"time", ts, now, -1, False, OKEY, 1 << 33, now, None)
    off, ln, tables, pitch = dev
    want, wctr, _, _ = emulated(val, cfg, b"time", tc.NGINX_FMT, now, -1, False, OKEY, 1 << 33, now, None, off, ln,
                                tables, pitch)
    assert got == want and ctr == wctr
    data, nev, hctr = _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, b"time", ts, now, -1, False, OKEY,
                            1 << 33, now, None)
    assert data == want and [int(x) for x in hctr] == wctr and nev == off.size
    assert int(hctr[7]) > 0


def test_refusals(eng):
    import loongcollector_b200 as lc
    cfg = rc.config(tc.KEYS, "content", None, True, False, False, regex=tc.PATTERN)
    ts = _ts(tc.NGINX_FMT)
    val = b"a 1 b\nx\n"
    calls = [lambda k, o: _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, k, ts, tc.NOW, -1, False, o, 0,
                                0, None),
             lambda k, o: _host(eng, eng.split_regex_timestamp_parse_sls_lz4, val, cfg, k, ts, tc.NOW, -1, False, o, 0,
                                0, None, tail=b""),
             lambda k, o: _host(eng, eng.multiline_split_regex_timestamp_parse_sls, val, cfg, k, ts, tc.NOW, -1,
                                False, o, 0, 0, None, ml=(None, None, None, False)),
             lambda k, o: eng.split_regex_timestamp_tap_dev(None, 0, None, None, 0, None, None, None, 3,
                                                            [b"time", b"level", b"msg"], b"content", k, None, None,
                                                            keep_fail=True, offset_key=o)]
    for i, call in enumerate(calls):
        with pytest.raises(lc.LcError) as ei:  # tkey holds the offset digits
            call(OKEY, OKEY)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
        if i != 2:
            call(b"time", OKEY)  # accepted
    # a source time_ns without enable_ns: the records that keep the source time would carry Time_ns, the parsed ones not
    mixed = [lambda: _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, b"time", ts, tc.NOW, -1, False, OKEY, 0,
                           0, 5),
             lambda: _host(eng, eng.split_regex_timestamp_parse_sls_lz4, val, cfg, b"time", ts, tc.NOW, -1, False,
                           OKEY, 0, 0, 5, tail=b""),
             lambda: eng.sls_serialize_split_regex_timestamp_dev(None, 0, None, None, 0, None, None, None, 3,
                                                                 [b"time", b"level", b"msg"], b"content", None, None,
                                                                 None, enable_ns=False, keep_fail=True, time_ns=5)]
    for call in mixed:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    _host(eng, eng.split_regex_timestamp_parse_sls, val, cfg, b"time", ts, tc.NOW, -1, True, OKEY, 0, 0, 5)


# ---- the host classes through lc_host_chain3_serialize_sls
def _procs(split_type, split_cfg, rcfg, tcfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor(split_type, split_cfg),
            lc.HostProcessor("processor_parse_regex_native", dict(rc.oracle_config(rcfg))),
            lc.HostProcessor("processor_parse_timestamp_native", tcfg))


def _group(vals, offset_key=None, extra=None, ns=True):
    g = {"metadata": {}, "tags": {"__topic__": "t"}, "events": []}
    if offset_key is not None:
        g["metadata"]["log.file.offset"] = offset_key
    for i, v in enumerate(vals):
        ev = {"type": 1, "timestamp": 1700000000 + i, "fileOffset": 1000 * i, "rawSize": len(v),
              "contents": {"content": v}}
        if ns:
            ev["timestampNanosecond"] = 17 + i
        if extra:
            ev["contents"].update(extra)
        g["events"].append(ev)
    return g


def _counters(p):  # the event counters (the regex class's phase timers are wall time)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _regex_ran(p):
    """whether the regex class's Process ran: its batched path adds wall time to the b200_*_ns phase timers, which the
    device chain, never calling Process, leaves at 0"""
    return sum(v for k, v in p.counters().items() if k.endswith("_ns")) > 0


def _check_modes(split_type, split_cfg, rcfg, tcfg, group, enable_ns=True, device=None):
    """mode 0 and mode 2 against mode 1; device True / False: the splitter's SerializeSls took the device chain / ran
    the four host calls (None: not checked)"""
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, rcfg, tcfg)
    b = _procs(split_type, split_cfg, rcfg, tcfg)
    got = capi.host_chain3_serialize_sls(a[0], a[1], a[2], group, enable_ns, 0)
    want = capi.host_chain3_serialize_sls(b[0], b[1], b[2], group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    for k in range(3):
        assert _counters(a[k]) == _counters(b[k]), k
    c = _procs(split_type, split_cfg, rcfg, tcfg)
    z = capi.host_chain3_serialize_sls(c[0], c[1], c[2], group, enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    for k in range(3):
        assert _counters(c[k]) == _counters(b[k]), k
    if device is not None:
        assert _regex_ran(a[1]) == (not device) and _regex_ran(c[1]) == (not device)
    return want


def _host_lines(rng, n):
    """nginx-style lines whose times are far from the discard threshold of the real clock: an hour old (kept), ten days
    old (discarded), garbage (failed), and lines the regex fails"""
    now = int(_time.time())
    pool = [tc.render(tc.NGINX_FMT, now - 3600 - k) for k in range(3)] + [tc.render(tc.NGINX_FMT, now - 864000),
                                                                         "garbage", ""]
    lines = []
    for _ in range(n):
        r = rng.random()
        line = "%s %s m%d" % (rng.choice(pool), rng.choice(["INFO", "E"]), rng.randint(0, 9))
        lines.append("nospace" if r < 0.1 else line)
    return "\n".join(lines)


SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"\S* \w+ .*", "UnmatchedContentTreatment": "single_line"})]


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(eng, split_type, split_cfg):
    rng = random.Random(5)
    vals = [_host_lines(rng, 40) for _ in range(3)]
    tcfg = {"SourceKey": "time", "SourceFormat": tc.NGINX_FMT}
    for keep_fail in (False, True):
        rcfg = rc.config(tc.KEYS, "content", "raw", keep_fail, False, True, regex=tc.PATTERN)
        for okey in (None, OKEY.decode()):
            for enable_ns in (False, True):
                for ns in (False, True):
                    _check_modes(split_type, split_cfg, rcfg, tcfg, _group(vals[:1], okey, ns=ns), enable_ns,
                                 device=True)
            # several source events: the host path
            _check_modes(split_type, split_cfg, rcfg, tcfg, _group(vals, okey), device=False)
    rcfg = rc.config(tc.KEYS, "content", "raw", True, False, True, regex=tc.PATTERN)
    _check_modes(split_type, split_cfg, rcfg, dict(tcfg, SourceKey="raw"), _group(vals[:1], OKEY.decode()),
                 device=True)
    _check_modes(split_type, split_cfg, rcfg, tcfg, _group(vals[:1], extra={"x": "y"}), device=False)  # non-flat
    # the offset key as tkey: refused by the device calls, so the host path runs
    _check_modes(split_type, split_cfg, rcfg, dict(tcfg, SourceKey=OKEY.decode()), _group(vals[:1], OKEY.decode()),
                 device=False)
    # errors: every event discarded, empty group
    old = "\n".join("%s INFO m" % tc.render(tc.NGINX_FMT, int(_time.time()) - 864000) for _ in range(20))
    assert _check_modes(split_type, split_cfg, rcfg, tcfg, _group([old]), device=True)[2] == "empty event group"
    assert _check_modes(split_type, split_cfg, rcfg, tcfg, _group([]))[2] == "empty event group"
