"""GPU tier: the delimiter -> SLS hand-over.  lc_sls_serialize_delim_dev after lc_delim_parse_dev, lc_delim_parse_sls
and ProcessorParseDelimiterNative::SerializeSls against the oracle (ProcessorParseDelimiterNative over flat events +
sls_serialize_logs / sls_serialize_group), byte for byte."""
import json
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import delim_sls_cases as dc  # noqa: E402
from tests.golden_util import input_with_metadata, load_cases  # noqa: E402

POISON, GUARD = 0xA5, 256


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _quote(cfg):
    return cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')


def _i32(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).cuda()


def device_serialize(eng, buf, off, ln, cfg, times, nss):
    """delim_parse_dev -> sls_serialize_delim_dev into a poisoned buffer followed by guard bytes; checks the guard, the
    sizing query and the capacity error; returns (wire bytes, status table)"""
    import torch

    import loongcollector_b200 as lc
    n, mf = off.size, cfg["max_fields"]
    d_buf = torch.from_numpy(np.concatenate([buf, np.zeros(16, np.uint8)])).cuda()
    d_off, d_len = _i32(off), _i32(ln)
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_nf = torch.empty(n, dtype=torch.int32, device="cuda")
    d_fo, d_fl, d_fd = (torch.empty(n * mf, dtype=torch.int32, device="cuda") for _ in range(3))
    d_t = _i32(times)
    d_ns = _i32(nss) if nss is not None else None
    keys = [k.encode() for k in cfg["keys"]]
    eng.delim_parse_dev(d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, cfg["sep"], _quote(cfg),
                        len(keys), cfg["treatment"] == "extend", cfg["allow_short"], mf, d_st.data_ptr(),
                        d_nf.data_ptr(), d_fo.data_ptr(), d_fl.data_ptr(), d_fd.data_ptr())
    args = (d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, d_st.data_ptr(), d_nf.data_ptr(),
            d_fo.data_ptr(), d_fl.data_ptr(), d_fd.data_ptr(), mf, cfg["sep"], _quote(cfg), cfg["treatment"], keys,
            cfg["source"].encode(), dc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"])
    kw = dict(d_ev_time=d_t.data_ptr(), d_ev_time_ns=d_ns.data_ptr() if d_ns is not None else None)
    need = eng.sls_serialize_delim_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_delim_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got = eng.sls_serialize_delim_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), d_st.cpu().numpy()


MATRIX = list(dc.all_cases(seed_base=2, per=2))


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_device_tables_to_wire_bytes_match_oracle(eng, case):
    _, cfg, rng = case
    lines = [dc.random_line(rng, cfg["sep"], cfg["quote"], wide=rng.random() < 0.05) for _ in range(400)]
    buf, off, ln = dc.arena(lines, gap=cfg["sep"][:1])  # separator bytes between the lines: no read may leave a line
    times, nss = dc.times_for(len(lines), rng.randint(0, 1 << 30))
    for ns in (nss, None):
        want, ctr, _ = dc.oracle_wire(lines, cfg, times, ns, ns is not None)
        got, _ = device_serialize(eng, buf, off, ln, cfg, times, ns)
        assert got == want
    # host buffers: same bytes, counters as the oracle's
    data, c = eng.delim_parse_sls(buf, off, ln, times, cfg["sep"], _quote(cfg), cfg["treatment"],
                                  [k.encode() for k in cfg["keys"]], cfg["source"].encode(), dc.renamed_key(cfg),
                                  cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], cfg["allow_short"],
                                  cfg["max_fields"], ev_time_ns=nss)
    want, ctr, _ = dc.oracle_wire(lines, cfg, times, nss, True)
    assert data == want
    assert (int(c[0]), int(c[1] + c[3]), int(c[2])) == (ctr["out_successful"], ctr["out_failed"], ctr["discarded"])


def test_c4_shaped_batch(eng):
    from loongcollector_b200 import synth
    buf, off, ln = synth.csv_lines(100_000, seed=21)
    lines = [bytes(buf[o:o + n]) for o, n in zip(off.tolist(), ln.tolist())]
    for tr, extra in (("extend", {}), ("keep", {"keep_succeed": True, "renamed": "raw"})):
        cfg = {"sep": b",", "quote": ord('"'), "treatment": tr, "keys": list(synth.CSV_KEYS), "source": "content",
               "renamed": None, "keep_fail": True, "keep_succeed": False, "copy_raw": False, "allow_short": True,
               "max_fields": 11}
        cfg.update(extra)
        times, nss = dc.times_for(len(lines), 9)
        want, _, _ = dc.oracle_wire(lines, cfg, times, nss)
        got, _ = device_serialize(eng, buf, off, ln, cfg, times, nss)
        assert got == want


def test_every_length_and_alignment(eng):
    rng = random.Random(5)
    cfg = {"sep": b",", "quote": ord('"'), "treatment": "keep", "keys": ["a", "b", "content"], "source": "content",
           "renamed": None, "keep_fail": True, "keep_succeed": True, "copy_raw": True, "allow_short": True,
           "max_fields": 4}
    buf = bytearray()
    off, ln, lines = [], [], []
    for length in range(0, 301):
        for mis in range(16):
            line = b""
            while len(line) < length:
                line += dc.random_line(rng, b",", ord('"')) + b","
            line = line[:length]
            buf += b'",' * 8
            buf += b"\"" * ((mis - len(buf)) % 16)
            off.append(len(buf))
            ln.append(length)
            lines.append(line)
            buf += line
    buf += b'"' * 32
    buf = np.frombuffer(bytes(buf), np.uint8)
    off, ln = np.array(off, np.uint32), np.array(ln, np.uint32)
    times, nss = dc.times_for(len(lines), 6)
    for tr in dc.TREATMENTS:
        cfg["treatment"] = tr
        want, _, _ = dc.oracle_wire(lines, cfg, times, nss)
        got, _ = device_serialize(eng, buf, off, ln, cfg, times, nss)
        assert got == want, tr


def _log_record(t, ns, contents):
    """one Log record as oracle.sls_serialize_logs writes it, joined in one pass (the oracle's serialiser appends to
    an immutable bytes object per content, which takes hours for a million contents); checked against it below"""
    body = b"".join([b"\x08" + orc._sls_varint(max(t, orc.SLS_MIN_LOG_TIME))] +
                    [orc._sls_pair(0x12, k, v) for k, v in contents] +
                    ([b"\x25" + int(ns).to_bytes(4, "little")] if ns is not None else []))
    return b"\x0a" + orc._sls_varint(len(body)) + body


def _hand_events_of_separator_line(cfg, nsep, sep):
    """contents of a line of nsep separators (nsep + 1 empty columns), derived by hand for a size the oracle's
    quadratic content look-up cannot take; checked against the oracle on a small instance first"""
    keys = [k.encode() for k in cfg["keys"]]
    nk, nf = len(keys), nsep + 1
    if cfg["treatment"] == "extend":
        return [(k, b"") for k in keys] + [(b"__column%d__" % j, b"") for j in range(nk, nf)]
    return [(k, b"") for k in keys] + [(b"__column%d__" % nk, sep[:1] * (nf - nk))]


# (keep with the multi-byte split has no wide rows: the split stops at nkeys + 1 columns)
@pytest.mark.parametrize("treatment,sep", [("extend", b","), ("keep", b","), ("extend", b"|#")])
def test_one_mib_line_of_separators_in_a_batch(eng, sep, treatment):
    cfg = {"sep": sep, "quote": ord('"'), "treatment": treatment, "keys": ["a", "b", "c"], "source": "content",
           "renamed": None, "keep_fail": False, "keep_succeed": False, "copy_raw": False, "allow_short": True,
           "max_fields": 4}
    small = sep * 700
    t1 = np.array([1700000000], np.uint32)
    want_small = dc.oracle_wire([small], cfg, t1, [123], True)[0]
    assert want_small == orc.sls_serialize_logs([(1700000000, 123, _hand_events_of_separator_line(cfg, 700, sep))],
                                                True)[0]
    assert want_small == _log_record(1700000000, 123, _hand_events_of_separator_line(cfg, 700, sep))
    rng = random.Random(8)
    nsep = (1 << 20) // len(sep)
    short = [dc.random_line(rng, sep, ord('"')) for _ in range(62)]
    lines = short[:31] + [sep * nsep] + short[31:]
    times, nss = dc.times_for(len(lines), 7)
    want = b""
    for i, line in enumerate(lines):
        if i == 31:
            want += _log_record(int(times[i]), None if nss[i] == 0xFFFFFFFF else int(nss[i]),
                                _hand_events_of_separator_line(cfg, nsep, sep))
        else:
            want += dc.oracle_wire([line], cfg, times[i:i + 1], nss[i:i + 1])[0]
    buf, off, ln = dc.arena(lines)
    got, st = device_serialize(eng, buf, off, ln, cfg, times, nss)
    assert st[31] == 0 and got == want


def test_host_buffers_across_pipeline_chunks(eng):
    """> 96 MB of C4 lines: several upload chunks; the bytes equal the device-resident path and the counters equal
    the status table's"""
    from loongcollector_b200 import synth
    buf, off, ln = synth.csv_lines(700_000, seed=23)
    assert buf.size > 100 << 20
    cfg = {"sep": b",", "quote": ord('"'), "treatment": "extend", "keys": list(synth.CSV_KEYS)[:8],
           "source": "content", "renamed": "raw", "keep_fail": True, "keep_succeed": True, "copy_raw": True,
           "allow_short": False, "max_fields": 9}
    times, nss = dc.times_for(off.size, 10)
    ref, st = device_serialize(eng, buf, off, ln, cfg, times, nss)
    data, c = eng.delim_parse_sls(buf, off, ln, times, cfg["sep"], _quote(cfg), cfg["treatment"],
                                  [k.encode() for k in cfg["keys"]], cfg["source"].encode(), b"raw", True, True, True,
                                  False, 9, ev_time_ns=nss)
    assert data == ref
    assert [int(x) for x in c] == [int((st == 0).sum()), int(((st == 1) | (st == 3)).sum()), 0, int((st == 2).sum())]
    assert c[0] > 0


# ---- host class: SerializeSls == Process + SLSEventGroupSerializer::Serialize on the same in-memory group
def _host_pair(cfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor("processor_parse_delimiter_native", cfg),
            lc.HostProcessor("processor_parse_delimiter_native", cfg))


def _check_host(cfg, group, oracle_too=True):
    fast, ref = _host_pair(cfg)
    for ns in (False, True):
        got = fast.serialize_sls(group, ns)
        want = ref.serialize_sls(group, ns, process_then_serialize=True)
        assert got == want, (cfg, ns, got[1], want[1])
        if oracle_too:
            g = orc.Group.from_json(json.loads(json.dumps(group)))
            orc.ProcessorParseDelimiterNative(cfg).process(g)
            o, oerr = orc.sls_serialize_group(g, ns)
            assert want[0] == o and (want[1] is None) == (oerr is None), (cfg, ns, want[1], oerr)
    assert fast.counters() == ref.counters()


def test_host_serialize_sls_on_reference_fixtures():
    import loongcollector_b200 as lc
    n = 0
    for case in load_cases("delimiter"):
        cfg = case["pipeline"][0]["config"]
        if case["pipeline"][0]["type"] != "processor_parse_delimiter_native" or len(case["pipeline"]) != 1:
            continue
        try:
            _host_pair(cfg)
        except lc.LcError:  # a fixture of a configuration Init refuses
            continue
        _check_host(cfg, input_with_metadata(case), oracle_too=False)
        n += 1
    assert n > 5


def test_host_serialize_sls_on_random_groups():
    rng = random.Random(31)
    for k in range(60):
        sname, sep, quote = dc.SEPARATORS[k % 4]
        cfg = dc.random_config(rng, dc.TREATMENTS[k % 3], sep, quote)
        evs = []
        for _ in range(rng.choice([0, 1, 5, 40])):
            ev = {"type": 1, "timestamp": rng.choice([5, 1700000000]),
                  "contents": {cfg["source"]: dc.random_line(rng, sep, quote, rng.random() < 0.05).decode("latin1")}}
            if rng.random() < 0.5:
                ev["timestampNanosecond"] = rng.randint(0, 999999999)
            if k % 5 == 4 and rng.random() < 0.3:  # not flat: Process + Serialize
                ev["contents"]["other"] = "x"
            evs.append(ev)
        root = {"events": evs, "tags": {"__topic__": "t", "host.name": "h" * rng.choice([1, 100])}}
        if k % 7 == 6:
            root["metadata"] = {"log.file.offset": "__offset__"}
        _check_host(dc.oracle_config(cfg), root)


def test_host_serialize_sls_size_limit_and_empty_groups():
    cfg = dc.oracle_config({"sep": b",", "quote": ord('"'), "treatment": "extend", "keys": ["a", "b"],
                            "source": "content", "renamed": None, "keep_fail": False, "keep_succeed": False,
                            "copy_raw": False, "allow_short": True, "max_fields": 3})
    big = {"events": [{"type": 1, "timestamp": 1, "contents": {"content": "x" * 4096 + ",y"}} for _ in range(3000)]}
    _check_host(cfg, big, oracle_too=True)  # > 10 MB: the size-limit error
    failing = {"events": [{"type": 1, "timestamp": 1, "contents": {"content": '"open'}}]}
    _check_host(cfg, failing)  # every event erased: "empty event group"
    _check_host(cfg, {"events": []})
    cfg2 = dict(cfg, Keys=["_", "_"], OverflowedFieldsTreatment="discard")
    _check_host(cfg2, {"events": [{"type": 1, "timestamp": 1, "contents": {"content": "1,2,3"}}]})  # all empty logs
