"""GPU tier: the split -> SLS hand-over.  lc_sls_serialize_spans_dev after lc_split_lines_dev and after
lc_multiline_split_dev, lc_split_sls / lc_multiline_split_sls and the splitters' SerializeSls against the oracle
(its splitters over one source event + sls_serialize_logs / sls_serialize_group), byte for byte."""
import json
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import split_sls_cases as sc  # noqa: E402
from tests.golden_util import input_with_metadata, load_cases  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = b"__file_offset__"


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _upload(val: bytes, align: int):
    """val on the device, starting `align` bytes past a 16-byte boundary; returns (tensor, device address)"""
    import torch
    d = torch.zeros(len(val) + 48, dtype=torch.uint8, device="cuda")
    base = (-d.data_ptr()) % 16 + align
    if val:
        d[base:base + len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    return d, d.data_ptr() + base


def device_pieces(eng, d_src, n_src, ml=None):
    """piece tables of lc_split_lines_dev (ml None) or lc_multiline_split_dev (ml = (start, cont, end, discard))"""
    import torch
    cap = max(n_src, 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    if ml is None:
        n = eng.split_lines_dev(d_src, n_src, 10, d_off.data_ptr(), d_len.data_ptr(), cap)
        ctr = None
    else:
        d_fl = torch.empty(cap, dtype=torch.uint8, device="cuda")
        n, ctr = eng.multiline_split_dev(d_src, n_src, *ml, d_off.data_ptr(), d_len.data_ptr(), d_fl.data_ptr(), cap)
    return d_off, d_len, n, ctr


def device_serialize(eng, val, key, okey, pos, time, ns, align=0, out_align=0, ml=None, check_refusal=True):
    """split (or multiline split) on the device, then sls_serialize_spans_dev into a poisoned buffer followed by guard
    bytes; checks the sizing query, the capacity refusal and the guard; returns the wire bytes"""
    import torch

    import loongcollector_b200 as lc
    d_buf, d_src = _upload(val, align)
    d_off, d_len, n, _ = device_pieces(eng, d_src, len(val), ml)
    args = (d_src, len(val), d_off.data_ptr(), d_len.data_ptr(), n, key, okey, pos, time, ns)
    need = eng.sls_serialize_spans_dev(*args)
    d_out = torch.full((need + GUARD + 16,), POISON, dtype=torch.uint8, device="cuda")
    o = (-d_out.data_ptr()) % 16 + out_align
    if need and check_refusal:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_spans_dev(*args, d_out=d_out.data_ptr() + o, out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got = eng.sls_serialize_spans_dev(*args, d_out=d_out.data_ptr() + o, out_cap=need)
    assert got == need
    host = d_out.cpu().numpy()
    assert (host[:o] == POISON).all() and (host[o + need:] == POISON).all(), "write outside the records"
    return bytes(host[o:o + need])


def test_split_then_serialize_matches_oracle(eng):
    rng = random.Random(1)
    for i in range(12):
        val = sc.random_value(rng, rng.randint(1, 200))
        t, ns = sc.TIMES[i % len(sc.TIMES)]
        okey = [None, OKEY, b"content"][i % 3]
        pos = sc.POSITIONS[i % len(sc.POSITIONS)]
        want = sc.oracle_split_wire(val, b"content", t, ns, pos, okey)
        assert device_serialize(eng, val, b"content", okey, pos, t, ns, i % 16, (3 * i) % 16) == want


def test_every_length_at_every_alignment(eng):
    rng = random.Random(2)
    alphabet = b"abcdefghij\n"
    for n in range(0, 301):
        val = bytes(rng.choice(alphabet) for _ in range(n))
        want = sc.oracle_split_wire(val, b"content", 1 << 29, 7, 1000, OKEY if n % 2 else None)
        for align in range(16):
            got = device_serialize(eng, val, b"content", OKEY if n % 2 else None, 1000, 1 << 29, 7, align,
                                   (align + n) % 16, check_refusal=align == 0)
            assert got == want, (n, align)


def test_megabyte_line_among_short_ones(eng):
    rng = random.Random(3)
    lines = [b"s" * rng.randint(0, 40) for _ in range(300)]
    lines[150] = bytes(rng.randrange(32, 127) for _ in range(4096)) * 256  # 1 MiB
    val = b"\n".join(lines)
    for okey in (None, OKEY):
        want = sc.oracle_split_wire(val, b"content", 1 << 30, None, 5, okey)
        assert device_serialize(eng, val, b"content", okey, 5, 1 << 30, None, 7, 9) == want


def test_c1_shaped_batch(eng):
    from loongcollector_b200 import synth
    buf, _, _ = synth.newline_lines(100_000)
    val = buf.tobytes()
    want = sc.oracle_split_wire(val, b"content", 1700000000, 123, 1 << 33, OKEY)
    assert device_serialize(eng, val, b"content", OKEY, 1 << 33, 1700000000, 123) == want
    data, nev = eng.split_sls(val, 10, b"content", OKEY, 1 << 33, 1700000000, 123)
    assert data == want and nev == 100_000


def _ml_handles(cfg):
    p = orc.ProcessorSplitMultilineLogStringNative(cfg)
    import loongcollector_b200 as lc
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


@pytest.mark.parametrize("discard", [False, True])
def test_c3_shaped_records(eng, discard):
    from loongcollector_b200 import synth
    buf, _, _ = synth.java_stack_records(3000)
    val = buf.tobytes()
    cfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
           "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    want, counters, nev = sc.oracle_multiline_wire(val, cfg, 1700000000, None, 4096, OKEY)
    h = _ml_handles(cfg)
    assert device_serialize(eng, val, b"content", OKEY, 4096, 1700000000, None, 5, 11, ml=h) == want
    data, n, ctr = eng.multiline_split_sls(val, *h, b"content", OKEY, 4096, 1700000000, None)
    assert data == want and n == nev
    assert int(ctr[0]) == counters["matched_events"]
    assert int(ctr[1]) - int(ctr[2]) == counters["matched_lines"] and int(ctr[2]) == counters["unmatched_lines"]


@pytest.mark.parametrize("name", sorted(sc.ML_CFGS))
@pytest.mark.parametrize("discard", [False, True])
def test_unit_test_patterns(eng, name, discard):
    rng = random.Random(hash(name) & 0xFFFF)
    val = sc.ml_value(rng, 300)
    cfg = sc.ml_config(name, discard)
    h = _ml_handles(cfg)
    for okey in (None, OKEY, b"content"):
        want, _, _ = sc.oracle_multiline_wire(val, cfg, 1 << 29, 99, 77, okey)
        assert device_serialize(eng, val, b"content", okey, 77, 1 << 29, 99, 3, 1, ml=h) == want
        data, _, _ = eng.multiline_split_sls(val, *h, b"content", okey, 77, 1 << 29, 99)
        assert data == want


def test_host_buffer_calls_match_device_path(eng):
    import loongcollector_b200 as lc
    rng = random.Random(4)
    val = sc.random_value(rng, 500)
    ref = device_serialize(eng, val, b"log", OKEY, 9, 1, 2)
    data, nev = eng.split_sls(val, 10, b"log", OKEY, 9, 1, 2)
    assert data == ref and nev == len(orc.split_lines(val)[0])
    with pytest.raises(lc.LcError) as ei:
        eng.split_sls(val, 10, b"log", OKEY, 9, 1, 2, out_cap=len(ref) - 1)
    assert ei.value.code == lc.capi.LC_ERR_CAPACITY
    assert eng.split_sls(b"", 10, b"log", OKEY, 9, 1, 2) == (b"", 0)


# ---- host classes: SerializeSls == Process + SLSEventGroupSerializer::Serialize on the same in-memory group
def oracle_group(ptype, cfg, group, ns):
    """the oracle's processor and serializer; RAW events serialise as "content" -> content"""
    g = orc.Group.from_json(json.loads(json.dumps(group)))
    proc = {"processor_split_string_native": orc.ProcessorSplitLogStringNative,
            "processor_split_multiline_log_string_native": orc.ProcessorSplitMultilineLogStringNative}[ptype](cfg)
    proc.process(g)
    kinds = {e.type for e in g.events}
    if orc.RAW in kinds:
        if kinds != {orc.RAW}:
            return None, "unsupported event type in event group"
        for e in g.events:
            c = e.raw
            e.type, e.contents = orc.LOG, [[b"content", c, True]]
    return orc.sls_serialize_group(g, ns)


def _check_host(ptype, cfg, group, oracle_too=True):
    import loongcollector_b200 as lc
    fast, ref = lc.HostProcessor(ptype, cfg), lc.HostProcessor(ptype, cfg)
    for ns in (False, True):
        got = fast.serialize_sls(group, ns)
        want = ref.serialize_sls(group, ns, process_then_serialize=True)
        assert got == want, (cfg, ns, got[1], want[1])
        if oracle_too:
            o, oerr = oracle_group(ptype, cfg, group, ns)
            assert want[0] == o and (want[1] is None) == (oerr is None), (cfg, ns, want[1], oerr)
            if oerr is not None:
                assert want[1].startswith(oerr)
    assert fast.counters() == ref.counters()
    return got


@pytest.mark.parametrize("kind,ptype", [("split", "processor_split_string_native"),
                                        ("multiline", "processor_split_multiline_log_string_native")])
def test_host_serialize_sls_on_reference_fixtures(kind, ptype):
    n = 0
    for case in load_cases(kind):
        if len(case["pipeline"]) != 1 or case["pipeline"][0]["type"] != ptype:
            continue
        got = _check_host(ptype, case["pipeline"][0]["config"], input_with_metadata(case))
        n += got[0] is not None
    assert n >= (3 if kind == "split" else 20)


def _random_group(rng, key, k, raw_ok=True):
    evs = []
    for _ in range(rng.choice([0, 1, 1, 3])):
        val = sc.random_value(rng, rng.randint(0, 30)) if rng.random() < 0.9 else b""
        ev = {"type": 1, "timestamp": rng.choice([5, 1700000000, 12345678901]), "contents": {key: val.decode()},
              "fileOffset": rng.choice(sc.POSITIONS[:12]), "rawSize": len(val)}
        if rng.random() < 0.5:
            ev["timestampNanosecond"] = rng.randint(0, 999999999)
        if k % 6 == 5 and rng.random() < 0.4:  # not flat: Process + Serialize
            ev["contents"]["other"] = "x"
        evs.append(ev)
    root = {"events": evs, "tags": {"__topic__": "t", "host.name": "h" * rng.choice([1, 100])}}
    if k % 3:
        root["metadata"] = {"log.file.offset": rng.choice(["__file_offset__", key])}
    return root


def test_host_split_on_random_groups():
    rng = random.Random(31)
    for k in range(40):
        key = rng.choice(["content", "log"])
        cfg = {"SourceKey": key, "SplitChar": rng.choice([10, 10, 0]), "EnableRawContent": k % 4 == 3}
        root = _random_group(rng, key, k)
        if cfg["SplitChar"] == 0:
            for ev in root["events"]:
                ev["contents"][key] = ev["contents"][key].replace("\n", "\0")
        _check_host("processor_split_string_native", cfg, root)


def test_host_multiline_on_random_groups():
    rng = random.Random(32)
    names = sorted(sc.ML_CFGS)
    for k in range(30):
        cfg = sc.ml_config(names[k % len(names)], discard=k % 2 == 1, raw=k % 5 == 4)
        root = _random_group(rng, "content", k)
        for ev in root["events"]:
            if ev["contents"]["content"]:
                ev["contents"]["content"] = sc.ml_value(rng, rng.randint(1, 20)).decode()
        _check_host("processor_split_multiline_log_string_native", cfg, root)


def test_host_special_groups():
    ptype = "processor_split_string_native"
    cfg = {"SourceKey": "content"}
    ev = lambda v, **kw: dict({"type": 1, "timestamp": 1, "contents": {"content": v}}, **kw)  # noqa: E731
    _check_host(ptype, cfg, {"events": []})  # empty group
    _check_host(ptype, cfg, {"events": [ev(""), ev("")]})  # only empty sources: "empty event group"
    _check_host(ptype, cfg, {"events": [ev("a\nb"), ev(""), ev("c\n\nd\n")]})  # several sources, in order
    mixed = {"events": [ev("a\nb"), {"type": 1, "timestamp": 2, "contents": {"x": "y"}}]}
    _check_host(ptype, cfg, mixed)  # non-flat: fallback path
    _check_host(ptype, dict(cfg, EnableRawContent=True), mixed)  # LOG + RAW: unsupported
    _check_host(ptype, dict(cfg, EnableRawContent=True), {"events": [ev("a\n\nb", timestampNanosecond=5)]})  # RAW
    # > 10 MB of records from short lines with offset metadata: the size-limit error, with the exact group size
    big = {"events": [ev("\n".join("x" * (i % 7) for i in range(200_000)))] * 2,
           "metadata": {"log.file.offset": "__file_offset__"}}
    got = _check_host(ptype, cfg, big)
    assert got[0] is None and got[1].startswith("log group exceeds size limit")


def test_host_multiline_counters():
    import loongcollector_b200 as lc
    cfg = sc.ml_config("start_end", discard=True)
    rng = random.Random(7)
    root = {"events": [{"type": 1, "timestamp": 3, "contents": {"content": sc.ml_value(rng, 200).decode()}}
                       for _ in range(3)]}
    fast = lc.HostProcessor("processor_split_multiline_log_string_native", cfg)
    ref = lc.HostProcessor("processor_split_multiline_log_string_native", cfg)
    assert fast.serialize_sls(root) == ref.serialize_sls(root, process_then_serialize=True)
    c = fast.counters()
    assert c == ref.counters() and c["matched_events"] > 0 and c["unmatched_lines"] > 0
    g = orc.Group.from_json(json.loads(json.dumps(root)))
    o = orc.ProcessorSplitMultilineLogStringNative(cfg)
    o.process(g)
    assert all(c[k] == v for k, v in o.counters.items())
