"""GPU tier: parse + serialise + LZ4 in one call.  lc_regex_parse_sls_lz4 / lc_delim_parse_sls_lz4 return one block
that decodes (strict decoder, tests/lz4_block.py) to lc_regex_parse_sls / lc_delim_parse_sls's bytes followed by the
tail, with the same counters; SerializeSlsLz4 decodes to SerializeSls's bytes, with the same errors and counters; the
GPU-backed LZ4Compressor round-trips."""
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402

TAIL = b"\x1a\x05topic\x22\x06source" + b"\x32\x0c\x0a\x04tag1\x12\x04val1"


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _regex_both(eng, buf, off, ln, cfg, times, nss, tail):
    import loongcollector_b200 as lc
    rx = None if rc.whole_line(cfg) else lc.Regex(cfg["regex"])
    args = (rx, buf, off, ln, times, [k.encode() for k in cfg["keys"]], cfg["source"].encode(), rc.renamed_key(cfg),
            cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], rc.whole_line(cfg))
    wire, c = eng.regex_parse_sls(*args, ev_time_ns=nss)
    block, raw, c2 = eng.regex_parse_sls_lz4(*args, ev_time_ns=nss, tail=tail)
    assert raw == len(wire) + len(tail)
    assert lz4_block.decode(block) == wire + tail
    assert list(c) == list(c2)
    return block


REGEX_MATRIX = list(rc.matrix()) + list(rc.whole_line_matrix())


@pytest.mark.parametrize("case", REGEX_MATRIX, ids=[c[0] for c in REGEX_MATRIX])
def test_regex_fused_decodes_to_sibling_plus_tail(eng, case):
    _, cfg = case
    rng = random.Random(sum(case[0].encode()) * 31 + len(case[0]))
    lines = [rc.random_line(rng) for _ in range(300)]
    buf, off, ln = rc.arena(lines)
    times, nss = rc.times_for(len(lines), 3)
    for tail in (TAIL, b""):
        _regex_both(eng, buf, off, ln, cfg, times, nss, tail)


def test_regex_fused_c2_batch_and_capacity(eng):
    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(100_000, seed=5)
    cfg = rc.config(list(synth.NGINX_KEYS), "content", None, True, False, False, regex=synth.NGINX_PATTERN)
    times, nss = rc.times_for(off.size, 4)
    block = _regex_both(eng, buf, off, ln, cfg, times, nss, TAIL)
    with pytest.raises(lc.LcError) as ei:
        eng.regex_parse_sls_lz4(lc.Regex(synth.NGINX_PATTERN), buf, off, ln, times, [k.encode() for k in cfg["keys"]],
                                b"content", None, True, ev_time_ns=nss, tail=TAIL, out_cap=len(block) - 1)
    assert ei.value.code == lc.capi.LC_ERR_CAPACITY


def test_fused_without_events_is_the_tail(eng):
    from loongcollector_b200 import synth
    e = np.zeros(0, np.uint32)
    block, raw, _ = eng.regex_parse_sls_lz4(None, b"", e, e, e, [b"a"], b"content", whole_line=True, tail=TAIL)
    assert raw == len(TAIL) and lz4_block.decode(block) == TAIL
    block, raw, _ = eng.delim_parse_sls_lz4(b"", e, e, e, b",", ord('"'), "extend", [k.encode() for k in synth.CSV_KEYS],
                                            b"content", tail=TAIL)
    assert raw == len(TAIL) and lz4_block.decode(block) == TAIL


def _quote(cfg):
    return cfg["quote"] if cfg["quote"] is not None else 0


def _delim_both(eng, buf, off, ln, cfg, times, nss, tail):
    args = (buf, off, ln, times, cfg["sep"], _quote(cfg), cfg["treatment"], [k.encode() for k in cfg["keys"]],
            cfg["source"].encode(), dc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"],
            cfg["allow_short"], cfg["max_fields"])
    wire, c = eng.delim_parse_sls(*args, ev_time_ns=nss)
    block, raw, c2 = eng.delim_parse_sls_lz4(*args, ev_time_ns=nss, tail=tail)
    assert raw == len(wire) + len(tail)
    assert lz4_block.decode(block) == wire + tail
    assert list(c) == list(c2)


DELIM_MATRIX = list(dc.all_cases(seed_base=3, per=1))


@pytest.mark.parametrize("case", DELIM_MATRIX, ids=[c[0] for c in DELIM_MATRIX])
def test_delim_fused_decodes_to_sibling_plus_tail(eng, case):
    _, cfg, rng = case
    lines = [dc.random_line(rng, cfg["sep"], cfg["quote"], wide=rng.random() < 0.05) for _ in range(300)]
    buf, off, ln = dc.arena(lines, gap=cfg["sep"][:1])
    times, nss = dc.times_for(len(lines), rng.randint(0, 1 << 30))
    for tail in (TAIL, b""):
        _delim_both(eng, buf, off, ln, cfg, times, nss, tail)


def test_delim_fused_c4_batch(eng):
    from loongcollector_b200 import synth
    buf, off, ln = synth.csv_lines(100_000, seed=21)
    cfg = {"sep": b",", "quote": ord('"'), "treatment": "extend", "keys": list(synth.CSV_KEYS), "source": "content",
           "renamed": None, "keep_fail": True, "keep_succeed": False, "copy_raw": False, "allow_short": True,
           "max_fields": len(synth.CSV_KEYS) + 16}
    times, nss = dc.times_for(off.size, 9)
    _delim_both(eng, buf, off, ln, cfg, times, nss, TAIL)


# ---- host classes: SerializeSlsLz4 decodes to SerializeSls's bytes, with the same errors and counters
def _groups(lines, pattern_line):
    flat = {"events": [{"type": 1, "timestamp": 1700000000 + i, "timestampNanosecond": 7,
                        "contents": {"content": x}} for i, x in enumerate(lines)],
            "tags": {"__topic__": "t", "__source__": "s", "k": "v"}}
    non_flat = {"events": [{"type": 1, "timestamp": 1700000000 + i, "contents": {"content": x, "other": "o"}}
                           for i, x in enumerate(lines)], "tags": {"__topic__": "t"}}
    big = {"events": [{"type": 1, "timestamp": 1700000000, "contents": {"content": pattern_line * ((11 << 20) // 64)}}
                      for _ in range(2)], "tags": {}}
    empty = {"events": [], "tags": {"__topic__": "t"}}
    return [flat, non_flat, big, empty]


def _check_host_lz4(ptype, cfg, groups):
    import loongcollector_b200 as lc
    a, b = lc.HostProcessor(ptype, cfg), lc.HostProcessor(ptype, cfg)
    for g in groups:
        for ns in (False, True):
            want, werr = a.serialize_sls(g, ns)
            block, raw, err = b.serialize_sls_lz4(g, ns)
            assert err == werr
            if want is not None:
                assert raw == len(want) and lz4_block.decode(block) == want
    # the event counters move alike; the host layer's phase timers (`*_ns`) are wall clocks
    ca, cb = ({k: v for k, v in p.counters().items() if not k.endswith("_ns")} for p in (a, b))
    assert ca == cb


def test_regex_serialize_sls_lz4():
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(500, seed=8)
    lines = [bytes(buf[o:o + n]).decode() for o, n in zip(off.tolist(), ln.tolist())]
    _check_host_lz4("processor_parse_regex_native",
                    {"SourceKey": "content", "Regex": synth.NGINX_PATTERN, "Keys": synth.NGINX_KEYS,
                     "KeepingSourceWhenParseFail": True},
                    _groups(lines, "x" * 64))


def test_delim_serialize_sls_lz4():
    from loongcollector_b200 import synth
    buf, off, ln = synth.csv_lines(500, seed=8)
    lines = [bytes(buf[o:o + n]).decode() for o, n in zip(off.tolist(), ln.tolist())]
    _check_host_lz4("processor_parse_delimiter_native",
                    {"SourceKey": "content", "Separator": ",", "Quote": '"', "Keys": synth.CSV_KEYS,
                     "KeepingSourceWhenParseFail": True},
                    _groups(lines, "x" * 64))


def test_host_lz4_compressor():
    from loongcollector_b200 import capi
    rng = random.Random(2)
    inputs = [b"", b"abc", rng.randbytes(70000), b"log line " * 20000]
    blocks, err = capi.host_lz4_compress(inputs)
    assert err is None and [lz4_block.decode(b) for b in blocks] == inputs
    blocks, err = capi.host_lz4_compress([])
    assert blocks == [] and err is None
