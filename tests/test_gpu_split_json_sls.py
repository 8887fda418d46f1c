"""GPU tier: the split -> JSON chain (lc_sls_serialize_split_json_dev, lc_split_json_parse_sls[_lz4],
lc_multiline_split_json_parse_sls[_lz4]) against the oracle's splitter + ProcessorParseJsonNative + sls_serialize_logs
and the host build of the resolve and row functions: bytes and counters, poisoned outputs with guard bytes, the
sizing query, the capacity refusal, the other refusals, and LZ4 blocks that decode to the records ‖ tail."""
import random

import numpy as np
import pytest

from oracle import json_parse as ojs  # noqa: E402  (checker only)
from oracle import oracle as orc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_json_sls_cases as jsc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_json_sls  # noqa: E402

pytestmark = pytest.mark.gpu

POISON, GUARD = 0xA5, 256
OKEY = jsc.OKEY
SPLIT = {"SourceKey": "content", "SplitChar": 10}
TAIL = b"\x1a\x05topic"


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _ml_handles(cfg):
    import loongcollector_b200 as lc
    p = orc.ProcessorSplitMultilineLogStringNative(cfg)
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


def _kw(jcfg, okey, pos, time, ns):
    return dict(renamed_key=jsc.renamed_key(jcfg), keep_fail=jcfg["KeepingSourceWhenParseFail"],
                keep_succeed=jcfg["KeepingSourceWhenParseSucceed"], copy_raw=jcfg["CopingRawLog"], offset_key=okey,
                src_pos=pos, time=time, time_ns=ns)


def _emul(val, jcfg, okey, pos, time, ns, ml=None):
    if ml is None:
        off, ln = orc.split_lines(val, 10)
    else:
        p = orc.ProcessorSplitMultilineLogStringNative(ml)
        off, ln, _fl, _c = orc.multiline_split(val, p.start, p.cont, p.end, p.opts.discard)
    sk = jcfg["SourceKey"].encode()
    st, first, ent, arena, _ = ojs.process(sk, np.frombuffer(val, np.uint8), off, ln)
    return split_json_sls.serialize(val, off, ln, (st, first, ent, arena), sk, jsc.renamed_key(jcfg),
                                    jcfg["KeepingSourceWhenParseFail"], jcfg["KeepingSourceWhenParseSucceed"],
                                    jcfg["CopingRawLog"], okey, pos, time, ns, 32)


def device_chain(eng, val, jcfg, okey, pos, time, ns, ml=None):
    """split, JSON and serialise on the device into a poisoned buffer with guard bytes; checks the sizing query, the
    capacity refusal and the guard; returns (wire bytes, counters)"""
    import torch

    import loongcollector_b200 as lc
    js = lc.Json(jcfg["SourceKey"])
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
        n, _ = eng.multiline_split_dev(d.data_ptr(), len(val), *_ml_handles(ml), d_off.data_ptr(), d_len.data_ptr(),
                                       d_fl.data_ptr(), cap)
    st = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    first = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    cnt = torch.empty(3, dtype=torch.int64, device="cuda")
    base = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n)
    ecap = acap = 0
    ent = ar = torch.empty(16, dtype=torch.uint8, device="cuda")
    for k in range(4):
        try:
            eng.json_parse_dev(js, *base, st.data_ptr(), first.data_ptr(), ent.data_ptr(), ecap, ar.data_ptr(), acap,
                               cnt.data_ptr())
            break
        except lc.LcError as e:
            assert e.code == lc.capi.LC_ERR_CAPACITY and k < 3
            ecap, acap = int(first[n].item()) + 1, (len(val) + 64) * 16 ** (k + 1)
            ent = torch.empty(ecap * 16, dtype=torch.uint8, device="cuda")
            ar = torch.empty(acap, dtype=torch.uint8, device="cuda")
    args = (js,) + base + (st.data_ptr(), first.data_ptr(), ent.data_ptr(), ar.data_ptr())
    kw = _kw(jcfg, okey, pos, time, ns)
    need, ctr0 = eng.sls_serialize_split_json_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_json_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_json_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr]


def _all_calls(eng, val, jcfg, okey, pos, time, ns, ml=None):
    """every call of the chain on one input equals the oracle chain and the host build"""
    import loongcollector_b200 as lc
    split_cfg = ml or {"SourceKey": jcfg["SourceKey"], "SplitChar": 10}
    want, wctr, wml, npieces = jsc.oracle_chain(val, split_cfg, jcfg, time, ns, pos, okey, multiline=ml is not None)
    assert _emul(val, jcfg, okey, pos, time, ns, ml) == (want, wctr)
    assert device_chain(eng, val, jcfg, okey, pos, time, ns, ml) == (want, wctr)
    js = lc.Json(jcfg["SourceKey"])
    kw = _kw(jcfg, okey, pos, time, ns)
    if ml is None:
        data, nev, ctr = eng.split_json_parse_sls(js, val, 10, **kw)
        block, raw, nev2, ctr2 = eng.split_json_parse_sls_lz4(js, val, 10, **kw, tail=TAIL)
    else:
        h = _ml_handles(ml)
        data, nev, ctr, mctr = eng.multiline_split_json_parse_sls(js, val, *h, **kw)
        block, raw, nev2, ctr2, mctr2 = eng.multiline_split_json_parse_sls_lz4(js, val, *h, **kw, tail=TAIL)
        assert [int(x) for x in mctr] == [int(x) for x in mctr2]
    assert data == want and [int(x) for x in ctr] == wctr and nev == npieces
    assert raw == len(want) + len(TAIL) and nev2 == nev and list(ctr2) == list(ctr)
    assert lz4_block.decode(block) == want + TAIL


CONFIGS = [(f"{r}_{i}", c) for r in (None, "raw", "__raw_log__", OKEY.decode()) for i, c in
           enumerate(jsc.flag_configs(r))]


@pytest.mark.parametrize("okey", [None, OKEY], ids=["no_offset", "offset"])
@pytest.mark.parametrize("cid,jcfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix(eng, cid, jcfg, okey):
    val = jsc.random_value(len(cid) * 7 + (0 if okey is None else 1))
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _all_calls(eng, val, jcfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns)


@pytest.mark.parametrize("okey", [b"a", b"raw", b"__raw_log__", b"dup"])
def test_offset_key_equal_to_member_or_added_keys(eng, okey):
    val = b"\n".join(jsc.special_lines(okey=okey))
    for f in (0, 3, 5, 7):
        jcfg = jsc.config("content", "raw", bool(f & 1), bool(f & 2), bool(f & 4))
        _all_calls(eng, val, jcfg, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("name", list(sc.ML_CFGS))
def test_multiline(eng, name):
    rng = random.Random(len(name))
    val = sc.ml_value(rng, 12) + b"\n" + b"\n".join(jsc.special_lines())
    _all_calls(eng, val, jsc.config("content", "raw", True, True, True), OKEY, 1 << 20, 1700000000, 7,
               ml=sc.ml_config(name))


def test_empty_and_erased_chunks(eng):
    for val in (b"", b"\n\n", b"x\ny\n", b"{}\n{}"):
        for f in (0, 1, 7):
            jcfg = jsc.config("content", None, bool(f & 1), bool(f & 2), bool(f & 4))
            for okey in (None, OKEY):
                _all_calls(eng, val, jcfg, okey, 5, 1700000000, None)


def test_wide_lines_among_short_ones(eng):
    """1 MiB-class lines of 10^5 members, distinct (some escaped) and all alike, in one call with short lines and
    with events the JSON walk hands to its slow path (deep nesting)"""
    deep = b'{"d":' + b"[" * 100 + b"]" * 100 + b', "d":2}'
    lines = [b'{"a":1}', jsc.big_doc(100000, escaped_every=7), b'{"a":2,"a":3}', jsc.big_doc(100000, alike=True),
             deep, b"bad", jsc.big_doc(33)] + jsc.special_lines()
    val = b"\n".join(lines)
    assert len(jsc.big_doc(100000)) > 1 << 20
    _all_calls(eng, val, jsc.config("content", "raw", True, True, False), OKEY, 1 << 40, 1700000000, 3)


def test_synth_json_lines(eng):
    from loongcollector_b200 import synth
    buf = synth.json_lines(3000, seed=5)[0]
    val = bytes(buf)
    _all_calls(eng, val, jsc.config("content", None, False, False), OKEY, 0, 1700000000, None)


def test_refusals(eng):
    import loongcollector_b200 as lc
    js = lc.Json("content")
    kw = dict(renamed_key=b"content", offset_key=b"content")
    calls = [lambda: eng.split_json_parse_sls(js, b"{}\n", 10, **kw),
             lambda: eng.split_json_parse_sls_lz4(js, b"{}\n", 10, **kw),
             lambda: eng.multiline_split_json_parse_sls(js, b"{}\n", None, None, None, False, **kw),
             lambda: eng.sls_serialize_split_json_dev(js, None, 0, None, None, 0, None, None, None, None, **kw)]
    for call in calls:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    # refused before the device is touched, so the tables may be any non-null address
    big = [lambda: eng.sls_serialize_split_json_dev(js, None, 1 << 31, None, None, 0, None, None, None, None,
                                                    renamed_key=b"content"),
           lambda: eng.sls_serialize_split_json_dev(js, 16, 16, 16, 16, 1 << 30, 16, 16, 16, 16,
                                                    renamed_key=b"content")]
    for call in big:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_TOO_LARGE
