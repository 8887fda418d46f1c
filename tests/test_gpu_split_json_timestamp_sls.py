"""GPU tier: the split -> JSON -> timestamp chain (lc_json_parse_dev, lc_split_json_timestamp_tap_dev,
lc_timestamp_parse_dev with one group over the tap's value buffer, lc_sls_serialize_split_json_timestamp_dev, and the
host-buffer calls lc_[multiline_]split_json_timestamp_parse_sls[_lz4]) against the oracle's splitter +
ProcessorParseJsonNative + a group-level ProcessorParseTimestampNative step + sls_serialize_logs and the host build of
the chain: bytes and all eight counters, poisoned outputs with guard bytes, the sizing query, the capacity refusal,
the other refusals, LZ4 blocks that decode to the records ‖ tail, and a 1 MiB time value among short ones."""
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import lz4_block  # noqa: E402
from tests import split_json_timestamp_sls_cases as jtc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_json_timestamp_sls as emul  # noqa: E402

pytestmark = pytest.mark.gpu

POISON, GUARD = 0xA5, 256
OKEY = jtc.OKEY
TAIL = b"\x1a\x05topic"


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _ts(fmt):
    import loongcollector_b200 as lc
    return lc.Timestamp(fmt)


def _kw(jcfg, okey):
    return dict(keep_fail=jcfg["KeepingSourceWhenParseFail"], keep_succeed=jcfg["KeepingSourceWhenParseSucceed"],
                copy_raw=jcfg["CopingRawLog"], offset_key=okey)


def emulated(val, jcfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns):
    off, ln = orc.split_lines(val, 10)
    tables = jtc.tables_of(val, off, ln, jcfg)
    return emul.serialize(val, off, ln, tables, jcfg["SourceKey"].encode(), jtc.renamed_key(jcfg),
                          jcfg["KeepingSourceWhenParseFail"], jcfg["KeepingSourceWhenParseSucceed"],
                          jcfg["CopingRawLog"], okey, pos, t, ns, tkey, fmt, now, di, enable_ns, nlanes=32)


def device_chain(eng, val, jcfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns):
    """split, JSON, tap, timestamp passes and serialiser on the device into poisoned buffers with guard bytes; checks
    the sizing query, the capacity refusal and the guards; returns (wire bytes, counters[8], tap table, timestamp
    status, value buffer)"""
    import torch

    import loongcollector_b200 as lc
    js = lc.Json(jcfg["SourceKey"])
    d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
    if val:
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    cap = max(len(val), 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), cap)
    st = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    first = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    cnt = torch.empty(3, dtype=torch.int64, device="cuda")
    base = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n)
    ecap = acap = 0
    ent = ar = torch.empty(16, dtype=torch.uint8, device="cuda")
    for k in range(4):
        try:
            _m, abytes = eng.json_parse_dev(js, *base, st.data_ptr(), first.data_ptr(), ent.data_ptr(), ecap,
                                            ar.data_ptr(), acap, cnt.data_ptr())
            break
        except lc.LcError as e:
            assert e.code == lc.capi.LC_ERR_CAPACITY and k < 3
            ecap, acap = int(first[n].item()) + 1, (len(val) + 64) * 16 ** (k + 1)
            ent = torch.empty(ecap * 16, dtype=torch.uint8, device="cuda")
            ar = torch.empty(acap, dtype=torch.uint8, device="cuda")
    args = (js,) + base + (st.data_ptr(), first.data_ptr(), ent.data_ptr(), ar.data_ptr())
    kw = _kw(jcfg, okey)
    m = max(n, 1)
    vcap = len(val) + abytes
    vbuf = torch.full((vcap + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    v_off = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    v_len = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    eng.split_json_timestamp_tap_dev(*args, jtc.renamed_key(jcfg), tkey, vbuf.data_ptr(), vcap, v_off.data_ptr(),
                                     v_len.data_ptr(), **kw)
    grp = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    sec = torch.empty(m, dtype=torch.int64, device="cuda")
    nsec = torch.empty(m, dtype=torch.int32, device="cuda")
    tst = torch.full((m,), 9, dtype=torch.uint8, device="cuda")
    tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
    eng.timestamp_parse_dev(ts, vbuf.data_ptr(), vcap, v_off.data_ptr(), v_len.data_ptr(), n, grp.data_ptr(), 1, now,
                            di, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(), tcnt.data_ptr())
    tsa = (tst.data_ptr(), sec.data_ptr(), nsec.data_ptr())
    kw.update(src_pos=pos, time=t, time_ns=ns, enable_ns=enable_ns)
    need, ctr0 = eng.sls_serialize_split_json_timestamp_dev(*args, jtc.renamed_key(jcfg), *tsa, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_json_timestamp_dev(*args, jtc.renamed_key(jcfg), *tsa, **kw,
                                                       d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_json_timestamp_dev(*args, jtc.renamed_key(jcfg), *tsa, **kw,
                                                          d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    vb = vbuf.cpu().numpy()
    assert (vb[vcap:] == POISON).all(), "the tap wrote past the value buffer"
    tap = (v_off[:n].cpu().numpy().view(np.uint32), v_len[:n].cpu().numpy().view(np.uint32))
    return bytes(host[:need]), [int(x) for x in ctr], tap, tst[:n].cpu().numpy(), vb[:vcap]


def _same_values(tap, vb, wtap, wvb):
    """the device's tap table equals the host build's, and so do the bytes of every value"""
    assert np.array_equal(tap[0], wtap[0]) and np.array_equal(tap[1], wtap[1])
    for o, n in zip(*tap):
        if n != 0xFFFFFFFF:
            assert bytes(vb[o:o + n]) == wvb[o:o + n]


CONFIGS = list(jtc.configs())


@pytest.mark.parametrize("fmt", jtc.FORMATS)
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_dev_chain_matrix(eng, case, fmt):
    cid, jcfg, tkey, member = case
    ts = _ts(fmt)
    rng = random.Random(zlib.crc32((cid + fmt).encode()))
    val = jtc.lines_value(rng, fmt, 80, member)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di, enable_ns in ((43200, True), (-1, False)):
            ns_in = ns if enable_ns else None
            want, wctr, _, _ = jtc.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, jcfg, tkey, fmt,
                                                jtc.NOW, di, t, ns_in, pos, okey, enable_ns=enable_ns)
            ewant, ectr, wst, wtap, wvb = emulated(val, jcfg, tkey, fmt, jtc.NOW, di, enable_ns, okey, pos, t, ns_in)
            assert (ewant, ectr) == (want, wctr)
            got, ctr, tap, st, vb = device_chain(eng, val, jcfg, tkey, ts, jtc.NOW, di, enable_ns, okey, pos, t,
                                                 ns_in)
            assert got == want and ctr == wctr, (cid, fmt, okey, di)
            assert np.array_equal(st, wst)
            _same_values(tap, vb, wtap, wvb)


def _host(eng, call, val, jcfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns, tail=None, ml=None):
    import loongcollector_b200 as lc
    js = lc.Json(jcfg["SourceKey"])
    kw = dict(_kw(jcfg, okey), src_pos=pos, time=t, time_ns=ns, discard_interval=di, enable_ns=enable_ns)
    if tail is not None:
        kw["tail"] = tail
    if ml is None:
        return call(js, val, 10, jtc.renamed_key(jcfg), tkey, ts, now, **kw)
    return call(js, val, *ml, jtc.renamed_key(jcfg), tkey, ts, now, **kw)


def _ml_handles(cfg):
    import loongcollector_b200 as lc
    p = orc.ProcessorSplitMultilineLogStringNative(cfg)
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


@pytest.mark.parametrize("fmt", jtc.FORMATS)
def test_host_calls(eng, fmt):
    """all four host-buffer calls against the oracle; the LZ4 blocks decode to the records ‖ tail"""
    ts = _ts(fmt)
    rng = random.Random(11)
    for cid, jcfg, tkey, member in CONFIGS:
        val = jtc.lines_value(rng, fmt, 120, member)
        for okey, di, enable_ns in ((OKEY, 43200, True), (None, -1, False)):
            ns = 77 if enable_ns else None
            want, wctr, _, npieces = jtc.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, jcfg, tkey,
                                                      fmt, jtc.NOW, di, 1 << 30, ns, 5, okey, enable_ns=enable_ns)
            data, nev, ctr = _host(eng, eng.split_json_timestamp_parse_sls, val, jcfg, tkey, ts, jtc.NOW, di,
                                   enable_ns, okey, 5, 1 << 30, ns)
            assert data == want and list(ctr) == wctr and nev == npieces, cid
            blk, raw, nev, ctr = _host(eng, eng.split_json_timestamp_parse_sls_lz4, val, jcfg, tkey, ts, jtc.NOW, di,
                                       enable_ns, okey, 5, 1 << 30, ns, tail=TAIL)
            assert lz4_block.decode(blk) == want + TAIL and raw == len(want) + len(TAIL) and list(ctr) == wctr
    mcfg = {"SourceKey": "content", "StartPattern": r"\{.*", "UnmatchedContentTreatment": "single_line"}
    val = jtc.lines_value(rng, fmt, 100)
    jcfg = jtc.config("content", "raw", True, False, True)
    for tkey in (b"time", b"raw"):
        want, wctr, _wml, npieces = jtc.oracle_chain(val, mcfg, jcfg, tkey, fmt, jtc.NOW, 43200, 1 << 30, 3, 9, OKEY,
                                                    multiline=True)
        ml = _ml_handles(mcfg)
        data, nev, ctr, mctr = _host(eng, eng.multiline_split_json_timestamp_parse_sls, val, jcfg, tkey, ts, jtc.NOW,
                                     43200, True, OKEY, 9, 1 << 30, 3, ml=ml)
        assert data == want and list(ctr) == wctr and nev == npieces
        blk, raw, nev, ctr, mctr2 = _host(eng, eng.multiline_split_json_timestamp_parse_sls_lz4, val, jcfg, tkey, ts,
                                       jtc.NOW, 43200, True, OKEY, 9, 1 << 30, 3, tail=TAIL, ml=ml)
        assert lz4_block.decode(blk) == want + TAIL and list(ctr) == wctr
        assert [int(x) for x in mctr] == [int(x) for x in mctr2]


def test_sizing_query_and_capacity(eng):
    import loongcollector_b200 as lc
    ts = _ts(jtc.YMD)
    val = jtc.lines_value(random.Random(3), jtc.YMD, 50)
    jcfg = jtc.config("content")
    want, wctr, _, _ = jtc.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, jcfg, b"time", jtc.YMD,
                                        jtc.NOW, 43200, 1 << 30, None, 0, OKEY, enable_ns=False)
    assert want
    with pytest.raises(lc.LcError) as ei:
        eng.split_json_timestamp_parse_sls(lc.Json("content"), val, 10, b"content", b"time", ts, jtc.NOW, 43200,
                                           offset_key=OKEY, time=1 << 30, out_cap=len(want) - 1)
    assert ei.value.code == lc.capi.LC_ERR_CAPACITY
    data, _n, ctr = eng.split_json_timestamp_parse_sls(lc.Json("content"), val, 10, b"content", b"time", ts, jtc.NOW,
                                                       43200, offset_key=OKEY, time=1 << 30, out_cap=len(want))
    assert data == want and list(ctr) == wctr
    # every piece discarded: no bytes, and the LZ4 call returns the block of the tail alone
    old = b"\n".join(b'{"time":"%s"}' % jtc.render(jtc.YMD, jtc.NOW - 86400).encode() for _ in range(10))
    data, _n, ctr = eng.split_json_timestamp_parse_sls(lc.Json("content"), old, 10, b"content", b"time", ts, jtc.NOW,
                                                       43200)
    assert data == b"" and ctr[6] == 10
    blk, raw, _n, _c = eng.split_json_timestamp_parse_sls_lz4(lc.Json("content"), old, 10, b"content", b"time", ts,
                                                               jtc.NOW, 43200, tail=TAIL)
    assert lz4_block.decode(blk) == TAIL and raw == len(TAIL)


def test_refusals(eng):
    import loongcollector_b200 as lc
    ts = _ts(jtc.YMD)
    js = lc.Json("content")
    val = b'{"time":"x"}\n'
    for kw in (dict(offset_key=OKEY, tkey=OKEY), dict(offset_key=b"content", tkey=b"time"),
               dict(offset_key=None, tkey=b"time", time_ns=5, enable_ns=False)):
        tkey = kw.pop("tkey")
        with pytest.raises(lc.LcError) as ei:
            eng.split_json_timestamp_parse_sls(js, val, 10, b"content", tkey, ts, jtc.NOW, **kw)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    import torch
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    p = d.data_ptr()
    with pytest.raises(lc.LcError) as ei:  # tkey == offset key
        eng.split_json_timestamp_tap_dev(js, p, 13, p, p, 1, p, p, p, p, b"content", OKEY, p, 64, p, p,
                                         offset_key=OKEY)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    with pytest.raises(lc.LcError) as ei:  # a value buffer smaller than the source
        eng.split_json_timestamp_tap_dev(js, p, 13, p, p, 1, p, p, p, p, b"content", b"time", p, 12, p, p)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    with pytest.raises(lc.LcError) as ei:  # a source Time_ns without enable_ns
        eng.sls_serialize_split_json_timestamp_dev(js, p, 13, p, p, 1, p, p, p, p, b"content", p, p, p,
                                                   enable_ns=False, time_ns=5)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


def test_long_value_among_short_ones(eng):
    """a 1 MiB time string (plain, then escaped into the arena) among short ones: its warp shares the copy"""
    ts = _ts("%s")
    t0 = str(jtc.NOW - 10)
    big = t0 + "9" * (1 << 20)
    for esc in (False, True):
        v = jtc.escaped(big) if esc else '"%s"' % big
        lines = [b'{"time":"%s","i":%d}' % (t0.encode(), i) for i in range(300)]
        lines[150] = b'{"time":%s}' % v.encode()
        lines[151] = b'{"time":%s}' % jtc.escaped(t0).encode()
        val = b"\n".join(lines)
        jcfg = jtc.config("content")
        want, wctr, _, _ = jtc.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, jcfg, b"time", "%s",
                                            jtc.NOW, 43200, 1 << 30, 5, 0, None)
        got, ctr, tap, _st, vb = device_chain(eng, val, jcfg, b"time", ts, jtc.NOW, 43200, True, None, 0, 1 << 30, 5)
        assert got == want and ctr == wctr
        o, n = tap[0][150], tap[1][150]
        assert n == len(big) and bytes(vb[o:o + n]) == big.encode()
