"""GPU tier: the split -> Apsara chain (lc_sls_serialize_split_apsara_dev, lc_split_apsara_parse_sls[_lz4],
lc_multiline_split_apsara_parse_sls[_lz4]) against the oracle's splitter + oracle/apsara.py's ProcessorParseApsaraNative
+ sls_serialize_logs and the host build of the chain: bytes and counters, poisoned outputs with guard bytes, the
sizing query, the capacity refusal, the other refusals, and LZ4 blocks that decode to the records ‖ tail."""
import numpy as np
import pytest

from oracle import oracle as orc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_apsara_sls_cases as ac  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_apsara_sls  # noqa: E402

pytestmark = pytest.mark.gpu

POISON, GUARD = 0xA5, 256
OKEY = ac.OKEY
TAIL = b"\x1a\x05topic"


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _ml_handles():
    import loongcollector_b200 as lc
    p = orc.ProcessorSplitMultilineLogStringNative(ac.ml_config())
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


def _kw(acfg, okey, pos, time, ns, enable_ns):
    return dict(renamed_key=ac.renamed_key(acfg), keep_fail=acfg["KeepingSourceWhenParseFail"],
                keep_succeed=acfg["KeepingSourceWhenParseSucceed"], copy_raw=acfg["CopingRawLog"], offset_key=okey,
                src_pos=pos, time=time, time_ns=ns if enable_ns else None, enable_ns=enable_ns)


def _emul(val, acfg, okey, pos, time, ns, enable_ns, ml, di):
    if not ml:
        off, ln = orc.split_lines(val, 10)
    else:
        p = orc.ProcessorSplitMultilineLogStringNative(ac.ml_config())
        off, ln, _fl, _c = orc.multiline_split(val, p.start, p.cont, p.end, p.opts.discard)
    return split_apsara_sls.serialize(val, off, ln, acfg["SourceKey"].encode(), ac.adjust(acfg), ac.NOW, di,
                                      ac.renamed_key(acfg), acfg["KeepingSourceWhenParseFail"],
                                      acfg["KeepingSourceWhenParseSucceed"], acfg["CopingRawLog"], okey, pos, time,
                                      ns if enable_ns else None, enable_ns, 32)


def device_chain(eng, val, acfg, okey, pos, time, ns, enable_ns, ml, di):
    """split, Apsara and serialise on the device into a poisoned buffer with guard bytes; checks the sizing query, the
    capacity refusal and the guard; returns (wire bytes, counters)"""
    import torch

    import loongcollector_b200 as lc
    ap = lc.Apsara(acfg["SourceKey"], ac.adjust(acfg))
    d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
    if val:
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    cap = max(len(val), 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    if not ml:
        n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), cap)
    else:
        d_fl = torch.empty(cap, dtype=torch.uint8, device="cuda")
        n, _ = eng.multiline_split_dev(d.data_ptr(), len(val), *_ml_handles(), d_off.data_ptr(), d_len.data_ptr(),
                                       d_fl.data_ptr(), cap)
    m1 = max(n, 1)
    st = torch.empty(m1, dtype=torch.uint8, device="cuda")
    sec = torch.empty(m1, dtype=torch.int64, device="cuda")
    nsec = torch.empty(m1, dtype=torch.int32, device="cuda")
    micro = torch.empty(m1, dtype=torch.int64, device="cuda")
    first = torch.empty(n + 1, dtype=torch.int64, device="cuda")
    cnt = torch.empty(5, dtype=torch.int64, device="cuda")
    grp = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    pargs = (ap, d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, grp.data_ptr(), 1, ac.NOW, di,
             st.data_ptr(), sec.data_ptr(), nsec.data_ptr(), micro.data_ptr(), first.data_ptr())
    ent = torch.empty(16, dtype=torch.uint8, device="cuda")
    try:
        eng.apsara_parse_dev(*pargs, ent.data_ptr(), 0, cnt.data_ptr())
    except lc.LcError as e:
        assert e.code == lc.capi.LC_ERR_CAPACITY
        m = int(first[n].item())
        ent = torch.empty(m * 16, dtype=torch.uint8, device="cuda")
        eng.apsara_parse_dev(*pargs, ent.data_ptr(), m, cnt.data_ptr())
    args = (ap, d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), sec.data_ptr(),
            nsec.data_ptr(), micro.data_ptr(), first.data_ptr(), ent.data_ptr())
    kw = _kw(acfg, okey, pos, time, ns, enable_ns)
    need, ctr0 = eng.sls_serialize_split_apsara_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_apsara_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_apsara_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr]


def _all_calls(eng, val, acfg, okey, pos, time, ns, enable_ns=True, ml=False, di=ac.DI):
    """every call of the chain on one input equals the oracle chain and the host build"""
    import loongcollector_b200 as lc
    split_cfg = ac.ml_config(acfg["SourceKey"]) if ml else {"SourceKey": acfg["SourceKey"], "SplitChar": 10}
    want, wctr, _, npieces = ac.oracle_chain(val, split_cfg, acfg, time, ns, pos, okey, multiline=ml,
                                               enable_ns=enable_ns, di=di)
    assert _emul(val, acfg, okey, pos, time, ns, enable_ns, ml, di) == (want, wctr)
    assert device_chain(eng, val, acfg, okey, pos, time, ns, enable_ns, ml, di) == (want, wctr)
    ap = lc.Apsara(acfg["SourceKey"], ac.adjust(acfg))
    kw = dict(_kw(acfg, okey, pos, time, ns, enable_ns), now=ac.NOW, discard_interval=di)
    if not ml:
        data, nev, ctr = eng.split_apsara_parse_sls(ap, val, 10, **kw)
        block, raw, nev2, ctr2 = eng.split_apsara_parse_sls_lz4(ap, val, 10, **kw, tail=TAIL)
    else:
        h = _ml_handles()
        data, nev, ctr, mctr = eng.multiline_split_apsara_parse_sls(ap, val, *h, **kw)
        block, raw, nev2, ctr2, mctr2 = eng.multiline_split_apsara_parse_sls_lz4(ap, val, *h, **kw, tail=TAIL)
        assert [int(x) for x in mctr] == [int(x) for x in mctr2]
    assert data == want and [int(x) for x in ctr] == wctr and nev == npieces
    assert raw == len(want) + len(TAIL) and nev2 == nev and list(ctr2) == list(ctr)
    assert lz4_block.decode(block) == want + TAIL
    return want, wctr


CONFIGS = [(f"{r}_{i}", c) for r in (None, "raw", "__raw_log__", OKEY.decode(), "microtime") for i, c in
           enumerate(ac.flag_configs(r))]


@pytest.mark.parametrize("okey", [None, OKEY], ids=["no_offset", "offset"])
@pytest.mark.parametrize("cid,acfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix(eng, cid, acfg, okey):
    val = ac.random_value(len(cid) * 7 + (0 if okey is None else 1))
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _all_calls(eng, val, acfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns, enable_ns=len(cid) % 2 == 0)


@pytest.mark.parametrize("source", ["content", "k1", "__THREAD__", "microtime"])
def test_source_and_offset_keys_equal_to_fields(eng, source):
    val = b"\n".join(ac.special_lines(source=source) + ac.special_lines(okey=b"__LEVEL__"))
    for f in (0, 3, 5, 7):
        for okey in (None, b"k1", b"__LEVEL__", b"microtime", b"raw", b"__raw_log__"):
            if okey == source.encode():
                continue  # refused: test_refusals
            acfg = ac.config(source, "raw", bool(f & 1), bool(f & 2), bool(f & 4))
            _all_calls(eng, val, acfg, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("seed", range(3))
def test_multiline(eng, seed):
    val = ac.ml_value(seed, 30) + b"\n" + b"\n".join(ac.special_lines())
    for acfg in (ac.config("content", "raw", True, True, True), ac.config("content", None, False, False)):
        _all_calls(eng, val, acfg, OKEY, 1 << 20, 1700000000, 7, ml=True)


def test_discard_off_and_pinned_corners(eng):
    """the history discard off; short time strings whose cache key runs into the chunk; the widest epochs"""
    short = b"[2024-1-1 1:2:3]"
    val = b"\n".join([short, short + b"[2024-01-01 00:00:00]", b"[2024-01-01 01:02:03.7]", short,
                      b"[%d]\tk:v" % ac.BIG_EPOCH, b"[19999999999999999999]"] + ac.special_lines())
    for f in (0, 7):
        _all_calls(eng, val, ac.config("content", "raw", bool(f & 1), bool(f & 2), bool(f & 4)), OKEY, 0,
                   1700000000, 3, di=-1)


def test_empty_and_erased_chunks(eng):
    for val in (b"", b"\n\n", b"x\ny\n", ac.date(ac.BOUNDARY - 500) + b"\n" + ac.date(ac.BOUNDARY - 900)):
        for f in (0, 1, 7):
            acfg = ac.config("content", None, bool(f & 1), bool(f & 2), bool(f & 4))
            for okey in (None, OKEY):
                want, _ = _all_calls(eng, val, acfg, okey, 5, 1700000000, None)
                if val.startswith(b"[") and not f & 1:
                    assert want == b""


def test_wide_lines_among_short_ones(eng):
    """lines of 1 MiB (a long key:value run, a long message) in one chunk with short ones"""
    t = ac.NOW - 10
    wide_kv = ac.date(t, b".1") + b"\t[INFO]\t" + b"\t".join(b"k%d:%s" % (i % 50, b"v" * 40) for i in range(24000))
    wide_msg = ac.date(t, b".2") + b"\tmsg:" + b"x" * (1 << 20)
    assert len(wide_kv) > 1 << 20
    lines = [ac.date(t) + b"\tk:v", wide_kv, b"", ac.date(t, b".3") + b"\tk:w", wide_msg, b"bad"] + \
        ac.special_lines()
    _all_calls(eng, b"\n".join(lines), ac.config("content", "raw", True, True, False), OKEY, 1 << 40, 1700000000, 3)


def test_synth_apsara_lines(eng):
    from loongcollector_b200 import synth
    buf, off, ln, _grp = synth.apsara_lines(3000, seed=5)
    b = bytes(buf)
    val = b"\n".join(b[o:o + n] for o, n in zip(off.tolist(), ln.tolist()))
    _all_calls(eng, val, ac.config("content", None, False, False), OKEY, 0, 1700000000, None, di=-1)


def test_refusals(eng):
    import loongcollector_b200 as lc
    ap = lc.Apsara("content")
    kw = dict(renamed_key=b"content", offset_key=b"content")
    calls = [lambda: eng.split_apsara_parse_sls(ap, b"x\n", 10, **kw),
             lambda: eng.split_apsara_parse_sls_lz4(ap, b"x\n", 10, **kw),
             lambda: eng.multiline_split_apsara_parse_sls(ap, b"x\n", None, None, None, False, **kw),
             lambda: eng.sls_serialize_split_apsara_dev(ap, None, 0, None, None, 0, None, None, None, None, None,
                                                        None, **kw),
             lambda: eng.split_apsara_parse_sls(ap, b"x\n", 10, renamed_key=b"c", time_ns=5, enable_ns=False)]
    for call in calls:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    # refused before the device is touched, so the tables may be any non-null address
    big = [lambda: eng.sls_serialize_split_apsara_dev(ap, 16, 0xFFFFFFF0, 16, 16, 0, 16, 16, 16, 16, 16, 16,
                                                      renamed_key=b"content"),
           lambda: eng.sls_serialize_split_apsara_dev(ap, 16, 16, 16, 16, 1 << 30, 16, 16, 16, 16, 16, 16,
                                                      renamed_key=b"content")]
    for call in big:
        with pytest.raises(lc.LcError) as ei:
            call()
        assert ei.value.code == lc.capi.LC_ERR_TOO_LARGE
    assert isinstance(np.uint8(0), np.uint8)
