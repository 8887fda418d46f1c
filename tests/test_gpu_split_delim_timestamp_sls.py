"""GPU tier: the split -> delimiter -> timestamp chain (lc_delim_parse_dev, lc_split_delim_timestamp_tap_dev,
lc_timestamp_parse_dev with one group over the tap's value buffer, lc_sls_serialize_split_delim_timestamp_dev, and the
host-buffer calls lc_[multiline_]split_delim_timestamp_parse_sls[_lz4]) against the oracle's splitter +
ProcessorParseDelimiterNative + a group-level ProcessorParseTimestampNative step + sls_serialize_logs and the host
build of the chain: bytes and all nine counters, poisoned outputs with guard bytes, the sizing query, the capacity
refusal, the other refusals, LZ4 blocks that decode to the records ‖ tail, and a 1 MiB piece and a 1 MiB quoted
column as time values among short ones."""
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_delim_timestamp_sls_cases as dtc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_delim_timestamp_sls as emul  # noqa: E402

pytestmark = pytest.mark.gpu

POISON, GUARD = 0xA5, 256
OKEY = dtc.OKEY
TAIL = b"\x1a\x05topic"
SPLIT = {"SourceKey": "content", "SplitChar": 10}


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _ts(fmt):
    import loongcollector_b200 as lc
    return lc.Timestamp(fmt)


def _dkw(cfg):
    """the delimiter stage's keyword arguments of the Engine bindings, without allow_short / max_fields"""
    a = dtc.device_args(cfg)
    return {k: v for k, v in a.items() if k not in ("allow_short", "max_fields")}


def emulated(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns):
    off, ln = orc.split_lines(val, 10)
    tabs = dtc.tables(val, off, ln, cfg)
    quote = cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')
    return emul.serialize(val, off, ln, tabs, cfg["max_fields"], cfg["sep"], quote, cfg["treatment"],
                          [k.encode() for k in cfg["keys"]], cfg["source"].encode(), dc.renamed_key(cfg),
                          cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], okey, pos, t, ns, tkey, fmt, now, di,
                          enable_ns, nlanes=32)


def device_chain(eng, val, cfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns):
    """split, delimiter, tap, timestamp passes and serialiser on the device into poisoned buffers with guard bytes;
    checks the sizing query, the capacity refusal and the guards; returns (wire bytes, counters[9], tap table,
    timestamp status, value buffer)"""
    import torch

    import loongcollector_b200 as lc
    d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
    if val:
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
    cap = max(len(val), 1)
    d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
    d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
    n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), cap)
    a = dtc.device_args(cfg)
    MF = a["max_fields"]
    m = max(n, 1)
    st = torch.empty(m, dtype=torch.uint8, device="cuda")
    nf = torch.empty(m, dtype=torch.int32, device="cuda")
    fo, fl, fd = (torch.empty(m * MF, dtype=torch.int32, device="cuda") for _ in range(3))
    if n:
        eng.delim_parse_dev(d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, a["sep"], a["quote"],
                            len(a["keys"]), a["treatment"] == "extend", a["allow_short"], MF, st.data_ptr(),
                            nf.data_ptr(), fo.data_ptr(), fl.data_ptr(), fd.data_ptr())
    args = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), nf.data_ptr(),
            fo.data_ptr(), fl.data_ptr(), fd.data_ptr(), MF)
    kw = _dkw(cfg)
    vcap = len(val)
    vbuf = torch.full((vcap + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    v_off = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    v_len = torch.full((m,), -1, dtype=torch.int32, device="cuda")
    dk = dict(kw)
    tk = dict(sep=dk.pop("sep"), quote=dk.pop("quote"), treatment=dk.pop("treatment"), keys=dk.pop("keys"),
              source_key=dk.pop("source_key"))
    eng.split_delim_timestamp_tap_dev(*args, tk["sep"], tk["quote"], tk["treatment"], tk["keys"], tk["source_key"],
                                      tkey, vbuf.data_ptr(), vcap, v_off.data_ptr(), v_len.data_ptr(), offset_key=okey,
                                      **dk)
    grp = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    sec = torch.empty(m, dtype=torch.int64, device="cuda")
    nsec = torch.empty(m, dtype=torch.int32, device="cuda")
    tst = torch.full((m,), 9, dtype=torch.uint8, device="cuda")
    tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
    eng.timestamp_parse_dev(ts, vbuf.data_ptr(), vcap, v_off.data_ptr(), v_len.data_ptr(), n, grp.data_ptr(), 1, now,
                            di, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(), tcnt.data_ptr())
    tsa = (tst.data_ptr(), sec.data_ptr(), nsec.data_ptr())
    skw = dict(dk, offset_key=okey, src_pos=pos, time=t, time_ns=ns, enable_ns=enable_ns)
    sargs = args + (tk["sep"], tk["quote"], tk["treatment"], tk["keys"], tk["source_key"]) + tsa
    need, ctr0 = eng.sls_serialize_split_delim_timestamp_dev(*sargs, **skw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_delim_timestamp_dev(*sargs, **skw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_delim_timestamp_dev(*sargs, **skw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    vb = vbuf.cpu().numpy()
    assert (vb[vcap:] == POISON).all(), "the tap wrote past the value buffer"
    tap = (v_off[:n].cpu().numpy().view(np.uint32), v_len[:n].cpu().numpy().view(np.uint32))
    return bytes(host[:need]), [int(x) for x in ctr], tap, tst[:n].cpu().numpy(), vb[:vcap]


def _same_values(tap, vb, wtap, wvb):
    """the device's tap table equals the host build's, and so do the bytes of every value"""
    assert np.array_equal(tap[1], wtap[1])
    for o, wo, n in zip(tap[0], wtap[0], tap[1]):
        if n != 0xFFFFFFFF:
            assert o == wo and bytes(vb[o:o + n]) == wvb[o:o + n]


CONFIGS = list(dtc.configs())
BARE = {"renamed_keep_succeed", "renamed_fail", "raw_log_fail"}
# the formats whose strings can stand where each configuration reads its time: a separator or a quote inside needs the
# quote state machine, and the piece itself is the value of the bare configurations
MATRIX = [(c, f) for c in CONFIGS for f in dtc.FORMATS
          if dtc.plain_fmt(f, c[1]) and not (c[0] in BARE and f in (dtc.COMMA_FMT, dtc.DQ_FMT))]


@pytest.mark.parametrize("case,fmt", MATRIX, ids=["%s-%s" % (c[0], f) for c, f in MATRIX])
def test_dev_chain_matrix(eng, case, fmt):
    cid, cfg, tkey, gen = case
    ts = _ts(fmt)
    rng = random.Random(zlib.crc32((cid + fmt).encode()))
    val = gen(rng, fmt)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di, enable_ns in ((43200, True), (-1, False)):
            ns_in = ns if enable_ns else None
            want, wctr, _, _ = dtc.oracle_chain(val, SPLIT, cfg, tkey, fmt, dtc.NOW, di, t, ns_in, pos, okey,
                                                enable_ns=enable_ns)
            ewant, ectr, wst, wtap, wvb = emulated(val, cfg, tkey, fmt, dtc.NOW, di, enable_ns, okey, pos, t, ns_in)
            assert (ewant, dtc.fold(ectr)) == (want, wctr)
            got, ctr, tap, st, vb = device_chain(eng, val, cfg, tkey, ts, dtc.NOW, di, enable_ns, okey, pos, t, ns_in)
            assert got == want and ctr == ectr, (cid, fmt, okey, di)
            assert np.array_equal(st, wst)
            _same_values(tap, vb, wtap, wvb)


def _host(eng, call, val, cfg, tkey, ts, now, di, enable_ns, okey, pos, t, ns, tail=None, ml=None):
    a = dtc.device_args(cfg)
    kw = dict(renamed_key=a["renamed_key"], keep_fail=a["keep_fail"], keep_succeed=a["keep_succeed"],
              copy_raw=a["copy_raw"], allow_short=a["allow_short"], max_fields=a["max_fields"], offset_key=okey,
              src_pos=pos, time=t, time_ns=ns, discard_interval=di, enable_ns=enable_ns)
    if tail is not None:
        kw["tail"] = tail
    head = (10,) if ml is None else ml
    return call(val, *head, a["sep"], a["quote"], a["treatment"], a["keys"], a["source_key"], tkey, ts, now, **kw)


def _ml_handles(cfg):
    import loongcollector_b200 as lc
    p = orc.ProcessorSplitMultilineLogStringNative(cfg)
    rx = lambda r: lc.Regex(r.pattern) if r is not None else None  # noqa: E731
    return rx(p.start), rx(p.cont), rx(p.end), p.opts.discard


@pytest.mark.parametrize("fmt", [dtc.YMD, "%s", dtc.COMMA_FMT, dtc.DQ_FMT])
def test_host_calls(eng, fmt):
    """all four host-buffer calls against the oracle; the LZ4 blocks decode to the records ‖ tail"""
    ts = _ts(fmt)
    rng = random.Random(11)
    for cid, cfg, tkey, gen in CONFIGS:
        if not dtc.plain_fmt(fmt, cfg) or (cid in BARE and fmt in (dtc.COMMA_FMT, dtc.DQ_FMT)):
            continue
        val = gen(rng, fmt)
        for okey, di, enable_ns in ((OKEY, 43200, True), (None, -1, False)):
            ns = 77 if enable_ns else None
            want, wctr, _, npieces = dtc.oracle_chain(val, SPLIT, cfg, tkey, fmt, dtc.NOW, di, 1 << 30, ns, 5, okey,
                                                      enable_ns=enable_ns)
            data, nev, ctr = _host(eng, eng.split_delim_timestamp_parse_sls, val, cfg, tkey, ts, dtc.NOW, di,
                                   enable_ns, okey, 5, 1 << 30, ns)
            assert data == want and dtc.fold(ctr) == wctr and nev == npieces, cid
            blk, raw, nev, ctr = _host(eng, eng.split_delim_timestamp_parse_sls_lz4, val, cfg, tkey, ts, dtc.NOW, di,
                                       enable_ns, okey, 5, 1 << 30, ns, tail=TAIL)
            assert lz4_block.decode(blk) == want + TAIL and raw == len(want) + len(TAIL) and dtc.fold(ctr) == wctr
    # the multiline splitter, with quoted time columns that hold the split char
    mcfg = {"SourceKey": "content", "StartPattern": r"\d.*", "UnmatchedContentTreatment": "single_line"}
    t0 = dtc.render(fmt, dtc.NOW - 30).encode()
    recs = []
    for i in range(60):
        q = dtc.field(t0, b",", ord('"')) if rng.random() < 0.5 else b'"' + t0.replace(b'"', b'""') + b'\n"'
        recs.append(b"%d,%s,m\nmore %d" % (i, q, i) if rng.random() < 0.5 else b"%d,%s,m" % (i, q))
    val = b"\n".join(recs)
    cfg = dtc.config(["i", "time", "msg"], renamed="raw", keep_fail=True, copy_raw=True)
    ml = _ml_handles(mcfg)
    for tkey in (b"time", b"raw"):
        want, wctr, _wml, npieces = dtc.oracle_chain(val, mcfg, cfg, tkey, fmt, dtc.NOW, 43200, 1 << 30, 3, 9, OKEY,
                                                     multiline=True)
        data, nev, ctr, mctr = _host(eng, eng.multiline_split_delim_timestamp_parse_sls, val, cfg, tkey, ts,
                                     dtc.NOW, 43200, True, OKEY, 9, 1 << 30, 3, ml=ml)
        assert data == want and dtc.fold(ctr) == wctr and nev == npieces
        blk, raw, nev, ctr, mctr2 = _host(eng, eng.multiline_split_delim_timestamp_parse_sls_lz4, val, cfg, tkey, ts,
                                          dtc.NOW, 43200, True, OKEY, 9, 1 << 30, 3, tail=TAIL, ml=ml)
        assert lz4_block.decode(blk) == want + TAIL and dtc.fold(ctr) == wctr
        assert [int(x) for x in mctr] == [int(x) for x in mctr2]


def test_lz4_blocks_are_the_siblings_bytes_and_tail(eng):
    """with a tkey the stage leaves absent, every record keeps the source time: the chain's bytes are the split ->
    delimiter chain's"""
    ts = _ts(dtc.YMD)
    val = dtc.lines_value(random.Random(2), dtc.YMD, 200)
    cfg = dtc.config(["time", "level", "msg"], keep_fail=True)
    a = dtc.device_args(cfg)
    kw = dict(renamed_key=a["renamed_key"], keep_fail=True, allow_short=a["allow_short"], max_fields=a["max_fields"],
              offset_key=OKEY, src_pos=3, time=1 << 30)
    sib, _n, sctr = eng.split_delim_parse_sls(val, 10, a["sep"], a["quote"], a["treatment"], a["keys"],
                                              a["source_key"], **kw)
    blk, raw, _n, ctr = eng.split_delim_timestamp_parse_sls_lz4(val, 10, a["sep"], a["quote"], a["treatment"],
                                                                a["keys"], a["source_key"], b"nope", ts, dtc.NOW,
                                                                43200, tail=TAIL, **kw)
    assert lz4_block.decode(blk) == sib + TAIL and raw == len(sib) + len(TAIL)
    assert list(ctr[:4]) == list(sctr) and ctr[4] == sctr[0] + sctr[3] + sctr[1] - sctr[2]


def test_sizing_query_and_capacity(eng):
    import loongcollector_b200 as lc
    ts = _ts(dtc.YMD)
    val = dtc.lines_value(random.Random(3), dtc.YMD, 50)
    cfg = dtc.config(["time", "level", "msg"], keep_fail=False)
    a = dtc.device_args(cfg)
    pos = (val, 10, a["sep"], a["quote"], a["treatment"], a["keys"], a["source_key"], b"time", ts, dtc.NOW, 43200)
    kw = dict(offset_key=OKEY, time=1 << 30, max_fields=a["max_fields"])
    want, wctr, _, _ = dtc.oracle_chain(val, SPLIT, cfg, b"time", dtc.YMD, dtc.NOW, 43200, 1 << 30, None, 0, OKEY,
                                        enable_ns=False)
    assert want
    with pytest.raises(lc.LcError) as ei:
        eng.split_delim_timestamp_parse_sls(*pos, **kw, out_cap=len(want) - 1)
    assert ei.value.code == lc.capi.LC_ERR_CAPACITY
    data, _n, ctr = eng.split_delim_timestamp_parse_sls(*pos, **kw, out_cap=len(want))
    assert data == want and dtc.fold(ctr) == wctr
    # every piece discarded: no bytes, and the LZ4 call returns the block of the tail alone
    old = b"\n".join(b"%s,%d" % (dtc.render(dtc.YMD, dtc.NOW - 86400).encode(), i) for i in range(10))
    data, _n, ctr = eng.split_delim_timestamp_parse_sls(old, *pos[1:])
    assert data == b"" and ctr[7] == 10
    blk, raw, _n, _c = eng.split_delim_timestamp_parse_sls_lz4(old, *pos[1:], tail=TAIL)
    assert lz4_block.decode(blk) == TAIL and raw == len(TAIL)
    # every piece erased by the delimiter stage
    data, _n, ctr = eng.split_delim_timestamp_parse_sls(b'"a\n"b\n"c', *pos[1:])
    assert data == b"" and list(ctr) == [0, 3, 3, 0, 0, 0, 0, 0, 0]


def test_refusals(eng):
    import loongcollector_b200 as lc
    ts = _ts(dtc.YMD)
    val = b"x,1\n"
    for keys, treatment, tkey, kw in (
            ([b"a", b"b"], "extend", OKEY, dict(offset_key=OKEY)),
            ([b"a", b"b"], "extend", b"__column2__", {}),
            ([b"a", b"b"], "keep", b"__column0__", dict(offset_key=OKEY)),
            ([b"a", b"b"], "extend", b"a", dict(offset_key=b"content")),
            ([b"a", b"b"], "extend", b"a", dict(time_ns=5, enable_ns=False)),
            ([b"a", b"a"], "extend", b"a", {})):
        with pytest.raises(lc.LcError) as ei:
            eng.split_delim_timestamp_parse_sls(val, 10, b",", ord('"'), treatment, keys, b"content", tkey, ts,
                                                dtc.NOW, **kw)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG, (keys, tkey, kw)
    # an overflow-form tkey is an ordinary key when overflow columns are discarded
    eng.split_delim_timestamp_parse_sls(val, 10, b",", ord('"'), "discard", [b"a", b"b"], b"content", b"__column2__",
                                        ts, dtc.NOW)
    import torch
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    p = d.data_ptr()
    tab = (p, 13, p, p, 1, p, p, p, p, p, 4)
    with pytest.raises(lc.LcError) as ei:  # tkey == offset key
        eng.split_delim_timestamp_tap_dev(*tab, b",", ord('"'), "extend", [b"a", b"b"], b"content", OKEY, p, 64, p, p,
                                          offset_key=OKEY)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    with pytest.raises(lc.LcError) as ei:  # a value buffer smaller than the source
        eng.split_delim_timestamp_tap_dev(*tab, b",", ord('"'), "extend", [b"a", b"b"], b"content", b"a", p, 12, p, p)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    with pytest.raises(lc.LcError) as ei:  # a source Time_ns without enable_ns
        eng.sls_serialize_split_delim_timestamp_dev(*tab, b",", ord('"'), "extend", [b"a", b"b"], b"content", p, p,
                                                    p, enable_ns=False, time_ns=5)
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


def test_long_values_among_short_ones(eng):
    """a 1 MiB piece (the whole line under RenamedSourceKey) and a 1 MiB quoted column with doubled quotes as time
    values among short ones: their warps share the copy and the collapse"""
    ts = _ts("%s")
    t0 = str(dtc.NOW - 10).encode()
    big = t0 + b"9" * (1 << 20)
    cfg = dtc.config(["time", "i"], renamed="raw", keep_succeed=True)
    lines = [b"%s,%d" % (t0, i) for i in range(300)]
    lines[150] = b'"%s%s"' % (t0, b'""' * (1 << 19))  # collapses to t0 + 2^19 quotes
    lines[151] = big  # one column: the short row keeps the piece under "raw"
    lines[152] = b'"%s"' % t0
    val = b"\n".join(lines)
    for tkey in (b"time", b"raw"):
        want, wctr, _, _ = dtc.oracle_chain(val, SPLIT, cfg, tkey, "%s", dtc.NOW, 43200, 1 << 30, 5, 0, None)
        ewant, ectr, wst, wtap, wvb = emulated(val, cfg, tkey, "%s", dtc.NOW, 43200, True, None, 0, 1 << 30, 5)
        assert (ewant, dtc.fold(ectr)) == (want, wctr)
        got, ctr, tap, st, vb = device_chain(eng, val, cfg, tkey, ts, dtc.NOW, 43200, True, None, 0, 1 << 30, 5)
        assert got == want and ctr == ectr
        assert np.array_equal(st, wst)
        _same_values(tap, vb, wtap, wvb)
        if tkey == b"time":
            o, n = tap[0][150], tap[1][150]
            assert n == len(t0) + (1 << 19) and bytes(vb[o:o + n]) == t0 + b'"' * (1 << 19)
        else:
            o, n = tap[0][151], tap[1][151]
            assert n == len(big) and bytes(vb[o:o + n]) == big
