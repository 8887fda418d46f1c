"""GPU tier: the split -> delimiter -> SLS chain.  lc_sls_serialize_split_delim_dev over the device tables of
lc_split_lines_dev / lc_multiline_split_dev and lc_delim_parse_dev, the four host calls, and the splitters'
SerializeSls(group, delimiter) against the oracle chain (its splitter, then its ProcessorParseDelimiterNative, then
sls_serialize_logs) and against Process + Process + Serialize, byte for byte and counter for counter."""
import random
import zlib

import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import split_delim_sls_cases as sdc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = sdc.OKEY


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


def device_chain(eng, val, cfg, okey, pos, time, ns, ml=None):
    """split, delimiter and serialise on the device into a poisoned buffer with guard bytes; checks the sizing query,
    the capacity refusal and the guard; returns (wire bytes, counters[4])"""
    import torch

    import loongcollector_b200 as lc
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
        n, _ = eng.multiline_split_dev(d.data_ptr(), len(val), *ml, d_off.data_ptr(), d_len.data_ptr(),
                                       d_fl.data_ptr(), cap)
    a = sdc.device_args(cfg)
    MF = a["max_fields"]
    st = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    nf = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
    fo, fl, fd = (torch.empty(max(n, 1) * MF, dtype=torch.int32, device="cuda") for _ in range(3))
    if n:
        eng.delim_parse_dev(d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, a["sep"], a["quote"],
                            len(a["keys"]), a["treatment"] == "extend", a["allow_short"], MF, st.data_ptr(),
                            nf.data_ptr(), fo.data_ptr(), fl.data_ptr(), fd.data_ptr())
    args = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), nf.data_ptr(),
            fo.data_ptr(), fl.data_ptr(), fd.data_ptr(), MF)
    kw = {k: v for k, v in a.items() if k not in ("allow_short", "max_fields")}
    kw.update(offset_key=okey, src_pos=pos, time=time, time_ns=ns)
    need, ctr0 = eng.sls_serialize_split_delim_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_delim_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_delim_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    return bytes(host[:need]), [int(x) for x in ctr]


def _check_dev(eng, val, cfg, okey, pos, time, ns, mcfg=None):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": 10}
    want, wctr, _, _ = sdc.oracle_chain(val, split_cfg, cfg, time, ns, pos, okey, multiline=mcfg is not None)
    got, ctr = device_chain(eng, val, cfg, okey, pos, time, ns, ml=_ml_handles(mcfg) if mcfg else None)
    assert got == want and sdc.fold(ctr) == wctr, (cfg, okey)


CASES = list(dc.all_cases(seed_base=5, per=1))


@pytest.mark.parametrize("cid,cfg,rng", CASES, ids=[c[0] for c in CASES])
def test_dev_chain_matrix(eng, cid, cfg, rng):
    val = sdc.random_value(rng, cfg, 80, wide_every=23)
    for i, okey in enumerate([None, OKEY, b""]):
        t, ns = sc.TIMES[i % len(sc.TIMES)]
        _check_dev(eng, val, cfg, okey, sc.POSITIONS[(3 * i + len(cid)) % len(sc.POSITIONS)], t, ns)


CORNERS = list(sdc.offset_corners())


@pytest.mark.parametrize("name,cfg,okey", CORNERS, ids=[c[0] for c in CORNERS])
def test_offset_key_corners(eng, name, cfg, okey):
    rng = random.Random(zlib.crc32(name.encode()))
    for flags in (0, 3, 5, 7):
        c = sdc.with_flags(cfg, flags)
        val = b"1,2,3,4,5,6\n1\n\n   \n\"open,1\n".replace(b",", cfg["sep"]) + sdc.random_value(rng, c, 40)
        _check_dev(eng, val, c, okey, 123456789, 1 << 29, 5)


def test_refusals(eng):
    """an offset key equal to SourceKey, or of the form __column<N>__ unless discarding, is refused by the device-fed
    and the host-buffer calls"""
    import loongcollector_b200 as lc
    for okey, tr in ((b"content", "extend"), (b"content", "discard"), (b"__column2__", "extend"),
                     (b"__column0__", "keep")):
        a = sdc.device_args(sdc.config(["a", "b", "c"], treatment=tr))
        kw = dict(a, offset_key=okey)
        dkw = {k: v for k, v in kw.items() if k not in ("allow_short", "max_fields")}
        calls = [lambda: eng.split_delim_parse_sls(b"a,1\n", 10, **kw),
                 lambda: eng.split_delim_parse_sls_lz4(b"a,1\n", 10, **kw),
                 lambda: eng.multiline_split_delim_parse_sls(b"a,1\n", None, None, None, False, **kw),
                 lambda: eng.multiline_split_delim_parse_sls_lz4(b"a,1\n", None, None, None, False, **kw),
                 lambda: eng.sls_serialize_split_delim_dev(None, 0, None, None, 0, None, None, None, None, None, 6,
                                                           **dkw)]
        for call in calls:
            with pytest.raises(lc.LcError) as ei:
                call()
            assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


@pytest.mark.parametrize("size", [0, 1, 512 * 1024])
def test_host_calls(eng, size):
    rng = random.Random(size)
    cfg = sdc.config(["a", "b", "c", "d"], renamed="raw", keep_fail=True, keep_succeed=True, copy_raw=True)
    val = sdc.random_value(rng, cfg, max(1, size // 40))[:size] if size else b""
    tail = b"\x1a\x05topic"
    a = sdc.device_args(cfg)
    for okey in (None, OKEY):
        want, wctr, _, npieces = sdc.oracle_chain(val, {"SourceKey": "content"}, cfg, 1700000000, 42, 4096, okey)
        kw = dict(a, offset_key=okey, src_pos=4096, time=1700000000, time_ns=42)
        data, nev, ctr = eng.split_delim_parse_sls(val, 10, **kw)
        assert data == want and sdc.fold(ctr) == wctr and nev == npieces
        block, raw, nev2, ctr2 = eng.split_delim_parse_sls_lz4(val, 10, **kw, tail=tail)
        assert raw == len(want) + len(tail) and nev2 == nev and list(ctr2) == list(ctr)
        assert lz4_block.decode(block) == want + tail
        # the multiline splitter without patterns: one event per line
        mwant, mwctr, _, mpieces = sdc.oracle_chain(val, {"SourceKey": "content"}, cfg, 1700000000, 42, 4096, okey,
                                                    multiline=True)
        mdata, mnev, mctr, _ml = eng.multiline_split_delim_parse_sls(val, None, None, None, False, **kw)
        assert mdata == mwant and mnev == mpieces and sdc.fold(mctr) == mwctr
        mblock, mraw, _n, _c, _m = eng.multiline_split_delim_parse_sls_lz4(val, None, None, None, False, **kw,
                                                                           tail=tail)
        assert mraw == len(mwant) + len(tail) and lz4_block.decode(mblock) == mwant + tail


def test_long_pieces_among_short_ones(eng):
    rng = random.Random(11)
    cfg = sdc.config(["a", "b", "c"], keep_fail=True, copy_raw=True)
    lines = []
    for i in range(40):
        if i % 9 == 8:
            lines.append(b",".join(bytes(rng.choice(b"abc -:") for _ in range(rng.randint(20000, 30000)))
                                   for _ in range(3)))
        else:
            lines.append(dc.random_line(rng, b",", ord('"')))
    val = b"\n".join(lines)
    _check_dev(eng, val, cfg, OKEY, 10 ** 9, 7, None)
    want, wctr, _, npieces = sdc.oracle_chain(val, {"SourceKey": "content"}, cfg, 7, None, 10 ** 9, OKEY)
    data, nev, ctr = eng.split_delim_parse_sls(val, 10, **sdc.device_args(cfg), offset_key=OKEY, src_pos=10 ** 9,
                                               time=7)
    assert data == want and nev == npieces and sdc.fold(ctr) == wctr


def test_c4_csv_lines(eng):
    from loongcollector_b200 import synth
    buf, _, _ = synth.csv_lines(20000)
    val = buf.tobytes()
    cfg = sdc.config(synth.CSV_KEYS, max_fields=11)
    _check_dev(eng, val, cfg, OKEY, 1 << 33, 1700000000, None)
    want, wctr, _, npieces = sdc.oracle_chain(val, {"SourceKey": "content"}, cfg, 1700000000, None, 1 << 33, OKEY)
    data, nev, ctr = eng.split_delim_parse_sls(val, 10, **sdc.device_args(cfg), offset_key=OKEY, src_pos=1 << 33,
                                               time=1700000000)
    assert data == want and nev == npieces and sdc.fold(ctr) == wctr


@pytest.mark.parametrize("discard", [False, True])
def test_multiline_records(eng, discard):
    """records of a dated first line and stack lines, the message a quoted field across them, among stray lines"""
    rng = random.Random(3)
    lines = []
    for i in range(400):
        if rng.random() < 0.2:
            lines.append(b"stray,%d" % i)
            continue
        lines.append(b'2024-01-0%d 10:00:0%d,%s,"msg %d' % (rng.randint(1, 9), rng.randint(0, 9),
                                                            rng.choice([b"INFO", b"ERROR"]), i))
        lines += [b"\tat frame %d" % j for j in range(rng.randint(0, 4))]
        lines[-1] += b'",tail'
    val = b"\n".join(lines)
    mcfg = dict(sc.ml_config("start", discard=discard))
    cfg = sdc.config(["when", "level", "msg", "tail"], treatment="keep", renamed="raw", keep_succeed=True)
    want, wctr, mctr, npieces = sdc.oracle_chain(val, mcfg, cfg, 1700000000, 9, 77, OKEY, multiline=True)
    h = _ml_handles(mcfg)
    got, ctr = device_chain(eng, val, cfg, OKEY, 77, 1700000000, 9, ml=h)
    assert got == want and sdc.fold(ctr) == wctr
    kw = dict(sdc.device_args(cfg), offset_key=OKEY, src_pos=77, time=1700000000, time_ns=9)
    data, nev, ctr, ml = eng.multiline_split_delim_parse_sls(val, *h, **kw)
    assert data == want and nev == npieces and sdc.fold(ctr) == wctr
    assert int(ml[0]) == mctr["matched_events"] and int(ml[2]) == mctr["unmatched_lines"]
    assert int(ml[1]) - int(ml[2]) == mctr["matched_lines"]
    block, raw, nev2, ctr2, ml2 = eng.multiline_split_delim_parse_sls_lz4(val, *h, **kw, tail=b"\x22\x01s")
    assert lz4_block.decode(block) == want + b"\x22\x01s" and list(ml2) == list(ml) and nev2 == nev


# ---- the host classes through lc_host_chain_serialize_sls
def _procs(split_type, split_cfg, cfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor(split_type, split_cfg),
            lc.HostProcessor("processor_parse_delimiter_native", dc.oracle_config(cfg)))


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


def _counters(p):  # the event counters (wall-time counters end in _ns)
    return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}


def _check_modes(split_type, split_cfg, cfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, cfg)
    b = _procs(split_type, split_cfg, cfg)
    got = capi.host_chain_serialize_sls(a[0], a[1], group, enable_ns, 0)
    want = capi.host_chain_serialize_sls(b[0], b[1], group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert _counters(a[0]) == _counters(b[0]) and _counters(a[1]) == _counters(b[1])
    c = _procs(split_type, split_cfg, cfg)
    z = capi.host_chain_serialize_sls(c[0], c[1], group, enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    assert _counters(c[0]) == _counters(b[0]) and _counters(c[1]) == _counters(b[1])
    return want


SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"[a-c].*", "UnmatchedContentTreatment": "single_line"})]


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(eng, split_type, split_cfg):
    rng = random.Random(5)
    base = sdc.config(["a", "b", "c"], renamed="raw", keep_fail=True, keep_succeed=True, copy_raw=True)
    vals = [sdc.random_value(rng, base, 40).decode("latin1") for _ in range(3)]
    cfgs = [base,
            sdc.config(["a", OKEY.decode(), "content"], treatment="keep", keep_fail=False, keep_succeed=True),
            sdc.config(["a", "_", "c"], treatment="discard", renamed=OKEY.decode(), keep_succeed=True),
            sdc.config(["x", "y"], sep=b"|#", keep_fail=True)]
    for cfg in cfgs:
        for okey in (None, OKEY.decode(), ""):
            _check_modes(split_type, split_cfg, cfg, _group(vals[:1], okey))  # the one-chunk LZ4 device path
            _check_modes(split_type, split_cfg, cfg, _group(vals, okey))      # several source events
    # fallbacks: raw content, another delimiter SourceKey, offset key = SourceKey, a __column<N>__ offset key in extend
    # mode, a non-flat group, an empty value
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), base, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(base, source="other"), _group(vals[:1]))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], "content"))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], "__column4__"))
    _check_modes(split_type, split_cfg, base, _group(vals[:1], extra={"x": "y"}))
    _check_modes(split_type, split_cfg, base, _group([""]))
    # errors: empty group, every event erased, size limit
    assert _check_modes(split_type, split_cfg, base, _group([]))[2] == "empty event group"
    erased = sdc.config(["a", "b", "c", "d", "e"], keep_fail=False, allow_short=False)
    for okey in (None, OKEY.decode()):
        assert _check_modes(split_type, split_cfg, erased, _group(["a,1\nb,2\nc\n"], okey))[2] == "empty event group"
    big = ("a,1," + "x" * 1000 + "\n") * 6000
    err = _check_modes(split_type, split_cfg, base, _group([big, big]))[2]
    assert err is not None and err.startswith("log group exceeds size limit")
