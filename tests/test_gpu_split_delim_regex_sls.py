"""GPU tier: the split -> delimiter -> regex -> SLS chain.  lc_sls_serialize_split_delim_regex_dev over the device
tables of lc_split_lines_dev / lc_multiline_split_dev, lc_delim_parse_dev, lc_delim_regex_tap_dev and
lc_regex_parse_dev, the four host calls, and the splitters' SerializeSls(group, delimiter, regex) against the oracle
chain (its splitter, ProcessorParseDelimiterNative, ProcessorParseRegexNative, then sls_serialize_logs), the emulation
and Process x 3 + Serialize, byte for byte and counter for counter."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import delim_regex_sls_cases as drc  # noqa: E402
from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402
from tests import split_delim_regex_sls_cases as sdrc  # noqa: E402
from tests import split_delim_sls_cases as sdc  # noqa: E402
from tests import split_sls_cases as sc  # noqa: E402
from tests.emul import split_delim_regex_sls  # noqa: E402

POISON, GUARD = 0xA5, 256
OKEY = sdrc.OKEY


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


def _rx(rcfg):
    import loongcollector_b200 as lc
    return None if rcfg["regex"] == drc.WHOLE_LINE else lc.Regex(rcfg["regex"])


def _cfgs(dcfg, rcfg):
    a = sdc.device_args(dcfg)
    delim = {k: v for k, v in a.items() if k not in ("allow_short", "max_fields")}
    r = sdrc.regex_args(rcfg)
    regex = dict(keys=r["rkeys"], source_key=r["rsource_key"], renamed_key=r["rrenamed_key"],
                 keep_fail=r["rkeep_fail"], keep_succeed=r["rkeep_succeed"], copy_raw=r["rcopy_raw"],
                 whole_line=r["whole_line"])
    return delim, regex, dict(allow_short=a["allow_short"], max_fields=a["max_fields"])


def device_chain(eng, val, dcfg, rcfg, okey, pos, time, ns, ml=None):
    """split, delimiter, tap, regex and serialise on the device into a poisoned buffer with guard bytes; checks the
    sizing query, the capacity refusal and the guard; returns (wire bytes, counters[8])"""
    import torch

    import loongcollector_b200 as lc
    side_at = (len(val) + 15) // 16 * 16
    d = torch.full((side_at + len(val) + 32,), POISON, dtype=torch.uint8, device="cuda")
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
    delim, regex, dk = _cfgs(dcfg, rcfg)
    MF = dk["max_fields"]
    st = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    nf = torch.empty(max(n, 1), dtype=torch.int32, device="cuda")
    fo, fl, fd = (torch.empty(max(n, 1) * MF, dtype=torch.int32, device="cuda") for _ in range(3))
    d_vo, d_vl = (torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda") for _ in range(2))
    side = 0
    if n:
        eng.delim_parse_dev(d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, delim["sep"],
                            delim["quote"], len(delim["keys"]), delim["treatment"] == "extend", dk["allow_short"], MF,
                            st.data_ptr(), nf.data_ptr(), fo.data_ptr(), fl.data_ptr(), fd.data_ptr())
    tabs = (d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), nf.data_ptr(), fo.data_ptr(), fl.data_ptr(),
            fd.data_ptr(), MF)
    if n:
        side = eng.delim_regex_tap_dev(d.data_ptr(), len(val), side_at + len(val), *tabs, delim, regex,
                                       d_vo.data_ptr(), d_vl.data_ptr())
        assert 0 <= side <= len(val)
    whole = regex["whole_line"]
    G = 0 if whole else _rx(rcfg).ngroups
    d_rs = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    d_co, d_cl = (torch.empty(max(n * G, 1), dtype=torch.int32, device="cuda") for _ in range(2))
    if n and not whole:
        eng.regex_parse_dev(_rx(rcfg), d.data_ptr(), side_at + side, d_vo.data_ptr(), d_vl.data_ptr(), n,
                            len(regex["keys"]), d_rs.data_ptr(), d_co.data_ptr(), d_cl.data_ptr())
    args = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), nf.data_ptr(),
            fo.data_ptr(), fl.data_ptr(), fd.data_ptr(), MF, delim, regex, d_vo.data_ptr(), d_vl.data_ptr(),
            None if whole else d_rs.data_ptr(), None if whole else d_co.data_ptr(),
            None if whole else d_cl.data_ptr(), G)
    kw = dict(offset_key=okey, src_pos=pos, time=time, time_ns=ns)
    need, ctr0 = eng.sls_serialize_split_delim_regex_dev(*args, **kw)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_delim_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_split_delim_regex_dev(*args, **kw, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    assert bool((d[side_at + side:] == POISON).all()), "a side copy past its slots"
    return bytes(host[:need]), [int(x) for x in ctr]


def _emul(val, dcfg, rcfg, okey, pos, time, ns, ml=None):
    off, ln = sdrc.pieces(val, 10, ml)
    tabs = sdrc.tables(val, off, ln, dcfg)
    got, ctr, _v, _s = split_delim_regex_sls.serialize(val, off, ln, tabs, dcfg, rcfg, okey, pos, time, ns)
    return got, [int(x) for x in ctr]


def _check_dev(eng, val, dcfg, rcfg, okey, pos, time, ns, mcfg=None):
    split_cfg = mcfg or {"SourceKey": dcfg["source"], "SplitChar": 10}
    want, wctr, _, _ = sdrc.oracle_chain(val, split_cfg, dcfg, rcfg, time, ns, pos, okey, multiline=mcfg is not None)
    got, ctr = device_chain(eng, val, dcfg, rcfg, okey, pos, time, ns, ml=_ml_handles(mcfg) if mcfg else None)
    assert got == want and sdrc.fold(ctr) == wctr, (dcfg, rcfg, okey)
    if mcfg is None:
        assert (got, ctr) == _emul(val, dcfg, rcfg, okey, pos, time, ns)


CASES = list(dc.all_cases(seed_base=17, per=1))


@pytest.mark.parametrize("cid,dcfg,rng", CASES, ids=[c[0] for c in CASES])
def test_dev_chain_matrix(eng, cid, dcfg, rng):
    val = sdc.random_value(rng, dcfg, 80, wide_every=23)
    for i, okey in enumerate([None, OKEY, b""]):
        t, ns = sc.TIMES[i % len(sc.TIMES)]
        for _ in range(4):
            rcfg = drc.random_regex(rng, dcfg)
            if not sdrc.refused(dcfg, rcfg, okey):
                _check_dev(eng, val, dcfg, rcfg, okey, sc.POSITIONS[(3 * i + len(cid)) % len(sc.POSITIONS)], t, ns)


CORNERS = list(sdc.offset_corners())


@pytest.mark.parametrize("name,cfg,okey", CORNERS, ids=[c[0] for c in CORNERS])
def test_offset_key_corners(eng, name, cfg, okey):
    rng = random.Random(zlib.crc32(name.encode()))
    for flags in (0, 3, 5, 7):
        dcfg = sdc.with_flags(cfg, flags)
        val = b'1,2,3,4,5,6\n1\n\n   \n"open,1\n"x""y",2\n'.replace(b",", cfg["sep"]) + sdc.random_value(rng, dcfg, 40)
        ks = [k for k in drc.delim_keys(dcfg) if k.encode() != okey]
        for rkeep_fail in (False, True):
            rcfg = rc.config(["r1", "r2"], ks[0], None, rkeep_fail, False, False, regex=drc.PAT_QUOTE)
            if not sdrc.refused(dcfg, rcfg, okey):
                _check_dev(eng, val, dcfg, rcfg, okey, 123456789, 1 << 29, 5)


def test_regex_failure_leaving_only_the_offset_content(eng):
    val = b"abc\n/p?k=1\n\nx y\n/q?k=zz\n  \n"
    for okey in (None, OKEY):
        for rkeep_fail in (False, True):
            _check_dev(eng, val, sdc.config(["url"]), sdrc.c4_regex(keep_fail=rkeep_fail), okey, 7, 1 << 30, 3)


def test_refusals(eng):
    """the chain's own refusals reach the device-fed and the host-buffer calls"""
    import loongcollector_b200 as lc
    for dcfg, rcfg, okey in ((sdc.config(["a", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD), b"b"),
                             (sdc.config(["a", "b"]), rc.config(["off"], "b", regex=drc.PAT_WORD), b"off"),
                             (sdc.config(["a", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD), b"content")):
        delim, regex, dk = _cfgs(dcfg, rcfg)
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_split_delim_regex_dev(0, 0, 0, 0, 0, 0, 0, 0, 0, 0, dk["max_fields"], delim, regex, 0,
                                                    0, 0, 0, 0, 2, offset_key=okey)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
        with pytest.raises(lc.LcError) as ei:
            eng.split_delim_regex_parse_sls(_rx(rcfg), b"x,1\n", 10, delim, regex, **dk, offset_key=okey)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


def test_four_gib_refusal_from_the_arguments(eng):
    """align16(len) + len reaching 4 GiB is refused before anything is read or allocated: the buffer passed is tiny"""
    import loongcollector_b200 as lc
    L = lc.lib()
    delim, regex, dk = _cfgs(sdc.config(["a", "url"]), sdrc.c4_regex())
    _keep, cfg = lc.Engine._chain_cfg(delim, regex)
    small = np.zeros(64, np.uint8)
    rx = _rx(sdrc.c4_regex())
    n, nev, raw = C.c_uint64(7), C.c_uint64(7), C.c_uint64(7)
    ctr = np.full(8, 9, np.uint64)
    tail = [OKEY, len(OKEY), 0, 1, 0xFFFFFFFF]
    for ln in (1 << 31, (1 << 32) - 64):
        rc_ = L.lc_split_delim_regex_parse_sls(eng._h, rx._h, small.ctypes.data_as(C.c_void_p), ln, 10, 1, 4, *cfg,
                                               *tail, None, 0, C.byref(n), C.byref(nev), ctr.ctypes.data_as(C.c_void_p))
        assert rc_ == lc.capi.LC_ERR_TOO_LARGE and n.value == 0 and nev.value == 0 and not ctr.any()
        assert "4 GiB" in L.lc_last_error().decode()
        rc_ = L.lc_split_delim_regex_parse_sls_lz4(eng._h, rx._h, small.ctypes.data_as(C.c_void_p), ln, 10, 1, 4,
                                                   *cfg, *tail, None, 0, None, 0, C.byref(n), C.byref(raw),
                                                   C.byref(nev), ctr.ctypes.data_as(C.c_void_p))
        assert rc_ == lc.capi.LC_ERR_TOO_LARGE and raw.value == 0
    # still usable afterwards
    data, nev2, _ctr = eng.split_delim_regex_parse_sls(rx, b"1,/a?k=b\n", 10, delim, regex, **dk)
    assert nev2 == 1 and data


@pytest.mark.parametrize("size", [0, 1, 512 * 1024])
def test_host_calls(eng, size):
    from loongcollector_b200 import synth
    buf, _, _ = synth.csv_lines(max(1, size // 100), seed=size)
    val = buf.tobytes()[:size]
    dcfg = sdc.config(synth.CSV_KEYS, max_fields=11)
    rcfg = sdrc.c4_regex(keep_fail=True, copy_raw=True, renamed="u")
    delim, regex, dk = _cfgs(dcfg, rcfg)
    rx = _rx(rcfg)
    tail = b"\x1a\x05topic"
    for okey in (None, OKEY):
        want, wctr, _, npieces = sdrc.oracle_chain(val, {"SourceKey": "content"}, dcfg, rcfg, 1700000000, 42, 4096,
                                                   okey)
        kw = dict(dk, offset_key=okey, src_pos=4096, time=1700000000, time_ns=42)
        data, nev, ctr = eng.split_delim_regex_parse_sls(rx, val, 10, delim, regex, **kw)
        assert data == want and sdrc.fold(ctr) == wctr and nev == npieces
        if val:
            assert (data, [int(x) for x in ctr]) == _emul(val, dcfg, rcfg, okey, 4096, 1700000000, 42)
        block, raw, nev2, ctr2 = eng.split_delim_regex_parse_sls_lz4(rx, val, 10, delim, regex, **kw, tail=tail)
        assert raw == len(want) + len(tail) and nev2 == nev and list(ctr2) == list(ctr)
        assert lz4_block.decode(block) == want + tail
        # the multiline splitter without patterns: one event per line
        mwant, mwctr, _, mpieces = sdrc.oracle_chain(val, {"SourceKey": "content"}, dcfg, rcfg, 1700000000, 42, 4096,
                                                     okey, multiline=True)
        mdata, mnev, mctr, _ml = eng.multiline_split_delim_regex_parse_sls(rx, val, None, None, None, False, delim,
                                                                           regex, **kw)
        assert mdata == mwant and mnev == mpieces and sdrc.fold(mctr) == mwctr
        mblock, mraw, _n, _c, _m = eng.multiline_split_delim_regex_parse_sls_lz4(rx, val, None, None, None, False,
                                                                                 delim, regex, **kw, tail=tail)
        assert mraw == len(mwant) + len(tail) and lz4_block.decode(mblock) == mwant + tail


def test_quoted_columns_and_whole_line(eng):
    """the regex on a quoted column with doubled quotes (side copies) and in whole-line mode, through the host call"""
    rng = random.Random(4)
    dcfg = sdc.config(["q", "b", "c"], keep_succeed=True, renamed="raw")
    lines = [b'"a""b""c",x,y', b'"""",1', b'"p" q,1', b"plain,2"] + [dc.random_line(rng, b",", ord('"'))
                                                                    for _ in range(300)]
    val = b"\n".join(lines)
    for rcfg in (rc.config(["r1", "r2"], "q", regex=drc.PAT_QUOTE), rc.config(["w"], "q", regex=drc.WHOLE_LINE)):
        _check_dev(eng, val, dcfg, rcfg, OKEY, 5, 6, None)
        delim, regex, dk = _cfgs(dcfg, rcfg)
        want, wctr, _, _ = sdrc.oracle_chain(val, {"SourceKey": "content"}, dcfg, rcfg, 6, None, 5, OKEY)
        data, _nev, ctr = eng.split_delim_regex_parse_sls(_rx(rcfg), val, 10, delim, regex, **dk, offset_key=OKEY,
                                                          src_pos=5, time=6)
        assert data == want and sdrc.fold(ctr) == wctr


@pytest.mark.parametrize("discard", [False, True])
def test_multiline_records(eng, discard):
    """records of a dated first line and stack lines, the message a quoted field across them, among stray lines"""
    rng = random.Random(3)
    lines = []
    for i in range(400):
        if rng.random() < 0.2:
            lines.append(b"stray,%d" % i)
            continue
        lines.append(b'2024-01-0%d 10:00:0%d,%s,"msg ""%d""' % (rng.randint(1, 9), rng.randint(0, 9),
                                                                rng.choice([b"INFO", b"ERROR"]), i))
        lines += [b"\tat frame %d" % j for j in range(rng.randint(0, 4))]
        lines[-1] += b'",tail'
    val = b"\n".join(lines)
    mcfg = dict(sc.ml_config("start", discard=discard))
    dcfg = sdc.config(["when", "level", "msg", "tail"], treatment="keep", renamed="raw", keep_succeed=True)
    rcfg = rc.config(["m1", "m2"], "msg", None, False, False, False, regex=drc.PAT_QUOTE)
    want, wctr, mctr, npieces = sdrc.oracle_chain(val, mcfg, dcfg, rcfg, 1700000000, 9, 77, OKEY, multiline=True)
    h = _ml_handles(mcfg)
    got, ctr = device_chain(eng, val, dcfg, rcfg, OKEY, 77, 1700000000, 9, ml=h)
    assert got == want and sdrc.fold(ctr) == wctr
    delim, regex, dk = _cfgs(dcfg, rcfg)
    kw = dict(dk, offset_key=OKEY, src_pos=77, time=1700000000, time_ns=9)
    rx = _rx(rcfg)
    data, nev, ctr, ml = eng.multiline_split_delim_regex_parse_sls(rx, val, *h, delim, regex, **kw)
    assert data == want and nev == npieces and sdrc.fold(ctr) == wctr
    assert int(ml[0]) == mctr["matched_events"] and int(ml[2]) == mctr["unmatched_lines"]
    assert int(ml[1]) - int(ml[2]) == mctr["matched_lines"]
    block, raw, nev2, ctr2, ml2 = eng.multiline_split_delim_regex_parse_sls_lz4(rx, val, *h, delim, regex, **kw,
                                                                                tail=b"\x22\x01s")
    assert lz4_block.decode(block) == want + b"\x22\x01s" and list(ml2) == list(ml) and nev2 == nev


def test_c4_two_mi_lines_in_512kb_chunks(eng):
    """2 Mi C4 lines, cut into 512 KB chunks at line ends as the reader hands them over, one host call per chunk:
    each chunk against the emulation fed with the oracle's tables, and every 64th against the oracle's processors"""
    from loongcollector_b200 import synth
    buf, _, _ = synth.csv_lines(2 * 1024 * 1024, seed=9)
    val = buf.tobytes()
    dcfg = sdc.config(synth.CSV_KEYS, max_fields=11)
    rcfg = sdrc.c4_regex()
    delim, regex, dk = _cfgs(dcfg, rcfg)
    rx = _rx(rcfg)
    pos, k, lines, total = 0, 0, 0, np.zeros(8, np.uint64)
    while pos < len(val):
        end = val.rfind(b"\n", pos, pos + 512 * 1024) + 1 if pos + 512 * 1024 < len(val) else len(val)
        chunk = val[pos:end]
        data, nev, ctr = eng.split_delim_regex_parse_sls(rx, chunk, 10, delim, regex, **dk, offset_key=OKEY,
                                                         src_pos=pos, time=1700000000 + k)
        assert (data, [int(x) for x in ctr]) == _emul(chunk, dcfg, rcfg, OKEY, pos, 1700000000 + k, None), k
        if k % 64 == 0:
            want, wctr, _, npieces = sdrc.oracle_chain(chunk, {"SourceKey": "content"}, dcfg, rcfg, 1700000000 + k,
                                                       None, pos, OKEY)
            assert data == want and sdrc.fold(ctr) == wctr and nev == npieces, k
        lines += nev
        total += ctr
        pos, k = end, k + 1
    assert lines == 2 * 1024 * 1024 and int(total[4]) > 0


# ---- the host classes through lc_host_chain3_serialize_sls
def _procs(split_type, split_cfg, dcfg, rcfg):
    import loongcollector_b200 as lc
    return (lc.HostProcessor(split_type, split_cfg),
            lc.HostProcessor("processor_parse_delimiter_native", dc.oracle_config(dcfg)),
            lc.HostProcessor("processor_parse_regex_native", rc.oracle_config(rcfg)))


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


def _check_modes(split_type, split_cfg, dcfg, rcfg, group, enable_ns=True):
    from loongcollector_b200 import capi
    a = _procs(split_type, split_cfg, dcfg, rcfg)
    b = _procs(split_type, split_cfg, dcfg, rcfg)
    got = capi.host_chain3_serialize_sls(*a, group, enable_ns, 0)
    want = capi.host_chain3_serialize_sls(*b, group, enable_ns, 1)
    assert got[0] == want[0] and got[2] == want[2]
    assert [_counters(p) for p in a] == [_counters(p) for p in b]
    c = _procs(split_type, split_cfg, dcfg, rcfg)
    z = capi.host_chain3_serialize_sls(*c, group, enable_ns, 2)
    if want[0] is None:
        assert z[0] is None and z[2] == want[2]
    else:
        assert z[1] == len(want[0]) and lz4_block.decode(z[0]) == want[0]
    assert [_counters(p) for p in c] == [_counters(p) for p in b]
    return want


SPLITTERS = [("processor_split_string_native", {"SourceKey": "content"}),
             ("processor_split_multiline_log_string_native",
              {"SourceKey": "content", "StartPattern": r"[0-9a-c].*", "UnmatchedContentTreatment": "single_line"})]


@pytest.mark.parametrize("split_type,split_cfg", SPLITTERS, ids=["split", "multiline"])
def test_host_classes(eng, split_type, split_cfg):
    from loongcollector_b200 import synth
    rng = random.Random(5)
    buf, _, _ = synth.csv_lines(300, seed=5)
    csv = buf.tobytes().decode("latin1")
    base = sdc.config(synth.CSV_KEYS, max_fields=11, keep_fail=True)
    c4 = sdrc.c4_regex()
    vals = [csv, sdc.random_value(rng, base, 40).decode("latin1"), csv[:5000] + "\n\n/x?k=1\n"]
    rcfgs = [c4, sdrc.c4_regex(keep_fail=True, keep_succeed=True, copy_raw=True, renamed="u"),
             rc.config(["w"], "url", regex=drc.WHOLE_LINE)]
    for rcfg in rcfgs:
        for okey in (None, OKEY.decode(), ""):
            _check_modes(split_type, split_cfg, base, rcfg, _group(vals[:1], okey))  # the one-chunk LZ4 device path
            _check_modes(split_type, split_cfg, base, rcfg, _group(vals, okey))      # several source events
    # fallbacks: raw content, another delimiter SourceKey, a regex SourceKey that is no delimiter key, refused
    # configurations (offset key = regex SourceKey, = a regex key), a non-flat group, an empty value
    _check_modes(split_type, dict(split_cfg, EnableRawContent=True), base, c4, _group(vals[:1]))
    _check_modes(split_type, split_cfg, dict(base, source="other"), c4, _group(vals[:1]))
    _check_modes(split_type, split_cfg, base, rc.config(["path", "k"], "zz", regex=synth.CSV_URL_PATTERN),
                 _group(vals[:1]))
    _check_modes(split_type, split_cfg, base, c4, _group(vals[:1], "url"))
    _check_modes(split_type, split_cfg, base, c4, _group(vals[:1], "path"))
    _check_modes(split_type, split_cfg, base, c4, _group(vals[:1], extra={"x": "y"}))
    _check_modes(split_type, split_cfg, base, c4, _group([""]))
    # errors: empty group, every event erased, size limit
    assert _check_modes(split_type, split_cfg, base, c4, _group([]))[2] == "empty event group"
    only_url = sdc.config(["url"], keep_fail=False)
    for okey in (None, OKEY.decode()):
        assert _check_modes(split_type, split_cfg, only_url, c4, _group(["abc\nxyz\n"], okey))[2] is not None
    big = ("1,2,3,/" + "x" * 1000 + "?k=1\n") * 6000
    err = _check_modes(split_type, split_cfg, base, c4, _group([big, big]))[2]
    assert err is not None and err.startswith("log group exceeds size limit")
