"""GPU tier: the delimiter -> regex -> SLS chain.  lc_delim_regex_tap_dev + lc_regex_parse_dev +
lc_sls_serialize_delim_regex_dev, lc_delim_regex_parse_sls[_lz4] and ProcessorParseDelimiterNative::SerializeSls(group,
regex) against the oracle (ProcessorParseDelimiterNative + ProcessorParseRegexNative over flat events +
sls_serialize_logs / sls_serialize_group), byte for byte, with both processors' counters."""
import json
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)
from tests import delim_regex_sls_cases as drc  # noqa: E402
from tests import delim_sls_cases as dc  # noqa: E402
from tests import lz4_block  # noqa: E402
from tests import regex_sls_cases as rc  # noqa: E402

POISON, GUARD = 0xA5, 256


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _quote(dcfg):
    return dcfg["quote"] if len(dcfg["sep"]) == 1 else ord('"')


def _i32(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).cuda()


def _cfgs(dcfg, rcfg):
    delim = dict(sep=dcfg["sep"], quote=_quote(dcfg), treatment=dcfg["treatment"],
                 keys=[k.encode() for k in dcfg["keys"]], source_key=dcfg["source"].encode(),
                 renamed_key=dc.renamed_key(dcfg), keep_fail=dcfg["keep_fail"], keep_succeed=dcfg["keep_succeed"],
                 copy_raw=dcfg["copy_raw"])
    regex = dict(keys=[k.encode() for k in rcfg["keys"]], source_key=rcfg["source"].encode(),
                 renamed_key=rc.renamed_key(rcfg), keep_fail=rcfg["keep_fail"], keep_succeed=rcfg["keep_succeed"],
                 copy_raw=rcfg["copy_raw"], whole_line=rcfg["regex"] == drc.WHOLE_LINE)
    return delim, regex


def _rx(rcfg):
    import loongcollector_b200 as lc
    return None if rcfg["regex"] == drc.WHOLE_LINE else lc.Regex(rcfg["regex"])


def device_serialize(eng, buf, off, ln, dcfg, rcfg, times, nss):
    """delim_parse_dev -> delim_regex_tap_dev -> regex_parse_dev -> sls_serialize_delim_regex_dev into a poisoned
    buffer followed by guard bytes; checks the guard, the tap's and the serialiser's sizing queries and capacity errors.
    Returns (wire bytes, counters[8], delimiter tables, value table, line buffer with its side copies)."""
    import torch

    import loongcollector_b200 as lc
    n, mf = off.size, dcfg["max_fields"]
    delim, regex = _cfgs(dcfg, rcfg)
    side_at = (buf.size + 15) // 16 * 16
    cap = side_at + int(ln.astype(np.uint64).sum()) + 16
    d_buf = torch.full((cap + 16,), POISON, dtype=torch.uint8, device="cuda")
    d_buf[:buf.size] = torch.from_numpy(np.array(buf)).cuda()
    d_off, d_len = _i32(off), _i32(ln)
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_nf = torch.empty(n, dtype=torch.int32, device="cuda")
    d_fo, d_fl, d_fd = (torch.empty(n * mf, dtype=torch.int32, device="cuda") for _ in range(3))
    d_vo, d_vl = (torch.full((n,), -1, dtype=torch.int32, device="cuda") for _ in range(2))
    eng.delim_parse_dev(d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, dcfg["sep"], _quote(dcfg),
                        len(dcfg["keys"]), dcfg["treatment"] == "extend", dcfg["allow_short"], mf, d_st.data_ptr(),
                        d_nf.data_ptr(), d_fo.data_ptr(), d_fl.data_ptr(), d_fd.data_ptr())
    tabs = (d_off.data_ptr(), d_len.data_ptr(), n, d_st.data_ptr(), d_nf.data_ptr(), d_fo.data_ptr(), d_fl.data_ptr(),
            d_fd.data_ptr(), mf)
    # the tap's sizing query: no room at all behind base_len
    try:
        side = eng.delim_regex_tap_dev(d_buf.data_ptr(), buf.size, buf.size, *tabs, delim, regex, d_vo.data_ptr(),
                                       d_vl.data_ptr())
    except lc.LcError as ex:
        assert ex.code == lc.capi.LC_ERR_CAPACITY
        side = ex.need
        assert side > 0
        assert bool((d_vo == -1).all()) and bool((d_buf[buf.size:] == POISON).all()), "a refused tap wrote"
    got_side = eng.delim_regex_tap_dev(d_buf.data_ptr(), buf.size, side_at + side, *tabs, delim, regex,
                                       d_vo.data_ptr(), d_vl.data_ptr())
    assert got_side == side
    arena = side_at + side
    whole = regex["whole_line"]
    G = 0 if whole else _rx(rcfg).ngroups
    d_rs = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    d_co, d_cl = (torch.empty(max(n * G, 1), dtype=torch.int32, device="cuda") for _ in range(2))
    if not whole:
        eng.regex_parse_dev(_rx(rcfg), d_buf.data_ptr(), arena, d_vo.data_ptr(), d_vl.data_ptr(), n, len(rcfg["keys"]),
                            d_rs.data_ptr(), d_co.data_ptr(), d_cl.data_ptr())
    d_t = _i32(times)
    d_ns = _i32(nss) if nss is not None else None
    args = (d_buf.data_ptr(), arena, *tabs, delim, regex, d_vo.data_ptr(), d_vl.data_ptr(),
            None if whole else d_rs.data_ptr(), None if whole else d_co.data_ptr(), None if whole else d_cl.data_ptr(),
            G, d_t.data_ptr(), d_ns.data_ptr() if d_ns is not None else None)
    need, ctr0 = eng.sls_serialize_delim_regex_dev(*args)
    d_out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    if need:
        with pytest.raises(lc.LcError) as ei:
            eng.sls_serialize_delim_regex_dev(*args, d_out=d_out.data_ptr(), out_cap=need - 1)
        assert ei.value.code == lc.capi.LC_ERR_CAPACITY
        assert bool((d_out == POISON).all()), "a refused call wrote"
    got, ctr = eng.sls_serialize_delim_regex_dev(*args, d_out=d_out.data_ptr(), out_cap=need)
    assert got == need and list(ctr) == list(ctr0)
    host = d_out.cpu().numpy()
    assert (host[need:] == POISON).all(), "write past the records"
    u32 = lambda t: t.cpu().numpy().view(np.uint32)  # noqa: E731
    tables = (d_st.cpu().numpy(), u32(d_nf), u32(d_fo).reshape(n, mf), u32(d_fl).reshape(n, mf),
              u32(d_fd).reshape(n, mf))
    return bytes(host[:need]), ctr, tables, (u32(d_vo), u32(d_vl)), d_buf[:arena].cpu().numpy()


def _host_calls(eng, buf, off, ln, dcfg, rcfg, times, nss):
    """lc_delim_regex_parse_sls and the LZ4 sibling: (bytes, counters); the block must decode to bytes ‖ tail"""
    delim, regex = _cfgs(dcfg, rcfg)
    kw = dict(allow_short=dcfg["allow_short"], max_fields=dcfg["max_fields"], ev_time_ns=nss)
    data, ctr = eng.delim_regex_parse_sls(_rx(rcfg), buf, off, ln, times, delim, regex, **kw)
    tail = b"\x1a\x05topic" + bytes(range(40))
    blk, raw, ctr2 = eng.delim_regex_parse_sls_lz4(_rx(rcfg), buf, off, ln, times, delim, regex, tail=tail, **kw)
    assert raw == len(data) + len(tail) and lz4_block.decode(blk) == data + tail
    assert list(ctr2) == list(ctr)
    return data, ctr


MATRIX = list(dc.all_cases(seed_base=5, per=2))


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_matrix_against_oracle(eng, case):
    _, dcfg, rng = case
    n = 0
    for _ in range(40):
        rcfg = drc.random_regex(rng, dcfg)
        if drc.refused(dcfg, rcfg):
            continue
        lines = [dc.random_line(rng, dcfg["sep"], dcfg["quote"], wide=rng.random() < 0.05) for _ in range(150)]
        times, nss = dc.times_for(len(lines), rng.randint(0, 1 << 30))
        want, wctr = drc.oracle_wire(lines, dcfg, rcfg, times, nss)
        buf, off, ln = dc.arena(lines)
        got, ctr, _, _, _ = device_serialize(eng, buf, off, ln, dcfg, rcfg, times, nss)
        assert got == want and drc.fold(ctr) == wctr, (dcfg, rcfg)
        data, hctr = _host_calls(eng, buf, off, ln, dcfg, rcfg, times, nss)
        assert data == want and list(hctr) == list(ctr)
        n += 1
        if n == 3:
            break
    assert n > 0


def test_refused_chains(eng):
    import loongcollector_b200 as lc
    dcfg = dict(sep=b",", quote=ord('"'), treatment="extend", keys=["a", "b"], source="content", renamed=None,
                keep_fail=True, keep_succeed=False, copy_raw=False, allow_short=True, max_fields=4)
    buf, off, ln = dc.arena([b"1,2"])
    for rcfg in (rc.config(["r"], "zz", regex=drc.PAT_QUOTE), rc.config(["a"], "b", regex=drc.PAT_QUOTE)):
        delim, regex = _cfgs(dcfg, rcfg)
        with pytest.raises(lc.LcError) as ei:
            eng.delim_regex_parse_sls(_rx(rcfg), buf, off, ln, [1], delim, regex)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


def _c4_cfgs():
    from loongcollector_b200 import synth
    dcfg = dict(sep=b",", quote=ord('"'), treatment="extend", keys=list(synth.CSV_KEYS), source="content",
                renamed=None, keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True, max_fields=11)
    rcfg = rc.config(["path", "k"], "url", regex=synth.CSV_URL_PATTERN)
    return dcfg, rcfg


def test_c4_batch_over_several_chunks(eng):
    """>= 1 Mi C4 lines (several upload chunks): rows whose column 3 has doubled quotes exist, and their captures index
    the collapsed bytes; the host call equals the device path, the counters the oracle's on a sample"""
    from loongcollector_b200 import synth
    buf, off, ln = synth.csv_lines(1 << 20, seed=29)
    dcfg, rcfg = _c4_cfgs()
    times, nss = dc.times_for(off.size, 12)
    got, ctr, tables, (vo, vl), arena = device_serialize(eng, buf, off, ln, dcfg, rcfg, times, nss)
    st, nf, fo, fl, fd = tables
    dq_rows = np.nonzero((st == 0) & (fd[:, 3] > 0))[0]
    assert dq_rows.size > 0
    for i in dq_rows[:200].tolist():
        raw = bytes(buf[fo[i, 3]:fo[i, 3] + fl[i, 3]])
        val = bytes(arena[vo[i]:vo[i] + vl[i]])
        assert vo[i] >= buf.size and val == raw.replace(b'""', b'"') and len(val) == fl[i, 3] - fd[i, 3]
    data, hctr = eng.delim_regex_parse_sls(_rx(rcfg), buf, off, ln, times, *_cfgs(dcfg, rcfg), max_fields=11,
                                           ev_time_ns=nss)
    assert data == got and list(hctr) == list(ctr)
    assert int(ctr[0]) + int(ctr[1]) + int(ctr[3]) == off.size
    # the doubled-quote rows and a slice of the rest against the oracle chain
    pick = sorted(set(dq_rows[:300].tolist()) | set(range(0, off.size, 4099)))
    lines = [bytes(buf[off[i]:off[i] + ln[i]]) for i in pick]
    want, wctr = drc.oracle_wire(lines, dcfg, rcfg, times[pick], nss[pick])
    sb, so, sl = dc.arena(lines)
    sub, sctr, _, _, _ = device_serialize(eng, sb, so, sl, dcfg, rcfg, times[pick], nss[pick])
    assert sub == want and drc.fold(sctr) == wctr


def test_every_length_and_alignment(eng):
    """the tapped column of every length 0..300 at every 16-byte alignment, with "" straddling chunk boundaries"""
    rng = random.Random(41)
    dcfg = dict(sep=b",", quote=ord('"'), treatment="extend", keys=["a", "b", "c"], source="content", renamed=None,
                keep_fail=True, keep_succeed=True, copy_raw=False, allow_short=True, max_fields=5)
    rcfg = rc.config(["r1", "r2"], "b", "raw", True, True, False, regex=drc.PAT_QUOTE)
    lines = []
    for L in range(301):
        for a in range(16):
            body = bytearray(rng.choice(b"abcxyz/?=") for _ in range(L))
            quoted = L >= 2 and (L + a) % 3 != 0
            if quoted:  # a "" pair at a position that moves across the 16-byte chunks
                p = (a * 7 + L) % (L - 1)
                body[p:p + 2] = b'""'
                col = b'"' + bytes(body) + b'"'
            else:
                col = bytes(body).replace(b'"', b"x")
            lines.append(b"p" * a + b"," + col + b",z")
    times, nss = dc.times_for(len(lines), 6)
    want, wctr = drc.oracle_wire(lines, dcfg, rcfg, times, nss)
    buf, off, ln = dc.arena(lines)
    got, ctr, _, _, _ = device_serialize(eng, buf, off, ln, dcfg, rcfg, times, nss)
    assert got == want and drc.fold(ctr) == wctr
    assert _host_calls(eng, buf, off, ln, dcfg, rcfg, times, nss)[0] == want


def test_long_values_and_wide_rows(eng):
    """tapped values >= 64 KB (the regex stage's long-event kernel), with and without doubled quotes, and rows wider
    than max_fields"""
    rng = random.Random(43)
    dcfg = dict(sep=b",", quote=ord('"'), treatment="keep", keys=["a", "b"], source="content", renamed=None,
                keep_fail=True, keep_succeed=False, copy_raw=False, allow_short=True, max_fields=3)
    rcfg = rc.config(["r1", "r2"], "b", None, True, False, False, regex=drc.PAT_QUOTE)
    big = b"q" * 70000
    lines = [b"x," + big + b'"' + big + b",z", b'x,"' + big + b'""' + big + b'",z',
             b'x,"' + b'""' * 40000 + b'",z', b"x," + b"y" * 100000]
    lines += [dc.random_line(rng, b",", ord('"'), wide=True) for _ in range(60)]
    lines += [b'1,"a""b",' + b",".join(b"c%d" % j for j in range(50))]
    times, nss = dc.times_for(len(lines), 7)
    want, wctr = drc.oracle_wire(lines, dcfg, rcfg, times, nss)
    buf, off, ln = dc.arena(lines)
    got, ctr, _, _, _ = device_serialize(eng, buf, off, ln, dcfg, rcfg, times, nss)
    assert got == want and drc.fold(ctr) == wctr
    assert _host_calls(eng, buf, off, ln, dcfg, rcfg, times, nss)[0] == want


# ---- host class: SerializeSls(group, regex) == Process + Process + SLSEventGroupSerializer::Serialize
def _check_host(dconf, rconf, group):
    import loongcollector_b200 as lc
    fast = (lc.HostProcessor("processor_parse_delimiter_native", dconf),
            lc.HostProcessor("processor_parse_regex_native", rconf))
    ref = (lc.HostProcessor("processor_parse_delimiter_native", dconf),
           lc.HostProcessor("processor_parse_regex_native", rconf))
    zfast = (lc.HostProcessor("processor_parse_delimiter_native", dconf),
             lc.HostProcessor("processor_parse_regex_native", rconf))
    for ns in (False, True):
        got = lc.capi.host_chain_serialize_sls(*fast, group, ns, 0)
        want = lc.capi.host_chain_serialize_sls(*ref, group, ns, 1)
        assert got == want, (dconf, rconf, ns, got[2], want[2])
        blk, raw, zerr = lc.capi.host_chain_serialize_sls(*zfast, group, ns, 2)
        assert zerr == want[2]
        if blk is not None:
            assert raw == len(want[0]) and lz4_block.decode(blk) == want[0]
        g = orc.Group.from_json(json.loads(json.dumps(group)))
        orc.ProcessorParseDelimiterNative(dconf).process(g)
        orc.ProcessorParseRegexNative(rconf).process(g)
        o, oerr = orc.sls_serialize_group(g, ns)
        assert want[0] == o and (want[2] is None) == (oerr is None), (dconf, rconf, ns, want[2], oerr)
    def events(p):  # the event counters (the regex class's phase timers are wall time)
        return {k: v for k, v in p.counters().items() if not k.endswith("_ns")}
    for a, b, c in zip(fast, ref, zfast):
        assert events(a) == events(b) == events(c)


def test_host_class_on_random_groups():
    rng = random.Random(47)
    done = 0
    for k in range(80):
        sname, sep, quote = dc.SEPARATORS[k % 4]
        dcfg = dc.random_config(rng, dc.TREATMENTS[k % 3], sep, quote)
        rcfg = drc.random_regex(rng, dcfg)
        evs = []
        for _ in range(rng.choice([0, 1, 5, 40])):
            ev = {"type": 1, "timestamp": rng.choice([5, 1700000000]),
                  "contents": {dcfg["source"]: dc.random_line(rng, sep, quote, rng.random() < 0.05).decode("latin1")}}
            if rng.random() < 0.5:
                ev["timestampNanosecond"] = rng.randint(0, 999999999)
            if k % 5 == 4 and rng.random() < 0.3:  # not flat: the three calls
                ev["contents"]["other"] = "x"
            evs.append(ev)
        root = {"events": evs, "tags": {"__topic__": "t", "host.name": "h" * rng.choice([1, 100])}}
        if k % 7 == 6:
            root["metadata"] = {"log.file.offset": "__offset__"}
        _check_host(dc.oracle_config(dcfg), rc.oracle_config(rcfg), root)
        done += not drc.refused(dcfg, rcfg)
    assert done > 20


def test_host_class_c4_group():
    from loongcollector_b200 import synth
    dcfg, rcfg = _c4_cfgs()
    lines = synth.csv_pool(3000, seed=3)
    evs = [{"type": 1, "timestamp": 1700000000 + i, "contents": {"content": x.rstrip(b"\n").decode()}}
           for i, x in enumerate(lines)]
    _check_host(dc.oracle_config(dcfg), rc.oracle_config(rcfg), {"events": evs, "tags": {"__topic__": "c4"}})
