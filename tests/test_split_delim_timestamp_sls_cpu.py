"""CPU tier: the split -> delimiter -> timestamp chain (lc_exec.cuh: lc_split_delim_ts_setup, lc_split_delim_ts_value,
lc_split_delim_ts_collapse, lc_ts_full, lc_ts_resolve, lc_split_delim_ts_time, lc_split_delim_ts_verdict and
lc_split_delim_sls_body, built for the host by tests/emul/split_delim_timestamp_sls.py), fed the oracle's split_lines /
multiline_split tables and delim_parse_batch tables over those pieces, against the oracle's splitter +
ProcessorParseDelimiterNative + a group-level ProcessorParseTimestampNative step + sls_serialize_logs on one flat source
event, with 1, 3 and 32 emulated lanes: bytes and all nine counters, in UTC and in a zone with daylight saving."""
import os
import random
import time
import zlib

import pytest

from oracle import oracle as orc
from tests import delim_sls_cases as dc
from tests import split_delim_timestamp_sls_cases as dtc
from tests import split_sls_cases as sc
from tests.emul import split_delim_timestamp_sls as emul

OKEY = dtc.OKEY


@pytest.fixture(params=("UTC", "America/New_York"))
def zone(request):
    saved = os.environ.get("TZ")
    os.environ["TZ"] = request.param
    time.tzset()
    yield request.param
    if saved is None:
        os.environ.pop("TZ", None)
    else:
        os.environ["TZ"] = saved
    time.tzset()


def _pieces(val, ml=None):
    if ml is None:
        return orc.split_lines(val, 10)
    off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    return off, ln


def _run(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml=None):
    off, ln = _pieces(val, ml)
    tabs = dtc.tables(val, off, ln, cfg)
    quote = cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')
    # time_ns is the source event's Time_ns as the serialiser writes it: none unless enable_ns
    return emul.serialize(val, off, ln, tabs, cfg["max_fields"], cfg["sep"], quote, cfg["treatment"],
                          [k.encode() for k in cfg["keys"]], cfg["source"].encode(), dc.renamed_key(cfg),
                          cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], okey, pos, t,
                          ns if enable_ns else None, tkey, fmt, now, di, enable_ns, nlanes=nlanes)


def _check(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, mcfg=None, lanes=(1, 3, 32)):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": 10}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = dtc.oracle_chain(val, split_cfg, cfg, tkey, fmt, now, di, t, ns if enable_ns else None, pos,
                                        okey, multiline=mcfg is not None, enable_ns=enable_ns)
    for nlanes in lanes:
        got, ctr, _st, _tab, _vb = _run(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml)
        assert got == want, (cfg, tkey, fmt, okey, enable_ns, nlanes)
        assert dtc.fold(ctr) == wctr, (cfg, tkey, fmt, okey, ctr, wctr)
    return want, ctr


CONFIGS = list(dtc.configs())
BARE = {"renamed_keep_succeed", "renamed_fail", "raw_log_fail"}  # the piece itself is the time value
# the formats whose strings can stand where each configuration reads its time: a separator or a quote inside needs the
# quote state machine, and the piece itself is the value of the bare configurations
MATRIX = [(c, f) for c in CONFIGS for f in dtc.FORMATS
          if dtc.plain_fmt(f, c[1]) and not (c[0] in BARE and f in (dtc.COMMA_FMT, dtc.DQ_FMT))]


@pytest.mark.parametrize("case,fmt", MATRIX, ids=["%s-%s" % (c[0], f) for c, f in MATRIX])
def test_matrix_matches_oracle(case, fmt, zone):
    cid, cfg, tkey, gen = case
    rng = random.Random(zlib.crc32((cid + fmt + zone).encode()))
    val = gen(rng, fmt)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di in (43200, -1):
            for enable_ns in (False, True):
                _check(val, cfg, tkey, fmt, dtc.NOW, di, enable_ns, okey, pos, t, ns,
                       lanes=(1, 3, 32) if (i == 1 and enable_ns) else (1,))


def test_every_status_and_counter_moves():
    rng = random.Random(5)
    cfg = dtc.config(["time", "level", "msg"], keep_fail=False)
    val = dtc.lines_value(rng, dtc.YMD, 400)
    _w, ctr = _check(val, cfg, b"time", dtc.YMD, dtc.NOW, 43200, True, OKEY, 9, 1 << 30, 4)
    assert all(c > 0 for c in ctr), ctr  # parsed, failed, erased and blank pieces; no key, failed, history, discarded
    # and parsed times


def test_quoted_time_column_holding_the_separator():
    """"Nov 14, 2023 22:13:20" with %b %d, %Y %H:%M:%S: the quoted column is one value; the tap reads it in place"""
    t0 = dtc.render(dtc.COMMA_FMT, dtc.NOW - 100).encode()
    val = b'"%s",INFO,a\n"%s",WARN,b\n%s,E,c' % (t0, t0, t0)
    cfg = dtc.config(["time", "level", "msg"])
    _check(val, cfg, b"time", dtc.COMMA_FMT, dtc.NOW, 43200, True, None, 0, 1, None)
    off, ln = orc.split_lines(val, 10)
    _b, _c, st, (voff, vlen), vbuf = _run(val, cfg, b"time", dtc.COMMA_FMT, dtc.NOW, 43200, True, None, 0, 1, None, 1)
    assert list(st) == [0, 0, 2]  # the unquoted one is cut at ", " and fails
    for i in (0, 1):
        assert voff[i] == off[i] + 1 and vbuf[voff[i]:voff[i] + vlen[i]] == t0


def test_doubled_quotes_are_collapsed():
    """a column holding doubled quotes is collapsed in place in the value buffer; the format parses only the collapsed
    value"""
    t0 = dtc.render(dtc.DQ_FMT, dtc.NOW - 7).encode()
    q = t0.replace(b'"', b'""')
    long_q = b'"' + b'""' * 40 + b'"'  # a column of 40 doubled quotes: collapsed across two 32-byte steps
    val = b'"%s",x\n"%s""",y\n"%s"\n%s,z\n"a""b%s""",w' % (q, q, long_q[1:-1], t0, b'""' * 20)
    cfg = dtc.config(["time", "level"])
    for nlanes in (1, 3, 32):
        _b, ctr, st, (voff, vlen), vbuf = _run(val, cfg, b"time", dtc.DQ_FMT, dtc.NOW, -1, False, None, 0, 1, None,
                                               nlanes)
        assert st[0] == 0 and st[1] == 0, list(st)
        assert vbuf[voff[0]:voff[0] + vlen[0]] == t0
        assert vbuf[voff[1]:voff[1] + vlen[1]] == t0 + b'"'
        assert vbuf[voff[2]:voff[2] + vlen[2]] == b'"' * 40
        assert vbuf[voff[4]:voff[4] + vlen[4]] == b'a"b' + b'"' * 21
    for okey in (None, OKEY):
        _check(val, cfg, b"time", dtc.DQ_FMT, dtc.NOW, -1, True, okey, 3, 1, 2)


def test_cache_hits_after_failed_parse_and_across_erased_pieces():
    t0 = dtc.render(dtc.YMD, dtc.NOW - 100).encode()
    lines = [t0 + b",a", b'"open,' + t0, t0 + b"Z,b", b"", t0 + b",c", b"garbage,d", t0 + b"7,e", b"   ",
             b'ab"c,' + t0, t0 + b",f", dtc.render(dtc.YMD, dtc.NOW - 86400).encode() + b",g", t0 + b",h"]
    val = b"\n".join(lines)
    for f in range(8):
        cfg = dtc.config(["time", "level"], renamed="raw", keep_fail=bool(f & 1), keep_succeed=bool(f & 2),
                         copy_raw=bool(f & 4))
        for tkey in (b"time", b"raw", b"__raw_log__", b"content"):
            for di in (43200, -1):
                _check(val, cfg, tkey, dtc.YMD, dtc.NOW, di, True, OKEY, 3, 7, None)


@pytest.mark.parametrize("fmt", [dtc.F_FMT, "%s"])
def test_fraction_and_epoch_formats_with_and_without_ns(fmt):
    rng = random.Random(len(fmt))
    val = dtc.lines_value(rng, fmt, 120)
    cfg = dtc.config(["time", "level", "msg"])
    for enable_ns in (False, True):
        for okey in (None, OKEY, b""):
            _check(val, cfg, b"time", fmt, dtc.NOW, 43200, enable_ns, okey, 1 << 33, 1700000000, 123)


@pytest.mark.parametrize("flags", range(8))
def test_blank_empty_and_failed_pieces(flags):
    cfg = dtc.config(["a", "b"], renamed="raw", keep_fail=bool(flags & 1), keep_succeed=bool(flags & 2),
                     copy_raw=bool(flags & 4), allow_short=bool(flags & 1))
    t0 = dtc.render("%s", dtc.NOW - 5).encode()
    for val in (b"\n\n\n", b"", b"   \n \r\n" + t0, t0 + b"\n" + t0 + b"x\n\n", b'"' + t0, t0 + b",1,2,3",
                b" " + t0 + b" "):
        for tkey in (b"a", b"raw", b"__raw_log__", b"content", b"nope"):
            for okey in (None, OKEY):
                _check(val, cfg, tkey, "%s", dtc.NOW, 43200, True, okey, 17, 1700000000, 5)


def test_whole_chunk_discarded():
    old = dtc.render(dtc.YMD, dtc.NOW - 86400).encode()
    val = b"\n".join(b"%s,%d" % (old, i) for i in range(50))
    want, ctr = _check(val, dtc.config(["time", "i"]), b"time", dtc.YMD, dtc.NOW, 43200, False, OKEY, 1, 2, 3)
    assert want == b"" and ctr[6] == 50 and ctr[7] == 50


def test_overflow_column_key_in_discard_mode_is_an_ordinary_key():
    cfg = dtc.config(["__column1__", "b"], treatment="discard")
    _check(b"1700000000,2,3\n5\n\n1699999999", cfg, b"__column1__", "%s", dtc.NOW, -1, False, OKEY, 3, 5, None)
    _check(b"1700000000,2,3\n5\n\n1699999999", cfg, b"__column2__", "%s", dtc.NOW, -1, False, OKEY, 3, 5, None)


@pytest.mark.parametrize("name", ["start", "start_cont", "end"])
def test_multiline_pieces_with_quoted_fields_across_lines(name, zone):
    rng = random.Random(zlib.crc32(name.encode()))
    mcfg = sc.ml_config(name)
    t0 = dtc.render(dtc.COMMA_FMT, dtc.NOW - 60).encode()
    recs = []
    for i in range(25):
        head = {"start": b"2024-01-0%d 10:00:0%d" % (rng.randint(1, 9), rng.randint(0, 9)),
                "start_cont": b"line %d" % i, "end": b"x%d" % i}[name]
        tq = b'"%s\n"' % t0 if rng.random() < 0.3 else b'"%s"' % t0
        body = b',"a\nb",' + tq if name != "start_cont" else b',' + tq + b"\ncontinue,\"q\"\ncontinue 2,x"
        tail = b"\nendLine %d" % i if name == "end" else b""
        recs.append(head + body + tail + (b"\nstray,1" if rng.random() < 0.3 else b""))
    val = b"\n".join(recs)
    for tr in dc.TREATMENTS:
        for tkey in (b"t", b"raw"):
            cfg = dtc.config(["h", "b", "t"], treatment=tr, renamed="raw", keep_succeed=True)
            _check(val, cfg, tkey, dtc.COMMA_FMT, dtc.NOW, 43200, True, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


@pytest.mark.parametrize("tkey,okey,treatment,why", [
    (OKEY, OKEY, "extend", "offset key"),
    (b"", b"", "extend", "offset key"),
    (b"__column3__", None, "extend", "__column"),
    (b"__column0__", OKEY, "keep", "__column"),
])
def test_refusals(tkey, okey, treatment, why):
    cfg = dtc.config(["a", "b"], treatment=treatment)
    with pytest.raises(emul.Refused, match=why):
        _run(b"x,1", cfg, tkey, "%s", dtc.NOW, -1, False, okey, 0, 0, None, 1)


def test_refusals_of_the_chain_and_the_timestamp_stage():
    cfg = dtc.config(["time", "b"])
    # the offset key is not an event key without log.file.offset metadata: absent, not refused
    _check(b"1700000000,1", cfg, OKEY, "%s", dtc.NOW, -1, False, None, 0, 0, None)
    with pytest.raises(emul.Refused, match="offset key equals SourceKey"):
        _run(b"x,1", cfg, b"time", "%s", dtc.NOW, -1, False, b"content", 0, 0, None, 1)
    with pytest.raises(emul.Refused, match="distinct"):
        _run(b"x,1", dtc.config(["a", "a"]), b"a", "%s", dtc.NOW, -1, False, None, 0, 0, None, 1)
    with pytest.raises(emul.Refused):
        _run(b"x,1", cfg, b"time", "%c", dtc.NOW, -1, False, OKEY, 0, 0, None, 1)
    # a source Time_ns without enable_ns: the records that keep the source time would carry Time_ns, the parsed ones
    # not
    off, ln = orc.split_lines(b"x,1", 10)
    tabs = dtc.tables(b"x,1", off, ln, cfg)
    args = [b"x,1", off, ln, tabs, cfg["max_fields"], b",", ord('"'), "extend", [b"time", b"b"], b"content",
            b"content", True, False, False, OKEY, 0, 0, 5, b"time", "%s", dtc.NOW, -1]
    with pytest.raises(emul.Refused, match="enable_ns"):
        emul.serialize(*args, False)
    emul.serialize(*args, True)
