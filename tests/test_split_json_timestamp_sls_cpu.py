"""CPU tier: the split -> JSON -> timestamp chain (lc_exec.cuh: lc_split_json_ts_setup, lc_json_ts_last_member,
lc_split_json_ts_value, lc_ts_full, lc_ts_resolve, lc_split_json_ts_time, lc_split_json_ts_verdict and
lc_split_json_sls_body, built for the host by tests/emul/split_json_timestamp_sls.py), fed the oracle's split_lines /
multiline_split tables and oracle/json_parse.py's tables over those pieces, against the oracle's splitter +
ProcessorParseJsonNative + a group-level ProcessorParseTimestampNative step + sls_serialize_logs on one flat source
event, with 1, 3 and 32 emulated lanes: bytes and all eight counters, in UTC and in a zone with daylight saving."""
import os
import random
import time
import zlib

import pytest

from oracle import oracle as orc
from tests import split_json_timestamp_sls_cases as jtc
from tests import split_sls_cases as sc
from tests.emul import split_json_timestamp_sls as emul

OKEY = jtc.OKEY


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


def _pieces(val, ml=None, split_char=10):
    if ml is None:
        return orc.split_lines(val, split_char)
    off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    return off, ln


def _run(val, jcfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml=None):
    off, ln = _pieces(val, ml)
    tables = jtc.tables_of(val, off, ln, jcfg)
    # time_ns is the source event's Time_ns as the serialiser writes it: none unless enable_ns
    return emul.serialize(val, off, ln, tables, jcfg["SourceKey"].encode(), jtc.renamed_key(jcfg),
                          jcfg["KeepingSourceWhenParseFail"], jcfg["KeepingSourceWhenParseSucceed"],
                          jcfg["CopingRawLog"], okey, pos, t, ns if enable_ns else None, tkey, fmt, now, di,
                          enable_ns, nlanes=nlanes)


def _check(val, jcfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, mcfg=None, lanes=(1, 3, 32)):
    split_cfg = mcfg or {"SourceKey": jcfg["SourceKey"], "SplitChar": 10}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = jtc.oracle_chain(val, split_cfg, jcfg, tkey, fmt, now, di, t, ns if enable_ns else None, pos,
                                        okey, multiline=mcfg is not None, enable_ns=enable_ns)
    for nlanes in lanes:
        got, ctr, _st, _tab, _vb = _run(val, jcfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml)
        assert got == want, (jcfg, tkey, fmt, okey, enable_ns, nlanes)
        assert ctr == wctr, (jcfg, tkey, fmt, okey, ctr, wctr)
    return want, wctr


CONFIGS = list(jtc.configs())


@pytest.mark.parametrize("fmt", jtc.FORMATS)
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix_matches_oracle(case, fmt, zone):
    cid, jcfg, tkey, member = case
    rng = random.Random(zlib.crc32((cid + fmt + zone).encode()))
    val = jtc.lines_value(rng, fmt, 80, member)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di in (43200, -1):
            for enable_ns in (False, True):
                _check(val, jcfg, tkey, fmt, jtc.NOW, di, enable_ns, okey, pos, t, ns,
                       lanes=(1, 3, 32) if (i == 1 and enable_ns) else (1,))


def test_every_status_and_counter_moves():
    rng = random.Random(5)
    val = jtc.lines_value(rng, jtc.YMD, 400)
    _w, ctr = _check(val, jtc.config("content"), b"time", jtc.YMD, jtc.NOW, 43200, True, OKEY, 9, 1 << 30, 4)
    assert all(c > 0 for c in ctr[:3]), ctr  # parsed, failed and erased pieces
    assert all(c > 0 for c in ctr[3:]), ctr  # no key, failed, history, discarded and parsed times


def test_values_from_chunk_and_arena():
    """the tap's table: a plain string member is read in place, an escaped one and a %f rendering from the arena's
    copy behind the chunk, and every value's bytes in the value buffer are the rendered value"""
    t0 = jtc.render(jtc.YMD, jtc.NOW - 100)
    lines = [b'{"time":"%s"}' % t0.encode(), b'{"time":%s}' % jtc.escaped(t0).encode(), b'{"x":1}',
             b'{"time":"a","time":"%s"}' % t0.encode(), b'{"\\u0074ime":%s,"y":2}' % jtc.escaped(t0).encode()]
    val = b"\n".join(lines)
    jcfg = jtc.config("content")
    off, ln = orc.split_lines(val, 10)
    tables = jtc.tables_of(val, off, ln, jcfg)
    _b, ctr, st, (voff, vlen), vbuf = emul.serialize(val, off, ln, tables, b"content", b"content", False, False,
                                                     False, None, 0, 1, None, b"time", jtc.YMD, jtc.NOW)
    assert list(st) == [0, 0, 1, 0, 0] and ctr[3:] == [1, 0, 0, 0, 4], (list(st), ctr)
    assert voff[0] < len(val) and voff[1] >= len(val) and voff[3] < len(val) and voff[4] >= len(val)
    for i in (0, 1, 3, 4):
        assert vbuf[voff[i]:voff[i] + vlen[i]] == t0.encode()
    num = b'{"ts":1700000000}\n{"ts":-0}\n{"ts":1699999999.25}'
    off, ln = orc.split_lines(num, 10)
    tables = jtc.tables_of(num, off, ln, jcfg)
    _b, ctr, st, (voff, vlen), vbuf = emul.serialize(num, off, ln, tables, b"content", b"content", False, False,
                                                     False, None, 0, 1, None, b"ts", "%s", jtc.NOW)
    got = [vbuf[o:o + n] for o, n in zip(voff, vlen)]
    assert got == [b"1700000000", b"0", b"1699999999.250000"], got
    assert voff[0] < len(num) and voff[1] < len(num) and voff[2] >= len(num)


def test_cache_hits_alternating_chunk_and_arena_across_erased_pieces():
    t0 = jtc.render(jtc.YMD, jtc.NOW - 100)
    e0 = jtc.escaped(t0).encode()
    lines = [b'{"time":"%s"}' % t0.encode(), b'{"time":%s}' % e0, b"broken", b'{"time":"%sZ"}' % t0.encode(),
             b"", b'{"time":"garbage"}', b'{"time":%s}' % e0, b'{"time":"%s"}' % t0.encode(),
             b'{"time":%s}' % jtc.escaped(t0 + "7").encode(), b"{}", b'{"time":"%s"}' % t0.encode()]
    val = b"\n".join(lines)
    for f in range(8):
        jcfg = jtc.config("content", None, bool(f & 1), bool(f & 2), bool(f & 4))
        for di in (43200, -1):
            _check(val, jcfg, b"time", jtc.YMD, jtc.NOW, di, True, OKEY, 3, 7, None)


@pytest.mark.parametrize("flags", range(8))
def test_empty_object_empty_pieces_and_failures(flags):
    jcfg = jtc.config("content", "raw", bool(flags & 1), bool(flags & 2), bool(flags & 4))
    t0 = jtc.render("%s", jtc.NOW - 5).encode()
    for val in (b"{}\n{}\n", b"\n\n\n", b"", b"{}", t0 + b"\n" + t0 + b"x\n\n{}", b'{\n}\n', b'{"raw":%s}' % t0):
        for tkey in (b"raw", b"__raw_log__", b"content", b"nope"):
            for okey in (None, OKEY):
                _check(val, jcfg, tkey, "%s", jtc.NOW, 43200, True, okey, 17, 1700000000, 5)


def test_whole_chunk_discarded():
    old = jtc.render(jtc.YMD, jtc.NOW - 86400).encode()
    val = b"\n".join(b'{"time":"%s","i":%d}' % (old, i) for i in range(50))
    want, ctr = _check(val, jtc.config("content"), b"time", jtc.YMD, jtc.NOW, 43200, False, OKEY, 1, 2, 3)
    assert want == b"" and ctr[5] == 50 and ctr[6] == 50


@pytest.mark.parametrize("name", list(sc.ML_CFGS))
def test_multiline_pieces(name, zone):
    rng = random.Random(len(name))
    val = sc.ml_value(rng, 12) + b"\n" + jtc.lines_value(rng, "%s", 30)
    mcfg = sc.ml_config(name)
    for jcfg, tkey in ((jtc.config("content", "raw", True, True, True), b"time"),
                       (jtc.config("content", None, True, False, True), b"__raw_log__")):
        _check(val, jcfg, tkey, "%s", jtc.NOW, 43200, True, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


def test_refusals():
    val = b'{"time":"x"}\n'
    jcfg = jtc.config("content", None, True)
    with pytest.raises(emul.Refused, match="offset key"):
        _run(val, jcfg, OKEY, jtc.YMD, jtc.NOW, -1, False, OKEY, 0, 0, None, 1)
    # the offset key is not an event key without log.file.offset metadata: absent, not refused
    _check(val, jcfg, OKEY, jtc.YMD, jtc.NOW, -1, False, None, 0, 0, None)
    with pytest.raises(emul.Refused, match="offset key equals SourceKey"):
        _run(val, jcfg, b"time", jtc.YMD, jtc.NOW, -1, False, b"content", 0, 0, None, 1)
    with pytest.raises(emul.Refused):
        _run(val, jcfg, b"time", "%c", jtc.NOW, -1, False, OKEY, 0, 0, None, 1)
    # a source Time_ns without enable_ns: the records that keep the source time would carry Time_ns, the parsed ones not
    off, ln = orc.split_lines(val, 10)
    tables = jtc.tables_of(val, off, ln, jcfg)
    args = [val, off, ln, tables, b"content", b"content", True, False, False, OKEY, 0, 0, 5, b"time", jtc.YMD,
            jtc.NOW, -1]
    with pytest.raises(emul.Refused, match="enable_ns"):
        emul.serialize(*args, False)
    emul.serialize(*args, True)
