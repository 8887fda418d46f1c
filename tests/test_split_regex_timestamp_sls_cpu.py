"""CPU tier: the split -> regex -> timestamp chain (lc_exec.cuh: lc_split_regex_ts_setup, lc_split_regex_ts_value,
lc_ts_full, lc_ts_resolve, lc_split_regex_ts_time, lc_split_regex_ts_verdict and lc_split_regex_sls_body, built for
the host by tests/emul/split_regex_timestamp_sls.py), fed the oracle's split_lines / multiline_split and
regex_parse_batch tables, against the oracle's splitter + ProcessorParseRegexNative + a group-level
ProcessorParseTimestampNative step + sls_serialize_logs on one flat source event, with 1, 3 and 32 emulated lanes:
bytes and all eight counters, in UTC and in a zone with daylight saving."""
import os
import random
import time
import zlib

import pytest

from oracle import oracle as orc
from tests import regex_sls_cases as rc
from tests import split_regex_timestamp_sls_cases as tc
from tests import split_sls_cases as sc
from tests.emul import split_regex_timestamp_sls as emul

OKEY = tc.OKEY


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


def _run(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml=None):
    if ml is None:
        off, ln = orc.split_lines(val, 10)
    else:
        off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    tables, pitch = tc.tables_of(val, off, ln, cfg)
    a = tc.device_args(cfg)
    # time_ns is the source event's Time_ns as the serialiser writes it: none unless enable_ns
    return emul.serialize(val, off, ln, tables, pitch, a["keys"], a["source_key"], a["renamed_key"], a["keep_fail"],
                          a["keep_succeed"], a["copy_raw"], a["whole_line"], okey, pos, t, ns if enable_ns else None,
                          tkey, fmt, now, di, enable_ns, nlanes=nlanes)


def _check(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, mcfg=None, lanes=(1, 3, 32)):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": 10}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = tc.oracle_chain(val, split_cfg, cfg, tkey, fmt, now, di, t, ns, pos, okey,
                                       multiline=mcfg is not None, enable_ns=enable_ns)
    for nlanes in lanes:
        got, ctr, _st, _tab = _run(val, cfg, tkey, fmt, now, di, enable_ns, okey, pos, t, ns, nlanes, ml)
        assert got == want, (cfg, tkey, fmt, okey, enable_ns, nlanes)
        assert ctr == wctr, (cfg, tkey, fmt, okey, ctr, wctr)
    return want, wctr


CONFIGS = list(tc.configs())
FORMATS = [tc.NGINX_FMT, tc.F_FMT, "%s"]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix_matches_oracle(case, fmt, zone):
    cid, cfg, tkey = case
    rng = random.Random(zlib.crc32((cid + fmt + zone).encode()))
    val = tc.lines_value(rng, fmt, 60)
    for i, okey in enumerate((None, OKEY, b"")):
        t, ns = sc.TIMES[(len(cid) + i) % len(sc.TIMES)]
        pos = sc.POSITIONS[(len(cid) + 3 * i) % len(sc.POSITIONS)]
        for di in (43200, -1):
            for enable_ns in (False, True):
                _check(val, cfg, tkey, fmt, tc.NOW, di, enable_ns, okey, pos, t, ns,
                       lanes=(1, 3, 32) if (i == 1 and enable_ns) else (1,))


def test_every_status_and_counter_moves():
    rng = random.Random(5)
    val = tc.lines_value(rng, tc.NGINX_FMT, 300)
    cfg = rc.config(tc.KEYS, "content", None, False, False, False, regex=tc.PATTERN)
    _w, ctr = _check(val, cfg, b"time", tc.NGINX_FMT, tc.NOW, 43200, True, OKEY, 9, 1 << 30, 4)
    assert all(c > 0 for c in ctr[:3]), ctr  # parsed, failed and erased pieces
    assert all(c > 0 for c in ctr[4:]), ctr  # failed, history, discarded and parsed times
    _w, ctr = _check(val, rc.config(tc.KEYS, "content", None, True, False, False, regex=tc.PATTERN), b"time",
                     tc.NGINX_FMT, tc.NOW, 43200, True, OKEY, 9, 1 << 30, 4)
    assert ctr[3] > 0  # kept failures have no "time" key


def test_cache_hit_after_failed_full_parse_and_erased_rows_between():
    t0 = tc.render(tc.NGINX_FMT, tc.NOW - 100).encode()
    lines = [t0 + b" INFO a", b"nospace", b"garbage X b", b"", t0 + b"zz INFO c", b"nospace2", t0 + b"9 E d",
             tc.render(tc.NGINX_FMT, tc.NOW - 5).encode() + b" E e", t0 + b" INFO f"]
    val = b"\n".join(lines)
    for keep_fail in (False, True):
        cfg = rc.config(tc.KEYS, "content", None, keep_fail, False, False, regex=tc.PATTERN)
        for di in (43200, -1):
            _check(val, cfg, b"time", tc.NGINX_FMT, tc.NOW, di, True, OKEY, 3, 7, None)


def test_epoch_seconds_beyond_32_bits_and_below_2_28():
    lines = [b"5000000123 INFO a", b"12345 INFO b", b"4294967296 E c", b"268435455 E d", b"-7 E e", b"0 E f"]
    val = b"\n".join(lines)
    cfg = rc.config(tc.KEYS, regex=tc.PATTERN)
    want, ctr = _check(val, cfg, b"time", "%s", tc.NOW, -1, True, None, 0, 1700000000, None)
    assert ctr[3:] == [0, 1, 1, 1, 4], ctr  # "0" fails, "-7" is discarded (time <= 0)


def test_whole_chunk_discarded():
    old = tc.render(tc.NGINX_FMT, tc.NOW - 86400).encode()
    val = b"\n".join(old + b" INFO %d" % i for i in range(50))
    cfg = rc.config(tc.KEYS, regex=tc.PATTERN)
    want, ctr = _check(val, cfg, b"time", tc.NGINX_FMT, tc.NOW, 43200, False, OKEY, 1, 2, 3)
    assert want == b"" and ctr[6] == 50 and ctr[5] == 50


@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_whole_line_mode(nkeys):
    keys = ["time", "content"][:nkeys]
    line = tc.render(tc.NGINX_FMT, tc.NOW - 10).encode()
    val = b"\n".join([line, b"", line + b" tail", b"bad", line])
    for f in (0, 3, 5, 7):
        cfg = rc.config(keys, "content", None, bool(f & 1), bool(f & 2), bool(f & 4), regex=rc.WHOLE_LINE)
        for tkey in (b"time", b"content", b"__raw_log__"):
            for okey in (None, OKEY):
                _check(val, cfg, tkey, tc.NGINX_FMT, tc.NOW, 43200, True, okey, 77, (1 << 28) - 1, 5)


@pytest.mark.parametrize("discard", [False, True])
def test_multiline_records(discard, zone):
    from loongcollector_b200 import synth
    from tests import split_regex_sls_cases as src
    buf, _, _ = synth.java_stack_records(60, seed=4)
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
            "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    for di in (-1, 86400 * 365 * 3):
        _check(buf.tobytes(), cfg, b"time", tc.F_FMT, 1790000000, di, True, OKEY, 123456, 1700000000, 3, mcfg=mcfg)


def test_refusals():
    val = b"a 1 b\nx\n"
    cfg = rc.config(tc.KEYS, "content", None, True, False, False, regex=tc.PATTERN)
    with pytest.raises(emul.Refused, match="offset"):
        _run(val, cfg, OKEY, tc.NGINX_FMT, tc.NOW, -1, False, OKEY, 0, 0, None, 1)
    # the offset key is not an event key without log.file.offset metadata: absent, not refused
    _check(val, cfg, OKEY, tc.NGINX_FMT, tc.NOW, -1, False, None, 0, 0, None)
    # a regex key named like the offset key replaces the digits on parsed rows, a kept failure still holds them
    cfg2 = rc.config(["a", OKEY.decode(), "c"], "content", None, True, False, False, regex=tc.PATTERN)
    with pytest.raises(emul.Refused, match="offset"):
        _run(val, cfg2, OKEY, tc.NGINX_FMT, tc.NOW, -1, False, OKEY, 0, 0, None, 1)
    with pytest.raises(emul.Refused):
        _run(val, cfg, b"time", "%c", tc.NOW, -1, False, OKEY, 0, 0, None, 1)
    # a source Time_ns without enable_ns: the records that keep the source time would carry Time_ns, the parsed ones not
    off, ln = orc.split_lines(val, 10)
    tables, pitch = tc.tables_of(val, off, ln, cfg)
    a = tc.device_args(cfg)
    args = [val, off, ln, tables, pitch, a["keys"], a["source_key"], a["renamed_key"], a["keep_fail"],
            a["keep_succeed"], a["copy_raw"], a["whole_line"], OKEY, 0, 0, 5, b"time", tc.NGINX_FMT, tc.NOW, -1]
    with pytest.raises(emul.Refused, match="enable_ns"):
        emul.serialize(*args, False)
    emul.serialize(*args, True)
