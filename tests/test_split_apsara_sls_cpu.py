"""CPU tier: the split -> Apsara chain (lc_exec.cuh: lc_ap_scan, lc_ap_resolve and lc_ap_fields over the pieces with
the chunk as their base, then lc_split_apsara_sls_setup, lc_split_apsara_sls_body and lc_split_apsara_verdict, built
for the host by tests/emul/split_apsara_sls.py), fed the oracle's split_lines / multiline_split tables, against the
oracle's splitter + oracle/apsara.py's ProcessorParseApsaraNative (fixed `now`) + sls_serialize_logs on one flat
source event, with 1, 3 and 32 emulated lanes, in UTC and in a zone with daylight saving: bytes and all five
counters."""
import os
import time

import numpy as np
import pytest

from oracle import apsara as oap
from oracle import oracle as orc
from tests import split_apsara_sls_cases as ac
from tests import split_sls_cases as sc
from tests.emul import split_apsara_sls as emul

OKEY = ac.OKEY


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


def _pieces(val, ml):
    if not ml:
        return orc.split_lines(val, 10)
    p = orc.ProcessorSplitMultilineLogStringNative(ac.ml_config())
    off, ln, _fl, _ctr = orc.multiline_split(val, p.start, p.cont, p.end, p.opts.discard)
    return off, ln


def _run(val, acfg, okey, pos, t, ns, enable_ns, nlanes, ml=False, now=ac.NOW, di=ac.DI):
    off, ln = _pieces(val, ml)
    return emul.serialize(val, off, ln, acfg["SourceKey"].encode(), ac.adjust(acfg), now, di, ac.renamed_key(acfg),
                          acfg["KeepingSourceWhenParseFail"], acfg["KeepingSourceWhenParseSucceed"],
                          acfg["CopingRawLog"], okey, pos, t, ns if enable_ns else None, enable_ns, nlanes=nlanes)


def _check(val, acfg, okey, pos, t, ns, ml=False, lanes=(1, 3, 32), now=ac.NOW, di=ac.DI):
    split_cfg = ac.ml_config(acfg["SourceKey"]) if ml else {"SourceKey": acfg["SourceKey"], "SplitChar": 10}
    for enable_ns in (True, False):
        want, wctr, _, _ = ac.oracle_chain(val, split_cfg, acfg, t, ns, pos, okey, multiline=ml, enable_ns=enable_ns,
                                           now=now, di=di)
        for nlanes in (lanes if enable_ns else (1,)):
            got, ctr = _run(val, acfg, okey, pos, t, ns, enable_ns, nlanes, ml, now, di)
            assert got == want, (acfg, okey, enable_ns, nlanes)
            assert ctr == wctr, (acfg, okey, ctr, wctr)
    return want, wctr


CONFIGS = [(f"{r}_{i}", c) for r in (None, "raw", "content", "__raw_log__", OKEY.decode(), "microtime", "__THREAD__",
                                     "k1") for i, c in enumerate(ac.flag_configs(r))]


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix_matches_oracle(case, okey):
    cid, acfg = case
    val = ac.random_value(len(cid) * 7 + (0 if okey is None else len(okey) + 1))
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _check(val, acfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns, lanes=(1, 32))


@pytest.mark.parametrize("okey", [b"k1", b"__LEVEL__", b"__THREAD__", b"microtime", b"raw", b"__raw_log__"])
@pytest.mark.parametrize("flags", range(8))
def test_offset_key_equal_to_fields_or_added_keys(okey, flags):
    """an offset key equal to a key:value key, a base-field name, "microtime", RenamedSourceKey or __raw_log__ is
    appended beside them, never merged; an added key equal to it is not added"""
    val = b"\n".join(ac.special_lines(okey=okey))
    for renamed in ("raw", "__raw_log__"):
        acfg = ac.config("content", renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4))
        _check(val, acfg, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("source", ["content", "k1", "__THREAD__", "__LEVEL__", "microtime", "raw"])
@pytest.mark.parametrize("flags", range(8))
def test_source_key_equal_to_fields(source, flags):
    """SourceKey equal to a key:value key (once and repeated: both SourceKey entries stay), to a base field (that
    field goes, the piece stays) and to "microtime" (the microtime entry goes)"""
    val = b"\n".join(ac.special_lines(source=source) + ac.special_lines(source="k1"))
    for renamed in (None, "raw", "microtime", "__THREAD__"):
        acfg = ac.config(source, renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4))
        for okey in (None, OKEY):
            _check(val, acfg, okey, 3, 1700000000, 5, lanes=(1, 3))


@pytest.mark.parametrize("flags", range(8))
def test_empty_failed_and_erased_pieces(flags):
    acfg = ac.config("content", None, bool(flags & 1), bool(flags & 2), bool(flags & 4))
    for val in (b"\n\n\n", b"", b"x", b"x\ny\n\nz", b"[\n]\n", ac.date(ac.BOUNDARY - 99) + b"\n\n",
                ac.date(ac.NOW) + b"\nx\n\n"):
        for okey in (None, OKEY):
            _check(val, acfg, okey, 17, 1700000000, 5)


def test_discard_boundary(zone):
    """pieces a second on either side of the boundary, epoch and date, with the discard on and off; the dates are
    rendered in the process's zone so that they land on the boundary there"""
    lines = []
    for d in (-2, -1, 0, 1, 2):
        t = ac.BOUNDARY + d
        lines.append(ac.epoch(t, 5) + b"\te:%d" % d)
        lines.append(b"[" + time.strftime("%Y-%m-%d %H:%M:%S", time.localtime(t)).encode() + b".25]\td:%d" % d)
    val = b"\n".join(lines)
    for f in (0, 7):
        acfg = ac.config("content", "raw", bool(f & 1), bool(f & 2), bool(f & 4))
        want, wctr = _check(val, acfg, OKEY, 0, 1700000000, 1)
        assert wctr[2] == 4 and wctr[4] == 6, wctr
        _, wctr = _check(val, acfg, OKEY, 0, 1700000000, 1, di=-1)
        assert wctr[2] == 0 and wctr[4] == 10, wctr


def test_time_cache_across_failed_and_erased_pieces(zone):
    """hits on the key of a full parse that came before failed, empty and discarded pieces"""
    t = ac.NOW - 50
    lines = [ac.date(t, b".1"), b"[2023-11-15 xx:00:00]", b"", ac.date(ac.BOUNDARY - 500, b".3"), b"garbage",
             ac.date(t, b".2") + b"\tk:v", ac.epoch(t + 1), ac.date(t, b",7"), ac.date(t)]
    for f in (0, 1):
        _check(b"\n".join(lines), ac.config("content", None, bool(f)), OKEY, 9, 1700000000, None)


def test_short_time_strings_read_the_chunk():
    """Pinned: the 19-byte cache key of a piece shorter than 20 bytes takes the chunk's next bytes (the pieces are
    views into the chunk), while oracle/apsara.py packs values back to back and sees other bytes there.  Neither can
    hit: a hit needs a time string of at least 19 bytes, and such a short key holds its ']'.  Each piece's record is
    the one it gets parsed on its own."""
    short = b"[2024-1-1 1:2:3]"
    lines = [short, short + short[:-1] + b".5]", short + b"\t[2024-01-01 01:02:03.7]", short, b"\t" + short,
             b"[2024-01-01 01:02:03]", short + b"[2024-01-01 00:00:00]"]
    val = b"\n".join(lines)
    acfg = ac.config("content", None, True, True)
    want, wctr = _check(val, acfg, None, 0, 1700000000, None, di=-1)
    alone = b"".join(ac.oracle_chain(v, {"SourceKey": "content", "SplitChar": 10}, acfg, 1700000000, None, 0,
                                     enable_ns=False, di=-1)[0] for v in lines)
    assert want == alone
    # the multiline splitter keeps the next line inside the piece: the key then reads it from the piece itself
    ml = b"\n".join([short, b"2024-1-1 1:2:3]", short, b"[2024-01-01 01:02:03.9]\tk:v"])
    _check(ml, acfg, None, 0, 1700000000, None, ml=True, di=-1)


def test_widest_epochs_render_microtime_in_full():
    """Pinned: "microtime" is the "%ld" rendering of logTime_in_micro, as ProcessorParseApsaraNative::Process renders
    it (std::to_string).  The reference's snprintf into 20 bytes would cut a 20-character rendering to 19, but the
    epoch parse keeps at most 10 digits of seconds (the digits after them are the fraction, and a number past int64
    reads as INT64_MAX), so even epochs of 14, 19 and 31 digits stay below 10^17 and render in full."""
    vals = [b"[%d]" % ac.BIG_EPOCH, b"[1999999999999999999]", b"[19999999999999999999]", b"[1" + b"9" * 30 + b"]",
            b"[1999999999]"]
    from tests.emul import timestamp as ets
    for v in vals:
        base, off, ln, grp = ets.layout([[v + b"\tk:v"]])
        micro = int(oap.process("content", 0, base, off, ln, grp, 0, -1)[3][0])
        assert 0 < micro < 10 ** 17, (v, micro)
        want, wctr = _check(v + b"\tk:v", ac.config("content"), None, 0, 1700000000, None, di=-1)
        assert orc._sls_pair(0x12, b"microtime", b"%d" % micro) in want
        assert wctr == [0, 0, 0, 0, 1]


@pytest.mark.parametrize("seed", range(4))
def test_multiline_records_with_stack_traces(seed, zone):
    val = ac.ml_value(seed, 25) + b"\n" + b"\n".join(ac.special_lines())
    for acfg in (ac.config("content", "raw", True, True, True), ac.config("content", None, False, False),
                 ac.config("content", "__raw_log__", True, False, True)):
        for okey in (None, OKEY):
            _check(val, acfg, okey, 1 << 20, 1700000000, 7, ml=True)


@pytest.mark.parametrize("tz", ["GMT+08:00", "GMT-03:30"])
def test_timezone_adjustment(tz, zone):
    val = ac.random_value(99)
    acfg = ac.config("content", None, True, False, False, tz=tz)
    _check(val, acfg, OKEY, 5, 1700000000, 3)


def test_refusals():
    acfg = ac.config("content", "raw")
    with pytest.raises(emul.Refused, match="offset key equals SourceKey"):
        _run(b"[1700000000]", acfg, b"content", 0, 1, None, True, 1)
    with pytest.raises(emul.Refused, match="source time_ns needs enable_ns"):
        off, ln = orc.split_lines(b"x", 10)
        emul.serialize(b"x", off, ln, b"content", 0, ac.NOW, -1, b"raw", 0, 0, 0, None, 0, 1, 5, False)


def test_oracle_counters_use_the_issue_order():
    """the oracle's counters agree with lc_apsara_parse's over the same pieces packed back to back"""
    val = ac.random_value(3)
    off, ln = orc.split_lines(val, 10)
    vals = [val[o:o + n] for o, n in zip(off.tolist(), ln.tolist())]
    from tests.emul import timestamp as ets
    base, o2, l2, grp = ets.layout([vals])
    cnt = oap.process("content", 0, base, o2, l2, grp, ac.NOW, ac.DI)[6]
    _, wctr, _, _ = ac.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, ac.config("content", None, True),
                                    1 << 29, None, 0)
    assert wctr == [int(x) for x in cnt]
    assert isinstance(np.uint64(cnt[4]), np.uint64)
