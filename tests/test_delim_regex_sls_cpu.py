"""CPU tier: the delimiter -> regex -> SLS chain's per-row functions (lc_exec.cuh: the tap rule and
lc_delim_regex_sls_body, built for the host by tests/emul/delim_regex_sls.py, with the oracle's matcher as the regex
stage over the tapped values) against the oracle's ProcessorParseDelimiterNative + ProcessorParseRegexNative +
sls_serialize_logs, over the separator x overflow-treatment matrix with random regex stages on top."""
import random

import pytest

from tests import delim_regex_sls_cases as drc
from tests import delim_sls_cases as dc
from tests import regex_sls_cases as rc
from tests.emul import delim_regex_sls

CASES = list(dc.all_cases(seed_base=3, per=4))


def _check(dcfg, rcfg, lines, times, nss, lanes=(1, 3, 32)):
    buf, off, ln = dc.arena(lines)
    want, wctr = drc.oracle_wire(lines, dcfg, rcfg, times, nss, True)
    for nlanes in lanes:
        got, ctr, _, _ = delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, times, nss, nlanes)
        assert got == want, (dcfg, rcfg, nlanes)
        assert drc.fold(ctr) == wctr, (dcfg, rcfg)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_chain_matches_oracle(case):
    _, dcfg, rng = case
    accepted = 0
    for _ in range(12):
        rcfg = drc.random_regex(rng, dcfg)
        lines = [dc.random_line(rng, dcfg["sep"], dcfg["quote"], wide=rng.random() < 0.05) for _ in range(80)]
        times, nss = dc.times_for(len(lines), rng.randint(0, 1 << 30))
        buf, off, ln = dc.arena(lines)
        if drc.refused(dcfg, rcfg):
            with pytest.raises(delim_regex_sls.Refused):
                delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, times, nss)
            continue
        accepted += 1
        _check(dcfg, rcfg, lines, times, nss)
        want_nons, _ = drc.oracle_wire(lines, dcfg, rcfg, times, None, False)
        assert delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, times, None)[0] == want_nons


def _dcfg(treatment="extend", keys=("a", "b", "c"), source="content", renamed=None, kf=True, ks=True, cr=True,
          allow_short=True, max_fields=5, sep=b",", quote=ord('"')):
    return {"sep": sep, "quote": quote, "treatment": treatment, "keys": list(keys), "source": source,
            "renamed": renamed, "keep_fail": kf, "keep_succeed": ks, "copy_raw": cr, "allow_short": allow_short,
            "max_fields": max_fields}


LINES = [b'x,"p""q",z', b'x,"pq",z', b"x,y", b"x", b"", b"  ", b'"open,1', b'x,"a""b""c",z,w,v,u',
         b'ab"c,1,2', b'x,"",z']


@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("rkeys,regex,renamed", [
    (["r1", "r2"], drc.PAT_QUOTE, None),
    (["b", "r2"], drc.PAT_QUOTE, None),          # a regex key equal to k: the capture replaces k in place
    (["r1", "b", "b"], drc.PAT_QUOTE, "raw"),     # repeated
    (["r1", "r1"], drc.PAT_WORD, "b"),
    ([], drc.WHOLE_LINE, None),
    (["b"], drc.WHOLE_LINE, "raw"),
    (["r1"], drc.WHOLE_LINE, None),
])
def test_quoted_column_flag_matrix(flags, rkeys, regex, renamed):
    """column 1 with and without doubled quotes, every keep / copy flag of the regex stage"""
    # (the delimiter's own __raw_log__ or "content" would refuse CopingRawLog / whole-line mode without keys)
    dcfg = _dcfg(source="src", cr=False)
    rcfg = rc.config(rkeys, "b", renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4), regex=regex)
    times, nss = dc.times_for(len(LINES), flags)
    _check(dcfg, rcfg, LINES, times, nss)


def test_collapsed_bytes_reach_the_regex():
    """the tap hands the regex the unquoted column: `p"q` parses to (p, q), where the raw span `p""q` would not"""
    dcfg = _dcfg()
    rcfg = rc.config(["r1", "r2"], "b", None, regex=drc.PAT_QUOTE)
    buf, off, ln = dc.arena([b'x,"p""q",z'])
    got, ctr, (vo, vl), side = delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, [1], None)
    assert side == b'p"q' and int(vl[0]) == 3
    assert b"\x0a\x02r1\x12\x01p" in got and b"\x0a\x02r2\x12\x01q" in got
    want, _ = drc.oracle_wire([b'x,"p""q",z'], dcfg, rcfg, [1], None)
    assert got == want


@pytest.mark.parametrize("dsrc,dren,dflags", [
    ("b", None, (True, True, True)),          # SourceKey is key k: short and blank rows keep the line under k
    ("content", "b", (True, True, False)),    # RenamedSourceKey is key k: kept failures and short rows
    ("content", "b", (False, True, False)),
    ("content", None, (True, False, True)),
])
def test_value_is_the_whole_line(dsrc, dren, dflags):
    dcfg = _dcfg(keys=("a", "b", "__raw_log__"), source=dsrc, renamed=dren, kf=dflags[0], ks=dflags[1],
                 cr=dflags[2])
    for rsrc in ("b", "__raw_log__"):
        for f in range(8):
            rcfg = rc.config(["r1", "r2"], rsrc, None, bool(f & 1), bool(f & 2), bool(f & 4), regex=drc.PAT_QUOTE)
            if drc.refused(dcfg, rcfg):
                continue
            times, nss = dc.times_for(len(LINES), f)
            _check(dcfg, rcfg, LINES, times, nss, lanes=(1, 32))


def test_rows_wider_than_the_tables():
    rng = random.Random(11)
    for sep in (b",", b"|#"):
        for tr in dc.TREATMENTS:
            dcfg = _dcfg(treatment=tr, keys=("a", "b"), sep=sep, max_fields=3, cr=False)
            rcfg = rc.config(["r1", "r2"], "b", None, True, True, True, regex=drc.PAT_QUOTE)
            lines = [dc.random_line(rng, sep, ord('"'), wide=True) for _ in range(30)] + [sep * 300]
            times, nss = dc.times_for(len(lines), 4)
            _check(dcfg, rcfg, lines, times, nss, lanes=(1, 32))


@pytest.mark.parametrize("dcfg,rcfg,why", [
    (_dcfg(), rc.config(["r1"], "zz"), "not one of the delimiter"),
    (_dcfg(treatment="discard", keys=("a", "_")), rc.config(["r1"], "_"), "not one of the delimiter"),
    (_dcfg(), rc.config(["a"], "b"), "names a content"),
    (_dcfg(), rc.config(["content"], "b"), "names a content"),
    (_dcfg(renamed="ren"), rc.config(["ren"], "b"), "names a content"),
    (_dcfg(), rc.config(["r1"], "b", keep_fail=True, copy_raw=True), "names a content"),
    (_dcfg(), rc.config(["__column4__"], "b"), "names a content"),
    (_dcfg(), rc.config(["r1"], "b", renamed="c", keep_succeed=True), "names a content"),
    (_dcfg(), rc.config(["r1"], "b", regex=drc.WHOLE_LINE), None),
    (_dcfg(), rc.config([], "b", regex=drc.WHOLE_LINE), "names a content"),
    (_dcfg(keys=("_time_", "_source_", "b")), rc.config(["r1"], "b"), "_time_"),
])
def test_refused_configurations(dcfg, rcfg, why):
    assert drc.refused(dcfg, rcfg) == (why is not None)
    buf, off, ln = dc.arena([b"1,2,3"])
    if why is None:
        delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, [1], None)
        return
    with pytest.raises(delim_regex_sls.Refused, match=why):
        delim_regex_sls.serialize(buf, off, ln, dcfg, rcfg, [1], None)


def test_repeated_and_overlapping_events_get_their_own_copies():
    """the same quoted line several times and overlapping spans: every row has its own side slot"""
    line = b'x,"p""q""r",z'
    buf = line + b"\n"
    off = [0, 0, 0, 2, 0]
    ln = [len(line), len(line), len(line), len(line) - 2, len(line)]
    lines = [buf[o:o + n] for o, n in zip(off, ln)]
    dcfg = _dcfg()
    rcfg = rc.config(["r1", "r2"], "b", None, regex=drc.PAT_QUOTE)
    import numpy as np
    got, ctr, (vo, vl), side = delim_regex_sls.serialize(np.frombuffer(buf, np.uint8), np.array(off, np.uint32),
                                                         np.array(ln, np.uint32), dcfg, rcfg, [1] * 5, None)
    want, wctr = drc.oracle_wire(lines, dcfg, rcfg, [1] * 5, None)
    assert got == want and drc.fold(ctr) == wctr
    assert side.count(b'p"q"r') == 4 and len(set(vo[[0, 1, 2, 4]].tolist())) == 4
