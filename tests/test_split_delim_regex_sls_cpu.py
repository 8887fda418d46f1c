"""CPU tier: the split -> delimiter -> regex chain's per-row functions (lc_exec.cuh: lc_split_delim_regex_sls_link, the
tap rule over the piece tables, lc_split_delim_regex_sls_body over lc_delim_sls_body and lc_split_delim_regex_verdict,
built for the host by tests/emul/split_delim_regex_sls.py), fed the oracle's split_lines / multiline_split,
delim_parse_batch and regex_parse_batch tables, against the oracle's splitter + ProcessorParseDelimiterNative +
ProcessorParseRegexNative + sls_serialize_logs on one flat source event, with 1, 3 and 32 emulated lanes: bytes and
counters."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import delim_regex_sls_cases as drc
from tests import delim_sls_cases as dc
from tests import regex_sls_cases as rc
from tests import split_delim_regex_sls_cases as sdrc
from tests import split_delim_sls_cases as sdc
from tests import split_sls_cases as sc
from tests.emul import split_delim_regex_sls

OKEY = sdrc.OKEY


def _run(val, dcfg, rcfg, okey, pos, time, ns, nlanes, split_char=10, ml=None, raw_args=None):
    """the emulated chain over the oracle's piece, delimiter and regex tables"""
    off, ln = sdrc.pieces(val, split_char, ml)
    tabs = sdrc.tables(val, off, ln, dcfg)
    return split_delim_regex_sls.serialize(val, off, ln, tabs, dcfg, rcfg, okey, pos, time, ns, nlanes, raw_args)


def _check(val, dcfg, rcfg, okey, pos, time, ns, split_char=10, mcfg=None):
    split_cfg = mcfg or {"SourceKey": dcfg["source"], "SplitChar": split_char}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = sdrc.oracle_chain(val, split_cfg, dcfg, rcfg, time, ns, pos, okey, multiline=mcfg is not None)
    for nlanes in (1, 3, 32):
        got, ctr, _, _ = _run(val, dcfg, rcfg, okey, pos, time, ns, nlanes, split_char, ml)
        assert got == want, (dcfg, rcfg, okey, nlanes)
        assert sdrc.fold(ctr) == wctr, (dcfg, rcfg, okey, list(ctr), wctr)
    if ns is not None:  # Time_ns off: the oracle without ns
        want_nons, _, _, _ = sdrc.oracle_chain(val, split_cfg, dcfg, rcfg, time, None, pos, okey,
                                              multiline=mcfg is not None)
        assert _run(val, dcfg, rcfg, okey, pos, time, None, 1, split_char, ml)[0] == want_nons
    return want


def _check_or_refused(val, dcfg, rcfg, okey, pos, time, ns):
    """the chain as _check does, or -- when the contract refuses it -- the refusal; returns whether it ran"""
    if sdrc.refused(dcfg, rcfg, okey):
        with pytest.raises(split_delim_regex_sls.Refused):
            _run(val, dcfg, rcfg, okey, pos, time, ns, 1)
        return False
    _check(val, dcfg, rcfg, okey, pos, time, ns)
    return True


CASES = list(dc.all_cases(seed_base=11, per=2))


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_matrix_matches_oracle(case, okey):
    """the separator x quote x overflow-treatment matrix (random delimiter keys, source / renamed keys, flags) with
    random regex stages on one of its keys, behind the splitter"""
    cid, dcfg, rng = case
    val = sdc.random_value(rng, dcfg, 50, wide_every=17)
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    ran = 0
    for _ in range(6):
        ran += _check_or_refused(val, dcfg, drc.random_regex(rng, dcfg), okey, sc.POSITIONS[len(cid) % 20], t, ns)
    # and one stage that reads a key every row has, so that each case runs at least once
    ks = drc.delim_keys(dcfg)
    if ks and not ran:
        rcfg = rc.config(["r1", "r2"], ks[0], None, rng.random() < 0.5, False, False, regex=drc.PAT_WORD)
        _check_or_refused(val, dcfg, rcfg, okey, 77, t, ns)


LINES = [b"1,2,3,4,5,6", b"1", b"1,2", b"", b"   ", b'"open,1', b'"x""y",2,3', b"a,b,c,d,e,f,g,h,i,j,k,l",
         b"9,8,7,6,5", b'w1 rest,"q""q",x']


def _corner_regex(dcfg, okey, keep_fail):
    """a regex stage on the first delimiter key that is neither the offset key nor a discarded "_" """
    ks = [k for k in drc.delim_keys(dcfg) if k.encode() != okey]
    return rc.config(["r1", "r2"], ks[0], None, keep_fail, False, False, regex=drc.PAT_WORD)


CORNERS = list(sdc.offset_corners())


@pytest.mark.parametrize("rkeep_fail", [False, True])
@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("name,cfg,okey", CORNERS, ids=[c[0] for c in CORNERS])
def test_offset_key_corners(name, cfg, okey, flags, rkeep_fail):
    """the offset key as a delimiter column every row reaches or short rows do not reach, beside SourceKey, as
    RenamedSourceKey, "__raw_log__" or "_" in discard mode, across the 8 delimiter keep / copy flag combinations and
    both regex KeepingSourceWhenParseFail settings"""
    rng = random.Random(zlib.crc32(name.encode()) + flags)
    dcfg = sdc.with_flags(cfg, flags)
    sep = cfg["sep"]
    val = b"\n".join(ln.replace(b",", sep) for ln in LINES) + b"\n" + sdc.random_value(rng, dcfg, 30)
    rcfg = _corner_regex(dcfg, okey, rkeep_fail)
    assert _check_or_refused(val, dcfg, rcfg, okey, 987654321, 1 << 29, 11) or sdrc.refused(dcfg, rcfg, okey)


@pytest.mark.parametrize("okey", [None, OKEY])
@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("where", ["source", "renamed", "quoted", "short_column"])
def test_regex_source_placements(where, flags, okey):
    """the regex SourceKey as the delimiter's SourceKey, as its RenamedSourceKey, as a quoted column with doubled
    quotes (side copies), and as a column short rows do not reach"""
    dcfg = {
        "source": sdc.config(["a", "content", "c"]),
        "renamed": sdc.config(["a", "b", "c"], renamed="b"),
        "quoted": sdc.config(["q", "b", "c"]),
        "short_column": sdc.config(["a", "b", "c", "d", "e"]),
    }[where]
    dcfg = sdc.with_flags(dcfg, flags)
    src = {"source": "content", "renamed": "b", "quoted": "q", "short_column": "e"}[where]
    rng = random.Random(flags)
    lines = LINES + [b'"a""b""c",x,y', b'"""",1', b'"p" q,1', b'  ,  ', b"x,y,z,w,e1 tail"]
    val = b"\n".join(lines + [dc.random_line(rng, b",", ord('"')) for _ in range(30)])
    for regex in (drc.PAT_QUOTE, drc.PAT_WORD, drc.WHOLE_LINE):
        for rkeep_fail in (False, True):
            keys = ["r1"] if regex == drc.WHOLE_LINE else ["r1", "r2"]
            rcfg = rc.config(keys, src, "raw" if rkeep_fail else None, rkeep_fail, flags & 2 != 0, flags & 4 != 0,
                             regex=regex)
            _check_or_refused(val, dcfg, rcfg, okey, 1 << 40, 1700000000, 5)


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
def test_regex_failure_leaving_only_the_offset_content(okey):
    """a regex failure without KeepingSourceWhenParseFail erases a piece whose only other content was key k: with the
    offset content left alone (ShouldEraseEvent), as without it; with KeepingSourceWhenParseFail it stays"""
    lines = [b"abc", b"/p?k=1", b"", b"x y", b"/q?k=zz", b"  "]
    val = b"\n".join(lines) + b"\n"
    dcfg = sdc.config(["url"], keep_fail=True)
    for rkeep_fail in (False, True):
        _check(val, dcfg, sdrc.c4_regex(keep_fail=rkeep_fail), okey, 12345, 1 << 30, 9)
    # the delimiter's SourceKey overwritten by key k: the blank piece keeps its line under key k
    dcfg = sdc.config(["content"], keep_fail=True)
    for rkeep_fail in (False, True):
        _check(val, dcfg, rc.config(["r1"], "content", None, rkeep_fail, False, False, regex=drc.PAT_WORD), okey,
               12345, 1 << 30, None)
    # another content left besides the offset content: kept
    dcfg = sdc.config(["url", "b"], keep_fail=False)
    _check(val.replace(b"\n", b",1\n"), dcfg, sdrc.c4_regex(), okey, 12345, 1 << 30, None)


@pytest.mark.parametrize("okey", [None, OKEY])
@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_whole_line_mode(nkeys, okey):
    rng = random.Random(nkeys)
    # (SourceKey "src": without regex keys the whole line goes to "content", which must not be a delimiter content)
    dcfg = sdc.config(["a", "b", "c"], source="src", keep_succeed=True, renamed="raw")
    rcfg = rc.config(["w%d" % i for i in range(nkeys)], "b", None, False, False, False, regex=drc.WHOLE_LINE)
    if nkeys == 2:
        rcfg["keys"] = ["b", "w1"]  # the first key overwrites key k in place
    _check(sdc.random_value(rng, dcfg, 40), dcfg, rcfg, okey, 99, 5, 17)


@pytest.mark.parametrize("split_char", [10, 0, ord(";")])
def test_blank_and_empty_pieces(split_char):
    rng = random.Random(split_char)
    dcfg = sdc.config(["a", "content", "c"], renamed="raw", keep_fail=True, keep_succeed=True, copy_raw=True)
    lines = [dc.random_line(rng, b",", ord('"')).replace(bytes([split_char]), b"") for _ in range(30)]
    lines += [b"", b"", b"   ", b"x,1"]
    for trailing in (False, True):
        val = bytes([split_char]).join(lines) + (bytes([split_char]) if trailing else b"")
        for okey in (None, OKEY):
            for rkeep_fail in (False, True):
                rcfg = rc.config(["r1", "r2"], "content", None, rkeep_fail, False, False, regex=drc.PAT_WORD)
                _check(val, dcfg, rcfg, okey, 10 ** 12, 5, 123, split_char=split_char)
    _check(bytes([split_char]), dcfg, rcfg, OKEY, 0, 5, None, split_char=split_char)


@pytest.mark.parametrize("name", ["start", "start_cont", "end"])
def test_multiline_pieces_with_quoted_newlines(name):
    """multiline records whose quoted CSV fields hold the split char, the regex on a quoted column"""
    rng = random.Random(zlib.crc32(name.encode()))
    mcfg = sc.ml_config(name)
    recs = []
    for i in range(25):
        head = {"start": b"2024-01-0%d 10:00:0%d" % (rng.randint(1, 9), rng.randint(0, 9)),
                "start_cont": b"line %d" % i, "end": b"x%d" % i}[name]
        body = b',"a\nb",c,"d""\ne"' if name != "start_cont" else b"\ncontinue,\"q\"\ncontinue 2,x"
        tail = b"\nendLine %d" % i if name == "end" else b""
        recs.append(head + b"," + body + tail + (b"\nstray,1" if rng.random() < 0.3 else b""))
    val = b"\n".join(recs)
    for tr in dc.TREATMENTS:
        dcfg = sdc.config(["t", "b", "c", "d"], treatment=tr, renamed="raw", keep_succeed=True)
        for src in ("b", "d"):
            rcfg = rc.config(["r1", "r2"], src, None, src == "d", False, False, regex=drc.PAT_QUOTE)
            _check(val, dcfg, rcfg, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
def test_c4_csv_lines(okey):
    from loongcollector_b200 import synth
    buf, _, _ = synth.csv_lines(400)
    dcfg = sdc.config(synth.CSV_KEYS, max_fields=11)
    val = buf.tobytes()
    _check(val, dcfg, sdrc.c4_regex(), okey, 4096, 1700000000, None)
    _check(val, dcfg, sdrc.c4_regex(keep_fail=True, keep_succeed=True, copy_raw=True, renamed="raw_url"), okey, 4096,
           1700000000, 3)


# (delimiter cfg, regex cfg, offset key, the reason's words)
REFUSALS = [
    ("offset_is_regex_source", sdc.config(["a", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD), b"b",
     "offset key equals the regex SourceKey"),
    ("offset_is_regex_key", sdc.config(["a", "b"]), rc.config(["r", "off"], "b", regex=drc.PAT_WORD), b"off",
     "names a content"),
    ("offset_is_whole_line_key", sdc.config(["a", "b"]), rc.config(["off"], "b", regex=drc.WHOLE_LINE), b"off",
     "names a content"),
    ("offset_is_regex_renamed", sdc.config(["a", "b"]), rc.config(["r"], "b", "off", True, regex=drc.PAT_WORD), b"off",
     "names a content"),
    ("offset_is_regex_raw_log", sdc.config(["a", "b"]),
     rc.config(["r"], "b", "x", True, False, True, regex=drc.PAT_WORD), b"__raw_log__", "names a content"),
    ("offset_with_source_time_rule", sdc.config(["_source_", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD),
     b"_time_", "_time_ and _source_"),
    ("offset_is_delimiter_source", sdc.config(["a", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD), b"content",
     "offset key equals SourceKey"),
    ("offset_column_form", sdc.config(["a", "b"]), rc.config(["r"], "b", regex=drc.PAT_WORD), b"__column4__",
     "__column"),
    ("regex_source_not_a_column", sdc.config(["a", "b"]), rc.config(["r"], "zz", regex=drc.PAT_WORD), OKEY,
     "not one of the delimiter's keys"),
    ("regex_key_is_a_column", sdc.config(["a", "b"]), rc.config(["a"], "b", regex=drc.PAT_WORD), OKEY,
     "names a content"),
]


@pytest.mark.parametrize("name,dcfg,rcfg,okey,why", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals(name, dcfg, rcfg, okey, why):
    assert sdrc.refused(dcfg, rcfg, okey)
    with pytest.raises(split_delim_regex_sls.Refused, match=why):
        _run(b"x,1", dcfg, rcfg, okey, 0, 1, None, 1)


def test_offset_key_is_no_regex_content_without_an_offset():
    """the same names are accepted when the group has no offset metadata"""
    for _name, dcfg, rcfg, okey, _why in REFUSALS[:6]:
        assert not sdrc.refused(dcfg, rcfg, None)
        _check(b"1,w x\n2\n\n,\n3,\"y\"\"z\"", dcfg, rcfg, None, 5, 1 << 29, None)


def test_c_abi_refuses_bad_arguments_without_a_device():
    """argument checks come before the engine is touched"""
    import loongcollector_b200 as lc
    L = lc.lib()
    n, nev = C.c_uint64(0), C.c_uint64(0)
    ctr = np.zeros(8, np.uint64)
    keys = (C.c_char_p * 1)(b"a")
    kl = np.array([1], np.uint32)
    sep = np.frombuffer(b",", np.uint8)
    pk = [C.cast(keys, C.c_void_p), kl.ctypes.data_as(C.c_void_p)]
    chain = [sep.ctypes.data_as(C.c_void_p), 1, ord('"'), 1, 0, *pk, 1, b"content", 7, b"content", 7, 0, 0, 0,
             *pk, 1, b"a", 1, b"a", 1, 0, 0, 0, 1, OKEY, len(OKEY), 0, 0, 0xFFFFFFFF]
    p = ctr.ctypes.data_as(C.c_void_p)
    assert L.lc_sls_serialize_split_delim_regex_dev(None, None, 0, None, None, 0, None, None, None, None, None, 4,
                                                    *chain, None, None, None, None, None, 0, None, 0, C.byref(n),
                                                    p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_split_delim_regex_parse_sls(None, None, None, 0, 10, 1, 4, *chain, None, 0, C.byref(n), C.byref(nev),
                                            p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_split_delim_regex_parse_sls_lz4(None, None, None, 0, 10, 1, 4, *chain, None, 0, None, 0, C.byref(n),
                                                C.byref(nev), C.byref(nev), p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_multiline_split_delim_regex_parse_sls(None, None, None, 0, None, None, None, 0, 1, 4, *chain, None, 0,
                                                      C.byref(n), C.byref(nev), p, None) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_multiline_split_delim_regex_parse_sls_lz4(None, None, None, 0, None, None, None, 0, 1, 4, *chain,
                                                          None, 0, None, 0, C.byref(n), C.byref(nev), C.byref(nev), p,
                                                          None) == lc.capi.LC_ERR_INVALID_ARG
