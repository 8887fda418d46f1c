"""CPU tier: the split -> regex -> filter chain's per-row functions (lc_exec.cuh: lc_filter_sls_setup, lc_filter_leaf,
lc_filter_eval and lc_split_regex_sls_body, built for the host by tests/emul/split_regex_filter_sls.py), fed the
oracle's split_lines / multiline_split and regex_parse_batch tables, against the oracle's splitter +
ProcessorParseRegexNative + ProcessorFilterNative + sls_serialize_logs on one flat source event, with 1, 3 and 32
emulated lanes: bytes and counters."""
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import regex_sls_cases as rc
from tests import split_regex_filter_sls_cases as fc
from tests import split_regex_sls_cases as src
from tests import split_sls_cases as sc
from tests.emul import split_regex_filter_sls as emul

OKEY = fc.OKEY


def _run(val, cfg, fcfg, okey, pos, time, ns, nlanes, ml=None, prog=None):
    if ml is None:
        off, ln = orc.split_lines(val, 10)
    else:
        off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    tables, pitch = None, 0
    if not rc.whole_line(cfg) and off.size:
        st, co, cl, pitch = rc.parse_tables(np.frombuffer(val, np.uint8), off, ln, cfg)
        tables = (st, co, cl)
    leaves, p = fc.program(fcfg)
    return emul.serialize(val, off, ln, tables, pitch, [k.encode() for k in cfg["keys"]], cfg["source"].encode(),
                          rc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"],
                          rc.whole_line(cfg), okey, pos, time, ns, [(k, orc.Regex(r)) for k, r in leaves],
                          p if prog is None else prog, nlanes)


def _check(val, cfg, fcfg, okey, pos, time, ns, mcfg=None, lanes=(1, 3, 32)):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": 10}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = fc.oracle_chain(val, split_cfg, cfg, fcfg, time, ns, pos, okey, multiline=mcfg is not None)
    for nlanes in lanes:
        got, ctr = _run(val, cfg, fcfg, okey, pos, time, ns, nlanes, ml)
        assert got == want, (cfg, fcfg, okey, nlanes)
        assert ctr == wctr, (cfg, fcfg, okey, ctr, wctr)
    return want, wctr


MATRIX = list(fc.matrix())


@pytest.mark.parametrize("fid", list(fc.FILTERS))
@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_matrix_matches_oracle(case, fid):
    cid, cfg = case
    rng = random.Random(zlib.crc32((cid + fid).encode()))
    val = src.random_lines_value(rng, 40)
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    pos = sc.POSITIONS[(len(cid) + len(fid)) % len(sc.POSITIONS)]
    for i, okey in enumerate((None, OKEY, b"")):
        _check(val, cfg, fc.FILTERS[fid], okey, pos, t, ns, lanes=(1, 3, 32) if i == 1 else (1,))


@pytest.mark.parametrize("fid", list(fc.FILTERS))
@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_whole_line_mode(fid, nkeys):
    keys = [OKEY.decode(), "content"][:nkeys]
    for f in (0, 3, 5, 7):
        cfg = rc.config(keys, "content", None, bool(f & 1), bool(f & 2), bool(f & 4), regex=rc.WHOLE_LINE)
        for okey in (None, OKEY):
            _check(b"a 1 b\n\nxyz 20\n15\n", cfg, fc.FILTERS[fid], okey, 77, (1 << 28) - 1, 5)


@pytest.mark.parametrize("fid", ["rule_offset", "nested", "rule_source_key"])
@pytest.mark.parametrize("discard", [False, True])
def test_multiline_records(fid, discard):
    from loongcollector_b200 import synth
    buf, _, _ = synth.java_stack_records(60, seed=4)
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*",
            "UnmatchedContentTreatment": "discard" if discard else "single_line"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    _check(buf.tobytes(), cfg, fc.FILTERS[fid], OKEY, 123456, 1700000000, 3, mcfg=mcfg)


def test_every_piece_removed_and_every_piece_kept():
    rng = random.Random(3)
    val = src.random_lines_value(rng, 50)
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, False)
    want, ctr = _check(val, cfg, fc.FILTERS["rule_missing"], OKEY, 5, 9, None)
    assert want == b"" and ctr[3] == ctr[0]  # every piece that reached the filter
    want, ctr = _check(val, cfg, fc.FILTERS["not_missing"], OKEY, 5, 9, None)
    assert want and ctr[3] == 0


def test_bypass_equals_the_unfiltered_chain():
    from tests.emul import split_regex_sls
    rng = random.Random(8)
    val = src.random_lines_value(rng, 60)
    cfg = rc.config([], "content", None, True, False, False)  # parsed pieces without contents
    got, ctr = _run(val, cfg, {}, OKEY, 1, 2, None, 3)
    off, ln = orc.split_lines(val, 10)
    st, co, cl, pitch = rc.parse_tables(np.frombuffer(val, np.uint8), off, ln, cfg)
    want, wctr = split_regex_sls.serialize(val, off, ln, (st, co, cl), pitch, [], b"content", b"content", True,
                                           False, False, False, OKEY, 1, 2, None, 3)
    assert got == want and ctr == wctr + [0]


def test_refusals():
    val = b"a 1 b\nx\n"
    cfg = rc.config(["a", "b", "c"])
    many = {"FilterKey": ["k%d" % i for i in range(33)], "FilterRegex": [".*"] * 33}
    with pytest.raises(emul.Refused, match="too many filter leaves"):
        _run(val, cfg, many, None, 0, 0, None, 1)
    one = {"FilterKey": ["a"], "FilterRegex": [".*"]}
    for prog in ([fc.AND], [0, 0], [0, fc.NOT, fc.OR], [1], [0, 7], [fc.NOT], [0] * 33 + [fc.AND] * 32, [0] * 129):
        with pytest.raises(emul.Refused):
            _run(val, cfg, one, None, 0, 0, None, 1, prog=prog)
    # a deep but valid program is accepted
    deep = [0] * 32 + [fc.AND] * 31
    _run(val, cfg, one, None, 0, 0, None, 1, prog=deep)
