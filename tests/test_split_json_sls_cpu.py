"""CPU tier: the split -> JSON chain's resolve and row functions (lc_exec.cuh: lc_json_resolve_warp,
lc_json_resolve_sort, lc_split_json_sls_body, built for the host by tests/emul/split_json_sls.py), fed the oracle's
split_lines / multiline_split tables and oracle/json_parse.py's tables over those pieces, against the oracle's
splitter + ProcessorParseJsonNative + sls_serialize_logs on one flat source event, with 1, 3 and 32 emulated lanes
and with every key hashed alike: bytes and counters."""
import random
import time as _time

import numpy as np
import pytest

from oracle import json_parse as ojs
from oracle import oracle as orc
from tests import split_json_sls_cases as jsc
from tests import split_sls_cases as sc
from tests.emul import split_json_sls

OKEY = jsc.OKEY


def _pieces(val, split_char=10, ml=None):
    if ml is None:
        return orc.split_lines(val, split_char)
    off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    return off, ln


def _run(val, jcfg, okey, pos, time, ns, nlanes, split_char=10, ml=None, const_hash=False):
    off, ln = _pieces(val, split_char, ml)
    st, first, ent, arena, _ = ojs.process(jcfg["SourceKey"].encode(), np.frombuffer(val, np.uint8), off, ln)
    return split_json_sls.serialize(val, off, ln, (st, first, ent, arena), jcfg["SourceKey"].encode(),
                                    jsc.renamed_key(jcfg), jcfg["KeepingSourceWhenParseFail"],
                                    jcfg["KeepingSourceWhenParseSucceed"], jcfg["CopingRawLog"], okey, pos, time, ns,
                                    nlanes, const_hash)


def _check(val, jcfg, okey, pos, time, ns, split_char=10, mcfg=None, lanes=(1, 3, 32)):
    split_cfg = mcfg or {"SourceKey": jcfg["SourceKey"], "SplitChar": split_char}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = jsc.oracle_chain(val, split_cfg, jcfg, time, ns, pos, okey, multiline=mcfg is not None)
    for nlanes in lanes:
        for const_hash in (False, True):
            got, ctr = _run(val, jcfg, okey, pos, time, ns, nlanes, split_char, ml, const_hash)
            assert got == want, (jcfg, okey, nlanes, const_hash)
            assert ctr == wctr, (jcfg, okey, ctr, wctr)
    if ns is not None:  # Time_ns off
        want_nons, _, _, _ = jsc.oracle_chain(val, split_cfg, jcfg, time, None, pos, okey,
                                              multiline=mcfg is not None)
        assert _run(val, jcfg, okey, pos, time, None, 1, split_char, ml)[0] == want_nons


CONFIGS = [(f"{r}_{i}", c) for r in (None, "raw", "content", "__raw_log__", OKEY.decode())
           for i, c in enumerate(jsc.flag_configs(r))]


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
@pytest.mark.parametrize("case", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_matrix_matches_oracle(case, okey):
    cid, jcfg = case
    val = jsc.random_value(len(cid) * 7 + (0 if okey is None else len(okey) + 1))
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _check(val, jcfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns)


@pytest.mark.parametrize("okey", [b"a", b"raw", b"__raw_log__", b"k1", b"dup"])
@pytest.mark.parametrize("flags", range(8))
def test_offset_key_equal_to_member_or_added_keys(okey, flags):
    """an offset key that is a member key takes the member's last value in place; a RenamedSourceKey or __raw_log__
    equal to it is not added; a failure without KeepingSourceWhenParseFail is erased although the offset is left"""
    lines = jsc.special_lines(okey=okey) + jsc.special_lines(okey=b"a")
    val = b"\n".join(lines)
    for renamed in ("raw", "__raw_log__"):
        jcfg = jsc.config("content", renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4))
        _check(val, jcfg, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("flags", range(8))
def test_empty_object_empty_pieces_and_all_erased(flags):
    jcfg = jsc.config("content", None, bool(flags & 1), bool(flags & 2), bool(flags & 4))
    for val in (b"{}\n{}\n", b"\n\n\n", b"", b"{}", b"x\ny\n\nz", b"{\n}\n"):
        for okey in (None, OKEY):
            _check(val, jcfg, okey, 17, 1700000000, 5)


@pytest.mark.parametrize("n", [2, 33, 100000])
def test_repeats_of_one_key(n):
    val = b"\n".join([jsc.big_doc(n, alike=True), b'{"a":1}', jsc.big_doc(3)])
    _check(val, jsc.config("content", None, True, True), OKEY, 5, 1 << 30, None, lanes=(1, 32))


def test_split_escaped_spellings():
    """duplicates of one key through escaped (arena) and plain (source) spellings, below and above 32 members"""
    lines = [jsc.doc([(jsc.escaped("k%d" % (i % 7)) if i % 2 else '"k%d"' % (i % 7), '"v%d"' % i)
                      for i in range(m)]) for m in (5, 31, 32, 33, 200)]
    for jcfg in jsc.flag_configs("k3"):
        _check(b"\n".join(lines), jcfg, OKEY, 3, 1 << 29, 1)


def test_distinct_keys_with_one_hash_resolve_in_m_log_m():
    """10^5 distinct keys in one event, every key hashed alike: the sort still splits them by bytes; a pairwise
    resolve would take ~5 * 10^9 key comparisons here"""
    val = jsc.big_doc(100000, escaped_every=10) + b"\n" + jsc.big_doc(40)
    jcfg = jsc.config("content", None, False, True)
    want, wctr, _, _ = jsc.oracle_chain(val, {"SourceKey": "content", "SplitChar": 10}, jcfg, 1 << 30, None, 0, OKEY)
    t0 = _time.perf_counter()
    got, ctr = _run(val, jcfg, OKEY, 0, 1 << 30, None, 1, const_hash=True)
    assert _time.perf_counter() - t0 < 20.0
    assert got == want and ctr == wctr


@pytest.mark.parametrize("name", list(sc.ML_CFGS))
def test_multiline_pieces(name):
    rng = random.Random(len(name))
    val = sc.ml_value(rng, 12) + b"\n" + b"\n".join(jsc.special_lines())
    mcfg = sc.ml_config(name)
    for jcfg in (jsc.config("content", "raw", True, True, True), jsc.config("content", None, False, False)):
        _check(val, jcfg, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


def test_other_source_key_and_split_char():
    val = b"\0".join(jsc.special_lines(source="log"))
    for jcfg in jsc.flag_configs("raw", source="log"):
        _check(val, jcfg, OKEY, 99, 1 << 28, 0, split_char=0)


def test_refusals():
    jcfg = jsc.config("content", "raw")
    with pytest.raises(split_json_sls.Refused, match="offset key equals SourceKey"):
        _run(b'{"a":1}', jcfg, b"content", 0, 1, None, 1)
    empty = jsc.config("", "raw")
    with pytest.raises(split_json_sls.Refused, match="offset key equals SourceKey"):
        _run(b'{"a":1}', empty, b"", 0, 1, None, 1)
