"""CPU tier: the regex-fed SLS serialiser's per-row function and content plans (lc_exec.cuh: lc_regex_sls_setup +
lc_regex_sls_body, built for the host by tests/emul/regex_sls.py) against the oracle's ProcessorParseRegexNative +
sls_serialize_logs on seeded flat groups, with 1, 3 and 32 emulated lanes: bytes and counters."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from tests import regex_sls_cases as rc
from tests.emul import regex_sls


def _run(cfg, lines, times, nss, nlanes, **kw):
    buf, off, ln = rc.arena(lines)
    tables, pitch = None, 0
    if not rc.whole_line(cfg):
        st, co, cl, pitch = rc.parse_tables(buf, off, ln, cfg)
        tables = (st, co, cl)
    return regex_sls.serialize(buf, off, ln, tables, pitch, [k.encode() for k in cfg["keys"]], cfg["source"].encode(),
                               rc.renamed_key(cfg), cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"],
                               rc.whole_line(cfg), times, nss, nlanes, **kw)


def _check(cfg, lines, seed):
    times, nss = rc.times_for(len(lines), seed)
    want, ctr, _ = rc.oracle_wire(lines, cfg, times, nss, True)
    for nlanes in (1, 3, 32):
        got, c = _run(cfg, lines, times, nss, nlanes)
        assert got == want, (cfg, nlanes)
        assert c == rc.counters_of(ctr), (cfg, c, ctr)
    want_nons, _, _ = rc.oracle_wire(lines, cfg, times, None, False)
    assert _run(cfg, lines, times, None, 1)[0] == want_nons


MATRIX = list(rc.matrix())


@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_matrix_matches_oracle(case):
    _, cfg = case
    rng = random.Random(zlib.crc32(case[0].encode()))
    lines = [rc.random_line(rng) for _ in range(120)] + [b"", b"x 1 ", b" 7 ", b"nomatch"]
    _check(cfg, lines, rng.randint(0, 1 << 30))


WHOLE = list(rc.whole_line_matrix())


@pytest.mark.parametrize("case", WHOLE, ids=[c[0] for c in WHOLE])
def test_whole_line_mode_matches_oracle(case):
    _, cfg = case
    rng = random.Random(3)
    _check(cfg, [rc.random_line(rng) for _ in range(40)] + [b""], 4)


RANDOM = list(rc.random_cases(1, 24))


@pytest.mark.parametrize("case", RANDOM, ids=[c[0] for c in RANDOM])
def test_random_configurations_match_oracle(case):
    _, cfg, rng = case
    _check(cfg, [rc.random_line(rng) for _ in range(100)], rng.randint(0, 1 << 30))


def test_whole_line_without_keys_empties_the_content_event():
    """Keys [] + SourceKey content: "content" gets the line, then the source (the same key) is deleted -- the event
    ends up empty and emits nothing, but it is not erased"""
    cfg = rc.config([], "content", regex=rc.WHOLE_LINE)
    times, _ = rc.times_for(3, 1)
    got, c = _run(cfg, [b"a", b"", b"bc"], times, None, 1)
    assert got == b"" and c == [3, 0, 0]


def test_pattern_without_groups():
    cfg = rc.config([], "content", "raw", True, True, True, regex=r"\d+")
    _check(cfg, [b"12", b"", b"x", b"007"], 9)


@pytest.mark.parametrize("arg,value", [(8, None), (9, None), (11, None), (13, None)],
                         ids=["keys", "key_lens", "source_key", "renamed_key"])
def test_refused_arguments(arg, value):
    cfg = rc.config(["a", "b"], "content", "raw")
    with pytest.raises(regex_sls.Refused, match="bad arguments"):
        _run(cfg, [b"x 1 y"], [1], None, 1, raw_args={arg: value})


def test_c_abi_refuses_bad_arguments_without_a_device():
    """argument checks come before the engine is touched"""
    import loongcollector_b200 as lc
    L = lc.lib()
    n = C.c_uint64(0)
    ctr = np.zeros(3, np.uint64)
    keys = (C.c_char_p * 1)(b"a")
    kl = np.array([1], np.uint32)
    cfg = [C.cast(keys, C.c_void_p), kl.ctypes.data_as(C.c_void_p), 1, b"content", 7, b"content", 7, 0, 0, 0]
    assert L.lc_sls_serialize_regex_dev(None, None, 0, None, None, 0, None, None, None, 1, *cfg, 0, None, None, None,
                                        0, C.byref(n), ctr.ctypes.data_as(C.c_void_p)) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_regex_parse_sls(None, None, None, 0, None, None, 0, None, None, *cfg, 0, None, 0, C.byref(n),
                                ctr.ctypes.data_as(C.c_void_p)) == lc.capi.LC_ERR_INVALID_ARG
