"""CPU tier: the split -> regex chain's per-row function and content plans (lc_exec.cuh: lc_split_regex_sls_setup,
lc_regex_sls_plans and lc_split_regex_sls_body, built for the host by tests/emul/split_regex_sls.py), fed the oracle's
split_lines / multiline_split and regex_parse_batch tables, against the oracle's splitter + ProcessorParseRegexNative
+ sls_serialize_logs on one flat source event, with 1, 3 and 32 emulated lanes: bytes and counters."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import regex_sls_cases as rc
from tests import split_regex_sls_cases as src
from tests import split_sls_cases as sc
from tests.emul import split_regex_sls

OKEY = src.OKEY


def _run(val, cfg, okey, pos, time, ns, nlanes, split_char=10, ml=None, raw_args=None):
    """the emulated chain over the oracle's piece and regex tables"""
    if ml is None:
        off, ln = orc.split_lines(val, split_char)
    else:
        off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    tables, pitch = None, 0
    if not rc.whole_line(cfg) and off.size:
        st, co, cl, pitch = rc.parse_tables(np.frombuffer(val, np.uint8), off, ln, cfg)
        tables = (st, co, cl)
    return split_regex_sls.serialize(val, off, ln, tables, pitch, [k.encode() for k in cfg["keys"]],
                                     cfg["source"].encode(), rc.renamed_key(cfg), cfg["keep_fail"],
                                     cfg["keep_succeed"], cfg["copy_raw"], rc.whole_line(cfg), okey, pos, time, ns,
                                     nlanes, raw_args)


def _check(val, cfg, okey, pos, time, ns, split_char=10, mcfg=None):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": split_char}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = src.oracle_chain(val, split_cfg, cfg, time, ns, pos, okey, multiline=mcfg is not None)
    for nlanes in (1, 3, 32):
        got, ctr = _run(val, cfg, okey, pos, time, ns, nlanes, split_char, ml)
        assert got == want, (cfg, okey, nlanes)
        assert ctr == wctr, (cfg, okey, ctr, wctr)
    if ns is not None:  # Time_ns off: the oracle without ns
        want_nons, _, _, _ = src.oracle_chain(val, split_cfg, cfg, time, None, pos, okey, multiline=mcfg is not None)
        assert _run(val, cfg, okey, pos, time, None, 1, split_char, ml)[0] == want_nons


MATRIX = list(src.matrix())


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
@pytest.mark.parametrize("case", MATRIX, ids=[c[0] for c in MATRIX])
def test_matrix_matches_oracle(case, okey):
    cid, cfg = case
    rng = random.Random(zlib.crc32(cid.encode()))
    val = src.random_lines_value(rng, 50)
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _check(val, cfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns)


@pytest.mark.parametrize("okey", [b"a", b"raw", b"__raw_log__", b"content2"])
@pytest.mark.parametrize("flags", range(8))
def test_offset_key_equal_to_regex_contents(okey, flags):
    """a regex key equal to the offset key overwrites the digits in place; a RenamedSourceKey or __raw_log__ equal to
    it is not added; a failure without KeepingSourceWhenParseFail is erased although the offset content is left"""
    rng = random.Random(flags)
    val = src.random_lines_value(rng, 40, trailing=True)
    for renamed in ("raw", "__raw_log__"):
        cfg = rc.config(["a", "raw", "c"], "content", renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4))
        _check(val, cfg, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("renamed", ["content", OKEY.decode(), "__raw_log__", "other"])
@pytest.mark.parametrize("flags", range(8))
def test_renamed_source_key(renamed, flags):
    rng = random.Random(100 + flags)
    val = src.random_lines_value(rng, 40)
    cfg = rc.config(["a", "b", "c"], "content", renamed, bool(flags & 1), bool(flags & 2), bool(flags & 4))
    for okey in (None, OKEY):
        _check(val, cfg, okey, 5, 3, None)


@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_whole_line_mode(nkeys):
    keys = [OKEY.decode(), "content"][:nkeys]
    for f in range(8):
        cfg = rc.config(keys, "content", None, bool(f & 1), bool(f & 2), bool(f & 4), regex=rc.WHOLE_LINE)
        for okey in (None, OKEY, b""):
            _check(b"a 1 b\n\nxyz\n", cfg, okey, 77, (1 << 28) - 1, 5)


@pytest.mark.parametrize("split_char", [10, 0, ord(";")])
def test_empty_pieces_trailing_and_other_split_chars(split_char):
    rng = random.Random(split_char)
    lines = [rc.random_line(rng) for _ in range(30)] + [b"", b"", b"x 1 "]
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, True)
    for trailing in (False, True):
        val = bytes([split_char]).join(lines) + (bytes([split_char]) if trailing else b"")
        for okey in (None, OKEY):
            _check(val, cfg, okey, 10 ** 12, 5, 123, split_char=split_char)
    _check(bytes([split_char]), cfg, OKEY, 0, 5, None, split_char=split_char)


@pytest.mark.parametrize("pos", sc.POSITIONS)
def test_offsets_across_digit_counts(pos):
    cfg = rc.config(["a", "b", "c"], "content", None, True, False, True)
    _check(src.random_lines_value(random.Random(1), 20), cfg, OKEY, pos, 1 << 30, None)


@pytest.mark.parametrize("name", list(sc.ML_CFGS))
def test_multiline_pieces(name):
    rng = random.Random(zlib.crc32(name.encode()))
    val = sc.ml_value(rng, 12)
    mcfg = sc.ml_config(name)
    cfg = rc.config(["a", "b", "c"], "content", "raw", True, True, False, regex=r"(\w+)\s(\d+)(.*)")
    _check(val, cfg, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


def test_java_records_with_the_record_regex():
    from loongcollector_b200 import synth
    buf, _, _ = synth.java_stack_records(200)
    mcfg = {"SourceKey": "content", "StartPattern": synth.JAVA_START_PATTERN, "ContinuePattern": r"\s+at\s.*"}
    cfg = rc.config(src.RECORD_KEYS, "content", None, True, False, False, regex=src.RECORD_PATTERN)
    _check(buf.tobytes(), cfg, OKEY, 4096, 1700000000, None, mcfg=mcfg)


def test_refusals():
    cfg = rc.config(["a", "b"], "content", "raw")
    with pytest.raises(split_regex_sls.Refused, match="offset key equals SourceKey"):
        _run(b"x 1 y", cfg, b"content", 0, 1, None, 1)
    empty = rc.config(["a", "b"], "", "raw")
    with pytest.raises(split_regex_sls.Refused, match="offset key equals SourceKey"):
        _run(b"x 1 y", empty, b"", 0, 1, None, 1)
    # keys, key_lens, source_key (non-zero length), renamed_key (non-zero length), offset_key with a length
    for arg, value in ((8, None), (9, None), (11, None), (13, None)):
        with pytest.raises(split_regex_sls.Refused, match="bad arguments"):
            _run(b"x 1 y", cfg, OKEY, 0, 1, None, 1, raw_args={arg: value})


def test_c_abi_refuses_bad_arguments_without_a_device():
    """argument checks come before the engine is touched"""
    import loongcollector_b200 as lc
    L = lc.lib()
    n, nev = C.c_uint64(0), C.c_uint64(0)
    ctr = np.zeros(3, np.uint64)
    keys = (C.c_char_p * 1)(b"a")
    kl = np.array([1], np.uint32)
    cfg = [C.cast(keys, C.c_void_p), kl.ctypes.data_as(C.c_void_p), 1, b"content", 7, b"content", 7, 0, 0, 0, 0,
           OKEY, len(OKEY), 0, 0, 0xFFFFFFFF]
    p = ctr.ctypes.data_as(C.c_void_p)
    assert L.lc_sls_serialize_split_regex_dev(None, None, 0, None, None, 0, None, None, None, 1, *cfg, None, 0,
                                              C.byref(n), p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_split_regex_parse_sls(None, None, None, 0, 10, *cfg, None, 0, C.byref(n), C.byref(nev),
                                      p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_multiline_split_regex_parse_sls(None, None, None, 0, None, None, None, 0, *cfg, None, 0, C.byref(n),
                                                C.byref(nev), p, None) == lc.capi.LC_ERR_INVALID_ARG
