"""CPU tier: the split -> delimiter chain's per-row function (lc_exec.cuh: lc_split_delim_sls_link and
lc_split_delim_sls_body over lc_delim_sls_body, built for the host by tests/emul/split_delim_sls.py), fed the oracle's
split_lines / multiline_split and delim_parse_batch tables, against the oracle's splitter +
ProcessorParseDelimiterNative + sls_serialize_logs on one flat source event, with 1, 3 and 32 emulated lanes: bytes and
counters."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

from oracle import oracle as orc
from tests import delim_sls_cases as dc
from tests import split_delim_sls_cases as sdc
from tests import split_sls_cases as sc
from tests.emul import split_delim_sls

OKEY = sdc.OKEY


def _run(val, cfg, okey, pos, time, ns, nlanes, split_char=10, ml=None, raw_args=None):
    """the emulated chain over the oracle's piece and delimiter tables"""
    if ml is None:
        off, ln = orc.split_lines(val, split_char)
    else:
        off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    tabs = sdc.tables(val, off, ln, cfg)
    quote = cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')
    return split_delim_sls.serialize(val, off, ln, tabs, cfg["max_fields"], cfg["sep"], quote, cfg["treatment"],
                                     [k.encode() for k in cfg["keys"]], cfg["source"].encode(), dc.renamed_key(cfg),
                                     cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], okey, pos, time, ns,
                                     nlanes, raw_args)


def _check(val, cfg, okey, pos, time, ns, split_char=10, mcfg=None):
    split_cfg = mcfg or {"SourceKey": cfg["source"], "SplitChar": split_char}
    ml = None
    if mcfg is not None:
        p = orc.ProcessorSplitMultilineLogStringNative(mcfg)
        ml = (p.start, p.cont, p.end, p.opts.discard)
    want, wctr, _, _ = sdc.oracle_chain(val, split_cfg, cfg, time, ns, pos, okey, multiline=mcfg is not None)
    for nlanes in (1, 3, 32):
        got, ctr = _run(val, cfg, okey, pos, time, ns, nlanes, split_char, ml)
        assert got == want, (cfg, okey, nlanes)
        assert sdc.fold(ctr) == wctr, (cfg, okey, ctr, wctr)
    if ns is not None:  # Time_ns off: the oracle without ns
        want_nons, _, _, _ = sdc.oracle_chain(val, split_cfg, cfg, time, None, pos, okey, multiline=mcfg is not None)
        assert _run(val, cfg, okey, pos, time, None, 1, split_char, ml)[0] == want_nons
    return want


CASES = list(dc.all_cases(seed_base=3, per=3))


@pytest.mark.parametrize("okey", [None, OKEY, b""], ids=["no_offset", "offset", "empty_offset_key"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_matrix_matches_oracle(case, okey):
    """delim_sls_cases' separator x treatment matrix (random keys, source / renamed keys, flags) behind the splitter"""
    cid, cfg, rng = case
    val = sdc.random_value(rng, cfg, 60, wide_every=17)
    t, ns = sc.TIMES[len(cid) % len(sc.TIMES)]
    _check(val, cfg, okey, sc.POSITIONS[len(cid) % len(sc.POSITIONS)], t, ns)


CORNERS = list(sdc.offset_corners())


@pytest.mark.parametrize("flags", range(8))
@pytest.mark.parametrize("name,cfg,okey", CORNERS, ids=[c[0] for c in CORNERS])
def test_offset_key_corners(name, cfg, okey, flags):
    """the offset key as a delimiter key (reached by every row or not), beside SourceKey, as RenamedSourceKey,
    "__raw_log__" or "_", across the 8 keep / copy flag combinations"""
    rng = random.Random(zlib.crc32(name.encode()) + flags)
    c = sdc.with_flags(cfg, flags)
    lines = [b"1,2,3,4,5,6", b"1", b"1,2", b"", b"   ", b'"open,1', b'"x""y",2,3', b"a,b,c,d,e,f,g,h,i,j,k,l",
             b"9,8,7,6,5"]
    sep = cfg["sep"]
    val = b"\n".join(ln.replace(b",", sep) for ln in lines) + b"\n" + sdc.random_value(rng, c, 30)
    _check(val, c, okey, 987654321, 1 << 29, 11)


@pytest.mark.parametrize("sep", [b",", b"|#"])
def test_rows_wider_than_the_tables(sep):
    rng = random.Random(7)
    for tr in dc.TREATMENTS:
        for okey in (OKEY, b"b"):
            cfg = sdc.config(["a", "b"], sep=sep, treatment=tr, renamed="__column5__" if tr != "discard" else "r",
                             keep_fail=False, keep_succeed=True, max_fields=3)
            lines = [dc.random_line(rng, sep, ord('"'), wide=True) for _ in range(30)] + [sep * 300, b"a" + sep + b"b"]
            _check(b"\n".join(lines), cfg, okey, 10 ** 7, 5, 123)


@pytest.mark.parametrize("split_char", [10, 0, ord(";")])
def test_empty_pieces_trailing_and_other_split_chars(split_char):
    rng = random.Random(split_char)
    cfg = sdc.config(["a", "b", "c"], renamed="raw", keep_fail=True, keep_succeed=True, copy_raw=True)
    lines = [dc.random_line(rng, b",", ord('"')).replace(bytes([split_char]), b"") for _ in range(30)]
    lines += [b"", b"", b"x,1"]
    for trailing in (False, True):
        val = bytes([split_char]).join(lines) + (bytes([split_char]) if trailing else b"")
        for okey in (None, OKEY):
            _check(val, cfg, okey, 10 ** 12, 5, 123, split_char=split_char)
    _check(bytes([split_char]), cfg, OKEY, 0, 5, None, split_char=split_char)


@pytest.mark.parametrize("pos", sc.POSITIONS)
def test_offsets_across_digit_counts(pos):
    cfg = sdc.config(["a", "b", "c"], keep_fail=True, copy_raw=True)
    _check(sdc.random_value(random.Random(1), cfg, 20), cfg, OKEY, pos, 1 << 30, None)


@pytest.mark.parametrize("name", ["start", "start_cont", "end"])
def test_multiline_pieces_with_quoted_newlines(name):
    """multiline records whose quoted CSV fields hold the split char"""
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
        cfg = sdc.config(["t", "b", "c", "d"], treatment=tr, renamed="raw", keep_succeed=True)
        _check(val, cfg, OKEY, 1 << 20, 1700000000, 7, mcfg=mcfg)


def test_c4_csv_lines():
    from loongcollector_b200 import synth
    buf, _, _ = synth.csv_lines(300)
    cfg = sdc.config(synth.CSV_KEYS, max_fields=11)
    for okey in (None, OKEY):
        _check(buf.tobytes(), cfg, okey, 4096, 1700000000, None)


@pytest.mark.parametrize("okey,treatment,why", [
    (b"content", "extend", "offset key equals SourceKey"),
    (b"content", "discard", "offset key equals SourceKey"),
    (b"__column3__", "extend", "__column"),
    (b"__column07__", "keep", "__column"),
])
def test_refusals(okey, treatment, why):
    cfg = sdc.config(["a", "b"], treatment=treatment)
    with pytest.raises(split_delim_sls.Refused, match=why):
        _run(b"x,1", cfg, okey, 0, 1, None, 1)


def test_refusals_of_the_delimiter_stage():
    with pytest.raises(split_delim_sls.Refused, match="distinct"):
        _run(b"x,1", sdc.config(["a", "a"]), OKEY, 0, 1, None, 1)
    with pytest.raises(split_delim_sls.Refused, match="max_fields"):
        _run(b"x,1", sdc.config(["a", "b"], max_fields=2), OKEY, 0, 1, None, 1)
    empty = sdc.config(["a", "b"], source="")
    with pytest.raises(split_delim_sls.Refused, match="offset key equals SourceKey"):
        _run(b"x,1", empty, b"", 0, 1, None, 1)


def test_column_form_offset_key_in_discard_mode_is_an_ordinary_key():
    cfg = sdc.config(["a", "__column1__", "c"], treatment="discard", keep_succeed=True)
    _check(b"1,2,3,4\n1\n\n5,6", cfg, b"__column1__", 3, 5, None)
    _check(b"1,2,3,4\n1\n\n5,6", cfg, b"__column9__", 3, 5, None)


def test_c_abi_refuses_bad_arguments_without_a_device():
    """argument checks come before the engine is touched"""
    import loongcollector_b200 as lc
    L = lc.lib()
    n, nev = C.c_uint64(0), C.c_uint64(0)
    ctr = np.zeros(4, np.uint64)
    keys = (C.c_char_p * 1)(b"a")
    kl = np.array([1], np.uint32)
    sep = np.frombuffer(b",", np.uint8)
    keycfg = [C.cast(keys, C.c_void_p), kl.ctypes.data_as(C.c_void_p), 1, b"content", 7, b"content", 7, 0, 0, 0,
              OKEY, len(OKEY), 0, 0, 0xFFFFFFFF]
    dcfg = [sep.ctypes.data_as(C.c_void_p), 1, ord('"'), 1, 0, 1, 4] + keycfg
    p = ctr.ctypes.data_as(C.c_void_p)
    assert L.lc_sls_serialize_split_delim_dev(None, None, 0, None, None, 0, None, None, None, None, None, 4,
                                              sep.ctypes.data_as(C.c_void_p), 1, ord('"'), 1, 0, *keycfg, None, 0,
                                              C.byref(n), p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_split_delim_parse_sls(None, None, 0, 10, *dcfg, None, 0, C.byref(n), C.byref(nev),
                                      p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_split_delim_parse_sls_lz4(None, None, 0, 10, *dcfg, None, 0, None, 0, C.byref(n), C.byref(nev),
                                          C.byref(nev), p) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_multiline_split_delim_parse_sls(None, None, 0, None, None, None, 0, *dcfg, None, 0, C.byref(n),
                                                C.byref(nev), p, None) == lc.capi.LC_ERR_INVALID_ARG
    assert L.lc_multiline_split_delim_parse_sls_lz4(None, None, 0, None, None, None, 0, *dcfg, None, 0, None, 0,
                                                    C.byref(n), C.byref(nev), C.byref(nev), p,
                                                    None) == lc.capi.LC_ERR_INVALID_ARG
