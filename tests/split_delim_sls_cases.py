"""Shared cases of the split -> delimiter -> SLS tests: the oracle's splitter over one flat source event, then its
ProcessorParseDelimiterNative, then sls_serialize_logs; and the configurations that put the offset content against the
delimiter's keys, RenamedSourceKey and "__raw_log__"."""
import numpy as np

from oracle import oracle as orc
from tests import delim_sls_cases as dc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"


def config(keys, sep=b",", quote=ord('"'), treatment="extend", source="content", renamed=None, keep_fail=True,
           keep_succeed=False, copy_raw=False, allow_short=True, max_fields=None):
    return {"sep": sep, "quote": quote, "treatment": treatment, "keys": list(keys), "source": source,
            "renamed": renamed, "keep_fail": keep_fail, "keep_succeed": keep_succeed, "copy_raw": copy_raw,
            "allow_short": allow_short, "max_fields": max_fields if max_fields is not None else len(keys) + 3}


def with_flags(cfg, flags):
    """cfg with KeepingSourceWhenParseFail / KeepingSourceWhenParseSucceed / CopingRawLog from the bits of flags"""
    return dict(cfg, keep_fail=bool(flags & 1), keep_succeed=bool(flags & 2), copy_raw=bool(flags & 4))


def random_value(rng, cfg, nlines, split_char=10, trailing=None, wide_every=0):
    """delim_sls_cases' random lines (blank, short, wide, quoted, broken) joined by split_char; a quoted field that
    would hold split_char is left as it is (the splitter cuts it: one more broken row)"""
    lines = [dc.random_line(rng, cfg["sep"], cfg["quote"], wide=bool(wide_every) and i % wide_every == 0)
             for i in range(nlines)]
    val = bytes([split_char]).join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += bytes([split_char])
    return val


def tables(val, off, ln, cfg):
    """the oracle's delimiter tables over the pieces (equal to lc_delim_parse's, pinned by the parity tests)"""
    return dc.parse_tables(np.frombuffer(bytes(val) or b"\0", np.uint8), off, ln, cfg)


def counters_of(ctr):
    """the oracle's delimiter counters in the order the chain's counters[4] fold to: successful, failed + blank,
    discarded"""
    return [ctr["out_successful"], ctr["out_failed"], ctr["discarded"]]


def fold(ctr):
    """the chain's counters[4] (successful, failed, discarded, blank) as counters_of orders the oracle's"""
    return [int(ctr[0]), int(ctr[1]) + int(ctr[3]), int(ctr[2])]


def oracle_chain(val, split_cfg, cfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True):
    """(Logs bytes, delimiter counters [3] as counters_of, splitter counters dict or None, piece count) of the oracle
    chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    dp = orc.ProcessorParseDelimiterNative(dc.oracle_config(cfg))
    dp.process(g)
    return sc.wire_of(g.events, enable_ns), counters_of(dp.counters), sp.counters if multiline else None, npieces


# offset-key corners (name, delimiter cfg, offset key): a key at a column every row reaches and at one short rows do not
# reach; the offset key as one key while another is SourceKey; RenamedSourceKey / "__raw_log__" / "_" as the offset key
def offset_corners():
    yield "key_col0", config(["off", "b", "c"]), b"off"
    yield "key_col_short", config(["a", "b", "c", "d", "off"]), b"off"
    yield "key_and_source", config(["a", "content", "off", "d"], keep_succeed=True), b"off"
    yield "source_then_key", config(["off", "b", "content"], keep_succeed=True), b"off"
    yield "renamed", config(["a", "b", "c"], renamed="off", keep_succeed=True), b"off"
    yield "raw_log", config(["a", "b", "c"], renamed="r", copy_raw=True), b"__raw_log__"
    yield "underscore_discard", config(["a", "_", "c", "_"], treatment="discard"), b"_"
    yield "underscore_extend", config(["a", "_", "c"], treatment="extend"), b"_"
    yield "underscore_keep", config(["a", "_", "c"], treatment="keep", max_fields=6), b"_"
    yield "column_form_discard", config(["a", "__column1__", "c"], treatment="discard"), b"__column1__"
    yield "multibyte_key", config(["a", "off", "c"], sep=b"|#"), b"off"
    yield "quote_is_sep_key", config(["a", "off"], quote=ord(",")), b"off"


def device_args(cfg):
    """the delimiter stage's keyword arguments of the Engine bindings"""
    return dict(sep=cfg["sep"], quote=cfg["quote"] if len(cfg["sep"]) == 1 else ord('"'),
                treatment=cfg["treatment"], keys=[k.encode() for k in cfg["keys"]],
                source_key=cfg["source"].encode(), renamed_key=dc.renamed_key(cfg), keep_fail=cfg["keep_fail"],
                keep_succeed=cfg["keep_succeed"], copy_raw=cfg["copy_raw"], allow_short=cfg["allow_short"],
                max_fields=cfg["max_fields"])
