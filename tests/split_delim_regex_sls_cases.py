"""Shared cases of the split -> delimiter -> regex -> SLS tests: the oracle's splitter over one flat source event, then
its ProcessorParseDelimiterNative, its ProcessorParseRegexNative on one of the delimiter's keys, then
sls_serialize_logs; an independent statement of which chains the device path refuses; and the C4 regex stage."""
from oracle import oracle as orc
from tests import delim_regex_sls_cases as drc
from tests import delim_sls_cases as dc
from tests import regex_sls_cases as rc
from tests import split_delim_sls_cases as sdc
from tests import split_sls_cases as sc

OKEY = sdc.OKEY


def c4_regex(keep_fail=False, keep_succeed=False, copy_raw=False, renamed=None):
    """C4's regex stage: synth.CSV_URL_PATTERN on the url column, keys path and k"""
    from loongcollector_b200 import synth
    return rc.config(["path", "k"], "url", renamed, keep_fail, keep_succeed, copy_raw, regex=synth.CSV_URL_PATTERN)


def refused(dcfg, rcfg, okey):
    """whether the device path refuses the chain (restated from its contract, not from its code)"""
    if okey is not None:
        o = okey.decode()
        if o == dcfg["source"] or o == rcfg["source"]:
            return True
        if dcfg["treatment"] != "discard" and drc.re.fullmatch(r"__column\d+__", o):
            return True
    if drc.refused(dcfg, rcfg):
        return True
    if okey is None:
        return False
    o = okey.decode()
    names = [rcfg["keys"][0] if rcfg["keys"] else "content"] if rcfg["regex"] == drc.WHOLE_LINE else list(rcfg["keys"])
    if rcfg["keep_fail"] or rcfg["keep_succeed"]:
        names.append(rcfg["renamed"] or rcfg["source"])
    if rcfg["keep_fail"] and rcfg["copy_raw"]:
        names.append("__raw_log__")
    if o in names:
        return True
    # ShouldEraseEvent's "_time_" + "_source_" rule, with the offset content as one more content left besides key k
    dren = dcfg["renamed"] or dcfg["source"]
    ks = drc.delim_keys(dcfg)

    def left(name):
        if name == rcfg["source"]:
            return False
        return (name == o or name in ks or name == dcfg["source"]
                or ((dcfg["keep_fail"] or dcfg["keep_succeed"]) and name == dren)
                or (dcfg["keep_fail"] and dcfg["copy_raw"] and name == "__raw_log__")
                or (dcfg["treatment"] != "discard" and drc.re.fullmatch(r"__column\d+__", name) is not None))
    return not rcfg["keep_fail"] and left("_time_") and left("_source_")


def oracle_chain(val, split_cfg, dcfg, rcfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True):
    """(Logs bytes, counters[7] as delim_regex_sls_cases.counters_of, splitter counters dict or None, piece count) of
    the oracle chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    dp = orc.ProcessorParseDelimiterNative(dc.oracle_config(dcfg))
    dp.process(g)
    rp = orc.ProcessorParseRegexNative(rc.oracle_config(rcfg))
    rp.process(g)
    return (sc.wire_of(g.events, enable_ns), drc.counters_of(dp.counters, rp.counters),
            sp.counters if multiline else None, npieces)


def pieces(val, split_char=10, ml=None):
    """the oracle's piece tables: split_lines, or multiline_split with ml = (start, cont, end, discard)"""
    if ml is None:
        return orc.split_lines(val, split_char)
    off, ln, _fl, _ctr = orc.multiline_split(val, *ml)
    return off, ln


def tables(val, off, ln, dcfg):
    """the oracle's delimiter tables over the pieces"""
    return sdc.tables(val, off, ln, dcfg)


def regex_args(rcfg):
    """the regex stage's keyword arguments of the Engine bindings"""
    return dict(rkeys=[k.encode() for k in rcfg["keys"]], rsource_key=rcfg["source"].encode(),
                rrenamed_key=rc.renamed_key(rcfg), rkeep_fail=rcfg["keep_fail"], rkeep_succeed=rcfg["keep_succeed"],
                rcopy_raw=rcfg["copy_raw"], whole_line=rcfg["regex"] == drc.WHOLE_LINE)


def value_bound(val):
    """bytes the device source buffer needs for the tap: the value, then its side copies from align16(len)"""
    return (len(val) + 15) // 16 * 16 + len(val)


fold = drc.fold
