"""Shared cases of the delimiter -> regex -> SLS chain tests: the delimiter matrix of tests/delim_sls_cases.py with
random regex stages on top (SourceKey = one of the delimiter's keys), an independent statement of which chains the
device path refuses, and the oracle's answer (ProcessorParseDelimiterNative, then ProcessorParseRegexNative, then
oracle.sls_serialize_logs)."""
import re

from oracle import oracle as orc
from tests import delim_sls_cases as dc
from tests import regex_sls_cases as rc

# quote-sensitive: a column with doubled quotes parses differently raw ("" = two bytes) and collapsed (one)
PAT_QUOTE = r'([^"]*)"(.*)'
PAT_WORD = r"(\w*)(.*)"
WHOLE_LINE = rc.WHOLE_LINE


def delim_keys(dcfg):
    """the delimiter keys a regex stage can read (a "_" in discard mode is no content)"""
    return [k for k in dcfg["keys"] if not (dcfg["treatment"] == "discard" and k == "_")]


def random_regex(rng, dcfg):
    ks = delim_keys(dcfg)
    source = rng.choice(ks) if ks and rng.random() < 0.9 else rng.choice(["content", "zz"])
    regex = rng.choice([PAT_QUOTE, PAT_QUOTE, PAT_WORD, WHOLE_LINE])
    pool = ["r1", "r2", "r3", source, source, "__raw_log__", "raw"] + (["a", "content"] if rng.random() < 0.2 else [])
    nkeys = rng.choice([0, 1, 2, 2, 3]) if regex == WHOLE_LINE else rng.choice([1, 2, 2, 3])
    keys = [rng.choice(pool) for _ in range(nkeys)]
    renamed = rng.choice([None, None, source, "raw", "__raw_log__", "r1"])
    return rc.config(keys, source, renamed, rng.random() < 0.5, rng.random() < 0.5, rng.random() < 0.5, regex=regex)


def refused(dcfg, rcfg):
    """whether the device path refuses the chain (restated from its contract, not from its code)"""
    ks = delim_keys(dcfg)
    src = rcfg["source"]
    if src not in ks:
        return True
    dren = dcfg["renamed"] or dcfg["source"]

    def left(name):  # a content the delimiter stage may leave under `name`, other than the regex source's
        if name == src:
            return False
        return (name in ks or name == dcfg["source"]
                or ((dcfg["keep_fail"] or dcfg["keep_succeed"]) and name == dren)
                or (dcfg["keep_fail"] and dcfg["copy_raw"] and name == "__raw_log__")
                or (dcfg["treatment"] != "discard" and re.fullmatch(r"__column\d+__", name) is not None))
    if rcfg["regex"] == WHOLE_LINE:
        names = [rcfg["keys"][0] if rcfg["keys"] else "content"]
    else:
        names = list(rcfg["keys"])
    if rcfg["keep_fail"] or rcfg["keep_succeed"]:
        names.append(rcfg["renamed"] or src)
    if rcfg["keep_fail"] and rcfg["copy_raw"]:
        names.append("__raw_log__")
    if any(left(x) for x in names):
        return True
    return not rcfg["keep_fail"] and left("_time_") and left("_source_")


def oracle_wire(lines, dcfg, rcfg, times, nss, enable_ns=True):
    """(Logs bytes, counters[8] in the C-ABI's order) of both Process calls over flat events + the serialiser"""
    d = orc.ProcessorParseDelimiterNative(dc.oracle_config(dcfg))
    r = orc.ProcessorParseRegexNative(rc.oracle_config(rcfg))
    g = orc.Group()
    for i, line in enumerate(lines):
        e = orc.Event()
        e.set(dcfg["source"].encode(), line)
        e.timestamp = int(times[i])
        e.ns = None if nss is None or nss[i] == 0xFFFFFFFF else int(nss[i])
        g.events.append(e)
    d.process(g)
    r.process(g)
    data, _ = orc.sls_serialize_logs([(e.timestamp, e.ns, e.live()) for e in g.events], enable_ns)
    return data, counters_of(d.counters, r.counters)


def counters_of(dctr, rctr):
    """both processors' counters in the C-ABI's order.  The delimiter's out_failed is failed + blank: the C-ABI
    reports the two apart, so the comparison folds them (see fold)."""
    return [dctr["out_successful"], dctr["out_failed"], dctr["discarded"], rctr["out_successful"],
            rctr["out_failed"], rctr["out_key_not_found"], rctr["discarded"]]


def fold(ctr):
    """C-ABI counters[8] -> counters_of's order"""
    c = [int(x) for x in ctr]
    return [c[0], c[1] + c[3], c[2], c[4], c[5], c[6], c[7]]
