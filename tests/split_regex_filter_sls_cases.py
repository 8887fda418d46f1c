"""Shared cases of the split -> regex -> filter -> SLS tests: the oracle's splitter over one flat source event, its
ProcessorParseRegexNative, its ProcessorFilterNative, then sls_serialize_logs; filter configurations whose leaves read
every kind of key the regex stage can leave behind; and the filter as the device calls take it."""
from oracle import oracle as orc
from tests import regex_sls_cases as rc
from tests import split_regex_sls_cases as src
from tests import split_sls_cases as sc

OKEY = src.OKEY
_O = OKEY.decode()
NOT, AND, OR = 0xFFFFFFFD, 0xFFFFFFFE, 0xFFFFFFFF


def _leaf(key, exp):
    return {"key": key, "exp": exp, "type": "regex"}


def _op(op, *operands):
    return {"operator": op, "operands": list(operands)}


# id -> processor_filter_regex_native configuration.  Keys: a regex key ("a", "b", "c"), SourceKey "content"
# (overwritten by a regex key or not, deleted or kept), RenamedSourceKey "raw", "__raw_log__", the offset key (its
# digits, or a regex key's capture when a regex key overwrote it), a key nobody sets, and the empty key.
FILTERS = {
    "bypass": {},
    "rule_regex_key": {"FilterKey": ["a"], "FilterRegex": [r"[abc0-4_]*"]},
    "rule_source_key": {"FilterKey": ["content"], "FilterRegex": [r".*\d.*"]},
    "rule_renamed": {"FilterKey": ["raw"], "FilterRegex": [r".*[xyz].*"]},
    "rule_raw_log": {"FilterKey": ["__raw_log__"], "FilterRegex": [r".+"]},
    "rule_offset": {"FilterKey": [_O], "FilterRegex": [r"\d*[02468]"]},
    "rule_two": {"FilterKey": ["b", _O], "FilterRegex": [r"\d*[0-6]", r".*[13579]"]},
    "rule_missing": {"FilterKey": ["nope"], "FilterRegex": [r".*"]},
    "rule_empty_key": {"FilterKey": [""], "FilterRegex": [r".*"]},
    "include": {"Include": {"c": r".*[a-m].*", "a": r".*"}},
    "not_missing": {"ConditionExp": _op("not", _leaf("nope", ".*"))},
    "nested": {"ConditionExp": _op(
        "and",
        _op("or", _leaf("b", r"\d\d?"), _leaf("__raw_log__", r".*x.*")),
        _op("not", _op("and", _leaf("c", r".*[yz].*"), _leaf(_O, r"\d*[13579]"))))},
    "or_offset_source": {"ConditionExp": _op("or", _leaf(_O, r"\d*[05]"), _leaf("content", r"[a-c].*"))},
}


def program(fcfg):
    """(leaves [(key bytes, pattern)], postfix program) of a filter configuration, as ProcessorFilterNative's
    DeviceFilter builds them"""
    ce = fcfg.get("ConditionExp")
    if ce is not None:
        leaves, prog = [], []

        def post(v):
            if "operator" in v:
                for o in v["operands"]:
                    post(o)
                prog.append({"not": NOT, "and": AND, "or": OR}[v["operator"].lower()])
            else:
                prog.append(len(leaves))
                leaves.append((v["key"].encode(), v["exp"]))
        post(ce)
        return leaves, prog
    if fcfg.get("FilterKey"):
        pairs = list(zip(fcfg["FilterKey"], fcfg["FilterRegex"]))
    elif fcfg.get("Include"):
        pairs = [(k, fcfg["Include"][k]) for k in sorted(fcfg["Include"])]
    else:
        return [], []
    prog = []
    for i in range(len(pairs)):
        prog += [i] if i == 0 else [i, AND]
    return [(k.encode(), r) for k, r in pairs], prog


def oracle_chain(val, split_cfg, rcfg, fcfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True):
    """(Logs bytes, counters [4] = the regex stage's three and the events the filter removed, splitter counters dict or
    None, piece count) of the oracle chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    rp = orc.ProcessorParseRegexNative(rc.oracle_config(rcfg))
    rp.process(g)
    before = len(g.events)
    orc.ProcessorFilterNative(fcfg).process(g)
    return (sc.wire_of(g.events, enable_ns), rc.counters_of(rp.counters) + [before - len(g.events)],
            sp.counters if multiline else None, npieces)


def matrix():
    """(id, regex cfg): split_regex_sls_cases' matrix and a regex stage that leaves parsed events without contents"""
    yield from src.matrix()
    for f in range(8):
        yield "no_contents-f%d" % f, rc.config([], "content", None, bool(f & 1), False, False)
