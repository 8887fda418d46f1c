"""Shared cases of the split -> JSON -> SLS tests: the oracle's splitter over one flat source event, then
oracle/json_parse.py's ProcessorParseJsonNative, then sls_serialize_logs; the CommonParserOptions matrix and values
built to hit the resolve's corners (repeated keys, escaped spellings, keys equal to the chain's own keys)."""
import json
import random

from oracle import json_parse as ojs
from oracle import oracle as orc
from tests import json_cases as jc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"


def config(source="content", renamed=None, keep_fail=False, keep_succeed=False, copy_raw=False):
    cfg = {"SourceKey": source, "KeepingSourceWhenParseFail": keep_fail,
           "KeepingSourceWhenParseSucceed": keep_succeed, "CopingRawLog": copy_raw}
    if renamed is not None:
        cfg["RenamedSourceKey"] = renamed
    return cfg


def renamed_key(cfg):
    """the effective RenamedSourceKey (SourceKey when unset or empty)"""
    return (cfg.get("RenamedSourceKey") or cfg["SourceKey"]).encode()


def flag_configs(renamed=None, source="content"):
    """the 8 CommonParserOptions combinations"""
    return [config(source, renamed, bool(f & 1), bool(f & 2), bool(f & 4)) for f in range(8)]


def oracle_chain(val, split_cfg, jcfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True):
    """(Logs bytes, JSON counters [3] = successful, failed, discarded, splitter counters or None, piece count)"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    jp = ojs.ProcessorParseJsonNative(jcfg)
    jp.process(g)
    c = jp.counters
    return (sc.wire_of(g.events, enable_ns), [c["out_successful"], c["out_failed"], c["discarded"]],
            sp.counters if multiline else None, npieces)


def escaped(key: str):
    """the key with every character as a \\u escape (its rendering lands in the arena)"""
    return '"' + "".join("\\u%04x" % ord(ch) for ch in key) + '"'


def doc(members):
    """an object of (key spelling, JSON value text) members, keys given as JSON string text"""
    return ("{" + ",".join("%s:%s" % (k, v) for k, v in members) + "}").encode()


def special_lines(source="content", okey=OKEY, renamed="raw"):
    """lines that put the chain's own keys among the members, once and repeated, plain and escaped"""
    s, o, r = json.dumps(source), json.dumps(okey.decode() if okey is not None else "off"), json.dumps(renamed)
    raw = json.dumps("__raw_log__")
    return [
        doc([(s, '"v1"')]),
        doc([('"a"', "1"), (s, '"v1"'), ('"b"', "2"), (s, '"v2"'), ('"a"', "3")]),
        doc([(o, "5")]),
        doc([('"x"', "1"), (o, '"o1"'), (o, '"o2"'), ('"x"', "2")]),
        doc([(r, '"r"'), ('"k"', "true")]),
        doc([(raw, '"rl"'), ('"k"', "null")]),
        doc([('"a"', "1"), ('"a"', "2")]),
        doc([('"a"', "1"), (escaped("a"), "2"), ('"a"', "3"), (escaped("a"), "4")]),
        doc([(escaped("a"), '"e"'), ('"b"', "[1, 2]"), ('"a"', '"p"')]),
        doc([(escaped(source), '"esc"'), ('"z"', "{}")]),
        doc([]),
        b"{ }",
        b"",
        b"not json",
        b'{"a":1',
        b'{"a":tru}',
        doc([('"k%d"' % (i % 5), str(i)) for i in range(40)]),
        doc([('"dup"', str(i)) for i in range(33)]),
        doc([('"k%d"' % i, str(i)) for i in range(32)]),
        doc([('"k%d"' % (i % 3), str(i)) for i in range(32)]),
    ]


def random_value(seed, nlines=60, trailing=None):
    """JSON lines: valid documents (duplicates through the generator), mutated ones, special lines, empty lines"""
    rng = random.Random(seed)
    docs = jc.valid_docs(nlines, seed)
    bad = jc.mutate(docs[:10], seed, per=1)
    lines = [d.replace(b"\n", b" ") for d in docs + bad + special_lines()]
    lines = [ln.replace(b"\x00", b"") for ln in lines]
    rng.shuffle(lines)
    val = b"\n".join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def big_doc(n, alike=False, escaped_every=0):
    """one line of n members: all keyed alike, or n distinct keys (some escaped)"""
    if alike:
        return doc([('"same"', str(i)) for i in range(n)])
    return doc([(escaped("k%d" % i) if escaped_every and i % escaped_every == 0 else '"k%d"' % i, str(i))
                for i in range(n)])
