"""Shared cases of the split -> regex -> SLS tests: the oracle's splitter over one flat source event, then its
ProcessorParseRegexNative, then sls_serialize_logs; and the configuration matrix over regex_sls_cases' key sets."""
from oracle import oracle as orc
from tests import regex_sls_cases as rc
from tests import split_sls_cases as sc

OKEY = b"__file_offset__"
# a Java record: its first line, then stack lines; the last group spans the rest of the record
RECORD_PATTERN = r"\[([^\]]+)\] \[(\w+)\] ([^:]+): (.*)"
RECORD_KEYS = ["time", "level", "class", "message"]


def random_lines_value(rng, nlines, trailing=None, long_every=0):
    """lines for regex_sls_cases.PATTERN (about 30 % non-matching or empty), some of 64 KiB and more"""
    lines = []
    for i in range(nlines):
        if long_every and i % long_every == long_every - 1:
            lines.append(b"w 12 " + bytes(rng.choice(b"abc -:") for _ in range(rng.randint(65536, 70000))))
        elif rng.random() < 0.3:
            lines.append(rng.choice([b"", b"no digits here x", b"x"]))
        else:
            lines.append(rc.random_line(rng))
    val = b"\n".join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += b"\n"
    return val


def oracle_chain(val, split_cfg, rcfg, time, ns, pos, offset_key=None, multiline=False, enable_ns=True):
    """(Logs bytes, regex counters [3], splitter counters dict or None, piece count) of the oracle chain"""
    g = sc.source_group(val, split_cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    sp = (orc.ProcessorSplitMultilineLogStringNative if multiline else orc.ProcessorSplitLogStringNative)(split_cfg)
    sp.process(g)
    npieces = len(g.events)
    rp = orc.ProcessorParseRegexNative(rc.oracle_config(rcfg))
    rp.process(g)
    return (sc.wire_of(g.events, enable_ns), rc.counters_of(rp.counters),
            sp.counters if multiline else None, npieces)


# offset keys: none, the default, empty, equal to a regex key / RenamedSourceKey / "__raw_log__"
OFFSET_KEYS = [None, OKEY, b"", b"a", b"raw", b"__raw_log__"]


def matrix():
    """(id, regex cfg) over regex_sls_cases' key sets x the 8 flag combinations, and whole-line mode"""
    yield from rc.matrix()
    for name, cfg in rc.whole_line_matrix():
        if cfg["source"] == "content":
            yield name, cfg
    yield "key_is_offset", rc.config(["a", OKEY.decode(), "c"], "content", None, True, True, True)
    yield "renamed_is_offset", rc.config(["a", "b", "c"], "content", OKEY.decode(), True, True, True)
    yield "whole_line_key_is_offset", rc.config([OKEY.decode()], "content", None, False, False, False,
                                                regex=rc.WHOLE_LINE)


def device_args(cfg):
    """the regex stage's keyword arguments of the Engine bindings"""
    return dict(keys=[k.encode() for k in cfg["keys"]], source_key=cfg["source"].encode(),
                renamed_key=rc.renamed_key(cfg), keep_fail=cfg["keep_fail"], keep_succeed=cfg["keep_succeed"],
                copy_raw=cfg["copy_raw"], whole_line=rc.whole_line(cfg))
