"""Shared cases of the regex -> SLS serialiser tests: seeded random lines and processor configurations, and the
oracle's answer (oracle.ProcessorParseRegexNative over flat events, then oracle.sls_serialize_logs)."""
import random

import numpy as np

from oracle import oracle as orc

PATTERN = r"(\w*)\s(\d+)\s(.*)"  # three groups; the third may be empty
WHOLE_LINE = "(.*)"
_ALPHA = "abcxyz0129_"


def random_line(rng) -> bytes:
    r = rng.random()
    if r < 0.06:
        return b""
    if r < 0.16:  # no match: no digits after the first blank
        return ("".join(rng.choice(_ALPHA) for _ in range(rng.randint(0, 12))) + " x").encode()
    w = "".join(rng.choice(_ALPHA) for _ in range(rng.choice([0, 1, 3, 9])))
    d = "".join(rng.choice("0123456789") for _ in range(rng.choice([1, 2, 6])))
    rest = "".join(rng.choice(_ALPHA + " -:/") for _ in range(rng.choice([0, 0, 1, 7, 40, 200])))
    return ("%s %s %s" % (w, d, rest)).encode()


def config(keys, source="content", renamed=None, keep_fail=False, keep_succeed=False, copy_raw=False,
           regex=PATTERN):
    return {"keys": list(keys), "source": source, "renamed": renamed, "keep_fail": keep_fail,
            "keep_succeed": keep_succeed, "copy_raw": copy_raw, "regex": regex}


def random_config(rng):
    source = rng.choice(["content", "content", "src", "__raw_log__"])
    nkeys = rng.choice([1, 2, 3, 3, 3, 4])  # 4 keys > 3 groups: every match is LC_REGEX_KEYS_MISMATCH
    pool = ["a", "b", "c", "content", "raw", "__raw_log__", source]
    keys = [rng.choice(pool) for _ in range(nkeys)]
    renamed = rng.choice([None, None, source, rng.choice(keys), "__raw_log__", "raw"])
    return config(keys, source, renamed, rng.random() < 0.5, rng.random() < 0.5, rng.random() < 0.5)


def oracle_config(cfg):
    c = {"SourceKey": cfg["source"], "Regex": cfg["regex"], "Keys": list(cfg["keys"]),
         "KeepingSourceWhenParseFail": cfg["keep_fail"], "KeepingSourceWhenParseSucceed": cfg["keep_succeed"],
         "CopingRawLog": cfg["copy_raw"]}
    if cfg["renamed"] is not None:
        c["RenamedSourceKey"] = cfg["renamed"]
    return c


def renamed_key(cfg) -> bytes:
    return (cfg["renamed"] or cfg["source"]).encode()


def whole_line(cfg):
    return cfg["regex"] == WHOLE_LINE


def arena(lines, gap=b"\n"):
    """lines back to back with one gap byte between them -> (buf uint8, off, len)"""
    buf = bytearray()
    off, ln = [], []
    for x in lines:
        off.append(len(buf))
        ln.append(len(x))
        buf += x + gap
    return np.frombuffer(bytes(buf) or b"\0", np.uint8), np.array(off, np.uint32), np.array(ln, np.uint32)


def parse_tables(buf, off, ln, cfg):
    """the oracle's regex tables (equal to lc_regex_parse's, pinned by the parity tests): (status, cap_off, cap_len,
    row pitch)"""
    rx = orc.Regex(cfg["regex"])
    st, co, cl = orc.regex_parse_batch(rx, buf, off, ln, len(cfg["keys"]))
    return st, co, cl, rx.ngroups


def oracle_wire(lines, cfg, times, nss, enable_ns=True):
    """(Logs bytes, counters dict, surviving event count) of Process over flat events + the serialiser"""
    p = orc.ProcessorParseRegexNative(oracle_config(cfg))
    g = orc.Group()
    for i, line in enumerate(lines):
        e = orc.Event()
        e.set(cfg["source"].encode(), line)
        e.timestamp = int(times[i])
        e.ns = None if nss is None or nss[i] == 0xFFFFFFFF else int(nss[i])
        g.events.append(e)
    p.process(g)
    data, _ = orc.sls_serialize_logs([(e.timestamp, e.ns, e.live()) for e in g.events], enable_ns)
    return data, p.counters, len(g.events)


def counters_of(ctr):
    """the oracle's counters dict in the C-ABI's order: successful, failed, discarded"""
    return [ctr["out_successful"], ctr["out_failed"], ctr["discarded"]]


def times_for(n, seed):
    rng = np.random.default_rng(seed)
    t = rng.choice([5, 1700000000, 0xFFFFFFF0], size=n).astype(np.uint32)
    ns = np.where(rng.random(n) < 0.5, 0xFFFFFFFF, rng.integers(0, 999999999, n)).astype(np.uint32)
    return t, ns


_KEY_SETS = {  # name -> (keys, renamed); source key "content"
    "distinct": (["a", "b", "c"], None),
    "repeated": (["a", "b", "a"], None),
    "source_among_keys": (["a", "content", "c"], None),
    "source_first_and_repeated": (["content", "b", "content"], "raw"),
    "key_is_renamed": (["a", "raw", "c"], "raw"),
    "key_is_raw_log": (["a", "__raw_log__", "c"], None),
    "renamed_is_source": (["a", "b", "c"], "content"),
    "keys_mismatch": (["a", "b", "c", "d"], "raw"),
}


def matrix():
    """(id, cfg) over key sets x the 8 flag combinations"""
    for name, (keys, renamed) in _KEY_SETS.items():
        for f in range(8):
            yield "%s-f%d" % (name, f), config(keys, "content", renamed, bool(f & 1), bool(f & 2), bool(f & 4))


def whole_line_matrix():
    """whole-line mode: Keys [], [S], [a], [a, S], with SourceKey "content" and another"""
    for source in ("content", "src"):
        for keys in ([], [source], ["a"], ["a", source]):
            for f in (0, 3, 5, 7):
                yield ("whole-%s-%s-f%d" % (source, "_".join(keys) or "none", f),
                       config(keys, source, None, bool(f & 1), bool(f & 2), bool(f & 4), regex=WHOLE_LINE))


def random_cases(seed_base, count):
    for k in range(count):
        rng = random.Random(seed_base * 1000 + k)
        yield "random-%d" % k, random_config(rng), rng
