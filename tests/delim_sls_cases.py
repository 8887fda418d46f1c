"""Shared cases of the delimiter -> SLS serialiser tests: seeded random lines and processor configurations, and the
oracle's answer (oracle.ProcessorParseDelimiterNative over flat events, then oracle.sls_serialize_logs)."""
import random

import numpy as np

from oracle import oracle as orc

SEPARATORS = [  # (name, separator, quote)
    ("comma", b",", ord('"')),            # one byte, quote state machine
    ("multibyte", b"|#", ord('"')),       # multi-byte split (a configured quote is ignored)
    ("blank", b" ", ord('"')),            # the blank as separator
    ("quote_is_sep", b",", ord(",")),     # quote == separator: split, no quote handling
]
TREATMENTS = ["extend", "keep", "discard"]
_ALPHA = "abcxyzABC0129-_./:"


def _field(rng, sep: bytes, quote: int, use_quote: bool):
    r = rng.random()
    if r < 0.12:
        return ""
    if r < 0.3 and use_quote:  # quoted, with separators and doubled quotes inside
        body = ""
        for _ in range(rng.randint(0, 8)):
            x = rng.random()
            body += (sep.decode("latin1") if x < 0.2 else chr(quote) * 2 if x < 0.35 else " " if x < 0.45
                     else rng.choice(_ALPHA))
        return chr(quote) + body + chr(quote)
    s = "".join(rng.choice(_ALPHA + "  ") for _ in range(rng.choice([1, 2, 5, 12, 40])))
    return s


def random_line(rng, sep: bytes, quote: int, wide=False) -> bytes:
    use_quote = len(sep) == 1 and quote != sep[0]
    r = rng.random()
    if r < 0.05:
        return rng.choice([b"", b" ", b"   ", b" \r", b"\r"])
    if r < 0.08 and use_quote:  # unterminated quote
        return (chr(quote) + "abc" + sep.decode("latin1") + "d").encode("latin1")
    if r < 0.11 and use_quote:  # quote inside a plain field (an error of the state machine)
        return ("ab" + chr(quote) + "c" + sep.decode("latin1") + "x").encode("latin1")
    ncols = rng.randint(30, 70) if wide else rng.choice([1, 2, 3, 4, 5, 6, 8, 12])
    line = sep.decode("latin1").join(_field(rng, sep, quote, use_quote) for _ in range(ncols))
    if rng.random() < 0.15:
        line = " " * rng.randint(1, 3) + line
    if rng.random() < 0.15:
        line += rng.choice([" ", "  ", "\r", " \r"])
    return line.encode("latin1")


def random_config(rng, treatment, sep, quote):
    nkeys = rng.randint(1, 6)
    pool = ["a", "b", "c", "d", "e", "f", "content", "msg"]
    if treatment == "discard":
        keys = [rng.choice(["_", "_"] + pool) for _ in range(nkeys)]
        seen, uniq = set(), []
        for k in keys:  # repeats only of "_"
            if k != "_" and k in seen:
                k = "_"
            seen.add(k)
            uniq.append(k)
        keys = uniq
    else:
        keys = rng.sample(pool + ["_"], nkeys)
    source = rng.choice(["content", "content", "src", "_"])
    renamed = rng.choice([None, None, rng.choice(keys), source, "__raw_log__", "__column%d__" % nkeys,
                          "__column%d__" % (nkeys + 2), "raw"])
    return {
        "sep": sep, "quote": quote, "treatment": treatment, "keys": keys, "source": source, "renamed": renamed,
        "keep_fail": rng.random() < 0.6, "keep_succeed": rng.random() < 0.5, "copy_raw": rng.random() < 0.5,
        "allow_short": rng.random() < 0.7, "max_fields": nkeys + rng.choice([1, 2, 3, 16]),
    }


def oracle_config(cfg):
    c = {"SourceKey": cfg["source"], "Separator": cfg["sep"].decode("latin1"), "Keys": list(cfg["keys"]),
         "OverflowedFieldsTreatment": cfg["treatment"], "AllowingShortenedFields": cfg["allow_short"],
         "KeepingSourceWhenParseFail": cfg["keep_fail"], "KeepingSourceWhenParseSucceed": cfg["keep_succeed"],
         "CopingRawLog": cfg["copy_raw"]}
    if len(cfg["sep"]) == 1:
        c["Quote"] = chr(cfg["quote"])
    if cfg["renamed"] is not None:
        c["RenamedSourceKey"] = cfg["renamed"]
    return c


def renamed_key(cfg) -> bytes:
    return (cfg["renamed"] or cfg["source"]).encode()


def arena(lines, rng=None, gap=b"\n"):
    """lines back to back with one gap byte between them -> (buf uint8, off, len)"""
    buf = bytearray()
    off, ln = [], []
    for ln_ in lines:
        off.append(len(buf))
        ln.append(len(ln_))
        buf += ln_ + gap
    return np.frombuffer(bytes(buf) or b"\0", np.uint8), np.array(off, np.uint32), np.array(ln, np.uint32)


def oracle_wire(lines, cfg, times, nss, enable_ns=True):
    """(Logs bytes, counters dict, surviving event count) of Process over flat events + the serialiser"""
    p = orc.ProcessorParseDelimiterNative(oracle_config(cfg))
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


def parse_tables(buf, off, ln, cfg):
    """the oracle's delimiter tables (equal to lc_delim_parse's, pinned by the parity tests)"""
    quote = cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')
    return orc.delim_parse_batch(buf, off, ln, cfg["sep"], quote, len(cfg["keys"]), cfg["treatment"] == "extend",
                                 cfg["allow_short"], cfg["max_fields"])


def times_for(n, seed):
    rng = np.random.default_rng(seed)
    t = rng.choice([5, 1700000000, 0xFFFFFFF0], size=n).astype(np.uint32)
    ns = np.where(rng.random(n) < 0.5, 0xFFFFFFFF, rng.integers(0, 999999999, n)).astype(np.uint32)
    return t, ns


def all_cases(seed_base=0, per=4):
    """(id, cfg, rng) over the separator x treatment matrix, `per` random configurations each"""
    for si, (sname, sep, quote) in enumerate(SEPARATORS):
        for ti, tr in enumerate(TREATMENTS):
            for k in range(per):
                rng = random.Random(seed_base * 1000 + si * 100 + ti * 10 + k)
                yield "%s-%s-%d" % (sname, tr, k), random_config(rng, tr, sep, quote), rng
