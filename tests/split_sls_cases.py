"""Shared inputs and oracle results of the split-fed SLS serialiser tests (CPU emulation and GPU): the oracle's
splitter (ProcessorSplitLogStringNative / ProcessorSplitMultilineLogStringNative) on one source event, followed by
sls_serialize_logs."""
import random

from oracle import oracle as O

OFFSET_META = O.META_LOG_FILE_OFFSET_KEY
# file offsets whose pieces cross every power of ten and 2^32
POSITIONS = [0, 1] + [10 ** k - 37 for k in range(2, 20)] + [(1 << 32) - 40, (1 << 64) - 100000]
TIMES = [(5, None), ((1 << 28) - 1, 7), (1 << 28, None), ((1 << 28) + 3, 999999999), ((1 << 32) - 1, 0),
         ((1 << 32) + 9, 12345)]


def random_value(rng: random.Random, nlines: int, split_char: int = 10, long_every: int = 0, trailing=None):
    """Lines of 0..300 random bytes (none equal to split_char), a few of 64 KiB and more when long_every > 0."""
    alphabet = bytes(b for b in range(32, 127) if b != split_char)
    lines = []
    for i in range(nlines):
        n = rng.randint(65536, 70000) if long_every and i % long_every == long_every - 1 else rng.choice(
            [0, 1, rng.randint(0, 20), rng.randint(0, 300)])
        lines.append(bytes(rng.choice(alphabet) for _ in range(min(n, 300))) * (n // 300 + 1) if n > 300 else
                     bytes(rng.choice(alphabet) for _ in range(n)))
    val = bytes([split_char]).join(lines)
    if trailing if trailing is not None else rng.random() < 0.5:
        val += bytes([split_char])
    return val


def source_group(val: bytes, key: bytes, time: int, ns, pos: int, offset_key=None):
    g = O.Group()
    if offset_key is not None:
        g.metadata[OFFSET_META] = offset_key.decode()
    e = O.Event(O.LOG)
    e.set(key, val)
    e.timestamp, e.ns, e.pos = time, ns, (pos, len(val))
    g.events.append(e)
    return g


def wire_of(events, enable_ns=True):
    """The `Logs` bytes of the oracle's output events, RAW events as "content" -> content"""
    evs = [(e.timestamp, e.ns, [(b"content", e.raw)] if e.type == O.RAW else e.live()) for e in events]
    return O.sls_serialize_logs(evs, enable_ns)[0]


def split_cfg(key: bytes, split_char=10, raw=False):
    return {"SourceKey": key.decode(), "SplitChar": split_char, "EnableRawContent": raw}


def oracle_split_wire(val, key, time, ns, pos, offset_key=None, split_char=10, raw=False, enable_ns=True):
    g = source_group(val, key, time, ns, pos, offset_key)
    O.ProcessorSplitLogStringNative(split_cfg(key, split_char, raw)).process(g)
    return wire_of(g.events, enable_ns)


def oracle_multiline_wire(val, cfg, time, ns, pos, offset_key=None, enable_ns=True):
    g = source_group(val, cfg.get("SourceKey", "content").encode(), time, ns, pos, offset_key)
    p = O.ProcessorSplitMultilineLogStringNative(cfg)
    p.process(g)
    return wire_of(g.events, enable_ns), p.counters, len(g.events)


# Multiline configurations of the reference's unit tests (ProcessorSplitMultilineLogStringNativeUnittest.cpp)
JAVA_START = r"\d+-\d+-\d+\s\d+:\d+:\d+.*"
ML_CFGS = {
    "start": {"StartPattern": JAVA_START},
    "start_cont": {"StartPattern": r"line.*", "ContinuePattern": r"continue.*"},
    "start_end": {"StartPattern": r"line.*", "EndPattern": r"endLine.*"},
    "cont_end": {"ContinuePattern": r"continue.*", "EndPattern": r"endLine.*"},
    "end": {"EndPattern": r"endLine.*"},
}


def ml_config(name, discard=False, raw=False, key="content"):
    cfg = dict(ML_CFGS[name])
    cfg.update({"SourceKey": key, "UnmatchedContentTreatment": "discard" if discard else "single_line",
                "EnableRawContent": raw})
    return cfg


def ml_value(rng: random.Random, nrec: int):
    """Records of the shapes the unit-test patterns match, with unmatched lines between them"""
    out = []
    for i in range(nrec):
        kind = rng.randrange(6)
        if kind == 0:
            out.append(b"2024-01-0%d 10:00:0%d ERROR boom" % (rng.randint(1, 9), rng.randint(0, 9)))
            out += [b"\tat com.example.Frame%d(Frame.java:%d)" % (j, rng.randint(1, 999)) for j in
                    range(rng.randint(0, 12))]
        elif kind == 1:
            out.append(b"line %d" % i)
            out += [b"continue %d" % j for j in range(rng.randint(0, 4))]
        elif kind == 2:
            out += [b"x" * rng.randint(0, 40) for _ in range(rng.randint(1, 3))] + [b"endLine %d" % i]
        elif kind == 3:
            out.append(b"unmatched %s" % (b"y" * rng.randint(0, 200)))
        elif kind == 4:
            out.append(b"")
        else:
            out.append(b"line start " + b"z" * rng.randint(0, 300))
            out.append(b"endLine")
    return b"\n".join(out) + (b"\n" if rng.random() < 0.5 else b"")
