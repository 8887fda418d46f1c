"""Shared inputs of the Apsara tests: the reference's fixtures (tests/golden/ref_apsara.json) as groups, and generated
groups that cover the time cache, the field scans and the undefined-read rules."""
import json
import os
import random

from oracle.oracle import Group

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_apsara.json")))
ZONES = ["UTC", "Asia/Shanghai", "America/New_York"]


def corner_values():
    """values for the corners the device pins: every one a separate event of one group, in this order"""
    long_v = b"[2024-01-02 03:04:05.1]\t" + b"\t".join(b"k%d:%s" % (i, b"v" * 50) for i in range(1400))
    return [
        b"", b"[", b"[1", b"[]", b"[1]", b"[0]", b"x", b"[2024-01-02 03:04:05]",
        b"[2024-01-02 03:04:05.123]\t[INFO]\t[12]\t[a/b.c:7]\tk:v",
        b"[2024-01-02 03:04:05,456]\tk:v",                 # hit with ',' after the seconds
        b"[2024-01-02 03:04:05]]\tk:v",                     # ']' right after the seconds
        b"[2024-01-02 03:04:0x.9]\tk:v",                    # %S reads "0": a miss that stores its own key
        b"[2024-01-02 03:04:05.77]\tk:v",                  # so this one misses too
        b"[2024-01-02 03:04:xx]\tk:v",                     # a failed full parse (a miss) ...
        b"[2024-01-02 03:04:05.66]\tk:v",                  # ... then a hit on the key of the line before it
        b"[2024-01-02         03:04:05]\tk:v",            # the key is "2024-01-02" and 9 blanks
        b"[2024-01-02         xx.5]\tk:v",                # a hit whose own full parse fails
        b"[1700000000123456]\t[WARN]\tk:v",                  # epoch between date lines
        b"[2024-01-02 03:04:05.88]\tk:v",
        b"[2024-1-2 3:4:5]",                                # short time string: key runs past the value
        b"[2024-1-2 3:4:6]\tk:v",
        b"[2024-01-02 03:04:06]\ta:b\nc:d\te:\t:f\t\tg",   # '\n' inside a value, empty key and value
        b"[2024-01-02 03:04:06]\t[A]\t[B]\t[C]\t[D]\t[E]\t[F]\t[G]\t[H]\t[I]\t[J]\t[K]\tk:v",  # > 10 slots
        b"[2024-01-02 03:04:06]\t[]\t[]\t[]\tk:v",          # empty fields
        b"[2024-01-02 03:04:06]x]\t[a]b]\t[1]\tk:v",        # stale begins
        b"[2024-01-02 03:04:06] k:v\tcontent:over",         # beg_index 0, a key equal to SourceKey
        b"[2024-01-02 03:04:06]\t[INFO]\n[2024-01-02 03:04:07]\t[ERROR]",
        b"[2024-01-02 03:04:06]\t[./x:]\t[5]\t[WARN]",
        long_v,
        b"[9999999999999]\tk:v", b"[1999-12-31 23:59:59.999999999]", b"[1969-12-31 23:59:59]",
        b"[2024-02-30 25:00:00]", b"[2024-01-02\t03:04:05]\tk:v", b"[2024-01-02 03:04:05\x00.5]\tk:v",
        b"[2024-01-02 03:04:0",                             # last value: the key runs past the base buffer
    ]


def random_value(r, t0):
    kind = r.random()
    if kind < 0.01:
        head = b"[%d%06d]" % (t0 + r.randrange(100), r.randrange(10 ** 6))
    elif kind < 0.03:
        head = r.choice([b"[2024-13-01 00:00:00]", b"2024-01-01", b"[2024-01-01 00:00", b"[", b"[x]"])
    else:
        import time
        tm = time.gmtime(t0 + r.randrange(0, 4))
        head = b"[" + time.strftime("%Y-%m-%d %H:%M:%S", tm).encode() + \
            r.choice([b"", b".%d" % r.randrange(10 ** 6), b",%03d" % r.randrange(1000), b".%09d" % r.randrange(10 ** 9)]) + b"]"
    base = [b"INFO", b"12345", b"src/x.cpp:%d" % r.randrange(999), b"ERROR", b"a.b"]
    r.shuffle(base)
    parts = [head] + [b"[" + f + b"]" for f in base[:r.randint(0, 4)]]
    for _ in range(r.randint(0, 8)):
        parts.append(b"k%d:%s" % (r.randrange(20), bytes(r.choice(b"abc:[]/.\n 09") for _ in range(r.randrange(40)))))
    return b"\t".join(parts)


def random_groups(seed, ngroups=40, t0=1700000000):
    r = random.Random(seed)
    groups = []
    for _ in range(ngroups):
        g = []
        for _ in range(r.choice([0, 1, 5, 31, 32, 33, 70])):
            x = r.random()
            g.append(None if x < 0.03 else (b"" if x < 0.05 else random_value(r, t0 + r.randrange(0, 30))))
        groups.append(g)
    return groups


def group_json(values, extra=None):
    evs = []
    for v in values:
        c = {"content": v.decode("latin-1")} if v is not None else {"other": "x"}
        if extra:
            c.update(extra)
        evs.append({"contents": c, "timestamp": 12345678901, "type": 1})
    return {"events": evs}


def oracle_group(js):
    return Group.from_json(js)
