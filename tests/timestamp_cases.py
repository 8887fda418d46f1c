"""Seeded inputs of the timestamp-parse tests: formats covering every strptime_ns directive, random dates from 1971 to
2037 rendered in them, damaged values, SourceYear modes and cache sequences.  Each case is
(name, format, source_year, adjust, now, discard_interval, groups) with groups as tests/emul/timestamp.layout takes."""
import calendar
import random
import time

NOW = 1700000000          # 2023-11-14 22:13:20 UTC
NOW_DEC31 = 1704024000    # 2023-12-31 12:00:00 UTC
NOW_JAN1 = 1704110400     # 2024-01-01 12:00:00 UTC
ZONES = ("UTC", "Asia/Shanghai", "America/New_York")

DAYS = ("Sunday", "Monday", "Tuesday", "Wednesday", "Thursday", "Friday", "Saturday")
MONTHS = ("January", "February", "March", "April", "May", "June", "July", "August", "September", "October",
          "November", "December")


def _fields(rng):
    return time.gmtime(rng.randint(calendar.timegm((1971, 1, 1, 0, 0, 0)), calendar.timegm((2037, 12, 31, 23, 59, 59))))


def render(fmt, g, rng):
    """fmt rendered for the broken-down time g, with random fractions, zones and name spellings"""
    out, i = [], 0
    while i < len(fmt):
        c = fmt[i]
        if c != "%":
            out.append(c)
            i += 1
            continue
        d = fmt[i + 1:i + 2]
        i += 2
        while d and d in "EO":
            d = fmt[i:i + 1]
            i += 1
        wd = (g.tm_wday + 1) % 7
        h12 = g.tm_hour % 12 or 12
        v = {
            "Y": "%04d" % g.tm_year, "y": "%02d" % (g.tm_year % 100), "C": "%02d" % (g.tm_year // 100),
            "m": "%02d" % g.tm_mon, "d": "%02d" % g.tm_mday, "e": "%2d" % g.tm_mday, "H": "%02d" % g.tm_hour,
            "k": "%2d" % g.tm_hour, "I": "%02d" % h12, "l": "%2d" % h12, "M": "%02d" % g.tm_min, "S": "%02d" % g.tm_sec,
            "j": "%03d" % g.tm_yday, "p": rng.choice(("AM", "am", "Am")) if g.tm_hour < 12 else rng.choice(("PM", "pm")),
            "a": DAYS[wd][:3], "A": DAYS[wd], "b": MONTHS[g.tm_mon - 1][:3], "h": MONTHS[g.tm_mon - 1][:3].upper(),
            "B": MONTHS[g.tm_mon - 1], "w": str(wd), "u": str(wd or 7), "U": "%02d" % rng.randint(0, 53),
            "W": "%02d" % rng.randint(0, 53), "V": "%02d" % rng.randint(1, 53), "g": "%02d" % (g.tm_year % 100),
            "G": "%04d" % g.tm_year, "n": rng.choice((" ", "\t", "")), "t": rng.choice(("  ", "\n")), "%": "%",
            "f": "".join(rng.choice("0123456789") for _ in range(rng.choice((1, 3, 6, 9, 9, 12)))),
            "z": rng.choice(("+0800", "-0530", "+08:00", "Z", "UT", "GMT", "EST", "pdt", "+08", "-12", "A", "M",
                             "Y", " +0100", "+0860", "+8", "J", "GMX")),
            "Z": rng.choice(("GMT", "utc", "CST", "", "UTC")),
            "D": "%02d/%02d/%02d" % (g.tm_mon, g.tm_mday, g.tm_year % 100),
            "F": "%04d-%02d-%02d" % (g.tm_year, g.tm_mon, g.tm_mday), "R": "%02d:%02d" % (g.tm_hour, g.tm_min),
            "T": "%02d:%02d:%02d" % (g.tm_hour, g.tm_min, g.tm_sec),
            "r": "%02d:%02d:%02d %s" % (h12, g.tm_min, g.tm_sec, "AM" if g.tm_hour < 12 else "PM"),
            "s": str(calendar.timegm(g)) + rng.choice(("", "", "123", "1", "123456789")),
        }.get(d, "")
        out.append(v)
    return "".join(out).encode()


FORMATS = (
    "%Y-%m-%d %H:%M:%S", "%Y-%m-%d %H:%M:%S.%f", "%d/%b/%Y:%H:%M:%S", "%d/%b/%Y:%H:%M:%S %z", "%s",
    "%Y-%m-%dT%H:%M:%S%z", "%a %b %e %H:%M:%S %Y", "%A, %d %B %Y %I:%M:%S %p", "%F %T", "%D %R", "%r %F",
    "%y%m%d %k:%M:%S", "%C%y-%j %l:%M %p", "%Y%m%d%H%M%S", "%m/%d %H:%M:%S", "%b %d %H:%M:%S", "%Y-%m-%d %T %Z",
    "%G-W%V-%u %H:%M:%S %Y", "%g %U %W %w %Y-%m-%d", "%Y-%m-%d%n%H:%M:%S%t", "%%%Y-%m-%d %H:%M:%S%%",
    "%Ey-%Od %OH:%OM:%OS %EY", "%EC%Ey/%m/%d", "%f %T", "%Y-%m-%d %H:%M:%S.%f %z", "%f", "[%Y-%m-%d %H:%M:%S.%f]",
    "%Ed %H", "%Ok %M", "%s %Y", "%q %Y", "%Y %", "%EEY", "%h %d %Y", "%Y-%m-%d %H:%M:%S %%f",
)


def damage(v, rng):
    k = rng.randrange(5)
    if not v or k == 0:
        return v[:rng.randint(0, len(v))] if v else v
    if k == 1:
        p = rng.randrange(len(v))
        return v[:p] + bytes([rng.choice(b"x9 :-+/.\x00\xff")]) + v[p + 1:]
    if k == 2:
        return b""
    if k == 3:
        return v + rng.choice((b" extra", b"7", b".5", b"Z"))
    return b" " + v


def random_cases(seed=20261017, per_format=150):
    rng = random.Random(seed)
    cases = []
    for fmt in FORMATS:
        for mode in (-1, 0, 2020):
            groups = []
            for _ in range(3):
                g = []
                for _ in range(per_format // 3):
                    v = render(fmt, _fields(rng), rng)
                    r = rng.random()
                    g.append(None if r < 0.05 else damage(v, rng) if r < 0.25 else v)
                groups.append(g)
            cases.append(("rand %s y%d" % (fmt, mode), fmt, mode, rng.choice((0, 0, -3600, 28800)), NOW,
                          rng.choice((43200, 43200, -1)), groups))
    return cases


def cache_cases(seed=7):
    """Hit / miss / failed-miss interleavings in groups of every size class."""
    rng = random.Random(seed)
    cases = []
    base = calendar.timegm((2023, 11, 14, 10, 0, 0))
    for fmt, step in (("%Y-%m-%d %H:%M:%S.%f", 1), ("%Y-%m-%d %H:%M:%S", 1), ("%s", 1), ("%Y-%m-%d %H:%M:%S.%f %z", 1),
                      ("%d/%b/%Y:%H:%M:%S", 1), ("%f", 1), ("%Y-%m-%d %H:%M:%S,%f", 1)):
        for per_sec in (1, 2, 3, 33, 1000):
            groups = []
            for gs in (1, 2, 31, 32, 33, 64, 65, 300):
                g, t = [], base + rng.randint(0, 100000)
                for k in range(gs):
                    if k % per_sec == 0:
                        t += step
                    v = render(fmt, time.gmtime(t), rng)
                    r = rng.random()
                    if r < 0.04:
                        v = None
                    elif r < 0.10:
                        v = damage(v, rng)
                    elif r < 0.13 and fmt == "%s":
                        v = v[:10] + b"77"
                    g.append(v)
                groups.append(g)
            cases.append(("cache %s x%d" % (fmt, per_sec), fmt, -1, rng.choice((0, 3600)), NOW, 43200 * 10 ** 5,
                          groups))
    # hand-made sequences
    hand = [
        ("%Y-%m-%d %H:%M:%S.%f", [b"2023-11-14 10:00:00.1", b"2023-11-14 10:00:00.2", b"2023-11-14 10:00:0x.3",
                                  b"2023-11-14 10:00:00.x", b"2023-11-14 10:00:00.", b"2023-11-14 10:00:00.9",
                                  b"2023-11-14 10:00:01.1", b"2023-11-14 10:00:0", b"2023-11-14 10:00:01.5"]),
        ("%Y-%m-%d %H:%M:%S", [b"2023-11-14 10:00:00", b"2023-11-14 10:00:00", b"2023-11-14 10:00:00 tail",
                               b"2023-11-14 10:99:00", b"2023-11-14 10:00:00", b"2023-11-14 1", b"2023-11-14 10:00:00"]),
        ("%s", [b"1700000000", b"1700000000123", b"1700000000", b"17000000001", b"1700000001", b"170000000",
                b"1700000001x", b"0", b"1700000001999999999999", b""]),
        ("%Y %m %d %f %H", [b"2023 11 14 5 10", b"2023 11 14 5 10", b"2023 11 14 6 10"]),
        ("%f", [b"1.5", b"1.7", b"1.x", b"2", b"2", b"1.9"]),
        ("%d/%b/%Y:%H:%M:%S", [b"14/Nov/2023:10:00:00", None, b"14/Nov/2023:10:00:00", b"bad",
                               b"14/Nov/2023:10:00:00", b"14/Nov/2023:10:00:01", b"14/Nov/2023:10:00:01"]),
    ]
    for fmt, vals in hand:
        cases.append(("hand %s" % fmt, fmt, -1, -7200, NOW, 43200 * 10 ** 5, [vals, vals[::-1], vals[:1]]))
    return cases


def year_cases():
    """SourceYear modes 0 / > 0 / -1 and the Dec 31 / Jan 1 deduction with an injected now."""
    vals = [b"01-01 00:00:01", b"12-31 23:59:59", b"06-15 12:00:00", b"02-29 12:00:00", b"00-00 00:00:00",
            b"13-01 00:00:00", b"01-00 00:00:00"]
    cases = []
    for now in (NOW, NOW_DEC31, NOW_JAN1):
        for mode in (-1, 0, 2000, 1999, 1969):
            for fmt in ("%m-%d %H:%M:%S", "%d/%m %T", "%H:%M:%S"):
                cases.append(("year %s y%d now%d" % (fmt, mode, now), fmt, mode, 0, now, -1, [vals, vals[2:]]))
    return cases


def all_cases():
    return random_cases() + cache_cases() + year_cases()
