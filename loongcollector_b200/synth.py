"""Seeded synthetic log generators for the BASELINE.json configs (SURVEY.md section 8d).

Every generator builds a pool of distinct template lines/records with Python's `random` (seeded),
then samples the pool with numpy to reach the requested size in seconds.  Buffers are one contiguous
uint8 array with '\\n' separators -- the shape LogFileReader hands to the splitters
(core/file_server/reader/LogFileReader.cpp:2511-2525) -- plus the (offset, length) table of the lines.
"""
import random

import numpy as np

DEFAULT_SEED = 20260922

# docs/cn/plugins/processor/native/processor-parse-regex-native.md:49  (10 capture groups)
NGINX_PATTERN = (r'([\d\.]+) \S+ \S+ \[(\S+) \S+\] \"(\w+) ([^\\"]*)\" ([\d\.]+) (\d+) (\d+) (\d+|-) '
                 r'\"([^\\"]*)\" \"([^\\"]*)\"')
NGINX_KEYS = ["ip", "time", "method", "url", "request_time", "request_length", "status", "length", "ref_url",
              "browser"]
# Apache combined (defined by this repo, SURVEY.md 8d; 11 groups)
APACHE_PATTERN = r'^(\S+) (\S+) (\S+) \[([^\]]+)\] "(\S+) (\S+) (\S+)" (\d{3}) (\d+|-) "([^"]*)" "([^"]*)"'
# docs/cn/plugins/input/native/input-file.md:185
JAVA_START_PATTERN = r"\[\d+-\d+-\w+:\d+:\d+.\d+]\s\[\w+]\s.*"
JAVA_PARSE_PATTERN = r"\[(\S+)]\s\[(\S+)]\s(.*)"

_MONTHS = ["Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"]
_METHODS = ["GET", "POST", "PUT", "DELETE", "HEAD", "PATCH"]
_PATHS = ["/PutData", "/api/v1/items", "/index.html", "/wp-admin/admin-ajax.php", "/static/js/app.js", "/health",
          "/logstores/access/shards/lb", "/search"]
_UAS = ["aliyun-sdk-java", "curl/7.68.0", "Mozilla/5.0 (Windows NT 10.0; Win64; x64) AppleWebKit/537.36",
        "python-requests/2.31.0", "Go-http-client/1.1", "okhttp/4.9.3"]
_REFS = ["-", "https://www.google.com/search?q=log", "https://example.com/a/b", "http://10.1.2.3/x"]
_ALNUM = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789"


def _rand_word(rng, n):
    return "".join(rng.choices(_ALNUM, k=n))


def _nginx_line(rng, target_len=None, bad=False):
    ip = "%d.%d.%d.%d" % (rng.randint(1, 223), rng.randint(0, 255), rng.randint(0, 255), rng.randint(1, 254))
    ts = "%02d/%s/%04d:%02d:%02d:%02d +0800" % (rng.randint(1, 28), rng.choice(_MONTHS), rng.randint(2020, 2026),
                                                 rng.randint(0, 23), rng.randint(0, 59), rng.randint(0, 59))
    method = rng.choice(_METHODS)
    path = rng.choice(_PATHS) + "?Category=" + _rand_word(rng, rng.randint(4, 18))
    rt = "%d.%03d" % (rng.randint(0, 9), rng.randint(0, 999))
    reqlen = str(rng.randint(10, 99999))
    status = str(rng.choice([200, 200, 200, 204, 301, 304, 400, 403, 404, 500, 502]))
    length = rng.choice([str(rng.randint(0, 999999)), "-"])
    ref = rng.choice(_REFS)
    ua = rng.choice(_UAS)
    if bad:
        status = "2x0"  # (\d+) cannot match -> regex_match fails

    def build(p):
        return '%s - - [%s] "%s %s" %s %s %s %s "%s" "%s"' % (ip, ts, method, p, rt, reqlen, status, length, ref, ua)

    line = build(path)
    if target_len is not None:
        if len(line) < target_len:
            path = path + "&pad=" if len(line) + 5 <= target_len else path
            line = build(path)
            path = path + _rand_word(rng, target_len - len(line))
            line = build(path)
        if len(line) > target_len:  # shrink the user agent / referrer, then the path
            over = len(line) - target_len
            cut = min(over, max(0, len(ua) - 1))
            ua = ua[:len(ua) - cut]
            over -= cut
            cut = min(over, max(0, len(ref) - 1))
            ref = ref[:len(ref) - cut]
            over -= cut
            path = path[:max(1, len(path) - over)]
            line = build(path)
        assert len(line) == target_len, (len(line), target_len)
    return line


def _apache_line(rng, target_len=None):
    ip = "%d.%d.%d.%d" % (rng.randint(1, 223), rng.randint(0, 255), rng.randint(0, 255), rng.randint(1, 254))
    ts = "%02d/%s/%04d:%02d:%02d:%02d +0000" % (rng.randint(1, 28), rng.choice(_MONTHS), rng.randint(2020, 2026),
                                                 rng.randint(0, 23), rng.randint(0, 59), rng.randint(0, 59))
    user = rng.choice(["-", "frank", "alice"])
    path = rng.choice(_PATHS) + "?id=" + _rand_word(rng, rng.randint(3, 12))
    status = str(rng.choice([200, 200, 301, 404, 500]))
    size = rng.choice([str(rng.randint(0, 999999)), "-"])
    ref = rng.choice(_REFS)
    ua = rng.choice(_UAS)

    def build(p):
        return '%s - %s [%s] "%s %s HTTP/1.1" %s %s "%s" "%s"' % (ip, user, ts, rng_method, p, status, size, ref, ua)

    rng_method = rng.choice(_METHODS)
    line = build(path)
    if target_len is not None:
        if len(line) < target_len:
            path = path + _rand_word(rng, target_len - len(line))
        elif len(line) > target_len:
            over = len(line) - target_len
            cut = min(over, max(0, len(ua) - 1))
            ua = ua[:len(ua) - cut]
            over -= cut
            path = path[:max(1, len(path) - over)]
        line = build(path)
        if len(line) != target_len:
            line = (line + "x" * target_len)[:target_len] if False else line
    return line


def pool_index(pool_n, n, seed):
    """The pool entry each of the n output lines/records was sampled from (same draw as _assemble)."""
    return np.random.default_rng(seed).integers(0, pool_n, size=n)


def _assemble(pool, n, seed):
    """Sample n entries from a pool of byte strings (each already ending with '\\n') into one buffer."""
    lens = np.array([len(p) for p in pool], np.int64)
    idx = pool_index(len(pool), n, seed)
    if np.all(lens == lens[0]):
        mat = np.frombuffer(b"".join(pool), np.uint8).reshape(len(pool), lens[0])
        buf = mat[idx].reshape(-1)
        off = (np.arange(n, dtype=np.int64) * lens[0])
        ln = np.full(n, lens[0] - 1, np.int64)
    else:
        l = lens[idx]
        off = np.zeros(n, np.int64)
        off[1:] = np.cumsum(l[:-1])
        buf = np.frombuffer(b"".join(map(pool.__getitem__, idx.tolist())), np.uint8)
        ln = l - 1
    return np.ascontiguousarray(buf), off.astype(np.uint32), ln.astype(np.uint32)


def newline_lines(n, line_bytes=512, seed=DEFAULT_SEED):
    """C1: n lines of printable ASCII, exactly line_bytes bytes each including the '\\n'."""
    rs = np.random.default_rng(seed)
    pool_n = min(n, 8192)
    mat = rs.integers(0x20, 0x7F, size=(pool_n, line_bytes), dtype=np.uint8)
    mat[:, -1] = 10
    idx = rs.integers(0, pool_n, size=n)
    buf = mat[idx].reshape(-1)
    off = (np.arange(n, dtype=np.int64) * line_bytes).astype(np.uint32)
    ln = np.full(n, line_bytes - 1, np.uint32)
    return np.ascontiguousarray(buf), off, ln


def nginx_pool(n, seed=DEFAULT_SEED, line_bytes=256, bad_fraction=0.01, pool=16384):
    """The distinct template lines nginx_lines() samples from (each ends with '\\n')."""
    rng = random.Random(seed)
    pool_n = max(8, min(n, pool))
    tl = None if line_bytes is None else line_bytes - 1
    lines = []
    for k in range(pool_n):
        bad = rng.random() < bad_fraction
        lines.append((_nginx_line(rng, tl, bad) + "\n").encode("ascii"))
    return lines


def nginx_lines(n, seed=DEFAULT_SEED, line_bytes=256, bad_fraction=0.01, pool=16384):
    """C2: nginx access-log lines for NGINX_PATTERN.  line_bytes includes the '\\n' (None = natural length);
    bad_fraction of the lines deliberately do not match.  Line i is pool entry pool_index(len(pool), n, seed + 1)[i]."""
    return _assemble(nginx_pool(n, seed, line_bytes, bad_fraction, pool), n, seed + 1)


def java_stack_records(n_records, seed=DEFAULT_SEED, mean_frames=20, unmatched_fraction=0.005, pool=4096):
    """C3: Java stack-trace records (first line matches JAVA_START_PATTERN, ~mean_frames '    at ...' lines).
    Returns (buffer, n_lines, n_records_expected_with_start_only)."""
    rng = random.Random(seed)
    rs = np.random.default_rng(seed + 7)
    pool_n = max(4, min(n_records, pool))
    recs = []
    nlines = []
    for k in range(pool_n):
        ts = "%04d-%02d-%02dT%02d:%02d:%02d.%09d" % (rng.randint(2020, 2026), rng.randint(1, 12), rng.randint(1, 28),
                                                      rng.randint(0, 23), rng.randint(0, 59), rng.randint(0, 59),
                                                      rng.randint(0, 999999999))
        lvl = rng.choice(["ERROR", "WARN", "INFO"])
        first = "[%s] [%s] java.lang.Exception: exception happened %s" % (ts, lvl, _rand_word(rng, 8))
        frames = max(0, int(rs.poisson(mean_frames)))
        body = [first]
        for f in range(frames):
            body.append("    at com.aliyun.sls.devops.logGenerator.type.%s.f%d(%s.java:%d)" %
                        (_rand_word(rng, 12), f, _rand_word(rng, 10), rng.randint(1, 999)))
        if rng.random() < unmatched_fraction * (frames + 1):
            body.append("unmatch log line without the continue prefix")
        recs.append(("\n".join(body) + "\n").encode("ascii"))
        nlines.append(len(body))
    buf, off, ln = _assemble(recs, n_records, seed + 1)
    rs2 = np.random.default_rng(seed + 1)
    idx = rs2.integers(0, pool_n, size=n_records)
    total_lines = int(np.array(nlines)[idx].sum())
    return buf, total_lines, n_records


def csv_lines(n, seed=DEFAULT_SEED, pool=16384):
    """C4: CSV lines, 10 fields, ~160 B, 5 % quoted fields, 0.5 % doubled quotes; field 3 is url-like."""
    return _assemble(csv_pool(n, seed, pool), n, seed + 1)


CSV_KEYS = ["ip", "f1", "f2", "url", "f4", "f5", "f6", "f7", "f8", "f9"]
CSV_URL_PATTERN = r"(/[^?]*)\?k=(\w+)"


def zipf_mixed_lines(n, seed=DEFAULT_SEED, s=1.1, lo=64, hi=8192, pool=8192):
    """C5: 50/50 nginx (NGINX_PATTERN) and apache (APACHE_PATTERN) lines, length ~ Zipf(s) clipped to [lo, hi].
    Returns (buffer, off, len, is_apache[n] bool)."""
    lines, kinds = zipf_mixed_pool(n, seed, s, lo, hi, pool)
    buf, off, ln = _assemble(lines, n, seed + 1)
    idx = pool_index(len(lines), n, seed + 1)
    return buf, off, ln, kinds[idx]


def zipf_mixed_pool(n, seed=DEFAULT_SEED, s=1.1, lo=64, hi=8192, pool=8192):
    """The distinct template lines zipf_mixed_lines() samples from (each ends with '\\n') and their kinds; line i of
    zipf_mixed_lines(n, seed, ...) is pool entry pool_index(len(pool), n, seed + 1)[i]."""
    rng = random.Random(seed)
    rs = np.random.default_rng(seed + 3)
    pool_n = max(8, min(n, pool))
    lens = np.clip(lo - 1 + rs.zipf(s, size=pool_n), lo, hi)
    lines, kinds = [], []
    for k in range(pool_n):
        L = int(lens[k])
        if rng.random() < 0.5:
            base = _nginx_line(rng, max(L - 1, 120))
            kinds.append(0)
        else:
            base = _apache_line(rng, max(L - 1, 120))
            kinds.append(1)
        lines.append((base + "\n").encode("ascii"))
    return lines, np.array(kinds, bool)


def csv_pool(n, seed=DEFAULT_SEED, pool=16384):
    """The distinct template lines csv_lines() samples from (same construction; index = pool_index(.., seed + 1))."""
    rng = random.Random(seed)
    pool_n = max(8, min(n, pool))
    lines = []
    for k in range(pool_n):
        cells = []
        for f in range(10):
            if f == 3:
                c = rng.choice(_PATHS) + "?k=" + _rand_word(rng, rng.randint(4, 24))
            elif f == 0:
                c = "%d.%d.%d.%d" % (rng.randint(1, 223), rng.randint(0, 255), rng.randint(0, 255), rng.randint(1, 254))
            else:
                c = _rand_word(rng, rng.randint(2, 22))
            r = rng.random()
            if r < 0.005:
                c = '"' + c[:3] + '""' + c[3:] + '"'
            elif r < 0.05:
                c = '"' + c + ',x"'
            cells.append(c)
        lines.append((",".join(cells) + "\n").encode("ascii"))
    return lines


def apsara_lines(n, seed=DEFAULT_SEED, t0=1700000000, groups_of=1024):
    """n Apsara log lines: "[YYYY-mm-dd HH:MM:SS.ffffff]" in runs of the same second (so the time cache hits), about
    1 % "[<epoch micros>]" lines and 0.5 % malformed heads; 2-4 base fields in varying order, 2-8 key:value fields,
    80 B - 2 KB.  Returns (buf u8, off u32, len u32, grp u32): one group per groups_of lines."""
    import time as _time
    rng = random.Random(seed)
    parts, off, ln, pos = [], np.empty(n, np.uint32), np.empty(n, np.uint32), 0
    sec, run = t0, 0
    for i in range(n):
        if run == 0:
            sec += rng.randrange(1, 3)
            run = rng.randrange(1, 64)
        run -= 1
        x = rng.random()
        if x < 0.01:
            head = b"[%d%06d]" % (sec, rng.randrange(10 ** 6))
        elif x < 0.015:
            head = rng.choice([b"[2024-13-01 00:00:00]", b"2024-01-01 00:00:00", b"[2024-01-01 00"])
        else:
            head = b"[" + _time.strftime("%Y-%m-%d %H:%M:%S", _time.gmtime(sec)).encode() + \
                b".%06d]" % rng.randrange(10 ** 6)
        base = [b"[" + rng.choice([b"INFO", b"WARNING", b"ERROR", b"DEBUG"]) + b"]",
                b"[%d]" % rng.randrange(1, 99999), b"[src/%s.cpp:%d]" % (_rand_word(rng, 8).encode(), rng.randrange(9999)),
                b"[" + _rand_word(rng, 6).encode() + b"]"]
        rng.shuffle(base)
        fields = [head] + base[:rng.randint(2, 4)]
        target = rng.randint(80, 2048)
        nkv = rng.randint(2, 8)
        per = max(1, (target - sum(len(f) + 1 for f in fields)) // nkv - 8)
        for k in range(nkv):
            fields.append(b"%s:%s" % (_rand_word(rng, rng.randint(3, 10)).encode(),
                                      _rand_word(rng, rng.randint(1, per)).encode()))
        line = b"\t".join(fields)
        off[i], ln[i] = pos, len(line)
        parts.append(line)
        pos += len(line)
    grp = np.arange(0, n + groups_of, groups_of, dtype=np.uint64)
    grp = np.minimum(grp, n).astype(np.uint32)
    grp = np.unique(grp)
    if grp[-1] != n or grp.size == 1:
        grp = np.append(grp, np.uint32(n))
    return np.frombuffer(b"".join(parts), np.uint8), off, ln, grp


def _json_line(rng, target):
    """one JSON access-log object of about target bytes: 8-40 members -- strings (about 10 % with escapes), ints, one
    or two floats (shortest round-trip doubles, small and large exponents among them), booleans and null, a nested
    label object and an array"""
    words = lambda k: _rand_word(rng, k)  # noqa: E731
    m = [b'"ts":%d' % rng.randrange(1_600_000_000, 1_800_000_000),
         b'"method":"%s"' % rng.choice([b"GET", b"POST", b"PUT", b"DELETE"]),
         b'"status":%d' % rng.choice([200, 200, 200, 301, 404, 500]),
         b'"latency":%s' % repr(rng.uniform(0, 5000)).encode()]  # shortest round-trip doubles, 17 digits mostly
    if rng.random() < 0.5:
        m.append(b'"ratio":%s' % rng.choice([b"-4.56e-3", b"0.25", b"1.5e3", b"0.0078125", b"3.14159",
                                             repr(rng.uniform(-1, 1) * 10.0 ** rng.randint(-30, 22)).encode()]))
    m.append(b'"ok":%s' % rng.choice([b"true", b"false"]))
    m.append(b'"trace":null')
    m.append(b'"labels":{"app":"%s","zone":"%s","tier":%d}' % (words(6).encode(), words(4).encode(), rng.randrange(9)))
    m.append(b'"hops":[%s]' % b",".join(b"%d" % rng.randrange(1000) for _ in range(rng.randint(0, 6))))
    nmem = rng.randint(8, 40)
    while len(m) < nmem:
        k = words(rng.randint(3, 12)).encode()
        if rng.random() < 0.7:
            v = words(rng.randint(1, 24)).encode()
            if rng.random() < 0.1:
                v += rng.choice([b"\\n", b"\\t", b'\\"', b"\\u00e9", b"\\/"]) + words(4).encode()
            m.append(b'"%s":"%s"' % (k, v))
        else:
            m.append(b'"%s":%d' % (k, rng.randrange(-10 ** 9, 10 ** 12)))
    line = b"{" + b",".join(m) + b"}"
    if len(line) < target:  # a message member brings the object to its length
        line = line[:-1] + b',"msg":"' + words(target - len(line) - 9).encode() + b'"}'
    return line


def json_lines(n, seed=DEFAULT_SEED, lo=150, hi=4096, groups_of=1024, pool=8192):
    """n JSON access-log lines of lo - hi bytes (_json_line), sampled from a seeded pool of distinct lines.  Returns
    (buf u8, off u32, len u32, grp u32): one group per groups_of lines."""
    rng = random.Random(seed)
    lines = [_json_line(rng, rng.randint(lo, hi)) + b"\n" for _ in range(min(pool, n))]
    buf, off, ln = _assemble(lines, n, seed)
    grp = np.minimum(np.arange(0, n + groups_of, groups_of, dtype=np.uint64), n).astype(np.uint32)
    grp = np.unique(grp)
    if grp[-1] != n or grp.size == 1:
        grp = np.append(grp, np.uint32(n))
    return buf, off, ln, grp
