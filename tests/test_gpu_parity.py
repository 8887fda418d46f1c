"""GPU tier: the CUDA path, called through the C-ABI (ctypes), must be bit-exact against the CPU oracle
on the same seeded inputs: offsets, lengths, statuses, flags and counters."""
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _lc():
    import loongcollector_b200 as lc
    return lc


# ------------------------------------------------------------------------------------------- split
def _rand_buf(rng, n, nl_prob, ch=10):
    a = rng.integers(32, 127, size=n, dtype=np.uint8)
    if n:
        a[rng.random(n) < nl_prob] = ch
    return a


@pytest.mark.parametrize("n", [0, 1, 2, 15, 16, 17, 31, 4095, 4096, 4097, 16383, 16384, 16385, 65536 + 3, 1 << 20,
                               (3 << 20) + 7])
@pytest.mark.parametrize("nl_prob", [0.0, 0.002, 0.05, 0.6])
def test_split_lines_matches_oracle(eng, n, nl_prob):
    rng = np.random.default_rng(n * 131 + int(nl_prob * 1000))
    for trailing in (False, True):
        a = _rand_buf(rng, n, nl_prob)
        if n and trailing:
            a[-1] = 10
        off, ln = eng.split_lines(a)
        eo, el = orc.split_lines(a)
        assert np.array_equal(off, eo) and np.array_equal(ln, el)


def test_split_lines_nul_char_and_all_newlines(eng):
    a = np.zeros(1000, np.uint8)
    off, ln = eng.split_lines(a, split_char=0)
    eo, el = orc.split_lines(a, 0)
    assert np.array_equal(off, eo) and np.array_equal(ln, el) and off.size == 1000
    b = np.frombuffer(b'{\n"k1":"v1"\n}\x00{\n"k2":"v2"\n}', np.uint8)
    off, ln = eng.split_lines(b, split_char=0)
    assert off.tolist() == [0, 14] and ln.tolist() == [13, 13]


def test_split_lines_capacity_error(eng):
    lc = _lc()
    a = np.full(100, 10, np.uint8)
    with pytest.raises(lc.LcError) as ei:
        eng.split_lines(a, cap=10)
    assert ei.value.code == 5


def test_split_dev_unaligned_pointer(eng):
    import torch
    rng = np.random.default_rng(5)
    a = _rand_buf(rng, 100000, 0.01)
    for shift in (1, 3, 8, 15):
        t = torch.zeros(a.size + 64, dtype=torch.uint8, device="cuda")
        t[shift:shift + a.size] = torch.from_numpy(a).cuda()
        d_off = torch.zeros(a.size, dtype=torch.int32, device="cuda")
        d_len = torch.zeros(a.size, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        n = eng.split_lines_dev(t.data_ptr() + shift, a.size, 10, d_off.data_ptr(), d_len.data_ptr(), a.size)
        eo, el = orc.split_lines(a)
        assert n == eo.size
        assert np.array_equal(d_off[:n].cpu().numpy().view(np.uint32), eo)
        assert np.array_equal(d_len[:n].cpu().numpy().view(np.uint32), el)


# ------------------------------------------------------------------------------------------- regex
def _misc():
    with open(os.path.join(HERE, "golden", "ref_misc.json"), encoding="utf-8") as f:
        return json.load(f)


def _events(lines):
    base = b"".join(lines)
    ln = np.array([len(x) for x in lines], np.uint32)
    off = np.zeros(len(lines), np.uint32)
    if len(lines) > 1:
        off[1:] = np.cumsum(ln[:-1])
    return np.frombuffer(base, np.uint8) if base else np.zeros(0, np.uint8), off, ln


def _check_parse(eng, pattern, lines, nkeys=None):
    lc = _lc()
    rx = lc.Regex(pattern)
    o = orc.Regex(pattern)
    base, off, ln = _events(lines)
    nk = rx.ngroups if nkeys is None else nkeys
    st, co, cl = eng.regex_parse(rx, base, off, ln, nk)
    est, eco, ecl = orc.regex_parse_batch(o, base, off, ln, nk)
    assert np.array_equal(st, est), (pattern, np.nonzero(st != est)[0][:5])
    assert np.array_equal(co, eco[:, :rx.ngroups]) and np.array_equal(cl, ecl[:, :rx.ngroups]), pattern
    return st


NGINX = _misc()["full_match_fields"][0]


def test_regex_doc_vector(eng):
    st = _check_parse(eng, NGINX["pattern"], [NGINX["input"].encode()] * 3 + [b"garbage", b""])
    assert st.tolist() == [0, 0, 0, 1, 1]
    lc = _lc()
    rx = lc.Regex(NGINX["pattern"])
    base, off, ln = _events([NGINX["input"].encode()])
    _, co, cl = eng.regex_parse(rx, base, off, ln, 10)
    got = [bytes(base[o:o + l]).decode() for o, l in zip(co[0], cl[0])]
    assert got == NGINX["fields"]


def test_regex_keys_mismatch_status(eng):
    st = _check_parse(eng, r"(\w+)\t(\w+).*", [b"value1\tvalue2", b"value1"], nkeys=3)
    assert st.tolist() == [2, 1]


PATTERNS = [
    r"(\w+)\t(\w+).*",
    r"\[(\S+)]\s\[(\S+)]\s(.*)",
    NGINX["pattern"],
    _misc()["benchmark_pattern"]["pattern"],
    r"(\d+)-(\d+)?(x|yy)*(.*?)(\s.*|)",
    r"^(\S+) (\S+) (\S+) \[([^\]]+)\] \"(\S+) (\S+) (\S+)\" (\d{3}) (\d+|-) \"([^\"]*)\" \"([^\"]*)\"",
    r"(a|ab)(c|bcd)(d*)",
    r"(?:(a)|b)*c",
    r"(\d{1,3})\.(\d{1,3})\.(\d{1,3})\.(\d{1,3}).*",
    r"\s*(\S+)\s*=\s*(\S*?)\s*",
    r"(?!\s)(\S+)\s(?=\[)(\S+)(?!.)",     # single-byte look-aheads (assertions on the next byte)
    r"(\w+)(?=[ =:])(.)(?![ab])(.*)",
]


def _noise_lines(rng, n):
    alpha = "ab c1-2\t\"[]x.=:/ yyd"
    out = []
    for _ in range(n):
        out.append("".join(rng.choice(alpha) for _ in range(rng.randint(0, 40))).encode())
    return out


def _nginx_lines(rng, n):
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(n, seed=rng.randint(0, 1 << 30), line_bytes=None)
    return [bytes(buf[o:o + l]) for o, l in zip(off, ln)]


@pytest.mark.parametrize("pattern", PATTERNS)
def test_regex_parse_matches_oracle_on_noise_and_logs(eng, pattern):
    rng = random.Random(hash(pattern) & 0xFFFF)
    lines = _noise_lines(rng, 3000) + _nginx_lines(rng, 2000)
    lines += [b"1-2xyy rest", b"10.0.0.1 tail", b"k = v ", b"abcd", b"abc", b"aabbc", b"[a] [b] c\nd\ne"]
    rng.shuffle(lines)
    _check_parse(eng, pattern, lines)


def test_regex_parse_long_and_ragged_lines(eng):
    rng = random.Random(9)
    lines = []
    for L in (0, 1, 7, 8, 9, 255, 256, 257, 4095, 8192, 70000):
        lines.append(("[" + "x" * L + "] [lvl] " + "m" * (L // 2)).encode())
        lines.append(("x" * L).encode())
    rng.shuffle(lines)
    _check_parse(eng, r"\[(\S+)]\s\[(\S+)]\s(.*)", lines)
    _check_parse(eng, r"(x*)(.*)", lines)


def test_prefix_match_matches_oracle(eng):
    lc = _lc()
    rng = random.Random(3)
    d = _misc()
    pats = [c["pattern"] for c in d["prefix_search"] + d["multiline_start"]] + [r"Exception.*", r"\s+at\s.*",
                                                                               r"\s*\.\.\.\d+ more"]
    lines = _noise_lines(rng, 2000) + [b"[2024-04-01] xxxxxx", b"aaa[2024-04-01] x", b"[138998928392] x",
                                       b"    at com.example(Book.java:16)", b"    ...23 more",
                                       b"Exception in thread"]
    base, off, ln = _events(lines)
    for p in pats:
        got = eng.regex_prefix_match(lc.Regex(p), base, off, ln)
        o = orc.Regex(p)
        want = np.array([o.prefix_match(x) for x in lines])
        assert np.array_equal(got, want), p


def test_multiline_start_pattern_with_a_look_ahead(eng):
    """A start pattern the reference's users write: "(?!\\s).*" = the record begins at a line that does not start with a
    blank.  Lines, flags and records against the oracle."""
    rng = random.Random(31)
    lines = []
    for _ in range(4000):
        head = rng.choice([b"", b" ", b"\t", b"    at ", b"Exception: ", b"x", b"[1] "])
        lines.append(head + bytes(rng.choice(b"ab c.") for _ in range(rng.randint(0, 30))))
    buf = np.frombuffer(b"\n".join(lines) + b"\n", np.uint8)
    lc = _lc()
    for discard in (False, True):
        off, ln, fl, ctr = eng.multiline_split(buf, lc.Regex(r"(?!\s).*"), None, None, discard)
        eo, el, ef, ectr = orc.multiline_split(buf, orc.Regex(r"(?!\s).*"), None, None, discard)
        assert np.array_equal(off, eo) and np.array_equal(ln, el) and np.array_equal(fl, ef)
        assert ctr.tolist() == ectr.tolist()
        assert 100 < len(eo) < 4000


def test_unsupported_regex_fails_loudly(eng):
    lc = _lc()
    with pytest.raises(lc.LcError) as ei:
        lc.Regex(r"(a)\1")
    assert ei.value.code == 4
    with pytest.raises(lc.LcError) as ei:
        lc.Regex(r"(a")
    assert ei.value.code == 3


# ------------------------------------------------------------------------------------------- multiline
BEGIN, CONT, END, UNM = (b"Exception in thread 'main' java.lang.NullPointerException",
                         b"    at com.example.myproject.Book.getTitle(Book.java:16)", b"    ...23 more", b"unmatch log")
ML_PAT = {"S": r"Exception.*", "C": r"\s+at\s.*", "E": r"\s*\.\.\.\d+ more"}
ML_MODES = ["S", "SC", "SE", "CE", "E", "SCE"]


def _ml_check(eng, buf, mode, discard):
    lc = _lc()
    rx = {k: (lc.Regex(ML_PAT[k]) if k in mode else None) for k in "SCE"}
    ox = {k: (orc.Regex(ML_PAT[k]) if k in mode else None) for k in "SCE"}
    off, ln, fl, ctr = eng.multiline_split(buf, rx["S"], rx["C"], rx["E"], discard)
    eo, el, ef, ectr = orc.multiline_split(buf, ox["S"], ox["C"], ox["E"], discard)
    assert np.array_equal(off, eo) and np.array_equal(ln, el), (mode, discard, bytes(buf[:200]))
    assert np.array_equal(fl, ef), (mode, discard)
    assert ctr.tolist() == ectr.tolist(), (mode, discard)


@pytest.mark.parametrize("mode", ML_MODES)
@pytest.mark.parametrize("discard", [False, True])
def test_multiline_random_soups(eng, mode, discard):
    rng = random.Random(hash(mode) & 0xFFF)
    vocab = [BEGIN, CONT, END, UNM, b"", b"  at x", b"...1 more"]
    for trial in range(60):
        k = rng.choice([0, 1, 2, 3, 5, 8, 40, 300])
        lines = [rng.choice(vocab) for _ in range(k)]
        s = b"\n".join(lines)
        if rng.random() < 0.4 and s:
            s += b"\n"
        if not s:
            continue
        _ml_check(eng, np.frombuffer(s, np.uint8), mode, discard)


@pytest.mark.parametrize("mode", ML_MODES)
def test_multiline_large_java_trace(eng, mode):
    from loongcollector_b200 import synth
    buf = synth.java_stack_records(4000, seed=11)[0]
    # the generator's own start pattern is exercised in bench; here the unit-test trio runs over the same bytes
    _ml_check(eng, buf, mode, False)
    _ml_check(eng, buf, mode, True)


def test_multiline_reference_fixtures_flat(eng):
    """Replays the reference's ~50 multiline unit-test inputs through the flat C-ABI call."""
    from tests.golden_util import load_cases
    lc = _lc()
    n = 0
    for case in load_cases("multiline"):
        cfg = case["pipeline"][0]["config"]
        pats = [cfg.get("StartPattern", ""), cfg.get("ContinuePattern", ""), cfg.get("EndPattern", "")]
        rx = [lc.Regex(p) if p else None for p in pats]
        ox = [orc.Regex(p) if p else None for p in pats]
        discard = cfg.get("UnmatchedContentTreatment") == "discard"
        for ev in case["input"]["events"]:
            val = ev["contents"]["content"].encode()
            buf = np.frombuffer(val, np.uint8)
            off, ln, fl, ctr = eng.multiline_split(buf, rx[0], rx[1], rx[2], discard)
            eo, el, ef, ectr = orc.multiline_split(buf, ox[0], ox[1], ox[2], discard)
            assert np.array_equal(off, eo) and np.array_equal(ln, el) and np.array_equal(fl, ef), case["name"]
            assert ctr.tolist() == ectr.tolist()
            n += 1
    assert n >= 50


# ------------------------------------------------------------------------------------------- delimiter
def _csv_lines(rng, n, sep, quote):
    out = []
    for _ in range(n):
        k = rng.randint(0, 8)
        cells = []
        for _ in range(k):
            r = rng.random()
            body = "".join(rng.choice("ab1 ,|@'\"x") for _ in range(rng.randint(0, 6)))
            if r < 0.25:
                q = chr(quote)
                cells.append(q + body.replace(q, q + q) + q)
            elif r < 0.35:
                cells.append(chr(quote) + body)  # often malformed
            else:
                cells.append(body.replace(chr(quote), "").replace(sep.decode(), ""))
        line = sep.decode().join(cells)
        if rng.random() < 0.2:
            line = " " * rng.randint(1, 3) + line + " " * rng.randint(0, 2) + ("\r" if rng.random() < 0.5 else "")
        out.append(line.encode())
    return out


@pytest.mark.parametrize("sep,quote", [(b",", ord('"')), (b",", ord("'")), (b"|", ord("'")), (b"@@", ord('"')),
                                       (b"||a", ord('"')), (b",", ord(",")), (b"\t", ord('"'))])
@pytest.mark.parametrize("extend,allow_short", [(True, True), (False, True), (False, False)])
def test_delim_matches_oracle(eng, sep, quote, extend, allow_short):
    rng = random.Random(len(sep) * 7 + quote)
    lines = _csv_lines(rng, 3000, sep, quote) + [b"", b"   ", b" \r", b"a", sep, sep * 3]
    base, off, ln = _events(lines)
    for nkeys, mf in ((4, 5), (4, 16), (1, 2), (9, 3), (4, 33), (20, 64)):
        got = eng.delim_parse(base, off, ln, sep, quote, nkeys, extend, allow_short, mf)
        want = orc.delim_parse_batch(base, off, ln, sep, quote, nkeys, extend, allow_short, mf)
        for g, w, name in zip(got, want, ("status", "nfields", "f_off", "f_len", "f_dq")):
            assert np.array_equal(g, w), (name, sep, quote, extend, allow_short, nkeys, mf)


# ------------------------------------------------------------------------------------------- kernel variants
@pytest.mark.timeout(300)
@pytest.mark.parametrize("variant", ["basic", "generic", "fast", "fast2", "tdfa"])
def test_regex_kernel_variants_agree(variant, monkeypatch):
    """The baseline (tables in global memory) and generic (smem interpreter) kernels stay parity-checked too."""
    lc = _lc()
    monkeypatch.setenv("LC_B200_REGEX_KERNEL", variant)
    e = lc.Engine(0)
    try:
        rng = random.Random(17)
        lines = _noise_lines(rng, 1500) + _nginx_lines(rng, 1500) + [b"x" * 5000, b"[" + b"y" * 3000 + b"] [z] q"]
        for pattern in PATTERNS[:6]:
            _check_parse(e, pattern, lines)
        # one event beyond the 16-bit capture registers of the stride-2 / single-pass kernels: they must hand the
        # whole batch to a kernel with 32-bit slots
        huge = lines[:200] + [b"GET /" + b"a" * 70000 + b" 200", b"k=" + b"v" * 66000]
        for pattern in (PATTERNS[0], r"(\w+) /(\w+) (\d+)", r"(\w)=(.*)"):
            _check_parse(e, pattern, huge)
    finally:
        e.close()


def test_regex_parse_pipelined_host_path_full_size(eng):
    """> 96 MB through the host-pointer API takes the chunked H2D / kernel / D2H pipeline; every row is checked."""
    lc = _lc()
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(600000, seed=4242, line_bytes=256)
    rx = lc.Regex(synth.NGINX_PATTERN)
    st, co, cl = eng.regex_parse(rx, buf, off, ln, 10)
    est, eco, ecl = orc.regex_parse_batch(orc.Regex(synth.NGINX_PATTERN), buf, off, ln, 10)
    assert np.array_equal(st, est) and np.array_equal(co, eco) and np.array_equal(cl, ecl)
    # ragged natural-length lines, same path
    buf, off, ln = synth.nginx_lines(700000, seed=4243, line_bytes=None)
    st, co, cl = eng.regex_parse(rx, buf, off, ln, 10)
    est, eco, ecl = orc.regex_parse_batch(orc.Regex(synth.NGINX_PATTERN), buf, off, ln, 10)
    assert np.array_equal(st, est) and np.array_equal(co, eco) and np.array_equal(cl, ecl)


def test_regex_ragged_batch_long_lines_and_length_order(monkeypatch):
    """Zipf-like ragged batch: lines beyond the shared-memory label budget keep their labels in the global slab;
    the opt-in length-bucket visiting order must not change any result."""
    lc = _lc()
    from loongcollector_b200 import synth
    buf, off, ln, kind = synth.zipf_mixed_lines(6000, seed=99, pool=600)
    rx = lc.Regex(synth.NGINX_PATTERN)
    o = orc.Regex(synth.NGINX_PATTERN)
    sel = ~kind
    est, eco, ecl = orc.regex_parse_batch(o, buf, off[sel], ln[sel], 10)
    for flag in ("0", "1"):
        monkeypatch.setenv("LC_B200_LENGTH_ORDER", flag)
        e = lc.Engine(0)
        try:
            st, co, cl = e.regex_parse(rx, buf, off[sel], ln[sel], 10)
        finally:
            e.close()
        assert np.array_equal(st, est) and np.array_equal(co, eco) and np.array_equal(cl, ecl), flag


# ------------------------------------------------------------------------------------------- BASELINE full sizes
def test_full_size_c2_every_row_bit_exact(eng):
    """C2 at BASELINE size (4 Mi x 256 B): the lines are samples of a 16 Ki-line pool, so the oracle's result on the
    pool expands to the exact expected table of the whole batch -- every status / offset / length is compared."""
    import torch
    lc = _lc()
    from loongcollector_b200 import synth
    n = 4 * 1024 * 1024
    buf, off, ln = synth.nginx_lines(n)
    pool = synth.nginx_pool(n)
    idx = synth.pool_index(len(pool), n, synth.DEFAULT_SEED + 1)
    pbuf, poff, plen = _events([p[:-1] for p in pool])
    o = orc.Regex(synth.NGINX_PATTERN)
    pst, pco, pcl = orc.regex_parse_batch(o, pbuf, poff, plen, 10)
    exp_st = pst[idx]
    rel = (pco.astype(np.int64) - poff[:, None].astype(np.int64)) * (pst == 0)[:, None]
    exp_co = ((rel[idx] + off[:, None].astype(np.int64)) * (exp_st == 0)[:, None]).astype(np.uint32)
    exp_cl = pcl[idx]
    rx = lc.Regex(synth.NGINX_PATTERN)
    G = rx.ngroups
    d_buf = torch.from_numpy(buf).cuda()
    d_off = torch.from_numpy(off.view(np.int32)).cuda()
    d_len = torch.from_numpy(ln.view(np.int32)).cuda()
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_co = torch.empty(n * G, dtype=torch.int32, device="cuda")
    d_cl = torch.empty(n * G, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    eng.regex_parse_dev(rx, d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, 10, d_st.data_ptr(),
                        d_co.data_ptr(), d_cl.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(d_st.cpu().numpy(), exp_st)
    assert np.array_equal(d_co.cpu().numpy().view(np.uint32).reshape(n, G), exp_co)
    assert np.array_equal(d_cl.cpu().numpy().view(np.uint32).reshape(n, G), exp_cl)
    # size-independent properties: captures are ordered, disjoint and inside their line
    co = exp_co.astype(np.int64)
    ok = exp_st == 0
    assert np.all(co[ok, 0] >= off[ok]) and np.all(co[ok, -1] + exp_cl[ok, -1] <= off[ok].astype(np.int64) + ln[ok])
    assert np.all(co[ok, 1:] >= co[ok, :-1] + exp_cl[ok, :-1])


def test_full_size_c1_split(eng):
    """C1 at BASELINE size (1 Mi x 512 B): the line table is known in closed form."""
    from loongcollector_b200 import synth
    n = 1 << 20
    buf, off, ln = synth.newline_lines(n, 512)
    g_off, g_len = eng.split_lines(buf, cap=n + 8)
    assert np.array_equal(g_off, off) and np.array_equal(g_len, ln)


def test_full_size_c3_multiline_records(eng):
    """C3 at BASELINE size (1 Mi Java records, ~1.8 KB): with a start pattern only, every record is one event that
    begins at a record start and runs to the byte before the next one; counters follow in closed form."""
    lc = _lc()
    from loongcollector_b200 import synth
    nrec = 1 << 20
    buf, nlines, _ = synth.java_stack_records(nrec)
    start = lc.Regex(synth.JAVA_START_PATTERN)
    off, ln, fl, ctr = eng.multiline_split(buf, start, None, None, False, cap=nrec + 8)
    assert off.size == nrec and ctr.tolist() == [nrec, nlines, 0]
    # record k starts where record k-1 ended + 1 ('\n'); the last one keeps the trailing '\n' (reference quirk)
    ends = off.astype(np.int64) + ln
    assert off[0] == 0 and np.array_equal(off[1:], ends[:-1] + 1) and ends[-1] == buf.size
    assert np.all(buf[off] == ord("[")) and np.all(fl[:-1] == 2) and fl[-1] == 3


def test_regex_match_boolean_matches_oracle(eng):
    """lc_regex_match (ProcessorFilterNative's arithmetic): reverse pass only, one boolean per value."""
    lc = _lc()
    rng = random.Random(31)
    lines = _noise_lines(rng, 2000) + _nginx_lines(rng, 1500) + [b"100", b"2008-08-08", b"192.168.1.1", b"x" * 3000]
    base, off, ln = _events(lines)
    ip = r"((2[0-4]\d|25[0-5]|[01]?\d\d?)\.){3}(2[0-4]\d|25[0-5]|[01]?\d\d?)"
    for p in PATTERNS[:6] + [r"\d+", r"20\d{1,2}-\d{1,2}-\d{1,2}", r"\S+", ip, r".*value1", r"^no-agent$"]:
        got = eng.regex_match(lc.Regex(p), base, off, ln)
        want = orc.regex_match_batch(orc.Regex(p), base, off, ln)
        assert np.array_equal(got, want), p


# ------------------------------------------------------------------------------------------- unaligned arenas
@pytest.mark.parametrize("shift", [1, 7, 16, 77])
def test_dev_entry_points_with_unaligned_base(eng, shift):
    """*_dev entry points take an arena that is already in HBM; nothing says it starts on a 16-byte boundary (a
    SourceBuffer value can start anywhere inside its chunk).  Every kernel that reads aligned 16-byte chunks has to
    fold the misalignment of `base` itself into its addressing -- checked here for split, regex parse (single-pass
    and two-pass kernels), multiline and delimiter."""
    import torch
    lc = _lc()
    from loongcollector_b200 import synth
    dev = torch.device("cuda", 0)

    def shifted(buf):
        t = torch.zeros(buf.size + shift + 64, dtype=torch.uint8, device=dev)
        t[shift:shift + buf.size] = torch.from_numpy(np.ascontiguousarray(buf)).to(dev)
        return t, t.data_ptr() + shift

    def dput(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    # split + regex parse over natural-length nginx lines
    buf, off, ln = synth.nginx_lines(5000, seed=shift, line_bytes=None)
    keep, ptr = shifted(buf)
    n = off.size
    d_off = torch.empty(n + 8, dtype=torch.int32, device=dev)
    d_len = torch.empty(n + 8, dtype=torch.int32, device=dev)
    got_n = eng.split_lines_dev(ptr, buf.size, 10, d_off.data_ptr(), d_len.data_ptr(), n + 8)
    assert got_n == n
    assert np.array_equal(d_off[:n].cpu().numpy().view(np.uint32), off)
    assert np.array_equal(d_len[:n].cpu().numpy().view(np.uint32), ln)
    o = orc.Regex(synth.NGINX_PATTERN)
    est, eco, ecl = orc.regex_parse_batch(o, buf, off, ln, 10)
    rx = lc.Regex(synth.NGINX_PATTERN)
    G = rx.ngroups
    for variant in ("tdfa", "fast2", "generic"):
        os.environ["LC_B200_REGEX_KERNEL"] = variant
        try:
            e2 = lc.Engine(0)
            st = torch.empty(n, dtype=torch.uint8, device=dev)
            co = torch.empty(n * G, dtype=torch.int32, device=dev)
            cl = torch.empty(n * G, dtype=torch.int32, device=dev)
            e2.regex_parse_dev(rx, ptr, buf.size, d_off.data_ptr(), d_len.data_ptr(), n, 10, st.data_ptr(),
                               co.data_ptr(), cl.data_ptr())
            e2.sync()
            assert np.array_equal(st.cpu().numpy(), est), variant
            assert np.array_equal(co.cpu().numpy().view(np.uint32).reshape(n, G), eco), variant
            assert np.array_equal(cl.cpu().numpy().view(np.uint32).reshape(n, G), ecl), variant
            e2.close()
        finally:
            os.environ.pop("LC_B200_REGEX_KERNEL", None)
    # multiline
    jb, _, _ = synth.java_stack_records(400, seed=shift)
    keep2, jptr = shifted(jb)
    s = lc.Regex(synth.JAVA_START_PATTERN)
    e_off, e_len, e_fl, ectr = orc.multiline_split(jb, orc.Regex(synth.JAVA_START_PATTERN), None, None, False)
    cap = e_off.size + 8
    m_off = torch.empty(cap, dtype=torch.int32, device=dev)
    m_len = torch.empty(cap, dtype=torch.int32, device=dev)
    m_fl = torch.empty(cap, dtype=torch.uint8, device=dev)
    k, ctr = eng.multiline_split_dev(jptr, jb.size, s, None, None, False, m_off.data_ptr(), m_len.data_ptr(),
                                     m_fl.data_ptr(), cap)
    assert k == e_off.size and ctr.tolist() == ectr.tolist()
    assert np.array_equal(m_off[:k].cpu().numpy().view(np.uint32), e_off)
    assert np.array_equal(m_len[:k].cpu().numpy().view(np.uint32), e_len)
    assert np.array_equal(m_fl[:k].cpu().numpy(), e_fl)
    # delimiter
    cb, c_off, c_len = synth.csv_lines(3000, seed=shift)
    keep3, cptr = shifted(cb)
    MF = 11
    want = orc.delim_parse_batch(cb, c_off, c_len, b",", ord('"'), 10, True, True, MF)
    nn = c_off.size
    d_co, d_cl = dput(c_off.view(np.int32)), dput(c_len.view(np.int32))
    st4 = torch.empty(nn, dtype=torch.uint8, device=dev)
    nf4 = torch.empty(nn, dtype=torch.int32, device=dev)
    fo4 = torch.empty(nn * MF, dtype=torch.int32, device=dev)
    fl4 = torch.empty(nn * MF, dtype=torch.int32, device=dev)
    fd4 = torch.empty(nn * MF, dtype=torch.int32, device=dev)
    eng.delim_parse_dev(cptr, cb.size, d_co.data_ptr(), d_cl.data_ptr(), nn, b",", ord('"'), 10, True, True, MF,
                        st4.data_ptr(), nf4.data_ptr(), fo4.data_ptr(), fl4.data_ptr(), fd4.data_ptr())
    eng.sync()
    got = (st4.cpu().numpy(), nf4.cpu().numpy().view(np.uint32), fo4.cpu().numpy().view(np.uint32).reshape(nn, MF),
           fl4.cpu().numpy().view(np.uint32).reshape(nn, MF), fd4.cpu().numpy().view(np.uint32).reshape(nn, MF))
    for g, w, name in zip(got, want, ("status", "nfields", "f_off", "f_len", "f_dq")):
        assert np.array_equal(g, w), name


def test_regex_every_length_at_every_alignment(eng):
    """The staged single-pass kernel decomposes a line into an optional head chunk, fully paired 16-byte chunks and
    an optional tail chunk (odd first / last byte peeled) in the line's own 16-byte frame: every line length 0..100
    at every start alignment 0..15, matching and non-matching, through the device entry point."""
    import torch
    lc = _lc()
    rng = random.Random(1234)
    dev = torch.device("cuda", 0)
    patterns = [r"(\w*)-(\d*)(x?)(.*)", r"([a-z]+)(?: (\d+))*", r'"([^"]*)" "([^"]*)"(.*)', r"(a|ab)(c|bcd)*(d*)(.*)"]
    alpha = 'ab cd-12x"'
    pieces, offs, lens = [], [], []
    at = 0
    for length in range(0, 101):
        for align in range(16):
            pad = (align - at) % 16
            pieces.append(b"#" * pad)
            at += pad
            kind = rng.random()
            if kind < 0.4:
                body = ("ab-%s%s" % ("1" * rng.randint(0, 3), "x" * rng.randint(0, 1))).encode()
            elif kind < 0.6:
                body = b'"' + b"q" * rng.randint(0, 5) + b'" "' + b"r" * rng.randint(0, 5) + b'"'
            else:
                body = b""
            line = (body + "".join(rng.choice(alpha) for _ in range(length)).encode())[:length]
            pieces.append(line)
            offs.append(at)
            lens.append(len(line))
            at += len(line)
    base = np.frombuffer(b"".join(pieces) + b"#" * 32, np.uint8)
    off = np.array(offs, np.uint32)
    ln = np.array(lens, np.uint32)
    n = off.size
    d_base = torch.from_numpy(base.copy()).to(dev)
    d_off = torch.from_numpy(off.view(np.int32).copy()).to(dev)
    d_len = torch.from_numpy(ln.view(np.int32).copy()).to(dev)
    for pattern in patterns:
        rx, o = lc.Regex(pattern), orc.Regex(pattern)
        G = rx.ngroups
        est, eco, ecl = orc.regex_parse_batch(o, base, off, ln, G)
        st = torch.empty(n, dtype=torch.uint8, device=dev)
        co = torch.empty(n * G, dtype=torch.int32, device=dev)
        cl = torch.empty(n * G, dtype=torch.int32, device=dev)
        eng.regex_parse_dev(rx, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n, G, st.data_ptr(),
                            co.data_ptr(), cl.data_ptr())
        eng.sync()
        bad = np.nonzero(st.cpu().numpy() != est)[0]
        assert bad.size == 0, (pattern, [(int(ln[i]), int(off[i]) % 16) for i in bad[:5]])
        assert np.array_equal(co.cpu().numpy().view(np.uint32).reshape(n, G), eco), pattern
        assert np.array_equal(cl.cpu().numpy().view(np.uint32).reshape(n, G), ecl), pattern
        assert 0 < int((est == 0).sum()) < n, pattern  # both verdicts occur


def test_regex_assertions_inside_the_pattern(eng):
    """Word boundaries and line anchors in the middle of a pattern: the single-pass tables carry the kind of the
    previous byte in the state (no kernel-side context logic), values contain embedded line separators."""
    rng = random.Random(77)
    patterns = [r"(\w+)\b.(\w+)\b(.*)", r"(.*)\bat\b(.*)", r"(a+)$.^(b+)(.*)", r"(\S+)$\s^(\S+)(?:$\s^(\S+))?",
                r"^(\w+) (\w+)$", r"(.*?)\b(\d+)\b(.*)", r"(\w+)\B(\w)(.*)", r"(.*?)a\Bb(.*)"]
    # (no \\r: boost treats \\r\\n as one separator, the PCRE2 oracle does not -- tests/test_regex_compiler_cpu.py pins that
    #  corner on the CPU tier; a trailing separator is avoided for the mid-pattern '^' corner described there)
    alpha = "ab at 12\n_-"
    lines = [b"ab cd ef", b"x at y", b"aa\nbb tail", b"w1\nw2\nw3", b"foo 12 bar", b"at", b""]
    for _ in range(3000):
        lines.append("".join(rng.choice(alpha) for _ in range(rng.randint(0, 40))).encode().rstrip(b"\n"))
    for pattern in patterns:
        _check_parse(eng, pattern, lines)


# ------------------------------------------------------------------------------------------- f3: last incomplete log
def _host_multiline_regs(cfg):
    """the (start, end) regexes of a reader for this Multiline config (MultilineOptions.cpp:125-160,205-222)"""
    lc = _lc()

    def reg(p):
        if not p:
            return None
        if p.endswith("$"):
            p = p[:-1]
        while p.endswith(".*"):
            p = p[:-2]
        return lc.Regex(p) if p else None
    return reg(cfg.get("StartPattern")), reg(cfg.get("EndPattern"))


def test_remove_last_incomplete_log_reference_fixtures(eng):
    """every case of core/unittest/reader/RemoveLastIncompleteLogUnittest.cpp (raw-text reader)"""
    with open(os.path.join(HERE, "golden", "ref_rollback.json"), encoding="utf-8") as f:
        cases = json.load(f)
    assert len(cases) == 29
    for c in cases:
        start, end = _host_multiline_regs(c["config"])
        if not c["input"]:
            continue  # size == 0 returns before anything is computed
        keep, rb = eng.remove_last_incomplete_log(c["input"].encode(), start, end, True)
        assert (keep, rb) == (c["expect_size"], c["expect_rollback"]), (c["name"], c["title"])


@pytest.mark.parametrize("mode", ["", "S", "E", "SE"])
def test_remove_last_incomplete_log_random_chunks_match_oracle(eng, mode):
    lc = _lc()
    rng = random.Random(len(mode) * 31 + 7)
    s_pat, e_pat = r"Exception", r"\s*\.\.\.\d+ more"
    start = lc.Regex(s_pat) if "S" in mode else None
    end = lc.Regex(e_pat) if "E" in mode else None
    o_start = orc.Regex(s_pat) if "S" in mode else None
    o_end = orc.Regex(e_pat) if "E" in mode else None
    pieces = [BEGIN, CONT, END, UNM, b"", b"x"]
    for trial in range(150):
        k = rng.randint(0, 12) if trial % 10 else rng.randint(2000, 6000)
        lines = [rng.choice(pieces) for _ in range(k)]
        buf = b"\n".join(lines) + (b"\n" if rng.random() < 0.5 else b"")
        if rng.random() < 0.1:
            buf = b"\n" * rng.randint(1, 3) + buf
        if not buf:
            continue
        got = eng.remove_last_incomplete_log(buf, start, end, True)
        want = orc.remove_last_incomplete_log(buf, o_start, o_end, True)
        assert got == want, (mode, buf[-200:])
    assert eng.remove_last_incomplete_log(b"a\nb", start, end, False)[0] == 3


def test_split_reports_too_large_beyond_2_pow_30_pieces(eng):
    """The line numbers keep 30 bits of piece count: a buffer with more split chars than that must be refused
    (LC_ERR_TOO_LARGE), not wrapped silently."""
    import ctypes as C

    import torch
    lc = _lc()
    n = (1 << 30) + 4096
    d = torch.full((n,), 10, dtype=torch.uint8, device="cuda")
    off = torch.empty(1024, dtype=torch.int32, device="cuda")
    ln = torch.empty(1024, dtype=torch.int32, device="cuda")
    got = C.c_uint64(0)
    rc = lc.lib().lc_split_lines_dev(eng._h, C.c_void_p(d.data_ptr()), n, 10, C.c_void_p(off.data_ptr()),
                                     C.c_void_p(ln.data_ptr()), 1024, C.byref(got))
    assert rc == lc.capi.LC_ERR_TOO_LARGE, (rc, got.value)
    del d
