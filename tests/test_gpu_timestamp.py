"""GPU tier: ProcessorParseTimestampNative on the device.  lc_timestamp_parse_dev, lc_timestamp_parse_capture_dev and
lc_timestamp_parse equal the host build of the same statements (tests/emul/timestamp.py) and the flat C oracle
(oracle/timestamp.py) event for event -- status, sec, nsec -- and in their counters.  Outputs are poisoned and followed
by guard words; the last value ends at the end of its device buffer."""
import os
import random
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import timestamp as ots  # noqa: E402
from tests import timestamp_cases as tc  # noqa: E402
from tests.emul import timestamp as ets  # noqa: E402

GUARD = 64
POISON = 0xA5


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


@pytest.fixture(params=tc.ZONES)
def zone(request):
    saved = os.environ.get("TZ")
    os.environ["TZ"] = request.param
    time.tzset()
    yield request.param
    if saved is None:
        os.environ.pop("TZ", None)
    else:
        os.environ["TZ"] = saved
    time.tzset()


def _dev_base(base):
    """base on the device so that its last byte is the last byte of the allocation the allocator handed out"""
    import torch
    n = max(base.size, 1)
    cap = (n + 511) // 512 * 512
    buf = torch.full((cap,), 0x37, dtype=torch.uint8, device="cuda")
    if base.size:
        buf[cap - base.size:] = torch.from_numpy(base.copy()).cuda()
    return buf, buf.data_ptr() + cap - base.size


def _outputs(n):
    import torch
    sec = torch.full((n + GUARD,), -0x5A5A5A5A5A5A5A5B, dtype=torch.int64, device="cuda")
    ns = torch.full((n + GUARD,), -0x5A5A5A5B, dtype=torch.int32, device="cuda")
    st = torch.full((n + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    cnt = torch.full((5 + GUARD,), -1, dtype=torch.int64, device="cuda")
    return sec, ns, st, cnt


def _fetch(eng, n, sec, ns, st, cnt):
    eng.sync()
    s, q, t, c = sec.cpu().numpy(), ns.cpu().numpy().view(np.uint32), st.cpu().numpy(), cnt.cpu().numpy()
    assert (s[n:] == -0x5A5A5A5A5A5A5A5B).all() and (q[n:] == np.uint32(0xA5A5A5A5)).all(), "wrote past sec / nsec"
    assert (t[n:] == POISON).all() and (c[5:] == -1).all(), "wrote past status / counters"
    return t[:n], s[:n], q[:n], c[:5].astype(np.uint64)


def run_dev(eng, ts, base, off, ln, grp, now, di):
    import torch
    n = off.size
    buf, d_base = _dev_base(base)
    d_off, d_len = torch.from_numpy(off.view(np.int32)).cuda(), torch.from_numpy(ln.view(np.int32)).cuda()
    d_grp = torch.from_numpy(grp.view(np.int32)).cuda()
    sec, ns, st, cnt = _outputs(n)
    eng.timestamp_parse_dev(ts, d_base, base.size, d_off.data_ptr(), d_len.data_ptr(), n, d_grp.data_ptr(),
                            grp.size - 1, now, di, sec.data_ptr(), ns.data_ptr(), st.data_ptr(), cnt.data_ptr())
    return _fetch(eng, n, sec, ns, st, cnt)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _diff(a, b, groups):
    """the first differing event of two (status, sec, nsec, counters) results, for the assertion message"""
    vals = [v for g in groups for v in g]
    for k, name in enumerate(("status", "sec", "nsec")):
        bad = np.nonzero(a[k] != b[k])[0]
        if bad.size:
            i = int(bad[0])
            return "%s of event %d (%r): %s != %s" % (name, i, vals[i], a[k][i], b[k][i])
    return "counters %s != %s" % (a[3].tolist(), b[3].tolist())


def _check(eng, fmt, sy, adj, now, di, groups, host=True):
    import loongcollector_b200 as lc
    base, off, ln, grp = ets.layout(groups)
    want = ots.process(fmt, sy, adj, base, off, ln, grp, now, di, "c")
    emu = ets.Compiled(fmt, sy, adj).parse(base, off, ln, grp, now, di, 32)
    assert _same(emu, want), (fmt, _diff(emu, want, groups))
    ts = lc.Timestamp(fmt, sy, adj)
    got = run_dev(eng, ts, base, off, ln, grp, now, di)
    assert _same(got, want), (fmt, _diff(got, want, groups))
    if host:
        got = eng.timestamp_parse(ts, base, off, ln, grp, now, di)
        assert _same(got, want), (fmt, _diff(got, want, groups))


def test_cases_equal_emulation_and_oracle(eng, zone):
    for name, fmt, sy, adj, now, di, groups in tc.all_cases():
        _check(eng, fmt, sy, adj, now, di, groups, host=name.startswith("cache"))


@pytest.mark.parametrize("fmt,per_sec", [("%Y-%m-%d %H:%M:%S.%f", 1), ("%Y-%m-%d %H:%M:%S.%f", 1000),
                                         ("%Y-%m-%d %H:%M:%S", 1), ("%d/%b/%Y:%H:%M:%S", 7)])
def test_group_sizes(eng, fmt, per_sec):
    """groups of 1 to 100 000 events in one call, and thousands of small groups"""
    rng = random.Random(per_sec)
    sizes = [1, 2, 31, 32, 33, 100, 1000, 100000] + [rng.randint(1, 40) for _ in range(3000)]
    head = fmt.replace(".%f", "")
    groups = []
    for gs in sizes:
        g = []
        t = 1699990000 + rng.randint(0, 5000)
        for k in range(gs):
            if k % per_sec == 0:
                t += 1
                sec = time.strftime(head, time.gmtime(t)).encode()
            v = sec + (b".%d" % rng.randrange(1000) if head != fmt else b"")
            r = rng.random()
            g.append(None if r < 0.01 else (v[:-2] if r < 0.02 else v))
        groups.append(g)
    _check(eng, fmt, -1, 0, tc.NOW, 43200, groups)


def test_capture_column_of_regex_result(eng, zone):
    """the nginx time capture of lc_regex_parse_dev, read in place; rows the regex did not parse are key_not_found"""
    import torch
    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    buf, off, ln = synth.nginx_lines(20000, seed=5)
    rx = lc.Regex(synth.NGINX_PATTERN)
    G = rx.ngroups
    n = off.size
    d_buf, d_base = _dev_base(buf)
    d_off = torch.from_numpy(off.astype(np.uint32).view(np.int32)).cuda()
    d_len = torch.from_numpy(ln.astype(np.uint32).view(np.int32)).cuda()
    rs = torch.zeros(n, dtype=torch.uint8, device="cuda")
    co = torch.zeros(n * G, dtype=torch.int32, device="cuda")
    cl = torch.zeros(n * G, dtype=torch.int32, device="cuda")
    eng.regex_parse_dev(rx, d_base, buf.size, d_off.data_ptr(), d_len.data_ptr(), n, G, rs.data_ptr(), co.data_ptr(),
                        cl.data_ptr())
    eng.sync()
    h_rs, h_co, h_cl = rs.cpu().numpy(), co.cpu().numpy().view(np.uint32), cl.cpu().numpy().view(np.uint32)
    assert (h_rs != 0).any() and (h_rs == 0).any()
    k = synth.NGINX_KEYS.index("time")
    rng = random.Random(1)
    cuts = [0] + sorted(rng.sample(range(1, n), 40)) + [n]
    grp = np.array(cuts, np.uint32)
    fmt = "%d/%b/%Y:%H:%M:%S"
    for sy, adj, now in ((-1, 0, tc.NOW), (0, 3600, tc.NOW_JAN1)):
        ts = lc.Timestamp(fmt, sy, adj)
        sec, ns, st, cnt = _outputs(n)
        d_grp = torch.from_numpy(grp.view(np.int32)).cuda()
        eng.timestamp_parse_capture_dev(ts, d_base, buf.size, rs.data_ptr(), co.data_ptr(), cl.data_ptr(), G, k, n,
                                        d_grp.data_ptr(), grp.size - 1, now, -1, sec.data_ptr(), ns.data_ptr(),
                                        st.data_ptr(), cnt.data_ptr())
        got = _fetch(eng, n, sec, ns, st, cnt)
        v_off = np.where(h_rs == 0, h_co.reshape(n, G)[:, k], 0).astype(np.uint32)
        v_len = np.where(h_rs == 0, h_cl.reshape(n, G)[:, k], ets.NO_KEY).astype(np.uint32)
        want = ots.process(fmt, sy, adj, buf, v_off, v_len, grp, now, -1, "c")
        assert _same(got, want)
        assert int(got[3][0]) == int((h_rs != 0).sum())


def test_refusals(eng):
    import loongcollector_b200 as lc
    for fmt in ("%c", "%x %Y", "%X"):
        with pytest.raises(lc.LcError):
            lc.Timestamp(fmt)
    ts = lc.Timestamp("%Y")
    base, off, ln, grp = ets.layout([[b"2020"]])
    with pytest.raises(lc.LcError):
        eng.timestamp_parse(ts, base, off, np.array([5], np.uint32), grp, tc.NOW)  # past the buffer
    with pytest.raises(lc.LcError):
        eng.timestamp_parse(ts, base, off, ln, np.array([0, 2], np.uint32), tc.NOW)  # groups do not cover n
