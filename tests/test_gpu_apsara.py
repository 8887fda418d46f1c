"""GPU tier of the Apsara parse: lc_apsara_parse and lc_apsara_parse_dev equal the host build of the device functions
and the C oracle on every output and counter, on poisoned outputs with guard words; the capacity refusal writes no
entry; an event past the buffer is refused."""
import os
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import apsara as oap  # noqa: E402
from tests import apsara_cases as ac  # noqa: E402
from tests.emul import apsara as eap  # noqa: E402
from tests.emul import timestamp as ets  # noqa: E402

NOW = 1700000000 + 43200
POISON = 0xA5


@pytest.fixture
def utc():
    old = os.environ.get("TZ")
    os.environ["TZ"] = "UTC"
    time.tzset()
    yield
    if old is None:
        os.environ.pop("TZ", None)
    else:
        os.environ["TZ"] = old
    time.tzset()


def _eng():
    import loongcollector_b200 as lc
    return lc, lc.Engine(0)


def _same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_host_call_equals_emulation_and_oracle(utc):
    lc, eng = _eng()
    groups = ac.random_groups(11, 200) + [ac.corner_values(), [None, b""]]
    base, off, ln, grp = ets.layout(groups)
    for adj, interval in ((0, -1), (8 * 3600, 43205)):
        ap = lc.Apsara("content", adj)
        got = eng.apsara_parse(ap, base, off, ln, grp, NOW, interval)
        want = oap.process("content", adj, base, off, ln, grp, NOW, interval)
        _same(got, want)
        _same(got, eap.parse("content", adj, base, off, ln, grp, NOW, interval))
    eng.close()


def test_dev_call_guards_and_capacity(utc):
    import torch
    lc, eng = _eng()
    groups = ac.random_groups(12, 300)
    base, off, ln, grp = ets.layout(groups)
    n, G = off.size, 64
    want = oap.process("content", 0, base, off, ln, grp, NOW, -1)
    m = int(want[4][-1])
    dev = lambda a: torch.from_numpy(np.array(a)).cuda()  # noqa: E731
    d_base, d_off, d_len, d_grp = dev(base), dev(off.view(np.int32)), dev(ln.view(np.int32)), dev(grp.view(np.int32))

    def guarded(nbytes):
        return torch.full((nbytes + 2 * G,), POISON, dtype=torch.uint8, device="cuda")

    bufs = {"st": guarded(n), "sec": guarded(8 * n), "ns": guarded(4 * n), "us": guarded(8 * n),
            "first": guarded(8 * (n + 1)), "ent": guarded(16 * m), "cnt": guarded(40)}
    ptr = {k: v.data_ptr() + G for k, v in bufs.items()}
    ap = lc.Apsara("content", 0)
    # the capacity refusal writes no entry
    with pytest.raises(lc.LcError) as ei:
        eng.apsara_parse_dev(ap, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n,
                             d_grp.data_ptr(), grp.size - 1, NOW, -1, ptr["st"], ptr["sec"], ptr["ns"], ptr["us"],
                             ptr["first"], ptr["ent"], m - 1, ptr["cnt"])
    assert ei.value.code == lc.capi.LC_ERR_CAPACITY
    assert bool((bufs["ent"] == POISON).all())
    got_m = eng.apsara_parse_dev(ap, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n,
                                 d_grp.data_ptr(), grp.size - 1, NOW, -1, ptr["st"], ptr["sec"], ptr["ns"], ptr["us"],
                                 ptr["first"], ptr["ent"], m, ptr["cnt"])
    assert got_m == m
    host = {k: v.cpu().numpy() for k, v in bufs.items()}
    for v in host.values():
        assert (v[:G] == POISON).all() and (v[-G:] == POISON).all()
    got = (host["st"][G:-G], host["sec"][G:-G].view(np.int64), host["ns"][G:-G].view(np.uint32),
           host["us"][G:-G].view(np.int64), host["first"][G:-G].view(np.uint64),
           host["ent"][G:-G].view(np.uint32).reshape(-1, 4), host["cnt"][G:-G].view(np.uint64))
    _same(got, want)
    # an event past the buffer is refused without being read
    bad = dev(np.array([base.size], np.uint32).view(np.int32))
    with pytest.raises(lc.LcError) as ei:
        eng.apsara_parse_dev(ap, d_base.data_ptr(), base.size - 1, d_off.data_ptr(), bad.data_ptr(), 1,
                             d_grp.data_ptr(), 1, NOW, -1, ptr["st"], ptr["sec"], ptr["ns"], ptr["us"], ptr["first"],
                             ptr["ent"], m, ptr["cnt"])
    assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG
    eng.close()


def test_million_lines(utc):
    lc, eng = _eng()
    from loongcollector_b200 import synth
    buf, off, ln, grp = synth.apsara_lines(1 << 20, seed=5)
    ap = lc.Apsara("content", 0)
    got = eng.apsara_parse(ap, buf, off, ln, grp, NOW, -1)
    want = oap.process("content", 0, buf, off, ln, grp, NOW, -1)
    _same(got, want)
    assert int(want[6][4]) > (1 << 20) * 0.9
    eng.close()
