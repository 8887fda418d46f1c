"""ProcessorParseTimestampNative without a GPU: the host build of the format compiler, the full-parse pass and the
warp resolution pass (tests/emul/lc_timestamp_emul.cpp, the statements of lc_exec.cuh the kernels run) with 1, 3 and
32 lanes, checked against the flat C restatement over libc's mktime (oracle/lc_timestamp_oracle.c), against the
reference's own strptime_ns (oracle/_ref/libref_strptime.so where it was built) and against that reference's stored
results (tests/golden/ref_strptime.json), in three zones."""
import json
import os
import random
import time

import numpy as np
import pytest

from oracle import timestamp as ots
from tests import timestamp_cases as tc
from tests.emul import timestamp as ets
from tests.golden import extract_strptime_vectors as xv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = tc.all_cases()


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


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def test_emulation_equals_oracles(zone):
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_strptime.json")))["results"][zone]
    for name, fmt, sy, adj, now, di, groups in CASES:
        base, off, ln, grp = ets.layout(groups)
        c = ets.Compiled(fmt, sy, adj)
        assert c.ok, (fmt, c.error)
        want = ots.process(fmt, sy, adj, base, off, ln, grp, now, di, "c")
        assert golden[name] == [[int(x) for x in want[3]], xv.digest(*want[:3])], (zone, name)
        if ots.have_reference():
            assert _same(ots.process(fmt, sy, adj, base, off, ln, grp, now, di, "ref"), want), (zone, name)
        for W in (1, 3, 32):
            assert _same(c.parse(base, off, ln, grp, now, di, W), want), (zone, name, W)


def test_every_case_has_a_stored_reference_result():
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_strptime.json")))["results"]
    names = {c[0] for c in CASES}
    assert len(names) == len(CASES)
    for zone in tc.ZONES:
        assert set(golden[zone]) == names


@pytest.mark.parametrize("fmt", ["%c", "%Y %x", "%X", "%Ec", "%Y\x00%m"])
def test_refused_formats(fmt):
    c = ets.Compiled(fmt.encode())
    assert not c.ok and c.error.startswith("SourceFormat:")


def test_program_capacity():
    assert ets.Compiled("%Y" * 96).ok
    c = ets.Compiled("%Y" * 97)
    assert not c.ok and "more directives" in c.error
    assert not ets.Compiled("%T" * 30).ok  # each %T is its recursive call's 6 steps


def test_directives_read_nothing_past_the_value(zone):
    """Values cut inside every directive, laid out so that the value ends exactly at the end of the buffer and the
    bytes behind a cut would continue it: the emulation must read them as NUL."""
    for fmt in tc.FORMATS:
        full = tc.render(fmt, time.gmtime(1500000000), random.Random(3))
        c = ets.Compiled(fmt)
        for cut in range(len(full) + 1):
            head = full[:cut]
            base = np.frombuffer(head + full[cut:], np.uint8).copy()
            off, ln = np.array([0], np.uint32), np.array([cut], np.uint32)
            grp = np.array([0, 1], np.uint32)
            got = c.parse(base, off, ln, grp, tc.NOW, -1, 32)
            want = ots.process(fmt, -1, 0, np.frombuffer(head, np.uint8).copy(), np.array([0], np.uint32),
                               ln, grp, tc.NOW, -1, "c")
            assert _same(got, want), (fmt, head)


def test_groups_reset_the_cache():
    """The same values in one group and in one group per event: the second-level cache does not cross groups.  A %s
    value that starts with the previous value hits it and keeps its second, the reference's quirk."""
    vals = [b"170000000", b"1700000000", b"170000000"]
    c = ets.Compiled("%s")
    one = c.parse(*ets.layout([vals]), tc.NOW, -1, 32)
    many = c.parse(*ets.layout([[v] for v in vals]), tc.NOW, -1, 32)
    assert one[1].tolist() == [170000000, 170000000, 170000000] and one[2].tolist() == [0, 0, 0]
    assert many[1].tolist() == [170000000, 1700000000, 170000000]
