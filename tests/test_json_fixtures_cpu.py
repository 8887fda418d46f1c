"""The reference unit test's ProcessorParseJsonNative cases (tests/golden/ref_json.json) on the CPU tier: the oracle's
group-level processor reproduces every expected group and counter, and the host build of the device walk
(tests/emul/lc_json_emul.cpp) equals the oracle on every fixture value with 1, 3 and 32 lanes."""
import numpy as np
import pytest

from oracle import json_parse as oj
from oracle.oracle import LOG
from tests import json_fixtures as jf
from tests.emul import json_parse as ej


@pytest.mark.parametrize("case", jf.PROCESS, ids=lambda c: c["name"])
def test_oracle_reproduces_fixture(case):
    g = jf.split_input(case)
    p = oj.ProcessorParseJsonNative(case["config"])
    p.process(g)
    jf.check_output(case, g.to_json(), p.counters)


def test_fixture_configs_accepted():
    init = [c for c in jf.FIXTURES if c.get("init")]
    assert init
    for c in init:
        oj.ProcessorParseJsonNative(c["config"])
    with pytest.raises(ValueError):
        oj.ProcessorParseJsonNative({})


@pytest.mark.parametrize("W", [1, 3, 32])
def test_emulation_equals_oracle_on_fixture_values(W):
    vals = []
    for c in jf.PROCESS:
        for e in jf.split_input(c).events:
            key = c["config"]["SourceKey"].encode()
            vals.append(e.get(key) if e.type == LOG and e.has(key) else None)
    base, off, ln = oj.table(vals)
    want = oj.process("content", base, off, ln)
    got = ej.parse("content", base, off, ln, W)
    for k in range(5):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
    assert int(want[4][2]) > 0 and int(want[4][1]) > 0
