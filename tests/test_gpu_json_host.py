"""GPU tier: the host class ProcessorParseJsonNative (loongcollector_b200/host) replays every case of the reference's unit
test (tests/golden/ref_json.json) to the reference's expected groups and counters, and equals the oracle's group-level
Process on generated groups (documents with NUL bytes inside and after the root among them) -- every CommonParserOptions combination, events without the key, empty and failing values,
SourceKey among the members -- through Process(group) and the batched Process(std::vector<PipelineEventGroup>&):
the same contents in the same order, the same erased events and the same counters; CreateProcessor knows the name and
Init refuses a missing SourceKey."""
import copy
import itertools
import random

import pytest

pytestmark = pytest.mark.gpu

from oracle import json_parse as oj  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from tests import json_cases as jc  # noqa: E402
from tests import json_fixtures as jf  # noqa: E402

NAME = "processor_parse_json_native"


def _norm(x):
    return orc.Group.from_json(x).to_json() if x is not None else None


def _groups(seed):
    from loongcollector_b200 import synth
    rng = random.Random(seed)
    buf, off, ln, _ = synth.json_lines(200, seed=seed)
    raw = buf.tobytes()
    lines = [raw[o:o + l] for o, l in zip(off.tolist(), ln.tolist())]
    valid = jc.valid_docs(120, seed=seed)
    special = [b"", b"{}", b'{"content":"over","x":1}', b'{"raw":"r","a":1.25}', b"not json", b'{"a":1}\x00{"b":2}',
         b'{"n":"\\u0000"} \x00tail', b"\x00{}", b'{"a":"x\x00y"}', b'{"__raw_log__":"kept","a":1}']
    pool = [d for d in lines + valid + jc.mutate(valid, seed=seed + 1, per=1) if _utf8(d)]
    groups = []
    for _ in range(12):
        evs = []
        for _ in range(rng.randint(0, 40)):
            x = rng.random()
            if x < 0.08:
                evs.append({"contents": {"other": "x"}, "timestamp": 1, "type": 1})
            elif x < 0.12:
                evs.append({"contents": {"content": "", "__path__": "p"}, "timestamp": 1, "type": 1})
            else:
                c = {"content": rng.choice(special if rng.random() < 0.2 else pool).decode("utf-8")}
                if rng.random() < 0.3:
                    c["tag"] = "t"
                evs.append({"contents": c, "timestamp": 1, "type": 1})
        groups.append({"events": evs})
    return [g for g in groups if g["events"]]


def _utf8(d):
    try:
        d.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


CONFIGS = [dict({"SourceKey": "content"}, **{k: v for k, v in zip(("KeepingSourceWhenParseFail",
                                                                       "KeepingSourceWhenParseSucceed",
                                                                       "CopingRawLog"), flags) if v},
                **({"RenamedSourceKey": "raw"} if rn else {}))
           for flags in itertools.product([False, True], repeat=3) for rn in (False, True)]


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "-".join("%s" % v for v in c.values()))
def test_host_class_equals_oracle(cfg):
    import loongcollector_b200 as lc
    groups = _groups(7)
    want = [orc.Group.from_json(copy.deepcopy(g)) for g in groups]
    ref = oj.ProcessorParseJsonNative(cfg)
    ref.process_groups(want)
    p = lc.HostProcessor(NAME, cfg)
    got = p.process_groups(copy.deepcopy(groups))
    assert [_norm(x) for x in got] == [w.to_json() for w in want]
    p2 = lc.HostProcessor(NAME, cfg)
    got1 = [p2.process(copy.deepcopy(g)) for g in groups]
    assert [_norm(x) for x in got1] == [w.to_json() for w in want]
    for k, v in ref.counters.items():
        assert p.counters()[k] == v and p2.counters()[k] == v, k
    assert ref.counters["out_successful"] > 0 and ref.counters["out_failed"] > 0
    assert ref.counters["out_key_not_found"] > 0


def test_init_refuses_missing_source_key():
    import loongcollector_b200 as lc
    with pytest.raises(Exception):
        lc.HostProcessor(NAME, {})
    assert lc.HostProcessor(NAME, {"SourceKey": "content"}) is not None


@pytest.mark.parametrize("case", jf.PROCESS, ids=lambda c: c["name"])
def test_host_class_fixtures(case):
    import loongcollector_b200 as lc
    g = jf.split_input(case)
    p = lc.HostProcessor(NAME, case["config"])
    out = p.process(g.to_json() or {"events": []})
    jf.check_output(case, out, p.counters())
    p2 = lc.HostProcessor(NAME, case["config"])
    out2 = p2.process_groups([jf.split_input(case).to_json() or {"events": []}])[0]
    jf.check_output(case, out2, p2.counters())
