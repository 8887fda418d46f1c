"""The reference unit test's ProcessorParseJsonNative cases (tests/golden/ref_json.json, written by
tests/golden/extract_json_vectors.py) and the helpers that replay them."""
import copy
import json
import os

from oracle import oracle as orc

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_json.json")
with open(_PATH, encoding="utf-8") as _f:
    FIXTURES = json.load(_f)["cases"]
PROCESS = [c for c in FIXTURES if "input" in c]


def norm(x):
    return orc.Group.from_json(copy.deepcopy(x)).to_json() if x is not None else None


def split_input(case):
    """the case's input group after its splitter, as an oracle Group"""
    g = orc.Group.from_json(copy.deepcopy(case["input"]))
    if case["split"]:
        orc.ProcessorSplitLogStringNative(case["config"]).process(g)
    return g


def check_output(case, out, counters):
    """out: the processed group as JSON (None when empty); counters: name -> value"""
    if "expect" in case:
        assert norm(out) == norm(case["expect"]), case["name"]
    else:
        text = json.dumps(out, ensure_ascii=False)
        for s in case["find"]:
            assert s in text, (case["name"], s)
        assert norm(out) == norm(case["pinned"]), case["name"]
    for k, v in case["counters"].items():
        assert counters[k] == v, (case["name"], k)
