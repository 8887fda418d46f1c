"""Writes tests/golden/ref_apsara.json from the reference's ProcessorParseApsaraNativeUnittest.cpp
(core/unittest/processor/), as data:

  * "time": TestApsaraEasyReadLogTimeParser's sequence over one cache (its Timezone and each value with the expected
    seconds, microseconds and whether the cache then holds that time);
  * "lines": TestApsaraLogLineParser's 31 lines (each one event in its own group, the config of the test) with the
    expected pairs.  The test checks only the first five pairs of each line ("pinned"); an empty list means the group
    becomes empty;
  * "process": every Process case (config, the input group, the expected group, the expected counters; "split" names a
    splitter that runs first).
The cases are pinned in a process zone at UTC.  Run with ilogtail_discard_old_data off, as the test sets it.

  python tests/golden/extract_apsara_vectors.py [reference root]
"""
import codecs
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "ref_apsara.json")
SRC = "core/unittest/processor/ProcessorParseApsaraNativeUnittest.cpp"
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_timestamp_vectors import bodies, config as _config  # noqa: E402

LIT = r'"((?:[^"\\]|\\.)*)"'


def config(body):
    return {k: {"true": True, "false": False}.get(v, v) for k, v in _config(body).items()}


def cpp(s):
    return codecs.decode(s, "unicode_escape")


def concat(expr):
    """the adjacent C++ string literals of expr, decoded"""
    return "".join(cpp(m) for m in re.findall(LIT, expr))


def time_steps(body):
    out = []
    for block in body.split("buffer = ")[1:]:
        m = re.match(LIT, block)
        step = {"value": cpp(m.group(1))}
        step["time"] = int(re.search(r"APSARA_TEST_EQUAL\(dateTime, (\d+)\)", block).group(1))
        step["micro"] = int(re.search(r"APSARA_TEST_EQUAL\(microTime, (\d+)\)", block).group(1))
        step["cached"] = "APSARA_TEST_EQUAL(dateTime, lastTime.tv_sec)" in block
        k = re.search(r"APSARA_TEST_EQUAL\(lastStr, " + LIT + r"\)", block)
        step["cache_key"] = cpp(k.group(1)) if k else None
        out.append(step)
    return out


def lines(body):
    arr = body[body.index("const char* logLine[] = {") + 1:]
    arr = arr[:arr.index("};")]
    raw_lines = re.findall(r"((?:\s*" + LIT + r")+)\s*(?:,\s*)?//\s*(\d+)", arr)
    vals = [json.loads('"' + concat(r[0]) + '"', strict=False) for r in raw_lines]
    res = body[body.index("logParseResult[][16] = {"):]
    res = res[:res.index("};\n")]
    names = {"APSARA_FIELD_LEVEL": "__LEVEL__", "APSARA_FIELD_THREAD": "__THREAD__", "APSARA_FIELD_FILE": "__FILE__",
             "APSARA_FIELD_LINE": "__LINE__"}
    exp = []
    for row in re.split(r"//\s*\d+", res[res.index("{") + 1:])[:-1]:
        toks = re.findall(LIT + r"|(APSARA_FIELD_\w+)|(NULL)", row)
        flat = []
        for lit, name, null in toks:
            if null:
                break
            flat.append(names[name] if name else cpp(lit))
        exp.append([flat[i:i + 2] for i in range(0, len(flat), 2)])
    assert len(vals) == len(exp) == 31, (len(vals), len(exp))
    return [{"value": v, "pairs": p, "pinned": min(5, len(p))} for v, p in zip(vals, exp)]


def raw_json(block, name):
    m = re.search(r"std::string " + name + r' = R"\((.*?)\)";', block, re.S)
    return json.loads(m.group(1), strict=False) if m else None


def counters(block):
    env = {k: int(v) for k, v in re.findall(r"int (\w+) = (\d+);", block)}
    out = {}
    for v, obj, k in re.findall(r"APSARA_TEST_EQUAL_FATAL\(uint64_t\((\w+)\), (processor|processorInstance)\.m(\w+)->",
                                block):
        out[("instance_" if obj == "processorInstance" else "") + k] = int(v) if v.isdigit() else env[v]
    return out


def process_cases(b):
    out = []
    for name in ("TestProcessWholeLine", "TestProcessWholeLinePart", "TestProcessKeyOverwritten", "TestUploadRawLog",
                 "TestProcessEventKeepUnmatch", "TestProcessEventDiscardUnmatch", "TestProcessEventMicrosecondUnmatch"):
        body = b[name]
        expect = raw_json(body, "expectJson")
        out.append({"name": name, "config": config(body), "split": None, "input": raw_json(body, "inJson"),
                    "expect": expect, "counters": counters(body)})
    body = b["TestMultipleLines"]
    inj, exp = raw_json(body, "inJson"), raw_json(body, "expectJson")
    for block, split in zip(body.split("// ProcessorSplit")[1:], ("string", "multiline")):
        out.append({"name": "TestMultipleLines/" + split, "config": config(block), "split": split, "input": inj,
                    "expect": exp, "counters": {}})
    return out


def extract(ref):
    text = open(os.path.join(ref, SRC)).read()
    b = bodies(text)
    tb = b["TestApsaraEasyReadLogTimeParser"]
    lb = b["TestApsaraLogLineParser"]
    return {"source": SRC, "zone": "UTC",
            "time": {"config": config(tb), "steps": time_steps(tb)},
            "lines": {"config": config(lb), "cases": lines(lb)},
            "process": process_cases(b)}


if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("LC_REFERENCE", "/root/reference")
    data = extract(ref)
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", OUT, len(data["time"]["steps"]), len(data["lines"]["cases"]), len(data["process"]))
