"""Writes tests/golden/ref_json.json from the reference's ProcessorParseJsonNativeUnittest.cpp
(core/unittest/processor/), as data.  One entry per input group of every test function:

  * "name": the test function (with "#k" for its k-th input group), "config": its Init parameters;
  * "input": the input group; "split": the splitter that runs first ("string" for ProcessorSplitLogStringNative,
    TestMultipleLines' "\\0" split), or null;
  * "expect": the group the test compares with (null for an empty group), or absent when the test only asserts
    find() on the output; then "find" lists the strings it asserts and "pinned" holds the oracle's full output
    (oracle/json_parse.py), pinned so that the device and the host class are held to it;
  * "counters": the processor counters the test asserts (DiscardedEventsTotal -> "discarded", ...).
TestInit is the "init" entry (a config that must be accepted); TestAddLog has no input.

  python tests/golden/extract_json_vectors.py [reference root]
"""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "ref_json.json")
SRC = "core/unittest/processor/ProcessorParseJsonNativeUnittest.cpp"
COUNTERS = {"mDiscardedEventsTotal": "discarded", "mOutFailedEventsTotal": "out_failed",
            "mOutKeyNotFoundEventsTotal": "out_key_not_found", "mOutSuccessfulEventsTotal": "out_successful"}


def bodies(text):
    heads = list(re.finditer(r"void ProcessorParseJsonNativeUnittest::(\w+)\(\) \{", text))
    for k, h in enumerate(heads):
        yield h.group(1), text[h.end():heads[k + 1].start() if k + 1 < len(heads) else len(text)]


def config(body):
    out = {}
    for k, v in re.findall(r'config\["(\w+)"\] = (.*?);', body):
        if v in ("true", "false"):
            out[k] = v == "true"
        elif v.startswith('"'):
            out[k] = v[1:-1]
        elif v == "'\\0'":
            out[k] = 0
        else:
            out[k] = int(v)
    return out


def raw(seg, name):
    m = re.search(name + r' = R"\((.*?)\)"', seg, re.S)
    return json.loads(m.group(1)) if m else None


def cases(text):
    sys.path.insert(0, ROOT)
    from oracle import oracle as orc
    from oracle import json_parse as oj
    out = []
    for fn, body in bodies(text):
        cfg = config(body)
        if fn == "TestInit":
            out.append({"name": fn, "config": cfg, "init": True})
            continue
        segs = body.split('std::string inJson = R"(')[1:]
        for k, seg in enumerate(segs):
            seg = 'std::string inJson = R"(' + seg
            c = {"name": fn + ("#%d" % k if len(segs) > 1 else ""), "config": cfg, "input": raw(seg, "inJson"),
                 "split": "string" if "ProcessorSplitLogStringNative" in seg else None}
            exp = raw(seg, "expectJson")
            if exp is not None:
                c["expect"] = exp
            elif 'APSARA_TEST_STREQ_FATAL("null"' in seg:
                c["expect"] = None
            else:
                c["find"] = re.findall(r'outJson\.find\("([^"]*)"\) != std::string::npos', seg)
            count = re.search(r"int count = (\d+);", seg)
            ctr = {}
            for v, name in re.findall(r"APSARA_TEST_EQUAL_FATAL\(uint64_t\((\w+)\), processor\.(\w+)->GetValue\(\)\)",
                                      seg):
                ctr[COUNTERS[name]] = int(count.group(1)) if v == "count" else int(v)
            c["counters"] = ctr
            if "find" in c:  # pin the oracle's output of a find()-only case
                g = orc.Group.from_json(json.loads(json.dumps(c["input"])))
                if c["split"]:
                    orc.ProcessorSplitLogStringNative(cfg).process(g)
                oj.ProcessorParseJsonNative(cfg).process(g)
                c["pinned"] = g.to_json()
            out.append(c)
    return out


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("LC_REFERENCE", "/root/reference")
    with open(os.path.join(ref, SRC), encoding="utf-8") as f:
        text = f.read()
    data = {"source": SRC, "cases": cases(text)}
    with open(OUT, "w", encoding="utf-8") as f:
        json.dump(data, f, indent=1, ensure_ascii=False)
        f.write("\n")
    print("%d cases -> %s" % (len(data["cases"]), OUT))


if __name__ == "__main__":
    main()
