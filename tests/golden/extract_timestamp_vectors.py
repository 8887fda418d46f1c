"""Writes tests/golden/ref_timestamp.json from the reference's ProcessorParseTimestampNativeUnittest.cpp
(core/unittest/processor/): every case of TestInit, TestProcessNoFormat, TestProcessRegularFormat,
TestProcessNoYearFormat, TestProcessRegularFormatFailed, TestProcessHistoryDiscard, TestParseLogTime,
TestParseLogTimeSecondCache and TestAdjustTimeZone, as data.

  * "init" cases: a config and whether Init accepts it.
  * "process" cases (the Process tests, whose values are the local "now" rendered by strftime): the config, the
    strftime format of the two values, the shift of their "now" (seconds), what the reference expects of each event
    ("parsed": timestamp now + shift - mLogTimeZoneOffsetSecond with the given nanoseconds, "unchanged", "erased") and
    the expected counters.
  * "parse" cases (ParseLogTime with an empty cache per sequence, SourceTimezone as configured): the format, the values
    in order and the expected (tv_sec, tv_nsec) of each.  The seeded cache of the second-cache tests ("2012-01-01
    15:04:59", ...) is a prefix of none of their values, so it behaves as an empty one.

  python tests/golden/extract_timestamp_vectors.py [reference root]
"""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "ref_timestamp.json")
SRC = "core/unittest/processor/ProcessorParseTimestampNativeUnittest.cpp"


def bodies(text):
    """{test name: body} of every `void ...Unittest::Test...() {` definition"""
    out = {}
    for m in re.finditer(r"void \w+Unittest::(Test\w+)\(\) \{", text):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            i += 1
        out[m.group(1)] = text[m.end():i - 1]
    return out


def config(body):
    cfg = {}
    for k, v in re.findall(r'config\["(\w+)"\] = ([^;]+);', body):
        v = v.strip()
        cfg[k] = json.loads(v) if v.startswith('"') else (int(v) if re.fullmatch(r"-?\d+", v) else v)
    return cfg


def counters(body):
    return {k: int(v) for v, k in re.findall(r"APSARA_TEST_EQUAL_FATAL\((\d+)UL, processor\.m(\w+)->GetValue\(\)\)",
                                             body)}


def cpp_expr(e):
    """the few C++ string expressions the generated cases use, as Python"""
    e = e.replace("std::string(second.data())", "second")
    e = re.sub(r'\(i < 10 \? "0" \+ std::to_string\(i\) : std::to_string\(i\)\)', '("0" + str(i) if i < 10 else str(i))',
               e)
    e = e.replace("std::to_string(expectLogTimeBase + i)", "str(base + i)")
    return re.sub(r"std::to_string\((\w+)\)", r"str(\1)", e)


def generated(block, tz):
    fmt = re.search(r'config\["SourceFormat"\] = "([^"]*)"', block).group(1)
    base = int(re.search(r"time_t expectLogTimeBase = (\d+);", block).group(1))
    second = cpp_expr(re.search(r"std::string second = (.+?);\n", block).group(1))
    m = re.search(r"inputTimes\.emplace_back\((.+?),\s*expectLogTimeBase \+ i,\s*(.+?),\s*expectLogTimeNanosecondBase",
                  block, re.S)
    value, nsec = cpp_expr(" ".join(m.group(1).split())), cpp_expr(m.group(2).strip())
    vals, want = [], []
    for i in range(5):
        for j in range(5):
            env = {"i": i, "j": j, "base": base, "str": str}
            env["second"] = eval(second, env)
            vals.append(eval(value, env))
            want.append([base + i, eval(nsec, env)])
    return {"format": fmt, "timezone": tz, "values": vals, "expect": want}


def extract(ref):
    text = open(os.path.join(ref, SRC)).read()
    b = bodies(text)
    out = {"source": SRC, "init": [], "process": [], "parse": []}
    out["init"].append({"name": "TestInit", "config": config(b["TestInit"]), "ok": True})
    out["init"].append({"name": "TestProcessNoFormat", "config": config(b["TestProcessNoFormat"]), "ok": False})
    for name, shift, expect in (("TestProcessRegularFormat", 0, "parsed"), ("TestProcessNoYearFormat", 0, "parsed"),
                                ("TestProcessRegularFormatFailed", -43201, "unchanged"),
                                ("TestProcessHistoryDiscard", -43201, "erased")):
        body = b[name]
        cfg = config(body)
        sf = re.search(r'strftime\(timebuff, sizeof\(timebuff\), ("[^"]*"|config\["SourceFormat"\]\.asString\(\)\.c_str\(\))',
                       body).group(1)
        strf = cfg["SourceFormat"] if sf.startswith("config") else json.loads(sf)
        if "ilogtail_discard_interval" in body.split("strftime")[0]:
            assert shift == -43201
        if cfg.get("SourceYear") == "now_tm->tm_year + 1900":
            cfg["SourceYear"] = "now"
        ns = re.findall(r'"timestampNanosecond" : (\d+),\n\s*"type"', body.split("judge result")[-1])
        out["process"].append({"name": name, "config": cfg, "strftime": strf, "now_shift": shift, "expect": expect,
                               "nanosecond": int(ns[0]) if ns and expect == "parsed" else 0,
                               "counters": counters(body)})
    body = b["TestParseLogTime"]
    tz = config(body)["SourceTimezone"]
    for v, f, s, ns in re.findall(r'\{"([^"]*)", "([^"]*)", (\d+), (\d+)\}', body):
        out["parse"].append({"format": f, "timezone": tz, "values": [v], "expect": [[int(s), int(ns)]],
                             "test": "TestParseLogTime"})
    for name in ("TestParseLogTimeSecondCache", "TestAdjustTimeZone"):
        body = b[name]
        outer_tz = re.search(r'config\["SourceTimezone"\] = "([^"]*)"', body.split("{ // case")[0])
        for block in body.split("{ // case")[1:]:
            m = re.search(r'config\["SourceTimezone"\] = "([^"]*)"', block)
            c = generated(block, (m or outer_tz).group(1))
            c["test"] = name
            out["parse"].append(c)
    return out


if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("LC_REFERENCE", "/root/reference")
    data = extract(ref)
    with open(OUT, "w") as f:
        json.dump(data, f, indent=1)
        f.write("\n")
    print("wrote", OUT, len(data["init"]), len(data["process"]), len(data["parse"]))
