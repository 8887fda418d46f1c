"""GPU tier: the reference's own unit-test fixtures (tests/golden/ref_*.json) replayed through the C++ host
layer (GPU-backed Processor classes behind the reference's plugin API) -- the drop-in claim."""
from collections import OrderedDict

import pytest

pytestmark = pytest.mark.gpu

from tests.golden_util import all_cases, run_cases_of_function  # noqa: E402

BY_FN = OrderedDict()
for c in all_cases():
    BY_FN.setdefault(c["name"].split("#")[0], []).append(c)


@pytest.mark.parametrize("fn", list(BY_FN), ids=list(BY_FN))
def test_host_processors_match_reference_fixture(fn):
    import loongcollector_b200 as lc

    def make(ptype, cfg):
        return lc.HostProcessor(ptype, cfg)

    def run(proc, group_json, enable_meta):
        n_in = len((group_json or {}).get("events", []))
        out = proc.process(group_json, True)
        return out, len((out or {}).get("events", [])), n_in

    n = run_cases_of_function(BY_FN[fn], make, run, lambda p: p.counters())
    assert n > 0


def test_merge_multiline_random_groups_match_oracle():
    """ProcessorMergeMultilineLogNative on random groups: every supported pattern combination, both unmatched
    treatments, the flag mode, empty events, events without the source key and unsupported events in the middle --
    the host class (batched GPU probes + host walk) against the oracle restatement, contents and counters."""
    import json
    import random

    import loongcollector_b200 as lc
    from oracle import oracle as orc

    rng = random.Random(20240607)
    words = ["S1 begin", "S2", "  cont a", "  cont", "E done", "Eof", "noise", "x", "", "S", "E"]
    combos = [("S.*", "", ""), ("S.*", r"\s+cont.*", ""), ("S\\d?.*", "", "E.*"), ("", r"\s+cont", "E\\w+"),
              ("", "", "E.*$"), ("S.*", r"\s+cont.*", "E.*")]
    name = "processor_merge_multiline_log_native"
    checked = 0
    for start, cont, end in combos:
        for treat in ("single_line", "discard"):
            cfg = {"MergeType": "regex", "UnmatchedContentTreatment": treat}
            if start:
                cfg["StartPattern"] = start
            if cont:
                cfg["ContinuePattern"] = cont
            if end:
                cfg["EndPattern"] = end
            host, ora = lc.HostProcessor(name, cfg), orc.PROCESSORS[name](cfg)
            for _ in range(12):
                evs = []
                for _ in range(rng.randint(0, 40)):
                    r = rng.random()
                    if r < 0.03:
                        evs.append({"name": "", "timestamp": 0, "type": 2, "value": {"type": "unknown"}})
                    elif r < 0.06:
                        evs.append({"type": 1, "timestamp": 7, "timestampNanosecond": 0})
                    elif r < 0.08:
                        evs.append({"type": 1, "timestamp": 7, "timestampNanosecond": 0, "contents": {"other": "v"}})
                    else:
                        evs.append({"type": 1, "timestamp": 7, "timestampNanosecond": 0,
                                    "contents": {"content": rng.choice(words), "tag": "t%d" % rng.randint(0, 3)}})
                root = {"events": evs} if evs else None
                got = host.process(json.loads(json.dumps(root)), True)
                g = orc.Group.from_json(json.loads(json.dumps(root)))
                ora.process(g)
                assert json.dumps(got, sort_keys=True) == json.dumps(g.to_json(True), sort_keys=True), (cfg, root)
                checked += 1
            hc = host.counters()
            assert hc["merged_events_total"] == ora.counters["merged_events"], cfg
            assert hc["unmatched_events_total"] == ora.counters["unmatched_events"], cfg
    # flag mode: docker partial logs
    cfg = {"MergeType": "flag"}
    host, ora = lc.HostProcessor(name, cfg), orc.PROCESSORS[name](cfg)
    for _ in range(30):
        evs = []
        for _ in range(rng.randint(1, 30)):
            c = {"content": rng.choice(words)}
            if rng.random() < 0.4:
                c["P"] = ""
            evs.append({"type": 1, "timestamp": 7, "timestampNanosecond": 0, "contents": c})
        root = {"events": evs, "metadata": {"has.part.log": "P"}} if rng.random() < 0.8 else {"events": evs}
        got = host.process(json.loads(json.dumps(root)), True)
        g = orc.Group.from_json(json.loads(json.dumps(root)))
        ora.process(g)
        assert json.dumps(got, sort_keys=True) == json.dumps(g.to_json(True), sort_keys=True), root
        checked += 1
    assert checked > 150


@pytest.mark.parametrize("treatment,nkeys", [(t, k) for k in (3, 20) for t in ("extend", "keep", "discard")],
                         ids=[t if k == 3 else "%s-%dkeys" % (t, k) for k in (3, 20) for t in ("extend", "keep", "discard")])
def test_delimiter_lines_with_far_more_columns_than_keys(treatment, nkeys):
    """Untrusted content: a few lines with hundreds / thousands of columns among ordinary ones.  The host class parses
    them again on their own (bounded tables, no group-wide re-run) and still produces exactly the reference's events
    (`__columnN__` keys in extend mode, the joined remainder in keep mode).  With 20 keys the tables are 36 columns
    wide, which the direct kernel (more than 32 columns) fills; long and blank-padded lines ride along."""
    import json

    import loongcollector_b200 as lc
    from oracle import oracle as orc

    name = "processor_parse_delimiter_native"
    keys = ["a", "b", "c"] if nkeys == 3 else ["k%d" % i for i in range(nkeys)]
    cfg = {"SourceKey": "content", "Separator": ",", "Quote": '"', "Keys": keys,
           "OverflowedFieldsTreatment": treatment, "KeepingSourceWhenParseFail": True}
    lines = ["1,2,3", "x,y", ",".join(str(i) for i in range(300)), "p,\"q,r\",s,t", ",".join(["z"] * 5000),
             "\"a\"\"b\",c", ",".join("\"v%d\"\"w\"" % i for i in range(40)), ""]
    lines += [" " * 300 + ",".join(str(i) for i in range(25)) + " \r" * 150, " " * 257, " \r" * 140,
              "\r" + " " * 40 + "a,b",
              ",".join("f%d" % i for i in range(19)) + ",\"" + "q,\"\"" * 1000 + "\"," + "y" * 4097,
              "m," * 33 + "\"" + "x" * 70001 + "\"", "u," * 10 + "\"" + "open" * 1100, " " * 129 + "d,\"e\"x"]
    evs = [{"type": 1, "timestamp": 5, "timestampNanosecond": 0, "contents": {"content": ln}} for ln in lines]
    root = {"events": evs}
    host, ora = lc.HostProcessor(name, cfg), orc.PROCESSORS[name](cfg)
    got = host.process(json.loads(json.dumps(root)), True)
    g = orc.Group.from_json(json.loads(json.dumps(root)))
    ora.process(g)
    assert json.dumps(got, sort_keys=True) == json.dumps(g.to_json(True), sort_keys=True)


def test_dynamic_plugins_process_groups_like_the_host_classes():
    """The lib<name>.so dynamic plugins, driven the way DynamicCProcessorProxy drives them (init -> process -> finalize
    through the exported processor_interface), produce exactly what the class-level processors produce."""
    import json

    import loongcollector_b200 as lc
    from loongcollector_b200 import _build
    from tests.test_cabi_cpu import _roundtrip

    cases = [
        ("processor_parse_regex_b200", "processor_parse_regex_native",
         {"SourceKey": "content", "Regex": r"(\w+)\t(\w+).*", "Keys": ["k1", "k2"], "KeepingSourceWhenParseFail": True,
          "RenamedSourceKey": "rawLog"}, ["value1\tvalue2 tail", "nomatch", "a\tb"]),
        ("processor_parse_delimiter_b200", "processor_parse_delimiter_native",
         {"SourceKey": "content", "Separator": ",", "Quote": "'", "Keys": ["a", "b", "c"]},
         ["1,2,3", "x,'y,z',w", "only"]),
        ("processor_split_string_b200", "processor_split_string_native", {}, ["l1\nl2\nl3", "single"]),
        ("processor_split_multiline_log_string_b200", "processor_split_multiline_log_string_native",
         {"Multiline": {"StartPattern": r"\[\d+\].*"}}, ["[1] a\n  cont\n[2] b\nnoise"]),
    ]
    for name, ptype, cfg, values in cases:
        grp = {"events": [{"type": 1, "timestamp": 9, "timestampNanosecond": 0, "contents": {"content": v}}
                          for v in values]}
        ver, nm, got, err = _roundtrip(_build.plugin_path(name), cfg, json.loads(json.dumps(grp)))
        assert err is None and ver == 100 and nm == name, (name, err)
        want = lc.HostProcessor(ptype, cfg).process(json.loads(json.dumps(grp)), True)
        assert json.dumps(got, sort_keys=True) == json.dumps(want, sort_keys=True), name
