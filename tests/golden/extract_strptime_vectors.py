"""Writes tests/golden/ref_strptime.json: the results of the reference's own strptime_ns (compiled in place by
oracle/build_ref_strptime.sh into oracle/_ref/libref_strptime.so, behind oracle/ref_strptime_driver.cpp) on the seeded
inputs of tests/timestamp_cases.py, in every zone of timestamp_cases.ZONES: per case the counters and one digest of the
status, sec and nsec tables.

  sh oracle/build_ref_strptime.sh && python tests/golden/extract_strptime_vectors.py
"""
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import timestamp as ots  # noqa: E402
from tests import timestamp_cases as tc  # noqa: E402
from tests.emul import timestamp as ets  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_strptime.json")


def digest(st, sec, ns):
    h = hashlib.sha256()
    for a in (st, sec, ns):
        h.update(a.tobytes())
    return h.hexdigest()[:24]


def results(which):
    """{zone: {case name: [counters, digest]}} of one oracle"""
    saved = os.environ.get("TZ")
    out = {}
    try:
        for zone in tc.ZONES:
            os.environ["TZ"] = zone
            time.tzset()
            out[zone] = {}
            for name, fmt, sy, adj, now, di, groups in tc.all_cases():
                base, off, ln, grp = ets.layout(groups)
                st, sec, ns, cnt = ots.process(fmt, sy, adj, base, off, ln, grp, now, di, which)
                out[zone][name] = [[int(x) for x in cnt], digest(st, sec, ns)]
    finally:
        if saved is None:
            os.environ.pop("TZ", None)
        else:
            os.environ["TZ"] = saved
        time.tzset()
    return out


if __name__ == "__main__":
    assert ots.have_reference(), "build oracle/_ref/libref_strptime.so first (oracle/build_ref_strptime.sh)"
    with open(OUT, "w") as f:
        json.dump({"source": "core/common/Strptime.cpp (strptime_ns) behind oracle/ref_strptime_driver.cpp",
                   "results": results("ref")}, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", OUT)
