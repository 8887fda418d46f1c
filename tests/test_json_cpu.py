"""ProcessorParseJsonNative on the CPU tier: the C oracle against Python's json module, the host build of the device
walk (tests/emul/lc_json_emul.cpp) against the oracle with 1, 3 and 32 lanes, and the walk under AddressSanitizer and
UBSan (tests/emul/lc_json_asan.cpp)."""
import json
import os
import re
import struct
import subprocess

import numpy as np
import pytest

from oracle import json_parse as oj
from tests import json_cases as jc
from tests.emul import json_parse as ej

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _py(doc):
    """Python's verdict and members of doc under the pinned rules: None when it does not parse"""
    def no_const(x):
        raise ValueError(x)
    try:
        text = doc
        items = json.loads(text.decode("utf-8"), object_pairs_hook=lambda kv: kv, parse_constant=no_const)
    except (ValueError, UnicodeDecodeError, RecursionError):
        return None
    if not isinstance(items, list) or (text.strip(b" \t\n\r")[:1] != b"{"):
        return None
    return items


def _render(v, raw):
    if isinstance(v, bool):
        return b"true" if v else b"false"
    if v is None:
        return b""
    if isinstance(v, str):
        return v.encode("utf-8", "surrogatepass")
    if isinstance(v, int):
        return b"%d" % v if -2 ** 63 <= v < 2 ** 64 else b""
    if isinstance(v, float):
        return b"" if v in (float("inf"), float("-inf")) else b"%f" % v
    return raw


def _compare(docs):
    base, off, ln = oj.table(docs)
    want = oj.process("content", base, off, ln)
    for W in (1, 3, 32):
        got = ej.parse("content", base, off, ln, W)
        for k in range(5):
            assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), (W, k)
    return want, got[5]


def test_pinned_renderings():
    docs = [b'{"v":' + v + b"}" for v, _ in jc.PINNED]
    got = oj.members(docs)
    for (v, want), m in zip(jc.PINNED, got):
        assert m == [(b"v", want)], v
    assert len(b"%f" % 1e308) == 316
    want, n_slow = _compare(docs)
    assert n_slow > 0


def test_edges_and_depths():
    got = oj.members(jc.EDGES + jc.DEPTHS)
    verdict = dict(zip(jc.EDGES + jc.DEPTHS, got))
    assert verdict[b"{}\x00junk"] == [] and verdict[b"{} \x00junk"] == [] and verdict[b"\x00{}"] is None
    assert verdict[b'{"a":[1,,2]}'] is None and verdict[b"{}x"] is None and verdict[b'{"a":tru}'] is None
    assert verdict[b'{"a":1,"a":2,"content":"x"}'] == [(b"a", b"1"), (b"a", b"2"), (b"content", b"x")]
    assert [verdict[d] is not None for d in jc.DEPTHS] == [True] * 6 + [False]
    _, n_slow = _compare(jc.EDGES + jc.DEPTHS)
    assert n_slow >= 3  # depths 65, 66 and 1024 (and 1025) need the slow walk


def test_overwritten_bit():
    base, off, ln = oj.table([b'{"content":"x"}', b'{"con\\u0074ent":1}', b'{"contents":1}', b'{"a":1}', None, b""])
    st = oj.process("content", base, off, ln)[0].tolist()
    assert st == [0x80, 0x80, 0, 0, oj.NOT_FOUND, oj.EMPTY]


def test_oracle_matches_python_on_valid_documents():
    docs = jc.valid_docs(600, seed=11)
    for d, m in zip(docs, oj.members(docs)):
        items = _py(d)
        assert items is not None and m is not None, d
        assert [k for k, _ in m] == [k.encode("utf-8", "surrogatepass") for k, _ in items]
        for (k, v), (_, pv) in zip(m, items):
            if isinstance(pv, (dict, list)):
                assert json.loads(v) is not None
            else:
                assert v == _render(pv, v), (d, k)


# The known differences between Python's json module and the pinned rule, and only these: Python accepts a lone
# surrogate escape, and Python rejects a NUL byte (and what follows) after the root object.
_ESC = re.compile(rb'\\(?:u([0-9A-Fa-f]{4})|.)', re.S)


def _lone_surrogate(doc):
    units = [int(m.group(1), 16) if m.group(1) else None for m in _ESC.finditer(doc)]
    for k, u in enumerate(units):
        nxt = units[k + 1] if k + 1 < len(units) else None
        prv = units[k - 1] if k else None
        if u is not None and 0xD800 <= u <= 0xDBFF and not (nxt is not None and 0xDC00 <= nxt <= 0xDFFF):
            return True
        if u is not None and 0xDC00 <= u <= 0xDFFF and not (prv is not None and 0xD800 <= prv <= 0xDBFF):
            return True
    return False


def _nul_after_root(doc):
    """a NUL byte right after a complete root object (and whitespace), where the pinned rule ends the input"""
    head = doc.split(b"\x00", 1)[0]
    if head == doc:
        return False
    try:
        json.loads(head.decode("utf-8"))
        return True
    except (ValueError, UnicodeDecodeError, RecursionError):
        return False


def _known_difference(doc):
    return _lone_surrogate(doc) or _nul_after_root(doc)


def test_oracle_verdicts_match_python_on_mutated_documents():
    docs = jc.mutate(jc.valid_docs(300, seed=12), seed=13)
    for d, m in zip(docs, oj.members(docs)):
        if _known_difference(d):
            continue
        assert (m is not None) == (_py(d) is not None), d


def test_emulation_matches_oracle():
    valid = jc.valid_docs(400, seed=21)
    docs = valid + jc.mutate(valid, seed=22, per=2) + [None, b""] + jc.EDGES
    _compare(docs)


def test_emulation_matches_oracle_on_generated_lines():
    from loongcollector_b200 import synth
    buf, off, ln, _ = synth.json_lines(3000, seed=5)
    base = buf
    want = oj.process("content", base, off, ln)
    got = ej.parse("content", base, off, ln, 32)
    for k in range(5):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
    assert int(want[4][2]) == 3000


def test_walk_under_sanitizers(tmp_path):
    exe = str(tmp_path / "lc_json_asan")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-o", exe, os.path.join(ROOT, "tests", "emul", "lc_json_asan.cpp")])
    valid = jc.valid_docs(150, seed=31)
    docs = valid + jc.mutate(valid, seed=32) + jc.EDGES + jc.DEPTHS + \
        [b'{"v":' + v + b"}" for v, _ in jc.PINNED]
    blob = b"".join(struct.pack("<I", len(d)) + d for d in docs)
    p = subprocess.run([exe], input=blob, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=600)
    assert p.returncode == 0, p.stderr.decode(errors="replace")[-3000:]
