"""CPU tier: the delimiter-fed SLS serialiser's per-row function (lc_exec.cuh: lc_delim_sls_body, built for the host
by tests/emul/delim_sls.py) against the oracle's ProcessorParseDelimiterNative + sls_serialize_logs on seeded random
lines, over the separator x overflow-treatment matrix with random keys, source / renamed keys and keep / copy flags."""
import pytest

from tests import delim_sls_cases as dc
from tests.emul import delim_sls

CASES = list(dc.all_cases(seed_base=1, per=6))


def _run(cfg, lines, times, nss, nlanes):
    buf, off, ln = dc.arena(lines)
    tables = dc.parse_tables(buf, off, ln, cfg)
    quote = cfg["quote"] if len(cfg["sep"]) == 1 else ord('"')
    return delim_sls.serialize(buf, off, ln, tables, cfg["max_fields"], cfg["sep"], quote, cfg["treatment"],
                               [k.encode() for k in cfg["keys"]], cfg["source"].encode(), dc.renamed_key(cfg),
                               cfg["keep_fail"], cfg["keep_succeed"], cfg["copy_raw"], times, nss, nlanes)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_per_row_function_matches_oracle(case):
    _, cfg, rng = case
    lines = [dc.random_line(rng, cfg["sep"], cfg["quote"], wide=rng.random() < 0.05) for _ in range(150)]
    times, nss = dc.times_for(len(lines), rng.randint(0, 1 << 30))
    want, _, _ = dc.oracle_wire(lines, cfg, times, nss, True)
    for nlanes in (1, 3, 32):
        assert _run(cfg, lines, times, nss, nlanes) == want, (cfg, nlanes)
    want_nons, _, _ = dc.oracle_wire(lines, cfg, times, None, False)
    assert _run(cfg, lines, times, None, 1) == want_nons


def test_source_key_among_keys_with_short_rows():
    for tr in dc.TREATMENTS:
        cfg = {"sep": b",", "quote": ord('"'), "treatment": tr, "keys": ["a", "b", "content"], "source": "content",
               "renamed": None, "keep_fail": True, "keep_succeed": True, "copy_raw": True, "allow_short": True,
               "max_fields": 4}
        lines = [b"1", b"1,2", b"1,2,3", b"1,2,3,4,5", b'"x""y",2,"3""""3"', b"", b'"open,1']
        times, nss = dc.times_for(len(lines), 3)
        want, _, _ = dc.oracle_wire(lines, cfg, times, nss)
        assert _run(cfg, lines, times, nss, 4) == want


@pytest.mark.parametrize("sep", [b",", b"|#"])
def test_rows_wider_than_the_tables(sep):
    import random
    rng = random.Random(7)
    for tr in dc.TREATMENTS:
        cfg = {"sep": sep, "quote": ord('"'), "treatment": tr, "keys": ["a", "b"], "source": "content",
               "renamed": "__column5__", "keep_fail": False, "keep_succeed": True, "copy_raw": False,
               "allow_short": True, "max_fields": 3}
        lines = [dc.random_line(rng, sep, ord('"'), wide=True) for _ in range(40)] + [sep * 300, b"a" + sep + b"b"]
        times, nss = dc.times_for(len(lines), 4)
        want, _, _ = dc.oracle_wire(lines, cfg, times, nss)
        assert _run(cfg, lines, times, nss, 32) == want


@pytest.mark.parametrize("keys,treatment,source,max_fields,why", [
    (["a", "a"], "extend", "content", 3, "distinct"),
    (["a", "a"], "discard", "content", 3, "distinct"),
    (["_", "_"], "keep", "content", 3, "distinct"),
    (["a", "__column2__"], "extend", "content", 3, "__column"),
    (["a", "__column07__"], "keep", "content", 3, "__column"),
    (["a"], "extend", "__column1__", 3, "source key"),
    (["a", "b"], "extend", "content", 2, "max_fields"),
])
def test_refused_configurations(keys, treatment, source, max_fields, why):
    cfg = {"sep": b",", "quote": ord('"'), "treatment": treatment, "keys": keys, "source": source, "renamed": None,
           "keep_fail": True, "keep_succeed": True, "copy_raw": True, "allow_short": True, "max_fields": max_fields}
    with pytest.raises(delim_sls.Refused, match=why):
        _run(cfg, [b"1,2"], [1], None, 1)


def test_accepted_in_discard_mode():
    """repeated "_" keys and __column<N>__ keys are plain keys when overflow columns are dropped"""
    cfg = {"sep": b",", "quote": ord('"'), "treatment": "discard", "keys": ["_", "__column1__", "_", "x"],
           "source": "content", "renamed": "__column1__", "keep_fail": True, "keep_succeed": True, "copy_raw": True,
           "allow_short": True, "max_fields": 5}
    lines = [b"1,2,3,4,5,6", b"1,2", b"", b'"a', b"1,2,3,4"]
    times, nss = dc.times_for(len(lines), 5)
    want, _, _ = dc.oracle_wire(lines, cfg, times, nss)
    assert _run(cfg, lines, times, nss, 2) == want
