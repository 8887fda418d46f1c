"""CPU tier: the split-fed SLS serialiser's record and tile functions (lc_exec.cuh: lc_span_sls_rec, lc_span_sls_tile,
built for the host by tests/emul/split_sls.py) against the oracle's splitters followed by sls_serialize_logs, with
output tiles that start anywhere: inside a header, a varint, a key, a value, the digits or the ns trailer."""
import random

import pytest

from oracle import oracle as O
from tests import split_sls_cases as sc
from tests.emul import split_sls

TILES = [1, 7, 16, 4096, 0]


def _emul(val, key, offset_key, pos, time, ns, split_char=10, **kw):
    off, ln = O.split_lines(val, split_char)
    return split_sls.serialize(val, off, ln, key, offset_key, pos, time, ns, **kw)


@pytest.mark.parametrize("split_char", [10, 0])
@pytest.mark.parametrize("tile", TILES)
def test_random_pieces_every_tile(split_char, tile):
    rng = random.Random(split_char * 100 + tile)
    for i in range(6):
        val = sc.random_value(rng, rng.randint(1, 60), split_char)
        t, ns = sc.TIMES[i % len(sc.TIMES)]
        want = sc.oracle_split_wire(val, b"content", t, ns, 0, None, split_char)
        for nlanes in (1, 3, 32):
            got = _emul(val, b"content", None, 0, t, ns, split_char, tile=tile, nlanes=nlanes,
                        src_align=rng.randrange(16), out_align=rng.randrange(16))
            assert got == want, (i, nlanes)


@pytest.mark.parametrize("tile", [7, 4096, 0])
def test_long_pieces(tile):
    rng = random.Random(tile)
    val = sc.random_value(rng, 12, 10, long_every=4, trailing=False)
    assert max(len(x) for x in val.split(b"\n")) >= 65536
    want = sc.oracle_split_wire(val, b"content", 1 << 29, 5, 1000, b"__file_offset__")
    assert _emul(val, b"content", b"__file_offset__", 1000, 1 << 29, 5, tile=tile, nlanes=32,
                 src_align=3, out_align=9) == want


def test_empty_pieces_and_trailing_split_char():
    for val in [b"\n", b"\n\n\n", b"a\n", b"a\n\nb\n\n", b"abc", b"\nx"]:
        for okey in (None, b"__file_offset__", b"content"):
            want = sc.oracle_split_wire(val, b"content", 1, 3, 77, okey)
            for tile in TILES:
                assert _emul(val, b"content", okey, 77, 1, 3, tile=tile, nlanes=3) == want, (val, okey, tile)


@pytest.mark.parametrize("ns_on", [True, False])
def test_times(ns_on):
    rng = random.Random(5)
    val = sc.random_value(rng, 30)
    for t, ns in sc.TIMES:
        want = sc.oracle_split_wire(val, b"content", t, ns, 0, enable_ns=ns_on)
        assert _emul(val, b"content", None, 0, t, ns if ns_on else None, tile=16, nlanes=32) == want, t


def test_raw_mode():
    rng = random.Random(6)
    val = sc.random_value(rng, 50)
    for t, ns in sc.TIMES:
        want = sc.oracle_split_wire(val, b"log", t, ns, 123, b"__file_offset__", raw=True)
        for tile in TILES:
            assert _emul(val, b"content", None, 123, t, ns, tile=tile, nlanes=32) == want


@pytest.mark.parametrize("okey", [b"__file_offset__", b"content", b"", b"k" * 200])
@pytest.mark.parametrize("tile", [1, 16, 0])
def test_offset_keys_across_digit_counts(okey, tile):
    rng = random.Random(len(okey) + tile)
    val = b"\n".join(b"x" * rng.randint(0, 9) for _ in range(40))  # offsets 0 .. ~400 from each position
    for pos in sc.POSITIONS:
        want = sc.oracle_split_wire(val, b"content", 1 << 30, 9, pos, okey)
        got = _emul(val, b"content", okey, pos, 1 << 30, 9, tile=tile, nlanes=3, src_align=pos % 16)
        assert got == want, pos


def test_long_keys_and_multibyte_varints():
    val = b"a" * 200 + b"\n" + b"b" * 20000 + b"\n\n" + b"c" * 3
    key = b"K" * 300
    for okey in (None, b"O" * 130, key):
        want = sc.oracle_split_wire(val, key, 1 << 31, 1, 1 << 40, okey)
        for tile in (1, 7, 0):
            assert _emul(val, key, okey, 1 << 40, 1 << 31, 1, tile=tile, nlanes=32) == want


@pytest.mark.parametrize("name", sorted(sc.ML_CFGS))
@pytest.mark.parametrize("discard", [False, True])
def test_multiline_records(name, discard):
    rng = random.Random(hash(name) & 0xFFFF)
    val = sc.ml_value(rng, 80)
    cfg = sc.ml_config(name, discard)
    want, _, _ = sc.oracle_multiline_wire(val, cfg, 1 << 29, 3, 4096, b"__file_offset__")
    p = O.ProcessorSplitMultilineLogStringNative(cfg)
    off, ln, _, _ = O.multiline_split(val, p.start, p.cont, p.end, discard)
    for tile in (7, 0):
        got = split_sls.serialize(val, off, ln, b"content", b"__file_offset__", 4096, 1 << 29, 3, tile=tile,
                                  nlanes=32, src_align=5)
        assert got == want
