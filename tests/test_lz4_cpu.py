"""CPU tier: the LZ4 block compressor's parse, size and emit functions (lc_exec.cuh, built for the host by
tests/emul/lz4.py) with 1, 3 and 32 emulated lanes.  Every block decodes, through the strict decoder of
tests/lz4_block.py and through the system's liblz4 when it is installed, to its segment; the lane counts agree byte
for byte; and on the bench shapes the blocks are at most 10 % larger than liblz4's LZ4_compress_default."""
import random

import pytest

from tests import lz4_block
from tests import lz4_cases as zc
from tests.emul import lz4

LANES = (1, 3, 32)
needs_liblz4 = pytest.mark.skipif(zc.liblz4() is None, reason="the system's liblz4 (liblz4.so.1) is not installed")


def _bound(n):
    return n + n // 255 + 16


def _check(segs, lanes=LANES):
    """compresses segs with every lane count; checks agreement, decoding and the bound; returns the blocks"""
    blocks = lz4.compress(segs, lanes[0])
    for w in lanes[1:]:
        assert lz4.compress(segs, w) == blocks, w
    for s, b in zip(segs, blocks):
        assert len(b) <= _bound(len(s))
        assert lz4_block.decode(b) == s
        if zc.liblz4() is not None:
            assert zc.lz4_decompress(b, len(s)) == s
    return blocks


@pytest.mark.parametrize("part", range(4))
def test_edge_matrix(part):
    segs = zc.edge_segments()
    _check([s for i, (_, s) in enumerate(segs) if i % 4 == part])


def test_short_segments_are_literals():
    for n in range(13):
        s = bytes(b"a" * n)
        [b] = _check([s])
        assert b == bytes([n << 4]) + s  # one literals-only sequence


def test_empty_segment_is_one_zero_byte():
    assert lz4.compress([b""]) == [b"\x00"]
    assert _check([b"", b"x" * 100, b"", b""])[::2] == [b"\x00", b"\x00"]


def test_runs_use_offset_one():
    s = b"q" * 1000
    [b] = _check([s])
    # token (1 literal, long match), match-length bytes, offset 1, then the 5+ closing literals
    assert b[1:2] == b"q" and b[2:4] == b"\x01\x00"
    assert len(b) < 20


def test_offset_65536_is_not_used():
    rng = random.Random(3)
    blk = rng.randbytes(64)
    # zeros between the copies hash to one table entry, so the first copy's positions stay in the table
    near = blk + bytes(65535 - 64) + blk + b"." * 20
    far = blk + bytes(65536 - 64) + blk + b"." * 20
    bn, bf = _check([near])[0], _check([far])[0]
    # at distance 65535 the second copy is (almost all) one match; at 65536 it is out of reach and stays literals
    assert len(bf) - len(bn) > 50
    assert b"\xff\xff" in bn[-80:]  # offset 65535


def test_cross_chunk_matches():
    rng = random.Random(4)
    period = bytes(rng.getrandbits(8) for _ in range(5000))
    s = (period * 60)[:3 * lz4.CHUNK + 123]
    [b] = _check([s])
    assert len(b) < 5000 + 3000  # every chunk after the first period copies from the previous one, across chunks


@pytest.mark.parametrize("mib", [1, 10])
def test_incompressible_segments(mib):
    rng = random.Random(mib)
    s = rng.randbytes(mib << 20)
    [b] = _check([s], lanes=(32,) if mib > 1 else LANES)
    assert len(b) <= _bound(len(s))


def test_many_segments():
    rng = random.Random(5)
    segs = []
    for i in range(300):
        k = rng.randrange(4)
        n = [0, rng.randrange(1, 40), rng.randrange(40, 3000), rng.randrange(3000, 70000)][k]
        segs.append((b"log line %d " % rng.randrange(50) * (n // 10 + 1))[:n] if i % 2 else rng.randbytes(n))
    _check(segs)


@needs_liblz4
def test_ratio_gate():
    """on the five bench shapes, as 512 KB groups: total block bytes <= 1.10 x liblz4's LZ4_compress_default"""
    groups = [zc.shape_group(s) for s in zc.SHAPES]
    ours = _check(groups, lanes=(32,))
    for name, g, b in zip(zc.SHAPES, groups, ours):
        assert len(b) <= 1.10 * len(zc.lz4_compress(g)), name
    assert sum(map(len, ours)) <= 1.10 * sum(len(zc.lz4_compress(g)) for g in groups)
