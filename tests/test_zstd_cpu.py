"""CPU tier: the zstd frame compressor's block and emit functions (lc_exec.cuh, built for the host by
tests/emul/zstd.py) over the LZ4 parse pass, with 1, 3 and 32 emulated lanes.  The lane counts agree byte for byte;
every frame decodes, through the strict RFC 8878 decoder of tests/zstd_frame.py and through the system's libzstd when
it loads, to its segment, and stays within ZSTD_compressBound; on the bench shapes each frame is at most 0.90 x our LZ4
block and the total at most 1.35 x libzstd level 1."""
import random

import pytest

from tests import lz4_cases as zc
from tests import zstd_cases as zs
from tests import zstd_frame
from tests.emul import lz4, zstd

LANES = (1, 3, 32)
needs_libzstd = pytest.mark.skipif(zs.libzstd() is None, reason="the system's libzstd (libzstd.so.1) is not installed")


def _check(segs, lanes=LANES):
    """compresses segs with every lane count; checks agreement, decoding and the bound; returns the frames"""
    frames = zstd.compress(segs, lanes[0])
    for w in lanes[1:]:
        assert zstd.compress(segs, w) == frames, w
    for s, f in zip(segs, frames):
        assert len(f) <= zs.bound(len(s))
        assert zstd_frame.decode(f) == s
        if zs.libzstd() is not None:
            assert zs.zstd_decompress(f, len(s)) == s
    return frames


@pytest.mark.parametrize("part", range(4))
def test_lz4_edge_matrix(part):
    _check([s for i, (_, s) in enumerate(zc.edge_segments()) if i % 4 == part])


@pytest.mark.parametrize("part", range(3))
def test_block_edges(part):
    _check([s for i, (_, s) in enumerate(zs.block_segments()) if i % 3 == part])


def test_empty_and_one_byte():
    assert zstd.compress([b""]) == [bytes.fromhex("28b52ffd2000010000")]
    assert _check([b"", b"x", b""]) == [bytes.fromhex("28b52ffd2000010000"), bytes.fromhex("28b52ffd2001090000") + b"x",
                                        bytes.fromhex("28b52ffd2000010000")]


def test_content_size_field():
    for n, desc, fcs in ((255, 0x20, b"\xff"), (256, 0x60, b"\x00\x00"), (65791, 0x60, b"\xff\xff"),
                         (65792, 0xA0, (65792).to_bytes(4, "little"))):
        [f] = _check([bytes(n)])
        assert f[4] == desc and f[5:5 + len(fcs)] == fcs


def test_one_repeated_byte_is_small():
    [f] = _check([b"z" * (10 << 20)])
    assert len(f) < 2000


@pytest.mark.parametrize("mib", [1, 10])
def test_random_bytes_are_raw_blocks(mib):
    s = random.Random(mib).randbytes(mib << 20)
    [f] = _check([s], lanes=(32,) if mib > 1 else LANES)
    hdr = 9  # magic, descriptor, 4-byte content size
    assert len(f) == hdr + 3 * (len(s) // zs.BLOCK) + len(s)
    assert all(f[hdr + k * (zs.BLOCK + 3)] & 6 == 0 for k in range(len(s) // zs.BLOCK))  # Raw block type


def test_many_segments():
    rng = random.Random(5)
    segs = []
    for i in range(300):
        k = rng.randrange(4)
        n = [0, rng.randrange(1, 40), rng.randrange(40, 3000), rng.randrange(3000, 300000)][k]
        segs.append((b"log line %d " % rng.randrange(50) * (n // 10 + 1))[:n] if i % 2 else rng.randbytes(n))
    _check(segs)


@needs_libzstd
@pytest.mark.parametrize("level", [1, 3])
def test_decoder_reads_libzstd_frames(level):
    for shape in zc.SHAPES:
        g = zc.shape_group(shape)
        assert zstd_frame.decode(zs.zstd_compress(g, level)) == g


def test_decoder_rejects_malformed_frames():
    [f] = zstd.compress([zc.shape_group("c4_csv")])
    bad = [f + b"\x00", f[:-1], f[:4] + bytes([f[4] | 8]) + f[5:],  # trailing byte, truncation, reserved bit
           f[:5] + bytes([f[5] ^ 1]) + f[6:]]                         # content size
    for b in bad:
        with pytest.raises(zstd_frame.ZstdError):
            zstd_frame.decode(b)


def test_ratio_gate_against_lz4():
    """on the five bench shapes, as 512 KB groups: each frame <= 0.90 x our LZ4 block of the same group"""
    groups = [zc.shape_group(s) for s in zc.SHAPES]
    ours = _check(groups, lanes=(32,))
    for name, g, f, b in zip(zc.SHAPES, groups, ours, lz4.compress(groups)):
        assert len(f) <= 0.90 * len(b), name


@needs_libzstd
def test_ratio_gate_against_libzstd():
    """the total over the five shapes <= 1.35 x libzstd level 1's"""
    groups = [zc.shape_group(s) for s in zc.SHAPES]
    ours = zstd.compress(groups)
    assert sum(map(len, ours)) <= 1.35 * sum(len(zs.zstd_compress(g, 1)) for g in groups)
