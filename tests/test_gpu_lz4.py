"""GPU tier: the LZ4 block compressor.  lc_lz4_compress_dev and lc_lz4_compress against the host build of the same
functions (tests/emul/lz4.py) byte for byte, every block decoded by the strict decoder (tests/lz4_block.py) and by the
system's liblz4 when it is installed.  Output buffers are poisoned and followed by guard bytes."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests import lz4_block  # noqa: E402
from tests import lz4_cases as zc  # noqa: E402
from tests.emul import lz4  # noqa: E402

POISON, GUARD = 0xA5, 256


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def _device_segments(segs, align=0):
    """the segments packed on the device (segment g at 16 * g + align bytes past its predecessor's end); returns
    (buffer, d_seg_off, d_seg_len)"""
    import torch
    offs, pos = [], align
    for s in segs:
        offs.append(pos)
        pos += len(s) + 16 + (16 - len(s) % 16) % 16
    host = np.zeros(pos + 16, np.uint8)
    for o, s in zip(offs, segs):
        host[o:o + len(s)] = np.frombuffer(s, np.uint8)
    d = torch.from_numpy(host).cuda()
    d_off = torch.tensor(np.array(offs or [0], np.int64), device="cuda")
    d_len = torch.tensor(np.array([len(s) for s in segs] or [0], np.uint32).view(np.int32), device="cuda")
    return d, d_off, d_len


def device_compress(eng, segs, align=0):
    """lc_lz4_compress_dev into poisoned buffers followed by guard bytes; checks the sizing query, the guards and the
    block table; returns the blocks"""
    import torch
    d, d_off, d_len = _device_segments(segs, align)
    n = len(segs)
    need = eng.lz4_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr())
    out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    boff = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda")
    blen = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    got = eng.lz4_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr(), out.data_ptr(), need,
                               boff.data_ptr(), blen.data_ptr())
    assert got == need
    h = out.cpu().numpy()
    assert (h[need:] == POISON).all(), "wrote past the output"
    bo, bl = boff.cpu().numpy(), blen.cpu().numpy().view(np.uint32)
    assert bo[n] == -1 and bl[n] == 0xFFFFFFFF, "wrote past the block table"
    assert bo[0] == 0 and all(bo[g] + bl[g] == (bo[g + 1] if g + 1 < n else need) for g in range(n))
    return [bytes(h[int(o):int(o) + int(ln)]) for o, ln in zip(bo[:n], bl[:n])]


def _verify(segs, blocks):
    for s, b in zip(segs, blocks):
        assert len(b) <= len(s) + len(s) // 255 + 16
        assert lz4_block.decode(b) == s
        if zc.liblz4() is not None:
            assert zc.lz4_decompress(b, len(s)) == s


@pytest.mark.parametrize("part", range(4))
def test_edge_matrix_equals_emulation(eng, part):
    segs = [s for i, (_, s) in enumerate(zc.edge_segments()) if i % 4 == part]
    got = device_compress(eng, segs, align=part * 5)
    assert got == lz4.compress(segs)
    _verify(segs, got)
    assert eng.lz4_compress(segs) == got


@pytest.mark.parametrize("shape", zc.SHAPES)
def test_shapes_equal_emulation(eng, shape):
    segs = [zc.shape_group(shape, seed) for seed in (1, 2)]
    got = device_compress(eng, segs)
    assert got == lz4.compress(segs)
    _verify(segs, got)
    assert eng.lz4_compress(segs) == got


def test_incompressible_10mib(eng):
    segs = [random.Random(10).randbytes(10 << 20), b"", random.Random(1).randbytes(1 << 20)]
    got = device_compress(eng, segs, align=3)
    assert got == lz4.compress(segs)
    _verify(segs, got)


def test_capacity_refusal_reports_exact_size(eng):
    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi
    segs = [zc.shape_group("c4_csv"), b"", b"abc" * 1000]
    d, d_off, d_len = _device_segments(segs)
    need = eng.lz4_compress_dev(d.data_ptr(), 3, d_off.data_ptr(), d_len.data_ptr())
    assert need == sum(map(len, lz4.compress(segs)))
    out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    boff = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    blen = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    got = C.c_uint64(0)
    rc = capi.lib().lc_lz4_compress_dev(eng._h, C.c_void_p(d.data_ptr()), 3, C.c_void_p(d_off.data_ptr()),
                                        C.c_void_p(d_len.data_ptr()), C.c_void_p(out.data_ptr()), need - 1,
                                        C.c_void_p(boff.data_ptr()), C.c_void_p(blen.data_ptr()), C.byref(got))
    assert rc == capi.LC_ERR_CAPACITY and got.value == need
    assert (out.cpu().numpy() == POISON).all()
    assert (boff.cpu().numpy() == -1).all() and (blen.cpu().numpy() == -1).all()
    with pytest.raises(lc.LcError):
        eng.lz4_compress(segs, out_cap=need - 1)


def test_too_large_segment_is_refused(eng):
    import torch

    import loongcollector_b200 as lc
    n = 0x7E000001
    d = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros(2, dtype=torch.int64, device="cuda")
    d_len = torch.tensor(np.array([5, n], np.uint32).view(np.int32), device="cuda")
    with pytest.raises(lc.LcError) as ei:
        eng.lz4_compress_dev(d.data_ptr(), 2, d_off.data_ptr(), d_len.data_ptr())
    assert ei.value.code == lc.capi.LC_ERR_TOO_LARGE
    del d


def test_2048_groups_and_a_10mb_segment_in_one_call(eng):
    """2 048 segments of 512 KB (the five shapes, several seeds each) plus one 10 MB segment"""
    base = [zc.shape_group(s, seed) for s in zc.SHAPES for seed in (1, 2, 3)]
    segs = [base[i % len(base)][:512 << 10] for i in range(2048)]
    segs.append(random.Random(9).randbytes(10 << 20))
    got = device_compress(eng, segs)
    # segments compress independently: the emulation of the distinct ones pins all of them
    want = dict(zip(range(len(base)), lz4.compress(segs[:len(base)])))
    for i in range(2048):
        assert got[i] == want[i % len(base)], i
    assert got[2048] == lz4.compress([segs[2048]])[0]
    _verify(segs[:len(base)] + segs[2048:], got[:len(base)] + got[2048:])
    assert eng.lz4_compress(segs) == got
