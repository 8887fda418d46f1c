"""GPU tier: the zstd frame compressor.  lc_zstd_compress_dev and lc_zstd_compress against the host build of the same
functions (tests/emul/zstd.py) byte for byte, every frame decoded by the strict decoder (tests/zstd_frame.py) and by
the system's libzstd when it loads.  Output buffers are poisoned and followed by guard bytes."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from tests import lz4_cases as zc  # noqa: E402
from tests import zstd_cases as zs  # noqa: E402
from tests import zstd_frame  # noqa: E402
from tests.emul import zstd  # noqa: E402
from tests.test_gpu_lz4 import GUARD, POISON, _device_segments  # noqa: E402


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


def device_compress(eng, segs, align=0):
    """lc_zstd_compress_dev into poisoned buffers followed by guard bytes; checks the sizing query, the guards and the
    frame table; returns the frames"""
    import torch
    d, d_off, d_len = _device_segments(segs, align)
    n = len(segs)
    need = eng.zstd_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr())
    out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    foff = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda")
    flen = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    got = eng.zstd_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr(), out.data_ptr(), need,
                                foff.data_ptr(), flen.data_ptr())
    assert got == need
    h = out.cpu().numpy()
    assert (h[need:] == POISON).all(), "wrote past the output"
    fo, fl = foff.cpu().numpy(), flen.cpu().numpy().view(np.uint32)
    assert fo[n] == -1 and fl[n] == 0xFFFFFFFF, "wrote past the frame table"
    assert fo[0] == 0 and all(fo[g] + fl[g] == (fo[g + 1] if g + 1 < n else need) for g in range(n))
    return [bytes(h[int(o):int(o) + int(ln)]) for o, ln in zip(fo[:n], fl[:n])]


def _verify(segs, frames):
    for s, f in zip(segs, frames):
        assert len(f) <= zs.bound(len(s))
        assert zstd_frame.decode(f) == s
        if zs.libzstd() is not None:
            assert zs.zstd_decompress(f, len(s)) == s


@pytest.mark.parametrize("part", range(4))
def test_edge_matrix_equals_emulation(eng, part):
    segs = [s for i, (_, s) in enumerate(zc.edge_segments() + zs.block_segments()) if i % 4 == part]
    got = device_compress(eng, segs, align=part * 5)
    assert got == zstd.compress(segs)
    _verify(segs, got)
    assert eng.zstd_compress(segs) == got


@pytest.mark.parametrize("shape", zc.SHAPES)
def test_shapes_equal_emulation(eng, shape):
    segs = [zc.shape_group(shape, seed) for seed in (1, 2)]
    got = device_compress(eng, segs)
    assert got == zstd.compress(segs)
    _verify(segs, got)
    assert eng.zstd_compress(segs) == got


def test_capacity_refusal_reports_exact_size(eng):
    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi
    segs = [zc.shape_group("c4_csv"), b"", b"abc" * 1000]
    d, d_off, d_len = _device_segments(segs)
    need = eng.zstd_compress_dev(d.data_ptr(), 3, d_off.data_ptr(), d_len.data_ptr())
    assert need == sum(map(len, zstd.compress(segs)))
    out = torch.full((need + GUARD,), POISON, dtype=torch.uint8, device="cuda")
    foff = torch.full((3,), -1, dtype=torch.int64, device="cuda")
    flen = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    got = C.c_uint64(0)
    rc = capi.lib().lc_zstd_compress_dev(eng._h, C.c_void_p(d.data_ptr()), 3, C.c_void_p(d_off.data_ptr()),
                                         C.c_void_p(d_len.data_ptr()), C.c_void_p(out.data_ptr()), need - 1,
                                         C.c_void_p(foff.data_ptr()), C.c_void_p(flen.data_ptr()), C.byref(got))
    assert rc == capi.LC_ERR_CAPACITY and got.value == need
    assert (out.cpu().numpy() == POISON).all()
    assert (foff.cpu().numpy() == -1).all() and (flen.cpu().numpy() == -1).all()
    with pytest.raises(lc.LcError):
        eng.zstd_compress(segs, out_cap=need - 1)


def test_too_large_segment_is_refused(eng):
    import torch

    import loongcollector_b200 as lc
    n = 0x7E000001
    d = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros(2, dtype=torch.int64, device="cuda")
    d_len = torch.tensor(np.array([5, n], np.uint32).view(np.int32), device="cuda")
    with pytest.raises(lc.LcError) as ei:
        eng.zstd_compress_dev(d.data_ptr(), 2, d_off.data_ptr(), d_len.data_ptr())
    assert ei.value.code == lc.capi.LC_ERR_TOO_LARGE
    del d


def test_2048_groups_and_a_10mb_segment_in_one_call(eng):
    """2 048 segments of 512 KB (the five shapes, several seeds each) plus one 10 MB segment"""
    base = [zc.shape_group(s, seed) for s in zc.SHAPES for seed in (1, 2, 3)]
    segs = [base[i % len(base)][:512 << 10] for i in range(2048)]
    segs.append(random.Random(9).randbytes(10 << 20))
    got = device_compress(eng, segs)
    # segments compress independently: the emulation of the distinct ones pins all of them
    want = zstd.compress(segs[:len(base)])
    for i in range(2048):
        assert got[i] == want[i % len(base)], i
    assert got[2048] == zstd.compress([segs[2048]])[0]
    _verify(segs[:len(base)] + segs[2048:], got[:len(base)] + got[2048:])
    assert eng.zstd_compress(segs) == got


def test_host_zstd_compressor(eng):
    """ZstdCompressor (lc_host_zstd_compress) returns lc_zstd_compress's frames"""
    from loongcollector_b200 import capi
    inputs = [zc.shape_group("c2_regex"), b"", b"x", b"hello " * 5000]
    frames, err = capi.host_zstd_compress(inputs)
    assert err is None
    assert frames == eng.zstd_compress(inputs)
    _verify(inputs, frames)
    assert capi.host_zstd_compress([]) == ([], None)
