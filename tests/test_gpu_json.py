"""GPU tier of the JSON parse: lc_json_parse and lc_json_parse_dev equal the host build of the device walk and the C
oracle on every output and counter, on poisoned outputs with guard words (generated lines, pinned renderings, edges,
depths, mutated documents, slow events among fast ones, 1 MiB lines sharing warps with short ones); the capacity
refusal writes nothing and the sizing query works; an event past the buffer is refused."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import json_parse as oj  # noqa: E402
from tests import json_cases as jc  # noqa: E402
from tests.emul import json_parse as ej  # noqa: E402

POISON = 0xA5


def _eng():
    import loongcollector_b200 as lc
    return lc, lc.Engine(0)


def _check_all(got, want):
    for k in range(5):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k


def _docs():
    from loongcollector_b200 import synth
    buf, off, ln, _ = synth.json_lines(4000, seed=9)
    raw = buf.tobytes()
    lines = [raw[o:o + l] for o, l in zip(off.tolist(), ln.tolist())]
    valid = jc.valid_docs(300, seed=41)
    big = b'{"msg":"' + b"x" * (1 << 20) + b'","n":1.5,"e":"a\\nb","deep":' + b"[" * 80 + b"]" * 80 + b"}"
    docs = lines + [b'{"v":' + v + b"}" for v, _ in jc.PINNED] + jc.EDGES + jc.DEPTHS + valid + \
        jc.mutate(valid, seed=42, per=2) + [None, b""]
    for k in range(0, len(docs), 97):  # 1 MiB lines in the same warps as short ones
        docs.insert(k, big if k % 2 else big[:-1])
    return docs


def test_host_call_equals_emulation_and_oracle():
    lc, eng = _eng()
    docs = _docs()
    base, off, ln = oj.table(docs)
    want = oj.process("content", base, off, ln)
    emu = ej.parse("content", base, off, ln, 32)
    _check_all(emu, want)
    assert emu[5] > 0  # slow events among the fast ones
    got = eng.json_parse(lc.Json("content"), base, off, ln)
    _check_all(got, want)


def test_dev_call_poisoned_with_guards():
    import torch
    lc, eng = _eng()
    docs = _docs()
    base, off, ln = oj.table(docs)
    st_w, first_w, ent_w, ar_w, cnt_w = oj.process("content", base, off, ln)
    n, m, a = off.size, ent_w.shape[0], len(ar_w)
    G = 64
    dev = torch.device("cuda:0")
    d_base = torch.from_numpy(base.copy()).to(dev)
    d_off, d_len = torch.from_numpy(off.astype(np.int32)).to(dev), torch.from_numpy(ln.view(np.int32)).to(dev)
    d_st = torch.full((n + G,), POISON, dtype=torch.uint8, device=dev)
    d_first = torch.full((n + 1 + G,), -1, dtype=torch.int64, device=dev)
    d_ent = torch.full((m * 4 + G,), -0x5A5A5A5B, dtype=torch.int32, device=dev)
    d_ar = torch.full((a + G,), POISON, dtype=torch.uint8, device=dev)
    d_cnt = torch.full((3 + 1,), -1, dtype=torch.int64, device=dev)
    js = lc.Json("content")
    # sizing query: caps of 0 write no entry and no arena byte
    with pytest.raises(lc.LcError) as ex:
        eng.json_parse_dev(js, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n, d_st.data_ptr(),
                           d_first.data_ptr(), d_ent.data_ptr(), 0, d_ar.data_ptr(), 0, d_cnt.data_ptr())
    assert ex.value.code == lc.capi.LC_ERR_CAPACITY
    assert bool((d_ent == -0x5A5A5A5B).all()) and bool((d_ar == POISON).all())
    assert np.array_equal(d_first[:n + 1].cpu().numpy().view(np.uint64), first_w)
    # one short of the arena: refused, nothing written
    if a:
        with pytest.raises(lc.LcError):
            eng.json_parse_dev(js, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n,
                               d_st.data_ptr(), d_first.data_ptr(), d_ent.data_ptr(), m, d_ar.data_ptr(), a - 1,
                               d_cnt.data_ptr())
        assert bool((d_ent == -0x5A5A5A5B).all()) and bool((d_ar == POISON).all())
    mm, aa = eng.json_parse_dev(js, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), n,
                                d_st.data_ptr(), d_first.data_ptr(), d_ent.data_ptr(), m, d_ar.data_ptr(), a,
                                d_cnt.data_ptr())
    assert (mm, aa) == (m, a)
    assert np.array_equal(d_st[:n].cpu().numpy(), st_w)
    assert bool((d_st[n:] == POISON).all())
    assert np.array_equal(d_first[:n + 1].cpu().numpy().view(np.uint64), first_w)
    assert bool((d_first[n + 1:] == -1).all())
    assert np.array_equal(d_ent[:m * 4].cpu().numpy().view(np.uint32).reshape(-1, 4), ent_w)
    assert bool((d_ent[m * 4:] == -0x5A5A5A5B).all())
    assert d_ar[:a].cpu().numpy().tobytes() == ar_w
    assert bool((d_ar[a:] == POISON).all())
    assert d_cnt[:3].cpu().numpy().view(np.uint64).tolist() == cnt_w.tolist()
    assert int(d_cnt[3]) == -1


def test_capacity_refusal_and_event_past_buffer():
    lc, eng = _eng()
    docs = [b'{"a":"x\\ny","b":1.5}', b'{"c":2}']
    base, off, ln = oj.table(docs)
    js = lc.Json("content")
    with pytest.raises(lc.LcError) as ex:
        eng.json_parse(js, base, off, ln, entry_cap=2, arena_cap=100)
    assert ex.value.code == lc.capi.LC_ERR_CAPACITY
    st, first, ent, ar, cnt = eng.json_parse(js, base, off, ln)
    assert first.tolist() == [0, 2, 3] and ar == b"x\ny1.500000" and cnt.tolist() == [0, 0, 2]
    bad = ln.copy()
    bad[1] = base.size  # off[1] + len > base_len
    with pytest.raises(lc.LcError) as ex:
        eng.json_parse(js, base, off, bad)
    assert ex.value.code == lc.capi.LC_ERR_INVALID_ARG
    import torch
    d_base = torch.from_numpy(base.copy()).cuda()
    d_off = torch.from_numpy(off.astype(np.int32)).cuda()
    d_len = torch.from_numpy(bad.view(np.int32)).cuda()
    d_st = torch.zeros(2, dtype=torch.uint8, device="cuda")
    d_first = torch.zeros(3, dtype=torch.int64, device="cuda")
    d_ent = torch.zeros(16, dtype=torch.int32, device="cuda")
    d_ar = torch.zeros(64, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    with pytest.raises(lc.LcError) as ex:
        eng.json_parse_dev(js, d_base.data_ptr(), base.size, d_off.data_ptr(), d_len.data_ptr(), 2, d_st.data_ptr(),
                           d_first.data_ptr(), d_ent.data_ptr(), 4, d_ar.data_ptr(), 64, d_cnt.data_ptr())
    assert ex.value.code == lc.capi.LC_ERR_INVALID_ARG
