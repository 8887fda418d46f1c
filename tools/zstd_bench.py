"""zstd frame compression of serialised SLS groups on the GPU (lc_zstd_compress_dev, lc_zstd_compress).

Reports, in one JSON line with the card's name and power limit (read in the same call):
  * per bench shape (tests/lz4_cases.py: C2 regex-parsed, C2 / C4 split only, C3 Java records, C1 random lines):
    compress GB/s of input and the ratio for 2 048 segments of 512 KB, device-resident, for lc_zstd_compress_dev and
    for lc_lz4_compress_dev on the same segments, the two alternated window by window (CUDA events over windows of at
    least --window-s after --warmup calls; median over --windows);
  * the same for one 512 KB segment and one 10 MB segment (C2 regex-parsed bytes);
  * the host-buffer call lc_zstd_compress on the 2 048 C2 regex-parsed groups (pinned buffers, host clock around calls
    that end in a synchronise), with the H2D and D2H bytes its arguments make it copy;
  * libzstd's ZSTD_compress at level 1 on one CPU core over 64 of the same groups per shape (GB/s and ratio), the CPU
    arm, through ctypes on the system's libzstd.so.1.
Needs a CUDA device; there is no CPU path."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.delim_sls_bench import card, pinned  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--segments", type=int, default=2048)
    ap.add_argument("--distinct", type=int, default=8, help="distinct groups per shape, repeated over the segments")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--window-s", type=float, default=1.0)
    ap.add_argument("--host-reps", type=int, default=5)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from tests import lz4_cases as zc
    from tests import zstd_cases as zs
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = lc.capi.lib()
    eng = lc.Engine(0)
    stream = torch.cuda.ExternalStream(eng.stream)

    def timed(segs):
        """{zstd, lz4}: (GB/s of input, ratio) of the two _dev calls over segs, device-resident, windows alternated"""
        lens = np.array([len(s) for s in segs], np.uint32)
        offs = np.zeros(len(segs), np.int64)
        offs[1:] = np.cumsum(((lens.astype(np.int64) + 15) // 16 * 16)[:-1])
        host = np.zeros(int(offs[-1]) + int(lens[-1]) + 16, np.uint8)
        for o, s in zip(offs.tolist(), segs):
            host[o:o + len(s)] = np.frombuffer(s, np.uint8)
        d = torch.from_numpy(host).cuda()
        d_off = torch.from_numpy(offs).cuda()
        d_len = torch.from_numpy(lens.view(np.int32)).cuda()
        n = len(segs)
        calls = {}
        for name, fn in (("zstd", eng.zstd_compress_dev), ("lz4", eng.lz4_compress_dev)):
            need = fn(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr())
            out = torch.empty(need, dtype=torch.uint8, device="cuda")
            bo = torch.empty(n, dtype=torch.int64, device="cuda")
            bl = torch.empty(n, dtype=torch.int32, device="cuda")
            calls[name] = (fn, need, out, bo, bl)
        rates = {k: [] for k in calls}
        for _ in range(a.warmup):
            for fn, need, out, bo, bl in calls.values():
                fn(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr(), out.data_ptr(), need, bo.data_ptr(),
                   bl.data_ptr())
        for _ in range(a.windows):
            for k, (fn, need, out, bo, bl) in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                c, t0 = 0, time.perf_counter()
                e0.record(stream)
                while time.perf_counter() - t0 < a.window_s:
                    assert fn(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr(), out.data_ptr(), need,
                              bo.data_ptr(), bl.data_ptr()) == need
                    c += 1
                e1.record(stream)
                e1.synchronize()
                rates[k].append(int(lens.sum()) * c / (e0.elapsed_time(e1) * 1e6))
        return {k: {"gpu_gb_per_s": round(float(np.median(rates[k])), 2),
                    "ratio": round(int(lens.sum()) / calls[k][1], 3)} for k in calls}

    res = {}
    groups = {}
    for shape in zc.SHAPES:
        base = [zc.shape_group(shape, seed)[:zc.GROUP_BYTES] for seed in range(1, a.distinct + 1)]
        groups[shape] = base
        res[shape] = timed([base[i % len(base)] for i in range(a.segments)])
    c2 = groups["c2_regex"]
    res["single_512k"] = timed([c2[0]])
    res["single_10m"] = timed([b"".join(c2[i % len(c2)] for i in range(20))[:10 << 20]])

    # host buffers: the 2 048 C2 groups from pinned memory, only the frames come back
    keep = []
    segs = [c2[i % len(c2)] for i in range(a.segments)]
    hs = []
    for s in segs:
        h = pinned(L, len(s), np.uint8, keep)
        h[:] = np.frombuffer(s, np.uint8)
        hs.append(h)
    ptrs = (C.c_void_p * len(hs))(*[h.ctypes.data for h in hs])
    lens = np.array([len(s) for s in segs], np.uint32)
    cap = int(sum(zs.bound(int(x)) for x in lens))
    h_out = pinned(L, cap, np.uint8, keep)
    foff, flen = np.zeros(len(segs), np.uint64), np.zeros(len(segs), np.uint32)
    need = C.c_uint64(0)
    p = lc.capi._p

    def host_call():
        lc.capi._check(L.lc_zstd_compress(eng._h, len(segs), C.cast(ptrs, C.c_void_p), p(lens), p(h_out), cap,
                                          p(foff), p(flen), C.byref(need)))
    host_call()
    ts = []
    for _ in range(a.host_reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host_call()
        ts.append((time.perf_counter() - t0) * 1e3)
    raw = int(lens.sum())
    res["host_c2_regex"] = {"ms_median": round(float(np.median(ts)), 2),
                            "gb_per_s": round(raw / (float(np.median(ts)) * 1e6), 2),
                            "h2d_bytes": raw + 28 * len(segs), "d2h_bytes": int(need.value) + 12 * len(segs)}
    for ptr in keep:
        L.lc_host_free(ptr)

    # CPU arm: libzstd level 1, one core
    cpu = {}
    if zs.libzstd() is not None:
        for shape, base in groups.items():
            data = [base[i % len(base)] for i in range(64)]
            t0 = time.perf_counter()
            outs = [zs.zstd_compress(g, 1) for g in data]
            dt = time.perf_counter() - t0
            cpu[shape] = {"gb_per_s": round(sum(map(len, data)) / dt / 1e9, 3),
                          "ratio": round(sum(map(len, data)) / sum(map(len, outs)), 3)}
    name, pl = card()
    print(json.dumps({"metric": "zstd_compress", "gpu": name, "power_limit_w": pl, "segments": a.segments,
                      "segment_bytes": zc.GROUP_BYTES, "gpu_dev": res, "libzstd_level1_1core": cpu,
                      "libzstd_version": int(zs.libzstd().ZSTD_versionNumber()) if zs.libzstd() is not None else None}))
    eng.close()


if __name__ == "__main__":
    main()
