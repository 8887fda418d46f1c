"""LZ4 block compression of serialised SLS groups on the GPU (lc_lz4_compress_dev, lc_lz4_compress).

Reports, in one JSON line with the card's name and power limit:
  * per bench shape (tests/lz4_cases.py: C2 regex-parsed, C2 / C4 split only, C3 Java records, C1 random lines):
    compress GB/s of input and the ratio for 2 048 segments of 512 KB, device-resident (CUDA events over windows of at
    least --window-s after --warmup calls; median over --windows);
  * the same for one 512 KB segment and one 10 MB segment (C2 regex-parsed bytes);
  * the host-buffer call lc_lz4_compress on the 2 048 C2 regex-parsed groups (pinned buffers, host clock around calls
    that end in a synchronise), with the H2D and D2H bytes its arguments make it copy;
  * lc_regex_parse_sls against lc_regex_parse_sls_lz4 on C2 lines and lc_delim_parse_sls against
    lc_delim_parse_sls_lz4 on C4 lines (--parse-lines lines, wall time median over --host-reps), with the H2D and D2H
    bytes each copies (counted from the arguments and the returned sizes);
  * liblz4's LZ4_compress_default on one CPU core over 64 of the same groups per shape (GB/s and ratio), the CPU arm.
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
    ap.add_argument("--parse-lines", type=int, default=1 << 20)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from tests import lz4_cases as zc
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = lc.capi.lib()
    eng = lc.Engine(0)
    stream = torch.cuda.ExternalStream(eng.stream)

    def timed(segs):
        """(GB/s of input, ratio) of lc_lz4_compress_dev over segs, device-resident"""
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
        need = eng.lz4_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr())
        out = torch.empty(need, dtype=torch.uint8, device="cuda")
        bo = torch.empty(n, dtype=torch.int64, device="cuda")
        bl = torch.empty(n, dtype=torch.int32, device="cuda")

        def call():
            return eng.lz4_compress_dev(d.data_ptr(), n, d_off.data_ptr(), d_len.data_ptr(), out.data_ptr(), need,
                                        bo.data_ptr(), bl.data_ptr())
        for _ in range(a.warmup):
            call()
        rates = []
        for _ in range(a.windows):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            calls, t0 = 0, time.perf_counter()
            e0.record(stream)
            while time.perf_counter() - t0 < a.window_s:
                assert call() == need
                calls += 1
            e1.record(stream)
            e1.synchronize()
            rates.append(int(lens.sum()) * calls / (e0.elapsed_time(e1) * 1e6))
        return float(np.median(rates)), int(lens.sum()) / need

    res = {}
    groups = {}
    for shape in zc.SHAPES:
        base = [zc.shape_group(shape, seed)[:zc.GROUP_BYTES] for seed in range(1, a.distinct + 1)]
        groups[shape] = base
        segs = [base[i % len(base)] for i in range(a.segments)]
        gbs, ratio = timed(segs)
        res[shape] = {"gpu_gb_per_s": round(gbs, 1), "ratio": round(ratio, 3)}
    c2 = groups["c2_regex"]
    res["single_512k"] = dict(zip(("gpu_gb_per_s", "ratio"), (round(x, 3) for x in timed([c2[0]]))))
    big = b"".join(c2[i % len(c2)] for i in range(20))[:10 << 20]
    res["single_10m"] = dict(zip(("gpu_gb_per_s", "ratio"), (round(x, 3) for x in timed([big]))))

    # host buffers: the 2 048 C2 groups from pinned memory, only the blocks come back
    keep = []
    segs = [c2[i % len(c2)] for i in range(a.segments)]
    hs = []
    for s in segs:
        h = pinned(L, len(s), np.uint8, keep)
        h[:] = np.frombuffer(s, np.uint8)
        hs.append(h)
    ptrs = (C.c_void_p * len(hs))(*[h.ctypes.data for h in hs])
    lens = np.array([len(s) for s in segs], np.uint32)
    cap = int(sum(int(x) + int(x) // 255 + 16 for x in lens))
    h_out = pinned(L, cap, np.uint8, keep)
    boff, blen = np.zeros(len(segs), np.uint64), np.zeros(len(segs), np.uint32)
    need = C.c_uint64(0)
    p = lc.capi._p

    def host_call():
        lc.capi._check(L.lc_lz4_compress(eng._h, len(segs), C.cast(ptrs, C.c_void_p), p(lens), p(h_out), cap, p(boff),
                                         p(blen), C.byref(need)))
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
                            "h2d_bytes": raw + 20 * len(segs), "d2h_bytes": int(need.value) + 12 * len(segs)}
    for ptr in keep:
        L.lc_host_free(ptr)

    # fused parse + serialise + compress against parse + serialise, host buffers
    from loongcollector_b200 import synth
    tail = b"\x1a\x05topic\x22\x06source"

    def wall(fn):
        fn()
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            out = fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), out
    buf, off, ln = synth.nginx_lines(a.parse_lines, seed=1)
    n = int(off.size)
    times = (1700000000 + np.arange(n) % 86400).astype(np.uint32)
    rx = lc.Regex(synth.NGINX_PATTERN)
    keys = [k.encode() for k in synth.NGINX_KEYS]
    t_sls, (wire, _) = wall(lambda: eng.regex_parse_sls(rx, buf, off, ln, times, keys, b"content"))
    t_lz4, (block, rawn, _) = wall(lambda: eng.regex_parse_sls_lz4(rx, buf, off, ln, times, keys, b"content",
                                                                    tail=tail))
    assert rawn == len(wire) + len(tail)
    h2d = int(buf.size) + 12 * n
    res["c2_regex_parse_sls"] = {"lines": n, "arena_bytes": int(buf.size), "sls_ms": round(t_sls, 2),
                                 "sls_lz4_ms": round(t_lz4, 2), "h2d_bytes": {"sls": h2d, "sls_lz4": h2d + len(tail)},
                                 "d2h_bytes": {"sls": len(wire), "sls_lz4": len(block)}}
    buf, off, ln = synth.csv_lines(a.parse_lines, seed=1)
    n = int(off.size)
    times = (1700000000 + np.arange(n) % 86400).astype(np.uint32)
    keys = [k.encode() for k in synth.CSV_KEYS]
    t_sls, (wire, _) = wall(lambda: eng.delim_parse_sls(buf, off, ln, times, b",", ord('"'), "extend", keys,
                                                        b"content"))
    t_lz4, (block, rawn, _) = wall(lambda: eng.delim_parse_sls_lz4(buf, off, ln, times, b",", ord('"'), "extend", keys,
                                                                    b"content", tail=tail))
    assert rawn == len(wire) + len(tail)
    h2d = int(buf.size) + 12 * n
    res["c4_delim_parse_sls"] = {"lines": n, "arena_bytes": int(buf.size), "sls_ms": round(t_sls, 2),
                                 "sls_lz4_ms": round(t_lz4, 2), "h2d_bytes": {"sls": h2d, "sls_lz4": h2d + len(tail)},
                                 "d2h_bytes": {"sls": len(wire), "sls_lz4": len(block)}}

    # CPU arm: liblz4, one core
    cpu = {}
    if zc.liblz4() is not None:
        for shape, base in groups.items():
            data = [base[i % len(base)] for i in range(64)]
            t0 = time.perf_counter()
            outs = [zc.lz4_compress(g) for g in data]
            dt = time.perf_counter() - t0
            cpu[shape] = {"gb_per_s": round(sum(map(len, data)) / dt / 1e9, 3),
                          "ratio": round(sum(map(len, data)) / sum(map(len, outs)), 3)}
    name, pl = card()
    print(json.dumps({"metric": "lz4_compress", "gpu": name, "power_limit_w": pl, "segments": a.segments,
                      "segment_bytes": zc.GROUP_BYTES, "gpu_dev": res, "liblz4_1core": cpu,
                      "liblz4_version": int(zc.liblz4().LZ4_versionNumber()) if zc.liblz4() is not None else None}))
    eng.close()


if __name__ == "__main__":
    main()
