"""Split -> Apsara -> SLS wire format on synth.apsara_lines (80 B - 2 KB) joined by "\n", with log.file.offset
metadata (offset key on) and no history discard (the generator's times start in 2023).

Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident chain lc_split_lines_dev + lc_apsara_parse_dev (one group) + lc_sls_serialize_split_apsara_dev,
    at one 512 KB reader chunk and at --lines lines -- CUDA events, median over --steps after --warmup;
  * the kernel time of one step at --lines lines, split into the Apsara scan and field passes (ap_scan / ap_emit),
    the time-cache resolve (ap_resolve: one warp walks the whole group), the size / emit passes (split_apsara_sls_*)
    and LZ4 (lz4_*, from one lc_split_apsara_parse_sls_lz4 call over the same lines) -- torch.profiler with CUDA
    activities, in a run of its own after the timed ones;
  * the same kernel split for one step over one 512 KB chunk;
  * lc_split_apsara_parse_sls and lc_split_apsara_parse_sls_lz4 over --chunks chunks of 512 KB with pinned host
    buffers (host clock around calls that end in a synchronise, sum over the chunks, median over --host-reps);
  * ProcessorSplitLogStringNative::SerializeSls(group, apsara) against Process + Process + Serialize on 512 KB groups
    of one source event, both through the JSON host API (lc_host_chain_serialize_sls modes 0 and 1, the history
    discard off; the JSON parse of the group description is in both).
Needs a CUDA device; there is no CPU path."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.delim_sls_bench import card, pinned  # noqa: E402

OKEY = b"__file_offset__"
CHUNK = 512 * 1024


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=1 << 20)
    ap.add_argument("--chunks", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--groups", type=int, default=8)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    apx = lc.Apsara("content")
    stream = torch.cuda.ExternalStream(eng.stream)
    p = lambda x: C.c_void_p(x) if isinstance(x, int) else capi._p(x)  # noqa: E731
    buf, off, ln, _grp = synth.apsara_lines(a.lines, seed=1)
    packed = bytes(buf)
    src = b"\n".join(packed[o:o + n] for o, n in zip(off.tolist(), ln.tolist()))
    cut = src.rfind(b"\n", 0, CHUNK) + 1
    chunk_val = src[:cut]
    cfg = [b"content", 7, 0, 0, 0, OKEY, len(OKEY), 4096, 1700000000, 0xFFFFFFFF, 0]
    NOW, DI = 1700000000, -1

    def device_setup(val):
        n_src = len(val)
        d = torch.from_numpy(np.frombuffer(val, np.uint8).copy()).cuda()
        t = dict(d=d, n_src=n_src, off=torch.empty(n_src, dtype=torch.int32, device="cuda"),
                 len=torch.empty(n_src, dtype=torch.int32, device="cuda"),
                 st=torch.empty(n_src, dtype=torch.uint8, device="cuda"),
                 sec=torch.empty(n_src, dtype=torch.int64, device="cuda"),
                 nsec=torch.empty(n_src, dtype=torch.int32, device="cuda"),
                 micro=torch.empty(n_src, dtype=torch.int64, device="cuda"),
                 first=torch.empty(n_src + 1, dtype=torch.int64, device="cuda"),
                 grp=torch.empty(2, dtype=torch.int32, device="cuda"),
                 cnt=torch.empty(5, dtype=torch.int64, device="cuda"), ctr=np.zeros(5, np.uint64))
        t["n"] = eng.split_lines_dev(d.data_ptr(), n_src, 10, t["off"].data_ptr(), t["len"].data_ptr(), n_src)
        t["grp"].copy_(torch.tensor([0, t["n"]], dtype=torch.int32))
        m = C.c_uint64(0)
        L.lc_apsara_parse_dev(eng._h, apx._h, p(d.data_ptr()), n_src, p(t["off"].data_ptr()),
                              p(t["len"].data_ptr()), t["n"], p(t["grp"].data_ptr()), 1, NOW, DI,
                              p(t["st"].data_ptr()), p(t["sec"].data_ptr()), p(t["nsec"].data_ptr()),
                              p(t["micro"].data_ptr()), p(t["first"].data_ptr()), None, 0, C.byref(m),
                              p(t["cnt"].data_ptr()))
        t["ecap"] = int(m.value)
        t["ent"] = torch.empty(max(t["ecap"], 1) * 16, dtype=torch.uint8, device="cuda")
        need = C.c_uint64(0)
        step(t, None, 0, need)
        t["wire"] = int(need.value)
        t["out"] = torch.empty(t["wire"] + 16, dtype=torch.uint8, device="cuda")
        return t

    def step(t, d_out, cap, need):
        d = t["d"].data_ptr()
        nn = C.c_uint64(0)
        capi._check(L.lc_split_lines_dev(eng._h, p(d), t["n_src"], 10, p(t["off"].data_ptr()),
                                         p(t["len"].data_ptr()), t["n_src"], C.byref(nn)))
        m = C.c_uint64(0)
        capi._check(L.lc_apsara_parse_dev(eng._h, apx._h, p(d), t["n_src"], p(t["off"].data_ptr()),
                                          p(t["len"].data_ptr()), nn.value, p(t["grp"].data_ptr()), 1, NOW, DI,
                                          p(t["st"].data_ptr()), p(t["sec"].data_ptr()), p(t["nsec"].data_ptr()),
                                          p(t["micro"].data_ptr()), p(t["first"].data_ptr()), p(t["ent"].data_ptr()),
                                          t["ecap"], C.byref(m), p(t["cnt"].data_ptr())))
        rc = L.lc_sls_serialize_split_apsara_dev(eng._h, apx._h, p(d), t["n_src"], p(t["off"].data_ptr()),
                                                 p(t["len"].data_ptr()), nn.value, p(t["st"].data_ptr()),
                                                 p(t["sec"].data_ptr()), p(t["nsec"].data_ptr()),
                                                 p(t["micro"].data_ptr()), p(t["first"].data_ptr()),
                                                 p(t["ent"].data_ptr()), *cfg, p(d_out), cap, C.byref(need),
                                                 capi._p(t["ctr"]))
        if d_out is not None:
            capi._check(rc)

    def timed(t):
        need = C.c_uint64(0)
        out = t["out"].data_ptr()
        for _ in range(a.warmup):
            step(t, out, t["wire"], need)
        ts = []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            step(t, out, t["wire"], need)
            e1.record(stream)
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    big = device_setup(src)
    small = device_setup(chunk_val)
    t_big, t_small = timed(big), timed(small)

    # ---- host-buffer calls over 512 KB chunks
    keep = []
    h_src = pinned(L, cut, np.uint8, keep)
    h_src[:] = np.frombuffer(chunk_val, np.uint8)
    est = 2 * cut + 4096
    h_out = pinned(L, est, np.uint8, keep)
    sizes = {}

    def host_sls():
        need, nev = C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(5, np.uint64)
        capi._check(L.lc_split_apsara_parse_sls(eng._h, apx._h, capi._p(h_src), cut, 10, *cfg, NOW, DI,
                                                capi._p(h_out), est, C.byref(need), C.byref(nev), capi._p(ctr)))
        sizes["wire"], sizes["n"] = int(need.value), int(nev.value)

    def host_lz4():
        need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(5, np.uint64)
        capi._check(L.lc_split_apsara_parse_sls_lz4(eng._h, apx._h, capi._p(h_src), cut, 10, *cfg, NOW, DI, None, 0,
                                                    capi._p(h_out), est, C.byref(need), C.byref(raw), C.byref(nev),
                                                    capi._p(ctr)))
        sizes["blk"] = int(need.value)

    res = {}
    for name, fn in (("host_sls", host_sls), ("host_lz4", host_lz4)):
        fn()
        ts = []
        for _ in range(a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _c in range(a.chunks):
                fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[name] = float(np.median(ts))
    for ptr in keep:
        L.lc_host_free(ptr)

    # ---- kernel time of one step at --lines lines (and of the LZ4 kernels behind the fused call over the same lines),
    # then of one step over one 512 KB chunk
    from torch.profiler import ProfilerActivity, profile

    def kernel_ms(run, runs):
        """kernel ms per run by group; `runs`: how many times the chain's own kernels run inside run()"""
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        groups = {"ap_scan_fields": 0.0, "ap_resolve": 0.0, "size_emit": 0.0, "lz4": 0.0, "other": 0.0}
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None)
            us = ev.cuda_time_total if us is None else us
            k = ev.key
            # the Apsara and size / emit kernels ran `runs` times over the same lines: their mean per run; the LZ4
            # kernels ran once, in the fused call
            g = ("lz4" if "lz4_" in k else "ap_resolve" if "ap_resolve" in k else "size_emit"
                 if "split_apsara_sls" in k else "ap_scan_fields" if ("ap_scan" in k or "ap_emit" in k) else "other")
            groups[g] += us / 1e3 / (1 if g == "lz4" else runs)
        return {k: round(v, 3) for k, v in groups.items()}

    need = C.c_uint64(0)

    def big_runs():
        step(big, big["out"].data_ptr(), big["wire"], need)
        eng.split_apsara_parse_sls_lz4(apx, src, 10, b"content", offset_key=OKEY, src_pos=4096, time=1700000000,
                                       now=NOW, discard_interval=DI)
    k_big = kernel_ms(big_runs, 2)
    k_small = kernel_ms(lambda: step(small, small["out"].data_ptr(), small["wire"], need), 1)

    # ---- the host class through the JSON host API, 512 KB groups of one source event with offset metadata
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": cut,
                         "contents": {"content": chunk_val.decode("latin-1")}}]}
    jres = {}
    for mode, mname in ((0, "serialize_sls"), (1, "process_process_serialize")):
        sp = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
        xp = lc.HostProcessor("processor_parse_apsara_native", {"SourceKey": "content"})
        xp.set_discard_old_data(False)
        capi.host_chain_serialize_sls(sp, xp, group, False, mode)
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for _g in range(a.groups):
                out = capi.host_chain_serialize_sls(sp, xp, group, False, mode)
            ts.append((time.perf_counter() - t0) * 1e3 / a.groups)
        jres[mname] = (float(np.median(ts)), out[0])
    assert jres["serialize_sls"][1] == jres["process_process_serialize"][1]

    name, pl = card()
    print(json.dumps({
        "metric": "split_apsara_sls", "gpu": name, "power_limit_w": pl,
        "lines": big["n"], "bytes": big["n_src"], "wire_bytes": big["wire"],
        "dev_chain_ms_median": round(t_big, 3),
        "chunk_bytes": small["n_src"], "chunk_lines": small["n"], "chunk_dev_chain_ms_median": round(t_small, 3),
        "dev_steps": a.steps,
        "kernel_ms_per_step": k_big, "chunk_kernel_ms_per_step": k_small,
        "chunks": a.chunks, "host_split_apsara_sls_ms_median": round(res["host_sls"], 2),
        "host_split_apsara_sls_lz4_ms_median": round(res["host_lz4"], 2), "host_reps": a.host_reps,
        "chunk_wire_bytes": sizes["wire"], "chunk_lz4_bytes": sizes["blk"],
        "serialize_sls_ms_per_group": round(jres["serialize_sls"][0], 2),
        "process_process_serialize_ms_per_group": round(jres["process_process_serialize"][0], 2),
    }))
    eng.close()


if __name__ == "__main__":
    main()
