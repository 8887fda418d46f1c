"""Split -> JSON -> SLS wire format on synth.json_lines (150 B - 2 KB), with log.file.offset metadata (offset key on).

Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident chain lc_split_lines_dev + lc_json_parse_dev + lc_sls_serialize_split_json_dev, at one
    512 KB reader chunk and at --lines lines -- CUDA events, median over --steps after --warmup;
  * the kernel time of one step at --lines lines, split into the JSON passes (json_*_kernel), the resolve
    (json_resolve_*), the size / emit passes (split_json_sls_*) and LZ4 (lz4_*, from one lc_split_json_parse_sls_lz4
    call over the same lines) -- torch.profiler with CUDA activities, in a run of its own after the timed ones;
  * the same kernel split for one step over one 512 KB chunk, with the step's wall time beside it, so that the
    chunk's time can be told apart from its kernels' (the rest is launches and host synchronisations);
  * lc_split_json_parse_sls and lc_split_json_parse_sls_lz4 over --chunks chunks of 512 KB with pinned host buffers
    (host clock around calls that end in a synchronise, sum over the chunks, median over --host-reps);
  * ProcessorSplitLogStringNative::SerializeSls(group, json) against Process + Process + Serialize on 512 KB groups
    of one source event, both through the JSON host API (lc_host_chain_serialize_sls modes 0 and 1; the JSON parse
    of the group description is in both).
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
    ap.add_argument("--json-groups", type=int, default=8)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    js = lc.Json("content")
    stream = torch.cuda.ExternalStream(eng.stream)
    p = lambda x: C.c_void_p(x) if isinstance(x, int) else capi._p(x)  # noqa: E731
    # lines of 150 B - 2 KB, so that 1 Mi of them stay below the chain's 2 GiB source limit
    buf = synth.json_lines(a.lines, seed=1, hi=2048)[0]
    src = bytes(buf)
    cut = src.rfind(b"\n", 0, CHUNK) + 1
    chunk_val = src[:cut]
    cfg = [b"content", 7, 0, 0, 0, OKEY, len(OKEY), 4096, 1700000000, 0xFFFFFFFF]

    def device_setup(val):
        n_src = len(val)
        d = torch.from_numpy(np.frombuffer(val, np.uint8).copy()).cuda()
        t = dict(d=d, n_src=n_src, off=torch.empty(n_src, dtype=torch.int32, device="cuda"),
                 len=torch.empty(n_src, dtype=torch.int32, device="cuda"),
                 st=torch.empty(n_src, dtype=torch.uint8, device="cuda"),
                 first=torch.empty(n_src + 1, dtype=torch.int64, device="cuda"),
                 cnt=torch.empty(3, dtype=torch.int64, device="cuda"), ctr=np.zeros(3, np.uint64))
        t["n"] = eng.split_lines_dev(d.data_ptr(), n_src, 10, t["off"].data_ptr(), t["len"].data_ptr(), n_src)
        m, ab = C.c_uint64(0), C.c_uint64(0)
        L.lc_json_parse_dev(eng._h, js._h, p(d.data_ptr()), n_src, p(t["off"].data_ptr()), p(t["len"].data_ptr()),
                            t["n"], p(t["st"].data_ptr()), p(t["first"].data_ptr()), None, 0, C.byref(m), None, 0,
                            C.byref(ab), p(t["cnt"].data_ptr()))
        t["ecap"], t["acap"] = int(m.value), int(ab.value)
        t["ent"] = torch.empty(max(t["ecap"], 1) * 16, dtype=torch.uint8, device="cuda")
        t["ar"] = torch.empty(max(t["acap"], 1), dtype=torch.uint8, device="cuda")
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
        m, ab = C.c_uint64(0), C.c_uint64(0)
        capi._check(L.lc_json_parse_dev(eng._h, js._h, p(d), t["n_src"], p(t["off"].data_ptr()),
                                        p(t["len"].data_ptr()), nn.value, p(t["st"].data_ptr()),
                                        p(t["first"].data_ptr()), p(t["ent"].data_ptr()), t["ecap"], C.byref(m),
                                        p(t["ar"].data_ptr()), t["acap"], C.byref(ab), p(t["cnt"].data_ptr())))
        rc = L.lc_sls_serialize_split_json_dev(eng._h, js._h, p(d), t["n_src"], p(t["off"].data_ptr()),
                                               p(t["len"].data_ptr()), nn.value, p(t["st"].data_ptr()),
                                               p(t["first"].data_ptr()), p(t["ent"].data_ptr()),
                                               p(t["ar"].data_ptr()), *cfg, p(d_out), cap, C.byref(need),
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
        ctr = np.zeros(3, np.uint64)
        capi._check(L.lc_split_json_parse_sls(eng._h, js._h, capi._p(h_src), cut, 10, *cfg, capi._p(h_out), est,
                                              C.byref(need), C.byref(nev), capi._p(ctr)))
        sizes["wire"], sizes["n"] = int(need.value), int(nev.value)

    def host_lz4():
        need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        capi._check(L.lc_split_json_parse_sls_lz4(eng._h, js._h, capi._p(h_src), cut, 10, *cfg, None, 0,
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
        groups = {"json_walk": 0.0, "resolve": 0.0, "size_emit": 0.0, "lz4": 0.0, "other": 0.0}
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None)
            us = ev.cuda_time_total if us is None else us
            k = ev.key
            # the JSON, resolve and size / emit kernels ran `runs` times over the same lines: their mean per run;
            # the LZ4 kernels ran once, in the fused call
            g = ("lz4" if "lz4_" in k else "resolve" if "json_resolve" in k else "size_emit"
                 if "split_json_sls" in k else "json_walk" if "json_" in k else "other")
            groups[g] += us / 1e3 / (1 if g == "lz4" else runs)
        return {k: round(v, 3) for k, v in groups.items()}

    need = C.c_uint64(0)

    def big_runs():
        step(big, big["out"].data_ptr(), big["wire"], need)
        eng.split_json_parse_sls_lz4(js, src, 10, b"content", offset_key=OKEY, src_pos=4096, time=1700000000)
    k_big = kernel_ms(big_runs, 2)
    k_small = kernel_ms(lambda: step(small, small["out"].data_ptr(), small["wire"], need), 1)

    # ---- the host class through the JSON host API, 512 KB groups of one source event with offset metadata
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": cut,
                         "contents": {"content": chunk_val.decode("latin-1")}}]}
    jres = {}
    for mode, mname in ((0, "json_serialize_sls"), (1, "json_process_process_serialize")):
        sp = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
        jp = lc.HostProcessor("processor_parse_json_native", {"SourceKey": "content"})
        capi.host_chain_serialize_sls(sp, jp, group, False, mode)
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for _g in range(a.json_groups):
                out = capi.host_chain_serialize_sls(sp, jp, group, False, mode)
            ts.append((time.perf_counter() - t0) * 1e3 / a.json_groups)
        jres[mname] = (float(np.median(ts)), out[0])
    assert jres["json_serialize_sls"][1] == jres["json_process_process_serialize"][1]

    name, pl = card()
    print(json.dumps({
        "metric": "split_json_sls", "gpu": name, "power_limit_w": pl,
        "lines": big["n"], "bytes": big["n_src"], "wire_bytes": big["wire"],
        "dev_chain_ms_median": round(t_big, 3),
        "chunk_bytes": small["n_src"], "chunk_lines": small["n"], "chunk_dev_chain_ms_median": round(t_small, 3),
        "dev_steps": a.steps,
        "kernel_ms_per_step": k_big, "chunk_kernel_ms_per_step": k_small,
        "chunks": a.chunks, "host_split_json_sls_ms_median": round(res["host_sls"], 2),
        "host_split_json_sls_lz4_ms_median": round(res["host_lz4"], 2), "host_reps": a.host_reps,
        "chunk_wire_bytes": sizes["wire"], "chunk_lz4_bytes": sizes["blk"],
        "json_serialize_sls_ms_per_group": round(jres["json_serialize_sls"][0], 2),
        "json_process_process_serialize_ms_per_group": round(jres["json_process_process_serialize"][0], 2),
    }))
    eng.close()


if __name__ == "__main__":
    main()
