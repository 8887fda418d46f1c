"""Regex -> SLS wire format on C2's data (synth.nginx_lines: 4 Mi lines of 256 B, ten keys, 1 % that do not match).

Reports, in one JSON line with the card's name and power limit:
  * the device-resident step lc_regex_parse_dev + lc_sls_serialize_regex_dev (CUDA events, median over --steps after
    --warmup);
  * the host-buffer call lc_regex_parse_sls (wire bytes back) against lc_regex_parse (its tables back), both with
    pinned host buffers (host clock around calls that end in a synchronise, median over --host-reps);
  * the H2D and D2H bytes of each, computed from shapes (the wire count is the measured one);
  * ProcessorParseRegexNative::SerializeSls against Process + SLSEventGroupSerializer::Serialize over --groups groups
    of 512 KB (wall time per group, median; both include the JSON parse of the group by the host layer's entry point).
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=4 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--groups", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    buf, off, ln = synth.nginx_lines(a.lines, seed=a.seed)
    n, base_len = int(off.size), int(buf.size)
    keys = [k.encode() for k in synth.NGINX_KEYS]
    K = len(keys)
    rx = lc.Regex(synth.NGINX_PATTERN)
    G = rx.ngroups
    src = b"content"
    times = (1700000000 + np.arange(n) % 86400).astype(np.uint32)

    # ---- device-resident step
    i32 = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()  # noqa: E731
    d_buf = torch.from_numpy(np.concatenate([buf, np.zeros(16, np.uint8)])).cuda()
    d_off, d_len, d_t = i32(off), i32(ln), i32(times)
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_co, d_cl = (torch.empty(n * G, dtype=torch.int32, device="cuda") for _ in range(2))

    def parse():
        eng.regex_parse_dev(rx, d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n, K,
                            d_st.data_ptr(), d_co.data_ptr(), d_cl.data_ptr())

    def ser(d_out=None, cap=0):
        return eng.sls_serialize_regex_dev(d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n,
                                           d_st.data_ptr(), d_co.data_ptr(), d_cl.data_ptr(), G, keys, src,
                                           d_ev_time=d_t.data_ptr(), d_out=d_out, out_cap=cap)
    parse()
    wire, ctr = ser()
    d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.ExternalStream(eng.stream)
    dev_ms = []
    for k in range(a.warmup + a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        parse()
        got, _ = ser(d_out.data_ptr(), wire)
        e1.record(stream)
        e1.synchronize()
        assert got == wire
        if k >= a.warmup:
            dev_ms.append(e0.elapsed_time(e1))
    parsed = int(ctr[0])

    # ---- host buffers (pinned): wire bytes back vs tables back
    keep = []
    h_buf = pinned(L, base_len, np.uint8, keep)
    h_buf[:] = buf
    h_off, h_len, h_t = (pinned(L, 4 * n, np.uint32, keep) for _ in range(3))
    h_off[:], h_len[:], h_t[:] = off, ln, times
    h_wire = pinned(L, wire + 16, np.uint8, keep)
    h_st = pinned(L, n, np.uint8, keep)
    h_co, h_cl = (pinned(L, 4 * n * G, np.uint32, keep) for _ in range(2))
    _kk, kargs = capi.Engine._delim_sls_cfg(keys, src, None, False, False, False)
    p = capi._p

    def host_sls():
        need = C.c_uint64(0)
        c = np.zeros(3, np.uint64)
        capi._check(L.lc_regex_parse_sls(eng._h, rx._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(h_t), None,
                                         *kargs, 0, p(h_wire), wire + 16, C.byref(need), p(c)))
        assert need.value == wire

    def host_tables():
        capi._check(L.lc_regex_parse(eng._h, rx._h, p(h_buf), base_len, p(h_off), p(h_len), n, K, p(h_st), p(h_co),
                                     p(h_cl)))

    res = {}
    for name, fn in (("host_sls", host_sls), ("host_tables", host_tables)):
        fn()
        ts = []
        for _ in range(a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[name] = float(np.median(ts))
    assert bytes(h_wire[:wire]) == bytes(d_out[:wire].cpu().numpy())
    for ptr in keep:
        L.lc_host_free(ptr)

    # ---- host class over 512 KB groups: SerializeSls vs Process + Serialize
    per = (512 << 10) // 256
    cfg = {"SourceKey": "content", "Regex": synth.NGINX_PATTERN, "Keys": synth.NGINX_KEYS}
    fast, slow = lc.HostProcessor("processor_parse_regex_native", cfg), lc.HostProcessor("processor_parse_regex_native",
                                                                                         cfg)
    group_ms = {"serialize_sls": [], "process_then_serialize": []}
    for g in range(a.groups + 1):
        lo = (g * per) % max(n - per, 1)
        evs = [{"type": 1, "timestamp": int(times[i]), "contents": {"content": bytes(buf[off[i]:off[i] + ln[i]]).decode()}}
               for i in range(lo, lo + per)]
        root = {"events": evs, "tags": {"__topic__": "t"}}
        outs = []
        for name, kw in (("serialize_sls", {}), ("process_then_serialize", {"process_then_serialize": True})):
            proc = fast if not kw else slow
            t0 = time.perf_counter()
            outs.append(proc.serialize_sls(root, False, **kw))
            if g:  # the first group warms both paths up
                group_ms[name].append((time.perf_counter() - t0) * 1e3)
        assert outs[0] == outs[1]

    name, pl = card()
    dev = float(np.median(dev_ms))
    cap_bytes = n + 2 * n * G * 4
    print(json.dumps({
        "metric": "regex_sls_c2", "gpu": name, "power_limit_w": pl, "lines": n, "arena_bytes": base_len, "groups": G,
        "keys": K, "parsed_events": parsed, "wire_bytes": wire,
        "dev_step_ms_median": round(dev, 3), "dev_step_gb_per_s": round(base_len / dev / 1e6, 1),
        "dev_steps": a.steps, "host_sls_ms_median": round(res["host_sls"], 2),
        "host_tables_ms_median": round(res["host_tables"], 2), "host_reps": a.host_reps,
        "h2d_bytes": {"regex_parse_sls": base_len + 12 * n, "regex_parse": base_len + 8 * n},
        "d2h_bytes": {"regex_parse_sls": wire, "regex_parse": cap_bytes},
        "group_512k_ms_median": {k: round(float(np.median(v)), 2) for k, v in group_ms.items()},
        "group_count": a.groups,
    }))
    eng.close()


if __name__ == "__main__":
    main()
