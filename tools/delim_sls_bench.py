"""Delimiter -> SLS wire format on C4's data (synth.csv_lines: 8 Mi lines, max_fields 11, ten keys, extend).

Reports, in one JSON line with the card's name and power limit:
  * the device-resident step lc_delim_parse_dev + lc_sls_serialize_delim_dev (CUDA events, median over --steps after
    --warmup);
  * the host-buffer call lc_delim_parse_sls (wire bytes back) against lc_delim_parse (its tables back), both with
    pinned host buffers (host clock around calls that end in a synchronise, median over --host-reps);
  * the H2D and D2H bytes of each, computed from shapes.
Needs a CUDA device; there is no CPU path."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, pl = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), None


def pinned(lib, nbytes, dtype, keep):
    p = lib.lc_host_alloc(max(int(nbytes), 16))
    if not p:
        raise MemoryError("lc_host_alloc(%d)" % nbytes)
    keep.append(p)
    buf = (C.c_uint8 * max(int(nbytes), 16)).from_address(p)
    return np.frombuffer(buf, np.uint8)[:int(nbytes)].view(dtype)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=8 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    buf, off, ln = synth.csv_lines(a.lines, seed=a.seed)
    n, MF, base_len = int(off.size), 11, int(buf.size)
    keys = [k.encode() for k in synth.CSV_KEYS]
    sep, quote, src = b",", ord('"'), b"content"
    times = (1700000000 + np.arange(n) % 86400).astype(np.uint32)
    cfg = dict(sep=sep, quote=quote, treatment="extend", keys=keys, source_key=src)

    # ---- device-resident step
    i32 = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()  # noqa: E731
    d_buf = torch.from_numpy(np.concatenate([buf, np.zeros(16, np.uint8)])).cuda()
    d_off, d_len, d_t = i32(off), i32(ln), i32(times)
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_nf = torch.empty(n, dtype=torch.int32, device="cuda")
    d_fo, d_fl, d_fd = (torch.empty(n * MF, dtype=torch.int32, device="cuda") for _ in range(3))
    tab = (d_st.data_ptr(), d_nf.data_ptr(), d_fo.data_ptr(), d_fl.data_ptr(), d_fd.data_ptr())

    def parse():
        eng.delim_parse_dev(d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n, sep, quote, len(keys),
                            True, True, MF, *tab)

    def ser(d_out=None, cap=0):
        return eng.sls_serialize_delim_dev(d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n, *tab, MF,
                                           sep, quote, "extend", keys, src, d_ev_time=d_t.data_ptr(), d_out=d_out,
                                           out_cap=cap)
    parse()
    wire = ser()
    d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.ExternalStream(eng.stream)
    dev_ms = []
    for k in range(a.warmup + a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        parse()
        got = ser(d_out.data_ptr(), wire)
        e1.record(stream)
        e1.synchronize()
        assert got == wire
        if k >= a.warmup:
            dev_ms.append(e0.elapsed_time(e1))

    # ---- host buffers (pinned): wire bytes back vs tables back
    keep = []
    h_buf = pinned(L, base_len, np.uint8, keep)
    h_buf[:] = buf
    h_off, h_len, h_t = (pinned(L, 4 * n, np.uint32, keep) for _ in range(3))
    h_off[:], h_len[:], h_t[:] = off, ln, times
    h_wire = pinned(L, wire + 16, np.uint8, keep)
    h_st = pinned(L, n, np.uint8, keep)
    h_nf = pinned(L, 4 * n, np.uint32, keep)
    h_fo, h_fl, h_fd = (pinned(L, 4 * n * MF, np.uint32, keep) for _ in range(3))
    _kk, kargs = capi.Engine._delim_sls_cfg(keys, src, None, False, False, False)
    sp = np.frombuffer(sep, np.uint8)
    p = capi._p

    def host_sls():
        need = C.c_uint64(0)
        ctr = np.zeros(4, np.uint64)
        capi._check(L.lc_delim_parse_sls(eng._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(h_t), None, p(sp), 1,
                                         quote, 1, 0, 1, MF, *kargs, p(h_wire), wire + 16, C.byref(need), p(ctr)))
        assert need.value == wire

    def host_tables():
        capi._check(L.lc_delim_parse(eng._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(sp), 1, quote, len(keys), 1,
                                     1, MF, p(h_st), p(h_nf), p(h_fo), p(h_fl), p(h_fd)))

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

    name, pl = card()
    dev = float(np.median(dev_ms))
    print(json.dumps({
        "metric": "delim_sls_c4", "gpu": name, "power_limit_w": pl, "lines": n, "arena_bytes": base_len,
        "max_fields": MF, "wire_bytes": wire,
        "dev_step_ms_median": round(dev, 3), "dev_step_gb_per_s": round(base_len / dev / 1e6, 1),
        "dev_steps": a.steps, "host_sls_ms_median": round(res["host_sls"], 2),
        "host_tables_ms_median": round(res["host_tables"], 2), "host_reps": a.host_reps,
        "h2d_bytes": {"delim_parse_sls": base_len + 12 * n, "delim_parse": base_len + 8 * n},
        "d2h_bytes": {"delim_parse_sls": wire, "delim_parse": n * 5 + 3 * n * MF * 4},
    }))
    eng.close()


if __name__ == "__main__":
    main()
