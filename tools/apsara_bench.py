"""ProcessorParseApsaraNative on the GPU (lc_apsara_parse_dev, lc_apsara_parse): bytes and lines per second.

Reports, in one JSON line with the card's name and power limit (read in the same call), over synth.apsara_lines
(--lines lines, 80 B - 2 KB, groups of --group lines):
  * device-resident: CUDA events on the engine's stream around --steps lc_apsara_parse_dev calls after --warmup (each
    call waits once midway for its entry count and again at its end, so the call time includes those two round trips);
  * kernel time: the device time of the call's four kernels (scan, resolve, exclusive sum, emit) summed per call,
    from torch.profiler in a run of its own after the timed window;
  * algorithmic bytes over that kernel time as a fraction of 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth).
    Algorithmic bytes: the value bytes read twice (the scan pass and the emit pass), the event table (8 B per line)
    and the outputs (status 1 + sec 8 + nsec 4 + micro 8 + first 8 B per line, 16 B per entry);
  * the host-buffer call end to end (a host clock around calls that end in a synchronise);
  * the C oracle (oracle/lc_apsara_oracle.c, sequential per group) on all cores, one process per core.
The device result is checked against the oracle first.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import multiprocessing as mp
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.delim_sls_bench import card  # noqa: E402

HBM = 3.35e12
NOW = 1700000000 + 43200


KERNELS = ("ap_scan_kernel", "ap_resolve_kernel", "exclusive_sum_kernel", "ap_emit_kernel")


def _oracle_chunk(args):
    from oracle import apsara as oap
    buf, off, ln, grp = args
    t = time.perf_counter()
    oap.process("content", 0, buf, off, ln, grp, NOW, -1)
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=1 << 20)
    ap.add_argument("--group", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    from oracle import apsara as oap
    buf, off, ln, grp = synth.apsara_lines(a.lines, seed=1, groups_of=a.group)
    n = off.size
    eng = lc.Engine(0)
    h = lc.Apsara("content", 0)
    want = oap.process("content", 0, buf, off, ln, grp, NOW, -1)
    got = eng.apsara_parse(h, buf, off, ln, grp, NOW, -1)
    for x, y in zip(got, want):
        assert np.array_equal(x, y), "device result differs from the oracle"
    m = int(want[4][-1])
    dev = lambda x: torch.from_numpy(np.array(x)).cuda()  # noqa: E731
    d_buf, d_off, d_len, d_grp = dev(buf), dev(off.view(np.int32)), dev(ln.view(np.int32)), dev(grp.view(np.int32))
    out = [torch.empty(k, dtype=torch.uint8, device="cuda") for k in (n, 8 * n, 4 * n, 8 * n, 8 * (n + 1),
                                                                       16 * max(m, 1), 40)]

    def call():
        return eng.apsara_parse_dev(h, d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n,
                                    d_grp.data_ptr(), grp.size - 1, NOW, -1, *[t.data_ptr() for t in out[:6]], m,
                                    out[6].data_ptr())
    for _ in range(a.warmup):
        call()
    eng.sync()
    s = torch.cuda.ExternalStream(eng.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(a.steps):
        call()
    e1.record(s)
    e1.synchronize()
    dt = e0.elapsed_time(e1) / 1e3 / a.steps
    from torch.profiler import ProfilerActivity, profile
    prof_calls = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(prof_calls):
            call()
        eng.sync()
    kus = sum(ev.device_time_total for ev in prof.key_averages() if any(k in ev.key for k in KERNELS))
    kdt = kus / 1e6 / prof_calls if kus else None  # None: the profiler saw no kernel, "not measured"
    alg = 2 * buf.size + 8 * n + 29 * n + 16 * m
    t = time.perf_counter()
    for _ in range(max(1, a.steps // 4)):
        eng.apsara_parse(h, buf, off, ln, grp, NOW, -1, entry_cap=m)
    host_dt = (time.perf_counter() - t) / max(1, a.steps // 4)
    ncpu = os.cpu_count() or 1
    cuts = np.linspace(0, grp.size - 1, ncpu + 1).astype(int)
    chunks = []
    for i in range(ncpu):  # whole groups per core; each task carries only its own bytes
        g0, g1 = int(grp[cuts[i]]), int(grp[cuts[i + 1]])
        if g1 > g0:
            b0, b1 = int(off[g0]), int(off[g1 - 1]) + int(ln[g1 - 1])
            chunks.append((buf[b0:b1].copy(), (off[g0:g1] - b0).astype(np.uint32), ln[g0:g1].copy(),
                           (grp[cuts[i]:cuts[i + 1] + 1] - g0).astype(np.uint32)))
    t = time.perf_counter()
    with mp.Pool(len(chunks)) as pool:
        pool.map(_oracle_chunk, chunks)
    cpu_dt = time.perf_counter() - t
    name, plimit = card()
    print(json.dumps({"bench": "apsara", "card": name, "power_limit": plimit, "lines": n, "bytes": int(buf.size),
                      "entries": m, "device_call_s": dt, "device_call_GBps": buf.size / dt / 1e9,
                      "device_call_lines_per_s": n / dt, "kernel_s": kdt,
                      "kernel_GBps": buf.size / kdt / 1e9 if kdt else None, "alg_bytes": alg,
                      "alg_fraction_of_3.35TBps": alg / kdt / HBM if kdt else None,
                      "host_call_s": host_dt, "host_call_GBps": buf.size / host_dt / 1e9,
                      "cpu_oracle_cores": ncpu, "cpu_oracle_s": cpu_dt, "cpu_oracle_GBps": buf.size / cpu_dt / 1e9}))
    eng.close()


if __name__ == "__main__":
    main()
