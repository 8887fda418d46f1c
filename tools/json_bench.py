"""ProcessorParseJsonNative on the GPU (lc_json_parse_dev, lc_json_parse): bytes and lines per second.

Reports, in one JSON line with the card's name and power limit (read in the same call), over synth.json_lines
(--lines lines of 150 B - 4 KB, 8-40 members each):
  * device-resident: CUDA events on the engine's stream around --steps lc_json_parse_dev calls after --warmup (each
    call waits once for its totals and again at its end, so the call time includes those two round trips);
  * kernel time: the device time of the call's kernels (fast and slow count, two exclusive sums, fast and slow emit)
    per call and per kernel, from torch.profiler in a run of its own after the timed window;
  * algorithmic bytes over that kernel time as a fraction of 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth).
    Algorithmic bytes: the value bytes read twice (the count pass and the emit pass), the event table (8 B per line),
    the per-line outputs (status 1 + first 8 B) and the outputs (16 B per entry, the arena bytes);
  * the host-buffer call end to end (a host clock around calls that end in a synchronise);
  * the C oracle (oracle/lc_json_oracle.c) on all cores, one process per core;
  * the number of events the fast walk handed to the slow one.
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
KERNELS = ("json_count_kernel", "json_count_slow_kernel", "exclusive_sum_kernel", "json_emit_kernel",
           "json_emit_slow_kernel")


def _oracle_chunk(args):
    from oracle import json_parse as oj
    buf, off, ln = args
    t = time.perf_counter()
    oj.process("content", buf, off, ln)
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
    from oracle import json_parse as oj
    from tests.emul import json_parse as ej
    buf, off, ln, _ = synth.json_lines(a.lines, seed=1, groups_of=a.group)
    n = off.size
    eng = lc.Engine(0)
    h = lc.Json("content")
    # one call takes under 2 GiB of values (the arena tag bit), so the lines go in as few calls as that allows,
    # cut at line boundaries as the host class cuts its batches
    ends = (off.astype(np.int64) + ln).tolist()
    parts, l0 = [], 0
    while l0 < n:
        b0 = int(off[l0])
        l1 = int(np.searchsorted(np.asarray(ends), b0 + (1 << 31) - 1, side="right"))
        b1 = ends[l1 - 1]
        parts.append((buf[b0:b1], (off[l0:l1] - b0).astype(np.uint32), ln[l0:l1].copy()))
        l0 = l1
    m = ab = n_slow = 0
    dev = lambda x: torch.from_numpy(np.array(x)).cuda()  # noqa: E731
    calls = []
    for pb, po, pl in parts:
        want = oj.process("content", pb, po, pl)
        got = eng.json_parse(h, pb, po, pl)
        for x, y in zip(got, want):
            assert np.array_equal(np.asarray(x), np.asarray(y)), "device result differs from the oracle"
        n_slow += ej.parse("content", pb, po, pl)[5]
        pm, pa, pn = int(want[1][-1]), len(want[3]), po.size
        m, ab = m + pm, ab + pa
        ins = [dev(pb), dev(po.view(np.int32)), dev(pl.view(np.int32))]
        out = [torch.empty(k, dtype=torch.uint8, device="cuda") for k in (pn, 8 * (pn + 1), 16 * max(pm, 1),
                                                                           max(pa, 1), 24)]
        calls.append((pb.size, pn, pm, pa, ins, out))
        del want, got

    def call():
        for nb, pn, pm, pa, ins, out in calls:
            eng.json_parse_dev(h, ins[0].data_ptr(), nb, ins[1].data_ptr(), ins[2].data_ptr(), pn, out[0].data_ptr(),
                               out[1].data_ptr(), out[2].data_ptr(), pm, out[3].data_ptr(), pa, out[4].data_ptr())
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
    per = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                per[k] = per.get(k, 0) + ev.device_time_total / 1e6 / prof_calls
    kdt = sum(per.values()) or None  # None: the profiler saw no kernel, "not measured"
    alg = 2 * buf.size + 8 * n + 9 * n + 16 * m + ab
    t = time.perf_counter()
    for _ in range(max(1, a.steps // 4)):
        for (pb, po, pl), c in zip(parts, calls):
            eng.json_parse(h, pb, po, pl, entry_cap=c[2], arena_cap=c[3])
    host_dt = (time.perf_counter() - t) / max(1, a.steps // 4)
    ncpu = os.cpu_count() or 1
    cuts = np.linspace(0, n, ncpu + 1).astype(int)
    chunks = []
    for i in range(ncpu):  # each task carries only its own bytes
        l0, l1 = int(cuts[i]), int(cuts[i + 1])
        if l1 > l0:
            b0, b1 = int(off[l0]), int(off[l1 - 1]) + int(ln[l1 - 1])
            chunks.append((buf[b0:b1].copy(), (off[l0:l1] - b0).astype(np.uint32), ln[l0:l1].copy()))
    t = time.perf_counter()
    with mp.Pool(len(chunks)) as pool:
        pool.map(_oracle_chunk, chunks)
    cpu_dt = time.perf_counter() - t
    name, plimit = card()
    print(json.dumps({"bench": "json", "card": name, "power_limit": plimit, "lines": n, "bytes": int(buf.size),
                      "calls_per_pass": len(parts),
                      "entries": m, "arena_bytes": ab, "slow_events": n_slow, "device_call_s": dt,
                      "device_call_GBps": buf.size / dt / 1e9, "device_call_lines_per_s": n / dt,
                      "kernel_s": kdt, "kernel_s_per_kernel": per,
                      "kernel_GBps": buf.size / kdt / 1e9 if kdt else None, "alg_bytes": alg,
                      "alg_fraction_of_3.35TBps": alg / kdt / HBM if kdt else None,
                      "host_call_s": host_dt, "host_call_GBps": buf.size / host_dt / 1e9,
                      "cpu_oracle_cores": ncpu, "cpu_oracle_s": cpu_dt, "cpu_oracle_GBps": buf.size / cpu_dt / 1e9}))
    eng.close()


if __name__ == "__main__":
    main()
