"""ProcessorParseTimestampNative on the GPU (lc_timestamp_parse_dev, lc_timestamp_parse_capture_dev,
lc_timestamp_parse): events per second.

Reports, in one JSON line with the card's name and power limit (read in the same call):
  * C2's nginx time column, `%d/%b/%Y:%H:%M:%S`, read in place from the regex stage's capture tables
    (lc_timestamp_parse_capture_dev over one lc_regex_parse_dev result), device-resident;
  * `%Y-%m-%d %H:%M:%S.%f` with 1, 10, 100 and 1000 events per second, device-resident and through the host-buffer call;
  * the cache's worst case: `%Y-%m-%d %H:%M:%S`, no %f, every event a new second;
  each over --events events in groups of --group events (a 512 KB chunk of 256-byte lines is 2 048), CUDA events
  around --steps calls after --warmup; the host-buffer call with a host clock around calls that end in a synchronise;
  * the CPU oracle (oracle/lc_timestamp_oracle.c, sequential per group) on all cores, one process per core.
Every device result is checked against the oracle first.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import multiprocessing as mp
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.delim_sls_bench import card  # noqa: E402


def dated_values(fmt, n, per_sec, seed):
    """n values of fmt (`...%S` or `...%S.%f` with 3 fraction digits), per_sec events in each second"""
    rng = random.Random(seed)
    head = fmt.replace(".%f", "")
    t0, out, sec = 1699990000, [], b""
    for k in range(n):
        if k % per_sec == 0:
            sec = time.strftime(head, time.gmtime(t0 + k // per_sec)).encode()
        out.append(sec + (b".%03d" % rng.randrange(1000) if head != fmt else b""))
    return out


def _oracle_chunk(args):
    from oracle import timestamp as ots
    fmt, base, off, ln, grp, now = args
    t = time.perf_counter()
    ots.process(fmt, -1, 0, base, off, ln, grp, now, 43200, "c")
    return time.perf_counter() - t


def oracle_rate(fmt, base, off, ln, grp, now):
    """events/s of the C oracle with the groups spread over all cores (wall clock of the pool); each process gets only
    the bytes of its own groups"""
    cores = os.cpu_count() or 1
    ng = grp.size - 1
    parts = []
    for c in range(cores):
        g0, g1 = ng * c // cores, ng * (c + 1) // cores
        if g1 > g0:
            e0, e1 = int(grp[g0]), int(grp[g1])
            o, ln_ = off[e0:e1].astype(np.int64), ln[e0:e1]
            have = ln_ != 0xFFFFFFFF
            b0 = int(o[have].min()) if have.any() else 0
            b1 = int((o[have] + ln_[have]).max()) if have.any() else 0
            parts.append((fmt, base[b0:b1].copy(), np.where(have, o - b0, 0).astype(np.uint32), ln_.copy(),
                          (grp[g0:g1 + 1] - grp[g0]).astype(np.uint32), now))
    # spawned, not forked: the parent holds a CUDA context and the runtime's threads
    with mp.get_context("spawn").Pool(len(parts)) as pool:
        pool.map(_oracle_chunk, parts[:1])
        t = time.perf_counter()
        pool.map(_oracle_chunk, parts)
        dt = time.perf_counter() - t
    return off.size / dt, cores


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--events", type=int, default=1 << 20)
    ap.add_argument("--group", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=5)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    from oracle import timestamp as ots
    from tests.emul import timestamp as ets
    assert torch.cuda.is_available(), "needs a CUDA device"
    eng = lc.Engine(0)
    now = 1700000000
    n = a.events
    grp = np.arange(0, n + a.group, a.group, dtype=np.int64)
    grp[-1] = n
    grp = np.unique(np.minimum(grp, n)).astype(np.uint32)
    ng = grp.size - 1
    d_grp = torch.from_numpy(grp.view(np.int32)).cuda()
    d_sec = torch.empty(n, dtype=torch.int64, device="cuda")
    d_ns = torch.empty(n, dtype=torch.int32, device="cuda")
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_cnt = torch.empty(5, dtype=torch.int64, device="cuda")

    def timed(call):
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
        return n * a.steps / (e0.elapsed_time(e1) / 1e3)

    def check(want):
        eng.sync()
        got = (d_st.cpu().numpy(), d_sec.cpu().numpy(), d_ns.cpu().numpy().view(np.uint32),
               d_cnt.cpu().numpy().astype(np.uint64))
        assert all(np.array_equal(x, y) for x, y in zip(got, want)), "device result differs from the oracle"

    res = {}
    # C2's time column, from the regex stage's captures
    buf, off, ln = synth.nginx_lines(n, seed=1)
    rx = lc.Regex(synth.NGINX_PATTERN)
    G, k = rx.ngroups, synth.NGINX_KEYS.index("time")
    d_buf = torch.from_numpy(buf.copy()).cuda()
    d_off = torch.from_numpy(off.astype(np.uint32).view(np.int32)).cuda()
    d_len = torch.from_numpy(ln.astype(np.uint32).view(np.int32)).cuda()
    rs = torch.empty(n, dtype=torch.uint8, device="cuda")
    co = torch.empty(n * G, dtype=torch.int32, device="cuda")
    cl = torch.empty(n * G, dtype=torch.int32, device="cuda")
    eng.regex_parse_dev(rx, d_buf.data_ptr(), buf.size, d_off.data_ptr(), d_len.data_ptr(), n, G, rs.data_ptr(),
                        co.data_ptr(), cl.data_ptr())
    eng.sync()
    fmt = "%d/%b/%Y:%H:%M:%S"
    ts = lc.Timestamp(fmt)
    cap = lambda: eng.timestamp_parse_capture_dev(  # noqa: E731
        ts, d_buf.data_ptr(), buf.size, rs.data_ptr(), co.data_ptr(), cl.data_ptr(), G, k, n, d_grp.data_ptr(), ng,
        now, 43200, d_sec.data_ptr(), d_ns.data_ptr(), d_st.data_ptr(), d_cnt.data_ptr())
    h_rs = rs.cpu().numpy()
    v_off = np.where(h_rs == 0, co.cpu().numpy().view(np.uint32).reshape(n, G)[:, k], 0).astype(np.uint32)
    v_len = np.where(h_rs == 0, cl.cpu().numpy().view(np.uint32).reshape(n, G)[:, k], ets.NO_KEY).astype(np.uint32)
    cap()
    check(ots.process(fmt, -1, 0, buf, v_off, v_len, grp, now, 43200, "c"))
    ok_frac = float((d_st.cpu().numpy() == 0).mean())
    res["c2_nginx_capture_dev"] = {"events_per_s": timed(cap), "ok_fraction": ok_frac,
                                   "oracle_all_cores_events_per_s": oracle_rate(fmt, buf, v_off, v_len, grp, now)[0]}
    print("c2_nginx_capture_dev", res["c2_nginx_capture_dev"], file=sys.stderr, flush=True)

    shapes = [("%Y-%m-%d %H:%M:%S.%f", p) for p in (1, 10, 100, 1000)] + [("%Y-%m-%d %H:%M:%S", 1)]
    for fmt, per_sec in shapes:
        vals = dated_values(fmt, n, per_sec, seed=per_sec)
        base, off, ln, _ = ets.layout([vals])
        d_base = torch.from_numpy(base.copy()).cuda()
        d_o = torch.from_numpy(off.view(np.int32)).cuda()
        d_l = torch.from_numpy(ln.view(np.int32)).cuda()
        ts = lc.Timestamp(fmt)
        dev = lambda: eng.timestamp_parse_dev(  # noqa: E731
            ts, d_base.data_ptr(), base.size, d_o.data_ptr(), d_l.data_ptr(), n, d_grp.data_ptr(), ng, now, 43200,
            d_sec.data_ptr(), d_ns.data_ptr(), d_st.data_ptr(), d_cnt.data_ptr())
        want = ots.process(fmt, -1, 0, base, off, ln, grp, now, 43200, "c")
        dev()
        check(want)
        r_dev = timed(dev)
        got = eng.timestamp_parse(ts, base, off, ln, grp, now)
        assert all(np.array_equal(x, y) for x, y in zip(got, want)), "host call differs from the oracle"
        t = time.perf_counter()
        for _ in range(a.host_reps):
            eng.timestamp_parse(ts, base, off, ln, grp, now)
        r_host = n * a.host_reps / (time.perf_counter() - t)
        orc, cores = oracle_rate(fmt, base, off, ln, grp, now)
        res["%s x%d/s" % (fmt, per_sec)] = {"dev_events_per_s": r_dev, "host_call_events_per_s": r_host,
                                             "oracle_all_cores_events_per_s": orc}
        print(fmt, per_sec, res["%s x%d/s" % (fmt, per_sec)], file=sys.stderr, flush=True)
    name, pl = card()
    print(json.dumps({"bench": "timestamp_parse", "gpu": name, "power_limit_w": pl, "events": n, "group": a.group,
                      "cpu_cores": os.cpu_count(), "results": res}))
    eng.close()


if __name__ == "__main__":
    main()
