"""Split -> delimiter -> timestamp -> SLS wire format on synth.csv_lines with a time column in front, tkey = time.

The CSV file pipeline whose logs take their time from a column: the splitter, processor_parse_delimiter_native (keys
time + synth.CSV_KEYS), processor_parse_timestamp_native on `time`, then the SLS flusher.  Two time forms: a plain
"%Y-%m-%d %H:%M:%S" column ("ymd"), and "%b %d, %Y %H:%M:%S" quoted around its comma and ending in a doubled
quote, which the tap collapses and the format's trailing literal quote matches ("quoted").  One JSON line, with the
card's name and power limit read in the same run:
  * device-resident steps (CUDA events, median over --steps after --warmup, the arms alternated), at one 512 KB reader
    chunk and at --lines lines: "plain" = lc_split_lines_dev + lc_delim_parse_dev + lc_sls_serialize_split_delim_dev
    (each record stamped with the source event's time, the split -> delimiter chain without the timestamp stage),
    against "ts" = the same with lc_split_delim_timestamp_tap_dev + lc_timestamp_parse_dev (one group, discard_interval
    -1) + lc_sls_serialize_split_delim_timestamp_dev;
  * algorithmic bytes of a "ts" step (the chunk read once plus the wire bytes written) and their fraction of the
    H100's 3.35 TB/s;
  * the kernel split of one "ts" step: split, delimiter, the tap, ts_full, ts_resolve and the size / emit passes
    (torch.profiler with CUDA activities, in a run of its own after the timed ones);
  * the host-buffer calls over --chunks chunks of 512 KB (host clock around calls that end in a synchronise, median
    of the per-chunk time): lc_split_delim_parse_sls against lc_split_delim_timestamp_parse_sls and its _lz4 variant;
  * the CPU oracle's rate (oracle splitter + ProcessorParseDelimiterNative + timestamp step + serialiser) on
    --oracle-lines lines.
The cache pass (ts_resolve_kernel) walks the one group serially in one warp, so the chain is meant for reader-sized
chunks.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.delim_sls_bench import card  # noqa: E402

OKEY = b"__file_offset__"
YMD = "%Y-%m-%d %H:%M:%S"
QFMT = '%b %d, %Y %H:%M:%S"'
CHUNK = 512 * 1024
HBM_BPS = 3.35e12
NOW = 1700000000
_MON = (b"Jan", b"Feb", b"Mar", b"Apr", b"May", b"Jun", b"Jul", b"Aug", b"Sep", b"Oct", b"Nov", b"Dec")


def with_time(buf, quoted):
    """the CSV lines with a time column in front: one second per 16 lines back from NOW (the cache hits within a
    second); quoted: "Mon DD, YYYY HH:MM:SS" plus a doubled quote the format's trailing literal matches"""
    out = []
    for k, ln in enumerate(bytes(buf).split(b"\n")):
        s = time.gmtime(NOW - 3600 + k // 16)
        if quoted:
            t = b'"%s %02d, %04d %02d:%02d:%02d"""' % (_MON[s.tm_mon - 1], s.tm_mday, s.tm_year, s.tm_hour, s.tm_min,
                                                       s.tm_sec)
        else:
            t = time.strftime(YMD, s).encode()
        out.append(t + b"," + ln)
    return b"\n".join(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=1 << 20)
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--oracle-lines", type=int, default=4000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    os.environ["TZ"] = "UTC"
    time.tzset()
    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, plimit = card()
    eng = lc.Engine(0)
    # the engine and torch queue on one stream of their own, so that the CUDA events bracket the calls that return
    # without waiting (the tap and the timestamp passes)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    keys = [b"time"] + [k.encode() for k in synth.CSV_KEYS]
    MF = len(keys) + 16
    dargs = (b",", ord('"'), "extend", keys, b"content")
    kw = dict(keep_fail=True, offset_key=OKEY)
    skw = dict(kw, src_pos=1 << 33, time=NOW)

    def device_arms(val, fmt):
        ts = lc.Timestamp(fmt)
        n_max = val.count(b"\n") + 2
        d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
        d_off = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        d_len = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        st = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        nf = torch.empty(n_max, dtype=torch.int32, device="cuda")
        fo, fl, fd = (torch.empty(n_max * MF, dtype=torch.int32, device="cuda") for _ in range(3))
        vbuf = torch.empty(len(val) + 16, dtype=torch.uint8, device="cuda")
        v_off = torch.empty(n_max, dtype=torch.int32, device="cuda")
        v_len = torch.empty(n_max, dtype=torch.int32, device="cuda")
        sec = torch.empty(n_max, dtype=torch.int64, device="cuda")
        nsec = torch.empty(n_max, dtype=torch.int32, device="cuda")
        tst = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
        grp1 = torch.empty(2, dtype=torch.int32, device="cuda")
        d_out = torch.empty(len(val) * 3 + 4096, dtype=torch.uint8, device="cuda")

        def split_delim():
            n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), len(val) + 1)
            eng.delim_parse_dev(d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, b",", ord('"'),
                                len(keys), True, True, MF, st.data_ptr(), nf.data_ptr(), fo.data_ptr(), fl.data_ptr(),
                                fd.data_ptr())
            return n, (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), nf.data_ptr(),
                       fo.data_ptr(), fl.data_ptr(), fd.data_ptr(), MF)

        def plain():
            _n, args = split_delim()
            return eng.sls_serialize_split_delim_dev(*args, *dargs, **skw, d_out=d_out.data_ptr(),
                                                     out_cap=d_out.numel())

        def with_ts():
            n, args = split_delim()
            eng.split_delim_timestamp_tap_dev(*args, *dargs, b"time", vbuf.data_ptr(), len(val), v_off.data_ptr(),
                                              v_len.data_ptr(), **kw)
            grp1.copy_(torch.tensor([0, n], dtype=torch.int32))
            eng.timestamp_parse_dev(ts, vbuf.data_ptr(), len(val), v_off.data_ptr(), v_len.data_ptr(), n,
                                    grp1.data_ptr(), 1, NOW, -1, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(),
                                    tcnt.data_ptr())
            return eng.sls_serialize_split_delim_timestamp_dev(*args, *dargs, tst.data_ptr(), sec.data_ptr(),
                                                               nsec.data_ptr(), **skw, d_out=d_out.data_ptr(),
                                                               out_cap=d_out.numel())

        arms = {"plain": plain, "ts": with_ts}
        times = {k: [] for k in arms}
        for it in range(a.warmup + a.steps):
            for k, f in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                s.record()
                f()
                e.record()
                torch.cuda.synchronize()
                if it >= a.warmup:
                    times[k].append(s.elapsed_time(e))
        out = {k + "_ms": round(statistics.median(v), 4) for k, v in times.items()}
        out["bytes"] = len(val)
        nb, c9 = with_ts()
        out["ts_counters"] = [int(x) for x in c9]
        out["wire_bytes"] = int(nb)
        alg = len(val) + int(nb)
        out["alg_bytes"] = alg
        out["ts_frac_of_3.35TBps"] = round(alg / (out["ts_ms"] * 1e-3) / HBM_BPS, 5)
        # the kernel split of one step, in a run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with_ts()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            k = ev.key
            grp = ("tap" if "split_delim_ts_tap" in k else "ts_full" if "ts_full" in k else
                   "ts_resolve" if "ts_resolve" in k else
                   "size_emit" if "split_delim_ts_sls" in k or "exclusive" in k or "scan" in k else
                   "delim" if "delim" in k else "split" if "split" in k else "other")
            t_us = getattr(ev, "device_time_total", None)
            if t_us is None:
                t_us = ev.cuda_time_total
            split[grp] = round(split.get(grp, 0.0) + t_us / 1e3, 4)
        out["kernel_ms"] = split
        return out

    res = {"card": name, "power_limit_w": plimit}
    chunk = synth.csv_lines(CHUNK // 150, seed=7)[0].tobytes()
    big = synth.csv_lines(a.lines, seed=8)[0].tobytes()
    for fmt, tag, quoted in ((YMD, "ymd", False), (QFMT, "quoted", True)):
        c = with_time(chunk, quoted)[:CHUNK]
        c = c[:c.rfind(b"\n") + 1]
        res["device_512KB_" + tag] = device_arms(c, fmt)
        res["device_lines_" + tag] = device_arms(with_time(big, quoted), fmt)
        res["device_lines_" + tag]["lines"] = a.lines
    del big

    # host-buffer calls over 512 KB chunks (ymd form)
    chunks = []
    for i in range(a.chunks):
        c = with_time(synth.csv_lines(CHUNK // 150, seed=100 + i)[0].tobytes(), False)[:CHUNK]
        chunks.append(c[:c.rfind(b"\n") + 1])
    ts = lc.Timestamp(YMD)
    cap = 3 * CHUNK + 65536
    calls = {
        "plain": lambda v: eng.split_delim_parse_sls(v, 10, *dargs, **skw, max_fields=MF, out_cap=cap),
        "ts": lambda v: eng.split_delim_timestamp_parse_sls(v, 10, *dargs, b"time", ts, NOW, -1, **skw,
                                                            max_fields=MF, out_cap=cap),
        "ts_lz4": lambda v: eng.split_delim_timestamp_parse_sls_lz4(v, 10, *dargs, b"time", ts, NOW, -1, **skw,
                                                                    max_fields=MF, tail=b"\x1a\x01t", out_cap=cap),
    }
    host = {k: [] for k in calls}
    for v in chunks[:2]:
        for f in calls.values():
            f(v)
    for v in chunks:
        for k, f in calls.items():
            t0 = time.perf_counter()
            f(v)
            host[k].append((time.perf_counter() - t0) * 1e3)
    res["host_calls_512KB_ms"] = {k: round(statistics.median(x), 4) for k, x in host.items()}

    # the CPU oracle on a slice of the same lines
    from tests import split_delim_timestamp_sls_cases as dtc
    cfg = dtc.config([k.decode() for k in keys], keep_fail=True, max_fields=MF)
    sample = with_time(synth.csv_lines(a.oracle_lines, seed=9)[0].tobytes(), False)
    t0 = time.perf_counter()
    dtc.oracle_chain(sample, {"SourceKey": "content", "SplitChar": 10}, cfg, b"time", YMD, NOW, -1, NOW, None,
                     1 << 33, OKEY, enable_ns=False)
    dt = time.perf_counter() - t0
    res["cpu_oracle"] = {"lines": a.oracle_lines, "lines_per_s": round(a.oracle_lines / dt, 1),
                         "MB_per_s": round(len(sample) / dt / 1e6, 4)}
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
