"""Split -> JSON -> timestamp -> SLS wire format on synth.json_lines (150 B - 2 KB), tkey = ts.

The JSON-lines file pipeline whose logs take their time from a member: the splitter, processor_parse_json_native,
processor_parse_timestamp_native on `ts`, then the SLS flusher.  Two value forms: synth's epoch integers with
SourceFormat %s ("epoch"), and the same lines with `ts` rewritten to a "%Y-%m-%d %H:%M:%S" string, escaped in every
fourth line so that its rendering lands in the arena ("ymd").  One JSON line, with the card's name and power limit read
in the same run:
  * device-resident steps (CUDA events, median over --steps after --warmup, the arms alternated), at one 512 KB reader
    chunk and at --lines lines: "plain" = lc_split_lines_dev + lc_json_parse_dev + lc_sls_serialize_split_json_dev
    (each record stamped with the source event's time), against "ts" = the same with lc_split_json_timestamp_tap_dev
    + lc_timestamp_parse_dev (one group, discard_interval -1) + lc_sls_serialize_split_json_timestamp_dev;
  * the kernel split of one "ts" step: the JSON passes, the resolve, the tap, ts_full, ts_resolve and the size / emit
    passes (torch.profiler with CUDA activities, in a run of its own after the timed ones);
  * the host-buffer calls over --chunks chunks of 512 KB (host clock around calls that end in a synchronise, median
    of the per-chunk time): lc_split_json_parse_sls against lc_split_json_timestamp_parse_sls and its _lz4 variant;
  * the host classes on 512 KB groups through the JSON host API (lc_host_chain3_serialize_sls): mode 0, the
    splitter's SerializeSls(group, json, timestamp), against mode 1, Process x 3 + Serialize.  The timestamp processor
    keeps its default history discard, so the times are rewritten to an hour before the real clock.
The cache pass (ts_resolve_kernel) walks the one group serially in one warp, so the chain is meant for reader-sized
chunks.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import re
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.delim_sls_bench import card  # noqa: E402

OKEY = b"__file_offset__"
YMD = "%Y-%m-%d %H:%M:%S"
CHUNK = 512 * 1024
TS = re.compile(rb'"ts":(\d+)')


def ymd_lines(buf, base=None):
    """the lines with "ts" as a "%Y-%m-%d %H:%M:%S" string (local time; base: the first line's time, one line per
    second after it, else the integer's own time), its first digit escaped in every fourth line"""
    out = []
    for k, ln in enumerate(bytes(buf).split(b"\n")):
        def sub(m, k=k):
            t = time.strftime(YMD, time.localtime(int(m.group(1)) if base is None else base + k // 16)).encode()
            if k % 4 == 0:
                t = b"\\u%04x" % t[0] + t[1:]
            return b'"ts":"' + t + b'"'
        out.append(TS.sub(sub, ln, count=1))
    return b"\n".join(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=1 << 20)
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--json-groups", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, plimit = card()
    eng = lc.Engine(0)
    # the engine and torch queue on one stream of their own, so that the CUDA events bracket the calls that return
    # without waiting (the tap and the timestamp passes)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    torch.cuda.set_stream(stream)
    js = lc.Json("content")
    now = 1700000000
    kw = dict(keep_fail=True, offset_key=OKEY)
    skw = dict(kw, src_pos=1 << 33, time=now)

    def device_arms(val, fmt):
        ts = lc.Timestamp(fmt)
        n_max = val.count(b"\n") + 2
        d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
        d_off = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        d_len = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        st = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        first = torch.empty(n_max + 1, dtype=torch.int64, device="cuda")
        cnt = torch.empty(3, dtype=torch.int64, device="cuda")
        ecap, acap = len(val) // 16 + 64, len(val) // 2 + 4096  # synth's members average about 45 B
        ent = torch.empty(ecap * 16, dtype=torch.uint8, device="cuda")
        ar = torch.empty(acap, dtype=torch.uint8, device="cuda")
        vbuf = torch.empty(len(val) + acap, dtype=torch.uint8, device="cuda")
        v_off = torch.empty(n_max, dtype=torch.int32, device="cuda")
        v_len = torch.empty(n_max, dtype=torch.int32, device="cuda")
        sec = torch.empty(n_max, dtype=torch.int64, device="cuda")
        nsec = torch.empty(n_max, dtype=torch.int32, device="cuda")
        tst = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
        grp1 = torch.empty(2, dtype=torch.int32, device="cuda")
        d_out = torch.empty(len(val) * 2 + 4096, dtype=torch.uint8, device="cuda")

        def split_json():
            n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), len(val) + 1)
            base = (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n)
            _m, ab = eng.json_parse_dev(js, *base, st.data_ptr(), first.data_ptr(), ent.data_ptr(), ecap,
                                        ar.data_ptr(), acap, cnt.data_ptr())
            return n, ab, (js,) + base + (st.data_ptr(), first.data_ptr(), ent.data_ptr(), ar.data_ptr())

        def plain():
            _n, _ab, args = split_json()
            return eng.sls_serialize_split_json_dev(*args, b"content", **skw, d_out=d_out.data_ptr(),
                                                    out_cap=d_out.numel())

        def with_ts():
            n, ab, args = split_json()
            eng.split_json_timestamp_tap_dev(*args, b"content", b"ts", vbuf.data_ptr(), len(val) + ab,
                                             v_off.data_ptr(), v_len.data_ptr(), **kw)
            grp1.copy_(torch.tensor([0, n], dtype=torch.int32))
            eng.timestamp_parse_dev(ts, vbuf.data_ptr(), len(val) + ab, v_off.data_ptr(), v_len.data_ptr(), n,
                                    grp1.data_ptr(), 1, now, -1, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(),
                                    tcnt.data_ptr())
            return eng.sls_serialize_split_json_timestamp_dev(*args, b"content", tst.data_ptr(), sec.data_ptr(),
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
        nb, c8 = with_ts()
        out["ts_counters"] = [int(x) for x in c8]
        out["wire_bytes"] = int(nb)
        # the kernel split of one step, in a run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with_ts()
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            k = ev.key
            grp = ("resolve" if "json_resolve" in k else "tap" if "split_json_ts_tap" in k else
                   "ts_full" if "ts_full" in k else "ts_resolve" if "ts_resolve" in k else
                   "size_emit" if "split_json_ts_sls" in k or "exclusive" in k or "scan" in k else
                   "json" if "json_" in k else "split" if "split" in k else "other")
            t_us = getattr(ev, "device_time_total", None)
            if t_us is None:
                t_us = ev.cuda_time_total
            split[grp] = round(split.get(grp, 0.0) + t_us / 1e3, 4)
        out["kernel_ms"] = split
        return out

    res = {"card": name, "power_limit_w": plimit}
    chunk, _, _, _ = synth.json_lines(CHUNK // 600, seed=7, hi=2048)
    chunk = chunk.tobytes()[:CHUNK]
    chunk = chunk[:chunk.rfind(b"\n") + 1]
    big, _, _, _ = synth.json_lines(a.lines, seed=8, hi=2048)
    big = big.tobytes()
    for fmt, tag, conv in (("%s", "epoch", lambda v: v), (YMD, "ymd", ymd_lines)):
        res["device_512KB_" + tag] = device_arms(conv(chunk), fmt)
        res["device_lines_" + tag] = device_arms(conv(big), fmt)
        res["device_lines_" + tag]["lines"] = a.lines
    del big

    # host-buffer calls over 512 KB chunks (epoch form)
    chunks = []
    for i in range(a.chunks):
        c = synth.json_lines(CHUNK // 600, seed=100 + i, hi=2048)[0].tobytes()[:CHUNK]
        chunks.append(c[:c.rfind(b"\n") + 1])
    ts = lc.Timestamp("%s")
    cap = 2 * CHUNK + 65536
    calls = {
        "plain": lambda v: eng.split_json_parse_sls(js, v, 10, b"content", **skw, out_cap=cap),
        "ts": lambda v: eng.split_json_timestamp_parse_sls(js, v, 10, b"content", b"ts", ts, now, -1, **skw,
                                                           out_cap=cap),
        "ts_lz4": lambda v: eng.split_json_timestamp_parse_sls_lz4(js, v, 10, b"content", b"ts", ts, now, -1, **skw,
                                                                   tail=b"\x1a\x01t", out_cap=cap),
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

    # host classes through the JSON host API, times an hour before the real clock (YMD, local time)
    recent = int(time.time()) - 3600
    groups = []
    for i in range(a.json_groups):
        v = ymd_lines(chunks[i % len(chunks)], base=recent).decode("utf-8")
        groups.append({"metadata": {"log.file.offset": OKEY.decode()}, "tags": {}, "events": [
            {"type": 1, "timestamp": now, "fileOffset": 4096, "rawSize": len(v), "contents": {"content": v}}]})
    procs = (lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"}),
             lc.HostProcessor("processor_parse_json_native", {"SourceKey": "content",
                                                              "KeepingSourceWhenParseFail": True}),
             lc.HostProcessor("processor_parse_timestamp_native", {"SourceKey": "ts", "SourceFormat": YMD}))
    hc = {0: [], 1: []}
    for g in groups[:1]:
        for mode in (0, 1):
            capi.host_chain3_serialize_sls(*procs, g, False, mode)
    for g in groups:
        outs = {}
        for mode in (0, 1):
            t0 = time.perf_counter()
            outs[mode] = capi.host_chain3_serialize_sls(*procs, g, False, mode)
            hc[mode].append((time.perf_counter() - t0) * 1e3)
        assert outs[0][0] == outs[1][0], "mode 0 and mode 1 differ"
    res["host_class_512KB_ms"] = {"device_path": round(statistics.median(hc[0]), 3),
                                  "process_x3_serialize": round(statistics.median(hc[1]), 3),
                                  "timestamp_counters": procs[2].counters()}
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
