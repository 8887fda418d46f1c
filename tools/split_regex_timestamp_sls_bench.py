"""Split -> regex -> timestamp -> SLS wire format on C2's nginx lines, tkey = time, SourceFormat %d/%b/%Y:%H:%M:%S.

The processor documentation's file pipeline: the splitter, the nginx regex, processor_parse_timestamp_native on the
regex's `time` key, then the SLS flusher.  One JSON line, with the card's name and power limit read in the same run:
  * device-resident steps (CUDA events, median over --steps after --warmup, the arms alternated), at one 512 KB reader
    chunk and at --lines lines of 256 B (C2's size):
      - "plain": lc_split_lines_dev + lc_regex_parse_dev + lc_sls_serialize_split_regex_dev (the chain without the
        timestamp stage, each record stamped with the source event's time);
      - "ts": the same with lc_split_regex_timestamp_tap_dev + lc_timestamp_parse_dev (one group) +
        lc_sls_serialize_split_regex_timestamp_dev;
      - "ts_passes_1grp" / "ts_passes_32grp": the tap and the two timestamp passes alone, over the whole chunk as one
        group and, for comparison only, cut into groups of 32 events (the cache pass then has no serial walk; the
        results differ).  Their difference is the cost of the one-warp cache pass over one group.
  * host-buffer calls over --chunks C2 chunks of 512 KB (host clock around calls that end in a synchronise, median of
    the per-chunk time over the chunks): lc_split_regex_parse_sls against lc_split_regex_timestamp_parse_sls and its
    _lz4 variant;
  * the host classes on 512 KB groups through the JSON host API (lc_host_chain3_serialize_sls): mode 0, the splitter's
    SerializeSls(group, regex, timestamp), against mode 1, Process x 3 + Serialize (the JSON parse is in both).
Needs a CUDA device; there is no CPU path."""
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
FMT = "%d/%b/%Y:%H:%M:%S"
CHUNK = 512 * 1024
TIME_FIELD = re.compile(r"^([^\[]*)\[\d\d/\w\w\w/\d{4}:\d\d:\d\d:\d\d")  # an nginx line's [time


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=4 << 20)
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
    rx = lc.Regex(synth.NGINX_PATTERN)
    ts = lc.Timestamp(FMT)
    keys = [k.encode() for k in synth.NGINX_KEYS]
    G = rx.ngroups
    now = 1700000000  # C2's times span 2020-2026: with discard_interval -1 none is discarded
    kw = dict(offset_key=OKEY, src_pos=1 << 33, time=now)

    def device_arms(val):
        n_max = len(val) // 64 + 16
        d = torch.zeros(len(val) + 32, dtype=torch.uint8, device="cuda")
        d[:len(val)] = torch.frombuffer(bytearray(val), dtype=torch.uint8).cuda()
        d_off = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        d_len = torch.empty(len(val) + 1, dtype=torch.int32, device="cuda")
        st = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        co = torch.empty(n_max * G + 1, dtype=torch.int32, device="cuda")
        cl = torch.empty(n_max * G + 1, dtype=torch.int32, device="cuda")
        v_off = torch.empty(n_max, dtype=torch.int32, device="cuda")
        v_len = torch.empty(n_max, dtype=torch.int32, device="cuda")
        sec = torch.empty(n_max, dtype=torch.int64, device="cuda")
        nsec = torch.empty(n_max, dtype=torch.int32, device="cuda")
        tst = torch.empty(n_max, dtype=torch.uint8, device="cuda")
        tcnt = torch.empty(5, dtype=torch.int64, device="cuda")
        grp1 = torch.empty(2, dtype=torch.int32, device="cuda")
        d_out = torch.empty(len(val) * 2 + 4096, dtype=torch.uint8, device="cuda")
        state = {}

        def split_regex():
            n = eng.split_lines_dev(d.data_ptr(), len(val), 10, d_off.data_ptr(), d_len.data_ptr(), len(val) + 1)
            eng.regex_parse_dev(rx, d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, len(keys),
                                st.data_ptr(), co.data_ptr(), cl.data_ptr())
            state["n"] = n
            return n, (d.data_ptr(), len(val), d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), co.data_ptr(),
                       cl.data_ptr(), G)

        def ts_passes(n, args, grp_ptr, ngroups):
            eng.split_regex_timestamp_tap_dev(*args, keys, b"content", b"time", v_off.data_ptr(), v_len.data_ptr(),
                                              offset_key=OKEY)
            eng.timestamp_parse_dev(ts, d.data_ptr(), len(val), v_off.data_ptr(), v_len.data_ptr(), n, grp_ptr,
                                    ngroups, now, -1, sec.data_ptr(), nsec.data_ptr(), tst.data_ptr(),
                                    tcnt.data_ptr())

        def plain():
            n, args = split_regex()
            return eng.sls_serialize_split_regex_dev(*args, keys, b"content", **kw, d_out=d_out.data_ptr(),
                                                     out_cap=d_out.numel())

        def with_ts():
            n, args = split_regex()
            grp1.copy_(torch.tensor([0, n], dtype=torch.int32))
            ts_passes(n, args, grp1.data_ptr(), 1)
            return eng.sls_serialize_split_regex_timestamp_dev(
                *args, keys, b"content", tst.data_ptr(), sec.data_ptr(), nsec.data_ptr(), **kw,
                d_out=d_out.data_ptr(), out_cap=d_out.numel())

        _, args0 = split_regex()
        n0 = state["n"]
        grp1.copy_(torch.tensor([0, n0], dtype=torch.int32))
        ng32 = (n0 + 31) // 32
        grp32_last = torch.arange(0, ng32 * 32 + 1, 32, dtype=torch.int32, device="cuda")
        grp32_last[-1] = n0
        arms = {"plain": plain, "ts": with_ts,
                "ts_passes_1grp": lambda: ts_passes(n0, args0, grp1.data_ptr(), 1),
                "ts_passes_32grp": lambda: ts_passes(n0, args0, grp32_last.data_ptr(), ng32)}
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
        out["lines"] = int(n0)
        out["bytes"] = len(val)
        nb, c8 = with_ts()
        out["ts_counters"] = [int(x) for x in c8]
        out["wire_bytes"] = int(nb)
        return out

    res = {"card": name, "power_limit_w": plimit, "format": FMT}
    big, _, _ = synth.nginx_lines(a.lines)
    chunk, _, _ = synth.nginx_lines(CHUNK // 256)
    res["device_512KB"] = device_arms(chunk.tobytes())
    res["device_c2"] = device_arms(big.tobytes())
    del big

    # host-buffer calls over 512 KB chunks
    chunks = [synth.nginx_lines(CHUNK // 256, seed=100 + i)[0].tobytes() for i in range(a.chunks)]
    cap = 2 * CHUNK + 65536
    host = {"plain": [], "ts": [], "ts_lz4": []}
    calls = {
        "plain": lambda v: eng.split_regex_parse_sls(rx, v, 10, keys, b"content", **kw, out_cap=cap),
        "ts": lambda v: eng.split_regex_timestamp_parse_sls(rx, v, 10, keys, b"content", b"time", ts, now, -1,
                                                            **kw, out_cap=cap),
        "ts_lz4": lambda v: eng.split_regex_timestamp_parse_sls_lz4(rx, v, 10, keys, b"content", b"time", ts, now,
                                                                    -1, **kw, tail=b"\x1a\x01t", out_cap=cap),
    }
    for v in chunks[:2]:
        for f in calls.values():
            f(v)
    for v in chunks:
        for k, f in calls.items():
            t0 = time.perf_counter()
            f(v)
            host[k].append((time.perf_counter() - t0) * 1e3)
    res["host_calls_512KB_ms"] = {k: round(statistics.median(x), 4) for k, x in host.items()}

    # host classes through the JSON host API.  processor_parse_timestamp_native keeps its default history discard
    # (43200 s behind the real clock), so each line's time is rewritten to an hour ago, 16 lines per second, with the
    # line lengths unchanged: every event the regex parses is kept.
    split_cfg = {"SourceKey": "content"}
    rcfg = {"SourceKey": "content", "Regex": synth.NGINX_PATTERN, "Keys": synth.NGINX_KEYS}
    tcfg = {"SourceKey": "time", "SourceFormat": FMT}
    mon = ("Jan", "Feb", "Mar", "Apr", "May", "Jun", "Jul", "Aug", "Sep", "Oct", "Nov", "Dec")
    recent = int(time.time()) - 3600

    def stamp(k):
        g = time.localtime(recent + k // 16)
        return "[%02d/%s/%04d:%02d:%02d:%02d" % (g.tm_mday, mon[g.tm_mon - 1], g.tm_year, g.tm_hour, g.tm_min,
                                                 g.tm_sec)

    groups = []
    for i in range(a.json_groups):
        lines = chunks[i % len(chunks)].decode("ascii").split("\n")
        v = "\n".join(TIME_FIELD.sub(lambda m, k=k: m.group(1) + stamp(k), ln, count=1) for k, ln in enumerate(lines))
        groups.append({"metadata": {"log.file.offset": OKEY.decode()}, "tags": {}, "events": [
            {"type": 1, "timestamp": now, "fileOffset": 4096, "rawSize": len(v), "contents": {"content": v}}]})
    procs = (lc.HostProcessor("processor_split_string_native", split_cfg),
             lc.HostProcessor("processor_parse_regex_native", rcfg),
             lc.HostProcessor("processor_parse_timestamp_native", tcfg))
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
