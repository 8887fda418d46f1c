"""Split -> regex -> SLS wire format on C2's and C3's data, with log.file.offset metadata (offset key on).

Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident step lc_split_lines_dev (or lc_multiline_split_dev) + lc_regex_parse_dev +
    lc_sls_serialize_split_regex_dev against split + regex alone (tables left on the device) -- CUDA events, median
    over --steps after --warmup, the two alternated.  C2: --lines nginx lines of 256 B, synth.NGINX_PATTERN (ten
    keys).  C3: --records Java records, split on synth.JAVA_START_PATTERN, parsed by a record regex whose last group
    spans the rest of the record;
  * lc_split_regex_parse_sls and lc_split_regex_parse_sls_lz4 over --chunks C2 chunks of 512 KB, against
    lc_split_lines + lc_regex_parse with their tables back, all with pinned host buffers (host clock around calls
    that end in a synchronise, sum over the chunks, median over --host-reps), and the H2D / D2H bytes of each computed
    from the shapes;
  * ProcessorSplitLogStringNative::SerializeSls(group, regex) against Process + Process + Serialize on 512 KB groups,
    both through the JSON host API (lc_host_chain_serialize_sls modes 0 and 1; the JSON parse is in both).
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
RECORD_PATTERN = r"\[([^\]]+)\] \[(\w+)\] ([^:]+): (.*)"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=4 << 20)
    ap.add_argument("--records", type=int, default=200_000)
    ap.add_argument("--chunks", type=int, default=2048)
    ap.add_argument("--json-groups", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    stream = torch.cuda.ExternalStream(eng.stream)

    def device_step(val, rx, keys, ml):
        """(median ms of split + regex + serialise, median ms of split + regex, pieces, wire bytes)"""
        n_src = len(val)
        d = torch.from_numpy(np.frombuffer(val, np.uint8).copy()).cuda()
        d_off = torch.empty(n_src, dtype=torch.int32, device="cuda")
        d_len = torch.empty(n_src, dtype=torch.int32, device="cuda")
        d_fl = torch.empty(n_src, dtype=torch.uint8, device="cuda")
        G = rx.ngroups
        st = [None]
        tabs = [None]

        def split_regex():
            if ml is None:
                n = eng.split_lines_dev(d.data_ptr(), n_src, 10, d_off.data_ptr(), d_len.data_ptr(), n_src)
            else:
                n, _ = eng.multiline_split_dev(d.data_ptr(), n_src, *ml, d_off.data_ptr(), d_len.data_ptr(),
                                               d_fl.data_ptr(), n_src)
            if st[0] is None or st[0].numel() < n:
                st[0] = torch.empty(n, dtype=torch.uint8, device="cuda")
                tabs[0] = [torch.empty(n * G, dtype=torch.int32, device="cuda") for _ in range(2)]
            eng.regex_parse_dev(rx, d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, len(keys),
                                st[0].data_ptr(), tabs[0][0].data_ptr(), tabs[0][1].data_ptr())
            return n

        def sls(d_out=None, cap=0):
            n = split_regex()
            need, _ = eng.sls_serialize_split_regex_dev(
                d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, st[0].data_ptr(), tabs[0][0].data_ptr(),
                tabs[0][1].data_ptr(), G, keys, b"content", offset_key=OKEY, src_pos=1 << 30, time=1700000000,
                d_out=d_out, out_cap=cap)
            return n, need
        n, wire = sls()
        d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
        ms = {"sls": [], "tables": []}
        for k in range(a.warmup + a.steps):
            for name in ("sls", "tables"):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                if name == "sls":
                    assert sls(d_out.data_ptr(), wire) == (n, wire)
                else:
                    split_regex()
                e1.record(stream)
                e1.synchronize()
                if k >= a.warmup:
                    ms[name].append(e0.elapsed_time(e1))
        return float(np.median(ms["sls"])), float(np.median(ms["tables"])), n, wire

    # ---- C2 / C3 device-resident steps
    nginx = lc.Regex(synth.NGINX_PATTERN)
    nkeys = [k.encode() for k in synth.NGINX_KEYS]
    buf, _, _ = synth.nginx_lines(a.lines, line_bytes=256)
    c2 = device_step(buf.tobytes(), nginx, nkeys, None)
    del buf
    rec = lc.Regex(RECORD_PATTERN)
    rkeys = [b"time", b"level", b"class", b"message"]
    jbuf, _, _ = synth.java_stack_records(a.records)
    ml = (lc.Regex(synth.JAVA_START_PATTERN), None, None, False)
    c3 = device_step(jbuf.tobytes(), rec, rkeys, ml)
    c3_bytes = int(jbuf.size)
    del jbuf

    # ---- host calls over 512 KB chunks (pinned)
    chunk = 512 * 1024
    cbuf, _, _ = synth.nginx_lines(chunk // 256 * 8, line_bytes=256)
    src = cbuf.tobytes()
    keep = []
    h_src = pinned(L, chunk, np.uint8, keep)
    h_src[:] = np.frombuffer(src[:chunk], np.uint8)
    _kk, cfg = capi.Engine._delim_sls_cfg(nkeys, b"content", b"content", False, False, False)
    wcap = 4 * chunk + 65536
    h_wire = pinned(L, wcap, np.uint8, keep)
    h_blk = pinned(L, wcap, np.uint8, keep)
    h_off, h_len = pinned(L, 4 * chunk, np.uint32, keep), pinned(L, 4 * chunk, np.uint32, keep)
    G = nginx.ngroups
    h_st = pinned(L, chunk, np.uint8, keep)
    h_co, h_cl = pinned(L, 4 * chunk * G, np.uint32, keep), pinned(L, 4 * chunk * G, np.uint32, keep)
    p = capi._p
    sizes = {"wire": 0, "blk": 0, "n": 0}
    tail = b"\x1a\x05topic"
    h_tail = np.frombuffer(tail, np.uint8)

    def host_sls():
        need, nev = C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        capi._check(L.lc_split_regex_parse_sls(eng._h, nginx._h, p(h_src), chunk, 10, *cfg, 0, OKEY, len(OKEY),
                                               1 << 30, 1700000000, 0xFFFFFFFF, p(h_wire), wcap, C.byref(need),
                                               C.byref(nev), p(ctr)))
        sizes["wire"], sizes["n"] = int(need.value), int(nev.value)

    def host_lz4():
        need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        capi._check(L.lc_split_regex_parse_sls_lz4(eng._h, nginx._h, p(h_src), chunk, 10, *cfg, 0, OKEY, len(OKEY),
                                                   1 << 30, 1700000000, 0xFFFFFFFF, p(h_tail), len(tail), p(h_blk),
                                                   wcap, C.byref(need), C.byref(raw), C.byref(nev), p(ctr)))
        sizes["blk"] = int(need.value)

    def host_tables():
        nn = C.c_uint64(0)
        capi._check(L.lc_split_lines(eng._h, p(h_src), chunk, 10, p(h_off), p(h_len), chunk, C.byref(nn)))
        n = int(nn.value)
        capi._check(L.lc_regex_parse(eng._h, nginx._h, p(h_src), chunk, p(h_off), p(h_len), n, len(nkeys), p(h_st),
                                     p(h_co), p(h_cl)))

    res = {}
    for name, fn in (("host_sls", host_sls), ("host_lz4", host_lz4), ("host_tables", host_tables)):
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

    # ---- the host class through the JSON host API, 512 KB groups of one source event with offset metadata
    text = src[:chunk].decode("latin-1")
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": chunk,
                         "contents": {"content": text}}]}
    rconf = {"SourceKey": "content", "Regex": synth.NGINX_PATTERN, "Keys": synth.NGINX_KEYS}
    jres = {}
    for mode, name in ((0, "json_serialize_sls"), (1, "json_process_process_serialize")):
        sp = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
        rp = lc.HostProcessor("processor_parse_regex_native", rconf)
        capi.host_chain_serialize_sls(sp, rp, group, False, mode)
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for _g in range(a.json_groups):
                out = capi.host_chain_serialize_sls(sp, rp, group, False, mode)
            ts.append((time.perf_counter() - t0) * 1e3 / a.json_groups)
        jres[name] = (float(np.median(ts)), out[0])
    assert jres["json_serialize_sls"][1] == jres["json_process_process_serialize"][1]

    name, pl = card()
    n = sizes["n"]
    print(json.dumps({
        "metric": "split_regex_sls", "gpu": name, "power_limit_w": pl,
        "c2_lines": c2[2], "c2_bytes": a.lines * 256, "c2_wire_bytes": c2[3],
        "c2_dev_step_ms_median": round(c2[0], 3), "c2_split_regex_ms_median": round(c2[1], 3),
        "c3_records": c3[2], "c3_bytes": c3_bytes, "c3_wire_bytes": c3[3],
        "c3_dev_step_ms_median": round(c3[0], 3), "c3_split_regex_ms_median": round(c3[1], 3),
        "dev_steps": a.steps, "chunks": a.chunks, "chunk_bytes": chunk, "chunk_pieces": n,
        "host_split_regex_sls_ms_median": round(res["host_sls"], 2),
        "host_split_regex_sls_lz4_ms_median": round(res["host_lz4"], 2),
        "host_split_regex_tables_ms_median": round(res["host_tables"], 2), "host_reps": a.host_reps,
        "h2d_bytes_per_chunk": {"split_regex_parse_sls": chunk, "split_lines+regex_parse": 2 * chunk + 8 * n},
        "d2h_bytes_per_chunk": {"split_regex_parse_sls": sizes["wire"], "split_regex_parse_sls_lz4": sizes["blk"],
                                "split_lines+regex_parse": 8 * n + n + 2 * n * G * 4},
        "json_serialize_sls_ms_per_group": round(jres["json_serialize_sls"][0], 2),
        "json_process_process_serialize_ms_per_group": round(jres["json_process_process_serialize"][0], 2),
        "per_kernel_ms": "not measured",
    }))
    eng.close()


if __name__ == "__main__":
    main()
