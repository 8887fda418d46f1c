"""Split -> regex -> filter -> SLS wire format on C2's data, with log.file.offset metadata (offset key on).

The pipeline of the reference's file-to-blackhole benchmark: the splitter, the nginx regex, then a
processor_filter_regex_native.  Three filters, each in the same run:
  * status: FilterKey [status], FilterRegex [^[45]\\d\\d$] (RULE mode; 5 of C2's 11 status values pass);
  * expr: and(status ^[45]\\d\\d$, not(browser ^curl.*)) (EXPRESSION mode);
  * no_agent: the reference benchmark's own ^no-agent$ on the last key, which C2's vocabulary never passes.
For each it reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident step lc_split_lines_dev + lc_regex_parse_dev + lc_sls_serialize_split_regex_filter_dev
    against the same without the filter (lc_sls_serialize_split_regex_dev) -- CUDA events, median over --steps after
    --warmup, the two alternated, over --lines nginx lines of 256 B;
  * lc_split_regex_filter_parse_sls and its _lz4 variant over --chunks C2 chunks of 512 KB, with pinned host buffers
    (host clock around calls that end in a synchronise, sum over the chunks, median over --host-reps), and the H2D /
    D2H bytes of each counted from the arguments;
  * ProcessorSplitLogStringNative::SerializeSls(group, regex, filter) against Process x 3 + Serialize on 512 KB
    groups, both through the JSON host API (lc_host_chain3_serialize_sls modes 0 and 1; the JSON parse is in both).
Kernel times are not measured here.  Needs a CUDA device; there is no CPU path."""
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
STATUS = r"[45]\d\d"  # regex_match is a whole-value match: ^[45]\d\d$
FILTERS = {
    "status": {"FilterKey": ["status"], "FilterRegex": [STATUS]},
    "expr": {"ConditionExp": {"operator": "and", "operands": [
        {"key": "status", "exp": STATUS, "type": "regex"},
        {"operator": "not", "operands": [{"key": "browser", "exp": "curl.*", "type": "regex"}]}]}},
    "no_agent": {"FilterKey": ["browser"], "FilterRegex": ["no-agent"]},
}


def _program(fcfg):
    """(leaves [(key, pattern)], postfix program) as ProcessorFilterNative builds them for these two shapes"""
    if "FilterKey" in fcfg:
        return [(fcfg["FilterKey"][0].encode(), fcfg["FilterRegex"][0])], [0]
    a, n = fcfg["ConditionExp"]["operands"]
    b = n["operands"][0]
    return [(a["key"].encode(), a["exp"]), (b["key"].encode(), b["exp"])], [0, 1, 0xFFFFFFFD, 0xFFFFFFFE]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=1 << 20)
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
    nginx = lc.Regex(synth.NGINX_PATTERN)
    nkeys = [k.encode() for k in synth.NGINX_KEYS]
    G = nginx.ngroups
    filters = {}
    for name, fcfg in FILTERS.items():
        leaves, prog = _program(fcfg)
        filters[name] = capi.Filter([(k, lc.Regex(r)) for k, r in leaves], prog)

    # ---- device-resident steps over one C2 buffer
    buf, _, _ = synth.nginx_lines(a.lines, line_bytes=256)
    n_src = int(buf.size)
    d = torch.from_numpy(buf.copy()).cuda()
    del buf
    d_off = torch.empty(n_src, dtype=torch.int32, device="cuda")
    d_len = torch.empty(n_src, dtype=torch.int32, device="cuda")
    st = torch.empty(a.lines + 16, dtype=torch.uint8, device="cuda")
    co = torch.empty((a.lines + 16) * G, dtype=torch.int32, device="cuda")
    cl = torch.empty((a.lines + 16) * G, dtype=torch.int32, device="cuda")

    def split_regex():
        n = eng.split_lines_dev(d.data_ptr(), n_src, 10, d_off.data_ptr(), d_len.data_ptr(), n_src)
        assert n <= a.lines + 16
        eng.regex_parse_dev(nginx, d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, len(nkeys),
                            st.data_ptr(), co.data_ptr(), cl.data_ptr())
        return n

    def step(filt, d_out=None, cap=0):
        n = split_regex()
        tabs = (d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, st.data_ptr(), co.data_ptr(),
                cl.data_ptr(), G, nkeys, b"content")
        kw = dict(offset_key=OKEY, src_pos=1 << 30, time=1700000000, d_out=d_out, out_cap=cap)
        if filt is None:
            need, ctr = eng.sls_serialize_split_regex_dev(*tabs, **kw)
        else:
            need, ctr = eng.sls_serialize_split_regex_filter_dev(*tabs, filt, **kw)
        return n, need, [int(x) for x in ctr]

    plain = step(None)
    d_out = torch.empty(plain[1] + 16, dtype=torch.uint8, device="cuda")
    dev = {}
    for name, filt in filters.items():
        n, wire, ctr = step(filt)
        ms = {"filter": [], "plain": []}
        for k in range(a.warmup + a.steps):
            for which, f, cap in (("filter", filt, wire), ("plain", None, plain[1])):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                step(f, d_out.data_ptr(), cap)
                e1.record(stream)
                e1.synchronize()
                if k >= a.warmup:
                    ms[which].append(e0.elapsed_time(e1))
        dev[name] = {"lines": n, "kept": ctr[0] - ctr[3], "removed": ctr[3], "wire_bytes": wire,
                     "dev_step_ms_median": round(float(np.median(ms["filter"])), 3),
                     "dev_step_no_filter_ms_median": round(float(np.median(ms["plain"])), 3)}
    del d, d_off, d_len, st, co, cl, d_out
    torch.cuda.empty_cache()

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
    p = capi._p
    tail = b"\x1a\x05topic"
    h_tail = np.frombuffer(tail, np.uint8)
    host = {}
    for name, filt in filters.items():
        sizes = {}

        def host_sls():
            need, nev = C.c_uint64(0), C.c_uint64(0)
            ctr = np.zeros(4, np.uint64)
            capi._check(L.lc_split_regex_filter_parse_sls(eng._h, nginx._h, p(h_src), chunk, 10, *cfg, 0, OKEY,
                                                          len(OKEY), 1 << 30, 1700000000, 0xFFFFFFFF, filt.ptr(),
                                                          p(h_wire), wcap, C.byref(need), C.byref(nev), p(ctr)))
            sizes["wire"], sizes["n"], sizes["removed"] = int(need.value), int(nev.value), int(ctr[3])

        def host_lz4():
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr = np.zeros(4, np.uint64)
            capi._check(L.lc_split_regex_filter_parse_sls_lz4(eng._h, nginx._h, p(h_src), chunk, 10, *cfg, 0, OKEY,
                                                              len(OKEY), 1 << 30, 1700000000, 0xFFFFFFFF, filt.ptr(),
                                                              p(h_tail), len(tail), p(h_blk), wcap, C.byref(need),
                                                              C.byref(raw), C.byref(nev), p(ctr)))
            sizes["blk"] = int(need.value)

        res = {}
        for call, fn in (("host_sls", host_sls), ("host_lz4", host_lz4)):
            fn()
            ts = []
            for _ in range(a.host_reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _c in range(a.chunks):
                    fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            res[call] = float(np.median(ts))
        host[name] = {"chunk_pieces": sizes["n"], "chunk_removed": sizes["removed"],
                      "host_sls_ms_median": round(res["host_sls"], 2),
                      "host_sls_lz4_ms_median": round(res["host_lz4"], 2),
                      "h2d_bytes_per_chunk": chunk + len(tail),
                      "d2h_bytes_per_chunk": {"sls": sizes["wire"], "sls_lz4": sizes["blk"]}}
    for ptr in keep:
        L.lc_host_free(ptr)

    # ---- the host classes through the JSON host API, 512 KB groups of one source event with offset metadata
    text = src[:chunk].decode("latin-1")
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": chunk,
                         "contents": {"content": text}}]}
    rconf = {"SourceKey": "content", "Regex": synth.NGINX_PATTERN, "Keys": synth.NGINX_KEYS}
    jres = {}
    for name, fcfg in FILTERS.items():
        out = {}
        for mode, which in ((0, "json_serialize_sls_ms_per_group"), (1, "json_process3_serialize_ms_per_group")):
            sp = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
            rp = lc.HostProcessor("processor_parse_regex_native", rconf)
            fp = lc.HostProcessor("processor_filter_regex_native", fcfg)
            capi.host_chain3_serialize_sls(sp, rp, fp, group, False, mode)
            ts = []
            for _ in range(a.host_reps):
                t0 = time.perf_counter()
                for _g in range(a.json_groups):
                    r = capi.host_chain3_serialize_sls(sp, rp, fp, group, False, mode)
                ts.append((time.perf_counter() - t0) * 1e3 / a.json_groups)
            out[which] = (round(float(np.median(ts)), 2), r[0], r[2])
        assert out["json_serialize_sls_ms_per_group"][1:] == out["json_process3_serialize_ms_per_group"][1:]
        jres[name] = {k: v[0] for k, v in out.items()}

    gpu, pl = card()
    print(json.dumps({
        "metric": "split_regex_filter_sls", "gpu": gpu, "power_limit_w": pl,
        "c2_lines": plain[0], "c2_bytes": n_src, "dev_steps": a.steps,
        "no_filter_wire_bytes": plain[1], "chunks": a.chunks, "chunk_bytes": chunk, "host_reps": a.host_reps,
        "filters": {k: dict(dev[k], **host[k], **jres[k]) for k in FILTERS},
        "per_kernel_ms": "not measured",
    }))
    eng.close()


if __name__ == "__main__":
    main()
