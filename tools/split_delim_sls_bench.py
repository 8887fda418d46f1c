"""Split -> delimiter -> SLS wire format on C4's CSV lines, with log.file.offset metadata (offset key on).

The delimiter stage is C4's: synth.CSV_KEYS, comma separator, double-quote quote, extend mode, max_fields 11.
Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident step lc_split_lines_dev + lc_delim_parse_dev + lc_sls_serialize_split_delim_dev against split
    + delimiter alone (tables left on the device) -- CUDA events, median over --steps after --warmup, the two
    alternated, over --lines CSV lines;
  * lc_split_delim_parse_sls and lc_split_delim_parse_sls_lz4 over --chunks chunks of 512 KB, against lc_split_lines +
    lc_delim_parse with their tables back, all with pinned host buffers (host clock around calls that end in a
    synchronise, sum over the chunks, median over --host-reps), and the H2D / D2H bytes of each computed from the
    shapes;
  * ProcessorSplitLogStringNative::SerializeSls(group, delimiter) against Process + Process + Serialize on 512 KB
    groups, both through the JSON host API (lc_host_chain_serialize_sls modes 0 and 1; the JSON parse is in both).
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
MAX_FIELDS = 11
SEP, QUOTE = b",", ord('"')


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=2 << 20)
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
    keys = [k.encode() for k in synth.CSV_KEYS]
    nkeys = len(keys)

    # ---- C4 device-resident step
    buf, _, _ = synth.csv_lines(a.lines)
    val = buf.tobytes()
    del buf
    n_src = len(val)
    d = torch.from_numpy(np.frombuffer(val, np.uint8).copy()).cuda()
    d_off = torch.empty(n_src, dtype=torch.int32, device="cuda")
    d_len = torch.empty(n_src, dtype=torch.int32, device="cuda")
    tabs = {}

    def split_delim():
        n = eng.split_lines_dev(d.data_ptr(), n_src, 10, d_off.data_ptr(), d_len.data_ptr(), n_src)
        if not tabs or tabs["st"].numel() < n:
            tabs["st"] = torch.empty(n, dtype=torch.uint8, device="cuda")
            tabs["nf"] = torch.empty(n, dtype=torch.int32, device="cuda")
            for k in ("fo", "fl", "fd"):
                tabs[k] = torch.empty(n * MAX_FIELDS, dtype=torch.int32, device="cuda")
        eng.delim_parse_dev(d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, SEP, QUOTE, nkeys, True, True,
                            MAX_FIELDS, *(tabs[k].data_ptr() for k in ("st", "nf", "fo", "fl", "fd")))
        return n

    def sls(d_out=None, cap=0):
        n = split_delim()
        need, _ = eng.sls_serialize_split_delim_dev(
            d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n,
            *(tabs[k].data_ptr() for k in ("st", "nf", "fo", "fl", "fd")), MAX_FIELDS, SEP, QUOTE, "extend", keys,
            b"content", offset_key=OKEY, src_pos=1 << 30, time=1700000000, d_out=d_out, out_cap=cap)
        return n, need

    n_lines, wire = sls()
    d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
    ms = {"sls": [], "tables": []}
    for k in range(a.warmup + a.steps):
        for name in ("sls", "tables"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            if name == "sls":
                assert sls(d_out.data_ptr(), wire) == (n_lines, wire)
            else:
                split_delim()
            e1.record(stream)
            e1.synchronize()
            if k >= a.warmup:
                ms[name].append(e0.elapsed_time(e1))
    dev = (float(np.median(ms["sls"])), float(np.median(ms["tables"])))
    del d, d_off, d_len, d_out
    tabs.clear()

    # ---- host calls over 512 KB chunks (pinned)
    chunk = 512 * 1024
    src = val[:chunk]
    keep = []
    h_src = pinned(L, chunk, np.uint8, keep)
    h_src[:] = np.frombuffer(src, np.uint8)
    _kk, cfg = capi.Engine._delim_sls_cfg(keys, b"content", b"content", False, False, False)
    sp = np.frombuffer(SEP, np.uint8)
    dcfg = [capi._p(sp), 1, QUOTE, 1, 0, 1, MAX_FIELDS]  # sep .. max_fields: extend, allow_short
    wcap = 4 * chunk + 65536
    h_wire = pinned(L, wcap, np.uint8, keep)
    h_blk = pinned(L, wcap, np.uint8, keep)
    h_off, h_len = pinned(L, chunk, np.uint32, keep), pinned(L, chunk, np.uint32, keep)
    h_st, h_nf = pinned(L, chunk, np.uint8, keep), pinned(L, chunk, np.uint32, keep)
    h_fo, h_fl, h_fd = (pinned(L, chunk * MAX_FIELDS, np.uint32, keep) for _ in range(3))
    p = capi._p
    sizes = {"wire": 0, "blk": 0, "n": 0}
    tail = b"\x1a\x05topic"
    h_tail = np.frombuffer(tail, np.uint8)

    def host_sls():
        need, nev = C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(4, np.uint64)
        capi._check(L.lc_split_delim_parse_sls(eng._h, p(h_src), chunk, 10, *dcfg, *cfg, OKEY, len(OKEY), 1 << 30,
                                               1700000000, 0xFFFFFFFF, p(h_wire), wcap, C.byref(need), C.byref(nev),
                                               p(ctr)))
        sizes["wire"], sizes["n"] = int(need.value), int(nev.value)

    def host_lz4():
        need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(4, np.uint64)
        capi._check(L.lc_split_delim_parse_sls_lz4(eng._h, p(h_src), chunk, 10, *dcfg, *cfg, OKEY, len(OKEY),
                                                   1 << 30, 1700000000, 0xFFFFFFFF, p(h_tail), len(tail), p(h_blk),
                                                   wcap, C.byref(need), C.byref(raw), C.byref(nev), p(ctr)))
        sizes["blk"] = int(need.value)

    def host_tables():
        nn = C.c_uint64(0)
        capi._check(L.lc_split_lines(eng._h, p(h_src), chunk, 10, p(h_off), p(h_len), chunk, C.byref(nn)))
        n = int(nn.value)
        capi._check(L.lc_delim_parse(eng._h, p(h_src), chunk, p(h_off), p(h_len), n, p(sp), 1, QUOTE, nkeys, 1, 1,
                                     MAX_FIELDS, p(h_st), p(h_nf), p(h_fo), p(h_fl), p(h_fd)))

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
    text = src.decode("latin-1")
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": chunk,
                         "contents": {"content": text}}]}
    dconf = {"SourceKey": "content", "Separator": ",", "Quote": '"', "Keys": synth.CSV_KEYS,
             "OverflowedFieldsTreatment": "extend"}
    jres = {}
    for mode, name in ((0, "json_serialize_sls"), (1, "json_process_process_serialize")):
        spl = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
        dp = lc.HostProcessor("processor_parse_delimiter_native", dconf)
        capi.host_chain_serialize_sls(spl, dp, group, False, mode)
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for _g in range(a.json_groups):
                out = capi.host_chain_serialize_sls(spl, dp, group, False, mode)
            ts.append((time.perf_counter() - t0) * 1e3 / a.json_groups)
        jres[name] = (float(np.median(ts)), out[0])
    assert jres["json_serialize_sls"][1] == jres["json_process_process_serialize"][1]

    name, pl = card()
    n = sizes["n"]
    print(json.dumps({
        "metric": "split_delim_sls", "gpu": name, "power_limit_w": pl,
        "c4_lines": n_lines, "c4_bytes": n_src, "c4_wire_bytes": wire, "max_fields": MAX_FIELDS,
        "c4_dev_step_ms_median": round(dev[0], 3), "c4_split_delim_ms_median": round(dev[1], 3),
        "dev_steps": a.steps, "chunks": a.chunks, "chunk_bytes": chunk, "chunk_pieces": n,
        "host_split_delim_sls_ms_median": round(res["host_sls"], 2),
        "host_split_delim_sls_lz4_ms_median": round(res["host_lz4"], 2),
        "host_split_delim_tables_ms_median": round(res["host_tables"], 2), "host_reps": a.host_reps,
        "h2d_bytes_per_chunk": {"split_delim_parse_sls": chunk, "split_lines+delim_parse": 2 * chunk + 8 * n},
        "d2h_bytes_per_chunk": {"split_delim_parse_sls": sizes["wire"], "split_delim_parse_sls_lz4": sizes["blk"],
                                "split_lines+delim_parse": 8 * n + n + 4 * n + 3 * n * MAX_FIELDS * 4},
        "json_serialize_sls_ms_per_group": round(jres["json_serialize_sls"][0], 2),
        "json_process_process_serialize_ms_per_group": round(jres["json_process_process_serialize"][0], 2),
        "per_kernel_ms": "not measured",
    }))
    eng.close()


if __name__ == "__main__":
    main()
