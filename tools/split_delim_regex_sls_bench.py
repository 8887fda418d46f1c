"""Split -> delimiter -> regex -> SLS wire format on C4's CSV lines, with log.file.offset metadata (offset key on).

The delimiter stage is C4's: synth.CSV_KEYS, comma separator, double-quote quote, extend mode, max_fields 11.  The
regex stage is C4's too: synth.CSV_URL_PATTERN on the url column, keys path and k.
Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident step lc_split_lines_dev + lc_delim_parse_dev + lc_delim_regex_tap_dev + lc_regex_parse_dev +
    lc_sls_serialize_split_delim_regex_dev against the same without the serialise (tables left on the device) --
    CUDA events, median over --steps after --warmup, the two alternated, over --lines CSV lines;
  * the four host calls lc_[multiline_]split_delim_regex_parse_sls[_lz4] over --chunks chunks of 512 KB, against
    lc_split_delim_parse_sls in the same run, all with pinned host buffers (host clock around calls that end in a
    synchronise, sum over the chunks, median over --host-reps), and the H2D / D2H bytes of each computed from the
    shapes;
  * ProcessorSplitLogStringNative::SerializeSls(group, delimiter, regex) against Process x 3 + Serialize on 512 KB
    groups, both through the JSON host API (lc_host_chain3_serialize_sls modes 0 and 1; the JSON parse is in both).
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
RKEYS = [b"path", b"k"]


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
    rx = lc.Regex(synth.CSV_URL_PATTERN)
    G = rx.ngroups
    delim = dict(sep=SEP, quote=QUOTE, treatment="extend", keys=keys, source_key=b"content")
    regex = dict(keys=RKEYS, source_key=b"url")

    # ---- C4 device-resident step
    buf, _, _ = synth.csv_lines(a.lines)
    val = buf.tobytes()
    del buf
    n_src = len(val)
    side_at = (n_src + 15) // 16 * 16
    d = torch.zeros(side_at + n_src + 16, dtype=torch.uint8, device="cuda")
    d[:n_src] = torch.from_numpy(np.frombuffer(val, np.uint8).copy()).cuda()
    d_off = torch.empty(n_src, dtype=torch.int32, device="cuda")
    d_len = torch.empty(n_src, dtype=torch.int32, device="cuda")
    tabs = {}
    names = ("st", "nf", "fo", "fl", "fd")

    def tables():
        """split, delimiter, tap, regex: every table the serialiser reads, left on the device"""
        n = eng.split_lines_dev(d.data_ptr(), n_src, 10, d_off.data_ptr(), d_len.data_ptr(), n_src)
        if not tabs or tabs["st"].numel() < n:
            tabs["st"], tabs["rs"] = (torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(2))
            tabs["nf"], tabs["vo"], tabs["vl"] = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
            for k in ("fo", "fl", "fd"):
                tabs[k] = torch.empty(n * MAX_FIELDS, dtype=torch.int32, device="cuda")
            tabs["co"], tabs["cl"] = (torch.empty(n * G, dtype=torch.int32, device="cuda") for _ in range(2))
        t = [tabs[k].data_ptr() for k in names]
        eng.delim_parse_dev(d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, SEP, QUOTE, nkeys, True, True,
                            MAX_FIELDS, *t)
        side = eng.delim_regex_tap_dev(d.data_ptr(), n_src, side_at + n_src, d_off.data_ptr(), d_len.data_ptr(), n,
                                       *t, MAX_FIELDS, delim, regex, tabs["vo"].data_ptr(), tabs["vl"].data_ptr())
        eng.regex_parse_dev(rx, d.data_ptr(), side_at + side, tabs["vo"].data_ptr(), tabs["vl"].data_ptr(), n,
                            len(RKEYS), tabs["rs"].data_ptr(), tabs["co"].data_ptr(), tabs["cl"].data_ptr())
        return n

    def sls(d_out=None, cap=0):
        n = tables()
        need, _ = eng.sls_serialize_split_delim_regex_dev(
            d.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, *(tabs[k].data_ptr() for k in names),
            MAX_FIELDS, delim, regex, tabs["vo"].data_ptr(), tabs["vl"].data_ptr(), tabs["rs"].data_ptr(),
            tabs["co"].data_ptr(), tabs["cl"].data_ptr(), G, offset_key=OKEY, src_pos=1 << 30, time=1700000000,
            d_out=d_out, out_cap=cap)
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
                tables()
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
    _kk, dkcfg = capi.Engine._delim_sls_cfg(keys, b"content", b"content", False, False, False)
    _kc, chain = capi.Engine._chain_cfg(delim, regex)
    sp = np.frombuffer(SEP, np.uint8)
    dcfg = [capi._p(sp), 1, QUOTE, 1, 0, 1, MAX_FIELDS]  # sep .. max_fields: extend, allow_short
    wcap = 4 * chunk + 65536
    h_wire = pinned(L, wcap, np.uint8, keep)
    h_blk = pinned(L, wcap, np.uint8, keep)
    p = capi._p
    sizes = {}
    tail = b"\x1a\x05topic"
    h_tail = np.frombuffer(tail, np.uint8)
    okt = [OKEY, len(OKEY), 1 << 30, 1700000000, 0xFFFFFFFF]

    def call(name, fn, lead, lz4, ml):
        def run():
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(8, np.uint64), np.zeros(3, np.uint64)
            z = [p(h_tail), len(tail)] if lz4 else []
            outs = [p(h_blk if lz4 else h_wire), wcap, C.byref(need)] + ([C.byref(raw)] if lz4 else []) + \
                [C.byref(nev), p(ctr)] + ([p(mctr)] if ml else [])
            capi._check(fn(*lead, *okt, *z, *outs))
            sizes[name] = (int(need.value), int(nev.value))
        return run

    sdr = [1, MAX_FIELDS] + chain  # allow_short, max_fields, both stages
    mlh = [None, None, None, 0]
    calls = [
        ("split_delim_regex_parse_sls", call("sls", L.lc_split_delim_regex_parse_sls,
                                             [eng._h, rx._h, p(h_src), chunk, 10] + sdr, False, False)),
        ("split_delim_regex_parse_sls_lz4", call("lz4", L.lc_split_delim_regex_parse_sls_lz4,
                                                 [eng._h, rx._h, p(h_src), chunk, 10] + sdr, True, False)),
        ("multiline_split_delim_regex_parse_sls", call("ml", L.lc_multiline_split_delim_regex_parse_sls,
                                                       [eng._h, rx._h, p(h_src), chunk] + mlh + sdr, False, True)),
        ("multiline_split_delim_regex_parse_sls_lz4", call("ml_lz4", L.lc_multiline_split_delim_regex_parse_sls_lz4,
                                                           [eng._h, rx._h, p(h_src), chunk] + mlh + sdr, True, True)),
        ("split_delim_parse_sls", call("sd", L.lc_split_delim_parse_sls,
                                       [eng._h, p(h_src), chunk, 10] + dcfg + dkcfg, False, False)),
    ]
    res = {}
    for name, fn in calls:
        fn()
        ts = []
        for _ in range(a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _c in range(a.chunks):
                fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[name] = round(float(np.median(ts)), 2)
    for ptr in keep:
        L.lc_host_free(ptr)

    # ---- the host class through the JSON host API, 512 KB groups of one source event with offset metadata
    text = src.decode("latin-1")
    group = {"metadata": {"log.file.offset": OKEY.decode()}, "tags": {"__topic__": "t"},
             "events": [{"type": 1, "timestamp": 1700000000, "fileOffset": 4096, "rawSize": chunk,
                         "contents": {"content": text}}]}
    dconf = {"SourceKey": "content", "Separator": ",", "Quote": '"', "Keys": synth.CSV_KEYS,
             "OverflowedFieldsTreatment": "extend"}
    rconf = {"SourceKey": "url", "Regex": synth.CSV_URL_PATTERN, "Keys": ["path", "k"]}
    jres = {}
    for mode, name in ((0, "json_serialize_sls"), (1, "json_process_x3_serialize")):
        spl = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
        dp = lc.HostProcessor("processor_parse_delimiter_native", dconf)
        rp = lc.HostProcessor("processor_parse_regex_native", rconf)
        capi.host_chain3_serialize_sls(spl, dp, rp, group, False, mode)
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            for _g in range(a.json_groups):
                out = capi.host_chain3_serialize_sls(spl, dp, rp, group, False, mode)
            ts.append((time.perf_counter() - t0) * 1e3 / a.json_groups)
        jres[name] = (float(np.median(ts)), out[0])
    assert jres["json_serialize_sls"][1] == jres["json_process_x3_serialize"][1]

    name, pl = card()
    n = sizes["sls"][1]
    h2d = chunk  # the chunk goes up once; keys and plans are a few hundred bytes
    print(json.dumps({
        "metric": "split_delim_regex_sls", "gpu": name, "power_limit_w": pl,
        "c4_lines": n_lines, "c4_bytes": n_src, "c4_wire_bytes": wire, "max_fields": MAX_FIELDS,
        "c4_dev_step_ms_median": round(dev[0], 3), "c4_tables_ms_median": round(dev[1], 3),
        "dev_steps": a.steps, "chunks": a.chunks, "chunk_bytes": chunk, "chunk_pieces": n,
        "host_ms_median": res, "host_reps": a.host_reps,
        "h2d_bytes_per_chunk": {k: h2d for k, _f in calls},
        "d2h_bytes_per_chunk": {"split_delim_regex_parse_sls": sizes["sls"][0],
                                "split_delim_regex_parse_sls_lz4": sizes["lz4"][0],
                                "multiline_split_delim_regex_parse_sls": sizes["ml"][0],
                                "multiline_split_delim_regex_parse_sls_lz4": sizes["ml_lz4"][0],
                                "split_delim_parse_sls": sizes["sd"][0]},
        "json_serialize_sls_ms_per_group": round(jres["json_serialize_sls"][0], 2),
        "json_process_x3_serialize_ms_per_group": round(jres["json_process_x3_serialize"][0], 2),
        "per_kernel_ms": "not measured",
    }))
    eng.close()


if __name__ == "__main__":
    main()
