"""Delimiter -> regex -> SLS wire format on C4's data (synth.csv_lines, max_fields 11, ten keys, extend; the regex
stage parses column 3 with synth.CSV_URL_PATTERN into two keys).

Reports, in one JSON line with the card's name and power limit read in the same run:
  * the device-resident step lc_delim_parse_dev + lc_delim_regex_tap_dev + lc_regex_parse_dev +
    lc_sls_serialize_delim_regex_dev against C4's chain step (lc_delim_parse_tap_dev + lc_regex_parse_dev, the tables
    left on the device) -- CUDA events, median over --steps after --warmup, the two alternated;
  * the host-buffer call lc_delim_regex_parse_sls (wire bytes back) against lc_delim_regex_chain (both stages' tables
    back), and the fused lc_delim_regex_parse_sls_lz4, all with pinned host buffers (host clock around calls that end
    in a synchronise, median over --host-reps);
  * the H2D and D2H bytes of each host call, computed from its arguments.
The tables-back call leaves the host the per-event object work of both processors; this tool does not time that.
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=8 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    rx = lc.Regex(synth.CSV_URL_PATTERN)
    G = rx.ngroups
    buf, off, ln = synth.csv_lines(a.lines, seed=a.seed)
    n, MF, base_len = int(off.size), 11, int(buf.size)
    keys = [k.encode() for k in synth.CSV_KEYS]
    sep, quote = b",", ord('"')
    delim = dict(sep=sep, quote=quote, treatment="extend", keys=keys, source_key=b"content")
    regex = dict(keys=[b"path", b"k"], source_key=b"url")
    times = (1700000000 + np.arange(n) % 86400).astype(np.uint32)

    # ---- device-resident step
    i32 = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()  # noqa: E731
    side_at = (base_len + 15) // 16 * 16
    base_cap = side_at + int(ln.astype(np.uint64).sum())
    d_buf = torch.zeros(base_cap + 16, dtype=torch.uint8, device="cuda")
    d_buf[:base_len] = torch.from_numpy(np.array(buf)).cuda()
    d_off, d_len, d_t = i32(off), i32(ln), i32(times)
    d_st = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_nf = torch.empty(n, dtype=torch.int32, device="cuda")
    d_fo, d_fl, d_fd = (torch.empty(n * MF, dtype=torch.int32, device="cuda") for _ in range(3))
    d_vo, d_vl = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
    d_rs = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_co, d_cl = (torch.empty(n * G, dtype=torch.int32, device="cuda") for _ in range(2))
    tab = (d_st.data_ptr(), d_nf.data_ptr(), d_fo.data_ptr(), d_fl.data_ptr(), d_fd.data_ptr())
    dtabs = (d_off.data_ptr(), d_len.data_ptr(), n) + tab + (MF,)
    side = [0]

    def chain_step():  # C4's step: the tapped raw column is the regex stage's event table
        eng.delim_parse_dev(d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n, sep, quote, len(keys),
                            True, True, MF, *tab, 3, d_vo.data_ptr(), d_vl.data_ptr())
        eng.regex_parse_dev(rx, d_buf.data_ptr(), base_len, d_vo.data_ptr(), d_vl.data_ptr(), n, 2, d_rs.data_ptr(),
                            d_co.data_ptr(), d_cl.data_ptr())

    def sls_step(d_out=None, cap=0):
        eng.delim_parse_dev(d_buf.data_ptr(), base_len, d_off.data_ptr(), d_len.data_ptr(), n, sep, quote, len(keys),
                            True, True, MF, *tab)
        side[0] = eng.delim_regex_tap_dev(d_buf.data_ptr(), base_len, base_cap, *dtabs, delim, regex, d_vo.data_ptr(),
                                          d_vl.data_ptr())
        arena = side_at + side[0]
        eng.regex_parse_dev(rx, d_buf.data_ptr(), arena, d_vo.data_ptr(), d_vl.data_ptr(), n, 2, d_rs.data_ptr(),
                            d_co.data_ptr(), d_cl.data_ptr())
        return eng.sls_serialize_delim_regex_dev(d_buf.data_ptr(), arena, *dtabs, delim, regex, d_vo.data_ptr(),
                                                 d_vl.data_ptr(), d_rs.data_ptr(), d_co.data_ptr(), d_cl.data_ptr(),
                                                 G, d_t.data_ptr(), d_out=d_out, out_cap=cap)
    wire, _ = sls_step()
    d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.ExternalStream(eng.stream)
    ms = {"sls": [], "chain": []}
    for k in range(a.warmup + a.steps):
        for name in ("sls", "chain"):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            if name == "sls":
                got, ctr = sls_step(d_out.data_ptr(), wire)
                assert got == wire
            else:
                chain_step()
            e1.record(stream)
            e1.synchronize()
            if k >= a.warmup:
                ms[name].append(e0.elapsed_time(e1))

    # ---- host buffers (pinned): wire bytes / LZ4 block back vs both stages' tables back
    keep = []
    h_buf = pinned(L, base_len, np.uint8, keep)
    h_buf[:] = buf
    h_off, h_len, h_t = (pinned(L, 4 * n, np.uint32, keep) for _ in range(3))
    h_off[:], h_len[:], h_t[:] = off, ln, times
    h_wire = pinned(L, wire + 16, np.uint8, keep)
    zcap = wire + wire // 255 + 64
    h_blk = pinned(L, zcap, np.uint8, keep)
    h_st, h_rs = pinned(L, n, np.uint8, keep), pinned(L, n, np.uint8, keep)
    h_nf = pinned(L, 4 * n, np.uint32, keep)
    h_fo, h_fl, h_fd = (pinned(L, 4 * n * MF, np.uint32, keep) for _ in range(3))
    h_co, h_cl = (pinned(L, 4 * n * G, np.uint32, keep) for _ in range(2))
    _kk, cfg = capi.Engine._chain_cfg(delim, regex)
    p = capi._p
    sp = np.frombuffer(sep, np.uint8)
    blk_len = [0]

    def host_sls():
        need = C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        capi._check(L.lc_delim_regex_parse_sls(eng._h, rx._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(h_t), None,
                                               1, MF, *cfg, p(h_wire), wire + 16, C.byref(need), p(ctr)))
        assert need.value == wire

    def host_lz4():
        need, raw = C.c_uint64(0), C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        capi._check(L.lc_delim_regex_parse_sls_lz4(eng._h, rx._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(h_t),
                                                   None, 1, MF, *cfg, None, 0, p(h_blk), zcap, C.byref(need),
                                                   C.byref(raw), p(ctr)))
        assert raw.value == wire
        blk_len[0] = int(need.value)

    def host_tables():
        capi._check(L.lc_delim_regex_chain(eng._h, p(h_buf), base_len, p(h_off), p(h_len), n, p(sp), 1, quote,
                                           len(keys), 1, 1, MF, p(h_st), p(h_nf), p(h_fo), p(h_fl), p(h_fd), 3, rx._h,
                                           2, p(h_rs), p(h_co), p(h_cl)))

    res = {}
    for name, fn in (("host_sls", host_sls), ("host_lz4", host_lz4), ("host_tables", host_tables)):
        fn()
        ts = []
        for _ in range(a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t0) * 1e3)
        res[name] = float(np.median(ts))
    assert bytes(h_wire[:wire]) == bytes(d_out[:wire].cpu().numpy())
    for ptr in keep:
        L.lc_host_free(ptr)

    name, pl = card()
    dev, chain = float(np.median(ms["sls"])), float(np.median(ms["chain"]))
    print(json.dumps({
        "metric": "delim_regex_sls_c4", "gpu": name, "power_limit_w": pl, "lines": n, "arena_bytes": base_len,
        "side_copy_bytes": side[0], "max_fields": MF, "wire_bytes": wire, "lz4_block_bytes": blk_len[0],
        "dev_step_ms_median": round(dev, 3), "dev_chain_step_ms_median": round(chain, 3), "dev_steps": a.steps,
        "host_sls_ms_median": round(res["host_sls"], 2), "host_lz4_ms_median": round(res["host_lz4"], 2),
        "host_tables_ms_median": round(res["host_tables"], 2), "host_reps": a.host_reps,
        "h2d_bytes": {"delim_regex_parse_sls": base_len + 12 * n, "delim_regex_chain": base_len + 8 * n},
        "d2h_bytes": {"delim_regex_parse_sls": wire, "delim_regex_parse_sls_lz4": blk_len[0],
                      "delim_regex_chain": n * 5 + 3 * n * MF * 4 + n + 2 * n * G * 4},
    }))
    eng.close()


if __name__ == "__main__":
    main()
