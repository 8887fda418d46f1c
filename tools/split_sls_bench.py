"""Split -> SLS wire format on C1's shape (synth.newline_lines: 1 Mi lines of 512 B) and C3's (synth.java_stack_records).

Reports, in one JSON line with the card's name and power limit:
  * the device-resident step split + lc_sls_serialize_spans_dev against the split alone (lc_split_lines_dev, or
    lc_multiline_split_dev for C3), with log.file.offset metadata; CUDA events, median over --steps after --warmup;
  * the host-buffer call lc_split_sls (wire bytes back) against lc_split_lines (line table back), pinned buffers;
  * ProcessorSplitLogStringNative::SerializeSls against Process + SLSEventGroupSerializer::Serialize over 512 KB groups
    of C1 lines (both through the JSON host API, so both times include the same JSON parse of the group);
  * the wire and input bytes, and the H2D and D2H bytes of each host call, computed from shapes.
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


def median_ms(fn, stream, warmup, steps):
    import torch
    ts = []
    for k in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        if k >= warmup:
            ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def host_ms(fn, reps):
    import torch
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lines", type=int, default=1 << 20)
    ap.add_argument("--records", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=5)
    ap.add_argument("--groups", type=int, default=20)
    a = ap.parse_args()

    import torch

    import loongcollector_b200 as lc
    from loongcollector_b200 import capi, synth
    assert torch.cuda.is_available(), "needs a CUDA device"
    L = capi.lib()
    eng = lc.Engine(0)
    stream = torch.cuda.ExternalStream(eng.stream)
    out = {"metric": "split_sls"}

    # ---- device-resident steps: C1 (split) and C3 (multiline split)
    buf, _, _ = synth.newline_lines(a.lines)
    c1_len = int(buf.size)
    c3, _, _ = synth.java_stack_records(a.records)
    c3_len = int(c3.size)
    start, cont = lc.Regex(synth.JAVA_START_PATTERN), lc.Regex(r"\s+at\s.*")
    for shape, src, ml in (("c1", buf, None), ("c3", c3, (start, cont, None, False))):
        d_src = torch.from_numpy(np.concatenate([src, np.zeros(16, np.uint8)])).cuda()
        n_src = int(src.size)
        cap = n_src
        d_off = torch.empty(cap, dtype=torch.int32, device="cuda")
        d_len = torch.empty(cap, dtype=torch.int32, device="cuda")
        d_fl = torch.empty(cap, dtype=torch.uint8, device="cuda")
        if ml is None:
            split = lambda: eng.split_lines_dev(d_src.data_ptr(), n_src, 10, d_off.data_ptr(), d_len.data_ptr(),  # noqa
                                                cap)
        else:
            split = lambda: eng.multiline_split_dev(d_src.data_ptr(), n_src, *ml, d_off.data_ptr(),  # noqa: E731
                                                    d_len.data_ptr(), d_fl.data_ptr(), cap)[0]
        n = split()
        args = (d_src.data_ptr(), n_src, d_off.data_ptr(), d_len.data_ptr(), n, b"content", OKEY, 1 << 20,
                1700000000, None)
        wire = eng.sls_serialize_spans_dev(*args)
        d_out = torch.empty(wire + 16, dtype=torch.uint8, device="cuda")
        split_ms = median_ms(split, stream, a.warmup, a.steps)
        step_ms = median_ms(lambda: (split(), eng.sls_serialize_spans_dev(*args, d_out=d_out.data_ptr(),
                                                                          out_cap=wire)), stream, a.warmup, a.steps)
        out[shape] = {"input_bytes": n_src, "events": int(n), "wire_bytes": int(wire),
                      "dev_split_ms_median": round(split_ms, 3), "dev_split_sls_ms_median": round(step_ms, 3),
                      "dev_split_sls_gb_per_s": round(n_src / step_ms / 1e6, 1)}
        if shape == "c1":
            c1_wire, c1_n, c1_dev = int(wire), int(n), d_out
        del d_src, d_off, d_len, d_fl, d_out

    # ---- host buffers (pinned): wire bytes back vs the line table back, C1
    keep = []
    h_buf = pinned(L, c1_len, np.uint8, keep)
    h_buf[:] = buf
    h_wire = pinned(L, c1_wire + 16, np.uint8, keep)
    h_off, h_len = (pinned(L, 4 * c1_n, np.uint32, keep) for _ in range(2))
    p = capi._p
    keys = capi.Engine._span_keys(b"content", OKEY, 1 << 20, 1700000000, None)

    def host_sls():
        need, nev = C.c_uint64(0), C.c_uint64(0)
        capi._check(L.lc_split_sls(eng._h, p(h_buf), c1_len, 10, *keys, p(h_wire), c1_wire + 16, C.byref(need),
                                   C.byref(nev)))
        assert need.value == c1_wire and nev.value == c1_n

    def host_table():
        nn = C.c_uint64(0)
        capi._check(L.lc_split_lines(eng._h, p(h_buf), c1_len, 10, p(h_off), p(h_len), c1_n, C.byref(nn)))

    out["c1"]["host_split_sls_ms_median"] = round(host_ms(host_sls, a.host_reps), 2)
    out["c1"]["host_split_lines_ms_median"] = round(host_ms(host_table, a.host_reps), 2)
    assert bytes(h_wire[:c1_wire]) == bytes(c1_dev[:c1_wire].cpu().numpy())
    out["c1"]["h2d_bytes"] = {"split_sls": c1_len, "split_lines": c1_len}
    out["c1"]["d2h_bytes"] = {"split_sls": c1_wire, "split_lines": 8 * c1_n}
    for ptr in keep:
        L.lc_host_free(ptr)

    # ---- host class over 512 KB groups of C1 lines with log.file.offset metadata
    per = (512 << 10) // 512
    text = bytes(buf[:per * 512]).decode()
    group = {"events": [{"type": 1, "timestamp": 1700000000, "contents": {"content": text}, "fileOffset": 4096,
                         "rawSize": len(text)}], "metadata": {"log.file.offset": "__file_offset__"},
             "tags": {"__topic__": "bench"}}
    fast = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
    ref = lc.HostProcessor("processor_split_string_native", {"SourceKey": "content"})
    got, want = fast.serialize_sls(group), ref.serialize_sls(group, process_then_serialize=True)
    assert got == want and got[0] is not None
    gs = host_ms(lambda: [fast.serialize_sls(group) for _ in range(a.groups)], a.host_reps) / a.groups
    gp = host_ms(lambda: [ref.serialize_sls(group, process_then_serialize=True) for _ in range(a.groups)],
                 a.host_reps) / a.groups
    out["group_512k"] = {"input_bytes": len(text), "events": per, "wire_bytes": len(got[0]),
                         "serialize_sls_ms_median": round(gs, 3), "process_serialize_ms_median": round(gp, 3)}

    name, pl = card()
    out.update({"gpu": name, "power_limit_w": pl, "steps": a.steps, "host_reps": a.host_reps})
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
