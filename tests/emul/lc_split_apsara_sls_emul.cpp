// lc_split_apsara_sls_emul.cpp -- TEST-ONLY host build of the split -> Apsara chain (loongcollector_b200/csrc/
// lc_exec.cuh: lc_ap_scan, lc_ap_resolve, lc_ap_fields over the pieces with the chunk as their base and one group, as
// lc_apsara_parse_dev runs them, then lc_split_apsara_sls_setup, lc_split_apsara_sls_body and lc_split_apsara_verdict
// as the size and emit kernels run them), so that the "not gpu" tier can check them against the oracle.  Not part of
// the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// The pieces (off, len) of src, Apsara-parsed with SourceKey skey, the Timezone adjustment, now and the history
// discard (-1 = none) over W emulated lanes, then serialised.  offset_key NULL = no log.file.offset metadata; time_ns
// 0xFFFFFFFF = no Time_ns.  The writing pass runs `nlanes` lanes one after the other, as the lanes of the emit
// kernel's warp share a record.  counters[5] += lc_apsara_parse's order.  Returns the total size (out written when it
// fits out_cap), -1 when the arguments are refused (err = why), -2 when a record's writer did not end exactly at the
// size the counting pass gave it.
int64_t emul_split_apsara_sls(const uint8_t* src, uint64_t src_len, const uint32_t* off, const uint32_t* len,
                              uint64_t n, const char* source_key, uint32_t source_len, int32_t adjust, int64_t now,
                              int32_t discard_interval, uint32_t W, const char* renamed_key, uint32_t renamed_len,
                              int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                              uint32_t offset_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, int enable_ns,
                              uint32_t nlanes, uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err,
                              uint32_t err_cap) {
    LcSplitApsaraSlsCfg c;
    const char* why = lc_split_apsara_sls_setup(source_key, source_len, renamed_key, renamed_len, offset_key,
                                                offset_len, keep_fail, keep_succeed, copy_raw, src_pos, time, time_ns,
                                                enable_ns, &c);
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    // the Apsara passes (tests/emul/lc_apsara_emul.cpp's statements) over the pieces, the chunk as base, one group
    static LcTsConf tc;
    memset(&tc, 0, sizeof tc);
    tc.adjust = adjust;
    lc_ts_probe_zone(tc);
    LcTsNow t;
    memset(&t, 0, sizeof t);
    t.now = now;
    t.discard_interval = discard_interval;
    const uint8_t* skey = reinterpret_cast<const uint8_t*>(source_key);
    std::vector<LcApEv> ev(n);
    for (uint64_t i = 0; i < n; ++i)
        ev[i] = lc_ap_scan(tc, src, src_len, off[i], len[i], skey, source_len);
    std::vector<uint8_t> status(n);
    std::vector<int64_t> sec(n), micro(n);
    std::vector<uint32_t> nsec(n), nent(n);
    std::vector<uint64_t> first(n + 1);
    uint64_t ap_cnt[5] = {0, 0, 0, 0, 0};
    LcApWarp w;
    lc_ap_resolve(t, ev.data(), 0, n, status.data(), sec.data(), nsec.data(), micro.data(), nent.data(), ap_cnt, w, 0,
                  W);
    uint64_t run = 0;
    for (uint64_t i = 0; i < n; ++i) {
        first[i] = run;
        run += nent[i];
    }
    first[n] = run;
    std::vector<LcApEntry> ent(run + 1);
    for (uint64_t i = 0; i < n; ++i) {
        if ((status[i] & 7u) != LC_AP_ST_OK)
            continue;
        LcApEmit em{ent.data() + first[i], off[i]};
        lc_ap_fields(src + off[i], len[i], em);
    }
    auto row = [&](uint64_t i) {
        LcSplitApsaraSlsRow r;
        r.po = off[i];
        r.plen = len[i];
        r.status = status[i];
        r.sec = sec[i];
        r.nsec = nsec[i];
        r.micro = micro[i];
        r.e = ent.data() + first[i];
        r.m = (status[i] & 7u) == LC_AP_ST_OK ? (uint32_t)(first[i + 1] - first[i]) : 0u;
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount64 s{0};
        const LcSplitApsaraSlsRow r = row(i);
        const uint32_t cnt = lc_split_apsara_sls_body(c, src, r, s);
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const uint32_t v = lc_split_apsara_verdict(c, r.status);
        for (int k = 0; k < LC_AP_SLS_COUNTERS; ++k)
            counters[k] += (v >> k) & 1u;
    }
    if (total > out_cap)
        return (int64_t)total;
    uint64_t o = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (!body[i])
            continue;
        uint8_t h[6];
        h[0] = 0x0A;
        const uint32_t hn = 1 + lc_put_varint(h + 1, body[i]), rec = hn + body[i];
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, 0u, rec, lane, nlanes};
            s.put(h, hn);
            lc_split_apsara_sls_body(c, src, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}

} // extern "C"
