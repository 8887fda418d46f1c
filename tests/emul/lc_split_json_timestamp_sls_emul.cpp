// lc_split_json_timestamp_sls_emul.cpp -- TEST-ONLY host build of the split -> JSON -> timestamp chain
// (loongcollector_b200/csrc/lc_exec.cuh: lc_split_json_sls_setup, lc_split_json_ts_setup, lc_json_resolve_*,
// lc_json_ts_last_member, lc_split_json_ts_value, lc_ts_compile / lc_ts_full / lc_ts_resolve, lc_split_json_ts_time,
// lc_split_json_ts_verdict and lc_split_json_sls_body), the statements the resolve, tap, timestamp, size and emit
// kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

int refuse(const char* why, char* err, uint32_t err_cap) {
    strncpy(err, why, err_cap - 1);
    err[err_cap - 1] = 0;
    return -1;
}

} // namespace

extern "C" {

// The whole chain over the pieces off / len of src and the tables of lc_json_parse over them (entries of 4 words,
// arena_len arena bytes): the resolve, the tap with W = nlanes lanes into a value buffer of src_len + arena_len bytes,
// the full parse per value, the cache pass over the pieces as one group with W = nlanes lanes, then the records with
// `nlanes` lanes one after the other.  fmt / source_year / adjust: the timestamp stage (compiled and zone-probed
// here); now_tm = localtime_r(now)'s (tm_year, tm_mon, tm_mday).  val_off / val_len[n] receive the tap's table, vbuf
// (src_len + arena_len bytes, may be NULL) the value buffer, ts_status[n] the timestamp stage's verdicts;
// counters[8] += the chain's.  Returns the total size (out written when it fits out_cap), -1 when refused
// (err = why), -2 when a record's writer did not end at the size the counting pass gave it.
int64_t emul_split_json_ts_sls(const uint8_t* src, uint64_t src_len, const uint32_t* off, const uint32_t* len,
                               uint64_t n, const uint8_t* status, const uint64_t* first, const uint32_t* ent,
                               const uint8_t* arena, uint64_t arena_len, const char* source_key, uint32_t source_len,
                               const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                               int copy_raw, const char* offset_key, uint32_t offset_len, uint64_t src_pos,
                               uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len, const char* fmt,
                               uint64_t fmt_len, int32_t source_year, int32_t adjust, int64_t now,
                               const int32_t* now_tm, int32_t discard_interval, int enable_ns, uint32_t nlanes,
                               uint32_t* val_off, uint32_t* val_len, uint8_t* vbuf, uint8_t* ts_status, uint8_t* out,
                               uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    LcSplitJsonSlsCfg c;
    LcSplitJsonTsCfg t;
    const char* why = lc_split_json_sls_setup(source_key, source_len, renamed_key, renamed_len, offset_key, offset_len,
                                              keep_fail, keep_succeed, copy_raw, src_pos, time, time_ns, &c);
    if (!why)
        why = lc_split_json_ts_setup(c, tkey, tkey_len, enable_ns, &t);
    if (why)
        return refuse(why, err, err_cap);
    t.arena_at = src_len;
    t.val_cap = src_len + arena_len;
    static LcTsConf conf;
    memset(&conf, 0, sizeof conf);
    if (lc_ts_compile(fmt, fmt_len, conf, &why) != 0)
        return refuse(why, err, err_cap);
    conf.source_year = source_year;
    conf.adjust = adjust;
    lc_ts_probe_zone(conf);
    const LcTsNow tn{now, now_tm[0], now_tm[1], now_tm[2], discard_interval};
    const LcJsonEntry* e = reinterpret_cast<const LcJsonEntry*>(ent);
    auto members = [&](uint64_t i) {
        return (status[i] & 0x7Fu) == LC_JSON_ST_OK ? (uint32_t)(first[i + 1] - first[i]) : 0u;
    };
    // the resolve, as the split -> JSON chain runs it
    const uint64_t m_all = first[n];
    std::vector<uint32_t> win(m_all + 1), scratch(3 * m_all + 3);
    std::vector<LcJsonSlsEv> ev(n);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t m = members(i);
        const uint64_t f = first[i];
        if (m <= LC_JSON_SLS_WARP) {
            LcJsonResolveWarp w;
            lc_json_resolve_warp<LcJsonKeyHash>(c, src, arena, e + f, m, win.data() + f, &ev[i], w, 0u);
        } else {
            lc_json_resolve_sort<LcJsonKeyHash>(c, src, arena, e + f, m, win.data() + f, &ev[i], scratch.data() + f,
                                                scratch.data() + m_all + f, scratch.data() + 2 * m_all + f);
        }
    }
    // the tap: the value table and the value buffer (bytes no value covers are left as 0xEE)
    std::vector<uint8_t> val(src_len + arena_len + 1, 0xEE);
    std::vector<uint32_t> v(nlanes);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t w = lc_json_ts_last_member(t, src, arena, e + first[i], members(i), v.data(), 0u, nlanes);
        uint32_t from;
        lc_split_json_ts_value(c, t, status[i], off[i], len[i], e + first[i], w, &from, &val_off[i], &val_len[i]);
        if (val_len[i] != LC_TS_NO_KEY && val_len[i])
            memcpy(val.data() + val_off[i], lc_json_span(src, arena, from), val_len[i]);
    }
    if (vbuf && src_len + arena_len)
        memcpy(vbuf, val.data(), src_len + arena_len);
    const LcTsSpans sp{val_off, val_len, nullptr, 1};
    std::vector<LcTsFull> full(n);
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t o, l;
        if (sp.get(i, o, l))
            full[i] = lc_ts_full(conf, tn, val.data() + o, l);
    }
    std::vector<int64_t> sec(n);
    std::vector<uint32_t> nsec(n);
    uint64_t tcnt[5] = {0, 0, 0, 0, 0}; // the passes' own counters: the chain takes its from the verdicts
    static LcTsWarp tw;
    lc_ts_resolve(conf, tn, val.data(), sp, full.data(), 0, n, sec.data(), nsec.data(), ts_status, tcnt, tw, 0,
                  nlanes);
    auto row = [&](uint64_t i) {
        LcSplitJsonSlsRow r;
        r.po = off[i];
        r.plen = len[i];
        r.status = status[i];
        r.e = e + first[i];
        r.win = win.data() + first[i];
        r.m = members(i);
        r.ev = ev[i];
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const LcSplitJsonSlsRow r = row(i);
        const LcSplitRegexTsTime tm = lc_split_json_ts_time(c, t, ts_status[i], sec[i], nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_json_sls_body(c, src, arena, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const uint32_t bits = lc_split_json_ts_verdict(c, r.status, ts_status[i]);
        for (uint32_t k = 0; k < LC_SRTS_COUNTERS; ++k)
            counters[k] += (bits >> k) & 1u;
    }
    if (total > out_cap)
        return (int64_t)total;
    uint64_t o = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (!body[i])
            continue;
        const LcSplitRegexTsTime tm = lc_split_json_ts_time(c, t, ts_status[i], sec[i], nsec[i]);
        uint8_t h[6];
        h[0] = 0x0A;
        const uint32_t hn = 1 + lc_put_varint(h + 1, body[i]), rec = hn + body[i];
        memcpy(out + o, h, hn);
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, hn, rec, lane, nlanes};
            lc_split_json_sls_body(c, src, arena, row(i), tm.time, tm.has_ns, tm.ns, s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
