// lc_split_delim_timestamp_sls_emul.cpp -- TEST-ONLY host build of the split -> delimiter -> timestamp chain
// (loongcollector_b200/csrc/lc_exec.cuh: lc_delim_sls_setup, lc_split_delim_sls_link, lc_split_delim_ts_setup,
// lc_split_delim_ts_value, lc_split_delim_ts_collapse, lc_ts_compile / lc_ts_full / lc_ts_resolve,
// lc_split_delim_ts_time, lc_split_delim_ts_verdict and lc_split_delim_sls_body), the statements the tap, timestamp,
// size and emit kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product
// library.
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

// Piece tables over src as the splitters return them and the delimiter tables over those pieces (f_off relative to
// src; src must keep 16 readable bytes on both sides, as the state machine reads aligned 16-byte chunks when it walks
// a wide row again).  offset_key NULL = no log.file.offset metadata.  The chain: the tap with W = nlanes lanes into a
// value buffer as long as src, the full parse per value, the cache pass over the pieces as one group with W = nlanes
// lanes, then the records with `nlanes` lanes one after the other.  fmt / source_year / adjust: the timestamp stage
// (compiled and zone-probed here); now_tm = localtime_r(now)'s (tm_year, tm_mon, tm_mday).  val_off / val_len[n]
// receive the tap's table, vbuf (src_len bytes, may be NULL) the value buffer, ts_status[n] the timestamp stage's
// verdicts; counters[9] += the chain's.  Returns the total size (out written when it fits out_cap), -1 when refused
// (err = why), -2 when a record's writer did not end at the size the counting pass gave it.
int64_t emul_split_delim_ts_sls(const uint8_t* src, uint64_t src_len, const uint32_t* off, const uint32_t* len,
                                uint64_t n, const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                                const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, const uint8_t* sep,
                                uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                                const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_len,
                                const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                                int copy_raw, const char* offset_key, uint32_t offset_len, uint64_t src_pos,
                                uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len, const char* fmt,
                                uint64_t fmt_len, int32_t source_year, int32_t adjust, int64_t now,
                                const int32_t* now_tm, int32_t discard_interval, int enable_ns, uint32_t nlanes,
                                uint32_t* val_off, uint32_t* val_len, uint8_t* vbuf, uint8_t* ts_status, uint8_t* out,
                                uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    uint64_t kbytes = (uint64_t)source_len + renamed_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 4);
    LcDelimSlsCfg d;
    LcSplitDelimSlsCfg c;
    LcSplitDelimTsCfg t;
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, &d, kb.data(), at.data());
    if (!why)
        why = lc_split_delim_sls_link(d, keys, key_lens, source_key, source_len, renamed_key, renamed_len, offset_key,
                                      offset_len, src_pos, time, time_ns, &c);
    if (!why)
        why = lc_split_delim_ts_setup(c, keys, key_lens, source_key, source_len, renamed_key, renamed_len, offset_key,
                                      offset_len, tkey, tkey_len, enable_ns, &t);
    if (why)
        return refuse(why, err, err_cap);
    c.d.keys = kb.data();
    c.d.key_at = at.data();
    c.okey = reinterpret_cast<const uint8_t*>(offset_key);
    static LcTsConf conf;
    memset(&conf, 0, sizeof conf);
    if (lc_ts_compile(fmt, fmt_len, conf, &why) != 0)
        return refuse(why, err, err_cap);
    conf.source_year = source_year;
    conf.adjust = adjust;
    lc_ts_probe_zone(conf);
    const LcTsNow tn{now, now_tm[0], now_tm[1], now_tm[2], discard_interval};
    auto row = [&](uint64_t i) { // as the kernels' split_delim_sls_row
        LcDelimSlsRow r;
        r.eo = off[i];
        r.elen = len[i];
        r.status = status[i];
        r.nf = nfields[i];
        r.fo = f_off + i * max_fields;
        r.fl = f_len + i * max_fields;
        r.fd = f_dq + i * max_fields;
        r.time = c.time;
        r.has_ns = c.has_ns;
        r.ns = c.ns;
        return r;
    };
    // the tap: the value table and the value buffer (bytes no value covers are left as 0xEE)
    std::vector<uint8_t> val(src_len + 1, 0xEE);
    std::vector<uint32_t> v(nlanes);
    for (uint64_t i = 0; i < n; ++i) {
        const LcSplitDelimTsValue x = lc_split_delim_ts_value(c, t, row(i));
        val_off[i] = x.off;
        val_len[i] = x.n == LC_TS_NO_KEY ? LC_TS_NO_KEY : x.n - x.dq;
        if (x.n == LC_TS_NO_KEY || !x.n)
            continue;
        if (x.dq)
            lc_split_delim_ts_collapse(val.data() + x.off, src + x.off, x.n, c.d.quote, v.data(), 0u, nlanes);
        else
            memcpy(val.data() + x.off, src + x.off, x.n);
    }
    if (vbuf && src_len)
        memcpy(vbuf, val.data(), src_len);
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
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const LcDelimSlsRow r = row(i);
        const LcSplitRegexTsTime tm = lc_split_delim_ts_time(c, t, ts_status[i], sec[i], nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_delim_sls_body(c, src, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const uint32_t bits = lc_split_delim_ts_verdict(c, r.status, ts_status[i]);
        for (uint32_t k = 0; k < LC_SDTS_COUNTERS; ++k)
            counters[k] += (bits >> k) & 1u;
    }
    if (total > out_cap)
        return (int64_t)total;
    uint64_t o = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (!body[i])
            continue;
        const LcSplitRegexTsTime tm = lc_split_delim_ts_time(c, t, ts_status[i], sec[i], nsec[i]);
        uint8_t h[6];
        h[0] = 0x0A;
        const uint32_t hn = 1 + lc_put_varint(h + 1, body[i]), rec = hn + body[i];
        memcpy(out + o, h, hn);
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, hn, rec, lane, nlanes};
            lc_split_delim_sls_body(c, src, row(i), tm.time, tm.has_ns, tm.ns, s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
