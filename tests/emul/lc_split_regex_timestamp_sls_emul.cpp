// lc_split_regex_timestamp_sls_emul.cpp -- TEST-ONLY host build of the split -> regex -> timestamp chain
// (loongcollector_b200/csrc/lc_exec.cuh: lc_split_regex_sls_setup, lc_split_regex_ts_setup, lc_split_regex_ts_value,
// lc_ts_compile / lc_ts_full / lc_ts_resolve, lc_split_regex_ts_time, lc_split_regex_ts_verdict and
// lc_split_regex_sls_body), the statements the tap, timestamp, size and emit kernels run, so that the "not gpu" tier
// can check them against the oracle.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

struct Chain {
    LcSplitRegexSlsCfg c;
    LcSplitRegexTsCfg t;
    std::vector<uint32_t> plan, at;
    std::vector<uint8_t> kb;
};

// the chain's configuration, as the C-ABI builds it; nullptr or why it is refused
const char* setup(Chain& ch, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                  uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                  int copy_raw, int whole_line, const char* offset_key, uint32_t offset_len, uint64_t src_pos,
                  uint32_t time, uint32_t time_ns, uint32_t pitch, const char* tkey, uint32_t tkey_len,
                  int enable_ns) {
    ch.plan.assign(3 * (size_t)nkeys + 24, 0);
    const char* why = lc_split_regex_sls_setup(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len,
                                               offset_key, offset_len, keep_fail, keep_succeed, copy_raw, whole_line,
                                               pitch, src_pos, time, time_ns, &ch.c, ch.plan.data());
    if (why)
        return why;
    std::vector<const char*> strings(nkeys + LC_SPLIT_REGEX_SLS_NSTR);
    std::vector<uint32_t> lens(nkeys + LC_SPLIT_REGEX_SLS_NSTR);
    lc_split_regex_sls_strings(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len, offset_key,
                               offset_len, strings.data(), lens.data());
    why = lc_split_regex_ts_setup(ch.c, ch.plan.data(), strings.data(), lens.data(), tkey, tkey_len, enable_ns,
                                  &ch.t);
    if (why)
        return why;
    uint64_t kbytes = 0;
    for (uint32_t l : lens)
        kbytes += l;
    ch.kb.assign(kbytes + 1, 0);
    ch.at.assign(nkeys + LC_SPLIT_REGEX_SLS_NSTR + 1, 0);
    lc_sls_key_table(strings.data(), lens.data(), nkeys + LC_SPLIT_REGEX_SLS_NSTR, ch.kb.data(), ch.at.data());
    ch.c.x.plan = ch.plan.data();
    ch.c.x.key_at = ch.at.data();
    ch.c.x.keys = ch.kb.data();
    return nullptr;
}

LcSplitRegexSlsRow row(const Chain& ch, const uint32_t* off, const uint32_t* len, const uint8_t* status,
                       const uint32_t* cap_off, const uint32_t* cap_len, uint32_t pitch, uint64_t i) {
    LcSplitRegexSlsRow r;
    r.po = off[i];
    r.plen = len[i];
    r.status = ch.c.x.whole_line ? 0u : status[i];
    r.co = cap_off ? cap_off + i * pitch : nullptr;
    r.cl = cap_len ? cap_len + i * pitch : nullptr;
    return r;
}

int refuse(const char* why, char* err, uint32_t err_cap) {
    strncpy(err, why, err_cap - 1);
    err[err_cap - 1] = 0;
    return -1;
}

} // namespace

extern "C" {

// The whole chain over the pieces off / len of src and the regex tables over them: the tap, the full parse per value,
// the cache pass over the pieces as one group with W = nlanes lanes, then the records with `nlanes` lanes one after
// the other.  fmt / source_year / adjust: the timestamp stage (compiled and zone-probed here); now_tm =
// localtime_r(now)'s (tm_year, tm_mon, tm_mday).  val_off / val_len[n] receive the tap's table, ts_status[n] the
// timestamp stage's verdicts; counters[8] += the chain's.  Returns the total size (out written when it fits out_cap),
// -1 when refused (err = why), -2 when a record's writer did not end at the size the counting pass gave it.
int64_t emul_split_regex_ts_sls(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                                const uint8_t* status, const uint32_t* cap_off, const uint32_t* cap_len,
                                uint32_t pitch, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                const char* source_key, uint32_t source_len, const char* renamed_key,
                                uint32_t renamed_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                                const char* offset_key, uint32_t offset_len, uint64_t src_pos, uint32_t time,
                                uint32_t time_ns, const char* tkey, uint32_t tkey_len, const char* fmt,
                                uint64_t fmt_len, int32_t source_year, int32_t adjust, int64_t now,
                                const int32_t* now_tm, int32_t discard_interval, int enable_ns, uint32_t nlanes,
                                uint32_t* val_off, uint32_t* val_len, uint8_t* ts_status, uint8_t* out,
                                uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    Chain ch;
    const char* why = setup(ch, keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len, keep_fail,
                            keep_succeed, copy_raw, whole_line, offset_key, offset_len, src_pos, time, time_ns, pitch,
                            tkey, tkey_len, enable_ns);
    if (why)
        return refuse(why, err, err_cap);
    static LcTsConf conf;
    memset(&conf, 0, sizeof conf);
    if (lc_ts_compile(fmt, fmt_len, conf, &why) != 0)
        return refuse(why, err, err_cap);
    conf.source_year = source_year;
    conf.adjust = adjust;
    lc_ts_probe_zone(conf);
    const LcTsNow tn{now, now_tm[0], now_tm[1], now_tm[2], discard_interval};
    for (uint64_t i = 0; i < n; ++i)
        lc_split_regex_ts_value(ch.c, ch.t, row(ch, off, len, status, cap_off, cap_len, pitch, i), &val_off[i],
                                &val_len[i]);
    const LcTsSpans sp{val_off, val_len, nullptr, 1};
    std::vector<LcTsFull> full(n);
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t o, l;
        if (sp.get(i, o, l))
            full[i] = lc_ts_full(conf, tn, src + o, l);
    }
    std::vector<int64_t> sec(n);
    std::vector<uint32_t> nsec(n);
    uint64_t tcnt[5] = {0, 0, 0, 0, 0}; // the passes' own counters: the chain takes its from the verdicts
    static LcTsWarp w;
    lc_ts_resolve(conf, tn, src, sp, full.data(), 0, n, sec.data(), nsec.data(), ts_status, tcnt, w, 0, nlanes);
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const LcSplitRegexSlsRow r = row(ch, off, len, status, cap_off, cap_len, pitch, i);
        const LcSplitRegexTsTime tm = lc_split_regex_ts_time(ch.c, ch.t, ts_status[i], sec[i], nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_regex_sls_body(ch.c, src, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const uint32_t bits = lc_split_regex_ts_verdict(ch.c, r.status, ts_status[i]);
        for (uint32_t k = 0; k < LC_SRTS_COUNTERS; ++k)
            counters[k] += (bits >> k) & 1u;
    }
    if (total > out_cap)
        return (int64_t)total;
    uint64_t o = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (!body[i])
            continue;
        const LcSplitRegexTsTime tm = lc_split_regex_ts_time(ch.c, ch.t, ts_status[i], sec[i], nsec[i]);
        uint8_t h[6];
        h[0] = 0x0A;
        const uint32_t hn = 1 + lc_put_varint(h + 1, body[i]), rec = hn + body[i];
        memcpy(out + o, h, hn);
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, hn, rec, lane, nlanes};
            lc_split_regex_sls_body(ch.c, src, row(ch, off, len, status, cap_off, cap_len, pitch, i), tm.time,
                                    tm.has_ns, tm.ns, s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
