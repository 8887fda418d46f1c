// lc_regex_sls_emul.cpp -- TEST-ONLY host build of the regex-fed SLS serialiser's per-row function
// (loongcollector_b200/csrc/lc_exec.cuh: lc_regex_sls_setup + lc_regex_sls_body), the statements the size and emit
// kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Tables as lc_regex_parse returns them (cap_off relative to base, rows of `pitch`); status / cap tables may be NULL
// in whole-line mode.  The writing pass runs `nlanes` lanes one after the other, as the lanes of the emit kernel's warp
// share a record.  counters[3] += successful, failed, discarded, as the size kernel counts them.  Returns the total
// size (out written when it fits out_cap), -1 when the arguments are refused (err = why), -2 when a record's writer
// did not end exactly at the size the counting pass gave it.
int64_t emul_regex_sls(const uint8_t* base, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                       const uint8_t* status, const uint32_t* cap_off, const uint32_t* cap_len, uint32_t pitch,
                       const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                       uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail,
                       int keep_succeed, int copy_raw, int whole_line, const uint32_t* ev_time, const uint32_t* ev_ns,
                       uint32_t nlanes, uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err,
                       uint32_t err_cap) {
    LcRegexSlsCfg c;
    std::vector<uint32_t> plan(3 * (size_t)nkeys + 12);
    const char* why = lc_regex_sls_setup(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len,
                                         keep_fail, keep_succeed, copy_raw, whole_line, pitch, &c, plan.data());
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    std::vector<const char*> strings(keys, keys + nkeys);
    std::vector<uint32_t> lens(key_lens, key_lens + nkeys);
    strings.insert(strings.end(), {source_key, renamed_key, "__raw_log__", "content"});
    lens.insert(lens.end(), {source_len, renamed_len, 11u, 7u});
    uint64_t kbytes = 0;
    for (uint32_t l : lens)
        kbytes += l;
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 5);
    lc_sls_key_table(strings.data(), lens.data(), nkeys + 4, kb.data(), at.data());
    c.plan = plan.data();
    c.key_at = at.data();
    c.keys = kb.data();
    auto row = [&](uint64_t i) {
        LcRegexSlsRow r;
        r.eo = ev_off[i];
        r.elen = ev_len[i];
        r.status = c.whole_line ? 0u : status[i];
        r.co = cap_off ? cap_off + i * pitch : nullptr;
        r.cl = cap_len ? cap_len + i * pitch : nullptr;
        r.time = ev_time[i];
        r.has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
        r.ns = r.has_ns ? ev_ns[i] : 0u;
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount s{0};
        const LcRegexSlsRow r = row(i);
        const uint32_t cnt = lc_regex_sls_body(c, base, r, s);
        body[i] = cnt ? s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const uint32_t v = lc_regex_sls_verdict(c, r.status);
        const bool kept = v == 0u || c.keep_fail;
        counters[0] += kept;
        counters[1] += v == 1u;
        counters[2] += !kept;
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
        memcpy(out + o, h, hn);
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, hn, rec, lane, nlanes};
            lc_regex_sls_body(c, base, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
