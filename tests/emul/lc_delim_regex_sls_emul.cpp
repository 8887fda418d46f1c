// lc_delim_regex_sls_emul.cpp -- TEST-ONLY host build of the delimiter -> regex -> SLS chain's per-row functions
// (loongcollector_b200/csrc/lc_exec.cuh: lc_delim_sls_setup + lc_regex_sls_setup + lc_delim_regex_sls_link, the tap
// rule lc_delim_regex_tap / lc_delim_regex_copy and the row function lc_delim_regex_sls_body), the statements the tap,
// size and emit kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product
// library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

struct Chain {
    LcDelimRegexSlsCfg c;
    std::vector<uint8_t> dkb, rkb;
    std::vector<uint32_t> dat, rat, plan;
};

// 0, or -1 with err = why the configuration is refused
int setup(Chain& ch, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
          const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
          uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
          int copy_raw, uint32_t max_fields, const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
          const char* rsource, uint32_t rsource_len, const char* rrenamed, uint32_t rrenamed_len, int rkeep_fail,
          int rkeep_succeed, int rcopy_raw, int whole_line, uint32_t pitch, char* err, uint32_t err_cap) {
    uint64_t kbytes = (uint64_t)source_len + renamed_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    ch.dkb.assign(kbytes + 1, 0);
    ch.dat.assign(nkeys + 4, 0);
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, &ch.c.d, ch.dkb.data(), ch.dat.data());
    ch.plan.assign(3 * (size_t)rnkeys + 12, 0);
    if (!why)
        why = lc_regex_sls_setup(rkeys, rkey_lens, rnkeys, rsource, rsource_len, rrenamed, rrenamed_len, rkeep_fail,
                                 rkeep_succeed, rcopy_raw, whole_line, pitch, &ch.c.x, ch.plan.data());
    if (!why)
        why = lc_delim_regex_sls_link(ch.c.d, keys, key_lens, source_key, source_len, renamed_key, renamed_len, rkeys,
                                      rkey_lens, rnkeys, rsource, rsource_len, rrenamed, rrenamed_len, rkeep_fail,
                                      rkeep_succeed, rcopy_raw, whole_line, &ch.c);
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    std::vector<const char*> strings(rkeys, rkeys + rnkeys);
    std::vector<uint32_t> lens(rkey_lens, rkey_lens + rnkeys);
    strings.insert(strings.end(), {rsource, rrenamed, "__raw_log__", "content"});
    lens.insert(lens.end(), {rsource_len, rrenamed_len, 11u, 7u});
    uint64_t rb = 0;
    for (uint32_t l : lens)
        rb += l;
    ch.rkb.assign(rb + 1, 0);
    ch.rat.assign(rnkeys + 5, 0);
    lc_sls_key_table(strings.data(), lens.data(), rnkeys + 4, ch.rkb.data(), ch.rat.data());
    ch.c.d.keys = ch.dkb.data();
    ch.c.d.key_at = ch.dat.data();
    ch.c.x.keys = ch.rkb.data();
    ch.c.x.key_at = ch.rat.data();
    ch.c.x.plan = ch.plan.data();
    return 0;
}

LcDelimSlsRow delim_row(const uint32_t* ev_off, const uint32_t* ev_len, const uint8_t* status, const uint32_t* nfields,
                        const uint32_t* f_off, const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields,
                        const uint32_t* ev_time, const uint32_t* ev_ns, uint64_t i) {
    LcDelimSlsRow r;
    r.eo = ev_off[i];
    r.elen = ev_len[i];
    r.status = status[i];
    r.nf = nfields[i];
    r.fo = f_off + i * max_fields;
    r.fl = f_len + i * max_fields;
    r.fd = f_dq + i * max_fields;
    r.time = ev_time ? ev_time[i] : 0u;
    r.has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
    r.ns = r.has_ns ? ev_ns[i] : 0u;
    return r;
}

} // namespace

extern "C" {

// The tap: val_off / val_len of every row, and the collapsed copies in base[side_at, ...) in row order (the kernels'
// exclusive sum over the copy sizes).  Returns the side bytes used, or -1 (err = why the chain is refused).  A row's
// copy is written exactly to its counted size, else -2.
int64_t emul_delim_regex_tap(uint8_t* base, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                             const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                             const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, const uint8_t* sep,
                             uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                             const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_len,
                             const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                             int copy_raw, const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                             const char* rsource, uint32_t rsource_len, const char* rrenamed, uint32_t rrenamed_len,
                             int rkeep_fail, int rkeep_succeed, int rcopy_raw, int whole_line, uint32_t pitch,
                             uint32_t side_at, uint32_t* val_off, uint32_t* val_len, char* err, uint32_t err_cap) {
    Chain ch;
    if (setup(ch, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key, source_len, renamed_key,
              renamed_len, keep_fail, keep_succeed, copy_raw, max_fields, rkeys, rkey_lens, rnkeys, rsource,
              rsource_len, rrenamed, rrenamed_len, rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, pitch, err,
              err_cap))
        return -1;
    uint64_t at = side_at;
    for (uint64_t i = 0; i < n; ++i) {
        const LcDelimSlsRow r =
            delim_row(ev_off, ev_len, status, nfields, f_off, f_len, f_dq, max_fields, nullptr, nullptr, i);
        const LcDrTap t = lc_delim_regex_tap(ch.c, r);
        val_off[i] = t.copy ? (uint32_t)at : t.off;
        val_len[i] = t.len;
        if (t.copy) {
            lc_delim_regex_copy(ch.c, base, r, base + at, t.copy);
            at += t.copy;
        }
    }
    return (int64_t)(at - side_at);
}

// The wire bytes, with counters[8] = the delimiter's successful, failed, discarded, blank and the regex stage's
// successful, failed, key-not-found, discarded events (the size kernel's verdicts).  The writing pass runs `nlanes`
// lanes one after the other, as the lanes of the emit kernel's warp share a record.  Returns the total size (out
// written when it fits out_cap), -1 when the configuration is refused, -2 when a record's writer did not end exactly
// at the size the counting pass gave it.
int64_t emul_delim_regex_sls(const uint8_t* base, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                             const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                             const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, const uint8_t* sep,
                             uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                             const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_len,
                             const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                             int copy_raw, const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                             const char* rsource, uint32_t rsource_len, const char* rrenamed, uint32_t rrenamed_len,
                             int rkeep_fail, int rkeep_succeed, int rcopy_raw, int whole_line, uint32_t pitch,
                             const uint32_t* val_off, const uint32_t* val_len, const uint8_t* re_status,
                             const uint32_t* cap_off, const uint32_t* cap_len, const uint32_t* ev_time,
                             const uint32_t* ev_ns, uint32_t nlanes, uint8_t* out, uint64_t out_cap, uint64_t* counters,
                             char* err, uint32_t err_cap) {
    Chain ch;
    if (setup(ch, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key, source_len, renamed_key,
              renamed_len, keep_fail, keep_succeed, copy_raw, max_fields, rkeys, rkey_lens, rnkeys, rsource,
              rsource_len, rrenamed, rrenamed_len, rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, pitch, err,
              err_cap))
        return -1;
    auto row = [&](uint64_t i) {
        LcDelimRegexSlsRow r;
        r.d = delim_row(ev_off, ev_len, status, nfields, f_off, f_len, f_dq, max_fields, ev_time, ev_ns, i);
        r.vo = val_off[i];
        r.vl = val_len[i];
        r.status = re_status ? re_status[i] : 0u;
        r.co = cap_off ? cap_off + i * pitch : nullptr;
        r.cl = cap_len ? cap_len + i * pitch : nullptr;
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    memset(counters, 0, 8 * sizeof(uint64_t));
    for (uint64_t i = 0; i < n; ++i) {
        const LcDelimRegexSlsRow r = row(i);
        LcSlsCount s{0};
        const uint32_t cnt = lc_delim_regex_sls_body(ch.c, base, r, s);
        body[i] = cnt ? s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcDelimRegexVerdict v = lc_delim_regex_verdict(ch.c, r, cnt);
        for (uint32_t k = 0; k < 8; ++k)
            counters[k] += v.ctr[k];
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
            lc_delim_regex_sls_body(ch.c, base, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
