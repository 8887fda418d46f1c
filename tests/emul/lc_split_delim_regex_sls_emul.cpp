// lc_split_delim_regex_sls_emul.cpp -- TEST-ONLY host build of the split -> delimiter -> regex -> SLS chain's per-row
// functions (loongcollector_b200/csrc/lc_exec.cuh: lc_delim_sls_setup + lc_regex_sls_setup +
// lc_split_delim_regex_sls_link, the tap rule lc_delim_regex_tap / lc_delim_regex_copy over the piece tables, the row
// function lc_split_delim_regex_sls_body and lc_split_delim_regex_verdict), the statements the tap, size and emit
// kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

struct Chain {
    LcSplitDelimRegexSlsCfg c;
    std::vector<uint8_t> dkb, rkb;
    std::vector<uint32_t> dat, rat, plan;
};

#define EMUL_CFG_PARAMS                                                                                                \
    const uint8_t *sep, uint32_t sep_len, uint8_t quote, int extend, int discard, const char *const *keys,             \
        const uint32_t *key_lens, uint32_t nkeys, const char *source_key, uint32_t source_len,                         \
        const char *renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed, int copy_raw,                  \
        const char *const *rkeys, const uint32_t *rkey_lens, uint32_t rnkeys, const char *rsource,                     \
        uint32_t rsource_len, const char *rrenamed, uint32_t rrenamed_len, int rkeep_fail, int rkeep_succeed,          \
        int rcopy_raw, int whole_line, uint32_t pitch, const char *offset_key, uint32_t offset_len, uint64_t src_pos,  \
        uint32_t time, uint32_t time_ns
#define EMUL_CFG_ARGS                                                                                                  \
    sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len,     \
        keep_fail, keep_succeed, copy_raw, rkeys, rkey_lens, rnkeys, rsource, rsource_len, rrenamed, rrenamed_len,     \
        rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, pitch, offset_key, offset_len, src_pos, time, time_ns

// 0, or -1 with err = why the configuration is refused
int setup(Chain& ch, uint32_t max_fields, EMUL_CFG_PARAMS, char* err, uint32_t err_cap) {
    uint64_t kbytes = (uint64_t)source_len + renamed_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    ch.dkb.assign(kbytes + 1, 0);
    ch.dat.assign(nkeys + 4, 0);
    memset(&ch.c, 0, sizeof ch.c);
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, &ch.c.r.d, ch.dkb.data(), ch.dat.data());
    ch.plan.assign(3 * (size_t)rnkeys + 12, 0);
    if (!why)
        why = lc_regex_sls_setup(rkeys, rkey_lens, rnkeys, rsource, rsource_len, rrenamed, rrenamed_len, rkeep_fail,
                                 rkeep_succeed, rcopy_raw, whole_line, pitch, &ch.c.r.x, ch.plan.data());
    if (!why) {
        ch.c.r.d.keys = ch.dkb.data();
        ch.c.r.d.key_at = ch.dat.data();
        why = lc_split_delim_regex_sls_link(keys, key_lens, source_key, source_len, renamed_key, renamed_len, rkeys,
                                            rkey_lens, rnkeys, rsource, rsource_len, rrenamed, rrenamed_len,
                                            rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, offset_key, offset_len,
                                            src_pos, time, time_ns, &ch.c);
    }
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
    ch.c.r.x.keys = ch.rkb.data();
    ch.c.r.x.key_at = ch.rat.data();
    ch.c.r.x.plan = ch.plan.data();
    ch.c.s.okey = reinterpret_cast<const uint8_t*>(offset_key);
    return 0;
}

// piece i and its delimiter row, with the source event's time and ns (as the kernels' split_delim_sls_row)
LcDelimSlsRow piece_row(const LcSplitDelimRegexSlsCfg& c, const uint32_t* off, const uint32_t* len,
                        const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off, const uint32_t* f_len,
                        const uint32_t* f_dq, uint64_t i) {
    const uint32_t mf = c.r.d.max_fields;
    LcDelimSlsRow r;
    r.eo = off[i];
    r.elen = len[i];
    r.status = status[i];
    r.nf = nfields[i];
    r.fo = f_off + i * mf;
    r.fl = f_len + i * mf;
    r.fd = f_dq + i * mf;
    r.time = c.s.time;
    r.has_ns = c.s.has_ns;
    r.ns = c.s.ns;
    return r;
}

} // namespace

extern "C" {

// The tap over the piece tables: val_off / val_len of every piece, and the collapsed copies in src[side_at, ...) in
// piece order (the kernels' exclusive sum over the copy sizes).  Returns the side bytes used, or -1 (err = why the
// chain is refused).
int64_t emul_split_delim_regex_tap(uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                                   const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                                   const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, EMUL_CFG_PARAMS,
                                   uint64_t side_at, uint32_t* val_off, uint32_t* val_len, char* err,
                                   uint32_t err_cap) {
    Chain ch;
    if (setup(ch, max_fields, EMUL_CFG_ARGS, err, err_cap))
        return -1;
    uint64_t at = side_at;
    for (uint64_t i = 0; i < n; ++i) {
        const LcDelimSlsRow r = piece_row(ch.c, off, len, status, nfields, f_off, f_len, f_dq, i);
        const LcDrTap t = lc_delim_regex_tap(ch.c.r, r);
        val_off[i] = t.copy ? (uint32_t)at : t.off;
        val_len[i] = t.len;
        if (t.copy) {
            lc_delim_regex_copy(ch.c.r, src, r, src + at, t.copy);
            at += t.copy;
        }
    }
    return (int64_t)(at - side_at);
}

// The wire bytes, with counters[8] as lc_delim_regex_verdict orders them (the size kernel's verdicts).  The writing
// pass runs `nlanes` lanes one after the other, as the lanes of the emit kernel's warp share a record.  Returns the
// total size (out written when it fits out_cap), -1 when the configuration is refused, -2 when a record's writer did not
// end exactly at the size the counting pass gave it.
int64_t emul_split_delim_regex_sls(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                                   const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                                   const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, EMUL_CFG_PARAMS,
                                   const uint32_t* val_off, const uint32_t* val_len, const uint8_t* re_status,
                                   const uint32_t* cap_off, const uint32_t* cap_len, uint32_t nlanes, uint8_t* out,
                                   uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    Chain ch;
    if (setup(ch, max_fields, EMUL_CFG_ARGS, err, err_cap))
        return -1;
    auto row = [&](uint64_t i) {
        LcDelimRegexSlsRow r;
        r.d = piece_row(ch.c, off, len, status, nfields, f_off, f_len, f_dq, i);
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
        LcSlsCount64 s{0};
        const uint32_t cnt = lc_split_delim_regex_sls_body(ch.c, src, r, s);
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcDelimRegexVerdict v = lc_split_delim_regex_verdict(ch.c, r, cnt);
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
            lc_split_delim_regex_sls_body(ch.c, src, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
