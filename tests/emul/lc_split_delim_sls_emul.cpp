// lc_split_delim_sls_emul.cpp -- TEST-ONLY host build of the split -> delimiter chain's per-row function
// (loongcollector_b200/csrc/lc_exec.cuh: lc_delim_sls_setup + lc_split_delim_sls_link + lc_split_delim_sls_body), the
// statements the size and emit kernels run, so that the "not gpu" tier can check them against the oracle.  Not part
// of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Piece tables over src as the splitters return them, and the delimiter tables over those pieces (f_off relative to
// src; src must keep 16 readable bytes on both sides, as the state machine reads aligned 16-byte chunks when it walks
// a wide row again).  offset_key NULL = no log.file.offset metadata.  The writing pass runs `nlanes` lanes one after
// the other, as the lanes of the emit kernel's warp share a record.  counters[4] += successful, failed, discarded,
// blank, as the size kernel counts them.  Returns the total size (out written when it fits out_cap), -1 when the
// arguments are refused (err = why), -2 when a record's writer did not end exactly at the size the counting pass gave
// it.
int64_t emul_split_delim_sls(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                             const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off,
                             const uint32_t* f_len, const uint32_t* f_dq, uint32_t max_fields, const uint8_t* sep,
                             uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                             const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_len,
                             const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                             int copy_raw, const char* offset_key, uint32_t offset_len, uint64_t src_pos, uint32_t time,
                             uint32_t time_ns, uint32_t nlanes, uint8_t* out, uint64_t out_cap, uint64_t* counters,
                             char* err, uint32_t err_cap) {
    uint64_t kbytes = (uint64_t)source_len + renamed_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 4);
    LcDelimSlsCfg d;
    LcSplitDelimSlsCfg c;
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, &d, kb.data(), at.data());
    if (!why)
        why = lc_split_delim_sls_link(d, keys, key_lens, source_key, source_len, renamed_key, renamed_len, offset_key,
                                      offset_len, src_pos, time, time_ns, &c);
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    c.d.keys = kb.data();
    c.d.key_at = at.data();
    c.okey = reinterpret_cast<const uint8_t*>(offset_key);
    auto row = [&](uint64_t i) {
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
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount64 s{0};
        const LcDelimSlsRow r = row(i);
        const uint32_t cnt = lc_split_delim_sls_body(c, src, r, s);
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcDelimSlsVerdict v = lc_delim_sls_verdict(c.d, r.status);
        counters[0] += v.ok;
        counters[1] += v.failed;
        counters[2] += v.erased;
        counters[3] += v.blank;
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
            lc_split_delim_sls_body(c, src, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
