// lc_delim_sls_emul.cpp -- TEST-ONLY host build of the delimiter-fed SLS serialiser's per-row function
// (loongcollector_b200/csrc/lc_exec.cuh: lc_delim_sls_setup + lc_delim_sls_body), the statements the size and emit
// kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Tables as lc_delim_parse returns them (f_off relative to base).  base must keep 16 readable bytes on both sides (the
// state machine reads aligned 16-byte chunks when it walks a wide row again).  The writing pass runs `nlanes` lanes
// one after the other, as the lanes of the emit kernel's warp share a record.  Returns the total size (out written
// when it fits out_cap), -1 when the configuration is refused (err = why), -2 when a record's writer did not end
// exactly at the size the counting pass gave it.
int64_t emul_delim_sls(const uint8_t* base, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                       const uint8_t* status, const uint32_t* nfields, const uint32_t* f_off, const uint32_t* f_len,
                       const uint32_t* f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                       int extend, int discard, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                       const char* source_key, uint32_t source_len, const char* renamed_key, uint32_t renamed_len,
                       int keep_fail, int keep_succeed, int copy_raw, const uint32_t* ev_time, const uint32_t* ev_ns,
                       uint32_t nlanes, uint8_t* out, uint64_t out_cap, char* err, uint32_t err_cap) {
    uint64_t kbytes = (uint64_t)source_len + renamed_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 4);
    LcDelimSlsCfg c;
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, &c, kb.data(), at.data());
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    c.keys = kb.data();
    c.key_at = at.data();
    auto row = [&](uint64_t i) {
        LcDelimSlsRow r;
        r.eo = ev_off[i];
        r.elen = ev_len[i];
        r.status = status[i];
        r.nf = nfields[i];
        r.fo = f_off + i * max_fields;
        r.fl = f_len + i * max_fields;
        r.fd = f_dq + i * max_fields;
        r.time = ev_time[i];
        r.has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
        r.ns = r.has_ns ? ev_ns[i] : 0u;
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount s{0};
        const uint32_t cnt = lc_delim_sls_body(c, base, row(i), s);
        body[i] = cnt ? s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
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
            lc_delim_sls_body(c, base, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
