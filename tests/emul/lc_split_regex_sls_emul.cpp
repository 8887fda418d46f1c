// lc_split_regex_sls_emul.cpp -- TEST-ONLY host build of the split -> regex chain's per-row function
// (loongcollector_b200/csrc/lc_exec.cuh: lc_split_regex_sls_setup + lc_split_regex_sls_body), the statements the
// size and emit kernels run, so that the "not gpu" tier can check them against the oracle.  Not part of the product
// library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Piece tables over src as the splitters return them, and the regex tables over those pieces (rows of `pitch`;
// status / cap tables may be NULL in whole-line mode).  offset_key NULL = no log.file.offset metadata.  The writing
// pass runs `nlanes` lanes one after the other, as the lanes of the emit kernel's warp share a record.  counters[3] +=
// successful, failed, discarded, as the size kernel counts them.  Returns the total size (out written when it fits
// out_cap), -1 when the arguments are refused (err = why), -2 when a record's writer did not end exactly at the size
// the counting pass gave it.
int64_t emul_split_regex_sls(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                             const uint8_t* status, const uint32_t* cap_off, const uint32_t* cap_len, uint32_t pitch,
                             const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                             uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail,
                             int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
                             uint32_t offset_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, uint32_t nlanes,
                             uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    LcSplitRegexSlsCfg c;
    std::vector<uint32_t> plan(3 * (size_t)nkeys + 24);
    const char* why = lc_split_regex_sls_setup(keys, key_lens, nkeys, source_key, source_len, renamed_key,
                                               renamed_len, offset_key, offset_len, keep_fail, keep_succeed, copy_raw,
                                               whole_line, pitch, src_pos, time, time_ns, &c, plan.data());
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    std::vector<const char*> strings(keys, keys + nkeys);
    std::vector<uint32_t> lens(key_lens, key_lens + nkeys);
    strings.insert(strings.end(), {source_key, renamed_key, "__raw_log__", "content", offset_key});
    lens.insert(lens.end(), {source_len, renamed_len, 11u, 7u, offset_key ? offset_len : 0u});
    uint64_t kbytes = 0;
    for (uint32_t l : lens)
        kbytes += l;
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 6);
    lc_sls_key_table(strings.data(), lens.data(), nkeys + 5, kb.data(), at.data());
    c.x.plan = plan.data();
    c.x.key_at = at.data();
    c.x.keys = kb.data();
    auto row = [&](uint64_t i) {
        LcSplitRegexSlsRow r;
        r.po = off[i];
        r.plen = len[i];
        r.status = c.x.whole_line ? 0u : status[i];
        r.co = cap_off ? cap_off + i * pitch : nullptr;
        r.cl = cap_len ? cap_len + i * pitch : nullptr;
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount64 s{0};
        const LcSplitRegexSlsRow r = row(i);
        const uint32_t cnt = lc_split_regex_sls_body(c, src, r, s);
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcSplitRegexVerdict v = lc_split_regex_verdict(c, r.status);
        counters[0] += v.ok;
        counters[1] += v.failed;
        counters[2] += v.erased;
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
            lc_split_regex_sls_body(c, src, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
