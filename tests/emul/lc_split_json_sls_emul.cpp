// lc_split_json_sls_emul.cpp -- TEST-ONLY host build of the split -> JSON chain's resolve and row functions
// (loongcollector_b200/csrc/lc_exec.cuh: lc_split_json_sls_setup, lc_json_resolve_warp / lc_json_resolve_sort,
// lc_split_json_sls_body), the statements the resolve, size and emit kernels run, so that the "not gpu" tier can check
// them against the oracle.  The resolve picks its path from the member count alone, as the kernels do.  Not part of
// the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

// every key in one hash bucket: the resolve must still split keys by their bytes, in O(m log m) comparisons
struct ConstHash {
    uint32_t operator()(const uint8_t*, uint32_t) const { return 7u; }
};

template <class H>
int64_t run(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n, const uint8_t* status,
            const uint64_t* first, const LcJsonEntry* ent, const uint8_t* arena, const char* source_key,
            uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
            int copy_raw, const char* offset_key, uint32_t offset_len, uint64_t src_pos, uint32_t time,
            uint32_t time_ns, uint32_t nlanes, uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err,
            uint32_t err_cap) {
    LcSplitJsonSlsCfg c;
    const char* why = lc_split_json_sls_setup(source_key, source_len, renamed_key, renamed_len, offset_key, offset_len,
                                              keep_fail, keep_succeed, copy_raw, src_pos, time, time_ns, &c);
    if (why) {
        strncpy(err, why, err_cap - 1);
        err[err_cap - 1] = 0;
        return -1;
    }
    const uint64_t m_all = first[n];
    std::vector<uint32_t> win(m_all + 1), scratch(3 * m_all + 3);
    std::vector<LcJsonSlsEv> ev(n);
    auto members = [&](uint64_t i) {
        return (status[i] & 0x7Fu) == LC_JSON_ST_OK ? (uint32_t)(first[i + 1] - first[i]) : 0u;
    };
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t m = members(i);
        const uint64_t f = first[i];
        if (m <= LC_JSON_SLS_WARP) {
            LcJsonResolveWarp w;
            lc_json_resolve_warp<H>(c, src, arena, ent + f, m, win.data() + f, &ev[i], w, 0u);
        } else {
            lc_json_resolve_sort<H>(c, src, arena, ent + f, m, win.data() + f, &ev[i], scratch.data() + f,
                                    scratch.data() + m_all + f, scratch.data() + 2 * m_all + f);
        }
    }
    auto row = [&](uint64_t i) {
        LcSplitJsonSlsRow r;
        r.po = off[i];
        r.plen = len[i];
        r.status = status[i];
        r.e = ent + first[i];
        r.win = win.data() + first[i];
        r.m = members(i);
        r.ev = ev[i];
        return r;
    };
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        LcSlsCount64 s{0};
        const LcSplitJsonSlsRow r = row(i);
        const uint32_t cnt = lc_split_json_sls_body(c, src, arena, r, s);
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcSplitRegexVerdict v = lc_split_json_verdict(c, r.status);
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
        for (uint32_t lane = 0; lane < nlanes; ++lane) {
            LcSlsWrite s{out + o, 0u, rec, lane, nlanes};
            s.put(h, hn);
            lc_split_json_sls_body(c, src, arena, row(i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}

} // namespace

extern "C" {

// Piece tables over src as the splitters return them, and the tables of lc_json_parse over those pieces (entries of
// 4 words).  offset_key NULL = no log.file.offset metadata; time_ns 0xFFFFFFFF = no Time_ns.  The writing pass runs
// `nlanes` lanes one after the other, as the lanes of the emit kernel's warp share a record; const_hash resolves with
// every key hashed alike.  counters[3] += successful, failed, discarded.  Returns the total size (out written when it
// fits out_cap), -1 when the arguments are refused (err = why), -2 when a record's writer did not end exactly at the
// size the counting pass gave it.
int64_t emul_split_json_sls(const uint8_t* src, const uint32_t* off, const uint32_t* len, uint64_t n,
                            const uint8_t* status, const uint64_t* first, const uint32_t* ent, const uint8_t* arena,
                            const char* source_key, uint32_t source_len, const char* renamed_key, uint32_t renamed_len,
                            int keep_fail, int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_len,
                            uint64_t src_pos, uint32_t time, uint32_t time_ns, uint32_t nlanes, int const_hash,
                            uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    const LcJsonEntry* e = reinterpret_cast<const LcJsonEntry*>(ent);
    return const_hash ? run<ConstHash>(src, off, len, n, status, first, e, arena, source_key, source_len, renamed_key,
                                       renamed_len, keep_fail, keep_succeed, copy_raw, offset_key, offset_len, src_pos,
                                       time, time_ns, nlanes, out, out_cap, counters, err, err_cap)
                      : run<LcJsonKeyHash>(src, off, len, n, status, first, e, arena, source_key, source_len,
                                           renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw, offset_key,
                                           offset_len, src_pos, time, time_ns, nlanes, out, out_cap, counters, err,
                                           err_cap);
}

} // extern "C"
