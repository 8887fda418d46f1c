// lc_split_regex_filter_sls_emul.cpp -- TEST-ONLY host build of the split -> regex -> filter chain's per-row functions
// (loongcollector_b200/csrc/lc_exec.cuh: lc_split_regex_sls_setup, lc_filter_sls_setup, lc_filter_leaf,
// lc_filter_eval and lc_split_regex_sls_body), the statements the tap, eval, size and emit kernels run, so that the
// "not gpu" tier can check them against the oracle.  The boolean match between the tap and the eval is the caller's.
// Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

namespace {

struct Chain {
    LcSplitRegexSlsCfg c;
    LcFilterSlsCfg f;
    std::vector<uint32_t> plan, at;
    std::vector<uint8_t> kb;
};

// the chain's and the filter's configuration, as the C-ABI builds them; nullptr or why they are refused
const char* setup(Chain& ch, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                  uint32_t source_len, const char* renamed_key, uint32_t renamed_len, int keep_fail, int keep_succeed,
                  int copy_raw, int whole_line, const char* offset_key, uint32_t offset_len, uint64_t src_pos,
                  uint32_t time, uint32_t time_ns, uint32_t pitch, uint32_t nleaves, const char* const* leaf_keys,
                  const uint32_t* leaf_lens, uint32_t nprog, const uint32_t* prog) {
    ch.plan.assign(3 * (size_t)nkeys + 24, 0);
    const char* why = lc_split_regex_sls_setup(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len,
                                               offset_key, offset_len, keep_fail, keep_succeed, copy_raw, whole_line,
                                               pitch, src_pos, time, time_ns, &ch.c, ch.plan.data());
    if (why)
        return why;
    std::vector<const char*> strings(keys, keys + nkeys);
    std::vector<uint32_t> lens(key_lens, key_lens + nkeys);
    strings.insert(strings.end(), {source_key, renamed_key, "__raw_log__", "content", offset_key});
    lens.insert(lens.end(), {source_len, renamed_len, 11u, 7u, offset_key ? offset_len : 0u});
    why = lc_filter_sls_setup(ch.plan.data(), ch.c.x.n_ok, ch.c.x.n_fail, strings.data(), lens.data(), nleaves,
                              leaf_keys, leaf_lens, nprog, prog, &ch.f);
    if (why)
        return why;
    uint64_t kbytes = 0;
    for (uint32_t l : lens)
        kbytes += l;
    ch.kb.assign(kbytes + 1, 0);
    ch.at.assign(nkeys + 6, 0);
    lc_sls_key_table(strings.data(), lens.data(), nkeys + 5, ch.kb.data(), ch.at.data());
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

#define EMUL_CHAIN_PARAMS                                                                                              \
    const uint32_t *off, const uint32_t *len, uint64_t n, const uint8_t *status, const uint32_t *cap_off,              \
        const uint32_t *cap_len, uint32_t pitch, const char *const *keys, const uint32_t *key_lens, uint32_t nkeys,    \
        const char *source_key, uint32_t source_len, const char *renamed_key, uint32_t renamed_len, int keep_fail,     \
        int keep_succeed, int copy_raw, int whole_line, const char *offset_key, uint32_t offset_len, uint64_t src_pos, \
        uint32_t time, uint32_t time_ns, uint32_t nleaves, const char *const *leaf_keys, const uint32_t *leaf_lens,    \
        uint32_t nprog, const uint32_t *prog
#define EMUL_SETUP_ARGS                                                                                                \
    keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len, keep_fail, keep_succeed, copy_raw,        \
        whole_line, offset_key, offset_len, src_pos, time, time_ns, pitch, nleaves, leaf_keys, leaf_lens, nprog, prog

extern "C" {

// The tap: for every leaf l and row i, src[l * n + i] = the value source (lc_filter_leaf), off / len its value in the
// source value, or (source LC_REGEX_SLS_DIGITS) its digits written at dig + 20 i as the tap kernel writes them.
// Returns 0, or -1 when the chain or the filter is refused (err = why).
int emul_filter_tap(EMUL_CHAIN_PARAMS, uint32_t* src, uint32_t* voff, uint32_t* vlen, uint8_t* dig, char* err,
                    uint32_t err_cap) {
    Chain ch;
    const char* why = setup(ch, EMUL_SETUP_ARGS);
    if (why)
        return refuse(why, err, err_cap);
    for (uint32_t l = 0; l < nleaves; ++l)
        for (uint64_t i = 0; i < n; ++i) {
            const LcSplitRegexSlsRow r = row(ch, off, len, status, cap_off, cap_len, pitch, i);
            uint32_t o, vl;
            const uint32_t s = lc_filter_leaf(ch.c, ch.f, l, r, &o, &vl);
            src[l * n + i] = s;
            voff[l * n + i] = o;
            vlen[l * n + i] = vl;
            if (s == LC_REGEX_SLS_DIGITS)
                for (uint32_t j = 0; j < vl; ++j)
                    dig[i * LC_FILTER_SLS_DIGIT_PITCH + j] = lc_dec_digit(ch.c.src_pos + r.po, j, vl);
        }
    return 0;
}

// The eval and the records: m = the match bytes ([l * n + i] over the source value, [(nleaves + l) * n + i] over the
// digits), the eval kernel's verdict per row, then the kept rows' records with `nlanes` lanes one after the other.
// counters[4] += successful, failed, discarded, removed by the filter.  Returns the total size (out written when it
// fits out_cap), -1 when refused, -2 when a record's writer did not end at the size the counting pass gave it.
int64_t emul_split_regex_filter_sls(const uint8_t* src, EMUL_CHAIN_PARAMS, const uint8_t* m, uint32_t nlanes,
                                    uint8_t* out, uint64_t out_cap, uint64_t* counters, char* err, uint32_t err_cap) {
    Chain ch;
    const char* why = setup(ch, EMUL_SETUP_ARGS);
    if (why)
        return refuse(why, err, err_cap);
    std::vector<uint32_t> body(n);
    uint64_t total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const LcSplitRegexSlsRow r = row(ch, off, len, status, cap_off, cap_len, pitch, i);
        bool reached, empty;
        lc_filter_row_state(ch.c, ch.f, r.status, &reached, &empty);
        uint32_t bits = 0;
        for (uint32_t l = 0; l < nleaves; ++l) {
            const uint32_t s = lc_filter_leaf_src(ch.c, ch.f, l, r.status);
            if (s != LC_FILTER_SLS_ABSENT)
                bits |= (uint32_t)m[(uint64_t)(s == LC_REGEX_SLS_DIGITS ? nleaves + l : l) * n + i] << l;
        }
        const uint32_t keep = reached ? lc_filter_eval(ch.f, bits, empty) : 0u;
        counters[3] += reached && !keep;
        LcSlsCount64 s{0};
        const uint32_t cnt = keep ? lc_split_regex_sls_body(ch.c, src, r, s) : 0u;
        body[i] = cnt ? (uint32_t)s.n : 0u;
        total += cnt ? 1 + lc_varint_size(body[i]) + body[i] : 0u;
        const LcSplitRegexVerdict v = lc_split_regex_verdict(ch.c, r.status);
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
            lc_split_regex_sls_body(ch.c, src, row(ch, off, len, status, cap_off, cap_len, pitch, i), s);
            if (s.at != rec)
                return -2;
        }
        o += rec;
    }
    return (int64_t)total;
}
}
