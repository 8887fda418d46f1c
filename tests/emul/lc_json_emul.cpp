// lc_json_emul.cpp -- TEST-ONLY host build of the JSON parse (loongcollector_b200/csrc/lc_exec.cuh: lc_json_count,
// lc_json_emit and the walk under them), in the kernels' order: the fast count pass, the slow count pass over the
// compacted slow events, the two exclusive sums, the fast and slow emit passes.  W emulated lanes per warp only change
// the order in which slow events are appended to the list (each warp's lanes last to first), which no output may
// depend on.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// status[n], first[n + 1], counters[3] are written; entries (4 words each) and arena bytes only when both totals fit.
// Returns 0, or 7 when an emit pass would have left its event's ranges; *n_slow receives the slow-event count.
int emul_json_parse(const uint8_t* skey, uint32_t sklen, const uint8_t* base, const uint32_t* ev_off,
                    const uint32_t* ev_len, uint64_t n, uint32_t W, uint8_t* status, uint64_t* first, uint32_t* ent,
                    uint64_t ent_cap, uint64_t* n_ent, uint8_t* arena, uint64_t arena_cap, uint64_t* n_arena,
                    uint64_t* counters, uint64_t* n_slow) {
    std::vector<uint32_t> nent(n), narena(n), list;
    std::vector<uint8_t> slow(n);
    memset(counters, 0, 3 * sizeof(uint64_t));
    auto count = [&](uint32_t st) {
        const uint32_t s = st & 0x7Fu;
        counters[0] += s == LC_JSON_ST_NOT_FOUND;
        counters[1] += s == LC_JSON_ST_FAILED;
        counters[2] += s == LC_JSON_ST_OK;
    };
    for (uint64_t w0 = 0; w0 < n; w0 += W) {
        const uint64_t w1 = w0 + W < n ? w0 + W : n;
        for (uint64_t i = w1; i-- > w0;) {
            bool sl;
            const uint32_t st = lc_json_count<false>(base, ev_len[i] == LC_JSON_NO_KEY ? 0u : ev_off[i], ev_len[i],
                                                     skey, sklen, lc_json_pow5, &nent[i], &narena[i], &sl);
            status[i] = (uint8_t)st;
            slow[i] = sl;
            if (sl)
                list.push_back((uint32_t)i);
            else
                count(st);
        }
    }
    for (uint32_t i : list) {
        bool sl;
        const uint32_t st = lc_json_count<true>(base, ev_off[i], ev_len[i], skey, sklen, lc_json_pow5, &nent[i], &narena[i], &sl);
        status[i] = (uint8_t)st;
        count(st);
    }
    *n_slow = list.size();
    std::vector<uint64_t> afirst(n + 1);
    uint64_t e = 0, a = 0;
    for (uint64_t i = 0; i < n; ++i) {
        first[i] = e;
        afirst[i] = a;
        e += nent[i];
        a += narena[i];
    }
    first[n] = *n_ent = e;
    afirst[n] = *n_arena = a;
    if (e > ent_cap || a > arena_cap)
        return 0;
    int rc = 0;
    auto emit = [&](uint64_t i, bool s) {
        LcJsonEntry* en = reinterpret_cast<LcJsonEntry*>(ent) + first[i];
        const uint32_t ec = (uint32_t)(first[i + 1] - first[i]), ac = (uint32_t)(afirst[i + 1] - afirst[i]);
        const bool ok = s ? lc_json_emit<true>(base, ev_off[i], ev_len[i], skey, sklen, lc_json_pow5, en, ec, arena + afirst[i],
                                               (uint32_t)afirst[i], ac)
                          : lc_json_emit<false>(base, ev_off[i], ev_len[i], skey, sklen, lc_json_pow5, en, ec, arena + afirst[i],
                                                (uint32_t)afirst[i], ac);
        if (!ok)
            rc = 7;
    };
    for (uint64_t i = 0; i < n; ++i)
        if (!slow[i] && (status[i] & 0x7Fu) == LC_JSON_ST_OK)
            emit(i, false);
    for (uint32_t i : list)
        if ((status[i] & 0x7Fu) == LC_JSON_ST_OK)
            emit(i, true);
    return rc;
}

} // extern "C"
