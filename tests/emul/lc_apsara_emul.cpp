// lc_apsara_emul.cpp -- TEST-ONLY host build of the Apsara parse (loongcollector_b200/csrc/lc_exec.cuh: lc_ap_scan,
// lc_ap_resolve, lc_ap_fields), the statements the three kernels run, with W emulated lanes per warp, so that the
// "not gpu" tier can check them against the oracle and pin the GPU's results.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// The three passes over n events in ngroups groups (grp: ngroups + 1 starts), W lanes, the process zone probed here.
// first[n + 1] is the exclusive sum of the parsed events' entry counts; entries (4 words each) are written only when
// they fit in ent_cap.  counters[5] are written.
void emul_apsara_parse(int32_t adjust, const uint8_t* skey, uint32_t sklen, const uint8_t* base, uint64_t base_len,
                       const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* grp,
                       uint64_t ngroups, int64_t now, int32_t discard_interval, uint32_t W, uint8_t* status,
                       int64_t* sec, uint32_t* nsec, int64_t* micro, uint64_t* first, uint32_t* ent, uint64_t ent_cap,
                       uint64_t* n_ent, uint64_t* counters) {
    static LcTsConf c;
    memset(&c, 0, sizeof c);
    c.adjust = adjust;
    lc_ts_probe_zone(c);
    LcTsNow t;
    memset(&t, 0, sizeof t);
    t.now = now;
    t.discard_interval = discard_interval;
    std::vector<LcApEv> ev(n);
    for (uint64_t i = 0; i < n; ++i)
        ev[i] = lc_ap_scan(c, base, base_len, ev_len[i] == LC_AP_NO_KEY ? 0u : ev_off[i], ev_len[i], skey, sklen);
    std::vector<uint32_t> nent(n);
    LcApWarp w;
    memset(counters, 0, 5 * sizeof(uint64_t));
    for (uint64_t g = 0; g < ngroups; ++g)
        lc_ap_resolve(t, ev.data(), grp[g], grp[g + 1], status, sec, nsec, micro, nent.data(), counters, w, 0, W);
    uint64_t run = 0;
    for (uint64_t i = 0; i < n; ++i) {
        first[i] = run;
        run += nent[i];
    }
    first[n] = run;
    *n_ent = run;
    if (run > ent_cap)
        return;
    for (uint64_t i = 0; i < n; ++i) {
        if ((status[i] & 7u) != LC_AP_ST_OK)
            continue;
        LcApEmit em{reinterpret_cast<LcApEntry*>(ent) + first[i], ev_off[i]};
        lc_ap_fields(base + ev_off[i], ev_len[i], em);
    }
}

} // extern "C"
