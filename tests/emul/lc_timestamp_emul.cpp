// lc_timestamp_emul.cpp -- TEST-ONLY host build of the timestamp parse (loongcollector_b200/csrc/lc_exec.cuh:
// lc_ts_compile, lc_ts_probe_zone, lc_ts_full, lc_ts_resolve), the statements the two kernels run, with W emulated
// lanes per warp, so that the "not gpu" tier can check them against the oracle and pin the GPU's results.  Not part of
// the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Compiles fmt into *conf (sizeof(LcTsConf) bytes) and probes the process zone.  Returns 0, or -1 with the message
// in err (256 bytes).
int emul_ts_compile(const char* fmt, uint64_t len, int32_t source_year, int32_t adjust, void* conf, char* err) {
    LcTsConf& c = *(LcTsConf*)conf;
    memset(&c, 0, sizeof c);
    const char* e = nullptr;
    if (lc_ts_compile(fmt, len, c, &e) != 0) {
        strncpy(err, e, 255);
        return -1;
    }
    c.source_year = source_year;
    c.adjust = adjust;
    lc_ts_probe_zone(c);
    return 0;
}

uint64_t emul_ts_conf_size(void) { return sizeof(LcTsConf); }

// Both passes over n events in ngroups groups (grp: ngroups + 1 starts), W lanes; now_tm = localtime_r(now)'s
// (tm_year, tm_mon, tm_mday).  counters[5] are written.
void emul_ts_parse(void* conf, const uint8_t* base, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                   const uint32_t* grp, uint64_t ngroups, int64_t now, const int32_t* now_tm, int32_t discard_interval,
                   uint32_t W, int64_t* sec, uint32_t* nsec, uint8_t* status, uint64_t* counters) {
    const LcTsConf& c = *(const LcTsConf*)conf;
    const LcTsNow t{now, now_tm[0], now_tm[1], now_tm[2], discard_interval};
    const LcTsSpans sp{ev_off, ev_len, nullptr, 1};
    std::vector<LcTsFull> full(n);
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t o, l;
        if (sp.get(i, o, l))
            full[i] = lc_ts_full(c, t, base + o, l);
    }
    static LcTsWarp w;
    memset(counters, 0, 5 * sizeof(uint64_t));
    for (uint64_t g = 0; g < ngroups; ++g)
        lc_ts_resolve(c, t, base, sp, full.data(), grp[g], grp[g + 1], sec, nsec, status, counters, w, 0, W);
}

// the full parse of one value: raw tv_sec, nsec, key length (LC_TS_KFAIL = failed)
} // extern "C"
