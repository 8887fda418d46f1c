// Driver around the reference's own strptime_ns (core/common/Strptime.cpp, compiled in place by
// oracle/build_ref_strptime.sh).  It restates, in this project's words, the Strptime wrapper (TimeUtil.cpp:112-160)
// and ParseLogTime's second-level cache with ProcessEvent's verdict (ProcessorParseTimestampNative.cpp:100-235), with
// the same C interface as oracle/lc_timestamp_oracle.c's orc_ts_process.  Values are copied into NUL-padded buffers.
#include <limits.h>
#include <stdint.h>
#include <string.h>
#include <time.h>

#include <string>
#include <vector>

namespace logtail {
const char* strptime_ns(const char* buf, const char* fmt, struct tm* tm, long* nanosecond, int* nanosecondLength);
}

namespace {

const char* wrapper(const char* buf, const char* fmt, int64_t* sec, long* ns, int& nslen, int32_t year_mode,
                    time_t now) {
    struct tm tm = {};
    tm.tm_year = INT_MIN;
    const char* r = logtail::strptime_ns(buf, fmt, &tm, ns, &nslen);
    if (strcmp("%f", fmt) == 0)
        return r;
    if (year_mode >= 0 && tm.tm_year == INT_MIN) {
        if (year_mode > 0) {
            tm.tm_year = year_mode - 1900;
        } else {
            struct tm cur = {};
            localtime_r(&now, &cur);
            if (tm.tm_mon == 0 && tm.tm_mday == 1 && cur.tm_mon == 11 && cur.tm_mday == 31)
                tm.tm_year = cur.tm_year + 1;
            else if (tm.tm_mon == 11 && tm.tm_mday == 31 && cur.tm_mon == 0 && cur.tm_mday == 1)
                tm.tm_year = cur.tm_year - 1;
            else
                tm.tm_year = cur.tm_year;
        }
    }
    *sec = (int64_t)mktime(&tm);
    return r;
}

} // namespace

extern "C" void ref_ts_process(const char* fmt, int32_t year_mode, int32_t adjust, const uint8_t* base,
                               const uint32_t* off, const uint32_t* len, const uint32_t* grp, uint64_t ngroups,
                               int64_t now, int32_t discard_interval, int64_t* sec_out, uint32_t* nsec_out,
                               uint8_t* status, uint64_t* cnt) {
    const std::string format(fmt);
    const char* f = strstr(fmt, "%f");
    const bool have_f = f != nullptr, end_f = have_f && f == fmt + format.size() - 2;
    std::vector<char> buf;
    for (uint64_t g = 0; g < ngroups; g++) {
        int64_t tv_sec = 0;
        long tv_nsec = 0;
        uint64_t key_at = 0, key_len = 0;
        for (uint64_t i = grp[g]; i < grp[g + 1]; i++) {
            sec_out[i] = 0;
            nsec_out[i] = 0;
            if (len[i] == 0xFFFFFFFFu) {
                status[i] = 1;
                cnt[0]++;
                continue;
            }
            const uint32_t n = len[i];
            buf.assign((size_t)n + 64, 0);
            memcpy(buf.data(), base + off[i], n);
            int nslen = -1;
            const char* r;
            const bool hit = (!have_f || end_f) && key_len && n >= key_len &&
                             memcmp(base + off[i], base + key_at, key_len) == 0;
            if (hit) {
                if (end_f || (format == "%s" && n > key_len)) {
                    int64_t unused = tv_sec;
                    r = wrapper(buf.data() + key_len, "%f", &unused, &tv_nsec, nslen, -1, (time_t)now);
                } else {
                    r = buf.data() + key_len;
                    tv_nsec = 0;
                }
            } else {
                r = wrapper(buf.data(), fmt, &tv_sec, &tv_nsec, nslen, year_mode, (time_t)now);
                if (r) {
                    key_at = off[i];
                    key_len = nslen < 0 ? n : n - (uint32_t)nslen;
                    tv_sec -= adjust;
                }
            }
            if (!r) {
                status[i] = 2;
                cnt[1]++;
                continue;
            }
            sec_out[i] = tv_sec;
            nsec_out[i] = (uint32_t)tv_nsec;
            if (tv_sec <= 0 || (discard_interval >= 0 && now - tv_sec > discard_interval)) {
                status[i] = 3;
                cnt[2]++;
                cnt[3]++;
            } else {
                status[i] = 0;
                cnt[4]++;
            }
        }
    }
}
