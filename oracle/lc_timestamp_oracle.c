/* lc_timestamp_oracle.c -- CPU oracle of ProcessorParseTimestampNative (test infrastructure only, never linked into
 * the product).  A flat, sequential restatement of strptime_ns (core/common/Strptime.cpp), the Strptime wrapper
 * (core/common/TimeUtil.cpp:112-160) and ParseLogTime's second-level cache with ProcessEvent's verdict
 * (core/plugin/processor/ProcessorParseTimestampNative.cpp:100-235), over libc's own mktime / localtime_r in the
 * process's zone.  It shares no code with the device program.  Values are copied into NUL-padded buffers, so a
 * directive that reads past a value's end reads NUL bytes, as the device does. */
#define _DEFAULT_SOURCE
#include <ctype.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <time.h>

static const char* const k_day[7] = {"Sunday", "Monday", "Tuesday", "Wednesday", "Thursday", "Friday", "Saturday"};
static const char* const k_abday[7] = {"Sun", "Mon", "Tue", "Wed", "Thu", "Fri", "Sat"};
static const char* const k_mon[12] = {"January", "February", "March",     "April",   "May",      "June",
                                      "July",    "August",   "September", "October", "November", "December"};
static const char* const k_abmon[12] = {"Jan", "Feb", "Mar", "Apr", "May", "Jun",
                                        "Jul", "Aug", "Sep", "Oct", "Nov", "Dec"};
static const char* const k_ampm[2] = {"AM", "PM"};
static const char* const k_std[4] = {"EST", "CST", "MST", "PST"};
static const char* const k_dst[4] = {"EDT", "CDT", "MDT", "PDT"};

/* decimal field of at most as many digits as hi has, in [lo, hi]; NULL (dest untouched) otherwise */
static const unsigned char* o_num(const unsigned char* p, int* dest, unsigned lo, unsigned hi) {
    if (!isdigit(*p))
        return NULL;
    unsigned v = 0, budget = hi;
    do {
        v = v * 10 + (unsigned)(*p++ - '0');
        budget /= 10;
    } while (v * 10 <= hi && budget && isdigit(*p));
    if (v < lo || v > hi)
        return NULL;
    *dest = (int)v;
    return p;
}

/* fraction digits scaled to nanoseconds in unsigned 32-bit arithmetic */
static const unsigned char* o_frac(const unsigned char* p, long* dest, int* count) {
    if (!isdigit(*p))
        return NULL;
    const unsigned char* start = p;
    unsigned v = 0;
    int k = 0;
    while (isdigit(*p)) {
        v = v * 10 + (unsigned)(*p++ - '0');
        k++;
    }
    for (; k < 9; k++)
        v *= 10;
    *dest = (long)v;
    *count = (int)(p - start);
    return p;
}

static const unsigned char* o_names(const unsigned char* p, int* idx, const char* const* a, const char* const* b,
                                    int cnt) {
    const char* const* lists[2] = {a, b};
    for (int t = 0; t < 2 && lists[t]; t++)
        for (int i = 0; i < cnt; i++) {
            size_t n = strlen(lists[t][i]);
            if (strncasecmp(lists[t][i], (const char*)p, n) == 0) {
                *idx = i;
                return p + n;
            }
        }
    return NULL;
}

static const char* o_strptime(const char* buf, const char* fmt, struct tm* tm, long* ns, int* nslen);

static const char* o_epoch(const char* buf, struct tm* tm, long* ns, int* nslen) {
    char* end;
    long long v = strtoll(buf, &end, 10);
    char digits[32];
    size_t width = (size_t)snprintf(digits, sizeof digits, "%lld", v);
    size_t keep = width < 10 ? width : 10;
    for (size_t i = keep; i < width; i++)
        v /= 10;
    time_t t = (time_t)v;
    if (v == 0 || localtime_r(&t, tm) == NULL)
        return NULL;
    *ns = 0;
    *nslen = 0;
    o_frac((const unsigned char*)buf + keep, ns, nslen);
    return end;
}

static const char* o_strptime(const char* buf, const char* fmt, struct tm* tm, long* ns, int* nslen) {
    if (strcmp(fmt, "%s") == 0)
        return o_epoch(buf, tm, ns, nslen);
    const unsigned char* p = (const unsigned char*)buf;
    int split = 0;
    *ns = 0;
    while (p) {
        unsigned char c = (unsigned char)*fmt++;
        if (c == 0)
            break;
        if (isspace(c)) {
            while (isspace(*p))
                p++;
            continue;
        }
        if (c != '%') {
            if (*p++ != c)
                return NULL;
            continue;
        }
        int alt = 0, i = 0;
        /* allowed: a mask of the modifiers the conversion accepts, checked after it ran (-1: no check) */
        int allowed = -1;
        for (;;) {
            c = (unsigned char)*fmt++;
            if (c == 'E' || c == 'O') {
                if (alt)
                    return NULL;
                alt = c == 'E' ? 1 : 2;
                continue;
            }
            break;
        }
        const char* sub = NULL;
        switch (c) {
        case '%':
            if (*p++ != '%' || alt)
                return NULL;
            continue;
        case 'D': sub = "%m/%d/%y"; break;
        case 'F': sub = "%Y-%m-%d"; break;
        case 'R': sub = "%H:%M"; break;
        case 'r': sub = "%I:%M:%S %p"; break;
        case 'T': sub = "%H:%M:%S"; break;
        case 'A': case 'a': p = o_names(p, &tm->tm_wday, k_day, k_abday, 7); allowed = 0; break;
        case 'B': case 'b': case 'h': p = o_names(p, &tm->tm_mon, k_mon, k_abmon, 12); allowed = 0; break;
        case 'C':
            i = 20;
            p = o_num(p, &i, 0, 99);
            i = i * 100 - 1900;
            if (split)
                i += tm->tm_year % 100;
            split = 1;
            tm->tm_year = i;
            allowed = 1;
            break;
        case 'd': case 'e': p = o_num(p, &tm->tm_mday, 1, 31); allowed = 2; break;
        case 'f': p = o_frac(p, ns, nslen); allowed = 2; break;
        case 'k': case 'H':
            if (c == 'k' && alt)
                return NULL;
            p = o_num(p, &tm->tm_hour, 0, 23);
            allowed = 2;
            break;
        case 'l': case 'I':
            if (c == 'l' && alt)
                return NULL;
            p = o_num(p, &tm->tm_hour, 1, 12);
            if (tm->tm_hour == 12)
                tm->tm_hour = 0;
            allowed = 2;
            break;
        case 'j': i = 1; p = o_num(p, &i, 1, 366); tm->tm_yday = i - 1; allowed = 0; break;
        case 'M': p = o_num(p, &tm->tm_min, 0, 59); allowed = 2; break;
        case 'm': i = 1; p = o_num(p, &i, 1, 12); tm->tm_mon = i - 1; allowed = 2; break;
        case 'p':
            p = o_names(p, &i, k_ampm, NULL, 2);
            if (tm->tm_hour > 11)
                return NULL;
            tm->tm_hour += i * 12;
            allowed = 0;
            break;
        case 'S': p = o_num(p, &tm->tm_sec, 0, 61); allowed = 2; break;
        case 'U': case 'W': p = o_num(p, &i, 0, 53); allowed = 2; break;
        case 'V': p = o_num(p, &i, 0, 53); break;
        case 'w': p = o_num(p, &tm->tm_wday, 0, 6); allowed = 2; break;
        case 'u': i = 1; p = o_num(p, &i, 1, 7); tm->tm_wday = i % 7; allowed = 2; break;
        case 'g': p = o_num(p, &i, 0, 99); break;
        case 'G':
            do
                p++;
            while (isdigit(*p));
            break;
        case 'Y': i = 1900; p = o_num(p, &i, 0, 9999); tm->tm_year = i - 1900; allowed = 1; break;
        case 'y':
            p = o_num(p, &i, 0, 99);
            if (split) {
                i += (tm->tm_year / 100) * 100;
            } else {
                split = 1;
                i += i <= 68 ? 100 : 0;
            }
            tm->tm_year = i;
            break;
        case 'Z':
            if (strncasecmp((const char*)p, "GMT", 3) == 0 || strncasecmp((const char*)p, "UTC", 3) == 0) {
                tm->tm_isdst = 0;
                p += 3;
            }
            break;
        case 'z': {
            while (isspace(*p))
                p++;
            int neg = 0;
            if (*p == 'Z' || (p[0] == 'U' && p[1] == 'T') || (p[0] == 'G' && p[1] == 'M' && p[2] == 'T')) {
                p += *p == 'Z' ? 1 : (*p == 'U' ? 2 : 3);
                tm->tm_isdst = 0;
                break;
            }
            if (*p == 'G' || *p == 'U')
                return NULL;
            if (*p == '+' || *p == '-') {
                neg = *p++ == '-';
                int v = 0, k = 0;
                while (k < 4) {
                    if (isdigit(*p)) {
                        v = v * 10 + (*p++ - '0');
                        k++;
                    } else if (k == 2 && *p == ':') {
                        p++;
                    } else {
                        break;
                    }
                }
                if (!(k == 2 || (k == 4 && v % 100 < 60)))
                    return NULL;
                (void)neg;
                tm->tm_isdst = 0;
                break;
            }
            const unsigned char* q;
            if ((q = o_names(p, &i, k_std, NULL, 4)) != NULL) {
                p = q;
                break;
            }
            if ((q = o_names(p, &i, k_dst, NULL, 4)) != NULL) {
                p = q;
                tm->tm_isdst = 1;
                break;
            }
            if ((*p >= 'A' && *p <= 'I') || (*p >= 'L' && *p <= 'Y')) {
                p++;
                break;
            }
            return NULL;
        }
        case 'n': case 't':
            if (alt)
                return NULL;
            while (isspace(*p))
                p++;
            break;
        default:
            return NULL;
        }
        if (sub) {
            if (alt)
                return NULL;
            p = (const unsigned char*)o_strptime((const char*)p, sub, tm, ns, nslen);
            continue;
        }
        if (allowed >= 0 && (alt & ~allowed))
            return NULL;
    }
    return (const char*)p;
}

/* the Strptime wrapper: tv_sec is written whether or not the parse succeeded */
static const char* o_wrapper(const char* buf, const char* fmt, int64_t* sec, long* ns, int* nslen, int32_t year_mode,
                             time_t now) {
    struct tm tm;
    memset(&tm, 0, sizeof tm);
    tm.tm_year = INT_MIN;
    const char* r = o_strptime(buf, fmt, &tm, ns, nslen);
    if (strcmp(fmt, "%f") == 0)
        return r;
    if (year_mode >= 0 && tm.tm_year == INT_MIN) {
        if (year_mode > 0) {
            tm.tm_year = year_mode - 1900;
        } else {
            struct tm cur;
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

/* ProcessorParseTimestampNative::Process over ngroups groups of events; len[i] == 0xFFFFFFFF = no SourceKey.
 * status: 0 ok, 1 key not found, 2 failed, 3 discarded.  cnt[5] += key_not_found, out_failed, history_failure,
 * discarded, out_successful. */
void orc_ts_process(const char* fmt, int32_t year_mode, int32_t adjust, const uint8_t* base, const uint32_t* off,
                    const uint32_t* len, const uint32_t* grp, uint64_t ngroups, int64_t now, int32_t discard_interval,
                    int64_t* sec_out, uint32_t* nsec_out, uint8_t* status, uint64_t* cnt) {
    const char* f = strstr(fmt, "%f");
    const int have_f = f != NULL, end_f = have_f && f == fmt + strlen(fmt) - 2, is_s = strcmp(fmt, "%s") == 0;
    size_t cap = 0;
    char* buf = NULL;
    for (uint64_t g = 0; g < ngroups; g++) {
        int64_t tv_sec = 0;
        long tv_nsec = 0;
        uint64_t key_at = 0, key_len = 0; /* the cache: base[key_at, + key_len), empty = none */
        for (uint64_t i = grp[g]; i < grp[g + 1]; i++) {
            sec_out[i] = 0;
            nsec_out[i] = 0;
            if (len[i] == 0xFFFFFFFFu) {
                status[i] = 1;
                cnt[0]++;
                continue;
            }
            const uint32_t n = len[i];
            if (cap < (size_t)n + 64) {
                cap = (size_t)n + 64;
                buf = (char*)realloc(buf, cap);
            }
            memset(buf, 0, (size_t)n + 64);
            memcpy(buf, base + off[i], n);
            int nslen = -1;
            const char* r;
            int hit = (!have_f || end_f) && key_len && n >= key_len && memcmp(base + off[i], base + key_at, key_len) == 0;
            if (hit) {
                if (end_f || (is_s && n > key_len)) {
                    tv_nsec = 0;
                    r = o_strptime(buf + key_len, "%f", &(struct tm){0}, &tv_nsec, &nslen);
                } else {
                    r = buf + key_len;
                    tv_nsec = 0;
                }
            } else {
                r = o_wrapper(buf, fmt, &tv_sec, &tv_nsec, &nslen, year_mode, (time_t)now);
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
    free(buf);
}
