/* lc_apsara_oracle.c -- CPU oracle of ProcessorParseApsaraNative (test infrastructure only, never linked into the
 * product).  A flat, sequential restatement of core/plugin/processor/ProcessorParseApsaraNative.cpp over the
 * strptime_ns / Strptime restatement of lc_timestamp_oracle.c (included below, not copied), with libc's own mktime in
 * the process's zone.  It shares no code with the device program.
 * The reference's undefined reads are pinned as the device pins them (loongcollector_b200/csrc/lc_exec.cuh):
 *   - the cache key is the 19 bytes at value + 1 whatever they are; bytes past the end of the base buffer read NUL;
 *   - a time string shorter than the key misses (the comparison reaches its NUL terminator first);
 *   - a value shorter than 2 bytes fails the time parse. */
#include "lc_timestamp_oracle.c"

#define AP_KEY 19
#define AP_NO_KEY 0xFFFFFFFFu
#define K_LEVEL 0xFFFFFFF0u
#define K_THREAD 0xFFFFFFF1u
#define K_FILE 0xFFFFFFF2u
#define K_LINE 0xFFFFFFF3u

typedef struct {
    uint32_t* ent; /* 4 words per entry */
    uint64_t n, cap;
} ents_t;

static void add(ents_t* e, uint32_t ko, uint32_t kl, uint32_t vo, uint32_t vl) {
    if (e->n < e->cap) {
        uint32_t* p = e->ent + 4 * e->n;
        p[0] = ko, p[1] = kl, p[2] = vo, p[3] = vl;
    }
    e->n++;
}

/* FindBaseFields (342-361) */
static int find_base_fields(const uint8_t* b, uint32_t n, int32_t* beg, int32_t* end) {
    int num = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (b[i] == '[') {
            beg[num] = (int32_t)i + 1;
        } else if (b[i] == ']') {
            uint8_t nx = i + 1 < n ? b[i + 1] : 0;
            if (i + 1 == n || nx == '\t' || nx == '\n') {
                end[num] = (int32_t)i;
                num++;
            }
            if (num >= 10)
                break;
            if (nx == '\t' && (i + 2 == n || b[i + 2] != '['))
                break;
        }
    }
    return num;
}

/* ParseApsaraBaseFields (433-463): the returned index, entries appended (offsets relative to the base buffer) */
static int32_t base_fields(const uint8_t* b, uint32_t n, uint32_t o, ents_t* e) {
    int32_t beg[10] = {0}, end[10] = {0};
    int num = find_base_fields(b, n, beg, end);
    if (num == 0)
        return 0;
    int bits = 0;
    for (int i = 1; bits != 0x111 && i < num; i++) {
        int32_t bi = beg[i], ei = end[i], k;
        int lvl = 1, thr = 1, fil = 0;
        for (k = bi; k < ei; k++) {
            if (b[k] > 'Z' || b[k] < 'A')
                lvl = 0;
            if (b[k] > '9' || b[k] < '0')
                thr = 0;
            if (b[k] == '/' || b[k] == '.')
                fil = 1;
        }
        if (!(bits & 0x1) && lvl) {
            bits |= 0x1;
            add(e, K_LEVEL, 0, o + bi, ei - bi);
        } else if (!(bits & 0x10) && thr) {
            bits |= 0x10;
            add(e, K_THREAD, 0, o + bi, ei - bi);
        } else if (!(bits & 0x100) && fil) {
            bits |= 0x100;
            int32_t c = bi;
            while (c < ei && b[c] != ':')
                c++;
            add(e, K_FILE, 0, o + bi, c - bi);
            if (c < ei)
                add(e, K_LINE, 0, o + c + 1, ei - c - 1);
        }
    }
    return end[num - 1];
}

/* ProcessorParseApsaraNative::Process over ngroups groups; len[i] == AP_NO_KEY = no SourceKey.  status: 0 ok, 1 not
 * found, 2 empty, 3 failed, 4 discarded, | 0x80 SourceKey overwritten.  cnt[5] += key_not_found, out_failed,
 * history_failure, discarded (history only), out_successful.  Entries (4 words each) of the ok events go to ent while
 * they fit in ent_cap; first[n + 1] and *n_ent are always written. */
void orc_apsara_process(int32_t adjust, const uint8_t* skey, uint32_t sklen, const uint8_t* base, uint64_t base_len,
                        const uint32_t* off, const uint32_t* len, const uint32_t* grp, uint64_t ngroups, int64_t now,
                        int32_t discard_interval, uint8_t* status, int64_t* sec_out, uint32_t* nsec_out,
                        int64_t* micro_out, uint64_t* first, uint32_t* ent, uint64_t ent_cap, uint64_t* n_ent,
                        uint64_t* cnt) {
    ents_t E = {ent, 0, ent_cap};
    char* st = NULL;
    size_t cap = 0;
    for (uint64_t g = 0; g < ngroups; g++) {
        int have_key = 0;
        uint64_t key_at = 0;  /* the cache: 19 bytes at base + key_at */
        int64_t cached = 0;   /* cachedLogTime.tv_sec */
        for (uint64_t i = grp[g]; i < grp[g + 1]; i++) {
            first[i] = E.n;
            status[i] = 3;
            sec_out[i] = micro_out[i] = 0;
            nsec_out[i] = 0;
            if (len[i] == AP_NO_KEY) {
                status[i] = 1;
                cnt[0]++;
                continue;
            }
            const uint32_t n = len[i];
            const uint8_t* b = base + off[i];
            if (n == 0) {
                status[i] = 2;
                cnt[1]++;
                continue;
            }
            /* ApsaraEasyReadLogTimeParser (251-323) */
            int64_t t = 0, us = 0;
            if (n >= 2 && b[0] == '[') {
                uint32_t pos = 1;
                while (pos < n && b[pos] != ']')
                    pos++;
                if (pos < n) {
                    if (cap < (size_t)pos + 64) {
                        cap = (size_t)pos + 64;
                        st = (char*)realloc(st, cap);
                    }
                    memset(st, 0, (size_t)pos + 64);
                    memcpy(st, b + 1, pos); /* strTime = buffer.substr(1, pos) */
                    int64_t s = 0;
                    long ns = 0;
                    int nl = 0;
                    if (b[1] == '1') {
                        const char* r = o_wrapper(st, "%s", &s, &ns, &nl, -1, (time_t)now);
                        if (r && r[0] == ']') {
                            t = s;
                            us = (int64_t)((uint64_t)s * 1000000u + (uint64_t)(ns / 1000));
                        }
                    } else {
                        int hit = have_key && pos >= AP_KEY;
                        for (int k = 0; hit && k < AP_KEY; k++)
                            hit = (uint8_t)st[k] == (key_at + k < base_len ? base[key_at + k] : 0);
                        if (hit) {
                            ns = 0;
                            if (pos > AP_KEY && !o_wrapper(st + AP_KEY + 1, "%f", &s, &ns, &nl, -1, (time_t)now))
                                ns = 0;
                            t = cached;
                            us = (int64_t)((uint64_t)cached * 1000000u + (uint64_t)(ns / 1000));
                        } else {
                            const char* r = o_wrapper(st, "%Y-%m-%d %H:%M:%S", &s, &ns, &nl, -1, (time_t)now);
                            if (r) {
                                if (*r != '\0' && !o_wrapper(r + 1, "%f", &s, &ns, &nl, -1, (time_t)now))
                                    ns = 0;
                                s -= adjust;
                                us = (int64_t)((uint64_t)s * 1000000u + (uint64_t)(ns / 1000));
                                have_key = 1;
                                key_at = off[i] + 1;
                                cached = s;
                                t = s;
                            }
                        }
                    }
                }
            }
            if (t <= 0) {
                cnt[1]++;
                continue;
            }
            sec_out[i] = t;
            micro_out[i] = us;
            nsec_out[i] = (uint32_t)((int64_t)((uint64_t)us * 1000u) % 1000000000);
            if (discard_interval >= 0 && now - t > discard_interval) {
                status[i] = 4;
                cnt[2]++;
                cnt[3]++;
                continue;
            }
            /* the fields (ProcessEvent 195-219) */
            int32_t idx = base_fields(b, n, off[i], &E);
            int32_t beg = 0, colon = -1, over = 0;
            for (idx = idx + 1; idx <= (int32_t)n; ++idx) {
                if (idx == (int32_t)n || b[idx] == '\t') {
                    if (colon >= 0) {
                        add(&E, off[i] + beg, colon - beg, off[i] + colon + 1, idx - colon - 1);
                        if ((uint32_t)(colon - beg) == sklen && memcmp(b + beg, skey, sklen) == 0)
                            over = 1;
                        colon = -1;
                    }
                    beg = idx + 1;
                } else if (b[idx] == ':' && colon == -1) {
                    colon = idx;
                }
            }
            status[i] = over ? 0x80 : 0;
            cnt[4]++;
        }
    }
    if (ngroups)
        first[grp[ngroups]] = E.n;
    *n_ent = E.n;
    free(st);
}
