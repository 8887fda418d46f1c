/* lc_json_oracle.c -- flat C restatement of ProcessorParseJsonNative's per-event rules as pinned in include/lc_b200.h
 * (lc_json_parse): a recursive-descent validator of strict RFC 8259 with the 1024 depth limit, strtod and
 * snprintf("%f") in the C locale for doubles, the integer range rules, and the same entry / arena layout as the
 * device.  Test infrastructure only: it shares no code with the product. */
#define _GNU_SOURCE
#include <errno.h>
#include <inttypes.h>
#include <locale.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define NO_KEY 0xFFFFFFFFu
#define ARENA 0x80000000u
#define MAX_DEPTH 1024

typedef struct {
    const uint8_t* s;
    size_t n, p;
    int ok;
} P;

typedef struct {
    uint8_t* b;
    size_t n, cap;
} Buf;

static void put(Buf* b, const void* d, size_t k) {
    if (b->n + k > b->cap) {
        b->cap = (b->n + k) * 2 + 64;
        b->b = (uint8_t*)realloc(b->b, b->cap);
    }
    memcpy(b->b + b->n, d, k);
    b->n += k;
}

static int at(P* q) { return q->p < q->n ? q->s[q->p] : -1; }
static void ws(P* q) {
    while (q->p < q->n && (q->s[q->p] == ' ' || q->s[q->p] == '\t' || q->s[q->p] == '\n' || q->s[q->p] == '\r'))
        q->p++;
}

static int hex4(P* q, size_t p) {
    if (p + 4 > q->n)
        return -1;
    int v = 0;
    for (int k = 0; k < 4; ++k) {
        int c = q->s[p + k], d;
        if (c >= '0' && c <= '9') d = c - '0';
        else if (c >= 'a' && c <= 'f') d = c - 'a' + 10;
        else if (c >= 'A' && c <= 'F') d = c - 'A' + 10;
        else return -1;
        v = v * 16 + d;
    }
    return v;
}

static void utf8(Buf* o, unsigned v) {
    uint8_t b[4];
    size_t k;
    if (v < 0x80) { b[0] = v; k = 1; }
    else if (v < 0x800) { b[0] = 0xC0 | (v >> 6); b[1] = 0x80 | (v & 63); k = 2; }
    else if (v < 0x10000) { b[0] = 0xE0 | (v >> 12); b[1] = 0x80 | ((v >> 6) & 63); b[2] = 0x80 | (v & 63); k = 3; }
    else { b[0] = 0xF0 | (v >> 18); b[1] = 0x80 | ((v >> 12) & 63); b[2] = 0x80 | ((v >> 6) & 63); b[3] = 0x80 | (v & 63); k = 4; }
    put(o, b, k);
}

/* a string after its opening quote; its unescaped bytes go to o (may be NULL); *esc: it had an escape */
static int str(P* q, Buf* o, int* esc) {
    *esc = 0;
    for (;;) {
        if (q->p >= q->n) return 0;
        unsigned c = q->s[q->p];
        if (c == '"') { q->p++; return 1; }
        if (c < 0x20) return 0;
        if (c == '\\') {
            *esc = 1;
            if (q->p + 1 >= q->n) return 0;
            unsigned x = q->s[q->p + 1], r;
            const char* from = "\"\\/bfnrt";
            const char* to = "\"\\/\b\f\n\r\t";
            const char* f = x ? strchr(from, (int)x) : NULL;
            if (f) { r = (uint8_t)to[f - from]; if (o) { uint8_t b = (uint8_t)r; put(o, &b, 1); } q->p += 2; continue; }
            if (x != 'u') return 0;
            int cp = hex4(q, q->p + 2);
            if (cp < 0 || (cp >= 0xDC00 && cp <= 0xDFFF)) return 0;
            q->p += 6;
            if (cp >= 0xD800 && cp <= 0xDBFF) {
                if (q->p + 1 >= q->n || q->s[q->p] != '\\' || q->s[q->p + 1] != 'u') return 0;
                int lo = hex4(q, q->p + 2);
                if (lo < 0xDC00 || lo > 0xDFFF) return 0;
                q->p += 6;
                cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
            }
            if (o) utf8(o, (unsigned)cp);
            continue;
        }
        size_t k = 1;
        if (c >= 0x80) {
            unsigned lo = 0x80, hi = 0xBF;
            if (c >= 0xC2 && c <= 0xDF) k = 2;
            else if (c >= 0xE0 && c <= 0xEF) { k = 3; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
            else if (c >= 0xF0 && c <= 0xF4) { k = 4; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
            else return 0;
            if (q->p + k > q->n) return 0;
            if (q->s[q->p + 1] < lo || q->s[q->p + 1] > hi) return 0;
            for (size_t j = 2; j < k; ++j)
                if ((q->s[q->p + j] & 0xC0) != 0x80) return 0;
        }
        if (o) put(o, q->s + q->p, k);
        q->p += k;
    }
}

static int isdig(P* q) { return q->p < q->n && q->s[q->p] >= '0' && q->s[q->p] <= '9'; }

/* a number by the JSON grammar; *isint: no fraction, no exponent */
static int num(P* q, int* isint) {
    if (at(q) == '-') q->p++;
    if (!isdig(q)) return 0;
    if (q->s[q->p] == '0') q->p++;
    else while (isdig(q)) q->p++;
    *isint = 1;
    if (at(q) == '.') {
        q->p++;
        if (!isdig(q)) return 0;
        while (isdig(q)) q->p++;
        *isint = 0;
    }
    if (at(q) == 'e' || at(q) == 'E') {
        q->p++;
        if (at(q) == '+' || at(q) == '-') q->p++;
        if (!isdig(q)) return 0;
        while (isdig(q)) q->p++;
        *isint = 0;
    }
    return 1;
}

static int lit(P* q, const char* w) {
    size_t k = strlen(w);
    if (q->p + k > q->n || memcmp(q->s + q->p, w, k)) return 0;
    q->p += k;
    return 1;
}

/* any value at nesting depth `depth` (the depth a container opened here would have) */
static int value(P* q, int depth) {
    ws(q);
    int c = at(q), esc, isint;
    if (c == '{' || c == '[') {
        if (depth > MAX_DEPTH) return 0;
        int close = c == '{' ? '}' : ']';
        q->p++;
        ws(q);
        if (at(q) == close) { q->p++; return 1; }
        for (;;) {
            if (c == '{') {
                ws(q);
                if (at(q) != '"') return 0;
                q->p++;
                if (!str(q, NULL, &esc)) return 0;
                ws(q);
                if (at(q) != ':') return 0;
                q->p++;
            }
            if (!value(q, depth + 1)) return 0;
            ws(q);
            if (at(q) == ',') { q->p++; continue; }
            if (at(q) == close) { q->p++; return 1; }
            return 0;
        }
    }
    if (c == '"') { q->p++; return str(q, NULL, &esc); }
    if (c == 't') return lit(q, "true");
    if (c == 'f') return lit(q, "false");
    if (c == 'n') return lit(q, "null");
    if (c == '-' || (c >= '0' && c <= '9')) return num(q, &isint);
    return 0;
}

typedef struct {
    uint32_t ko, kl, vo, vl;
} Ent;

/* one event: 0 = parsed (entries appended to E, arena bytes to A), 1 = failed; *hit: a key equals SourceKey */
static int event(const uint8_t* s, size_t n, uint32_t base_off, const uint8_t* sk, size_t skl, Buf* E, Buf* A,
                 uint32_t arena0, int* hit) {
    P q = {s, n, 0, 1};
    *hit = 0;
    ws(&q);
    if (at(&q) != '{') return 1;
    q.p++;
    ws(&q);
    if (at(&q) == '}') {
        q.p++;
    } else {
        for (;;) {
            ws(&q);
            if (at(&q) != '"') return 1;
            q.p++;
            size_t k0 = q.p;
            Buf key = {0};
            int esc;
            if (!str(&q, &key, &esc)) { free(key.b); return 1; }
            Ent e;
            e.kl = (uint32_t)key.n;
            if (key.n == skl && (skl == 0 || !memcmp(key.b, sk, skl))) *hit = 1;
            if (esc) { e.ko = ARENA | (uint32_t)(arena0 + A->n); put(A, key.b, key.n); }
            else e.ko = base_off + (uint32_t)k0;
            free(key.b);
            ws(&q);
            if (at(&q) != ':') return 1;
            q.p++;
            ws(&q);
            size_t v0 = q.p;
            int c = at(&q), isint;
            e.vo = base_off + (uint32_t)v0;
            e.vl = 0;
            if (c == '"') {
                q.p++;
                Buf v = {0};
                if (!str(&q, &v, &esc)) { free(v.b); return 1; }
                e.vl = (uint32_t)v.n;
                if (esc) { e.vo = ARENA | (uint32_t)(arena0 + A->n); put(A, v.b, v.n); }
                else e.vo = base_off + (uint32_t)v0 + 1;
                free(v.b);
            } else if (c == '{' || c == '[') {
                if (!value(&q, 2)) return 1;
                e.vl = (uint32_t)(q.p - v0);
            } else if (c == 't' || c == 'f') {
                if (!lit(&q, c == 't' ? "true" : "false")) return 1;
                e.vl = (uint32_t)(q.p - v0);
            } else if (c == 'n') {
                if (!lit(&q, "null")) return 1;
            } else if (c == '-' || (c >= '0' && c <= '9')) {
                if (!num(&q, &isint)) return 1;
                char t[64];
                size_t tl = q.p - v0;
                if (isint && tl >= sizeof t) {
                    /* out of range of both integer types: empty */
                } else if (isint) {
                    memcpy(t, s + v0, tl);
                    t[tl] = 0;
                    char* end;
                    errno = 0;
                    if (c == '-') {
                        long long v = strtoll(t, &end, 10);
                        if (errno != ERANGE) {
                            if (v == 0) { e.vo = base_off + (uint32_t)v0 + 1; e.vl = 1; }
                            else e.vl = (uint32_t)tl;
                        }
                    } else {
                        strtoull(t, &end, 10);
                        if (errno != ERANGE) e.vl = (uint32_t)tl;
                    }
                } else {
                    size_t L = q.p - v0;
                    char* tmp = (char*)malloc(L + 1);
                    memcpy(tmp, s + v0, L);
                    tmp[L] = 0;
                    double d = strtod(tmp, NULL);
                    free(tmp);
                    if (!isinf(d)) {
                        char out[400];
                        int k = snprintf(out, sizeof out, "%f", d);
                        e.vo = ARENA | (uint32_t)(arena0 + A->n);
                        e.vl = (uint32_t)k;
                        put(A, out, (size_t)k);
                    }
                }
            } else {
                return 1;
            }
            put(E, &e, sizeof e);
            ws(&q);
            if (at(&q) == ',') { q.p++; continue; }
            if (at(&q) == '}') { q.p++; break; }
            return 1;
        }
    }
    ws(&q);
    return q.p < n && s[q.p] != 0;
}

/* status[n], first[n + 1], entries / arena written only when both fit, counters[3] */
void orc_json_process(const uint8_t* sk, uint32_t skl, const uint8_t* base, uint64_t base_len, const uint32_t* off,
                      const uint32_t* len, uint64_t n, uint8_t* status, uint64_t* first, uint32_t* ent,
                      uint64_t ent_cap, uint64_t* n_ent, uint8_t* arena, uint64_t arena_cap, uint64_t* n_arena,
                      uint64_t* counters) {
    (void)base_len;
    setlocale(LC_NUMERIC, "C");
    Buf E = {0}, A = {0};
    memset(counters, 0, 3 * sizeof(uint64_t));
    for (uint64_t i = 0; i < n; ++i) {
        first[i] = E.n / sizeof(Ent);
        if (len[i] == NO_KEY) { status[i] = 1; counters[0]++; continue; }
        if (len[i] == 0) { status[i] = 2; continue; }
        size_t e0 = E.n, a0 = A.n;
        int hit;
        if (event(base + off[i], len[i], off[i], sk, skl, &E, &A, 0, &hit)) {
            E.n = e0;
            A.n = a0;
            status[i] = 3;
            counters[1]++;
        } else {
            status[i] = hit ? 0x80 : 0;
            counters[2]++;
        }
    }
    first[n] = E.n / sizeof(Ent);
    *n_ent = first[n];
    *n_arena = A.n;
    if (*n_ent <= ent_cap && *n_arena <= arena_cap) {
        if (E.n) memcpy(ent, E.b, E.n);
        if (A.n) memcpy(arena, A.b, A.n);
    }
    free(E.b);
    free(A.b);
}
