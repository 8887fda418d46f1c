// lc_json_asan.cpp -- TEST-ONLY driver that runs the host build of the JSON walk (lc_exec.cuh: lc_json_count and
// lc_json_emit, both instantiations) under -fsanitize=address,undefined.  Every event sits in its own heap allocation
// of exactly its length (nothing addressable before or after it), and every emit goes to allocations of exactly the counted sizes, so a read past the event or
// a write past its ranges stops the run.  Corpus: the documents given on stdin (4-byte little-endian length, bytes),
// every length 0..300 at every 16-byte alignment, the depths 63, 64, 65, 1024 and 1025, 1 MiB strings, and every
// truncation of every valid document.  Exit 0 when clean, 1 when the fast and slow walks disagree.
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

static const uint8_t kKey[] = "content";
static uint64_t g_events, g_ok, g_slow;

// count and emit one event with both instantiations; returns whether it parsed.  The event is an allocation of exactly
// its length (an empty one gets a 0-byte allocation), so one byte read past either end is reported; `align` only
// varies the lengths the callers ask for.
static bool one(const std::string& doc, uint32_t align) {
    (void)align;
    uint8_t* mem = (uint8_t*)malloc(doc.size());
    uint8_t* s = mem;
    if (!doc.empty())
        memcpy(s, doc.data(), doc.size());
    const uint32_t n = (uint32_t)doc.size();
    const uint8_t* base = s; // offset 0: the event is the whole base
    uint32_t ne = 0, na = 0, ne2 = 0, na2 = 0;
    bool sl = false, sl2 = false;
    uint32_t st = lc_json_count<false>(base, 0, n, kKey, 7, lc_json_pow5, &ne, &na, &sl);
    const uint32_t st2 = lc_json_count<true>(base, 0, n, kKey, 7, lc_json_pow5, &ne2, &na2, &sl2);
    if (sl2) {
        fprintf(stderr, "slow walk gave up\n");
        exit(1);
    }
    if (!sl && (st != st2 || ne != ne2 || na != na2)) {
        fprintf(stderr, "fast and slow walks disagree on a %u-byte event\n", n);
        exit(1);
    }
    g_events++;
    g_slow += sl;
    st = st2;
    if ((st & 0x7Fu) == LC_JSON_ST_OK) {
        g_ok++;
        LcJsonEntry* ent = (LcJsonEntry*)malloc(sizeof(LcJsonEntry) * (ne2 ? ne2 : 1));
        uint8_t* ar = (uint8_t*)malloc(na2 ? na2 : 1);
        if (!sl && !lc_json_emit<false>(base, 0, n, kKey, 7, lc_json_pow5, ent, ne2, ar, 0, na2)) {
            fprintf(stderr, "fast emit did not fill its ranges\n");
            exit(1);
        }
        if (!lc_json_emit<true>(base, 0, n, kKey, 7, lc_json_pow5, ent, ne2, ar, 0, na2)) {
            fprintf(stderr, "slow emit did not fill its ranges\n");
            exit(1);
        }
        // ranges one short: nothing may be written past them
        if (ne2 && lc_json_emit<true>(base, 0, n, kKey, 7, lc_json_pow5, ent, ne2 - 1, ar, 0, na2)) {
            fprintf(stderr, "short entry range accepted\n");
            exit(1);
        }
        if (na2 && lc_json_emit<true>(base, 0, n, kKey, 7, lc_json_pow5, ent, ne2, ar, 0, na2 - 1)) {
            fprintf(stderr, "short arena range accepted\n");
            exit(1);
        }
        free(ent);
        free(ar);
    }
    free(mem);
    return (st & 0x7Fu) == LC_JSON_ST_OK;
}

static std::string nest(int depth) { // a root object holding depth - 1 nested arrays
    return "{\"a\":" + std::string(depth - 1, '[') + std::string(depth - 1, ']') + "}";
}

int main(int argc, char** argv) {
    std::vector<std::string> docs;
    uint8_t h[4];
    while (fread(h, 1, 4, stdin) == 4) {
        const uint32_t l = h[0] | h[1] << 8 | h[2] << 16 | (uint32_t)h[3] << 24;
        std::string d(l, '\0');
        if (l && fread(&d[0], 1, l, stdin) != l)
            return 2;
        docs.push_back(d);
    }
    for (const std::string& d : docs) {
        const bool ok = one(d, 0);
        if (ok && d.size() <= 4096) // every truncation of a valid document
            for (size_t k = 0; k < d.size(); ++k)
                one(d.substr(0, k), (uint32_t)(k & 15));
    }
    // every length 0..300 at every 16-byte alignment: a valid prefix padded with a string, and its cuts
    const std::string fill = "{\"k\":\"" + std::string(300, 'x') + "\"}";
    for (uint32_t l = 0; l <= 300; ++l)
        for (uint32_t a = 0; a < 16; ++a) {
            std::string d = fill.substr(0, l);
            if (l >= 8)
                d = "{\"k\":\"" + std::string(l - 8, 'x') + "\"}";
            one(d, a);
        }
    const int depths[] = {63, 64, 65, 1024, 1025};
    for (int d : depths) {
        const bool ok = one(nest(d), 0);
        if (ok != (d <= 1024)) {
            fprintf(stderr, "depth %d: wrong verdict\n", d);
            return 1;
        }
    }
    std::string big = "{\"a\":\"" + std::string(1 << 20, 'y') + "\",\"b\":\"" + std::string(1 << 20, 'z') + "\\n\"}";
    if (!one(big, 3))
        return 1;
    if (one(big.substr(0, big.size() - 1), 5))
        return 1;
    printf("events %llu ok %llu slow %llu\n", (unsigned long long)g_events, (unsigned long long)g_ok,
           (unsigned long long)g_slow);
    (void)argc;
    (void)argv;
    return 0;
}
