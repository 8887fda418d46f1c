// lc_split_sls_emul.cpp -- TEST-ONLY host build of the split-fed SLS serialiser (loongcollector_b200/csrc/lc_exec.cuh:
// lc_span_sls_rec + lc_span_sls_tile), the statements the size and emit kernels run, so that the "not gpu" tier can
// check them against the oracle with any tile size.  Not part of the product library.
#include <stdint.h>
#include <string.h>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Pieces (off, len) of src[0, src_len); okey NULL = no offset key; ns 0xFFFFFFFF = no Time_ns.  The writing pass cuts
// the output into tiles of `tile` bytes (0 = one tile) and runs `nlanes` lanes one after the other on each, as the
// lanes of the emit kernel's warp share a tile.  Returns the total size (out written when it fits out_cap).
int64_t emul_split_sls(const uint8_t* src, uint64_t src_len, const uint32_t* off, const uint32_t* len, uint64_t n,
                       const char* key, uint32_t klen, const char* okey, uint32_t oklen, uint64_t src_pos,
                       uint32_t time, uint32_t ns, uint64_t tile, uint32_t nlanes, uint8_t* out, uint64_t out_cap,
                       uint64_t* rec_off) {
    LcSpanSlsCfg c;
    memset(&c, 0, sizeof c);
    c.src = src;
    c.src_len = src_len;
    c.off = off;
    c.len = len;
    c.key = reinterpret_cast<const uint8_t*>(key);
    c.klen = klen;
    c.okey = reinterpret_cast<const uint8_t*>(okey);
    c.oklen = okey ? oklen : 0u;
    c.mode = !okey ? LC_SPAN_PIECE : (oklen == klen && !memcmp(okey, key, klen)) ? LC_SPAN_OFFSET : LC_SPAN_PIECE_OFFSET;
    c.time = time < (1u << 28) ? (1u << 28) : time;
    c.has_ns = ns != 0xFFFFFFFFu;
    c.ns = c.has_ns ? ns : 0u;
    c.src_pos = src_pos;
    uint64_t total = 0;
    for (uint64_t k = 0; k < n; ++k) {
        rec_off[k] = total;
        total += lc_span_sls_rec(c, off[k], len[k]).size;
    }
    if (total > out_cap || n == 0)
        return (int64_t)total;
    if (tile == 0)
        tile = total;
    for (uint64_t t0 = 0; t0 < total; t0 += tile) {
        const uint64_t t1 = t0 + tile < total ? t0 + tile : total;
        const uint64_t r = lc_span_sls_find(rec_off, n, t0);
        for (uint32_t lane = 0; lane < nlanes; ++lane)
            lc_span_sls_tile(c, rec_off, n, r, t0, t1, out, lane, nlanes);
    }
    return (int64_t)total;
}
}
