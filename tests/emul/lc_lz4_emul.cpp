// lc_lz4_emul.cpp -- TEST-ONLY host build of the LZ4 block compressor (loongcollector_b200/csrc/lc_exec.cuh:
// lc_lz4_parse_chunk, lc_lz4_seg_sizes, lc_lz4_emit_chunk), the statements the parse, size and emit kernels run, with
// W emulated lanes per batch, so that the "not gpu" tier can check the blocks and pin the GPU's bytes.  Not part of
// the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Segment g = in[seg_off[g], + seg_len[g]) -> one block; blocks packed back to back (blk_off, blk_len).  Returns the
// total size (out, blk_off and blk_len written when it fits out_cap).
int64_t emul_lz4_compress(const uint8_t* in, uint64_t nseg, const uint64_t* seg_off, const uint32_t* seg_len,
                          uint32_t W, uint8_t* out, uint64_t out_cap, uint64_t* blk_off, uint32_t* blk_len) {
    static LcLz4Warp w;
    std::vector<uint64_t> first(nseg + 1);
    for (uint64_t g = 0; g < nseg; ++g)
        first[g + 1] = first[g] + lc_lz4_nchunks(seg_len[g]);
    const uint64_t nch = first[nseg];
    std::vector<LcLz4Seq> seq(nch * LC_LZ4_SEQ_CAP);
    std::vector<LcLz4Chunk> info(nch);
    std::vector<uint32_t> csize(nch), anchor(nch);
    std::vector<uint64_t> choff(nch + 1);
    for (uint64_t g = 0; g < nseg; ++g) {
        const uint8_t* s = in + seg_off[g];
        const uint32_t n = seg_len[g];
        for (uint64_t k = first[g]; k < first[g + 1]; ++k) {
            const uint32_t c0 = (uint32_t)(k - first[g]) * LC_LZ4_CHUNK;
            const uint32_t c1 = n - c0 < LC_LZ4_CHUNK ? n : c0 + LC_LZ4_CHUNK;
            lc_lz4_parse_chunk(s, n, c0, c1, w, &seq[k * LC_LZ4_SEQ_CAP], &info[k], 0, W);
        }
        lc_lz4_seg_sizes(n, (uint32_t)(first[g + 1] - first[g]), &info[first[g]], &csize[first[g]], &anchor[first[g]]);
    }
    for (uint64_t k = 0; k < nch; ++k)
        choff[k + 1] = choff[k] + csize[k];
    const uint64_t total = choff[nch];
    if (total > out_cap)
        return (int64_t)total;
    for (uint64_t g = 0; g < nseg; ++g) {
        blk_off[g] = choff[first[g]];
        blk_len[g] = (uint32_t)(choff[first[g + 1]] - choff[first[g]]);
        for (uint64_t k = first[g]; k < first[g + 1]; ++k)
            lc_lz4_emit_chunk(in + seg_off[g], seg_len[g], (uint32_t)(k - first[g]) * LC_LZ4_CHUNK,
                              &seq[k * LC_LZ4_SEQ_CAP], info[k].nseq, anchor[k], k + 1 == first[g + 1],
                              out + choff[k], 0, W);
    }
    return (int64_t)total;
}
}
