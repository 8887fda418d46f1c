// lc_zstd_emul.cpp -- TEST-ONLY host build of the zstd frame compressor (loongcollector_b200/csrc/lc_exec.cuh:
// lc_lz4_parse_chunk, lc_zstd_block, lc_zstd_emit_block), the statements the parse, block and emit kernels run, with
// W emulated lanes per batch, so that the "not gpu" tier can check the frames and pin the GPU's bytes.  Not part of
// the product library.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../loongcollector_b200/csrc/lc_exec.cuh"

extern "C" {

// Segment g = in[seg_off[g], + seg_len[g]) -> one frame; frames packed back to back (frm_off, frm_len).  Returns the
// total size (out, frm_off and frm_len written when it fits out_cap).
int64_t emul_zstd_compress(const uint8_t* in, uint64_t nseg, const uint64_t* seg_off, const uint32_t* seg_len,
                           uint32_t W, uint8_t* out, uint64_t out_cap, uint64_t* frm_off, uint32_t* frm_len) {
    static LcLz4Warp w;
    static LcZstdWarp zw;
    std::vector<uint64_t> first(nseg + 1), bfirst(nseg + 1);
    for (uint64_t g = 0; g < nseg; ++g) {
        first[g + 1] = first[g] + lc_lz4_nchunks(seg_len[g]);
        bfirst[g + 1] = bfirst[g] + lc_zstd_nblocks(seg_len[g]);
    }
    const uint64_t nch = first[nseg], nblk = bfirst[nseg];
    std::vector<LcLz4Seq> seq(nch * LC_LZ4_SEQ_CAP);
    std::vector<LcLz4Chunk> info(nch);
    std::vector<uint8_t> slot(nblk * LC_ZSTD_BLOCK);
    std::vector<uint32_t> body(nblk);
    std::vector<uint64_t> boff(nblk + 1);
    for (uint64_t g = 0; g < nseg; ++g) {
        const uint8_t* s = in + seg_off[g];
        const uint32_t n = seg_len[g];
        for (uint64_t k = first[g]; k < first[g + 1]; ++k) {
            const uint32_t c0 = (uint32_t)(k - first[g]) * LC_LZ4_CHUNK;
            const uint32_t c1 = n - c0 < LC_LZ4_CHUNK ? n : c0 + LC_LZ4_CHUNK;
            lc_lz4_parse_chunk(s, n, c0, c1, w, &seq[k * LC_LZ4_SEQ_CAP], &info[k], 0, W);
        }
        for (uint64_t k = bfirst[g]; k < bfirst[g + 1]; ++k) {
            const uint32_t j = (uint32_t)(k - bfirst[g]), b0 = j * LC_ZSTD_BLOCK;
            const uint64_t c = first[g] + 2 * j;
            LcZstdBlk b{s, b0, n - b0 < LC_ZSTD_BLOCK ? n : b0 + LC_ZSTD_BLOCK, {&seq[c * LC_LZ4_SEQ_CAP], nullptr},
                        {info[c].nseq, 0}};
            if (b.b1 - b.b0 > LC_LZ4_CHUNK) {
                b.seq[1] = &seq[(c + 1) * LC_LZ4_SEQ_CAP];
                b.nseq[1] = info[c + 1].nseq;
            }
            body[k] = lc_zstd_block(b, &slot[k * LC_ZSTD_BLOCK], zw, 0, W);
            boff[k + 1] = boff[k] + lc_zstd_emit_size(n, j, body[k]);
        }
    }
    const uint64_t total = boff[nblk];
    if (total > out_cap)
        return (int64_t)total;
    for (uint64_t g = 0; g < nseg; ++g) {
        frm_off[g] = boff[bfirst[g]];
        frm_len[g] = (uint32_t)(boff[bfirst[g + 1]] - boff[bfirst[g]]);
        for (uint64_t k = bfirst[g]; k < bfirst[g + 1]; ++k)
            lc_zstd_emit_block(in + seg_off[g], seg_len[g], (uint32_t)(k - bfirst[g]), &slot[k * LC_ZSTD_BLOCK],
                               body[k], out + boff[k], 0, W);
    }
    return (int64_t)total;
}
}
