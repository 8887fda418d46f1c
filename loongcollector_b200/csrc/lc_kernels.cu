// lc_kernels.cu -- sm_90a kernels of the log-parsing engine.
//
// All work is HBM-bound byte / integer indexing (no tensor cores): the split passes stream the
// SourceBuffer bytes once with 16-byte coalesced loads and number every line from a scan of
// per-tile line counts; the regex kernels interpret the automaton tables produced by
// regex_compiler.cpp once per log line; the multiline splitter turns the reference's sequential
// start/continue/end state machine into a prefix scan over 2-state transition functions.
//
// Reference behaviour reproduced (paths relative to the reference checkout):
//   split      core/plugin/processor/inner/ProcessorSplitLogStringNative.cpp:127-174
//   multiline  core/plugin/processor/inner/ProcessorSplitMultilineLogStringNative.cpp:162-393
//   regex      core/plugin/processor/ProcessorParseRegexNative.cpp:186-253, core/common/StringTools.cpp:183-288
//   delimiter  core/plugin/processor/ProcessorParseDelimiterNative.cpp:219-409, core/parser/DelimiterModeFsmParser.cpp:49-294
#include "lc_kernels.cuh"

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "lc_exec.cuh"
#include "lc_scan.cuh"

namespace lck {

using namespace lcscan;

// ================================================================================================ split
// 16 input bytes -> 16-bit mask of bytes equal to the (replicated) split char
__device__ __forceinline__ uint32_t match16(uint4 v, uint32_t splat) {
    uint32_t m = 0;
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t eq = __vcmpeq4(w[k], splat) & 0x01010101u; // bit 0 of each equal byte
        m |= (((eq * 0x01020408u) >> 24) & 0xFu) << (4 * k);
    }
    return m;
}

// PROBE (multiline, a2): the anchored prefix probes of the start / continue / end patterns (regex_search +
// match_continuous, StringTools.cpp:263-288) are evaluated by the same pass that finds the lines -- a line's first bytes
// were fetched a moment ago (same tile or the one before: L1 / L2 hits), so the separate probe pass that re-read the
// first sector of every line is gone.  A line's owner (the thread that holds its terminating newline) only applies a
// first-byte filter: most lines cannot start a match of any pattern and get flags = 0 at once.  Candidates go to a
// queue in shared memory and are probed DENSELY, one thread per queued line, after the tile's lines are written --
// otherwise a warp in which a single lane owns a 35-step start line would idle its other 31 lanes for 35 steps.
struct SplitProbe {
    uint32_t any_first[8]; // union of first[]: bytes that can start a match of any pattern
    const void* blob[3];   // device blobs of the start / continue / end patterns (nullptr = not configured)
    uint32_t first[3][8];  // per pattern: bit b set <=> a line whose first byte is b can match (prefix DFA, host-built)
    uint32_t empty_flags;  // flags of an empty line (patterns that match the empty prefix)
    uint8_t* flags;        // [line] bit0/1/2 = start / continue / end matches a prefix
};
constexpr uint32_t kProbeTable = 2048; // u16 entries of a prefix DFA that is staged in shared memory (states x classes)

// The prefix DFAs of the (up to three) patterns, staged in shared memory by every block of the split + probe pass: a
// queued line is probed with three DEPENDENT look-ups per byte (byte -> class -> next state), which from global memory
// costs a few hundred cycles per step and left a 35-step tail on every tile.
struct ProbeSmem {
    uint8_t cls[3][256];
    uint16_t next[3][kProbeTable];
    uint8_t acc[3][256];
    uint32_t nc[3], start[3], staged[3];
};

__device__ __forceinline__ void probe_stage(const SplitProbe& pr, ProbeSmem& ps) {
    for (int p = 0; p < 3; ++p) {
        if (!pr.blob[p]) {
            if (threadIdx.x == 0)
                ps.staged[p] = 0;
            continue;
        }
        const LcProgView v = lc_view(pr.blob[p]);
        const uint32_t ns = v.h->pre_nstates, nc = v.h->nclasses;
        const bool fits = ns * nc <= kProbeTable && ns <= 256;
        if (threadIdx.x == 0) {
            ps.nc[p] = nc;
            ps.start[p] = v.h->pre_start;
            ps.staged[p] = fits ? 1u : 0u;
        }
        if (!fits)
            continue;
        for (uint32_t k = threadIdx.x; k < 256; k += blockDim.x)
            ps.cls[p][k] = v.byte_class[k];
        for (uint32_t k = threadIdx.x; k < ns * nc; k += blockDim.x)
            ps.next[p][k] = v.pre_next[k];
        for (uint32_t k = threadIdx.x; k < ns; k += blockDim.x)
            ps.acc[p][k] = v.pre_acc[k];
    }
}

__device__ __forceinline__ uint8_t probe_line_smem(const SplitProbe& pr, const ProbeSmem& ps,
                                                   const uint8_t* __restrict__ s, uint32_t l) {
    uint8_t f = 0;
#pragma unroll
    for (int p = 0; p < 3; ++p) {
        if (!pr.blob[p])
            continue;
        if (!ps.staged[p]) {
            if (lc_prefix_match(lc_view(pr.blob[p]), s, l))
                f |= (uint8_t)(1u << p);
            continue;
        }
        const uint32_t nc = ps.nc[p];
        uint32_t st = ps.start[p];
        bool hit = false, done = false;
        for (uint32_t i = 0; i < l; ++i) {
            const uint32_t e = ps.next[p][st * nc + ps.cls[p][s[i]]];
            if (e == LC_PREFIX_ACCEPT) {
                hit = true;
                done = true;
                break;
            }
            if (e == LC_PREFIX_DEAD) {
                done = true;
                break;
            }
            st = e;
        }
        if (!done)
            hit = ps.acc[p][st] != 0;
        if (hit)
            f |= (uint8_t)(1u << p);
    }
    return f;
}

__device__ __forceinline__ uint8_t probe_line(const SplitProbe& pr, const uint8_t* __restrict__ s, uint32_t l) {
    uint8_t f = 0;
#pragma unroll
    for (int p = 0; p < 3; ++p)
        if (pr.blob[p] && lc_prefix_match(lc_view(pr.blob[p]), s, l))
            f |= (uint8_t)(1u << p);
    return f;
}
// which patterns may match a non-empty line whose first byte is b
__device__ __forceinline__ uint32_t probe_first(const SplitProbe& pr, uint32_t b) {
    uint32_t m = 0;
#pragma unroll
    for (int p = 0; p < 3; ++p)
        m |= ((pr.first[p][b >> 5] >> (b & 31)) & 1u) << p;
    return m;
}

// bit 7 of every byte of w that equals the splat byte (exact, no cross-byte borrows)
__device__ __forceinline__ uint32_t eq_bytes(uint32_t w, uint32_t splat) {
    const uint32_t x = w ^ splat;
    return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u;
}
// 16 input bytes -> 16-bit mask of the bytes equal to the splat byte
__device__ __forceinline__ uint32_t match16b(uint4 v, uint32_t splat) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) // bits 7 / 15 / 23 / 31 -> one nibble (the partial products never collide)
        m |= ((((eq_bytes(w[k], splat) >> 7) * 0x00204081u) >> 21) & 0xFu) << (4 * k);
    return m;
}

// ---- three-pass split: masks -> tile scan -> emission ------------------------------------------------------------------
// What a single-pass kernel cannot get around (measured with per-tile phase timestamps, three restructurings tried:
// persistent + prefetched tiles, a scanner warp beside the byte work, two tiles of slack, 256-descriptor walks): lines
// must be numbered in buffer order, so with a decoupled look-back a tile finishes only after EVERY earlier tile has
// published its count, and the per-tile service time has a heavy tail (with two 1024-thread blocks on an SM).  All the
// resident tiles (two per SM) wait for the slowest of them, every generation, and in the per-tile %globaltimer stamps
// the look-back was the largest phase in every variant: persistent blocks with cp.async-prefetched tiles (the loads
// fully hidden), 8 descriptors per lane and round, a scanner warp beside 31 data warps with two tiles of slack (one
// round of 256 descriptors, re-polled while it waits for unpublished predecessors), and three tickets per block (a
// serial chain).  (None of those kernels is kept; the plain single-pass look-back split was 5 % slower than the three
// passes below on an H100.)
// The order constraint only concerns the NUMBERS, though, not the bytes:
//   pass 1  split_mask_kernel   reads the buffer once (a warp covers 2 KiB with four 16-byte loads per lane), and
//                               writes one mask bit per byte (len/8 bytes) plus {count, end of last newline} per tile;
//                               tiles are independent -- no descriptor, no ticket, no waiting;
//   pass 2  split_scan_kernel   one block turns the per-tile pairs into exclusive prefixes (8 K tiles for 512 MiB);
//   pass 3  split_emit_kernel   reads the MASKS (1/8 of the bytes, mostly still in L2), numbers the lines of a tile from
//                               its prefix and writes the table.
// Traffic: len + 2 * len/8 instead of len; in exchange no pass ever waits for another block.  With per-line probes (the
// multiline front half) pass 1 also records, per newline, whether the byte after it can start a match of any pattern
// (a second bit per byte), so that pass 3 neither re-reads line heads from DRAM for the first-byte filter nor probes
// the ~95 % of lines that cannot match.
constexpr uint32_t kSplitTileChunks = 4096; // 16-byte chunks per tile (64 KiB, 1024 threads x 4)

__device__ __forceinline__ uint32_t match16c(uint4 v, uint32_t splat) {
    constexpr uint32_t M0 = (1u << 25) | (1u << 18) | (1u << 11) | (1u << 4), M4 = M0 << 4;
    // bit 8j+7 of a word's marks times 2^(25+C-7j) lands on bit 32+C+j; all 16 partial products fall on distinct bits,
    // so the high word of the product holds the word's nibble at C..C+3 exactly (no carries)
    const uint32_t p0 = (__umulhi(eq_bytes(v.x, splat), M0) & 0x0Fu) | (__umulhi(eq_bytes(v.y, splat), M4) & 0xF0u);
    const uint32_t p1 = (__umulhi(eq_bytes(v.z, splat), M0) & 0x0Fu) | (__umulhi(eq_bytes(v.w, splat), M4) & 0xF0u);
    return p0 | (p1 << 8);
}

template <bool PROBE>
__global__ void __launch_bounds__(1024, 2)
    split_mask_kernel(const uint8_t* __restrict__ buf, uint32_t len, uint32_t shift, uint32_t splat,
                      uint16_t* __restrict__ masks /* [chunk] newline bits; PROBE: + [chunk] candidate bits behind them */,
                      uint64_t nchunks /* chunks the mask arrays hold (tiles x 4096) */,
                      uint64_t* __restrict__ agg /* [tile] */, uint64_t* __restrict__ wagg /* [tile][warp] */,
                      SplitProbe pr) {
    __shared__ uint32_t s_cnt, s_last;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t tile = blockIdx.x;
    if (tid == 0)
        s_cnt = s_last = 0;
    __syncthreads();
    const uint4* vbuf = reinterpret_cast<const uint4*>(buf - shift);
    const uint64_t total_v = (uint64_t)len + shift; // virtual length including the alignment lead-in
    // The warp's 2 KiB = 128 chunks, four per lane.  Plain split: slot r = chunk 32 r + lane (every load instruction reads
    // one contiguous 512-byte row; measured best).  With probes a lane owns two ADJACENT chunks in each of two 1 KiB rows
    // (slot r: row r / 2, half r % 2), so that newline and candidate masks leave as 4-byte stores -- 2-byte stores into
    // two arrays slowed the pass down.
    const uint64_t c0 = (uint64_t)tile * kSplitTileChunks + (uint32_t)wid * 128 + (uint32_t)lane * (PROBE ? 2 : 1);
#define LC_SLOT_CHUNK(r) (PROBE ? c0 + 64 * ((r) >> 1) + ((r)&1) : c0 + 32 * (r))
    const bool full = ((uint64_t)(tile + 1) * kSplitTileChunks * 16 <= total_v) && !(tile == 0 && shift);
    uint4 v[4];
    uint32_t m[4];
    if (full) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
            v[r] = __ldg(vbuf + LC_SLOT_CHUNK(r));
#pragma unroll
        for (int r = 0; r < 4; ++r)
            m[r] = match16c(v[r], splat);
    } else {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const uint64_t vpos = LC_SLOT_CHUNK(r) * 16;
            m[r] = 0;
            v[r] = make_uint4(0, 0, 0, 0);
            if (vpos < total_v) {
                v[r] = __ldg(vbuf + LC_SLOT_CHUNK(r));
                m[r] = match16c(v[r], splat);
                if (vpos == 0 && shift) // alignment lead-in bytes in front of the buffer (shift < 16)
                    m[r] &= ~((1u << shift) - 1u);
                if (total_v - vpos < 16)
                    m[r] &= (1u << (total_v - vpos)) - 1u;
            }
        }
    }
    uint32_t last = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r)
        if (m[r]) // slots ascend, so the last hit wins
            last = (uint32_t)(LC_SLOT_CHUNK(r) * 16 + (31 - __clz(m[r])) + 1 - shift);
    const uint32_t cnt = __popc(m[0] | (m[1] << 16)) + __popc(m[2] | (m[3] << 16));
    if constexpr (!PROBE) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
            masks[LC_SLOT_CHUNK(r)] = (uint16_t)m[r];
    } else {
        uint32_t* nl32 = reinterpret_cast<uint32_t*>(masks); // (c0 is even)
        nl32[c0 >> 1] = m[0] | (m[1] << 16);
        nl32[(c0 + 64) >> 1] = m[2] | (m[3] << 16);
        uint32_t* cand32 = reinterpret_cast<uint32_t*>(masks + nchunks);
        uint32_t cm[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            uint32_t c16 = 0, mm = m[r];
            while (mm) {
                const uint32_t b = __ffs(mm) - 1;
                mm &= mm - 1;
                if (b == 15) { // the next byte lives in another chunk: leave the decision to the probe
                    c16 |= 1u << 15;
                } else {
                    const uint32_t i = (b + 1) >> 2;
                    const uint32_t w = i < 2 ? (i == 0 ? v[r].x : v[r].y) : (i == 2 ? v[r].z : v[r].w);
                    const uint32_t nb = (w >> (8 * ((b + 1) & 3))) & 0xFFu;
                    c16 |= ((pr.any_first[nb >> 5] >> (nb & 31)) & 1u) << b;
                }
            }
            cm[r] = c16;
        }
        cand32[c0 >> 1] = cm[0] | (cm[1] << 16);
        cand32[(c0 + 64) >> 1] = cm[2] | (cm[3] << 16);
    }
#undef LC_SLOT_CHUNK
    const uint32_t wc = __reduce_add_sync(0xFFFFFFFFu, cnt), wl = __reduce_max_sync(0xFFFFFFFFu, last);
    if (lane == 0) {
        wagg[(uint64_t)tile * 32 + wid] = ((uint64_t)wc << 32) | wl; // the warp's 2 KiB: pass 3 needs no block scan
        if (wc) {
            atomicAdd(&s_cnt, wc);
            atomicMax(&s_last, wl);
        }
    }
    __syncthreads();
    if (tid == 0)
        agg[tile] = ((uint64_t)s_cnt << 32) | s_last;
}

// exclusive {sum of counts, max of ends} over the tiles, in tile order.  One block: warp w owns a contiguous range of
// tiles and walks it in coalesced groups of 32 (a REDUX pair per group for the range totals, then, with the totals of the
// earlier warps known, a shuffle scan per group that writes the prefixes).
__global__ void __launch_bounds__(1024)
    split_scan_kernel(const uint64_t* __restrict__ agg, uint32_t ntiles, uint64_t* __restrict__ prefix,
                      unsigned long long* total_chars) {
    __shared__ unsigned long long s_c[32];
    __shared__ uint32_t s_l[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const uint32_t per = ((ntiles + 31) / 32 + 31) & ~31u; // tiles per warp, a multiple of 32
    const uint32_t t0 = min((uint32_t)wid * per, ntiles), t1 = min(t0 + per, ntiles);
    unsigned long long c = 0;
    uint32_t l = 0;
#pragma unroll 4
    for (uint32_t t = t0 + lane; t < t1; t += 32) {
        const uint64_t a = __ldg(agg + t);
        c += a >> 32;
        l = max(l, (uint32_t)a);
    }
    const uint32_t c_lo = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)c), c_hi = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)(c >> 32));
    (void)c_hi; // (a warp's range holds < 2^32 newlines: at most 2^26 tiles... the low word is exact per lane, sums below)
    unsigned long long wc = c;
#pragma unroll
    for (int d = 16; d; d >>= 1)
        wc += shfl_down64(wc, d);
    const uint32_t wl = __reduce_max_sync(0xFFFFFFFFu, l);
    (void)c_lo;
    if (lane == 0) {
        s_c[wid] = wc;
        s_l[wid] = wl;
    }
    __syncthreads();
    unsigned long long run_c = 0; // totals of the warps before mine
    uint32_t run_l = 0;
    for (int w = 0; w < wid; ++w) {
        run_c += s_c[w];
        run_l = max(run_l, s_l[w]);
    }
    for (uint32_t tb = t0; tb < t1; tb += 32) {
        const uint32_t t = tb + lane;
        const uint64_t a = t < t1 ? __ldg(agg + t) : 0ull;
        const uint32_t ac = (uint32_t)(a >> 32), al = (uint32_t)a;
        uint32_t ic = ac, il = al;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t tc = __shfl_up_sync(0xFFFFFFFFu, ic, d), tl = __shfl_up_sync(0xFFFFFFFFu, il, d);
            if (lane >= d) {
                ic += tc;
                il = max(il, tl);
            }
        }
        uint32_t el = __shfl_up_sync(0xFFFFFFFFu, il, 1);
        if (lane == 0)
            el = 0;
        if (t < t1)
            prefix[t] = ((uint64_t)((uint32_t)(run_c + (ic - ac)) & 0x3FFFFFFFu) << 32) | max(run_l, el);
        run_c += __shfl_sync(0xFFFFFFFFu, ic, 31);
        run_l = max(run_l, __shfl_sync(0xFFFFFFFFu, il, 31));
    }
    if (tid == 1023)
        *total_chars = run_c; // un-truncated count (the table index keeps 30 bits): > 2^30 pieces is an error
}

// Pass 3.  Persistent and warp-autonomous: a warp takes UNITS of 8 KiB (four mask words per lane, a quarter of a tile) in
// a grid stride -- units are independent, so a static stride is safe -- with the masks, the tile prefix and the per-warp
// counts of its next unit already requested.  It numbers its lines from {tile prefix, counts of the 2 KiB pieces before
// it} (two REDUX, no block barrier), compacts the newline positions into a list in shared memory and then emits
// LINE-parallel: lane j writes line j, so the table stores are coalesced and no lane idles behind a neighbour that owns
// three lines.  (One mask word per lane and iteration was instruction-bound: ~150 warp instructions per 2 KiB, most of
// them the fixed part -- scans, address arithmetic, prefetch.)  With probes the prefix DFAs are staged once per block
// and candidate lines collect in a per-warp queue until 32 of them fill a probe step.
constexpr uint32_t kSplitList = 192;   // newline positions a warp compacts per unit (8 KiB: lines of >= 43 bytes on average;
                                       // denser text takes the per-lane path)
constexpr uint32_t kEmitQueue = 64;    // per warp: candidate lines waiting until 32 of them fill a probe step
template <bool PROBE>
__global__ void __launch_bounds__(1024, 2)
    split_emit_kernel(const uint8_t* __restrict__ buf, uint32_t len, uint32_t shift,
                      const uint16_t* __restrict__ masks /* newline bits, then (PROBE) candidate bits */,
                      const uint64_t* __restrict__ prefix, const uint64_t* __restrict__ wagg, uint32_t ntiles,
                      uint32_t* __restrict__ out_off, uint32_t* __restrict__ out_len, uint32_t cap, uint32_t* n_out,
                      SplitProbe pr) {
    __shared__ uint32_t s_list[32][kSplitList];
    __shared__ uint32_t s_wq[PROBE ? 32 : 1][PROBE ? kEmitQueue : 1];
    __shared__ typename std::conditional<PROBE, ProbeSmem, uint32_t>::type s_probe;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    uint32_t qn = 0; // (warp-uniform) lines in the warp's queue
    if constexpr (PROBE) {
        probe_stage(pr, s_probe);
        __syncthreads();
    }
    // the lane's 16 chunks = four 64-bit words of newline bits
    auto mask_ptr = [&](uint32_t unit) { return reinterpret_cast<const uint4*>(masks) + ((uint64_t)unit * 32 + lane) * 2; };
    auto prefetch_unit = [&](uint32_t unit) { // the next unit's masks -> L2
        asm volatile("prefetch.global.L2 [%0];" ::"l"(mask_ptr(unit)));
    };
    // line k = [start, p); cand: can its first byte start a match (recorded by pass 1 at the newline in front of it).
    // Returns true when the line still has to be probed.
    auto line_out = [&](uint32_t k, uint32_t start, uint32_t p, uint32_t cand) -> bool {
        if (k >= cap)
            return false;
        out_off[k] = start;
        out_len[k] = p - start;
        if constexpr (PROBE) {
            const uint32_t ll = p - start;
            if (ll && cand)
                return true;
            pr.flags[k] = ll ? 0 : (uint8_t)pr.empty_flags;
        }
        return false;
    };
    // 32 queued lines, one per lane (a first version queued per BLOCK and probed between barriers: candidates that
    // overflowed that queue were walked by single lanes from global memory, which dominated the kernel's instructions)
    auto probe_step = [&](uint32_t first, uint32_t count) {
        if constexpr (PROBE) {
            if ((uint32_t)lane < count) {
                const uint32_t kk = s_wq[wid][first + lane];
                pr.flags[kk] = probe_line_smem(pr, s_probe, buf + out_off[kk], out_len[kk]);
            }
        }
    };
    const uint16_t* cand16 = masks + (uint64_t)ntiles * kSplitTileChunks;
    auto cand_at = [&](uint32_t start) -> uint32_t { // candidate bit of the line that starts at `start`
        if (!PROBE || !start)
            return 1;
        const uint64_t vp = (uint64_t)start - 1 + shift;
        return ((uint32_t)__ldg(cand16 + (vp >> 4)) >> (vp & 15)) & 1u;
    };
    const uint32_t nunits = ntiles * 8, ustride = gridDim.x * 32;
    uint32_t unit = blockIdx.x * 32 + wid;
    uint64_t prefix_n = 0, wa_n = 0;
    if (unit < nunits) {
        prefix_n = __ldg(prefix + (unit >> 3));
        wa_n = __ldg(wagg + (uint64_t)(unit >> 3) * 32 + lane);
    }
    for (; unit < nunits; unit += ustride) {
        {
            const uint64_t tile_prefix = prefix_n, wa = wa_n;
            const uint32_t un = unit + ustride;
            if (un < nunits) {
                prefetch_unit(un);
                prefix_n = __ldg(prefix + (un >> 3));
                wa_n = __ldg(wagg + (uint64_t)(un >> 3) * 32 + lane);
            }
            const uint32_t sub = unit & 7;
            const uint64_t vpos0 = ((uint64_t)unit * 32 + lane) * 256; // the lane's 256 bytes
            const uint4* mp = mask_ptr(unit);
            const uint4 q0 = __ldg(mp), q1 = __ldg(mp + 1);
            uint64_t mk[4] = {q0.x | ((uint64_t)q0.y << 32), q0.z | ((uint64_t)q0.w << 32), q1.x | ((uint64_t)q1.y << 32),
                              q1.z | ((uint64_t)q1.w << 32)};
            const uint32_t cnt = __popcll(mk[0]) + __popcll(mk[1]) + __popcll(mk[2]) + __popcll(mk[3]);
            // the 2 KiB pieces of the tile before my unit: their line count and the end of their last newline
            const uint32_t before = lane < sub * 4 ? 0xFFFFFFFFu : 0u;
            const uint32_t my_off = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)(wa >> 32) & before);
            uint32_t my_start = __reduce_max_sync(0xFFFFFFFFu, (uint32_t)wa & before);
            if (!my_start)
                my_start = OpCountMax::maxv(tile_prefix);
            uint32_t inc = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, inc, d);
                if (lane >= d)
                    inc += t;
            }
            const uint32_t total = __shfl_sync(0xFFFFFFFFu, inc, 31);
            const uint32_t k0 = OpCountMax::count(tile_prefix) + my_off;
            uint32_t end_start = my_start; // start of the piece that is open after the unit's last newline
            if (total <= kSplitList) {
                uint32_t idx = inc - cnt;
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    uint64_t m = mk[w];
                    while (m) {
                        const int b = __ffsll((long long)m) - 1;
                        m &= m - 1;
                        s_list[wid][idx++] = (uint32_t)(vpos0 + 64 * w + b - shift);
                    }
                }
                __syncwarp();
                for (uint32_t j0 = 0; j0 < total; j0 += 32) {
                    const uint32_t j = j0 + lane, k = (k0 + j) & 0x3FFFFFFFu;
                    bool want = false;
                    if (j < total) {
                        const uint32_t start = j ? s_list[wid][j - 1] + 1 : my_start;
                        want = line_out(k, start, s_list[wid][j], cand_at(start));
                    }
                    if constexpr (PROBE) {
                        const uint32_t bal = __ballot_sync(0xFFFFFFFFu, want);
                        if (want)
                            s_wq[wid][qn + __popc(bal & ((1u << lane) - 1u))] = k;
                        qn += __popc(bal);
                        __syncwarp(); // queue entries and the table entries of these lines are visible to the warp
                        if (qn >= 32) {
                            probe_step(qn - 32, 32);
                            qn -= 32;
                        }
                    }
                }
                if (total)
                    end_start = s_list[wid][total - 1] + 1;
                __syncwarp();
            } else {
                // dense text: every lane writes its own lines
                uint32_t last = 0;
#pragma unroll
                for (int w = 0; w < 4; ++w)
                    if (mk[w])
                        last = (uint32_t)(vpos0 + 64 * w + (63 - __clzll((long long)mk[w])) + 1 - shift);
                const uint32_t has = __ballot_sync(0xFFFFFFFFu, cnt != 0);
                const uint32_t below = has & ((1u << lane) - 1u);
                const uint32_t prev_last = __shfl_sync(0xFFFFFFFFu, last, below ? 31 - __clz(below) : 0);
                end_start = __shfl_sync(0xFFFFFFFFu, last, 31 - __clz(has)); // (has != 0: total > 0)
                uint32_t k = k0 + (inc - cnt), start = below ? prev_last : my_start;
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    uint64_t m = mk[w];
                    while (m) {
                        const int b = __ffsll((long long)m) - 1;
                        m &= m - 1;
                        const uint32_t p = (uint32_t)(vpos0 + 64 * w + b - shift);
                        if (line_out(k & 0x3FFFFFFFu, start, p, cand_at(start))) {
                            if constexpr (PROBE)
                                pr.flags[k & 0x3FFFFFFFu] = probe_line_smem(pr, s_probe, buf + start, p - start);
                        }
                        ++k;
                        start = p + 1;
                    }
                }
            }
            if (unit == nunits - 1 && lane == 0) {
                // inclusive total of the whole buffer: the unterminated last piece, if any
                uint32_t k = (k0 + total) & 0x3FFFFFFFu;
                if (end_start < len) {
                    if (k < cap) {
                        out_off[k] = end_start;
                        out_len[k] = len - end_start;
                        if (PROBE)
                            pr.flags[k] = probe_line(pr, buf + end_start, len - end_start);
                    }
                    ++k;
                }
                *n_out = k;
            }
        }
    }
    if constexpr (PROBE)
        probe_step(0, qn); // what is left in the warp's queue
}

uint64_t split_scratch_bytes(uint64_t len, bool probe) {
    const uint64_t nt = (len + 16 + kSplitTileChunks * 16 - 1) / (kSplitTileChunks * 16);
    return nt * 16 + nt * 256 + nt * kSplitTileChunks * (probe ? 4 : 2) + 256;
}

template <bool PROBE>
static int launch_split_impl(const uint8_t* d_buf, uint32_t len, uint8_t split_char, uint32_t* d_off, uint32_t* d_len,
                             uint32_t cap, uint32_t* d_n_out, unsigned long long* d_total, uint64_t* d_scratch,
                             const SplitProbe& pr, cudaStream_t st) {
    uint32_t shift = (uint32_t)((uintptr_t)d_buf & 15u);
    uint32_t splat = split_char * 0x01010101u;
    const uint32_t nt = (uint32_t)(((uint64_t)len + shift + kSplitTileChunks * 16 - 1) / (kSplitTileChunks * 16));
    uint64_t* agg = d_scratch;
    uint64_t* prefix = d_scratch + nt;
    uint64_t* wagg = d_scratch + 2 * (uint64_t)nt;
    uint16_t* masks = reinterpret_cast<uint16_t*>(d_scratch + 34 * (uint64_t)nt);
    split_mask_kernel<PROBE><<<nt, 1024, 0, st>>>(d_buf, len, shift, splat, masks, (uint64_t)nt * kSplitTileChunks, agg,
                                                 wagg, pr);
    split_scan_kernel<<<1, 1024, 0, st>>>(agg, nt, prefix, d_total);
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    const uint32_t grid = std::min<uint32_t>((nt + 3) / 4, (uint32_t)sms * 2);
    split_emit_kernel<PROBE><<<grid, 1024, 0, st>>>(d_buf, len, shift, masks, prefix, wagg, nt, d_off, d_len, cap,
                                                   d_n_out, pr);
    return 3;
}

int launch_split(const uint8_t* d_buf, uint32_t len, uint8_t split_char, uint32_t* d_off, uint32_t* d_len,
                 uint32_t cap, uint32_t* d_n_out, unsigned long long* d_total, uint64_t* d_scratch, cudaStream_t st) {
    SplitProbe pr;
    memset(&pr, 0, sizeof pr);
    return launch_split_impl<false>(d_buf, len, split_char, d_off, d_len, cap, d_n_out, d_total, d_scratch, pr, st);
}

int launch_split_probe(const MlConfig& cfg, const uint8_t* d_buf, uint32_t len, uint32_t* d_off, uint32_t* d_len,
                       uint8_t* d_flags, uint32_t cap, uint32_t* d_n_out, unsigned long long* d_total,
                       uint64_t* d_scratch, cudaStream_t st) {
    SplitProbe pr;
    memset(&pr, 0, sizeof pr);
    pr.blob[0] = cfg.blob_start;
    pr.blob[1] = cfg.blob_cont;
    pr.blob[2] = cfg.blob_end;
    for (int p = 0; p < 3; ++p) {
        memcpy(pr.first[p], cfg.first[p], sizeof pr.first[p]);
        for (int w = 0; w < 8; ++w)
            pr.any_first[w] |= cfg.first[p][w]; // (the set of an absent pattern is empty)
    }
    pr.empty_flags = cfg.empty_flags;
    pr.flags = d_flags;
    return launch_split_impl<true>(d_buf, len, '\n', d_off, d_len, cap, d_n_out, d_total, d_scratch, pr, st);
}

// ================================================================================================ sums
template <int THREADS, int ITEMS>
__global__ void __launch_bounds__(THREADS)
    exclusive_sum_kernel(const uint32_t* __restrict__ in, uint64_t n, uint64_t* __restrict__ out, uint64_t* total,
                         volatile uint64_t* desc, uint32_t* ticket, uint32_t ntiles) {
    __shared__ uint64_t s_scan[THREADS / 32 + 1];
    __shared__ uint32_t s_tile;
    __shared__ uint64_t s_part[4];
    __shared__ uint32_t s_flag[4];
    const int tid = threadIdx.x;
    if (tid == 0)
        s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t base = (uint64_t)tile * THREADS * ITEMS + (uint64_t)tid * ITEMS;
    uint32_t v[ITEMS];
    uint64_t sum = 0;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        v[k] = (base + k < n) ? in[base + k] : 0u;
        sum += v[k];
    }
    uint64_t tot;
    uint64_t ex = block_exclusive_scan<OpSum, THREADS>(sum, tot, s_scan);
    uint64_t run = lookback_block<OpSum, 4>(desc, tile, tot, s_part, s_flag) + ex;
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        if (base + k < n)
            out[base + k] = run;
        run += v[k];
    }
    if (tile == ntiles - 1 && tid == THREADS - 1)
        *total = run;
}

void launch_exclusive_sum(const uint32_t* d_in, uint64_t n, uint64_t* d_out, uint64_t* d_total, uint64_t* d_desc,
                          uint32_t* d_ticket, cudaStream_t st) {
    uint32_t ntiles = scan_tiles(n);
    if (ntiles == 0)
        return;
    exclusive_sum_kernel<kScanThreads, kScanItems>
        <<<ntiles, kScanThreads, 0, st>>>(d_in, n, d_out, d_total, (volatile uint64_t*)d_desc, d_ticket, ntiles);
}

// ================================================================================================ regex (baseline)
__global__ void label_sizes_kernel(const uint32_t* __restrict__ ev_len, uint64_t n, uint32_t* __restrict__ sizes) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        sizes[i] = (ev_len[i] + 1 + 7) & ~7u;
}
void launch_label_sizes(const uint32_t* d_ev_len, uint64_t n, uint32_t* d_sizes, cudaStream_t st) {
    if (!n)
        return;
    label_sizes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ev_len, n, d_sizes);
}

// max and sum of the event lengths (sizes the shared-memory label area of the persistent kernels)
__global__ void __launch_bounds__(256)
    len_stats_kernel(const uint32_t* __restrict__ ev_len, uint64_t n, unsigned long long* __restrict__ out /* [2] */) {
    uint32_t mx = 0;
    unsigned long long sum = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t l = ev_len[i];
        mx = max(mx, l);
        sum += l;
    }
    for (int d = 16; d; d >>= 1) {
        mx = max(mx, __shfl_down_sync(0xFFFFFFFFu, mx, d));
        sum += __shfl_down_sync(0xFFFFFFFFu, sum, d);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&out[0], (unsigned long long)mx);
        atomicAdd(&out[1], sum);
    }
}
void launch_len_stats(const uint32_t* d_ev_len, uint64_t n, unsigned long long* d_out, cudaStream_t st) {
    if (!n)
        return;
    unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256, 1184);
    len_stats_kernel<<<grid, 256, 0, st>>>(d_ev_len, n, d_out);
}

// Ragged batches: events are visited in descending length-bucket order so that the 32 lanes of a warp walk lines
// of similar length (a warp costs as much as its longest line).  bucket = 2*floor(log2(len)) + next bit.
__device__ __forceinline__ uint32_t len_bucket(uint32_t len) {
    if (len < 2)
        return len;
    uint32_t lg = 31 - __clz(len);
    return 2 * lg + ((len >> (lg - 1)) & 1);
}
__global__ void __launch_bounds__(256)
    bucket_hist_kernel(const uint32_t* __restrict__ ev_len, uint64_t n, uint32_t* __restrict__ hist /* [64] */) {
    __shared__ uint32_t sh[64];
    if (threadIdx.x < 64)
        sh[threadIdx.x] = 0;
    __syncthreads();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(&sh[len_bucket(ev_len[i])], 1u);
    __syncthreads();
    if (threadIdx.x < 64 && sh[threadIdx.x])
        atomicAdd(&hist[threadIdx.x], sh[threadIdx.x]);
}
__global__ void bucket_scan_kernel(uint32_t* hist /* [64] in: counts, out: start cursor, longest bucket first;
                                                       [64] out: 1 = ragged batch (lengths span > 2 adjacent buckets) */) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        uint32_t run = 0;
        int lo = 64, hi = -1;
        for (int b = 63; b >= 0; --b) {
            uint32_t c = hist[b];
            if (c) {
                lo = b;
                if (hi < 0)
                    hi = b;
            }
            hist[b] = run;
            run += c;
        }
        hist[64] = (hi - lo >= 2) ? 1u : 0u;
    }
}
__global__ void __launch_bounds__(256)
    bucket_fill_kernel(const uint32_t* __restrict__ ev_len, uint64_t n, uint32_t* __restrict__ cursor,
                       uint32_t* __restrict__ order) {
    // block-local ranking keeps the global atomics to one per (block, bucket)
    __shared__ uint32_t cnt[64], basep[64];
    if (threadIdx.x < 64)
        cnt[threadIdx.x] = 0;
    __syncthreads();
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t b = 0, r = 0;
    if (i < n) {
        b = len_bucket(ev_len[i]);
        r = atomicAdd(&cnt[b], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 64 && cnt[threadIdx.x])
        basep[threadIdx.x] = atomicAdd(&cursor[threadIdx.x], cnt[threadIdx.x]);
    __syncthreads();
    if (i < n)
        order[basep[b] + r] = (uint32_t)i;
}
void launch_length_order(const uint32_t* d_ev_len, uint64_t n, uint32_t* d_hist64, uint32_t* d_order,
                         cudaStream_t st) {
    if (!n)
        return;
    cudaMemsetAsync(d_hist64, 0, 65 * sizeof(uint32_t), st);
    unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256, 1184);
    bucket_hist_kernel<<<grid, 256, 0, st>>>(d_ev_len, n, d_hist64);
    bucket_scan_kernel<<<1, 32, 0, st>>>(d_hist64);
    bucket_fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ev_len, n, d_hist64, d_order);
}

// lc_regex_match on the kernels that always produce captures: parse status (0 ok, 2 keys mismatch = matched) -> bool
__global__ void status_to_bool_kernel(uint8_t* __restrict__ st, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        st[i] = st[i] != 1 ? 1 : 0;
}
void launch_status_to_bool(uint8_t* d_status, uint64_t n, cudaStream_t st) {
    if (n)
        status_to_bool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_status, n);
}

// One thread per event; tables read through the read-only path from global memory.
__global__ void __launch_bounds__(128)
    regex_parse_basic_kernel(const void* __restrict__ blob, uint32_t mode, uint32_t G, const uint8_t* __restrict__ base,
                             const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len, uint64_t n,
                             uint32_t nkeys, uint8_t* __restrict__ status, uint32_t* __restrict__ cap_off,
                             uint32_t* __restrict__ cap_len, const uint64_t* __restrict__ lab_off,
                             uint16_t* __restrict__ lab) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    LcProgView v = lc_view(blob);
    const uint32_t off = ev_off[i], len = ev_len[i];
    const uint8_t* s = base + off;
    uint32_t slots[2 * LC_MAX_GROUPS];
    for (uint32_t k = 0; k < 2 * G; ++k)
        slots[k] = LC_SLOT_UNSET;
    bool ok;
    if (mode == LC_MODE_FWD1) {
        ok = lc_full_match_fwd1(v, s, len, slots);
    } else {
        uint16_t* my = lab + lab_off[i];
        ok = lc_rev_label(v, s, len, my) && lc_fwd_walk(v, s, len, my, slots);
    }
    uint8_t st = ok ? (G + 1 <= nkeys ? 2 : 0) : 1;
    status[i] = st;
    uint32_t* co = cap_off + i * G;
    uint32_t* cl = cap_len + i * G;
    for (uint32_t g = 0; g < G; ++g) {
        uint32_t o = 0, l = 0;
        if (st == 0) {
            lc_slots_to_cap(slots, g, len, &o, &l);
            o += off;
        }
        co[g] = o;
        cl[g] = l;
    }
}

void launch_regex_parse_basic(const void* d_blob, uint32_t mode, uint32_t ngroups, const uint8_t* d_base,
                              const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                              uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len, const uint64_t* d_lab_off,
                              uint16_t* d_lab, cudaStream_t st) {
    if (!n)
        return;
    regex_parse_basic_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(
        d_blob, mode, ngroups, d_base, d_ev_off, d_ev_len, n, nkeys, d_status, d_cap_off, d_cap_len, d_lab_off, d_lab);
}


// ================================================================================================ regex (fast path)
// Thread-per-event kernels with the whole automaton blob staged in shared memory.
//
// Two-pass matcher: the reverse pass needs one label per input position.  Labels of short events live in
// shared memory, packed 4 (u8) or 2 (u16) per 32-bit word; a warp's words are interleaved
// [word][lane] so that lane == bank and the accesses are conflict-free whatever position each lane is at.
// Events longer than the shared-memory budget bump-allocate their label words from a global scratch slab
// (order is irrelevant); if the slab is exhausted the kernel raises *overflow and the host retries bigger.

struct LabSmem {
    uint32_t* p; // warp region base + lane
    __device__ __forceinline__ void st(uint32_t widx, uint32_t v) const { p[widx * 32] = v; }
    __device__ __forceinline__ uint32_t ld(uint32_t widx) const { return p[widx * 32]; }
};
struct LabGlobal {
    uint32_t* p;
    __device__ __forceinline__ void st(uint32_t widx, uint32_t v) const { p[widx] = v; }
    __device__ __forceinline__ uint32_t ld(uint32_t widx) const { return p[widx]; }
};

// byte `a` (absolute address) through aligned 32-bit read-only loads; `cur`/`cur_word` cache the last word
__device__ __forceinline__ uint32_t ld_byte(const uint8_t* __restrict__ base, uint64_t a, uint64_t& cur_word,
                                            uint32_t& cur) {
    uint64_t w = a >> 2;
    if (w != cur_word) {
        cur_word = w;
        cur = __ldg(reinterpret_cast<const uint32_t*>(base) + w);
    }
    return (cur >> (8 * (uint32_t)(a & 3))) & 0xFFu;
}

template <class LabT, class Lab>
__device__ __forceinline__ bool twopass_event(const LcProgView& v, const LabT* __restrict__ rev_byte,
                                              const uint8_t* __restrict__ abase, uint64_t a0, uint32_t n, Lab lab,
                                              uint32_t* slots) {
    constexpr uint32_t PER = 4 / sizeof(LabT);     // labels per word
    constexpr uint32_t BITS = 8 * sizeof(LabT);
    constexpr uint32_t MASK = (1u << BITS) - 1u;
    // ---- reverse labelling
    uint32_t d = v.h->rev_start;
    uint32_t lw = d << (BITS * (n % PER));
    uint64_t cw = ~0ull;
    uint32_t cur = 0;
    for (uint32_t i = n; i-- > 0;) {
        uint32_t b = ld_byte(abase, a0 + i, cw, cur);
        d = rev_byte[d * 256 + b];
        if (d == LC_REV_DEAD)
            return false;
        if ((i % PER) == PER - 1) {
            lab.st((i + 1) / PER, lw);
            lw = 0;
        }
        lw |= d << (BITS * (i % PER));
    }
    lab.st(0, lw);
    // ---- guided forward walk
    const uint32_t cols = v.h->fwd_cols;
    const uint32_t npc = v.h->npc;
    uint32_t w = 0, pk = 0;
    cw = ~0ull;
    for (uint32_t i = 0; i <= n; ++i) {
        if ((i % PER) == 0 && i)
            lw = lab.ld(i / PER);
        uint32_t l = (lw >> (BITS * (i % PER))) & MASK;
        uint32_t e = v.fwd[(w * npc + pk) * cols + l];
        if (e == LC_NONE_ENTRY)
            return false;
        uint32_t a = LC_ENTRY_ACT(e);
        if (a)
            lc_apply_action(v, a, i, slots);
        w = LC_ENTRY_NEXT(e);
        if (npc > 1 && i < n)
            pk = v.class_pc[v.byte_class[ld_byte(abase, a0 + i, cw, cur)]];
    }
    return true;
}

__device__ __forceinline__ bool fwd1_event(const LcProgView& v, const uint32_t* __restrict__ fwd_byte,
                                           const uint8_t* __restrict__ abase, uint64_t a0, uint32_t n,
                                           uint32_t* slots) {
    uint32_t w = 0;
    uint64_t cw = ~0ull;
    uint32_t cur = 0;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t b = ld_byte(abase, a0 + i, cw, cur);
        uint32_t e = fwd_byte[w * 256 + b];
        if (e == LC_NONE_ENTRY)
            return false;
        uint32_t a = LC_ENTRY_ACT(e);
        if (a)
            lc_apply_action(v, a, i, slots);
        w = LC_ENTRY_NEXT(e);
    }
    uint32_t e = v.fwd_eof[w];
    if (e == LC_NONE_ENTRY)
        return false;
    uint32_t a = LC_ENTRY_ACT(e);
    if (a)
        lc_apply_action(v, a, n, slots);
    return true;
}


// ---- fast two-pass kernel over the host-built fast blob (lc_tables.h: LcFastHeader) -------------------------
// Input bytes are consumed as 16-byte aligned chunks and the label of position i is stored at virtual index
// q = i + (address & 15), so input words and label words share their boundaries: full chunks run 16 fully
// unrolled steps without per-byte predicates.
//   reverse step : b = PRMT(word) ; d4 = rev[d4 * 65 + b] ; lw = lw * 256 + d4          (labels pre-multiplied by 4)
//   forward step : addr = PRMT(entry, lw) ; entry = fwd[addr] ; if (entry & 0xFF) slots[..] = pos   (predicated)
// Capture boundaries are rare per line but happen on SOME lane at almost every step of a warp, so they must not
// branch: a single-slot boundary is one predicated local store; only multi-slot boundaries take a branch.
struct FastView {
    const LcFastHeader* h;
    const uint8_t* rev;
    const uint8_t* fwd; // byte-addressed, 256-byte rows
    const uint8_t* cx;
    const uint64_t* masks;
};

__device__ __noinline__ void fast_multi_action(const FastView& f, uint32_t addr, uint32_t pos, uint32_t* slots) {
    uint64_t m = f.masks[f.cx[addr >> 2]];
    while (m) {
        int s = __ffsll((long long)m) - 1;
        slots[s] = pos;
        m &= m - 1;
    }
}

// slots live in shared memory ([thread][slot], odd word pitch): a capture boundary is one predicated STS
#define LC_FWD_STEP(K, POS)                                                                                           \
    {                                                                                                                  \
        const uint32_t addr = __byte_perm(e, lw, 0x2214 + (K)) /* (row << 8) | label4; entry byte 2 is always 0 */;                                                        \
        e = *reinterpret_cast<const uint32_t*>(fwd + addr);                                                            \
        const uint32_t sl = e & 0xFFu;                                                                                 \
        if (sl)                                                                                                        \
            *reinterpret_cast<uint32_t*>(slots_m4 + sl) = (POS);                                                       \
        if (MULTI && (int32_t)e < 0)                                                                                   \
            fast_multi_action(f, addr, (POS), reinterpret_cast<uint32_t*>(slots_m4 + 4));                              \
    }

template <bool MULTI, class Lab>
__device__ __forceinline__ bool twopass_event_fast(const FastView& f, const uint4* __restrict__ chunks, uint32_t mis,
                                                   uint32_t n, Lab lab, uint8_t* slots_m4 /* slot area - 4 bytes */) {
    const uint32_t Q = n + mis;
    const int top = (int)(Q >> 4);
    const uint32_t rev_start4 = f.h->rev_start4;
    const uint8_t* __restrict__ rev = f.rev;
    uint32_t d4 = rev_start4;
    // ---- reverse labelling (software-pipelined chunk loads)
    uint4 nxt = make_uint4(0, 0, 0, 0);
    if ((uint32_t)top * 16 < Q)
        nxt = __ldg(chunks + top);
    for (int qc = top; qc >= 0; --qc) {
        const uint32_t lo = (uint32_t)qc * 16;
        const uint4 vv = nxt;
        if (qc > 0)
            nxt = __ldg(chunks + qc - 1);
        const uint32_t w[4] = {vv.x, vv.y, vv.z, vv.w};
        if (lo >= mis && lo + 15 < Q) {
#pragma unroll
            for (int wi = 3; wi >= 0; --wi) {
                const uint32_t x = w[wi];
                uint32_t lw;
                d4 = rev[d4 * 65 + __byte_perm(x, 0, 0x4443)];
                lw = d4;
                d4 = rev[d4 * 65 + __byte_perm(x, 0, 0x4442)];
                lw = lw * 256 + d4;
                d4 = rev[d4 * 65 + __byte_perm(x, 0, 0x4441)];
                lw = lw * 256 + d4;
                d4 = rev[d4 * 65 + __byte_perm(x, 0, 0x4440)];
                lw = lw * 256 + d4;
                lab.st(qc * 4 + wi, lw);
            }
        } else {
#pragma unroll
            for (int wi = 3; wi >= 0; --wi) {
                const uint32_t x = w[wi];
                uint32_t lw = 0;
                bool any = false;
#pragma unroll
                for (int k = 3; k >= 0; --k) {
                    const uint32_t q = lo + wi * 4 + k;
                    if (q == Q) {
                        lw |= rev_start4 << (8 * k);
                        any = true;
                    } else if (q < Q && q >= mis) {
                        d4 = rev[d4 * 65 + ((x >> (8 * k)) & 0xFFu)];
                        lw |= d4 << (8 * k);
                        any = true;
                    }
                }
                if (any)
                    lab.st(qc * 4 + wi, lw);
            }
        }
        if (d4 == 0)
            return false;
    }
    // ---- guided forward walk; d4 == 4 * label of position 0
    const uint8_t* __restrict__ fwd = f.fwd;
    if (*reinterpret_cast<const uint32_t*>(fwd + d4) == LC_NONE_ENTRY)
        return false;
    uint32_t e = 0; // current entry: row index in bits 8.., START row = 0
    for (int qc = 0; qc <= top; ++qc) {
        const uint32_t lo = (uint32_t)qc * 16;
        const uint32_t pos0 = lo - mis;
        if (lo >= mis && lo + 15 <= Q) {
#pragma unroll
            for (int wi = 0; wi < 4; ++wi) {
                const uint32_t lw = lab.ld(qc * 4 + wi);
                LC_FWD_STEP(0, pos0 + wi * 4 + 0)
                LC_FWD_STEP(1, pos0 + wi * 4 + 1)
                LC_FWD_STEP(2, pos0 + wi * 4 + 2)
                LC_FWD_STEP(3, pos0 + wi * 4 + 3)
            }
        } else {
#pragma unroll
            for (int wi = 0; wi < 4; ++wi) {
                const uint32_t q0 = lo + wi * 4;
                if (q0 + 3 < mis || q0 > Q)
                    continue;
                const uint32_t lw = lab.ld(qc * 4 + wi);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint32_t q = q0 + k;
                    if (q >= mis && q <= Q)
                        LC_FWD_STEP(k, q - mis)
                }
            }
        }
    }
    return true;
}

template <bool MULTI>
__global__ void __launch_bounds__(1024, 1)
    regex_twopass_fast_kernel(const uint4* __restrict__ blob, uint32_t blob_bytes, const uint8_t* __restrict__ base,
                              const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len, uint64_t n,
                              uint32_t nkeys, uint8_t* __restrict__ status, uint32_t* __restrict__ cap_off,
                              uint32_t* __restrict__ cap_len, uint32_t lab_words, uint32_t slot_pitch,
                              uint32_t* __restrict__ scratch, unsigned long long scratch_words,
                              unsigned long long* bump, uint32_t* overflow, unsigned long long* next_batch, const uint32_t* __restrict__ order) {
    extern __shared__ uint4 smem[];
    for (uint32_t k = threadIdx.x; k < blob_bytes / 16; k += blockDim.x)
        smem[k] = __ldg(blob + k);
    __syncthreads();
    const uint8_t* sb = reinterpret_cast<const uint8_t*>(smem);
    FastView f;
    f.h = reinterpret_cast<const LcFastHeader*>(sb);
    f.rev = sb + f.h->off_rev;
    f.fwd = sb + f.h->off_fwd;
    f.cx = sb + f.h->off_cx;
    f.masks = reinterpret_cast<const uint64_t*>(sb + f.h->off_masks);
    const uint32_t G = f.h->ngroups;
    // shared memory: [blob][labels: warps x lab_words x 32 words][slots: threads x slot_pitch words]
    uint32_t* lab_base = reinterpret_cast<uint32_t*>(smem) + blob_bytes / 4;
    uint32_t* slots = lab_base + (size_t)(blockDim.x / 32) * lab_words * 32 + (size_t)threadIdx.x * slot_pitch;
    uint8_t* slots_m4 = reinterpret_cast<uint8_t*>(slots) - 4;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (;;) {
        unsigned long long batch = 0;
        if (lane == 0)
            batch = atomicAdd(next_batch, 32ull);
        batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
        if (batch >= n)
            break;
        if (batch + lane >= n)
            continue;
        const uint64_t i = order ? order[batch + lane] : batch + lane;
        const uint32_t off = ev_off[i], len = ev_len[i];
        for (uint32_t k = 0; k < 2 * G; ++k)
            slots[k] = LC_SLOT_UNSET;
        const uint64_t a16 = (uint64_t)(uintptr_t)(base + off);
        const uint32_t mis16 = (uint32_t)(a16 & 15u);
        const uint4* chunks = reinterpret_cast<const uint4*>(a16 - mis16);
        const uint32_t need = (len + mis16) / 4 + 1;
        bool ok;
        if (need <= lab_words) {
            LabSmem lab{lab_base + (size_t)wid * lab_words * 32 + lane};
            ok = twopass_event_fast<MULTI>(f, chunks, mis16, len, lab, slots_m4);
        } else {
            unsigned long long at = atomicAdd(bump, (unsigned long long)need);
            if (at + need > scratch_words) {
                atomicExch(overflow, 1u);
                ok = false;
            } else {
                LabGlobal lab{scratch + at};
                ok = twopass_event_fast<MULTI>(f, chunks, mis16, len, lab, slots_m4);
            }
        }
        uint8_t st = ok ? (G + 1 <= nkeys ? 2 : 0) : 1;
        status[i] = st;
        uint32_t* co = cap_off + i * G;
        uint32_t* cl = cap_len + i * G;
        for (uint32_t g = 0; g < G; ++g) {
            uint32_t o = 0, l = 0;
            if (st == 0) {
                lc_slots_to_cap(slots, g, len, &o, &l);
                o += off;
            }
            co[g] = o;
            cl[g] = l;
        }
    }
}

int launch_regex_twopass_fast(const void* d_fast_blob, uint32_t blob_bytes, bool multi, uint32_t ngroups,
                              const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                              uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                              uint32_t lab_words, uint32_t threads, uint32_t grid, uint32_t* d_scratch,
                              uint64_t scratch_words, unsigned long long* d_bump, uint32_t* d_overflow,
                              unsigned long long* d_next_batch, const uint32_t* d_order, cudaStream_t st) {
    if (!n)
        return 0;
    const uint32_t slot_pitch = fast_slot_pitch(ngroups);
    size_t smem = fast_smem_bytes(blob_bytes, ngroups, lab_words, threads);
    auto k = multi ? regex_twopass_fast_kernel<true> : regex_twopass_fast_kernel<false>;
    cudaError_t er = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er != cudaSuccess)
        return (int)er;
    k<<<grid, threads, smem, st>>>((const uint4*)d_fast_blob, blob_bytes, d_base, d_ev_off, d_ev_len, n, nkeys, d_status,
                                   d_cap_off, d_cap_len, lab_words, slot_pitch, d_scratch, scratch_words, d_bump,
                                   d_overflow, d_next_batch, d_order);
    return (int)cudaGetLastError();
}

// ---- stride-2 two-pass kernel over the fast2 layout (lc_tables.h: LcFast2Header) -------------------------------
// Two input bytes per dependent look-up and one label byte per byte pair: half the dependency chain and half the
// shared-memory label footprint of the stride-1 kernel, so twice the lines in flight at half the latency each.
//   reverse pair step : off = cls_hi[b1] + cls_lo[b0] ; e = t2[row + off] ; row = e & 0xFFFF (chain) ; P = e >> 16
//   forward pair step : idx = PRMT(entry, labels) = walker << 8 | P ; entry = f2[idx] (chain: PRMT + LDS) ;
//                       entry bytes 1,2 -> up to two predicated 16-bit STS into the thread's capture slots
// Pairs are aligned on even addresses; an odd first byte / odd end position is peeled as a single step.
struct Fast2Dev {
    const uint8_t* cls; // byte -> class (u8, conflict-free for ASCII)
    const uint8_t* t2;  // byte addressed u32 entries
    const uint8_t* f2;  // byte addressed u32 entries
    uint32_t rev_start, row_bytes, ncls;
};

struct LabSmemB { // label words interleaved [word][lane]; byte-level access for peeled / partial chunks
    uint32_t* p;
    __device__ __forceinline__ void st(uint32_t widx, uint32_t v) const { p[widx * 32] = v; }
    __device__ __forceinline__ uint32_t ld(uint32_t widx) const { return p[widx * 32]; }
    __device__ __forceinline__ void stb(uint32_t j, uint32_t v) const {
        reinterpret_cast<uint8_t*>(p + (j >> 2) * 32)[j & 3] = (uint8_t)v;
    }
};
struct LabGlobalB {
    uint32_t* p;
    __device__ __forceinline__ void st(uint32_t widx, uint32_t v) const { p[widx] = v; }
    __device__ __forceinline__ uint32_t ld(uint32_t widx) const { return p[widx]; }
    __device__ __forceinline__ void stb(uint32_t j, uint32_t v) const { reinterpret_cast<uint8_t*>(p)[j] = (uint8_t)v; }
};

#define LC2_REV_PAIR(X, HI)                                                                                           \
    {                                                                                                                  \
        const uint32_t c1 = t.cls[__byte_perm((X), 0, (HI) ? 0x4443 : 0x4441)];                                        \
        const uint32_t c0 = t.cls[__byte_perm((X), 0, (HI) ? 0x4442 : 0x4440)];                                        \
        const uint32_t e2 = *reinterpret_cast<const uint32_t*>(t.t2 + row + ((c1 * t.ncls + c0) << 2));               \
        row = e2 & 0xFFFFu;                                                                                            \
        P = e2 >> 16;                                                                                                  \
    }

// COMPACT: labels hold pair_id * 4 and PRMT(entry, labels) is the byte offset of the next entry (256-byte rows);
// otherwise PRMT gives the entry index in 256-entry rows.
#define LC2_FWD_PAIR(K, POS)                                                                                          \
    {                                                                                                                  \
        const uint32_t idx = __byte_perm(e, lw, 0x3304 + (K)); /* walker << 8 | label */                               \
        e = *reinterpret_cast<const uint32_t*>(t.f2 + (COMPACT ? idx : idx * 4));                                      \
        const uint32_t sa = (e >> 8) & 0x7Fu, sb = (e >> 16) & 0x7Fu;                                                  \
        if (sa)                                                                                                        \
            *reinterpret_cast<uint16_t*>(slots_m2 + sa) = (uint16_t)(POS);                                             \
        if (sb)                                                                                                        \
            *reinterpret_cast<uint16_t*>(slots_m2 + sb) = (uint16_t)((POS) + 1);                                       \
        if (MULTI && (e & LC_FAST2_ACT_MULTI))                                                                         \
            lc_fast2_pair_slow(v, idx >> 8, (idx & 0xFFu) >> (COMPACT ? 2 : 0), (POS),                                 \
                               reinterpret_cast<uint16_t*>(slots_m2 + 2));                                             \
    }

// One 16-byte chunk of the reverse pass: 8 byte pairs, highest first.  Pairs are restricted to [qlo, Qe).
// STORE: label words go to lab word index wbase (+1); partial chunks store single label bytes.
template <bool STORE, class Lab>
__device__ __forceinline__ void fast2_rev_chunk(const Fast2Dev& t, const uint4 vv, uint32_t lo, uint32_t qlo,
                                                uint32_t Qe, uint32_t& row, Lab lab, uint32_t wbase) {
    uint32_t P;
    if (lo >= qlo && lo + 16 <= Qe) {
        uint32_t lw;
        LC2_REV_PAIR(vv.w, 1)
        lw = P;
        LC2_REV_PAIR(vv.w, 0)
        lw = lw * 256 + P;
        LC2_REV_PAIR(vv.z, 1)
        lw = lw * 256 + P;
        LC2_REV_PAIR(vv.z, 0)
        lw = lw * 256 + P;
        if (STORE)
            lab.st(wbase + 1, lw);
        LC2_REV_PAIR(vv.y, 1)
        lw = P;
        LC2_REV_PAIR(vv.y, 0)
        lw = lw * 256 + P;
        LC2_REV_PAIR(vv.x, 1)
        lw = lw * 256 + P;
        LC2_REV_PAIR(vv.x, 0)
        lw = lw * 256 + P;
        if (STORE)
            lab.st(wbase, lw);
    } else {
        const uint32_t wd[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
        for (int pi = 7; pi >= 0; --pi) {
            const uint32_t q = lo + 2 * pi;
            if (q >= qlo && q < Qe) {
                LC2_REV_PAIR(wd[pi >> 1], pi & 1)
                if (STORE)
                    lab.stb(wbase * 4 + pi, P);
            }
        }
    }
}

// One 16-byte chunk of the forward walk: pairs restricted to [qlo, Qf); labels at word index wbase (+1).
template <bool MULTI, bool COMPACT, class Lab>
__device__ __forceinline__ void fast2_fwd_chunk(const LcFast2View& v, const Fast2Dev& t, uint32_t lo, uint32_t mis,
                                                uint32_t qlo, uint32_t Qf, uint32_t& e, Lab lab, uint32_t wbase,
                                                uint8_t* slots_m2) {
    const uint32_t pos0 = lo - mis;
    if (lo >= qlo && lo + 16 <= Qf) {
        uint32_t lw = lab.ld(wbase);
        LC2_FWD_PAIR(0, pos0 + 0)
        LC2_FWD_PAIR(1, pos0 + 2)
        LC2_FWD_PAIR(2, pos0 + 4)
        LC2_FWD_PAIR(3, pos0 + 6)
        lw = lab.ld(wbase + 1);
        LC2_FWD_PAIR(0, pos0 + 8)
        LC2_FWD_PAIR(1, pos0 + 10)
        LC2_FWD_PAIR(2, pos0 + 12)
        LC2_FWD_PAIR(3, pos0 + 14)
    } else {
#pragma unroll
        for (int wi = 0; wi < 2; ++wi) {
            const uint32_t q0 = lo + wi * 8;
            if (q0 + 8 <= qlo || q0 >= Qf)
                continue;
            const uint32_t lw = lab.ld(wbase + wi);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t q = q0 + 2 * k;
                if (q >= qlo && q < Qf)
                    LC2_FWD_PAIR(k, q - mis)
            }
        }
    }
}

// Whole event with all labels resident (`lab` holds (n + mis) / 8 + 1 words).
template <bool MULTI, bool COMPACT, class Lab>
__device__ __forceinline__ bool fast2_event(const LcFast2View& v, const Fast2Dev& t, const uint8_t* __restrict__ s,
                                            const uint4* __restrict__ chunks, uint32_t mis, uint32_t n, Lab lab,
                                            uint8_t* slots_m2 /* slot area - 2 bytes */, bool bool_only) {
    const uint32_t Q = n + mis;
    const uint32_t qlo = mis + (mis & 1);      // first even position whose pair lies inside the event
    const uint32_t Qe = Q & ~1u;               // reverse pairs cover [qlo, Qe)
    const uint32_t Qf = (Q + 1) & ~1u;         // forward pairs cover [qlo, Qf)
    const uint32_t ncls = v.h->ncls, nrev = v.h->nrev;
    uint32_t d = t.rev_start;
    // ---- reverse: peel the byte whose pair partner is the end position
    if ((Q & 1) && n) {
        const uint32_t b = s[n - 1];
        d = v.rev1[d * ncls + t.cls[b]];
        if (!d)
            return false;
        lab.stb((Q - 1) >> 1, v.pid[d * nrev + t.rev_start]);
    }
    uint32_t row = d * t.row_bytes;
    if (Qe > qlo) {
        const int c_hi = (int)((Qe - 1) >> 4), c_lo = (int)(qlo >> 4);
        uint4 nxt = __ldg(chunks + c_hi);
        for (int qc = c_hi; qc >= c_lo; --qc) {
            const uint4 vv = nxt;
            if (qc > c_lo)
                nxt = __ldg(chunks + qc - 1);
            fast2_rev_chunk<true>(t, vv, (uint32_t)qc * 16, qlo, Qe, row, lab, (uint32_t)qc * 2);
            if (row == 0)
                return false;
        }
    }
    d = row / t.row_bytes;
    // the first byte sits in the second slot of a pair whose first slot precedes the event
    if ((mis & 1) && n) {
        d = v.rev1[d * ncls + t.cls[s[0]]];
        if (!d)
            return false;
    }
    // ---- forward; d == label of position mis
    if (v.fwd1[d] == LC_NONE_ENTRY)
        return false;
    if (bool_only)
        return true; // regex_match as a boolean needs no captures: the reverse pass decides
    uint32_t e = 0; // forward entry; byte 0 = current walker
    if (mis & 1)
        e = lc_fast2_single(v, 0, d, 0, reinterpret_cast<uint16_t*>(slots_m2 + 2));
    if (Qf > qlo) {
        const int c_lo = (int)(qlo >> 4), c_hi = (int)((Qf - 1) >> 4);
        for (int qc = c_lo; qc <= c_hi; ++qc)
            fast2_fwd_chunk<MULTI, COMPACT>(v, t, (uint32_t)qc * 16, mis, qlo, Qf, e, lab, (uint32_t)qc * 2, slots_m2);
    }
    if (!(Q & 1))
        (void)lc_fast2_single(v, e & 0xFFu, t.rev_start, n, reinterpret_cast<uint16_t*>(slots_m2 + 2));
    return true;
}

// Long event: its labels would not fit the thread's shared-memory area.  Checkpointed evaluation keeps the
// footprint constant: (1) one reverse pass without label stores records the reverse state at every block
// boundary (2 bytes per block, in the global slab); (2) block by block, left to right, the reverse pass is re-run
// over just that block from its checkpoint to regenerate the block's labels in shared memory, followed by the
// forward walk over the block.  1.5x the look-ups of the resident variant, but full occupancy and no label
// traffic to HBM.  KC = chunks (16 B) per block, 2 * KC <= lab_words.
template <bool MULTI, bool COMPACT, class Lab>
__device__ __forceinline__ bool fast2_event_blocked(const LcFast2View& v, const Fast2Dev& t,
                                                    const uint8_t* __restrict__ s, const uint4* __restrict__ chunks,
                                                    uint32_t mis, uint32_t n, Lab lab, uint32_t KC,
                                                    uint16_t* __restrict__ ck, uint8_t* slots_m2, bool bool_only) {
    const uint32_t Q = n + mis;
    const uint32_t qlo = mis + (mis & 1);
    const uint32_t Qe = Q & ~1u;
    const uint32_t Qf = (Q + 1) & ~1u;
    const uint32_t ncls = v.h->ncls, nrev = v.h->nrev;
    const uint32_t nb = (Q >> 4) / KC + 1; // blocks 0 .. nb-1 cover chunks [j*KC, (j+1)*KC)
    uint32_t d = t.rev_start;
    uint32_t peel_label = 0;
    if ((Q & 1) && n) {
        d = v.rev1[d * ncls + t.cls[s[n - 1]]];
        if (!d)
            return false;
        peel_label = v.pid[d * nrev + t.rev_start];
    }
    uint32_t row = d * t.row_bytes;
    ck[nb] = (uint16_t)row; // state entering the top block
    // ---- pass 1: reverse over the whole event, checkpoints only
    if (Qe > qlo) {
        const int c_hi = (int)((Qe - 1) >> 4), c_lo = (int)(qlo >> 4);
        uint4 nxt = __ldg(chunks + c_hi);
        for (int qc = c_hi; qc >= c_lo; --qc) {
            const uint4 vv = nxt;
            if (qc > c_lo)
                nxt = __ldg(chunks + qc - 1);
            fast2_rev_chunk<false>(t, vv, (uint32_t)qc * 16, qlo, Qe, row, lab, 0);
            if (row == 0)
                return false;
            if ((uint32_t)qc % KC == 0)
                ck[(uint32_t)qc / KC] = (uint16_t)row; // state at the lower edge of block qc / KC
        }
    }
    d = row / t.row_bytes;
    if ((mis & 1) && n) {
        d = v.rev1[d * ncls + t.cls[s[0]]];
        if (!d)
            return false;
    }
    if (v.fwd1[d] == LC_NONE_ENTRY)
        return false;
    if (bool_only)
        return true;
    uint32_t e = 0;
    if (mis & 1)
        e = lc_fast2_single(v, 0, d, 0, reinterpret_cast<uint16_t*>(slots_m2 + 2));
    // ---- pass 2: per block, regenerate labels then walk forward
    const int rc_hi = Qe > qlo ? (int)((Qe - 1) >> 4) : -1, rc_lo = (int)(qlo >> 4);
    const int fc_hi = Qf > qlo ? (int)((Qf - 1) >> 4) : -1, fc_lo = (int)(qlo >> 4);
    for (uint32_t j = 0; j < nb; ++j) {
        const int b_lo = (int)(j * KC), b_hi = (int)((j + 1) * KC) - 1;
        const uint32_t wshift = j * KC * 2; // label words of this block start at 0
        // reverse over the block from the state at its upper edge
        int c1 = b_hi < rc_hi ? b_hi : rc_hi, c0 = b_lo > rc_lo ? b_lo : rc_lo;
        if (c1 >= c0) {
            uint32_t r2 = (b_hi < rc_hi) ? ck[j + 1] : ck[nb];
            uint4 nxt = __ldg(chunks + c1);
            for (int qc = c1; qc >= c0; --qc) {
                const uint4 vv = nxt;
                if (qc > c0)
                    nxt = __ldg(chunks + qc - 1);
                fast2_rev_chunk<true>(t, vv, (uint32_t)qc * 16, qlo, Qe, r2, lab, (uint32_t)qc * 2 - wshift);
            }
        }
        // the peeled top pair (Q-1, Q) belongs to the block that holds chunk (Q-1) >> 4
        if ((Q & 1) && n && (int)((Q - 1) >> 4) >= b_lo && (int)((Q - 1) >> 4) <= b_hi)
            lab.stb(((Q - 1) >> 1) - wshift * 4, peel_label);
        c1 = b_hi < fc_hi ? b_hi : fc_hi;
        c0 = b_lo > fc_lo ? b_lo : fc_lo;
        for (int qc = c0; qc <= c1; ++qc)
            fast2_fwd_chunk<MULTI, COMPACT>(v, t, (uint32_t)qc * 16, mis, qlo, Qf, e, lab, (uint32_t)qc * 2 - wshift, slots_m2);
    }
    if (!(Q & 1))
        (void)lc_fast2_single(v, e & 0xFFu, t.rev_start, n, reinterpret_cast<uint16_t*>(slots_m2 + 2));
    return true;
}

template <bool MULTI, bool COMPACT>
__global__ void __launch_bounds__(1024, 1)
    regex_fast2_kernel(const uint4* __restrict__ blob, uint32_t blob_bytes, const uint8_t* __restrict__ base,
                       const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len, uint64_t n,
                       uint32_t nkeys, uint8_t* __restrict__ status, uint32_t* __restrict__ cap_off,
                       uint32_t* __restrict__ cap_len, uint32_t lab_words, uint32_t slot_pitch /* halfwords */,
                       uint32_t* __restrict__ scratch, unsigned long long scratch_words, unsigned long long* bump,
                       uint32_t* overflow, unsigned long long* next_batch, const uint32_t* __restrict__ order) {
    extern __shared__ uint4 smem[];
    for (uint32_t k = threadIdx.x; k < blob_bytes / 16; k += blockDim.x)
        smem[k] = __ldg(blob + k);
    __syncthreads();
    const LcFast2View v = lc_fast2_view(smem);
    Fast2Dev t;
    t.cls = v.cls;
    t.t2 = v.t2;
    t.f2 = reinterpret_cast<const uint8_t*>(v.f2);
    t.ncls = v.h->ncls;
    t.rev_start = v.h->rev_start;
    t.row_bytes = v.h->row_bytes;
    const uint32_t G = v.h->ngroups;
    // shared memory: [blob][labels: warps x lab_words x 32 words][slots: threads x slot_pitch halfwords]
    uint32_t* lab_base = reinterpret_cast<uint32_t*>(smem) + blob_bytes / 4;
    uint16_t* slots = reinterpret_cast<uint16_t*>(lab_base + (size_t)(blockDim.x / 32) * lab_words * 32) +
                      (size_t)threadIdx.x * slot_pitch;
    uint8_t* slots_m2 = reinterpret_cast<uint8_t*>(slots) - 2;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // results leave through a per-warp staging area (the warp's label words, free once the walk is done) so that
    // the capture tables are written with fully coalesced 128-byte stores instead of 32 scattered rows
    const bool bool_only = cap_off == nullptr; // lc_regex_match: status[i] = 1 match / 0 no match, no captures
    const uint32_t pitch = G | 1u;
    const bool coop = !bool_only && order == nullptr && G > 0 && (size_t)lab_words * 32 >= (size_t)2 * 32 * pitch;
    uint32_t* stg = lab_base + (size_t)wid * lab_words * 32;
    for (;;) {
        unsigned long long batch = 0;
        if (lane == 0)
            batch = atomicAdd(next_batch, 32ull);
        batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
        if (batch >= n)
            break;
        const bool valid = batch + lane < n;
        const uint64_t i = valid ? (order ? order[batch + lane] : batch + lane) : 0;
        uint32_t off = 0, len = 0;
        uint8_t st = 1;
        if (valid) {
            off = ev_off[i];
            len = ev_len[i];
            for (uint32_t k = 0; k < 2 * G; ++k)
                slots[k] = LC_SLOT16_UNSET;
            const uint8_t* s = base + off;
            const uint64_t a16 = (uint64_t)(uintptr_t)s;
            const uint32_t mis16 = (uint32_t)(a16 & 15u);
            const uint4* chunks = reinterpret_cast<const uint4*>(a16 - mis16);
            const uint32_t need = (len + mis16) / 8 + 1; // label words: one byte per byte pair
            bool ok;
            if (need <= lab_words) {
                LabSmemB lab{lab_base + (size_t)wid * lab_words * 32 + lane};
                ok = fast2_event<MULTI, COMPACT>(v, t, s, chunks, mis16, len, lab, slots_m2, bool_only);
            } else {
                // long event: checkpointed blocks, labels stay in shared memory, 2 B per block in the global slab
                const uint32_t KC = lab_words / 2;
                const uint32_t nb = ((len + mis16) >> 4) / KC + 1;
                const unsigned long long ckw = (nb + 2) / 2 + 1;
                unsigned long long at = atomicAdd(bump, ckw);
                if (at + ckw > scratch_words) {
                    atomicExch(overflow, 1u);
                    ok = false;
                } else {
                    LabSmemB lab{lab_base + (size_t)wid * lab_words * 32 + lane};
                    ok = fast2_event_blocked<MULTI, COMPACT>(v, t, s, chunks, mis16, len, lab, KC,
                                                    reinterpret_cast<uint16_t*>(scratch + at), slots_m2, bool_only);
                }
            }
            st = ok ? (G + 1 <= nkeys ? 2 : 0) : 1;
            status[i] = bool_only ? (ok ? 1 : 0) : st;
        }
        if (bool_only)
            continue;
        if (coop) {
            __syncwarp();
            if (valid)
                for (uint32_t g = 0; g < G; ++g) {
                    uint32_t o = 0, l = 0;
                    if (st == 0) {
                        lc_slots16_to_cap(slots, g, len, &o, &l);
                        o += off;
                    }
                    stg[lane * pitch + g] = o;
                    stg[32 * pitch + lane * pitch + g] = l;
                }
            __syncwarp();
            const uint64_t left = n - batch;
            const uint32_t total = (uint32_t)(left < 32 ? left : 32) * G;
            uint32_t* go = cap_off + batch * G;
            uint32_t* gl = cap_len + batch * G;
            for (uint32_t j = lane; j < total; j += 32) {
                const uint32_t line = j / G, k = j - line * G;
                go[j] = stg[line * pitch + k];
                gl[j] = stg[32 * pitch + line * pitch + k];
            }
            __syncwarp();
        } else if (valid) {
            uint32_t* co = cap_off + i * G;
            uint32_t* cl = cap_len + i * G;
            for (uint32_t g = 0; g < G; ++g) {
                uint32_t o = 0, l = 0;
                if (st == 0) {
                    lc_slots16_to_cap(slots, g, len, &o, &l);
                    o += off;
                }
                co[g] = o;
                cl[g] = l;
            }
        }
    }
}

int launch_regex_fast2(const void* d_blob, uint32_t blob_bytes, bool multi, bool compact, uint32_t ngroups,
                       const uint8_t* d_base,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                       uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len, uint32_t lab_words,
                       uint32_t threads, uint32_t grid, uint32_t* d_scratch, uint64_t scratch_words,
                       unsigned long long* d_bump, uint32_t* d_overflow, unsigned long long* d_next_batch,
                       const uint32_t* d_order, cudaStream_t st) {
    if (!n)
        return 0;
    const uint32_t slot_pitch = fast2_slot_pitch(ngroups);
    size_t smem = fast2_smem_bytes(blob_bytes, ngroups, lab_words, threads);
    auto k = compact ? (multi ? regex_fast2_kernel<true, true> : regex_fast2_kernel<false, true>)
                     : (multi ? regex_fast2_kernel<true, false> : regex_fast2_kernel<false, false>);
    cudaError_t er = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er != cudaSuccess)
        return (int)er;
    k<<<grid, threads, smem, st>>>((const uint4*)d_blob, blob_bytes, d_base, d_ev_off, d_ev_len, n, nkeys, d_status,
                                   d_cap_off, d_cap_len, lab_words, slot_pitch, d_scratch, scratch_words, d_bump,
                                   d_overflow, d_next_batch, d_order);
    return (int)cudaGetLastError();
}

// ---- single-pass tagged-DFA kernel (lc_tables.h: LcTdfaHeader) ----------------------------------------------
// One forward pass, two input bytes per dependent look-up, no labels: per byte pair
//   c0 = cls[b0] ; c1 = cls[b1] ; e = t2[row + (c0 * ncls + c1) * 4] ; row = e & 0xFFFF           (the chain)
//   bytes 2,3 of e -> up to two predicated 16-bit STS into the thread's register file in shared memory
// The per-line state is the register file alone (2 * groups + spares halfwords), so all 32 warps stay resident
// whatever the line length, and the input is read exactly once.
// ---- staged input: the automaton fed through shared memory -----------------------------------------------------
// Why: with one line per lane, a per-lane 16-byte LDG touches 32 different 128-byte lines, i.e. 32 L1 tag
// wavefronts for 512 bytes -- measured to cost more than the automaton's own look-ups.  Here the warp fetches its
// 32 lines COOPERATIVELY: one cp.async (LDGSTS) instruction moves 4 full 128-byte lines (8 lanes x 16 B each, 4
// wavefronts) straight into a per-warp staging tile (tile_slot): line j of the warp owns the 128-byte row j, so every
// global line of an LDGSTS lands in one shared-memory row, and its 8 chunks are permuted by j inside the row, so that
// the per-lane LDS.128 reads of one chunk column stay bank-conflict free.  Lanes then consume their own line from
// the tile.  All hot-loop accesses use 32-bit shared-window addresses: the class
// table sits on a 256-byte boundary (address = PRMT(byte, base)), and the pair table's row offsets are rebased to
// absolute addresses while the automaton is staged, so a pair step is
//   PRMT PRMT LDS.U8 LDS.U8 IMAD LEA LDS LOP  + two predicated STS.U16 for capture boundaries.
#define LCT_STAGE_CHUNKS 8u /* 16-byte chunks per line per stage: 128 B = one L1 line per 8-lane group */

// The one place that knows the staging tile's layout: shared address of chunk q of line j (only q mod 8 counts) in
// the 4 KB tile at `tile` (128-byte aligned).  Row j holds line j, chunk q in 16-byte unit (q ^ j) mod 8: the 8 lanes
// that copy one global line write one row, and the 8 lanes 8g..8g+7 that read one chunk column hit 8 distinct bank
// quads.  Since only j mod 8 enters the permutation, tile_slot(tile + 1024 * g, r, q) == tile_slot(tile, 8 * g + r, q).
__device__ __forceinline__ uint32_t tile_slot(uint32_t tile, uint32_t j, uint32_t q) {
    return tile + (j << 7) + (((q ^ j) & 7u) << 4);
}

__device__ __forceinline__ uint32_t lds_u8(uint32_t a) {
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8_v(uint32_t a) { // mutable data (staging tile)
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds_u32_v(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint2 lds_u64_v(uint32_t a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint4 lds_u128_v(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u16(uint32_t a, uint32_t v) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((unsigned short)v) : "memory");
}
__device__ __forceinline__ void sts_u64(uint32_t a, uint32_t x, uint32_t y) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
// 16-byte cp.async if i < n.  The predicate lives inside the asm, so that the compiler forms the addresses once for
// all copies of a stage instead of sinking their arithmetic into one branch per copy.
__device__ __forceinline__ void cp_async_16_if_lt(uint32_t dst, const void* src, uint32_t i, uint32_t n) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %2, %3;\n\t@p cp.async.cg.shared.global [%0], [%1], 16;\n\t}"
                 ::"r"(dst), "l"(src), "r"(i), "r"(n)
                 : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

struct TdfaAbs {
    uint32_t cls;       // absolute shared address of the class table (256-byte aligned)
    uint32_t t2;        // absolute shared address of row 0 (= the dead state)
    uint32_t ncls;
    uint32_t row_bytes;
    uint32_t inv_row;   // ceil(2^32 / row_bytes): state = umulhi(row - t2, inv_row)
    uint32_t skip;      // absolute shared address of the run-skipping table (u32 per state, lc_tables.h)
};

// (Tried and measured slower on C2: a power-of-two row pitch with the address formed as row | index * 4 -- the same
// class pair of different states then always shares a bank; and storing both boundary fields under one predicate --
// two instructions fewer per pair but more shared-memory wavefronts.)
// Pair step over the STAGED tables (tdfa_stage_blob re-encodes them for this loop): the class table holds class * 4,
// a pair-table entry is  next_row_address << 16 | (register of the 2nd step) << 8 | (register of the 1st step)  (register
// fields = byte offset of the register + 2, 0 = none).  With the row in the HIGH half the address of the next look-up is
// one LEA.HI -- (entry >> 16) + index -- instead of a mask and an add, one instruction less on the dependent chain of
// every pair: PRMT PRMT LDS.U8 LDS.U8 IMAD LEA.HI LDS + two predicated STS.U16 for capture boundaries.
// ROWX = the address of the current row: `row` for the first pair of a chunk, (e_prev >> 16) afterwards.
// The capture stores keep the field test, the address and the store in one asm block each, so that ptxas takes the
// predicate and the masked field from one LOP3 instead of masking the second field twice.
__device__ __forceinline__ void sts_u16_reg_a(uint32_t e, uint32_t regs_m2, uint32_t pos) {
    asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 f;\n\tand.b32 f, %0, 0x7F;\n\tsetp.ne.u32 p, f, 0;\n\t"
                 "add.u32 f, f, %1;\n\t@p st.shared.u16 [f], %2;\n\t}"
                 ::"r"(e), "r"(regs_m2), "h"((unsigned short)pos) : "memory");
}
__device__ __forceinline__ void sts_u16_reg_b(uint32_t e, uint32_t regs_m2, uint32_t pos) {
    asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 f;\n\tand.b32 f, %0, 0x7F00;\n\tsetp.ne.u32 p, f, 0;\n\t"
                 "shr.u32 f, f, 8;\n\tadd.u32 f, f, %1;\n\t@p st.shared.u16 [f], %2;\n\t}"
                 ::"r"(e), "r"(regs_m2), "h"((unsigned short)pos) : "memory");
}
#define LCS_PAIR(ROWX, X, HI, POS)                                                                                     \
    {                                                                                                                  \
        const uint32_t c0 = lds_u8(__byte_perm((X), t.cls, (HI) ? 0x7652 : 0x7650));                                   \
        const uint32_t c1 = lds_u8(__byte_perm((X), t.cls, (HI) ? 0x7653 : 0x7651));                                   \
        const uint32_t e = lds_u32((ROWX) + (c0 * t.ncls + c1));                                                       \
        sts_u16_reg_a(e, regs_m2, (POS));                                                                              \
        sts_u16_reg_b(e, regs_m2, (POS) + 1);                                                                          \
        e_prev = e;                                                                                                    \
    }

// Out-of-line redo of one chunk whose fast pass met an entry that sets several registers in one step: single steps
// with full op lists over the same pairs, from the state at chunk entry.  Re-executing the single-register sets
// in order on top of the fast pass leaves exactly the sequential result.  Returns the state after the chunk.
__device__ __noinline__ uint32_t tdfa_chunk_slow(const LcTdfaView v, uint32_t st, uint4 vv, uint32_t pos0,
                                                 uint16_t* rg) {
    const uint32_t wd[4] = {vv.x, vv.y, vv.z, vv.w};
    for (uint32_t pi = 0; pi < 8; ++pi) {
        const uint32_t w = wd[pi >> 1] >> ((pi & 1) * 16);
        st = lc_tdfa_single(v, st, w & 0xFFu, pos0 + 2 * pi, rg);
        st = lc_tdfa_single(v, st, (w >> 8) & 0xFFu, pos0 + 2 * pi + 1, rg);
    }
    return st;
}

// A chunk that is not fully covered by byte pairs of the line (its first and/or last chunk): optional odd first
// byte, the pairs inside [qlo, Qe), optional odd last byte.  At most two calls per line.  caddr = shared address
// of the chunk in the tile, lo = index of its first byte in the line's 16-byte aligned frame.
__device__ __noinline__ uint32_t tdfa_partial_chunk(const LcTdfaView v, const TdfaAbs t, uint32_t row, uint32_t caddr,
                                                    uint32_t lo, uint32_t mis, uint32_t len, uint32_t regs_m2,
                                                    uint16_t* rg, uint32_t sink) {
    const uint32_t Q = len + mis, qlo = mis + (mis & 1), Qe = Q & ~1u;
    if (lo == 0 && (mis & 1)) { // odd first byte (frame index mis lies in chunk 0): single step from the start state
        const uint32_t st1 = lc_tdfa_single(v, v.h->start, lds_u8_v(caddr + mis), 0, rg);
        row = t.t2 + st1 * t.row_bytes;
    }
    const uint32_t a = lo > qlo ? lo : qlo, b = lo + 16 < Qe ? lo + 16 : Qe;
    for (uint32_t q = a; q < b; q += 2) {
        const uint32_t b0 = lds_u8_v(caddr + (q - lo)), b1 = lds_u8_v(caddr + (q - lo) + 1);
        const uint32_t e = lds_u32(row + (lds_u8(t.cls | b0) * t.ncls + lds_u8(t.cls | b1))); // (staged encoding)
        const uint32_t nrow = e >> 16;
        if (nrow == sink) {
            const uint32_t s1 = lc_tdfa_single(v, __umulhi(row - t.t2, t.inv_row), b0, q - mis, rg);
            row = t.t2 + t.row_bytes * lc_tdfa_single(v, s1, b1, q + 1 - mis, rg);
        } else {
            const uint32_t sa = e & 0x7Fu, sb = (e >> 8) & 0x7Fu;
            if (sa)
                sts_u16(regs_m2 + sa, q - mis);
            if (sb)
                sts_u16(regs_m2 + sb, q + 1 - mis);
            row = nrow;
        }
    }
    if ((Q & 1) && Q - 1 >= qlo && ((Q - 1) >> 4) == (lo >> 4)) { // odd last byte
        const uint32_t st1 = lc_tdfa_single(v, __umulhi(row - t.t2, t.inv_row), lds_u8_v(caddr + ((Q - 1) & 15)),
                                            len - 1, rg);
        row = t.t2 + st1 * t.row_bytes;
    }
    return row;
}

// (Tile fill alternatives measured on C2 and dropped as slower: cp.async.ca instead of .cg; LDG.128 into registers
// followed by STS.128 -- the loads stall the issuing warp and the extra live registers spill under the 64-register
// cap.  The shared-memory side of LDGSTS is cheap only when the 8 lanes of one global line write one 128-byte row:
// with the earlier [chunk][line ^ chunk] tile, where every lane of an LDGSTS wrote a row of its own, the fill alone
// (tools/tile_fill_probe.py, C2's 4 Mi x 256 B lines in HBM) took 1.39-1.59x as long as with tile_slot's layout.)
//
// The warp's 32 lines (one per lane; line = frame of `len` bytes starting `mis` bytes into its first 16-byte chunk,
// chunk list published in the warp's info slots as {first chunk index, chunk count}) walk through automaton `t`
// stage by stage: cooperative fetch of 8 chunks per line into the tile, then every lane consumes its own line.
// Lanes whose `row` is `dead` on entry (or becomes dead) only help fetching.  Returns the final row.
struct TdfaLoader {
    const uint4* gbase16; // 16-byte aligned base of the arena
    uint32_t ld_q;        // loader role: chunk column of lines ld_L0 + r (r = 0..7), ld_L0 = (lane >> 3) * 8
    uint32_t ld_info;     // info slots of those lines
    uint32_t ld_rows;     // tile + ld_L0 * 128: tile_slot(ld_rows, r, q) is the slot of chunk q of line ld_L0 + r
    uint32_t tile_abs;    // this warp's 4 KB tile (128-byte aligned)
    uint32_t lane;
    __device__ __forceinline__ void init(const uint8_t* base, uint32_t info_abs, uint32_t tile, uint32_t ln) {
        gbase16 = reinterpret_cast<const uint4*>((uintptr_t)base & ~(uintptr_t)15);
        ld_q = ln & 7;
        ld_info = info_abs + (ln >> 3) * 64;
        ld_rows = tile + (ln >> 3) * 1024;
        tile_abs = tile;
        lane = ln;
    }
    // shared address of chunk k of this lane's own line
    __device__ __forceinline__ uint32_t own(uint32_t k) const { return tile_slot(tile_abs, lane, k); }
    // cooperative fetch of chunks s0..s0+7 of the warp's 32 lines: instruction r moves lines r, r+8, r+16, r+24.
    // The 8 info loads go first, so that the copies do not wait on them one by one.
    __device__ __forceinline__ void stage(uint32_t s0) {
        const uint32_t cidx = s0 + ld_q;
        uint2 inf[8];
#pragma unroll
        for (uint32_t r = 0; r < 8; ++r)
            inf[r] = lds_u64_v(ld_info + r * 8);
#pragma unroll
        for (uint32_t r = 0; r < 8; ++r) // (chunk indices of the arena fit 32 bits: g0 is one)
            cp_async_16_if_lt(tile_slot(ld_rows, r, ld_q), gbase16 + (inf[r].x + cidx), cidx, inf[r].y);
        cp_async_wait_all();
        __syncwarp();
    }
};

template <bool SLOW>
__device__ __forceinline__ uint32_t tdfa_walk_lines(const LcTdfaView& v, const TdfaAbs& t, TdfaLoader& L,
                                                    uint32_t dead, uint32_t sink, uint32_t row, uint32_t len,
                                                    uint32_t mis, uint32_t max_nch, uint32_t regs_m2, uint16_t* rg) {
    // frame of the line: byte j of the line sits at frame index mis + j; pairs cover the even-aligned [qlo, Qe)
    const uint32_t Q = len + mis, qlo = mis + (mis & 1), Qe = Q & ~1u;
    const uint32_t kf_lo = (qlo + 15) >> 4, kf_hi = Qe >> 4; // fully paired chunks: [kf_lo, kf_hi)
    const uint32_t k_tail = len ? (Q - 1) >> 4 : 0;
    const bool has_head = len && !(kf_lo == 0 && kf_hi > 0);        // chunk 0 is not fully paired
    const bool has_tail = len && k_tail >= kf_hi && !(has_head && k_tail == 0);
    for (uint32_t s0 = 0; s0 < max_nch; s0 += LCT_STAGE_CHUNKS) {
        L.stage(s0); // chunks s0..s0+7 of the warp's 32 lines are in the tile when this returns
        // ---- every lane walks its own line through the tile
        if (row != dead && has_head && s0 == 0)
            row = tdfa_partial_chunk(v, t, row, L.own(0), 0, mis, len, regs_m2, rg, sink);
        // The fully paired chunks go in warp lockstep: in step j every lane that is alive and has a j-th fully
        // paired chunk in this stage walks that chunk of its own line, and the others sit the step out.  Run
        // skipping is decided for the warp as a whole, since a warp only saves issue slots when all of its walking
        // lanes skip: inside [^"]* / .* the state maps every byte but (at most) two back to itself without touching a
        // register, so a chunk without those bytes is a no-op.  The exit test runs only when the vote says every
        // walking lane is in such a state; otherwise they all walk their chunk, which is exact either way.
        const uint32_t ka = kf_lo > s0 ? kf_lo : s0;
        const uint32_t kb = kf_hi < s0 + LCT_STAGE_CHUNKS ? kf_hi : s0 + LCT_STAGE_CHUNKS;
        const uint32_t nk = row != dead && kb > ka ? kb - ka : 0;
        for (uint32_t j = 0; __any_sync(0xFFFFFFFFu, j < nk); ++j) {
            const uint32_t k = ka + j;
            // (both loads are in bounds for every lane: its own tile row, and the skip word of a valid row)
            const uint4 vv = lds_u128_v(L.own(k));
            const uint32_t sk = lds_u32(t.skip + __umulhi(row - t.t2, t.inv_row) * 4);
            const bool walk = row != dead && j < nk;
            if (__all_sync(0xFFFFFFFFu, sk != 0 || !walk)) {
                const uint32_t w[4] = {vv.x, vv.y, vv.z, vv.w};
                if (!__any_sync(0xFFFFFFFFu, walk && lc_tdfa_chunk_has_exit(sk, w)))
                    continue;
            }
            if (walk) {
                const uint32_t pos0 = k * 16 - mis;
                const uint32_t row_in = row;
                uint32_t e_prev;
                LCS_PAIR(row, vv.x, 0, pos0 + 0)
                LCS_PAIR(e_prev >> 16, vv.x, 1, pos0 + 2)
                LCS_PAIR(e_prev >> 16, vv.y, 0, pos0 + 4)
                LCS_PAIR(e_prev >> 16, vv.y, 1, pos0 + 6)
                LCS_PAIR(e_prev >> 16, vv.z, 0, pos0 + 8)
                LCS_PAIR(e_prev >> 16, vv.z, 1, pos0 + 10)
                LCS_PAIR(e_prev >> 16, vv.w, 0, pos0 + 12)
                LCS_PAIR(e_prev >> 16, vv.w, 1, pos0 + 14)
                row = e_prev >> 16;
                if (SLOW && row == sink) // some step set several registers: redo this chunk step by step
                    row = t.t2 + t.row_bytes * tdfa_chunk_slow(v, __umulhi(row_in - t.t2, t.inv_row), vv, pos0, rg);
            }
        }
        if (row != dead && has_tail && k_tail - s0 < LCT_STAGE_CHUNKS)
            row = tdfa_partial_chunk(v, t, row, L.own(k_tail), k_tail * 16, mis, len, regs_m2, rg, sink);
        __syncwarp();
    }
    return row;
}

// Stages one automaton: class table at the 256-byte aligned shared address cls_abs, blob right behind it; pair-table
// entries are rebased so that their low 16 bits are the ABSOLUTE shared address of the next row.  All threads call;
// the caller synchronises afterwards.
__device__ __forceinline__ void tdfa_stage_blob(uint8_t* g_cls, uint32_t cls_abs, const uint4* __restrict__ blob,
                                                uint32_t blob_bytes) {
    uint4* g_blob = reinterpret_cast<uint4*>(g_cls + 256);
    for (uint32_t k = threadIdx.x; k < blob_bytes / 16; k += blockDim.x)
        g_blob[k] = __ldg(blob + k);
    __syncthreads();
    const LcTdfaView v = lc_tdfa_view(g_blob);
    const uint32_t t2 = cls_abs + 256 + v.h->off_t2;
    if (t2 + (v.h->nstates + 1) * v.h->row_bytes > 65535u)
        __trap(); // rows could not be addressed with 16 bits: the host must not select this kernel
    if (v.h->ncls > 63)
        __trap(); // class * 4 must fit the byte-wide staged class table
    for (uint32_t k = threadIdx.x; k < 256; k += blockDim.x)
        g_cls[k] = (uint8_t)(v.cls[k] * 4); // pre-multiplied: c0 * ncls + c1 is then the BYTE offset of the entry
    uint32_t* t2w = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(g_blob) + v.h->off_t2);
    const uint32_t nent = (v.h->nstates + 1) * (v.h->row_bytes / 4);
    for (uint32_t k = threadIdx.x; k < nent; k += blockDim.x) {
        // blob entry: row offset | reg of step 1 << 16 | slow << 23 | reg of step 2 << 24  ->  the loop's encoding
        const uint32_t e = t2w[k];
        t2w[k] = ((e & 0xFFFFu) + t2) << 16 | ((e >> 24) & 0x7Fu) << 8 | ((e >> 16) & 0x7Fu);
    }
}

template <bool SLOW>
__global__ void __launch_bounds__(1024, 1)
    regex_tdfa_staged_kernel(const uint4* __restrict__ blob, uint32_t blob_bytes, const uint8_t* __restrict__ base,
                             const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len,
                             uint32_t ev_stride, uint64_t n, uint32_t nkeys, uint8_t* __restrict__ status,
                             uint32_t* __restrict__ cap_off, uint32_t* __restrict__ cap_len,
                             uint32_t reg_pitch /* halfwords */, unsigned long long* next_batch, uint32_t* overflow,
                             const uint32_t* __restrict__ order, const uint32_t* __restrict__ order_flag) {
    extern __shared__ uint4 smem[];
    // carve-out: [pad][class table, 256 B @ 256-aligned][blob][16 B][register files][pad to 128 B]
    // [line info: warps x 32 x 8 B][tiles: warps x 4 KB, 128-byte aligned rows (tile_slot)]
    const uint32_t s0abs = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t cls_abs = (s0abs + 255u) & ~255u;
    uint8_t* g_cls = reinterpret_cast<uint8_t*>(smem) + (cls_abs - s0abs);
    uint4* g_blob = reinterpret_cast<uint4*>(g_cls + 256);
    tdfa_stage_blob(g_cls, cls_abs, blob, blob_bytes);
    __syncthreads();
    const LcTdfaView v = lc_tdfa_view(g_blob);
    TdfaAbs t;
    t.cls = cls_abs;
    t.t2 = cls_abs + 256 + v.h->off_t2;
    t.ncls = v.h->ncls;
    t.row_bytes = v.h->row_bytes;
    t.inv_row = (uint32_t)((0x100000000ull + t.row_bytes - 1) / t.row_bytes);
    t.skip = cls_abs + 256 + v.h->off_skip;
    const uint32_t G = v.h->ngroups;
    const uint32_t invG = G ? 0xFFFFFFFFu / G + 1 : 0; // umulhi(j, invG) == j / G for j < 65536
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint8_t* g_regs0 = reinterpret_cast<uint8_t*>(g_blob) + blob_bytes + 16; // (+16: spare slot)
    uint16_t* wregs = reinterpret_cast<uint16_t*>(g_regs0) + (size_t)wid * 32 * reg_pitch;
    uint16_t* regs = wregs + (size_t)lane * reg_pitch;
    const uint32_t regs_abs = (uint32_t)__cvta_generic_to_shared(regs);
    const uint32_t regs_m2 = regs_abs - 2;
    const uint32_t aux_abs = ((uint32_t)__cvta_generic_to_shared(g_regs0 + (size_t)blockDim.x * reg_pitch * 2) + 127u) &
                             ~127u;
    const uint32_t info_abs = aux_abs + wid * 256;
    const uint32_t tile_abs = aux_abs + nwarps * 256 + wid * (LCT_STAGE_CHUNKS * 512);
    // bounce the class-table address through shared memory so that it lives in a per-thread register: with a
    // uniform-register operand PRMT cannot take its selector as an immediate (one extra MOV per look-up)
    sts_u64(info_abs + lane * 8, cls_abs, 0);
    asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(t.cls) : "r"(info_abs + lane * 8) : "memory");
    const uint32_t base_mis = (uint32_t)((uintptr_t)base & 15);
    const bool bool_only = cap_off == nullptr;
    const uint32_t dead = t.t2, sink = t.t2 + v.h->sink * t.row_bytes;
    uint16_t* rg = regs;
    if (order && order_flag && *order_flag == 0) // the length pre-pass found a uniform batch: natural order
        order = nullptr;
    TdfaLoader L;
    L.init(base, info_abs, tile_abs, lane);
    for (;;) {
        unsigned long long batch = 0;
        if (lane == 0)
            batch = atomicAdd(next_batch, 32ull);
        batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
        if (batch >= n)
            break;
        const bool valid = batch + lane < n;
        // ragged batches: `order` lists the events by descending length bucket, so that the 32 lines of a warp are of
        // similar length (a warp costs its longest line)
        const uint64_t i = (order && valid) ? order[batch + lane] : batch + lane;
        uint32_t off = 0, len = 0, mis = 0, nch = 0, g0 = 0;
        if (valid) {
            off = ev_off[i * ev_stride];
            len = ev_len[i * ev_stride];
            if (len >= 65535u) { // capture registers are 16-bit: regex_tdfa_long_kernel redoes this event afterwards
                atomicExch(overflow, 1u);
                len = 0;
            }
            const uint64_t a = (uint64_t)base_mis + off; // byte offset from gbase16
            mis = (uint32_t)(a & 15);
            g0 = (uint32_t)(a >> 4);
            nch = len ? (mis + len + 15) >> 4 : 0;
            for (uint32_t k = 0; k < G; ++k)
                reinterpret_cast<uint32_t*>(regs)[k] = 0xFFFFFFFFu; // home registers = LC_SLOT16_UNSET
        }
        sts_u64(info_abs + lane * 8, g0, nch);
        const uint32_t max_nch = __reduce_max_sync(0xFFFFFFFFu, nch);
        uint32_t row = t.t2 + v.h->start * t.row_bytes;
        __syncwarp();
        row = tdfa_walk_lines<SLOW>(v, t, L, dead, sink, row, len, mis, max_nch, regs_m2, rg);
        uint32_t st = 1;
        if (valid) {
            bool ok = false;
            const uint32_t fin = v.eof[__umulhi(row - t.t2, t.inv_row)];
            if (fin != LC_NONE_ENTRY) {
                lc_tdfa_run_ops(v, fin, len, rg);
                ok = true;
            }
            st = ok ? (G + 1 <= nkeys ? 2 : 0) : 1;
            status[i] = bool_only ? (ok ? 1 : 0) : (uint8_t)st;
        }
        if (bool_only || G == 0)
            continue;
        if (order) { // rows of the batch are scattered: every lane writes its own
            if (valid) {
                uint32_t* co = cap_off + i * G;
                uint32_t* cl = cap_len + i * G;
                for (uint32_t g = 0; g < G; ++g) {
                    uint32_t o = 0, l = 0;
                    if (st == 0) {
                        lc_slots16_to_cap(regs, g, len, &o, &l);
                        o += off;
                    }
                    co[g] = o;
                    cl[g] = l;
                }
            }
            continue;
        }
        // coalesced result rows: element j of the batch's [32][G] tables is produced by lane j % 32 straight from
        // the owning line's register file (one 32-bit LDS = begin | end << 16); the line's (off, len) travel
        // through the info slots
        sts_u64(info_abs + lane * 8, off, st == 0 ? len : 0xFFFFFFFFu);
        __syncwarp();
        const uint64_t left = n - batch;
        const uint32_t total = (uint32_t)(left < 32 ? left : 32) * G;
        uint32_t* go = cap_off + batch * G + lane;
        uint32_t* gl = cap_len + batch * G + lane;
        const uint32_t wbase = regs_m2 + 2 - lane * reg_pitch * 2; // register file of the warp's line 0
        for (uint32_t j = lane; j < total; j += 32, go += 32, gl += 32) {
            const uint32_t line = G == 1 ? j : __umulhi(j, invG), g = j - line * G; // (2^32 / 1 does not fit invG)
            const uint2 inf = lds_u64_v(info_abs + line * 8);
            uint32_t o = 0, l = 0;
            if (inf.y != 0xFFFFFFFFu) {
                const uint32_t be = lds_u32_v(wbase + line * reg_pitch * 2 + g * 4);
                const uint32_t b = be & 0xFFFFu, en = be >> 16;
                if (b == LC_SLOT16_UNSET || en == LC_SLOT16_UNSET || en < b) {
                    o = inf.x + inf.y;
                } else {
                    o = inf.x + b;
                    l = en - b;
                }
            }
            *go = o;
            *gl = l;
        }
        __syncwarp();
    }
}

int launch_regex_tdfa_staged(const void* d_blob, uint32_t blob_bytes, bool slow, uint32_t nregs, const uint8_t* d_base,
                             const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint32_t ev_stride, uint64_t n,
                             uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                             uint32_t threads, uint32_t grid, unsigned long long* d_next_batch, uint32_t* d_overflow,
                             const uint32_t* d_order, const uint32_t* d_order_flag, cudaStream_t st) {
    if (!n)
        return 0;
    const uint32_t reg_pitch = tdfa_reg_pitch(nregs);
    size_t smem = tdfa_staged_smem_bytes(blob_bytes, nregs, threads);
    auto k = slow ? regex_tdfa_staged_kernel<true> : regex_tdfa_staged_kernel<false>;
    cudaError_t er = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er != cudaSuccess)
        return (int)er;
    k<<<grid, threads, smem, st>>>((const uint4*)d_blob, blob_bytes, d_base, d_ev_off, d_ev_len, ev_stride, n, nkeys,
                                   d_status, d_cap_off, d_cap_len, reg_pitch, d_next_batch, d_overflow, d_order,
                                   d_order_flag);
    return (int)cudaGetLastError();
}

// ---- several patterns in one grid (BASELINE config C5 "multi-pattern") ---------------------------------------
// All automata are co-resident in shared memory (each with its own 256-byte aligned class table; every pair table
// must end below shared address 64 Ki, which the host checks).  Per 32-line batch the patterns are tried in array
// order: lanes whose line has not matched yet (and whose selector, if any, names this pattern) walk it, the others
// only help fetching the tiles.  First match wins == what `(?:p0)|(?:p1)|...` would return under regex_match, with
// the capture groups numbered per pattern.  which[i] = index of the matching pattern or 0xFF.
// RESUME (patterns that do not fit together are spread over several launches): which[] holds the result of the
// earlier launches; lines matched there are left alone, p_base = index of this launch's first pattern.
struct TdfaPatS {
    uint32_t cls, t2, ncls, row_bytes, inv_row, start_row, sink, G, nkeys, blob_off, skip;
};

template <bool SLOW, bool RESUME>
__global__ void __launch_bounds__(1024, 1)
    regex_tdfa_multi_kernel(TdfaMultiArgs a, uint32_t p_base, const uint8_t* __restrict__ base,
                            const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len, uint64_t n,
                            const uint8_t* __restrict__ sel, uint8_t* __restrict__ which, uint8_t* __restrict__ status,
                            uint32_t* __restrict__ cap_off, uint32_t* __restrict__ cap_len, uint32_t gpitch,
                            uint32_t reg_pitch /* halfwords */, unsigned long long* next_batch, uint32_t* overflow,
                            const uint32_t* __restrict__ order, const uint32_t* __restrict__ order_flag) {
    extern __shared__ uint4 smem[];
    __shared__ TdfaPatS pats[LC_MULTI_MAX];
    const uint32_t s0abs = (uint32_t)__cvta_generic_to_shared(smem);
    uint32_t cursor = (s0abs + 255u) & ~255u;
    uint8_t* const smem_b = reinterpret_cast<uint8_t*>(smem);
    const uint32_t P = a.npat;
    for (uint32_t p = 0; p < P; ++p) {
        uint8_t* g_cls = smem_b + (cursor - s0abs);
        tdfa_stage_blob(g_cls, cursor, reinterpret_cast<const uint4*>(a.blob[p]), a.blob_bytes[p]);
        if (threadIdx.x == 0) {
            const LcTdfaView v = lc_tdfa_view(g_cls + 256);
            TdfaPatS ps;
            ps.cls = cursor;
            ps.t2 = cursor + 256 + v.h->off_t2;
            ps.ncls = v.h->ncls;
            ps.row_bytes = v.h->row_bytes;
            ps.inv_row = (uint32_t)((0x100000000ull + ps.row_bytes - 1) / ps.row_bytes);
            ps.start_row = ps.t2 + v.h->start * ps.row_bytes;
            ps.sink = ps.t2 + v.h->sink * ps.row_bytes;
            ps.G = v.h->ngroups;
            ps.nkeys = a.nkeys[p];
            ps.blob_off = cursor + 256 - s0abs;
            ps.skip = cursor + 256 + v.h->off_skip;
            pats[p] = ps;
        }
        cursor += 256 + ((a.blob_bytes[p] + 255u) & ~255u);
    }
    __syncthreads();
    const uint32_t invG = gpitch ? 0xFFFFFFFFu / gpitch + 1 : 0;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    uint8_t* g_regs0 = smem_b + (cursor - s0abs) + 16;
    uint16_t* wregs = reinterpret_cast<uint16_t*>(g_regs0) + (size_t)wid * 32 * reg_pitch;
    uint16_t* regs = wregs + (size_t)lane * reg_pitch;
    const uint32_t regs_abs = (uint32_t)__cvta_generic_to_shared(regs);
    const uint32_t regs_m2 = regs_abs - 2;
    // line info and tiles behind the register files, 128-byte aligned (tile_slot)
    const uint32_t aux_abs = ((uint32_t)__cvta_generic_to_shared(g_regs0 + (size_t)blockDim.x * reg_pitch * 2) + 127u) &
                             ~127u;
    const uint32_t info_abs = aux_abs + wid * 256;
    const uint32_t tile_abs = aux_abs + nwarps * 256 + wid * (LCT_STAGE_CHUNKS * 512);
    const uint32_t pats_abs = (uint32_t)__cvta_generic_to_shared(pats);
    const uint32_t base_mis = (uint32_t)((uintptr_t)base & 15);
    if (order && order_flag && *order_flag == 0)
        order = nullptr;
    TdfaLoader L;
    L.init(base, info_abs, tile_abs, lane);
    for (;;) {
        unsigned long long batch = 0;
        if (lane == 0)
            batch = atomicAdd(next_batch, 32ull);
        batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
        if (batch >= n)
            break;
        const bool valid = batch + lane < n;
        const uint64_t i = (order && valid) ? order[batch + lane] : batch + lane;
        uint32_t off = 0, len = 0, mis = 0, nch = 0, g0 = 0, selp = 0xFFu;
        bool open = valid; // still looking for a matching pattern
        bool skip_out = false;
        if (valid) {
            off = ev_off[i];
            len = ev_len[i];
            if (len >= 65535u) { // regex_tdfa_long_kernel handles this event (all patterns) afterwards
                atomicExch(overflow, 1u);
                len = 0;
                open = false;
            }
            if (sel)
                selp = sel[i];
            if (RESUME && which[i] != 0xFFu) {
                open = false;
                skip_out = true;
            }
            const uint64_t ab = (uint64_t)base_mis + off;
            mis = (uint32_t)(ab & 15);
            g0 = (uint32_t)(ab >> 4);
            nch = len ? (mis + len + 15) >> 4 : 0;
        }
        uint32_t st = 1, wh = 0xFFu, Gw = 0;
        for (uint32_t p = 0; p < P; ++p) {
            const bool act = open && (selp == 0xFFu || selp == p_base + p);
            if (!__any_sync(0xFFFFFFFFu, act))
                continue;
            // this pattern's parameters, through volatile loads so that they live in per-thread registers (PRMT with
            // an immediate selector needs a non-uniform operand, see regex_tdfa_staged_kernel)
            TdfaAbs t;
            uint32_t start_row, sink, Gp, nkp, blob_off;
            {
                const uint32_t pa = pats_abs + p * (uint32_t)sizeof(TdfaPatS);
                asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(t.cls) : "r"(pa) : "memory");
                t.t2 = lds_u32_v(pa + 4);
                t.ncls = lds_u32_v(pa + 8);
                t.row_bytes = lds_u32_v(pa + 12);
                t.inv_row = lds_u32_v(pa + 16);
                start_row = lds_u32_v(pa + 20);
                sink = lds_u32_v(pa + 24);
                Gp = lds_u32_v(pa + 28);
                nkp = lds_u32_v(pa + 32);
                blob_off = lds_u32_v(pa + 36);
                t.skip = lds_u32_v(pa + 40);
            }
            const LcTdfaView v = lc_tdfa_view(smem_b + blob_off);
            const uint32_t dead = t.t2;
            if (act)
                for (uint32_t k = 0; k < Gp; ++k)
                    reinterpret_cast<uint32_t*>(regs)[k] = 0xFFFFFFFFu;
            const uint32_t nch_p = act ? nch : 0;
            sts_u64(info_abs + lane * 8, g0, nch_p);
            const uint32_t max_nch = __reduce_max_sync(0xFFFFFFFFu, nch_p);
            uint32_t row = act ? start_row : dead;
            __syncwarp();
            row = tdfa_walk_lines<SLOW>(v, t, L, dead, sink, row, len, mis, max_nch, regs_m2, regs);
            if (act) {
                const uint32_t fin = v.eof[__umulhi(row - t.t2, t.inv_row)];
                if (fin != LC_NONE_ENTRY) {
                    lc_tdfa_run_ops(v, fin, len, regs);
                    open = false;
                    wh = p_base + p;
                    Gw = Gp;
                    st = Gp + 1 <= nkp ? 2 : 0;
                }
            }
            __syncwarp();
        }
        if (valid && !skip_out) {
            status[i] = (uint8_t)st;
            which[i] = (uint8_t)wh;
        }
        if (gpitch == 0)
            continue;
        if (order) {
            if (valid && !skip_out) {
                uint32_t* co = cap_off + i * gpitch;
                uint32_t* cl = cap_len + i * gpitch;
                for (uint32_t g = 0; g < gpitch; ++g) {
                    uint32_t o = 0, l = 0;
                    if (st == 0 && g < Gw) {
                        lc_slots16_to_cap(regs, g, len, &o, &l);
                        o += off;
                    }
                    co[g] = o;
                    cl[g] = l;
                }
            }
            continue;
        }
        // coalesced rows of gpitch entries; info = {off, len | G << 16} of a matched line, 0xFFFFFFFF = zero row,
        // 0xFFFFFFFE = row owned by an earlier launch (left alone)
        sts_u64(info_abs + lane * 8, off, skip_out ? 0xFFFFFFFEu : (st == 0 ? (len | (Gw << 16)) : 0xFFFFFFFFu));
        __syncwarp();
        const uint64_t left = n - batch;
        const uint32_t total = (uint32_t)(left < 32 ? left : 32) * gpitch;
        uint32_t* go = cap_off + batch * gpitch + lane;
        uint32_t* gl = cap_len + batch * gpitch + lane;
        const uint32_t wbase = regs_m2 + 2 - lane * reg_pitch * 2;
        for (uint32_t j = lane; j < total; j += 32, go += 32, gl += 32) {
            const uint32_t line = gpitch == 1 ? j : __umulhi(j, invG), g = j - line * gpitch;
            const uint2 inf = lds_u64_v(info_abs + line * 8);
            if (inf.y == 0xFFFFFFFEu)
                continue;
            uint32_t o = 0, l = 0;
            if (inf.y != 0xFFFFFFFFu && g < (inf.y >> 16)) {
                const uint32_t ln = inf.y & 0xFFFFu;
                const uint32_t be = lds_u32_v(wbase + line * reg_pitch * 2 + g * 4);
                const uint32_t b = be & 0xFFFFu, en = be >> 16;
                if (b == LC_SLOT16_UNSET || en == LC_SLOT16_UNSET || en < b) {
                    o = inf.x + ln;
                } else {
                    o = inf.x + b;
                    l = en - b;
                }
            }
            *go = o;
            *gl = l;
        }
        __syncwarp();
    }
}

int launch_regex_tdfa_multi(const TdfaMultiArgs& a, uint32_t p_base, bool resume, bool slow, uint32_t max_nregs,
                            const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                            const uint8_t* d_sel, uint8_t* d_which, uint8_t* d_status, uint32_t* d_cap_off,
                            uint32_t* d_cap_len, uint32_t gpitch, uint32_t threads, uint32_t grid,
                            unsigned long long* d_next_batch, uint32_t* d_overflow, const uint32_t* d_order,
                            const uint32_t* d_order_flag, cudaStream_t st) {
    if (!n)
        return 0;
    const uint32_t reg_pitch = tdfa_reg_pitch(max_nregs);
    size_t smem = tdfa_multi_smem_bytes(a, max_nregs, threads);
    auto k = resume ? (slow ? regex_tdfa_multi_kernel<true, true> : regex_tdfa_multi_kernel<false, true>)
                    : (slow ? regex_tdfa_multi_kernel<true, false> : regex_tdfa_multi_kernel<false, false>);
    cudaError_t er = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er != cudaSuccess)
        return (int)er;
    k<<<grid, threads, smem, st>>>(a, p_base, d_base, d_ev_off, d_ev_len, n, d_sel, d_which, d_status, d_cap_off,
                                   d_cap_len, gpitch, reg_pitch, d_next_batch, d_overflow, d_order, d_order_flag);
    return (int)cudaGetLastError();
}

// ---- events of 65535 bytes or more: 32-bit capture registers, tables read from global memory ------------------
// Launched unconditionally behind the staged kernels (which skip such events and raise *overflow); returns at once
// when no event was that long, so the common case costs one empty launch and NO host round trip.  One thread per
// long event, bytes fetched directly; patterns tried in order as in regex_tdfa_multi_kernel (npat = 1, which ==
// nullptr: the single-pattern entry points).
__global__ void __launch_bounds__(128)
    regex_tdfa_long_kernel(TdfaMultiArgs a, const uint8_t* __restrict__ base, const uint32_t* __restrict__ ev_off,
                           const uint32_t* __restrict__ ev_len, uint32_t ev_stride, uint64_t n,
                           const uint8_t* __restrict__ sel, uint8_t* __restrict__ which, uint8_t* __restrict__ status,
                           uint32_t* __restrict__ cap_off, uint32_t* __restrict__ cap_len, uint32_t gpitch,
                           const uint32_t* __restrict__ overflow, int bool_only) {
    if (*overflow == 0)
        return;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t len = ev_len[i * ev_stride];
        if (len < 65535u)
            continue;
        const uint32_t off = ev_off[i * ev_stride];
        const uint8_t* s = base + off;
        uint32_t regs[LC_TDFA_MAX_REGS + 2];
        uint32_t st = 1, wh = 0xFFu, Gw = 0;
        const uint32_t selp = sel ? sel[i] : 0xFFu;
        for (uint32_t p = 0; p < a.npat && wh == 0xFFu; ++p) {
            if (selp != 0xFFu && selp != p)
                continue;
            const LcTdfaView v = lc_tdfa_view(a.blob[p]);
            for (uint32_t k = 0; k < 2 * v.h->ngroups; ++k)
                regs[k] = 0xFFFFFFFFu;
            if (lc_tdfa_event<uint32_t>(v, s, 0, len, regs)) {
                wh = p;
                Gw = v.h->ngroups;
                st = Gw + 1 <= a.nkeys[p] ? 2 : 0;
            }
        }
        if (bool_only) {
            status[i] = wh != 0xFFu ? 1 : 0;
            continue;
        }
        status[i] = (uint8_t)st;
        if (which)
            which[i] = (uint8_t)wh;
        for (uint32_t g = 0; g < gpitch; ++g) {
            uint32_t o = 0, l = 0;
            if (st == 0 && g < Gw) {
                lc_slots_to_cap(regs, g, len, &o, &l);
                o += off;
            }
            cap_off[i * gpitch + g] = o;
            cap_len[i * gpitch + g] = l;
        }
    }
}

void launch_regex_tdfa_long(const TdfaMultiArgs& a, const uint8_t* d_base, const uint32_t* d_ev_off,
                            const uint32_t* d_ev_len, uint32_t ev_stride, uint64_t n, const uint8_t* d_sel,
                            uint8_t* d_which, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                            uint32_t gpitch, const uint32_t* d_overflow, bool bool_only, cudaStream_t st) {
    if (!n)
        return;
    unsigned grid = (unsigned)std::min<uint64_t>((n + 127) / 128, 1184);
    regex_tdfa_long_kernel<<<grid, 128, 0, st>>>(a, d_base, d_ev_off, d_ev_len, ev_stride, n, d_sel, d_which, d_status,
                                                 d_cap_off, d_cap_len, gpitch, d_overflow, bool_only ? 1 : 0);
}

template <class LabT>
__global__ void __launch_bounds__(1024, 1)
    regex_parse_smem_kernel(const uint4* __restrict__ blob, uint32_t blob_bytes, uint32_t G,
                            const uint8_t* __restrict__ base, const uint32_t* __restrict__ ev_off,
                            const uint32_t* __restrict__ ev_len, uint64_t n, uint32_t nkeys,
                            uint8_t* __restrict__ status, uint32_t* __restrict__ cap_off,
                            uint32_t* __restrict__ cap_len, uint32_t lab_words /* per thread, in smem */,
                            uint32_t* __restrict__ scratch, unsigned long long scratch_words,
                            unsigned long long* bump, uint32_t* overflow, unsigned long long* next_batch, const uint32_t* __restrict__ order) {
    extern __shared__ uint4 smem[];
    // stage the automaton
    for (uint32_t k = threadIdx.x; k < blob_bytes / 16; k += blockDim.x)
        smem[k] = __ldg(blob + k);
    __syncthreads();
    const LcProgView v = lc_view(smem);
    uint32_t* lab_base = reinterpret_cast<uint32_t*>(smem) + blob_bytes / 4;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // persistent warps: each warp claims batches of 32 consecutive events from a global counter
    for (;;) {
    unsigned long long batch = 0;
    if (lane == 0)
        batch = atomicAdd(next_batch, 32ull);
    batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
    if (batch >= n)
        break;
    if (batch + lane >= n)
        continue;
    const uint64_t i = order ? order[batch + lane] : batch + lane;
    const uint32_t off = ev_off[i], len = ev_len[i];
    // aligned view of the arena: byte loads go through 32-bit words of the 4-byte aligned base
    const uint32_t mis = (uint32_t)((uintptr_t)base & 3u);
    const uint8_t* abase = base - mis;
    const uint64_t a0 = (uint64_t)off + mis;
    uint32_t slots[2 * LC_MAX_GROUPS];
    for (uint32_t k = 0; k < 2 * G; ++k)
        slots[k] = LC_SLOT_UNSET;
    bool ok;
    if (v.h->mode == LC_MODE_FWD1 && v.h->off_fwd_byte) {
        ok = fwd1_event(v, reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(smem) +
                                                             v.h->off_fwd_byte),
                        abase, a0, len, slots);
    } else if (v.h->mode == LC_MODE_FWD1) {
        ok = lc_full_match_fwd1(v, base + off, len, slots);
    } else {
        const LabT* rev_byte =
            reinterpret_cast<const LabT*>(reinterpret_cast<const uint8_t*>(smem) + v.h->off_rev_byte);
        constexpr uint32_t PER = 4 / sizeof(LabT);
        const uint32_t need = len / PER + 1; // words for labels 0..len
        if (need <= lab_words) {
            LabSmem lab{lab_base + (size_t)wid * lab_words * 32 + lane};
            ok = twopass_event<LabT>(v, rev_byte, abase, a0, len, lab, slots);
        } else {
            unsigned long long at = atomicAdd(bump, (unsigned long long)need);
            if (at + need > scratch_words) {
                atomicExch(overflow, 1u);
                ok = false;
            } else {
                LabGlobal lab{scratch + at};
                ok = twopass_event<LabT>(v, rev_byte, abase, a0, len, lab, slots);
            }
        }
    }
    uint8_t st = ok ? (G + 1 <= nkeys ? 2 : 0) : 1;
    status[i] = st;
    uint32_t* co = cap_off + i * G;
    uint32_t* cl = cap_len + i * G;
    for (uint32_t g = 0; g < G; ++g) {
        uint32_t o = 0, l = 0;
        if (st == 0) {
            lc_slots_to_cap(slots, g, len, &o, &l);
            o += off;
        }
        co[g] = o;
        cl[g] = l;
    }
    } // persistent loop
}

int launch_regex_parse_fast(const void* d_blob, uint32_t blob_bytes, uint32_t rev_label_bytes, uint32_t ngroups,
                            const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                            uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                            uint32_t lab_words, uint32_t threads, uint32_t grid, uint32_t* d_scratch,
                            uint64_t scratch_words, unsigned long long* d_bump, uint32_t* d_overflow,
                            unsigned long long* d_next_batch, const uint32_t* d_order, cudaStream_t st) {
    if (!n)
        return 0;
    size_t smem = blob_bytes + (size_t)(threads / 32) * lab_words * 32 * 4;
    auto k8 = regex_parse_smem_kernel<uint8_t>;
    auto k16 = regex_parse_smem_kernel<uint16_t>;
    cudaError_t er = cudaFuncSetAttribute(rev_label_bytes == 2 ? k16 : k8,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (er != cudaSuccess)
        return (int)er;
    if (rev_label_bytes == 2)
        k16<<<grid, threads, smem, st>>>((const uint4*)d_blob, blob_bytes, ngroups, d_base, d_ev_off, d_ev_len, n, nkeys,
                                         d_status, d_cap_off, d_cap_len, lab_words, d_scratch, scratch_words, d_bump,
                                         d_overflow, d_next_batch, d_order);
    else
        k8<<<grid, threads, smem, st>>>((const uint4*)d_blob, blob_bytes, ngroups, d_base, d_ev_off, d_ev_len, n, nkeys,
                                        d_status, d_cap_off, d_cap_len, lab_words, d_scratch, scratch_words, d_bump,
                                        d_overflow, d_next_batch, d_order);
    return (int)cudaGetLastError();
}

__global__ void __launch_bounds__(128)
    prefix_match_kernel(const void* __restrict__ blob, const uint8_t* __restrict__ base,
                        const uint32_t* __restrict__ ev_off, const uint32_t* __restrict__ ev_len, uint64_t n,
                        uint8_t* __restrict__ out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    LcProgView v = lc_view(blob);
    out[i] = lc_prefix_match(v, base + ev_off[i], ev_len[i]) ? 1 : 0;
}

void launch_prefix_match(const void* d_blob, const uint8_t* d_base, const uint32_t* d_ev_off,
                         const uint32_t* d_ev_len, uint64_t n, uint8_t* d_out, cudaStream_t st) {
    if (!n)
        return;
    prefix_match_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_blob, d_base, d_ev_off, d_ev_len, n, d_out);
}

// ================================================================================================ multiline
struct MlMode {
    bool S, C, E, discard;
};

// Transition of line `fl` from state s_in (0 not partial / 1 partial):
// s_out and which line (0 none, 1 this line, 2 the next line) becomes multiStartIndex.
// Restates ProcessorSplitMultilineLogStringNative.cpp:175-283 without the emission side effects.
__host__ __device__ __forceinline__ void ml_trans(const MlMode& m, uint32_t fl, uint32_t s_in, uint32_t& s_out,
                                         uint32_t& begin) {
    const bool mS = fl & 1, mC = fl & 2, mE = fl & 4;
    begin = 0;
    if (!s_in) {
        bool probe = m.S ? mS : (m.C ? mC : false);
        if (probe) {
            s_out = 1;
            begin = 1;
        } else {
            s_out = 0;
        }
        return;
    }
    if (m.C && mC) {
        s_out = 1;
        return;
    }
    if (m.E) {
        if (m.C) {
            s_out = 0;
        } else if (mE) {
            if (m.S) {
                s_out = 0;
            } else {
                s_out = 1;
                begin = 2;
            }
        } else {
            s_out = 1;
        }
        return;
    }
    if (!m.C) {
        s_out = 1;
        if (mS)
            begin = 1;
    } else {
        if (mS) {
            s_out = 1;
            begin = 1;
        } else {
            s_out = 0;
        }
    }
}

// Events produced by line j (or by the virtual end-of-buffer element j == n).  Sink methods:
//   single(j, matched)          the line itself                       (CreateNewEvent / HandleUnmatchLogs on one line)
//   to_end(lb, j)               [start of line lb, end of line j]     matched record
//   to_prev(lb, j)              [start of line lb, start of line j - 1) matched record
//   span(lb, j_last, flag_line) unmatched lines lb..j_last, each carrying flag_line's isLast flag
//   to_eof(lb)                  [start of line lb, end of buffer)     matched record, isLast = true
template <class Sink>
__host__ __device__ __forceinline__ void ml_actions(const MlMode& m, uint32_t fl, uint32_t s_in, uint32_t lb, uint32_t j,
                                           uint32_t n, Sink& sink) {
    if (j == n) { // :289-308
        if (s_in && lb < n) {
            if (!m.E)
                sink.to_eof(lb);
            else
                sink.span(lb, n - 1, n);
        }
        return;
    }
    const bool mS = fl & 1, mC = fl & 2, mE = fl & 4;
    if (!s_in) {
        bool probe = m.S ? mS : (m.C ? mC : false);
        if (probe)
            return;
        if (m.E && !m.S && m.C && mE)
            sink.single(j, true);
        else
            sink.single(j, false);
        return;
    }
    if (m.C && mC)
        return;
    if (m.E) {
        if (m.C) {
            if (mE)
                sink.to_end(lb, j);
            else
                sink.span(lb, j, j);
        } else if (mE) {
            sink.to_end(lb, j);
        }
        return;
    }
    if (!m.C) {
        if (mS)
            sink.to_prev(lb, j);
    } else {
        sink.to_prev(lb, j);
        if (!mS)
            sink.single(j, false);
    }
}

// HandleUnmatchLogs re-splits its span with `while (begin < size)` (:342-380): an EMPTY unmatched line yields
// nothing (not even unmatch_lines++), and a span that ends with an empty line loses that last line; only the
// end-of-buffer span (which includes the trailing '\n') keeps it.
__device__ __forceinline__ uint32_t ml_span_last(const uint32_t* len, uint32_t lb, uint32_t jl, bool tail,
                                                 bool& none) {
    none = false;
    if (!tail && len[jl] == 0) {
        if (jl == lb) {
            none = true;
            return jl;
        }
        return jl - 1;
    }
    return jl;
}

struct MlCountSink {
    bool discard;
    const uint32_t* len;
    uint32_t n;
    uint32_t cnt = 0;
    __device__ void single(uint32_t j, bool matched) {
        if (matched)
            cnt += 1;
        else if (!discard && len[j] != 0)
            cnt += 1;
    }
    __device__ void to_end(uint32_t, uint32_t) { cnt += 1; }
    __device__ void to_prev(uint32_t, uint32_t) { cnt += 1; }
    __device__ void to_eof(uint32_t) { cnt += 1; }
    __device__ void span(uint32_t lb, uint32_t jl, uint32_t flag_line) {
        bool none;
        uint32_t last = ml_span_last(len, lb, jl, flag_line == n, none);
        if (!none && !discard)
            cnt += last - lb + 1;
    }
};

struct MlEmitSink {
    bool discard;
    const uint32_t* off;
    const uint32_t* len;
    uint32_t total_len;
    uint32_t* out_off;
    uint32_t* out_len;
    uint8_t* out_flags;
    uint64_t cap;
    uint64_t pos;
    uint32_t is_last; // isLastLog of the line being processed
    uint32_t n;       // number of lines
    uint32_t matched_events = 0, unmatch_lines = 0;
    __device__ void put(uint32_t o, uint32_t l, uint32_t fl) {
        if (pos < cap) {
            out_off[pos] = o;
            out_len[pos] = l;
            out_flags[pos] = (uint8_t)fl;
        }
        ++pos;
    }
    __device__ void single(uint32_t j, bool matched) {
        if (matched) {
            put(off[j], len[j], is_last | 2u);
            ++matched_events;
        } else if (len[j] != 0) {
            ++unmatch_lines;
            if (!discard)
                put(off[j], len[j], is_last);
        }
    }
    __device__ void to_end(uint32_t lb, uint32_t j) {
        uint32_t o = off[lb];
        put(o, off[j] + len[j] - o, is_last | 2u);
        ++matched_events;
    }
    __device__ void to_prev(uint32_t lb, uint32_t j) {
        uint32_t o = off[lb];
        put(o, off[j] - 1 - o, is_last | 2u);
        ++matched_events;
    }
    __device__ void to_eof(uint32_t lb) {
        uint32_t o = off[lb];
        put(o, total_len - o, 1u | 2u);
        ++matched_events;
    }
    __device__ void span(uint32_t lb, uint32_t jl, uint32_t flag_line) {
        bool none;
        uint32_t last = ml_span_last(len, lb, jl, flag_line == n, none);
        if (none)
            return;
        unmatch_lines += last - lb + 1;
        if (!discard)
            for (uint32_t k = lb; k <= last; ++k)
                put(off[k], len[k], is_last);
    }
};

// ---- back half of the multiline split, without look-backs: state pass -> scan -> count pass -> scan -> emission ------
// A single kernel would chain two decoupled look-backs per tile, and a look-back waits for the slowest of the resident
// tiles (see the split above: same effect; measured 12 % slower on an H100).  The arithmetic, however,
// only needs the FLAGS (one byte per line) until the very last step, so the passes are cheap to repeat:
//   pass 1  per tile of 16384 lines: the composed 2-state transition function           -> agg1[tile]
//   scan    one block, OpMlState (ordered)                                              -> pre1[tile]
//   pass 2  per tile: incoming state of every line (from pre1) -> number of events      -> agg2[tile]
//   scan    one block, OpSum                                                            -> pre2[tile]
//   pass 3  per tile: states again, exclusive event slots (from pre2), emission (reads off/len of the emitted lines)
// Tiles never wait for each other.  Lines whose transition is the identity (in start-only mode: every line that does
// not match) skip the composition.
constexpr int kMlPassThreads = 256;
constexpr int kMlPassItems = 64; // lines per thread: the two block scans of a pass are paid once per 16 K lines
constexpr uint32_t kMlPassTile = kMlPassThreads * kMlPassItems;

uint32_t ml_pass_tiles(uint64_t line_cap) { return (uint32_t)((line_cap + 1 + kMlPassTile - 1) / kMlPassTile); }
// scratch of launch_ml_passes: four u64 per tile + {u64 incoming state, u32 event count} per thread of a tile
uint64_t ml_pass_scratch_bytes(uint64_t line_cap) {
    return (uint64_t)ml_pass_tiles(line_cap) * (32 + (uint64_t)kMlPassThreads * 12) + 64;
}

template <class Op>
__global__ void __launch_bounds__(1024)
    ml_tile_scan_kernel(const uint64_t* __restrict__ agg, const uint32_t* __restrict__ n_lines, uint32_t line_cap,
                        uint64_t* __restrict__ pre) {
    __shared__ uint64_t s_scan[33];
    const uint64_t n = min(*n_lines, line_cap);
    const uint32_t ntiles = (uint32_t)((n + 1 + kMlPassTile - 1) / kMlPassTile); // (element n = end of buffer)
    const uint32_t per = (ntiles + 1023) / 1024;
    const uint32_t t0 = min((uint32_t)threadIdx.x * per, ntiles), t1 = min(t0 + per, ntiles);
    uint64_t a = Op::identity();
    for (uint32_t t = t0; t < t1; ++t)
        a = Op::combine(a, __ldg(agg + t));
    uint64_t tot;
    uint64_t run = block_exclusive_scan<Op, 1024>(a, tot, s_scan);
    for (uint32_t t = t0; t < t1; ++t) {
        pre[t] = run;
        run = Op::combine(run, __ldg(agg + t));
    }
}

// The state machine as tables over (flags, state), built on the host from ml_trans / ml_actions themselves: stepping a
// line is then three shifts instead of the branch cascade (the generic code stays the single statement of the rules).
//   act codes: 0 nothing, 1 single(unmatched), 2 single(matched), 3 to_end, 4 span(lb, j, j), 5 to_prev,
//              6 to_prev + single(unmatched)
struct MlTab {
    uint32_t next;    // bit fl*2+s: state after the line
    uint32_t begin;   // 2 bits at (fl*2+s)*2: 0 none / 1 this line / 2 the next line becomes multiStartIndex
    uint64_t act;     // 3 bits at (fl*2+s)*3
    uint32_t ident;   // bit fl: the line changes neither state (and opens nothing)
    uint32_t skip[2]; // bit fl: in state s the line does nothing at all (no event, no change)
};

struct MlRecSink { // records which sink calls ml_actions makes for one (flags, state) pair
    uint32_t code = 0;
    bool bad = false;
    __host__ __device__ void single(uint32_t, bool matched) { code = code == 5 ? (matched ? (bad = true, 0u) : 6u) : (code ? (bad = true, 0u) : (matched ? 2u : 1u)); }
    __host__ __device__ void to_end(uint32_t, uint32_t) { code = code ? (bad = true, 0u) : 3u; }
    __host__ __device__ void to_prev(uint32_t, uint32_t) { code = code ? (bad = true, 0u) : 5u; }
    __host__ __device__ void to_eof(uint32_t) { bad = true; }
    __host__ __device__ void span(uint32_t, uint32_t jl, uint32_t fl) { code = (code || jl != 7 || fl != 7) ? (bad = true, 0u) : 4u; }
};

static bool ml_build_tab(const MlMode& m, MlTab& t) {
    memset(&t, 0, sizeof t);
    for (uint32_t fl = 0; fl < 8; ++fl) {
        bool id = true;
        for (uint32_t st = 0; st < 2; ++st) {
            uint32_t o, b;
            ml_trans(m, fl, st, o, b);
            MlRecSink rec;
            ml_actions(m, fl, st, 3u, 7u, 100u, rec); // (line 7 of 100, multiStartIndex 3)
            if (rec.bad)
                return false;
            const uint32_t idx = fl * 2 + st;
            t.next |= (o & 1u) << idx;
            t.begin |= (b & 3u) << (2 * idx);
            t.act |= (uint64_t)rec.code << (3 * idx);
            if (o != st || b)
                id = false;
            if (o == st && !b && !rec.code)
                t.skip[st] |= 1u << fl;
        }
        if (id)
            t.ident |= 1u << fl;
    }
    return true;
}

template <class Sink>
__device__ __forceinline__ void ml_apply(uint32_t code, uint32_t lb, uint32_t j, Sink& sink) {
    switch (code) {
    case 1: sink.single(j, false); break;
    case 2: sink.single(j, true); break;
    case 3: sink.to_end(lb, j); break;
    case 4: sink.span(lb, j, j); break;
    case 5: sink.to_prev(lb, j); break;
    case 6:
        sink.to_prev(lb, j);
        sink.single(j, false);
        break;
    default: break;
    }
}

template <int PASS>
__global__ void __launch_bounds__(kMlPassThreads)
    ml_pass_kernel(MlMode m, MlTab tb, const uint8_t* __restrict__ flags, const uint32_t* __restrict__ off,
                   const uint32_t* __restrict__ len, const uint32_t* __restrict__ n_lines, uint32_t line_cap,
                   uint32_t total_len, uint64_t* __restrict__ agg1, const uint64_t* __restrict__ pre1,
                   uint64_t* __restrict__ agg2, const uint64_t* __restrict__ pre2, uint32_t* __restrict__ out_off,
                   uint32_t* __restrict__ out_len, uint8_t* __restrict__ out_flags, uint64_t cap,
                   unsigned long long* counters, uint64_t* total_out,
                   uint64_t* __restrict__ t_run0 /* [tile][thread]: pass 2 -> pass 3 */,
                   uint32_t* __restrict__ t_cnt /* [tile][thread]: pass 2 -> pass 3 */) {
    constexpr int THREADS = kMlPassThreads, ITEMS = kMlPassItems;
    static_assert(ITEMS % 16 == 0, "16-byte loads of flags");
    constexpr int NWORDS = ITEMS / 4;
    __shared__ uint64_t s_scan[THREADS / 32 + 1];
    const int tid = threadIdx.x;
    const uint32_t tile = blockIdx.x;
    const uint64_t n = min(*n_lines, line_cap); // (more lines than the table holds: the host repeats the call)
    if ((uint64_t)tile * kMlPassTile > n)
        return;
    const uint64_t base = (uint64_t)tile * kMlPassTile + (uint64_t)tid * ITEMS;
    uint32_t fw[NWORDS];
    if (base + ITEMS <= n) {
#pragma unroll
        for (int q = 0; q < ITEMS / 16; ++q) {
            const uint4 f4 = __ldg(reinterpret_cast<const uint4*>(flags + base) + q);
            fw[4 * q + 0] = f4.x & 0x07070707u, fw[4 * q + 1] = f4.y & 0x07070707u;
            fw[4 * q + 2] = f4.z & 0x07070707u, fw[4 * q + 3] = f4.w & 0x07070707u;
        }
    } else {
#pragma unroll
        for (int w = 0; w < NWORDS; ++w) {
            fw[w] = 0;
            for (int b = 0; b < 4; ++b)
                if (base + 4 * w + b < n)
                    fw[w] |= (uint32_t)(flags[base + 4 * w + b] & 7u) << (8 * b);
        }
    }
    const uint32_t nvalid = base >= n ? 0u : (uint32_t)min((uint64_t)ITEMS, n - base); // lines (not the eof element)
    // ---- the thread's lines composed: both incoming states stepped side by side (passes 1 and 2; pass 3 takes the
    // thread's incoming state and its event count from pass 2)
    const uint64_t slot = (uint64_t)tile * THREADS + tid;
    uint32_t sA = 0, sB = 1, lbA = 0, lbB = 0; // lbX: (index + 1) of the last line opened inside the run, 0 = none
#pragma unroll
    for (int w = 0; w < NWORDS && PASS != 3; ++w) {
        if (fw[w] == 0 && (tb.ident & 1u))
            continue; // four lines that change nothing
#pragma unroll 1
        for (int b = 0; b < 4; ++b) {
            const int k = w * 4 + b;
            const uint32_t fl = (fw[w] >> (8 * b)) & 0xFFu;
            if ((uint32_t)k < nvalid && !((tb.ident >> fl) & 1u)) {
                const uint32_t j1 = (uint32_t)(base + k) + 1;
                const uint32_t ia = fl * 2 + sA, ib = fl * 2 + sB;
                const uint32_t ba = (tb.begin >> (2 * ia)) & 3u, bb = (tb.begin >> (2 * ib)) & 3u;
                if (ba)
                    lbA = j1 + ba - 1;
                if (bb)
                    lbB = j1 + bb - 1;
                sA = (tb.next >> ia) & 1u;
                sB = (tb.next >> ib) & 1u;
            }
        }
    }
    uint64_t run0;
    if (PASS != 3) {
        const uint64_t agg = OpMlState::make(sA, sB, lbA, lbB);
        uint64_t tot;
        const uint64_t ex = block_exclusive_scan<OpMlState, THREADS>(agg, tot, s_scan);
        if (PASS == 1) {
            if (tid == 0)
                agg1[tile] = tot;
            return;
        }
        run0 = OpMlState::combine(__ldg(pre1 + tile), ex);
        t_run0[slot] = run0;
    } else {
        run0 = __ldg(t_run0 + slot);
    }
    // initial condition (:165-169): End-only mode starts partial with multiStartIndex = line 0
    const uint32_t s0 = (!m.S && !m.C && m.E) ? 1u : 0u;
    const uint32_t st0 = OpMlState::f(run0, s0);
    uint32_t lb0 = OpMlState::lb(run0, s0);
    if (!lb0)
        lb0 = s0 ? 1u : 0u;
    lb0 = lb0 ? lb0 - 1 : 0u; // line index of multiStartIndex (valid only in the partial state)
    // one sweep over the thread's lines with a concrete state; `Sink` counts (pass 2) or writes (pass 3)
    auto sweep = [&](auto& sink) {
        uint32_t st = st0, lb = lb0;
#pragma unroll
        for (int w = 0; w < NWORDS; ++w) {
            if (fw[w] == 0 && (tb.skip[st] & 1u) && (uint32_t)(w * 4 + 4) <= nvalid)
                continue; // four lines without any effect in this state
#pragma unroll 1
            for (int b = 0; b < 4; ++b) {
                const int k = w * 4 + b;
                if ((uint32_t)k >= nvalid)
                    break;
                const uint32_t fl = (fw[w] >> (8 * b)) & 0xFFu;
                if ((tb.skip[st] >> fl) & 1u)
                    continue;
                const uint32_t j = (uint32_t)(base + k);
                const uint32_t idx = fl * 2 + st;
                const uint32_t code = (uint32_t)(tb.act >> (3 * idx)) & 7u;
                if (code) {
                    sink.prepare(j);
                    ml_apply(code, lb, j, sink);
                }
                const uint32_t bg = (tb.begin >> (2 * idx)) & 3u;
                if (bg)
                    lb = j + bg - 1;
                st = (tb.next >> idx) & 1u;
            }
        }
        if (base <= n && n < base + ITEMS) { // the virtual end-of-buffer element lives in this thread
            sink.prepare((uint32_t)n);
            ml_actions(m, 0u, st, lb, (uint32_t)n, (uint32_t)n, sink);
        }
    };
    struct CountSink : MlCountSink {
        __device__ void prepare(uint32_t) {}
    } cs;
    if (PASS == 2) {
        cs.discard = m.discard;
        cs.len = len;
        cs.n = (uint32_t)n;
        sweep(cs);
        t_cnt[slot] = cs.cnt;
    } else {
        cs.cnt = __ldg(t_cnt + slot);
    }
    uint64_t tot2;
    const uint64_t ex2 = block_exclusive_scan<OpSum, THREADS>((uint64_t)cs.cnt, tot2, s_scan);
    if (PASS == 2) {
        if (tid == 0)
            agg2[tile] = tot2;
        return;
    }
    // ---- emission at the exclusive prefix of the counts.  The sweep only RECORDS what each event is made of; the records
    // are then turned into output rows one per thread (independent gathers of off / len, coalesced stores) -- a thread
    // that emitted its three or four events one after the other paid a DRAM round trip for each of them.
    constexpr uint32_t LIST = 3072; // events of a tile that fit the list (more: the threads write their events directly)
    __shared__ uint32_t s_rec[LIST][2];
    const uint64_t pos0 = __ldg(pre2 + tile);
    struct EmitSink : MlEmitSink {
        uint32_t total_len_;
        // begin + content.size() == sourceVal.size() (:174): only the last line can end where the buffer ends (every
        // other line is followed by a '\n'); the end-of-buffer element always passes true
        __device__ void prepare(uint32_t j) {
            is_last = (j == n) ? 1u : ((j + 1 == n && off[j] + len[j] == total_len_) ? 1u : 0u);
        }
    };
    // kind: 0 one line (a) | 1 lines a..j up to the end of j | 2 lines a..j-1 (without the line feed) | 3 a..end of buffer
    struct RecSink {
        uint32_t (*rec)[2];
        const uint32_t* off;
        const uint32_t* len;
        uint64_t pos0, pos;
        uint32_t total_len, n, is_last, matched_events, unmatch_lines;
        bool discard;
        __device__ void prepare(uint32_t j) {
            is_last = (j == n) ? 1u : ((j + 1 == n && off[j] + len[j] == total_len) ? 1u : 0u);
        }
        __device__ void put(uint32_t kind, uint32_t a, uint32_t j, uint32_t matched) {
            const uint32_t idx = (uint32_t)(pos - pos0);
            rec[idx][0] = a | (kind << 30);
            rec[idx][1] = j | (matched << 30) | (is_last << 31);
            ++pos;
        }
        __device__ void single(uint32_t j, bool matched) {
            if (matched) {
                put(0, j, j, 1);
                ++matched_events;
            } else if (len[j] != 0) {
                ++unmatch_lines;
                if (!discard)
                    put(0, j, j, 0);
            }
        }
        __device__ void to_end(uint32_t lb, uint32_t j) {
            put(1, lb, j, 1);
            ++matched_events;
        }
        __device__ void to_prev(uint32_t lb, uint32_t j) {
            put(2, lb, j, 1);
            ++matched_events;
        }
        __device__ void to_eof(uint32_t lb) {
            is_last = 1;
            put(3, lb, 0, 1);
            ++matched_events;
        }
        __device__ void span(uint32_t lb, uint32_t jl, uint32_t flag_line) {
            bool none;
            const uint32_t last = ml_span_last(len, lb, jl, flag_line == n, none);
            if (none)
                return;
            unmatch_lines += last - lb + 1;
            if (!discard)
                for (uint32_t k = lb; k <= last; ++k)
                    put(0, k, k, 0);
        }
    };
    uint32_t me, ul;
    if (tot2 <= LIST) { // (block-uniform)
        RecSink rs;
        rs.rec = s_rec;
        rs.off = off;
        rs.len = len;
        rs.pos0 = pos0;
        rs.pos = pos0 + ex2;
        rs.total_len = total_len;
        rs.n = (uint32_t)n;
        rs.is_last = 0;
        rs.matched_events = rs.unmatch_lines = 0;
        rs.discard = m.discard;
        sweep(rs);
        if (base <= n && n < base + ITEMS)
            *total_out = rs.pos;
        me = rs.matched_events, ul = rs.unmatch_lines;
        __syncthreads();
        for (uint32_t e = tid; e < (uint32_t)tot2; e += THREADS) {
            const uint64_t at = pos0 + e;
            if (at >= cap)
                break;
            const uint32_t w0 = s_rec[e][0], w1 = s_rec[e][1];
            const uint32_t kind = w0 >> 30, a = w0 & 0x3FFFFFFFu, j = w1 & 0x3FFFFFFFu;
            const uint32_t o = __ldg(off + a);
            uint32_t l;
            if (kind == 0)
                l = __ldg(len + a);
            else if (kind == 1)
                l = __ldg(off + j) + __ldg(len + j) - o;
            else if (kind == 2)
                l = __ldg(off + j) - 1 - o;
            else
                l = total_len - o;
            out_off[at] = o;
            out_len[at] = l;
            out_flags[at] = (uint8_t)((w1 >> 31) | (((w1 >> 30) & 1u) << 1));
        }
    } else {
        EmitSink es;
        es.discard = m.discard;
        es.off = off;
        es.len = len;
        es.total_len = total_len;
        es.total_len_ = total_len;
        es.out_off = out_off;
        es.out_len = out_len;
        es.out_flags = out_flags;
        es.cap = cap;
        es.pos = pos0 + ex2;
        es.n = (uint32_t)n;
        es.is_last = 0;
        sweep(es);
        if (base <= n && n < base + ITEMS)
            *total_out = es.pos;
        me = es.matched_events, ul = es.unmatch_lines;
    }
    for (int d = 16; d; d >>= 1) {
        me += __shfl_down_sync(0xFFFFFFFFu, me, d);
        ul += __shfl_down_sync(0xFFFFFFFFu, ul, d);
    }
    if ((threadIdx.x & 31) == 0) {
        if (me)
            atomicAdd(&counters[0], (unsigned long long)me);
        if (ul)
            atomicAdd(&counters[1], (unsigned long long)ul);
    }
}

int launch_ml_passes(const MlConfig& cfg, const uint8_t* d_flags, const uint32_t* d_off, const uint32_t* d_len,
                     const uint32_t* d_n_lines, uint32_t line_cap, uint32_t total_len, uint32_t* d_out_off,
                     uint32_t* d_out_len, uint8_t* d_out_flags, uint64_t cap, uint64_t* d_scratch /* ml_pass_scratch_bytes */,
                     unsigned long long* d_counters, uint64_t* d_total, cudaStream_t st) {
    MlMode m{cfg.blob_start != nullptr, cfg.blob_cont != nullptr, cfg.blob_end != nullptr, cfg.discard != 0};
    const uint32_t nt = ml_pass_tiles(line_cap);
    uint64_t *agg1 = d_scratch, *pre1 = d_scratch + nt, *agg2 = d_scratch + 2 * (uint64_t)nt,
             *pre2 = d_scratch + 3 * (uint64_t)nt, *t_run0 = d_scratch + 4 * (uint64_t)nt;
    uint32_t* t_cnt = reinterpret_cast<uint32_t*>(t_run0 + (uint64_t)nt * kMlPassThreads);
    MlTab tb;
    if (!ml_build_tab(m, tb))
        return -1; // (cannot happen: every (flags, state) pair makes at most to_prev + single)
#define LC_ML_PASS(P)                                                                                                  \
    ml_pass_kernel<P><<<nt, kMlPassThreads, 0, st>>>(m, tb, d_flags, d_off, d_len, d_n_lines, line_cap, total_len,      \
                                                     agg1, pre1, agg2, pre2, d_out_off, d_out_len, d_out_flags, cap,   \
                                                     d_counters, d_total, t_run0, t_cnt)
    LC_ML_PASS(1);
    ml_tile_scan_kernel<OpMlState><<<1, 1024, 0, st>>>(agg1, d_n_lines, line_cap, pre1);
    LC_ML_PASS(2);
    ml_tile_scan_kernel<OpSum><<<1, 1024, 0, st>>>(agg2, d_n_lines, line_cap, pre2);
    LC_ML_PASS(3);
#undef LC_ML_PASS
    return 5;
}

// ---- f3 (next row): LogFileReader::RemoveLastIncompleteLog over the line table + probe flags of the split pass --------
// core/file_server/reader/LogFileReader.cpp:1997-2064 walks the chunk backwards line by line (RawTextParser::GetLastLine,
// :2186-2204) until a line matches the end pattern (and is newline-terminated) or, without an end pattern, the start
// pattern.  With flags[line] at hand that walk is "the last line whose flag is set": one block searches the table from
// the back, 1024 lines per step.  out[0] = bytes to keep, out[1] = rollbackLineFeedCount.
__global__ void __launch_bounds__(1024)
    last_record_kernel(const uint8_t* __restrict__ flags, const uint32_t* __restrict__ off,
                       const uint32_t* __restrict__ len, const uint32_t* __restrict__ n_lines, uint32_t line_cap,
                       uint32_t size, int has_start, int has_end, unsigned long long* __restrict__ out) {
    __shared__ long long s_best;
    __shared__ int s_any_end;
    const uint32_t n = min(*n_lines, line_cap);
    if (threadIdx.x == 0) {
        s_best = -1;
        s_any_end = 0;
    }
    __syncthreads();
    long long hit = -1;
    if (has_start || has_end) {
        const uint32_t want = has_end ? 4u : 1u;
        for (long long hi = (long long)n - 1; hi >= 0; hi -= 1024) {
            const long long j = hi - threadIdx.x;
            if (j >= 0 && (flags[j] & want)) {
                // an end line only counts when its newline is inside the chunk ("ensure the end line is complete")
                if (!has_end || off[j] + len[j] < size)
                    atomicMax(&s_best, j);
                else
                    s_any_end = 1; // foundEnd on the unterminated last line
            }
            __syncthreads();
            hit = s_best;
            __syncthreads(); // everyone has read s_best before the next step may raise it
            if (hit >= 0)
                break;
        }
    }
    if (threadIdx.x != 0)
        return;
    // rollback contribution of lines [a, n): one each, except a line that ends at offset 0 (GetLastLine(end == 0))
    auto rb_from = [&](long long a) -> unsigned long long {
        if (a >= (long long)n)
            return 0;
        unsigned long long c = (unsigned long long)(n - a);
        if (a == 0 && n > 0 && off[0] + len[0] == 0)
            --c;
        return c;
    };
    unsigned long long keep, rb;
    if (hit >= 0 && has_end) {
        keep = (unsigned long long)off[hit] + len[hit] + 1;
        rb = rb_from(hit + 1);
    } else if (hit >= 0) {
        keep = off[hit];
        rb = rb_from(hit);
    } else if (has_end && s_any_end) {
        keep = 0;
        rb = rb_from(0);
    } else if (n == 0) {
        keep = size;
        rb = 0;
    } else {
        // single-line rollback (or nothing matched): keep everything when the last line is complete
        const uint32_t L = n - 1, end = off[L] + len[L];
        if (end != 0 && end < size) {
            keep = (unsigned long long)end + 1;
            rb = 0;
        } else {
            keep = off[L];
            rb = end != 0 ? 1 : 0;
        }
    }
    out[0] = keep;
    out[1] = rb;
}

void launch_last_record(const uint8_t* d_flags, const uint32_t* d_off, const uint32_t* d_len, const uint32_t* d_n_lines,
                        uint32_t line_cap, uint32_t size, bool has_start, bool has_end, unsigned long long* d_out,
                        cudaStream_t st) {
    last_record_kernel<<<1, 1024, 0, st>>>(d_flags, d_off, d_len, d_n_lines, line_cap, size, has_start ? 1 : 0,
                                           has_end ? 1 : 0, d_out);
}

// ================================================================================================ delimiter
// STAGED (max_fields <= kDelimStagedMaxFields): the [32 lines][max_fields] blocks of f_off / f_len / f_dq that a warp
// produces are contiguous in the output tables, so they are assembled in shared memory (row pitch max_fields | 1:
// conflict-free for the per-line pushes) and leave as fully coalesced 128-byte stores, zero padding included; the
// direct variant writes every record with a 4-byte store into its line's row (32 different rows per warp
// instruction).
constexpr uint32_t kDelimStagedMaxFields = 32;
template <bool STAGED>
__global__ void __launch_bounds__(128)
    delim_kernel(DelimConfig cfg, const uint8_t* __restrict__ base, const uint32_t* __restrict__ ev_off,
                 const uint32_t* __restrict__ ev_len, uint64_t n, uint8_t* __restrict__ status,
                 uint32_t* __restrict__ nfields, uint32_t* __restrict__ f_off, uint32_t* __restrict__ f_len,
                 uint32_t* __restrict__ f_dq) {
    extern __shared__ uint32_t s_rows[]; // STAGED: [warp][3][32][pitch]
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t MF = cfg.max_fields;
    const uint32_t lane = threadIdx.x & 31, pitch = MF | 1u;
    uint32_t* fo;
    uint32_t* fl;
    uint32_t* fd;
    uint32_t* wrows = nullptr;
    if (STAGED) {
        wrows = s_rows + (size_t)(threadIdx.x >> 5) * 3 * 32 * pitch;
        fo = wrows + lane * pitch;
        fl = fo + 32 * pitch;
        fd = fl + 32 * pitch;
        for (uint32_t k = 0; k < MF; ++k) {
            fo[k] = 0;
            fl[k] = 0;
            fd[k] = 0;
        }
    } else {
        if (i >= n)
            return;
        fo = f_off + i * MF;
        fl = f_len + i * MF;
        fd = f_dq + i * MF;
    }
    if (i < n) {
    const uint32_t eo = ev_off[i];
    const uint8_t* v = base + eo;
    uint32_t nf = 0; // columns counted
    uint8_t st;
    // trim (:226-238)
    int32_t endIdx = (int32_t)ev_len[i];
    int32_t begIdx = 0;
    bool blank = endIdx == 0;
    if (!blank) {
        while (endIdx > 0 && (v[endIdx - 1] == ' ' || v[endIdx - 1] == '\r'))
            --endIdx;
        while (begIdx < endIdx && v[begIdx] == ' ')
            ++begIdx;
        blank = begIdx >= endIdx;
    }
    auto push = [&](uint32_t o, uint32_t l, uint32_t dq) {
        if (nf < MF) {
            fo[nf] = eo + o;
            fl[nf] = l;
            fd[nf] = dq;
        }
        ++nf;
    };
    bool ok = true;
    if (blank) {
        st = 2;
    } else if (cfg.nkeys == 0) {
        st = 1;
        ok = false;
    } else {
        const bool use_quote = cfg.sep_len == 1 && cfg.quote != cfg.sep[0];
        if (use_quote) {
            // DelimiterModeFsmParser::ParseDelimiterLine (zero-copy variant, :260-294), run-skipping formulation:
            // only separators and quotes step the state machine, runs of ordinary bytes are one step (lc_exec.cuh)
            ok = lc_delim_fsm(v, begIdx, endIdx, cfg.sep[0], cfg.quote, push);
        } else {
            // ProcessorParseDelimiterNative::SplitString (:366-409)
            const uint32_t d = cfg.sep_len;
            const uint32_t size = endIdx - begIdx;
            if (d > size) {
                push(begIdx, size, 0);
            } else {
                uint32_t pos = begIdx, top = endIdx - d;
                bool done = false;
                while (pos <= top && !done) {
                    uint32_t pos2 = endIdx;
                    for (uint32_t q = pos; q + d <= (uint32_t)endIdx; ++q) {
                        bool eq = true;
                        for (uint32_t t = 0; t < d; ++t)
                            eq = eq && v[q + t] == cfg.sep[t];
                        if (eq) {
                            pos2 = q;
                            break;
                        }
                    }
                    push(pos, pos2 - pos, 0);
                    if (pos2 == (uint32_t)endIdx) {
                        done = true;
                        break;
                    }
                    pos = pos2 + d;
                    if (nf >= cfg.nkeys && !cfg.extend) {
                        push(pos2, endIdx - pos2, 0);
                        done = true;
                    }
                }
                if (!done && pos <= (uint32_t)endIdx)
                    push(pos, endIdx - pos, 0);
            }
            if (nf == 0)
                ok = false;
        }
        if (!ok) {
            st = 1;
            nf = 0;
        } else {
            uint32_t cols = nf;
            if (use_quote && !cfg.extend && cols > cfg.nkeys)
                cols = cfg.nkeys + 1; // overflow columns are joined into one (:258-275)
            st = (cols == 0 || (!cfg.allow_short && cols < cfg.nkeys)) ? 3 : 0;
        }
    }
    status[i] = st;
    nfields[i] = nf;
    // rows of failed / blank lines are zero; so are the unused columns (STAGED rows start out zeroed)
    for (uint32_t k = (st == 1 || st == 2) ? 0 : (nf < MF ? nf : MF); k < MF && (!STAGED || st == 1 || st == 2); ++k) {
        fo[k] = 0;
        fl[k] = 0;
        fd[k] = 0;
    }
    if (cfg.tap_off && cfg.tap_col < MF) {
        cfg.tap_off[i] = fo[cfg.tap_col];
        cfg.tap_len[i] = fl[cfg.tap_col];
    }
    }
    if (STAGED) {
        __syncwarp();
        const uint64_t i0 = i - lane; // first line of this warp
        if (i0 < n) {
            const uint64_t left = n - i0;
            const uint32_t total = (uint32_t)(left < 32 ? left : 32) * MF;
            const uint32_t invMF = MF > 1 ? 0xFFFFFFFFu / MF + 1 : 0;
            uint32_t* go = f_off + i0 * MF;
            uint32_t* gl = f_len + i0 * MF;
            uint32_t* gd = f_dq + i0 * MF;
            for (uint32_t j = lane; j < total; j += 32) {
                const uint32_t line = MF > 1 ? __umulhi(j, invMF) : j, k = j - line * MF;
                const uint32_t at = line * pitch + k;
                go[j] = wrows[at];
                gl[j] = wrows[32 * pitch + at];
                gd[j] = wrows[64 * pitch + at];
            }
        }
    }
}

// ---- tiled variant for the quote FSM (the common configuration) -----------------------------------------------------
// Same structure as the staged regex kernel: persistent warps claim 32-line batches, fetch the lines COOPERATIVELY
// (TdfaLoader: cp.async, 4 full 128-byte segments per instruction, tile_slot layout) instead of every lane pulling its
// own line with LDG.128 (32 different 128-byte lines per instruction), and each lane then streams its line out of the
// tile through the resumable run-skipping FSM (lc_delim_chunk).  Only the trimmed range is fetched: the lane first looks
// at the last 16 bytes of its line for trailing blanks / CRs (:226-238); leading blanks are skipped in the stream.
// Field records are assembled in the per-warp row block in shared memory and leave as coalesced 128-byte stores, as
// in delim_kernel<true>.  Shared memory per warp: 256 B line info + 4 KB tile + 3 x 32 x (max_fields | 1) words, plus
// 128 B per block to align the tiles.
__global__ void __launch_bounds__(1024, 1)
    delim_tiled_kernel(DelimConfig cfg, const uint8_t* __restrict__ base, const uint32_t* __restrict__ ev_off,
                       const uint32_t* __restrict__ ev_len, uint64_t n, uint8_t* __restrict__ status,
                       uint32_t* __restrict__ nfields, uint32_t* __restrict__ f_off, uint32_t* __restrict__ f_len,
                       uint32_t* __restrict__ f_dq, unsigned long long* next_batch) {
    extern __shared__ uint4 smem[];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    // the warp's [32][MF] blocks of f_off / f_len / f_dq are built in shared memory in exactly the global layout (row
    // pitch MF), so that they leave -- zero padding included -- as plain 16-byte vector copies
    const uint32_t MF = cfg.max_fields;
    const uint32_t blk_words = 32 * MF, blk_pad = (blk_words + 3u) & ~3u; // words per table block (16-byte multiple)
    // line info and tiles from the first 128-byte boundary of the window (tile_slot), the row blocks behind them
    const uint32_t raw_abs = (uint32_t)__cvta_generic_to_shared(smem), s0abs = (raw_abs + 127u) & ~127u;
    const uint32_t info_abs = s0abs + wid * 256;
    const uint32_t tile_abs = s0abs + nwarps * 256 + wid * (LCT_STAGE_CHUNKS * 512);
    uint32_t* wrows = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(smem) + (s0abs - raw_abs) +
                                                  (size_t)nwarps * (256 + 4096)) +
                      (size_t)wid * 3 * blk_pad;
    uint32_t* fo = wrows + lane * MF;
    uint32_t* fl = fo + blk_pad;
    uint32_t* fd = fl + blk_pad;
    const uint32_t base_mis = (uint32_t)((uintptr_t)base & 15);
    TdfaLoader L;
    L.init(base, info_abs, tile_abs, lane);
    const uint32_t sep_splat = cfg.sep[0] * 0x01010101u, quote_splat = cfg.quote * 0x01010101u;
    for (;;) {
        unsigned long long batch = 0;
        if (lane == 0)
            batch = atomicAdd(next_batch, 32ull);
        batch = __shfl_sync(0xFFFFFFFFu, batch, 0);
        if (batch >= n)
            break;
        const bool valid = batch + lane < n;
        const uint64_t i = batch + lane;
        // zero the three row blocks (rows of failed / blank lines and unused columns are zero)
        for (uint32_t k = lane; k < 3 * blk_pad / 4; k += 32)
            reinterpret_cast<uint4*>(wrows)[k] = make_uint4(0, 0, 0, 0);
        uint32_t eo = 0, mis = 0, g0 = 0, nch = 0;
        int32_t endIdx = 0;
        if (valid) {
            eo = ev_off[i];
            endIdx = (int32_t)ev_len[i];
            const uint64_t a = (uint64_t)base_mis + eo;
            mis = (uint32_t)(a & 15);
            g0 = (uint32_t)(a >> 4);
            // trailing ' ' / '\r' (:226-232): look at the chunks of the tail, last one first
            while (endIdx > 0) {
                const uint32_t qlast = mis + (uint32_t)endIdx - 1; // frame position of the last byte
                const uint4 vv = __ldg(L.gbase16 + g0 + (qlast >> 4));
                const uint32_t blank = match16b(vv, 0x20202020u) | match16b(vv, 0x0D0D0D0Du);
                const uint32_t hi = qlast & 15u;                      // last byte's slot in this chunk
                const uint32_t lo = (qlast & ~15u) >= mis ? 0u : mis; // first slot of the chunk that belongs to the line
                const uint32_t inside = ((hi == 15u) ? 0xFFFFu : ((1u << (hi + 1)) - 1u)) & ~((1u << lo) - 1u);
                const uint32_t keep = ~blank & inside;                // non-blank bytes of the line in this chunk
                if (keep) {
                    endIdx = (int32_t)((qlast & ~15u) + (31 - __clz(keep)) + 1 - mis);
                    break;
                }
                endIdx = (int32_t)((qlast & ~15u) + lo) - (int32_t)mis; // all blank: go on with the chunk before
            }
            nch = endIdx > 0 ? (mis + (uint32_t)endIdx + 15) >> 4 : 0;
        }
        sts_u64(info_abs + lane * 8, g0, nch);
        const uint32_t max_nch = __reduce_max_sync(0xFFFFFFFFu, nch);
        uint32_t nf = 0;
        auto push = [&](uint32_t o, uint32_t l, uint32_t dq) { // (the state machine's columns: fallback only)
            if (nf < MF) {
                fo[nf] = eo + o;
                fl[nf] = l;
                fd[nf] = dq;
            }
            ++nf;
        };
        // bit-parallel path: a real separator (or the record's end) at offset p closes column nf, which holds `quotes`
        // quotes; offset and quote count are parked in the row and turned into the column record after the last byte
        auto mark = [&](uint32_t p, uint32_t quotes) {
            if (nf < MF) {
                fo[nf] = p;
                fd[nf] = quotes;
            }
            ++nf;
        };
        bool ok = true, started = false, slow = false; // slow: not well-formed for the bit-parallel path
        LcDelimFast run;
        lc_delim_fast_start(run);
        const uint32_t qe = mis + (uint32_t)endIdx;
        uint32_t qb = mis; // becomes the frame position of the first non-blank byte
        const bool parse = valid && endIdx > 0;
        __syncwarp();
        for (uint32_t s0 = 0; s0 < max_nch; s0 += LCT_STAGE_CHUNKS) {
            L.stage(s0);
            if (parse && ok && !slow) {
                const uint32_t kb = nch < s0 + LCT_STAGE_CHUNKS ? nch : s0 + LCT_STAGE_CHUNKS;
                for (uint32_t k = s0; k < kb; k += 2) { // 32 bytes per step (the second chunk may lie behind the record)
                    const uint4 v0 = lds_u128_v(L.own(k));
                    const uint4 v1 = lds_u128_v(L.own(k + 1));
                    const uint32_t q0 = k * 16;
                    if (!started) {
                        // leading ' ' (:233-238): the first byte that is not a blank starts the record
                        uint32_t nb = ~(match16c(v0, 0x20202020u) | (match16c(v1, 0x20202020u) << 16));
                        if (q0 < qb)
                            nb &= ~lc_low_bits(qb - q0);
                        nb &= lc_low_bits(qe - q0);
                        if (!nb)
                            continue;
                        qb = q0 + (uint32_t)(__ffs((int)nb) - 1);
                        started = true;
                        if (cfg.nkeys == 0) { // nothing to parse into: the line fails once it is known not to be blank
                            ok = false;
                            break;
                        }
                    }
                    // bit-parallel columns (lc_exec.cuh); a record with a quote the machine would not accept there is
                    // redone by the machine itself after the batch (rare, and it also decides about the error)
                    if (!lc_delim_fast_step<32>(run, match16c(v0, sep_splat) | (match16c(v1, sep_splat) << 16),
                                                match16c(v0, quote_splat) | (match16c(v1, quote_splat) << 16), q0, qb,
                                                qe, mis, mark)) {
                        slow = true;
                        break;
                    }
                }
            }
            __syncwarp();
        }
        if (valid) {
            uint8_t st;
            if (endIdx <= 0 || !started) {
                st = 2; // empty / all-blank value (:220-224,239-242)
            } else if (cfg.nkeys == 0) {
                st = 1;
                nf = 0;
            } else {
                if (!slow && !lc_delim_fast_finish(run, endIdx, mark))
                    slow = true;
                const uint32_t nf_fast = nf < MF ? nf : MF;
                if (!slow) {
                    // marks -> column records: a column starts behind the previous mark
                    uint32_t prev = qb - mis;
                    for (uint32_t k = 0; k < nf_fast; ++k) {
                        const uint32_t p = fo[k], c = fd[k];
                        fo[k] = eo + prev + (c ? 1u : 0u);
                        fl[k] = p - prev - (c ? 2u : 0u);
                        fd[k] = c ? (c - 2) >> 1 : 0u;
                        prev = p + 1;
                    }
                } else { // the state machine over the whole record, straight from global memory
                    nf = 0;
                    ok = lc_delim_fsm(base + eo, (int32_t)(qb - mis), endIdx, cfg.sep[0], cfg.quote, push);
                    for (uint32_t k = nf; ok && k < nf_fast; ++k) // marks only the first attempt left behind
                        fo[k] = fd[k] = 0;
                }
                if (!ok) {
                    st = 1;
                    nf = 0;
                } else {
                    uint32_t cols = nf;
                    if (!cfg.extend && cols > cfg.nkeys)
                        cols = cfg.nkeys + 1; // overflow columns are joined into one (:258-275)
                    st = (cols == 0 || (!cfg.allow_short && cols < cfg.nkeys)) ? 3 : 0;
                }
            }
            status[i] = st;
            nfields[i] = (st == 2) ? 0u : nf;
            if (st == 1 || st == 2) // rows of failed / blank lines are zero
                for (uint32_t k = 0; k < MF; ++k) {
                    fo[k] = 0;
                    fl[k] = 0;
                    fd[k] = 0;
                }
            if (cfg.tap_off && cfg.tap_col < MF) { // dense copy of one column: the chained processor's event table
                cfg.tap_off[i] = fo[cfg.tap_col];
                cfg.tap_len[i] = fl[cfg.tap_col];
            }
        }
        __syncwarp();
        // ---- the three [lines][MF] blocks leave as 16-byte vector copies (a batch starts at a multiple of 128 * MF
        // bytes; the table bases are 16-byte aligned allocations)
        const uint64_t left = n - batch;
        const uint32_t total = (uint32_t)(left < 32 ? left : 32) * MF; // words per table
        uint32_t* gt[3] = {f_off + batch * MF, f_len + batch * MF, f_dq + batch * MF};
#pragma unroll
        for (int tb = 0; tb < 3; ++tb) {
            const uint32_t* src = wrows + tb * blk_pad;
            uint32_t* dst = gt[tb];
            if ((((uintptr_t)dst) & 15u) == 0) {
                const uint32_t nv = total >> 2;
                for (uint32_t j = lane; j < nv; j += 32)
                    reinterpret_cast<uint4*>(dst)[j] = reinterpret_cast<const uint4*>(src)[j];
                for (uint32_t j = (nv << 2) + lane; j < total; j += 32)
                    dst[j] = src[j];
            } else {
                for (uint32_t j = lane; j < total; j += 32)
                    dst[j] = src[j];
            }
        }
        __syncwarp();
    }
}

void launch_delim(const DelimConfig& cfg, const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len,
                  uint64_t n, uint8_t* d_status, uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len,
                  uint32_t* d_f_dq, unsigned long long* d_next_batch /* zeroed, or nullptr */, cudaStream_t st) {
    if (!n)
        return;
    const unsigned grid = (unsigned)((n + 127) / 128);
    static const bool direct = getenv("LC_B200_DELIM_DIRECT") != nullptr; // A/B knob
    static const bool no_tiled = getenv("LC_B200_DELIM_NO_TILE") != nullptr; // A/B knob
    const bool use_quote = cfg.sep_len == 1 && cfg.quote != cfg.sep[0];
    if (!direct && !no_tiled && use_quote && d_next_batch && cfg.max_fields && cfg.max_fields <= kDelimStagedMaxFields) {
        // persistent tiled kernel: as many warps per block as the per-warp tile + row block allow
        int dev = 0, smem_max = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const size_t per_warp = 256 + 4096 + (size_t)3 * ((32 * cfg.max_fields + 3u) & ~3u) * 4;
        uint32_t warps = (uint32_t)std::min<size_t>(32, ((size_t)smem_max - 128) / per_warp);
        if (warps >= 8) {
            const size_t smem = per_warp * warps + 128;
            cudaFuncSetAttribute(delim_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            const uint64_t need = (n + warps * 32 - 1) / (warps * 32);
            const unsigned g = (unsigned)std::min<uint64_t>(need, (uint64_t)sms);
            delim_tiled_kernel<<<g, warps * 32, smem, st>>>(cfg, d_base, d_ev_off, d_ev_len, n, d_status, d_nfields,
                                                            d_f_off, d_f_len, d_f_dq, d_next_batch);
            return;
        }
    }
    if (!direct && cfg.max_fields && cfg.max_fields <= kDelimStagedMaxFields) {
        const size_t smem = (size_t)4 * 3 * 32 * (cfg.max_fields | 1u) * sizeof(uint32_t);
        if (smem > 48 * 1024)
            cudaFuncSetAttribute(delim_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        delim_kernel<true><<<grid, 128, smem, st>>>(cfg, d_base, d_ev_off, d_ev_len, n, d_status, d_nfields, d_f_off,
                                                    d_f_len, d_f_dq);
    } else {
        delim_kernel<false><<<grid, 128, 0, st>>>(cfg, d_base, d_ev_off, d_ev_len, n, d_status, d_nfields, d_f_off,
                                                  d_f_len, d_f_dq);
    }
}

// ================================================================================================ SLS serialise
// Next row (SURVEY.md 8f rank 4): the `Logs` fields of an sls_logs::LogGroup written straight from spans of the
// arena (lc_exec.cuh: lc_sls_log_size / lc_sls_emit_log).  sizes -> exclusive_sum_kernel -> emit.
__global__ void __launch_bounds__(256)
    sls_size_kernel(const uint64_t* __restrict__ ent_begin, const uint32_t* __restrict__ klen,
                    const uint32_t* __restrict__ vlen, const uint32_t* __restrict__ ev_ns, uint64_t n,
                    uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    uint32_t body;
    rec_size[i] = lc_sls_log_size(klen, vlen, ent_begin[i], ent_begin[i + 1], ev_ns && ev_ns[i] != 0xFFFFFFFFu, &body);
    body_size[i] = body;
}

// one warp per event: lane 0 writes tags and lengths, all lanes copy the key / value bytes
__global__ void __launch_bounds__(256)
    sls_emit_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ ev_time,
                    const uint32_t* __restrict__ ev_ns, const uint64_t* __restrict__ ent_begin,
                    const uint32_t* __restrict__ koff, const uint32_t* __restrict__ klen,
                    const uint32_t* __restrict__ voff, const uint32_t* __restrict__ vlen, uint64_t n,
                    const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ body_size,
                    uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint64_t e0 = ent_begin[i], e1 = ent_begin[i + 1];
    if (e0 == e1)
        return; // LogEvent::Empty: skipped (SLSSerializer.cpp:383-385)
    const bool has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
    lc_sls_emit_log(out + rec_off[i], base, ev_time[i], has_ns, has_ns ? ev_ns[i] : 0u, koff, klen, voff, vlen, e0, e1,
                    body_size[i], threadIdx.x & 31, 32);
}

void launch_sls_sizes(const uint64_t* d_ent_begin, const uint32_t* d_klen, const uint32_t* d_vlen,
                      const uint32_t* d_ev_ns, uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                      cudaStream_t st) {
    if (n)
        sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_ent_begin, d_klen, d_vlen, d_ev_ns, n,
                                                                     d_rec_size, d_body_size);
}

void launch_sls_emit(const uint8_t* d_base, const uint32_t* d_ev_time, const uint32_t* d_ev_ns,
                     const uint64_t* d_ent_begin, const uint32_t* d_koff, const uint32_t* d_klen,
                     const uint32_t* d_voff, const uint32_t* d_vlen, uint64_t n, const uint64_t* d_rec_off,
                     const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st) {
    if (n)
        sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(d_base, d_ev_time, d_ev_ns, d_ent_begin,
                                                                          d_koff, d_klen, d_voff, d_vlen, n, d_rec_off,
                                                                          d_body_size, d_out);
}

// ---- f4, regex-fed: Log records of the events a ProcessorParseRegexNative leaves behind, straight from the regex
// stage's tables.  Both passes run the same per-row function (lc_exec.cuh: lc_regex_sls_body) over the content plans
// of the configuration -- the size pass with a counting sink, one thread per event; the emit pass with a writing sink,
// one warp per event.
__device__ __forceinline__ LcRegexSlsRow regex_sls_row(const LcRegexSlsCfg& c, const RegexSlsTables& t,
                                                       const uint32_t* ev_time, const uint32_t* ev_ns, uint64_t i) {
    LcRegexSlsRow r;
    r.eo = t.ev_off[i];
    r.elen = t.ev_len[i];
    r.status = c.whole_line ? 0u : t.status[i];
    r.co = t.cap_off ? t.cap_off + i * c.pitch : nullptr;
    r.cl = t.cap_len ? t.cap_len + i * c.pitch : nullptr;
    r.time = ev_time ? ev_time[i] : 0u;
    r.has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
    r.ns = r.has_ns ? ev_ns[i] : 0u;
    return r;
}

__global__ void __launch_bounds__(256)
    regex_sls_size_kernel(LcRegexSlsCfg c, RegexSlsTables t, const uint32_t* __restrict__ ev_ns, uint64_t n,
                          uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                          unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t kept = 0, nomatch = 0, erased = 0;
    if (i < n) {
        const LcRegexSlsRow r = regex_sls_row(c, t, nullptr, ev_ns, i);
        LcSlsCount s{0};
        const uint32_t cnt = lc_regex_sls_body(c, t.base, r, s);
        const uint32_t body = cnt ? s.n : 0u;
        rec_size[i] = cnt ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        const uint32_t v = lc_regex_sls_verdict(c, r.status);
        kept = v == 0u || c.keep_fail;
        nomatch = v == 1u; // LC_REGEX_NOMATCH: out_failed (LC_REGEX_KEYS_MISMATCH does not count, :227-244)
        erased = !kept;
    }
    if (counters) { // successful, failed, discarded: one atomic per warp and counter
        kept = __reduce_add_sync(0xFFFFFFFFu, kept);
        nomatch = __reduce_add_sync(0xFFFFFFFFu, nomatch);
        erased = __reduce_add_sync(0xFFFFFFFFu, erased);
        if ((threadIdx.x & 31) == 0) {
            if (kept)
                atomicAdd(counters + 0, (unsigned long long)kept);
            if (nomatch)
                atomicAdd(counters + 1, (unsigned long long)nomatch);
            if (erased)
                atomicAdd(counters + 2, (unsigned long long)erased);
        }
    }
}

__global__ void __launch_bounds__(256)
    regex_sls_emit_kernel(LcRegexSlsCfg c, RegexSlsTables t, const uint32_t* __restrict__ ev_time,
                          const uint32_t* __restrict__ ev_ns, uint64_t n, const uint64_t* __restrict__ rec_off,
                          const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased or LogEvent::Empty: no record (SLSSerializer.cpp:383-385)
    const LcRegexSlsRow r = regex_sls_row(c, t, ev_time, ev_ns, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_regex_sls_body(c, t.base, r, s);
}

void launch_regex_sls_sizes(const LcRegexSlsCfg& c, const RegexSlsTables& t, const uint32_t* d_ev_ns, uint64_t n,
                            uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                            cudaStream_t st) {
    if (n)
        regex_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, d_ev_ns, n, d_rec_size, d_body_size,
                                                                            d_counters);
}

void launch_regex_sls_emit(const LcRegexSlsCfg& c, const RegexSlsTables& t, const uint32_t* d_ev_time,
                           const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off, const uint32_t* d_body_size,
                           uint8_t* d_out, cudaStream_t st) {
    if (n)
        regex_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, d_ev_time, d_ev_ns, n, d_rec_off,
                                                                                 d_body_size, d_out);
}

// ---- f4, split -> regex chain: Log records of the pieces a splitter cut and a ProcessorParseRegexNative parsed,
// straight from the piece tables and the regex tables over them (lc_exec.cuh: lc_split_regex_sls_body) -- the size
// pass one thread per piece, the emit pass one warp per piece.  counters: u64 [4] += successful, failed, discarded,
// pieces whose record would reach 4 GiB (their size is left 0 and the call is refused).
__device__ __forceinline__ LcSplitRegexSlsRow split_regex_sls_row(const LcSplitRegexSlsCfg& c, const RegexSlsTables& t,
                                                                  uint64_t i) {
    LcSplitRegexSlsRow r;
    r.po = t.ev_off[i];
    r.plen = t.ev_len[i];
    r.status = c.x.whole_line ? 0u : t.status[i];
    r.co = t.cap_off ? t.cap_off + i * c.x.pitch : nullptr;
    r.cl = t.cap_len ? t.cap_len + i * c.x.pitch : nullptr;
    return r;
}

// keep (or nullptr): a filter's verdict per piece; a removed piece gets size 0 and is never counted as too large
__global__ void __launch_bounds__(256)
    split_regex_sls_size_kernel(LcSplitRegexSlsCfg c, RegexSlsTables t, uint64_t n, const uint8_t* __restrict__ keep,
                                uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    LcSplitRegexVerdict v{0u, 0u, 0u};
    uint32_t big = 0;
    if (i < n) {
        const LcSplitRegexSlsRow r = split_regex_sls_row(c, t, i);
        LcSlsCount64 s{0};
        const uint32_t cnt = keep && !keep[i] ? 0u : lc_split_regex_sls_body(c, t.base, r, s);
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        v = lc_split_regex_verdict(c, r.status);
    }
    // one atomic per warp and counter
    const uint32_t ok = __reduce_add_sync(0xFFFFFFFFu, v.ok), failed = __reduce_add_sync(0xFFFFFFFFu, v.failed),
                   erased = __reduce_add_sync(0xFFFFFFFFu, v.erased);
    big = __reduce_add_sync(0xFFFFFFFFu, big);
    if ((threadIdx.x & 31) == 0) {
        if (ok)
            atomicAdd(counters + 0, (unsigned long long)ok);
        if (failed)
            atomicAdd(counters + 1, (unsigned long long)failed);
        if (erased)
            atomicAdd(counters + 2, (unsigned long long)erased);
        if (big)
            atomicAdd(counters + 3, (unsigned long long)big);
    }
}

__global__ void __launch_bounds__(256)
    split_regex_sls_emit_kernel(LcSplitRegexSlsCfg c, RegexSlsTables t, uint64_t n, const uint64_t* __restrict__ rec_off,
                                const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased or LogEvent::Empty: no record
    const LcSplitRegexSlsRow r = split_regex_sls_row(c, t, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_regex_sls_body(c, t.base, r, s);
}

void launch_split_regex_sls_sizes(const LcSplitRegexSlsCfg& c, const RegexSlsTables& t, uint64_t n,
                                  const uint8_t* d_keep, uint32_t* d_rec_size, uint32_t* d_body_size,
                                  unsigned long long* d_counters, cudaStream_t st) {
    if (n)
        split_regex_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_keep, d_rec_size,
                                                                                  d_body_size, d_counters);
}

// ---- f4, split -> regex -> filter chain (lc_exec.cuh: lc_filter_leaf, lc_filter_eval), one thread per piece.  The
// tap writes leaf l's values as a dense table over the source value (off / len; 0 / 0 where the value is absent or is
// the offset digits) and, with dig, a second table over the digit scratch (row i's digits at dig + 20 i; 0 / 0 where
// the value is not the digits), so that the boolean match runs over each base in turn.
__global__ void __launch_bounds__(256)
    filter_tap_kernel(LcSplitRegexSlsCfg c, LcFilterSlsCfg f, uint32_t leaf, RegexSlsTables t, uint64_t n,
                      uint32_t* __restrict__ off, uint32_t* __restrict__ len, uint32_t* __restrict__ doff,
                      uint32_t* __restrict__ dlen, uint8_t* __restrict__ dig) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const LcSplitRegexSlsRow r = split_regex_sls_row(c, t, i);
    uint32_t o, l;
    const uint32_t s = lc_filter_leaf(c, f, leaf, r, &o, &l);
    const bool digits = s == LC_REGEX_SLS_DIGITS;
    off[i] = digits ? 0u : o;
    len[i] = digits ? 0u : l;
    if (doff) {
        const uint32_t at = (uint32_t)i * LC_FILTER_SLS_DIGIT_PITCH;
        doff[i] = digits ? at : 0u;
        dlen[i] = digits ? l : 0u;
        const uint64_t pos = c.src_pos + r.po;
        for (uint32_t j = 0; digits && j < l; ++j)
            dig[at + j] = lc_dec_digit(pos, j, l);
    }
}

// keep[i] = the filter's verdict; counters[0] += pieces the filter removed (one atomic per warp).  m: the match bytes,
// [l * n + i] over the source value and, with f.any_digits, [(nleaves + l) * n + i] over the digit scratch.
__global__ void __launch_bounds__(256)
    filter_eval_kernel(LcSplitRegexSlsCfg c, LcFilterSlsCfg f, const uint8_t* __restrict__ status, uint64_t n,
                       const uint8_t* __restrict__ m, uint8_t* __restrict__ keep,
                       unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t removed = 0;
    if (i < n) {
        const uint32_t st = c.x.whole_line ? 0u : status[i];
        bool reached, empty;
        lc_filter_row_state(c, f, st, &reached, &empty);
        uint32_t bits = 0;
        for (uint32_t l = 0; l < f.nleaves; ++l) {
            const uint32_t s = lc_filter_leaf_src(c, f, l, st);
            if (s != LC_FILTER_SLS_ABSENT)
                bits |= (uint32_t)m[(uint64_t)(s == LC_REGEX_SLS_DIGITS ? f.nleaves + l : l) * n + i] << l;
        }
        const uint32_t k = reached ? lc_filter_eval(f, bits, empty) : 0u;
        keep[i] = (uint8_t)k;
        removed = reached && !k;
    }
    removed = __reduce_add_sync(0xFFFFFFFFu, removed);
    if ((threadIdx.x & 31) == 0 && removed)
        atomicAdd(counters, (unsigned long long)removed);
}

void launch_filter_tap(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, uint32_t leaf, const RegexSlsTables& t,
                       uint64_t n, uint32_t* d_off, uint32_t* d_len, uint32_t* d_doff, uint32_t* d_dlen,
                       uint8_t* d_dig, cudaStream_t st) {
    if (n)
        filter_tap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, f, leaf, t, n, d_off, d_len, d_doff, d_dlen,
                                                                        d_dig);
}

void launch_filter_eval(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, const uint8_t* d_status, uint64_t n,
                        const uint8_t* d_match, uint8_t* d_keep, unsigned long long* d_counters, cudaStream_t st) {
    if (n)
        filter_eval_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, f, d_status, n, d_match, d_keep,
                                                                         d_counters);
}

void launch_split_regex_sls_emit(const LcSplitRegexSlsCfg& c, const RegexSlsTables& t, uint64_t n,
                                 const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                 cudaStream_t st) {
    if (n)
        split_regex_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_off, d_body_size,
                                                                                       d_out);
}

// ---- f4, split -> regex -> timestamp chain (lc_exec.cuh: lc_split_regex_ts_value, _time, _verdict).  The tap, one
// thread per piece, writes the dense value table the timestamp passes take; the size pass (one thread per piece) and
// the emit pass (one warp per piece) run lc_split_regex_sls_body with each record's own time.
__global__ void __launch_bounds__(256)
    split_regex_ts_tap_kernel(LcSplitRegexSlsCfg c, LcSplitRegexTsCfg tc, RegexSlsTables t, uint64_t n,
                              uint32_t* __restrict__ off, uint32_t* __restrict__ len) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    uint32_t o, l;
    lc_split_regex_ts_value(c, tc, split_regex_sls_row(c, t, i), &o, &l);
    off[i] = o;
    len[i] = l;
}

// counters: u64 [9] += the LC_SRTS_COUNTERS verdicts (one atomic per warp and counter), then pieces whose record
// would reach 4 GiB
__global__ void __launch_bounds__(256)
    split_regex_ts_sls_size_kernel(LcSplitRegexSlsCfg c, LcSplitRegexTsCfg tc, RegexSlsTables t, TsRowTables ts,
                                   uint64_t n, uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                   unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bits = 0, big = 0;
    if (i < n) {
        const LcSplitRegexSlsRow r = split_regex_sls_row(c, t, i);
        const uint32_t st = ts.status[i];
        const LcSplitRegexTsTime tm = lc_split_regex_ts_time(c, tc, st, ts.sec[i], ts.nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_regex_sls_body(c, t.base, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        bits = lc_split_regex_ts_verdict(c, r.status, st);
    }
#pragma unroll
    for (uint32_t k = 0; k < LC_SRTS_COUNTERS; ++k) {
        const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, (bits >> k) & 1u);
        if ((threadIdx.x & 31) == 0 && v)
            atomicAdd(counters + k, (unsigned long long)v);
    }
    big = __reduce_add_sync(0xFFFFFFFFu, big);
    if ((threadIdx.x & 31) == 0 && big)
        atomicAdd(counters + LC_SRTS_COUNTERS, (unsigned long long)big);
}

__global__ void __launch_bounds__(256)
    split_regex_ts_sls_emit_kernel(LcSplitRegexSlsCfg c, LcSplitRegexTsCfg tc, RegexSlsTables t, TsRowTables ts,
                                   uint64_t n, const uint64_t* __restrict__ rec_off,
                                   const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased, discarded or LogEvent::Empty: no record
    const LcSplitRegexSlsRow r = split_regex_sls_row(c, t, i);
    const LcSplitRegexTsTime tm = lc_split_regex_ts_time(c, tc, ts.status[i], ts.sec[i], ts.nsec[i]);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_regex_sls_body(c, t.base, r, tm.time, tm.has_ns, tm.ns, s);
}

void launch_split_regex_ts_tap(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                               uint64_t n, uint32_t* d_off, uint32_t* d_len, cudaStream_t st) {
    if (n)
        split_regex_ts_tap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, tc, t, n, d_off, d_len);
}

void launch_split_regex_ts_sls_sizes(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                                     const TsRowTables& ts, uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                                     unsigned long long* d_counters, cudaStream_t st) {
    if (n)
        split_regex_ts_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_size,
                                                                                     d_body_size, d_counters);
}

void launch_split_regex_ts_sls_emit(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                                    const TsRowTables& ts, uint64_t n, const uint64_t* d_rec_off,
                                    const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st) {
    if (n)
        split_regex_ts_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_off,
                                                                                          d_body_size, d_out);
}

// ---- f4, delimiter-fed: Log records of the events a ProcessorParseDelimiterNative leaves behind, straight from the
// delimiter stage's tables.  Both passes run the same per-row function (lc_exec.cuh: lc_delim_sls_body) -- the size
// pass with a counting sink, one thread per event; the emit pass with a writing sink, one warp per event.
__device__ __forceinline__ LcDelimSlsRow delim_sls_row(const LcDelimSlsCfg& c, const DelimSlsTables& t,
                                                       const uint32_t* ev_time, const uint32_t* ev_ns, uint64_t i) {
    LcDelimSlsRow r;
    r.eo = t.ev_off[i];
    r.elen = t.ev_len[i];
    r.status = t.status[i];
    r.nf = t.nfields[i];
    r.fo = t.f_off + i * c.max_fields;
    r.fl = t.f_len + i * c.max_fields;
    r.fd = t.f_dq + i * c.max_fields;
    r.time = ev_time ? ev_time[i] : 0u;
    r.has_ns = ev_ns && ev_ns[i] != 0xFFFFFFFFu;
    r.ns = r.has_ns ? ev_ns[i] : 0u;
    return r;
}

__global__ void __launch_bounds__(256)
    delim_sls_size_kernel(LcDelimSlsCfg c, DelimSlsTables t, const uint32_t* __restrict__ ev_ns, uint64_t n,
                          uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                          unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t ok = 0, failed = 0, erased = 0, blank = 0;
    if (i < n) {
        const LcDelimSlsRow r = delim_sls_row(c, t, nullptr, ev_ns, i);
        LcSlsCount s{0};
        const uint32_t cnt = lc_delim_sls_body(c, t.base, r, s);
        const uint32_t body = cnt ? s.n : 0u;
        rec_size[i] = cnt ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        ok = r.status == 0;
        blank = r.status == 2;
        failed = !ok && !blank;
        erased = failed && !c.keep_fail;
    }
    if (counters) { // successful, failed, discarded, blank: one atomic per warp and counter
        ok = __reduce_add_sync(0xFFFFFFFFu, ok);
        failed = __reduce_add_sync(0xFFFFFFFFu, failed);
        erased = __reduce_add_sync(0xFFFFFFFFu, erased);
        blank = __reduce_add_sync(0xFFFFFFFFu, blank);
        if ((threadIdx.x & 31) == 0) {
            if (ok)
                atomicAdd(counters + 0, (unsigned long long)ok);
            if (failed)
                atomicAdd(counters + 1, (unsigned long long)failed);
            if (erased)
                atomicAdd(counters + 2, (unsigned long long)erased);
            if (blank)
                atomicAdd(counters + 3, (unsigned long long)blank);
        }
    }
}

__global__ void __launch_bounds__(256)
    delim_sls_emit_kernel(LcDelimSlsCfg c, DelimSlsTables t, const uint32_t* __restrict__ ev_time,
                          const uint32_t* __restrict__ ev_ns, uint64_t n, const uint64_t* __restrict__ rec_off,
                          const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased or LogEvent::Empty: no record (SLSSerializer.cpp:383-385)
    const LcDelimSlsRow r = delim_sls_row(c, t, ev_time, ev_ns, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_delim_sls_body(c, t.base, r, s);
}

void launch_delim_sls_sizes(const LcDelimSlsCfg& c, const DelimSlsTables& t, const uint32_t* d_ev_ns, uint64_t n,
                            uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                            cudaStream_t st) {
    if (n)
        delim_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, d_ev_ns, n, d_rec_size, d_body_size,
                                                                            d_counters);
}

void launch_delim_sls_emit(const LcDelimSlsCfg& c, const DelimSlsTables& t, const uint32_t* d_ev_time,
                           const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off, const uint32_t* d_body_size,
                           uint8_t* d_out, cudaStream_t st) {
    if (n)
        delim_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, d_ev_time, d_ev_ns, n, d_rec_off,
                                                                                 d_body_size, d_out);
}

// ---- f4, delimiter -> regex chain: the value tap (one thread per row; a row with doubled quotes in key k's column
// copies the collapsed value to its side slot, the common row only reads its table entries) and the Log records
// (lc_exec.cuh: lc_delim_regex_sls_body -- the size pass one thread per event, the emit pass one warp per event).
__global__ void __launch_bounds__(256)
    delim_regex_tap_size_kernel(LcDelimRegexSlsCfg c, DelimSlsTables t, uint64_t n, uint32_t* __restrict__ copy) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        copy[i] = lc_delim_regex_tap(c, delim_sls_row(c.d, t, nullptr, nullptr, i)).copy;
}

__global__ void __launch_bounds__(256)
    delim_regex_tap_kernel(LcDelimRegexSlsCfg c, DelimSlsTables t, uint64_t n, const uint64_t* __restrict__ slot,
                           uint64_t side_at, uint8_t* base, uint32_t* __restrict__ val_off,
                           uint32_t* __restrict__ val_len) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const LcDelimSlsRow r = delim_sls_row(c.d, t, nullptr, nullptr, i);
    const LcDrTap v = lc_delim_regex_tap(c, r);
    uint32_t off = v.off;
    if (v.copy) {
        off = (uint32_t)(side_at + slot[i]);
        lc_delim_regex_copy(c, base, r, base + off, v.copy);
    }
    val_off[i] = off;
    val_len[i] = v.len;
}

__device__ __forceinline__ LcDelimRegexSlsRow delim_regex_sls_row(const LcDelimRegexSlsCfg& c,
                                                                  const DelimRegexSlsTables& t, const uint32_t* ev_time,
                                                                  const uint32_t* ev_ns, uint64_t i) {
    LcDelimRegexSlsRow r;
    r.d = delim_sls_row(c.d, t.d, ev_time, ev_ns, i);
    r.vo = t.val_off[i];
    r.vl = t.val_len[i];
    r.status = t.status ? t.status[i] : 0u;
    r.co = t.cap_off ? t.cap_off + i * c.x.pitch : nullptr;
    r.cl = t.cap_len ? t.cap_len + i * c.x.pitch : nullptr;
    return r;
}

__global__ void __launch_bounds__(256)
    delim_regex_sls_size_kernel(LcDelimRegexSlsCfg c, DelimRegexSlsTables t, const uint32_t* __restrict__ ev_ns,
                                uint64_t n, uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    LcDelimRegexVerdict v = {};
    if (i < n) {
        const LcDelimRegexSlsRow r = delim_regex_sls_row(c, t, nullptr, ev_ns, i);
        LcSlsCount s{0};
        const uint32_t cnt = lc_delim_regex_sls_body(c, t.d.base, r, s);
        const uint32_t body = cnt ? s.n : 0u;
        rec_size[i] = cnt ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        v = lc_delim_regex_verdict(c, r, cnt);
    }
    if (counters) { // one atomic per warp and counter
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, v.ctr[k]);
            if ((threadIdx.x & 31) == 0 && w)
                atomicAdd(counters + k, (unsigned long long)w);
        }
    }
}

__global__ void __launch_bounds__(256)
    delim_regex_sls_emit_kernel(LcDelimRegexSlsCfg c, DelimRegexSlsTables t, const uint32_t* __restrict__ ev_time,
                                const uint32_t* __restrict__ ev_ns, uint64_t n, const uint64_t* __restrict__ rec_off,
                                const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased or LogEvent::Empty: no record (SLSSerializer.cpp:383-385)
    const LcDelimRegexSlsRow r = delim_regex_sls_row(c, t, ev_time, ev_ns, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_delim_regex_sls_body(c, t.d.base, r, s);
}

void launch_delim_regex_tap_sizes(const LcDelimRegexSlsCfg& c, const DelimSlsTables& t, uint64_t n, uint32_t* d_copy,
                                  cudaStream_t st) {
    if (n)
        delim_regex_tap_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_copy);
}

void launch_delim_regex_tap(const LcDelimRegexSlsCfg& c, const DelimSlsTables& t, uint64_t n, const uint64_t* d_slot,
                            uint64_t side_at, uint8_t* d_base, uint32_t* d_val_off, uint32_t* d_val_len,
                            cudaStream_t st) {
    if (n)
        delim_regex_tap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_slot, side_at, d_base,
                                                                             d_val_off, d_val_len);
}

void launch_delim_regex_sls_sizes(const LcDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, const uint32_t* d_ev_ns,
                                  uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                                  unsigned long long* d_counters, cudaStream_t st) {
    if (n)
        delim_regex_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, d_ev_ns, n, d_rec_size,
                                                                                  d_body_size, d_counters);
}

void launch_delim_regex_sls_emit(const LcDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, const uint32_t* d_ev_time,
                                 const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off,
                                 const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st) {
    if (n)
        delim_regex_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, d_ev_time, d_ev_ns, n,
                                                                                       d_rec_off, d_body_size, d_out);
}

// ---- f4, split -> delimiter chain: Log records of the pieces a splitter cut and a ProcessorParseDelimiterNative
// parsed, straight from the piece tables and the delimiter tables over them (lc_exec.cuh: lc_split_delim_sls_body) --
// the size pass one thread per piece, the emit pass one warp per piece.  counters: u64 [5] += successful, failed,
// discarded, blank, pieces whose record would reach 4 GiB (their size is left 0 and the call is refused).
__device__ __forceinline__ LcDelimSlsRow split_delim_sls_row(const LcSplitDelimSlsCfg& c, const DelimSlsTables& t,
                                                             uint64_t i) {
    LcDelimSlsRow r;
    r.eo = t.ev_off[i];
    r.elen = t.ev_len[i];
    r.status = t.status[i];
    r.nf = t.nfields[i];
    r.fo = t.f_off + i * c.d.max_fields;
    r.fl = t.f_len + i * c.d.max_fields;
    r.fd = t.f_dq + i * c.d.max_fields;
    r.time = c.time;
    r.has_ns = c.has_ns;
    r.ns = c.ns;
    return r;
}

__global__ void __launch_bounds__(256)
    split_delim_sls_size_kernel(LcSplitDelimSlsCfg c, DelimSlsTables t, uint64_t n, uint32_t* __restrict__ rec_size,
                                uint32_t* __restrict__ body_size, unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    LcDelimSlsVerdict v{0u, 0u, 0u, 0u};
    uint32_t big = 0;
    if (i < n) {
        const LcDelimSlsRow r = split_delim_sls_row(c, t, i);
        LcSlsCount64 s{0};
        const uint32_t cnt = lc_split_delim_sls_body(c, t.base, r, s);
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        v = lc_delim_sls_verdict(c.d, r.status);
    }
    // one atomic per warp and counter
    const uint32_t w[5] = {__reduce_add_sync(0xFFFFFFFFu, v.ok), __reduce_add_sync(0xFFFFFFFFu, v.failed),
                           __reduce_add_sync(0xFFFFFFFFu, v.erased), __reduce_add_sync(0xFFFFFFFFu, v.blank),
                           __reduce_add_sync(0xFFFFFFFFu, big)};
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 5; ++k)
            if (w[k])
                atomicAdd(counters + k, (unsigned long long)w[k]);
    }
}

__global__ void __launch_bounds__(256)
    split_delim_sls_emit_kernel(LcSplitDelimSlsCfg c, DelimSlsTables t, uint64_t n,
                                const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ body_size,
                                uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased: no record
    const LcDelimSlsRow r = split_delim_sls_row(c, t, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_delim_sls_body(c, t.base, r, s);
}

void launch_split_delim_sls_sizes(const LcSplitDelimSlsCfg& c, const DelimSlsTables& t, uint64_t n,
                                  uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                  cudaStream_t st) {
    if (n)
        split_delim_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_size, d_body_size,
                                                                                  d_counters);
}

void launch_split_delim_sls_emit(const LcSplitDelimSlsCfg& c, const DelimSlsTables& t, uint64_t n,
                                 const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                 cudaStream_t st) {
    if (n)
        split_delim_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_off, d_body_size,
                                                                                       d_out);
}

// ---- f4, split -> delimiter -> regex chain: Log records of the pieces a splitter cut, a ProcessorParseDelimiterNative
// parsed and a ProcessorParseRegexNative parsed one column of (lc_exec.cuh: lc_split_delim_regex_sls_body), from the
// piece, delimiter, value and regex tables -- the size pass one thread per piece, the emit pass one warp per piece.
// counters: u64 [9] += lc_delim_regex_verdict's 8, pieces whose record would reach 4 GiB (their size is left 0 and the
// call is refused).
__device__ __forceinline__ LcDelimRegexSlsRow split_delim_regex_sls_row(const LcSplitDelimRegexSlsCfg& c,
                                                                        const DelimRegexSlsTables& t, uint64_t i) {
    LcDelimRegexSlsRow r;
    r.d = split_delim_sls_row(c.s, t.d, i);
    r.vo = t.val_off[i];
    r.vl = t.val_len[i];
    r.status = t.status ? t.status[i] : 0u;
    r.co = t.cap_off ? t.cap_off + i * c.r.x.pitch : nullptr;
    r.cl = t.cap_len ? t.cap_len + i * c.r.x.pitch : nullptr;
    return r;
}

__global__ void __launch_bounds__(256)
    split_delim_regex_sls_size_kernel(LcSplitDelimRegexSlsCfg c, DelimRegexSlsTables t, uint64_t n,
                                      uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                      unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    LcDelimRegexVerdict v = {};
    uint32_t big = 0;
    if (i < n) {
        const LcDelimRegexSlsRow r = split_delim_regex_sls_row(c, t, i);
        LcSlsCount64 s{0};
        const uint32_t cnt = lc_split_delim_regex_sls_body(c, t.d.base, r, s);
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        v = lc_split_delim_regex_verdict(c, r, cnt);
    }
    // one atomic per warp and counter
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, k < 8 ? v.ctr[k] : big);
        if ((threadIdx.x & 31) == 0 && w)
            atomicAdd(counters + k, (unsigned long long)w);
    }
}

__global__ void __launch_bounds__(256)
    split_delim_regex_sls_emit_kernel(LcSplitDelimRegexSlsCfg c, DelimRegexSlsTables t, uint64_t n,
                                      const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ body_size,
                                      uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased: no record
    const LcDelimRegexSlsRow r = split_delim_regex_sls_row(c, t, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_delim_regex_sls_body(c, t.d.base, r, s);
}

void launch_split_delim_regex_sls_sizes(const LcSplitDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, uint64_t n,
                                        uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                        cudaStream_t st) {
    if (n)
        split_delim_regex_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_size,
                                                                                        d_body_size, d_counters);
}

void launch_split_delim_regex_sls_emit(const LcSplitDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, uint64_t n,
                                       const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                       cudaStream_t st) {
    if (n)
        split_delim_regex_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_off,
                                                                                             d_body_size, d_out);
}

// ---- f4, split-fed: Log records of the pieces a splitter cuts from one source value (lc_exec.cuh: lc_span_sls_rec,
// lc_span_sls_tile).  The size pass runs one thread per piece; the emit pass one warp per kSpanTile bytes of OUTPUT,
// so records of 0 B and of many MiB share a launch without one warp copying a whole long record.
__global__ void __launch_bounds__(256)
    span_sls_size_kernel(LcSpanSlsCfg c, uint64_t n, uint32_t* __restrict__ rec_size) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        rec_size[i] = lc_span_sls_rec(c, c.off[i], c.len[i]).size;
}

__global__ void __launch_bounds__(256)
    span_sls_emit_kernel(LcSpanSlsCfg c, const uint64_t* __restrict__ rec_off, uint64_t n, uint64_t total,
                         uint8_t* __restrict__ out) {
    const uint64_t t0 = (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * kSpanTile;
    if (t0 >= total)
        return;
    const uint64_t t1 = t0 + kSpanTile < total ? t0 + kSpanTile : total;
    lc_span_sls_tile(c, rec_off, n, lc_span_sls_find(rec_off, n, t0), t0, t1, out, threadIdx.x & 31, 32);
}

void launch_span_sls_sizes(const LcSpanSlsCfg& c, uint64_t n, uint32_t* d_rec_size, cudaStream_t st) {
    if (n)
        span_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, n, d_rec_size);
}

void launch_span_sls_emit(const LcSpanSlsCfg& c, const uint64_t* d_rec_off, uint64_t n, uint64_t total, uint8_t* d_out,
                          cudaStream_t st) {
    const uint64_t warps = (total + kSpanTile - 1) / kSpanTile;
    if (n && total)
        span_sls_emit_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(c, d_rec_off, n, total, d_out);
}

// ---- f4, LZ4: one block per segment (lc_exec.cuh: lc_lz4_parse_chunk, lc_lz4_seg_sizes, lc_lz4_emit_chunk).  The
// parse and emit passes run one warp per chunk of LC_LZ4_CHUNK bytes, each warp with its own hash table in shared
// memory; the size pass one thread per segment over that segment's chunk summaries.
constexpr int kLz4Warps = 4; // warps per block of the parse and emit kernels

__global__ void __launch_bounds__(256)
    lz4_chunks_kernel(const uint32_t* __restrict__ seg_len, uint64_t nseg, uint32_t* __restrict__ nch,
                      uint32_t* too_large) {
    const uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nseg)
        return;
    const uint32_t n = seg_len[s];
    if (n > LC_LZ4_MAX_INPUT)
        atomicOr(too_large, 1u);
    nch[s] = lc_lz4_nchunks(n > LC_LZ4_MAX_INPUT ? 0u : n);
}

// chunk k of [k0, k1): its segment, its range [c0, c1) and the segment's bytes
struct Lz4ChunkRef {
    const uint8_t* s;
    uint32_t n, c0, c1;
    bool last;
};
__device__ __forceinline__ Lz4ChunkRef lz4_chunk(const uint8_t* in, const uint64_t* seg_off, const uint32_t* seg_len,
                                                 const uint64_t* first, uint64_t nseg, uint64_t nchunks, uint64_t k) {
    const uint64_t g = lc_span_sls_find(first, nseg, k);
    const uint64_t next = g + 1 < nseg ? first[g + 1] : nchunks;
    Lz4ChunkRef r;
    r.s = in + seg_off[g];
    r.n = seg_len[g];
    r.c0 = (uint32_t)(k - first[g]) * LC_LZ4_CHUNK;
    r.c1 = r.n - r.c0 < LC_LZ4_CHUNK ? r.n : r.c0 + LC_LZ4_CHUNK;
    r.last = k + 1 == next;
    return r;
}

__global__ void __launch_bounds__(32 * kLz4Warps)
    lz4_parse_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ seg_off,
                     const uint32_t* __restrict__ seg_len, const uint64_t* __restrict__ first, uint64_t nseg,
                     uint64_t nchunks, uint64_t k0, uint64_t k1, LcLz4Seq* __restrict__ seq,
                     LcLz4Chunk* __restrict__ info) {
    __shared__ LcLz4Warp s_w[kLz4Warps];
    const uint32_t wid = threadIdx.x >> 5;
    const uint64_t k = k0 + (uint64_t)blockIdx.x * kLz4Warps + wid;
    if (k >= k1)
        return;
    const Lz4ChunkRef r = lz4_chunk(in, seg_off, seg_len, first, nseg, nchunks, k);
    lc_lz4_parse_chunk(r.s, r.n, r.c0, r.c1, s_w[wid], seq + k * LC_LZ4_SEQ_CAP, info + k, threadIdx.x & 31, 32);
}

__global__ void __launch_bounds__(256)
    lz4_sizes_kernel(const uint32_t* __restrict__ seg_len, const uint64_t* __restrict__ first, uint64_t nseg,
                     uint64_t nchunks, const LcLz4Chunk* __restrict__ info, uint32_t* __restrict__ csize,
                     uint32_t* __restrict__ anchor) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nseg)
        return;
    const uint64_t k = first[g], next = g + 1 < nseg ? first[g + 1] : nchunks;
    lc_lz4_seg_sizes(seg_len[g], (uint32_t)(next - k), info + k, csize + k, anchor + k);
}

__global__ void __launch_bounds__(256)
    lz4_blocks_kernel(const uint64_t* __restrict__ first, const uint64_t* __restrict__ choff,
                      const uint64_t* __restrict__ total, uint64_t nseg, uint64_t* __restrict__ blk_off,
                      uint32_t* __restrict__ blk_len) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nseg)
        return;
    const uint64_t a = choff[first[g]], b = g + 1 < nseg ? choff[first[g + 1]] : *total;
    blk_off[g] = a;
    blk_len[g] = (uint32_t)(b - a);
}

__global__ void __launch_bounds__(32 * kLz4Warps, 1)
    lz4_emit_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ seg_off,
                    const uint32_t* __restrict__ seg_len, const uint64_t* __restrict__ first, uint64_t nseg,
                    uint64_t nchunks, const LcLz4Seq* __restrict__ seq, const LcLz4Chunk* __restrict__ info,
                    const uint32_t* __restrict__ anchor, const uint64_t* __restrict__ choff, uint8_t* __restrict__ out) {
    const uint64_t k = (uint64_t)blockIdx.x * kLz4Warps + (threadIdx.x >> 5);
    if (k >= nchunks)
        return;
    const Lz4ChunkRef r = lz4_chunk(in, seg_off, seg_len, first, nseg, nchunks, k);
    lc_lz4_emit_chunk(r.s, r.n, r.c0, seq + k * LC_LZ4_SEQ_CAP, info[k].nseq, anchor[k], r.last, out + choff[k],
                      threadIdx.x & 31, 32);
}

void launch_lz4_chunks(const uint32_t* d_seg_len, uint64_t nseg, uint32_t* d_nch, uint32_t* d_too_large,
                       cudaStream_t st) {
    if (nseg)
        lz4_chunks_kernel<<<(unsigned)((nseg + 255) / 256), 256, 0, st>>>(d_seg_len, nseg, d_nch, d_too_large);
}

void launch_lz4_parse(const Lz4Segs& g, uint64_t k0, uint64_t k1, LcLz4Seq* d_seq, LcLz4Chunk* d_info,
                      cudaStream_t st) {
    if (k1 > k0)
        lz4_parse_kernel<<<(unsigned)((k1 - k0 + kLz4Warps - 1) / kLz4Warps), 32 * kLz4Warps, 0, st>>>(
            g.in, g.seg_off, g.seg_len, g.first, g.nseg, g.nchunks, k0, k1, d_seq, d_info);
}

void launch_lz4_sizes(const Lz4Segs& g, const LcLz4Chunk* d_info, uint32_t* d_csize, uint32_t* d_anchor,
                      cudaStream_t st) {
    if (g.nseg)
        lz4_sizes_kernel<<<(unsigned)((g.nseg + 255) / 256), 256, 0, st>>>(g.seg_len, g.first, g.nseg, g.nchunks,
                                                                            d_info, d_csize, d_anchor);
}

void launch_lz4_emit(const Lz4Segs& g, const LcLz4Seq* d_seq, const LcLz4Chunk* d_info, const uint32_t* d_anchor,
                     const uint64_t* d_choff, const uint64_t* d_total, uint8_t* d_out, uint64_t* d_blk_off,
                     uint32_t* d_blk_len, cudaStream_t st) {
    if (!g.nseg)
        return;
    lz4_blocks_kernel<<<(unsigned)((g.nseg + 255) / 256), 256, 0, st>>>(g.first, d_choff, d_total, g.nseg, d_blk_off,
                                                                         d_blk_len);
    lz4_emit_kernel<<<(unsigned)((g.nchunks + kLz4Warps - 1) / kLz4Warps), 32 * kLz4Warps, 0, st>>>(
        g.in, g.seg_off, g.seg_len, g.first, g.nseg, g.nchunks, d_seq, d_info, d_anchor, d_choff, d_out);
}

// ---- f4, zstd: one frame per segment (lc_exec.cuh: lc_zstd_block, lc_zstd_emit_block) over the matches of the LZ4
// parse pass.  The block pass runs one warp per 128 KiB block, the emit pass one warp per block.
constexpr int kZstdWarps = 4; // warps per block of the zstd block and emit kernels

__global__ void __launch_bounds__(256)
    zstd_nblocks_kernel(const uint32_t* __restrict__ seg_len, uint64_t nseg, uint32_t* __restrict__ nblk) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < nseg)
        nblk[g] = lc_zstd_nblocks(seg_len[g]);
}

__global__ void __launch_bounds__(32 * kZstdWarps)
    zstd_block_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ seg_off,
                      const uint32_t* __restrict__ seg_len, const uint64_t* __restrict__ first,
                      const uint64_t* __restrict__ bfirst, uint64_t nseg, uint64_t nblocks, LcLz4Seq* seq,
                      const LcLz4Chunk* __restrict__ info, uint8_t* __restrict__ slot, uint32_t* __restrict__ body,
                      uint32_t* __restrict__ esz) {
    __shared__ LcZstdWarp s_w[kZstdWarps];
    const uint32_t wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t k = (uint64_t)blockIdx.x * kZstdWarps + wid;
    if (k >= nblocks)
        return;
    const uint64_t g = lc_span_sls_find(bfirst, nseg, k);
    const uint32_t n = seg_len[g], j = (uint32_t)(k - bfirst[g]), b0 = j * LC_ZSTD_BLOCK;
    const uint64_t c = first[g] + 2 * j;
    LcZstdBlk b{in + seg_off[g], b0, n - b0 < LC_ZSTD_BLOCK ? n : b0 + LC_ZSTD_BLOCK, {seq + c * LC_LZ4_SEQ_CAP, nullptr},
                {info[c].nseq, 0}};
    if (b.b1 - b.b0 > LC_LZ4_CHUNK) {
        b.seq[1] = seq + (c + 1) * LC_LZ4_SEQ_CAP;
        b.nseq[1] = info[c + 1].nseq;
    }
    const uint32_t z = lc_zstd_block(b, slot + k * LC_ZSTD_BLOCK, s_w[wid], lane, 32);
    if (lane == 0) {
        body[k] = z;
        esz[k] = lc_zstd_emit_size(n, j, z);
    }
}

__global__ void __launch_bounds__(256)
    zstd_frames_kernel(const uint64_t* __restrict__ bfirst, const uint64_t* __restrict__ boff,
                       const uint64_t* __restrict__ total, uint64_t nseg, uint64_t* __restrict__ frm_off,
                       uint32_t* __restrict__ frm_len) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= nseg)
        return;
    const uint64_t a = boff[bfirst[g]], e = g + 1 < nseg ? boff[bfirst[g + 1]] : *total;
    frm_off[g] = a;
    frm_len[g] = (uint32_t)(e - a);
}

__global__ void __launch_bounds__(32 * kZstdWarps)
    zstd_emit_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ seg_off,
                     const uint32_t* __restrict__ seg_len, const uint64_t* __restrict__ bfirst, uint64_t nseg,
                     uint64_t nblocks, const uint8_t* __restrict__ slot, const uint32_t* __restrict__ body,
                     const uint64_t* __restrict__ boff, uint8_t* __restrict__ out) {
    const uint64_t k = (uint64_t)blockIdx.x * kZstdWarps + (threadIdx.x >> 5);
    if (k >= nblocks)
        return;
    const uint64_t g = lc_span_sls_find(bfirst, nseg, k);
    lc_zstd_emit_block(in + seg_off[g], seg_len[g], (uint32_t)(k - bfirst[g]), slot + k * LC_ZSTD_BLOCK, body[k],
                       out + boff[k], threadIdx.x & 31, 32);
}

void launch_zstd_nblocks(const uint32_t* d_seg_len, uint64_t nseg, uint32_t* d_nblk, cudaStream_t st) {
    if (nseg)
        zstd_nblocks_kernel<<<(unsigned)((nseg + 255) / 256), 256, 0, st>>>(d_seg_len, nseg, d_nblk);
}

void launch_zstd_blocks(const Lz4Segs& g, const uint64_t* d_bfirst, uint64_t nblocks, LcLz4Seq* d_seq,
                        const LcLz4Chunk* d_info, uint8_t* d_slot, uint32_t* d_body, uint32_t* d_esz, cudaStream_t st) {
    if (nblocks)
        zstd_block_kernel<<<(unsigned)((nblocks + kZstdWarps - 1) / kZstdWarps), 32 * kZstdWarps, 0, st>>>(
            g.in, g.seg_off, g.seg_len, g.first, d_bfirst, g.nseg, nblocks, d_seq, d_info, d_slot, d_body, d_esz);
}

void launch_zstd_emit(const Lz4Segs& g, const uint64_t* d_bfirst, uint64_t nblocks, const uint8_t* d_slot,
                      const uint32_t* d_body, const uint64_t* d_boff, const uint64_t* d_total, uint8_t* d_out,
                      uint64_t* d_frm_off, uint32_t* d_frm_len, cudaStream_t st) {
    if (!g.nseg)
        return;
    zstd_frames_kernel<<<(unsigned)((g.nseg + 255) / 256), 256, 0, st>>>(d_bfirst, d_boff, d_total, g.nseg, d_frm_off,
                                                                          d_frm_len);
    zstd_emit_kernel<<<(unsigned)((nblocks + kZstdWarps - 1) / kZstdWarps), 32 * kZstdWarps, 0, st>>>(
        g.in, g.seg_off, g.seg_len, d_bfirst, g.nseg, nblocks, d_slot, d_body, d_boff, d_out);
}

// ---------------------------------------------------------------------------------------------- timestamp parse
__global__ void __launch_bounds__(256)
    ts_full_kernel(const LcTsConf* __restrict__ conf, LcTsNow now, const uint8_t* __restrict__ base, LcTsSpans sp,
                   uint64_t n, LcTsFull* __restrict__ full) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t o, l;
    if (i >= n || !sp.get(i, o, l))
        return;
    full[i] = lc_ts_full(*conf, now, base + o, l);
}

constexpr int kTsWarps = 4;

__global__ void __launch_bounds__(32 * kTsWarps)
    ts_resolve_kernel(const LcTsConf* __restrict__ conf, LcTsNow now, const uint8_t* __restrict__ base, LcTsSpans sp,
                      const LcTsFull* __restrict__ full, const uint32_t* __restrict__ grp, uint64_t ngroups,
                      int64_t* __restrict__ sec, uint32_t* __restrict__ nsec, uint8_t* __restrict__ status,
                      unsigned long long* __restrict__ counters) {
    __shared__ LcTsWarp ws[kTsWarps];
    const uint32_t wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t cnt[5] = {0, 0, 0, 0, 0};
    for (uint64_t g = (uint64_t)blockIdx.x * kTsWarps + wi; g < ngroups; g += (uint64_t)gridDim.x * kTsWarps)
        lc_ts_resolve(*conf, now, base, sp, full, grp[g], grp[g + 1], sec, nsec, status, cnt, ws[wi], lane, 32);
    for (int k = 0; k < 5; ++k) {
        const uint32_t t = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)cnt[k]);
        if (lane == 0 && t)
            atomicAdd(&counters[k], (unsigned long long)t);
    }
}

void launch_ts_full(const LcTsConf* d_conf, const LcTsNow& now, const uint8_t* d_base, const LcTsSpans& sp, uint64_t n,
                    LcTsFull* d_full, cudaStream_t st) {
    if (n)
        ts_full_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_conf, now, d_base, sp, n, d_full);
}

void launch_ts_resolve(const LcTsConf* d_conf, const LcTsNow& now, const uint8_t* d_base, const LcTsSpans& sp, const LcTsFull* d_full,
                       const uint32_t* d_grp, uint64_t ngroups, int64_t* d_sec, uint32_t* d_nsec, uint8_t* d_status,
                       unsigned long long* d_counters, cudaStream_t st) {
    if (!ngroups)
        return;
    const uint64_t blocks = (ngroups + kTsWarps - 1) / kTsWarps;
    ts_resolve_kernel<<<(unsigned)(blocks < (1u << 20) ? blocks : (1u << 20)), 32 * kTsWarps, 0, st>>>(
        d_conf, now, d_base, sp, d_full, d_grp, ngroups, d_sec, d_nsec, d_status, d_counters);
}

// ================================================================================================ Apsara parse
__global__ void __launch_bounds__(256)
    ap_scan_kernel(const LcTsConf* __restrict__ conf, const uint8_t* __restrict__ base, uint64_t base_len,
                   const uint32_t* __restrict__ off, const uint32_t* __restrict__ len, uint64_t n,
                   const uint8_t* __restrict__ skey, uint32_t sklen, LcApEv* __restrict__ ev, uint32_t* bad) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n)
        return;
    const uint32_t l = len[i], o = l == LC_AP_NO_KEY ? 0u : off[i];
    if (l != LC_AP_NO_KEY && (uint64_t)o + l > base_len) {
        atomicOr(bad, 1u);
        ev[i] = LcApEv{0, 0, 0, {0, 0, 0, 0, 0}, 0, LC_AP_F_NONE, 0};
        return;
    }
    ev[i] = lc_ap_scan(*conf, base, base_len, o, l, skey, sklen);
}

constexpr int kApWarps = 4;

__global__ void __launch_bounds__(32 * kApWarps)
    ap_resolve_kernel(LcTsNow now, const LcApEv* __restrict__ ev, const uint32_t* __restrict__ grp, uint64_t ngroups,
                      uint8_t* __restrict__ status, int64_t* __restrict__ sec, uint32_t* __restrict__ nsec,
                      int64_t* __restrict__ micro, uint32_t* __restrict__ nent,
                      unsigned long long* __restrict__ counters) {
    __shared__ LcApWarp ws[kApWarps];
    const uint32_t wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t cnt[5] = {0, 0, 0, 0, 0};
    for (uint64_t g = (uint64_t)blockIdx.x * kApWarps + wi; g < ngroups; g += (uint64_t)gridDim.x * kApWarps)
        lc_ap_resolve(now, ev, grp[g], grp[g + 1], status, sec, nsec, micro, nent, cnt, ws[wi], lane, 32);
    for (int k = 0; k < 5; ++k) {
        const uint32_t t = __reduce_add_sync(0xFFFFFFFFu, (uint32_t)cnt[k]);
        if (lane == 0 && t)
            atomicAdd(&counters[k], (unsigned long long)t);
    }
}

__global__ void __launch_bounds__(256)
    ap_emit_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ off,
                   const uint32_t* __restrict__ len, const uint8_t* __restrict__ status, uint64_t n,
                   const uint64_t* __restrict__ first, LcApEntry* __restrict__ entries) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || (status[i] & 7u) != LC_AP_ST_OK)
        return;
    LcApEmit em{entries + first[i], off[i]};
    lc_ap_fields(base + off[i], len[i], em);
}

void launch_ap_scan(const LcTsConf* d_conf, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_off,
                    const uint32_t* d_len, uint64_t n, const uint8_t* d_skey, uint32_t sklen, LcApEv* d_ev,
                    uint32_t* d_bad, cudaStream_t st) {
    if (n)
        ap_scan_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_conf, d_base, base_len, d_off, d_len, n, d_skey,
                                                                     sklen, d_ev, d_bad);
}

void launch_ap_resolve(const LcTsNow& now, const LcApEv* d_ev, const uint32_t* d_grp, uint64_t ngroups,
                       uint8_t* d_status, int64_t* d_sec, uint32_t* d_nsec, int64_t* d_micro, uint32_t* d_nent,
                       unsigned long long* d_counters, cudaStream_t st) {
    if (!ngroups)
        return;
    const uint64_t blocks = (ngroups + kApWarps - 1) / kApWarps;
    ap_resolve_kernel<<<(unsigned)(blocks < (1u << 20) ? blocks : (1u << 20)), 32 * kApWarps, 0, st>>>(
        now, d_ev, d_grp, ngroups, d_status, d_sec, d_nsec, d_micro, d_nent, d_counters);
}

void launch_ap_emit(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len, const uint8_t* d_status,
                    uint64_t n, const uint64_t* d_first, LcApEntry* d_entries, cudaStream_t st) {
    if (n)
        ap_emit_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_base, d_off, d_len, d_status, n, d_first,
                                                                     d_entries);
}

// ================================================================================================ JSON parse
// counters[3] of the JSON count passes from one warp: every lane calls it
__device__ __forceinline__ void json_add_counters(uint32_t st, bool valid, unsigned long long* counters) {
    const uint32_t s = st & 0x7Fu;
    const uint32_t c0 = __reduce_add_sync(0xFFFFFFFFu, valid && s == LC_JSON_ST_NOT_FOUND ? 1u : 0u);
    const uint32_t c1 = __reduce_add_sync(0xFFFFFFFFu, valid && s == LC_JSON_ST_FAILED ? 1u : 0u);
    const uint32_t c2 = __reduce_add_sync(0xFFFFFFFFu, valid && s == LC_JSON_ST_OK ? 1u : 0u);
    if ((threadIdx.x & 31) == 0) {
        if (c0)
            atomicAdd(&counters[0], (unsigned long long)c0);
        if (c1)
            atomicAdd(&counters[1], (unsigned long long)c1);
        if (c2)
            atomicAdd(&counters[2], (unsigned long long)c2);
    }
}

__global__ void __launch_bounds__(256)
    json_count_kernel(const uint8_t* __restrict__ base, uint64_t base_len, const uint32_t* __restrict__ off,
                      const uint32_t* __restrict__ len, uint64_t n, const uint8_t* __restrict__ skey, uint32_t sklen, const uint64_t* __restrict__ pow5,
                      uint8_t* __restrict__ status, uint32_t* __restrict__ nent, uint32_t* __restrict__ narena,
                      uint8_t* __restrict__ slow, uint32_t* __restrict__ slow_list, uint32_t* nslow, uint32_t* bad,
                      unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < n;
    uint32_t st = LC_JSON_ST_FAILED, ne = 0, na = 0;
    bool sl = false;
    if (valid) {
        const uint32_t l = len[i], o = l == LC_JSON_NO_KEY ? 0u : off[i];
        if (l != LC_JSON_NO_KEY && (uint64_t)o + l > base_len)
            atomicOr(bad, 1u);
        else
            st = lc_json_count<false>(base, o, l, skey, sklen, pow5, &ne, &na, &sl);
        if (sl)
            slow_list[atomicAdd(nslow, 1u)] = (uint32_t)i;
        status[i] = (uint8_t)st;
        nent[i] = ne;
        narena[i] = na;
        slow[i] = sl ? 1 : 0;
    }
    json_add_counters(st, valid && !sl, counters);
}

__global__ void __launch_bounds__(128)
    json_count_slow_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ off,
                           const uint32_t* __restrict__ len, const uint8_t* __restrict__ skey, uint32_t sklen, const uint64_t* __restrict__ pow5,
                           const uint32_t* __restrict__ slow_list, const uint32_t* __restrict__ nslow,
                           uint8_t* __restrict__ status, uint32_t* __restrict__ nent, uint32_t* __restrict__ narena,
                           unsigned long long* __restrict__ counters) {
    const uint32_t m = *nslow, stride = gridDim.x * blockDim.x;
    for (uint32_t j0 = blockIdx.x * blockDim.x; j0 < m; j0 += stride) {
        const uint32_t j = j0 + threadIdx.x;
        const bool valid = j < m;
        uint32_t st = LC_JSON_ST_FAILED;
        if (valid) {
            const uint32_t i = slow_list[j];
            uint32_t ne, na;
            bool sl;
            st = lc_json_count<true>(base, off[i], len[i], skey, sklen, pow5, &ne, &na, &sl);
            status[i] = (uint8_t)st;
            nent[i] = ne;
            narena[i] = na;
        }
        json_add_counters(st, valid, counters);
    }
}

__global__ void __launch_bounds__(256)
    json_emit_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ off,
                     const uint32_t* __restrict__ len, uint64_t n, const uint8_t* __restrict__ skey, uint32_t sklen, const uint64_t* __restrict__ pow5,
                     const uint8_t* __restrict__ status, const uint8_t* __restrict__ slow,
                     const uint64_t* __restrict__ first, const uint64_t* __restrict__ afirst,
                     LcJsonEntry* __restrict__ entries, uint8_t* __restrict__ arena, uint32_t* bad) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || slow[i] || (status[i] & 0x7Fu) != LC_JSON_ST_OK)
        return;
    const uint64_t e0 = first[i], a0 = afirst[i];
    if (!lc_json_emit<false>(base, off[i], len[i], skey, sklen, pow5, entries + e0, (uint32_t)(first[i + 1] - e0),
                             arena + a0, (uint32_t)a0, (uint32_t)(afirst[i + 1] - a0)))
        atomicOr(bad, 2u);
}

__global__ void __launch_bounds__(128)
    json_emit_slow_kernel(const uint8_t* __restrict__ base, const uint32_t* __restrict__ off,
                          const uint32_t* __restrict__ len, const uint8_t* __restrict__ skey, uint32_t sklen, const uint64_t* __restrict__ pow5,
                          const uint8_t* __restrict__ status, const uint32_t* __restrict__ slow_list,
                          const uint32_t* __restrict__ nslow, const uint64_t* __restrict__ first,
                          const uint64_t* __restrict__ afirst, LcJsonEntry* __restrict__ entries,
                          uint8_t* __restrict__ arena, uint32_t* bad) {
    const uint32_t m = *nslow;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) {
        const uint32_t i = slow_list[j];
        if ((status[i] & 0x7Fu) != LC_JSON_ST_OK)
            continue;
        const uint64_t e0 = first[i], a0 = afirst[i];
        if (!lc_json_emit<true>(base, off[i], len[i], skey, sklen, pow5, entries + e0, (uint32_t)(first[i + 1] - e0),
                                arena + a0, (uint32_t)a0, (uint32_t)(afirst[i + 1] - a0)))
            atomicOr(bad, 2u);
    }
}

// the slow kernels run a fixed grid over the device-side count of slow events, so no host round trip is needed
constexpr unsigned kJsonSlowBlocks = 264;

void launch_json_count(const uint8_t* d_base, uint64_t base_len, const uint32_t* d_off, const uint32_t* d_len,
                       uint64_t n, const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, uint8_t* d_status, uint32_t* d_nent,
                       uint32_t* d_narena, uint8_t* d_slow, uint32_t* d_slow_list, uint32_t* d_nslow, uint32_t* d_bad,
                       unsigned long long* d_counters, cudaStream_t st) {
    if (n)
        json_count_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_base, base_len, d_off, d_len, n, d_skey,
                                                                        sklen, d_pow5, d_status, d_nent, d_narena, d_slow,
                                                                        d_slow_list, d_nslow, d_bad, d_counters);
}

void launch_json_count_slow(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len,
                            const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint32_t* d_slow_list, const uint32_t* d_nslow,
                            uint8_t* d_status, uint32_t* d_nent, uint32_t* d_narena, unsigned long long* d_counters,
                            cudaStream_t st) {
    json_count_slow_kernel<<<kJsonSlowBlocks, 128, 0, st>>>(d_base, d_off, d_len, d_skey, sklen, d_pow5, d_slow_list,
                                                            d_nslow, d_status, d_nent, d_narena, d_counters);
}

void launch_json_emit(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                      const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint8_t* d_status, const uint8_t* d_slow,
                      const uint64_t* d_first, const uint64_t* d_afirst, LcJsonEntry* d_entries, uint8_t* d_arena,
                      uint32_t* d_bad, cudaStream_t st) {
    if (n)
        json_emit_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_base, d_off, d_len, n, d_skey, sklen, d_pow5,
                                                                       d_status, d_slow, d_first, d_afirst, d_entries,
                                                                       d_arena, d_bad);
}

void launch_json_emit_slow(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len,
                           const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint8_t* d_status,
                           const uint32_t* d_slow_list, const uint32_t* d_nslow, const uint64_t* d_first,
                           const uint64_t* d_afirst, LcJsonEntry* d_entries, uint8_t* d_arena, uint32_t* d_bad,
                           cudaStream_t st) {
    json_emit_slow_kernel<<<kJsonSlowBlocks, 128, 0, st>>>(d_base, d_off, d_len, d_skey, sklen, d_pow5, d_status,
                                                           d_slow_list,
                                                           d_nslow, d_first, d_afirst, d_entries, d_arena, d_bad);
}

// ---- f4, split -> JSON chain (lc_exec.cuh: lc_json_resolve_*, lc_split_json_sls_body).  The resolve pass runs one warp
// per piece; a parsed piece of more than LC_JSON_SLS_WARP members goes to the list, which json_resolve_sort_kernel
// takes one thread per piece over a fixed grid.  The size pass runs one thread per piece, the emit pass one warp per
// piece.  counters: u64 [4] += successful, failed, discarded, pieces whose record would reach 4 GiB.
__device__ __forceinline__ uint32_t split_json_members(const SplitJsonSlsTables& t, uint64_t i) {
    return (t.status[i] & 0x7Fu) == LC_JSON_ST_OK ? (uint32_t)(t.first[i + 1] - t.first[i]) : 0u;
}

__global__ void __launch_bounds__(256)
    json_resolve_warp_kernel(LcSplitJsonSlsCfg c, SplitJsonSlsTables t, uint64_t n, uint32_t* __restrict__ list,
                             uint32_t* nlist) {
    __shared__ LcJsonResolveWarp ws[8];
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= n)
        return;
    const uint32_t m = split_json_members(t, i);
    if (m > LC_JSON_SLS_WARP) {
        if (lane == 0)
            list[atomicAdd(nlist, 1u)] = (uint32_t)i;
        return;
    }
    const uint64_t f = t.first[i];
    lc_json_resolve_warp<LcJsonKeyHash>(c, t.src, t.arena, t.ent + f, m, t.win + f, t.ev + i, ws[threadIdx.x >> 5],
                                        lane);
}

__global__ void __launch_bounds__(128)
    json_resolve_sort_kernel(LcSplitJsonSlsCfg c, SplitJsonSlsTables t, const uint32_t* __restrict__ list,
                             const uint32_t* __restrict__ nlist, uint32_t* __restrict__ scratch, uint64_t n_entries) {
    const uint32_t cnt = *nlist;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < cnt; j += gridDim.x * blockDim.x) {
        const uint32_t i = list[j];
        const uint64_t f = t.first[i];
        lc_json_resolve_sort<LcJsonKeyHash>(c, t.src, t.arena, t.ent + f, split_json_members(t, i), t.win + f,
                                            t.ev + i, scratch + f, scratch + n_entries + f,
                                            scratch + 2 * n_entries + f);
    }
}

__device__ __forceinline__ LcSplitJsonSlsRow split_json_sls_row(const SplitJsonSlsTables& t, uint64_t i) {
    LcSplitJsonSlsRow r;
    const uint64_t f = t.first[i];
    r.po = t.off[i];
    r.plen = t.len[i];
    r.status = t.status[i];
    r.e = t.ent + f;
    r.win = t.win + f;
    r.m = split_json_members(t, i);
    r.ev = t.ev[i];
    return r;
}

__global__ void __launch_bounds__(256)
    split_json_sls_size_kernel(LcSplitJsonSlsCfg c, SplitJsonSlsTables t, uint64_t n, uint32_t* __restrict__ rec_size,
                               uint32_t* __restrict__ body_size, unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    LcSplitRegexVerdict v{0u, 0u, 0u};
    uint32_t big = 0;
    if (i < n) {
        const LcSplitJsonSlsRow r = split_json_sls_row(t, i);
        LcSlsCount64 s{0};
        const uint32_t cnt = lc_split_json_sls_body(c, t.src, t.arena, r, s);
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        v = lc_split_json_verdict(c, r.status);
    }
    const uint32_t ok = __reduce_add_sync(0xFFFFFFFFu, v.ok), failed = __reduce_add_sync(0xFFFFFFFFu, v.failed),
                   erased = __reduce_add_sync(0xFFFFFFFFu, v.erased);
    big = __reduce_add_sync(0xFFFFFFFFu, big);
    if ((threadIdx.x & 31) == 0) {
        if (ok)
            atomicAdd(counters + 0, (unsigned long long)ok);
        if (failed)
            atomicAdd(counters + 1, (unsigned long long)failed);
        if (erased)
            atomicAdd(counters + 2, (unsigned long long)erased);
        if (big)
            atomicAdd(counters + 3, (unsigned long long)big);
    }
}

__global__ void __launch_bounds__(256)
    split_json_sls_emit_kernel(LcSplitJsonSlsCfg c, SplitJsonSlsTables t, uint64_t n,
                               const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ body_size,
                               uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased or LogEvent::Empty: no record
    const LcSplitJsonSlsRow r = split_json_sls_row(t, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_json_sls_body(c, t.src, t.arena, r, s);
}

void launch_json_resolve(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n, uint64_t n_entries,
                         uint32_t* d_list, uint32_t* d_nlist, uint32_t* d_scratch, cudaStream_t st) {
    if (!n)
        return;
    json_resolve_warp_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_list, d_nlist);
    json_resolve_sort_kernel<<<kJsonSlowBlocks, 128, 0, st>>>(c, t, d_list, d_nlist, d_scratch, n_entries);
}

void launch_split_json_sls_sizes(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n,
                                 uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                 cudaStream_t st) {
    if (n)
        split_json_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_size, d_body_size,
                                                                                 d_counters);
}

void launch_split_json_sls_emit(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n,
                                const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                cudaStream_t st) {
    if (n)
        split_json_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_off, d_body_size,
                                                                                      d_out);
}

// ---- f4, split -> JSON -> timestamp chain (lc_exec.cuh: lc_json_ts_last_member, lc_split_json_ts_value, _time,
// _verdict).  The tap runs one warp per piece: the lanes scan the piece's members backward for tkey, then share the
// copy of its value into the value buffer, so a long value (a 1 MiB string member) costs its warp n / 512 steps
// rather than n.  The size pass (one thread per piece) and the emit pass (one warp per piece) run
// lc_split_json_sls_body with each record's own time.

// n bytes s -> d by the 32 lanes of a warp: 16-byte words when both share their alignment (a chunk value, copied to
// its own offset), else bytes
__device__ __forceinline__ void split_json_ts_copy(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t n,
                                                   uint32_t lane) {
    uint32_t i = 0;
    if ((((uintptr_t)d ^ (uintptr_t)s) & 15u) == 0) {
        const uint32_t head = (uint32_t)((16u - ((uintptr_t)d & 15u)) & 15u);
        i = head < n ? head : n;
        if (lane < i)
            d[lane] = s[lane];
        const uint32_t words = (n - i) >> 4;
        uint4* dw = reinterpret_cast<uint4*>(d + i);
        const uint4* sw = reinterpret_cast<const uint4*>(s + i);
        for (uint32_t k = lane; k < words; k += 32)
            dw[k] = sw[k];
        i += words << 4;
    }
    for (uint32_t k = i + lane; k < n; k += 32)
        d[k] = s[k];
}

__global__ void __launch_bounds__(256)
    split_json_ts_tap_kernel(LcSplitJsonSlsCfg c, LcSplitJsonTsCfg tc, SplitJsonSlsTables t, uint64_t n,
                             uint8_t* __restrict__ val, uint32_t* __restrict__ off, uint32_t* __restrict__ len) {
    __shared__ uint32_t ws[8][32];
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= n)
        return;
    const LcJsonEntry* e = t.ent + t.first[i];
    const uint32_t w = lc_json_ts_last_member(tc, t.src, t.arena, e, split_json_members(t, i), ws[threadIdx.x >> 5],
                                              lane, 32);
    uint32_t from, o, l;
    lc_split_json_ts_value(c, tc, t.status[i], t.off[i], t.len[i], e, w, &from, &o, &l);
    if (lane == 0) {
        off[i] = o;
        len[i] = l;
    }
    if (l != LC_TS_NO_KEY)
        split_json_ts_copy(val + o, lc_json_span(t.src, t.arena, from), l, lane);
}

// counters: u64 [9] += the LC_SRTS_COUNTERS verdicts (one atomic per warp and counter), then pieces whose record
// would reach 4 GiB
__global__ void __launch_bounds__(256)
    split_json_ts_sls_size_kernel(LcSplitJsonSlsCfg c, LcSplitJsonTsCfg tc, SplitJsonSlsTables t, TsRowTables ts,
                                  uint64_t n, uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                  unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bits = 0, big = 0;
    if (i < n) {
        const LcSplitJsonSlsRow r = split_json_sls_row(t, i);
        const uint32_t st = ts.status[i];
        const LcSplitRegexTsTime tm = lc_split_json_ts_time(c, tc, st, ts.sec[i], ts.nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_json_sls_body(c, t.src, t.arena, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        bits = lc_split_json_ts_verdict(c, r.status, st);
    }
#pragma unroll
    for (uint32_t k = 0; k < LC_SRTS_COUNTERS; ++k) {
        const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, (bits >> k) & 1u);
        if ((threadIdx.x & 31) == 0 && v)
            atomicAdd(counters + k, (unsigned long long)v);
    }
    big = __reduce_add_sync(0xFFFFFFFFu, big);
    if ((threadIdx.x & 31) == 0 && big)
        atomicAdd(counters + LC_SRTS_COUNTERS, (unsigned long long)big);
}

__global__ void __launch_bounds__(256)
    split_json_ts_sls_emit_kernel(LcSplitJsonSlsCfg c, LcSplitJsonTsCfg tc, SplitJsonSlsTables t, TsRowTables ts,
                                  uint64_t n, const uint64_t* __restrict__ rec_off,
                                  const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased, discarded or LogEvent::Empty: no record
    const LcSplitJsonSlsRow r = split_json_sls_row(t, i);
    // lc_split_json_ts_time's rule for a piece with a record, as selects on the kernel parameters: a struct of the
    // three kept live across the body costs this kernel 20 bytes of spills
    const bool ok = ts.status[i] == LC_TS_ST_OK;
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_json_sls_body(c, t.src, t.arena, r, ok ? (uint32_t)ts.sec[i] : c.time, ok ? tc.enable_ns : c.has_ns,
                           ok ? ts.nsec[i] : c.ns, s);
}

void launch_split_json_ts_tap(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc, const SplitJsonSlsTables& t,
                              uint64_t n, uint8_t* d_val, uint32_t* d_off, uint32_t* d_len, cudaStream_t st) {
    if (n)
        split_json_ts_tap_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, tc, t, n, d_val, d_off, d_len);
}

void launch_split_json_ts_sls_sizes(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc,
                                    const SplitJsonSlsTables& t, const TsRowTables& ts, uint64_t n,
                                    uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                    cudaStream_t st) {
    if (n)
        split_json_ts_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_size,
                                                                                    d_body_size, d_counters);
}

void launch_split_json_ts_sls_emit(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc,
                                   const SplitJsonSlsTables& t, const TsRowTables& ts, uint64_t n,
                                   const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                   cudaStream_t st) {
    if (n)
        split_json_ts_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_off,
                                                                                         d_body_size, d_out);
}

// ---- f4, split -> delimiter -> timestamp chain (lc_exec.cuh: lc_split_delim_ts_value, _collapse, _time, _verdict).
// The tap runs one warp per piece and copies its value into the value buffer at the value's own offset: every value
// lies inside its piece and a collapsed column is never longer than the column, so no two values share bytes.  Unlike
// the delimiter -> regex tap (lc_delim_regex_tap), it needs no sizing pass for side copies and no region behind the
// source.  A plain value is the warp's shared copy (split_json_ts_copy); a column with doubled quotes is collapsed
// 32 bytes per step.  The size pass (one thread per piece) and the emit pass (one warp per piece) are the split ->
// delimiter chain's, with each record's own time.
__global__ void __launch_bounds__(256)
    split_delim_ts_tap_kernel(LcSplitDelimSlsCfg c, LcSplitDelimTsCfg tc, DelimSlsTables t, uint64_t n,
                              uint8_t* __restrict__ val, uint32_t* __restrict__ off, uint32_t* __restrict__ len) {
    __shared__ uint32_t ws[8][32];
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (i >= n)
        return;
    const LcSplitDelimTsValue v = lc_split_delim_ts_value(c, tc, split_delim_sls_row(c, t, i));
    if (lane == 0) {
        off[i] = v.off;
        len[i] = v.n == LC_TS_NO_KEY ? LC_TS_NO_KEY : v.n - v.dq;
    }
    if (v.n == LC_TS_NO_KEY)
        return;
    if (v.dq)
        lc_split_delim_ts_collapse(val + v.off, t.base + v.off, v.n, c.d.quote, ws[threadIdx.x >> 5], lane, 32);
    else
        split_json_ts_copy(val + v.off, t.base + v.off, v.n, lane);
}

// counters: u64 [10] += the LC_SDTS_COUNTERS verdicts (one atomic per warp and counter), then pieces whose record
// would reach 4 GiB
__global__ void __launch_bounds__(256)
    split_delim_ts_sls_size_kernel(LcSplitDelimSlsCfg c, LcSplitDelimTsCfg tc, DelimSlsTables t, TsRowTables ts,
                                   uint64_t n, uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                   unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bits = 0, big = 0;
    if (i < n) {
        const LcDelimSlsRow r = split_delim_sls_row(c, t, i);
        const uint32_t st = ts.status[i];
        const LcSplitRegexTsTime tm = lc_split_delim_ts_time(c, tc, st, ts.sec[i], ts.nsec[i]);
        LcSlsCount64 s{0};
        const uint32_t cnt = tm.keep ? lc_split_delim_sls_body(c, t.base, r, tm.time, tm.has_ns, tm.ns, s) : 0u;
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        bits = lc_split_delim_ts_verdict(c, r.status, st);
    }
#pragma unroll
    for (uint32_t k = 0; k < LC_SDTS_COUNTERS; ++k) {
        const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, (bits >> k) & 1u);
        if ((threadIdx.x & 31) == 0 && v)
            atomicAdd(counters + k, (unsigned long long)v);
    }
    big = __reduce_add_sync(0xFFFFFFFFu, big);
    if ((threadIdx.x & 31) == 0 && big)
        atomicAdd(counters + LC_SDTS_COUNTERS, (unsigned long long)big);
}

__global__ void __launch_bounds__(256)
    split_delim_ts_sls_emit_kernel(LcSplitDelimSlsCfg c, LcSplitDelimTsCfg tc, DelimSlsTables t, TsRowTables ts,
                                   uint64_t n, const uint64_t* __restrict__ rec_off,
                                   const uint32_t* __restrict__ body_size, uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased, discarded or without contents: no record
    const LcDelimSlsRow r = split_delim_sls_row(c, t, i);
    // lc_split_delim_ts_time's rule for a piece with a record, as selects on the kernel parameters (as in the split ->
    // JSON -> timestamp emit kernel, which a struct of the three kept live across the body made spill)
    const bool ok = ts.status[i] == LC_TS_ST_OK;
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_delim_sls_body(c, t.base, r, ok ? (uint32_t)ts.sec[i] : c.time, ok ? tc.enable_ns : c.has_ns,
                            ok ? ts.nsec[i] : c.ns, s);
}

void launch_split_delim_ts_tap(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc, const DelimSlsTables& t,
                               uint64_t n, uint8_t* d_val, uint32_t* d_off, uint32_t* d_len, cudaStream_t st) {
    if (n)
        split_delim_ts_tap_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, tc, t, n, d_val, d_off, d_len);
}

void launch_split_delim_ts_sls_sizes(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc,
                                     const DelimSlsTables& t, const TsRowTables& ts, uint64_t n,
                                     uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                     cudaStream_t st) {
    if (n)
        split_delim_ts_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_size,
                                                                                     d_body_size, d_counters);
}

void launch_split_delim_ts_sls_emit(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc,
                                    const DelimSlsTables& t, const TsRowTables& ts, uint64_t n,
                                    const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                    cudaStream_t st) {
    if (n)
        split_delim_ts_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, tc, t, ts, n, d_rec_off,
                                                                                          d_body_size, d_out);
}

// ---- f4, split -> Apsara chain (lc_exec.cuh: lc_split_apsara_sls_body, lc_split_apsara_verdict).  The size pass runs
// one thread per piece, the emit pass one warp per piece.  counters: u64 [6] += lc_apsara_parse's five, then pieces
// whose record would reach 4 GiB.
__device__ __forceinline__ LcSplitApsaraSlsRow split_apsara_sls_row(const SplitApsaraSlsTables& t, uint64_t i) {
    LcSplitApsaraSlsRow r;
    const uint64_t f = t.first[i];
    r.po = t.off[i];
    r.plen = t.len[i];
    r.status = t.status[i];
    r.sec = t.sec[i];
    r.nsec = t.nsec[i];
    r.micro = t.micro[i];
    r.e = t.ent + f;
    r.m = (r.status & 7u) == LC_AP_ST_OK ? (uint32_t)(t.first[i + 1] - f) : 0u;
    return r;
}

__global__ void __launch_bounds__(256)
    split_apsara_sls_size_kernel(LcSplitApsaraSlsCfg c, SplitApsaraSlsTables t, uint64_t n,
                                 uint32_t* __restrict__ rec_size, uint32_t* __restrict__ body_size,
                                 unsigned long long* __restrict__ counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bits = 0, big = 0;
    if (i < n) {
        const LcSplitApsaraSlsRow r = split_apsara_sls_row(t, i);
        LcSlsCount64 s{0};
        const uint32_t cnt = lc_split_apsara_sls_body(c, t.src, r, s);
        big = s.n + 16 > 0xFFFFFFFFull;
        const uint32_t body = cnt && !big ? (uint32_t)s.n : 0u;
        rec_size[i] = body ? 1 + lc_varint_size(body) + body : 0u;
        body_size[i] = body;
        bits = lc_split_apsara_verdict(c, r.status) | (big << LC_AP_SLS_COUNTERS);
    }
    for (uint32_t k = 0; k <= LC_AP_SLS_COUNTERS; ++k) {
        const uint32_t v = __reduce_add_sync(0xFFFFFFFFu, (bits >> k) & 1u);
        if ((threadIdx.x & 31) == 0 && v)
            atomicAdd(counters + k, (unsigned long long)v);
    }
}

__global__ void __launch_bounds__(256)
    split_apsara_sls_emit_kernel(LcSplitApsaraSlsCfg c, SplitApsaraSlsTables t, uint64_t n,
                                 const uint64_t* __restrict__ rec_off, const uint32_t* __restrict__ body_size,
                                 uint8_t* __restrict__ out) {
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n)
        return;
    const uint32_t body = body_size[i];
    if (!body)
        return; // erased: no record
    const LcSplitApsaraSlsRow r = split_apsara_sls_row(t, i);
    uint8_t h[6];
    h[0] = 0x0A;
    const uint32_t hn = 1 + lc_put_varint(h + 1, body);
    LcSlsWrite s{out + rec_off[i], 0u, hn + body, threadIdx.x & 31, 32};
    s.put(h, hn);
    lc_split_apsara_sls_body(c, t.src, r, s);
}

void launch_split_apsara_sls_sizes(const LcSplitApsaraSlsCfg& c, const SplitApsaraSlsTables& t, uint64_t n,
                                   uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                   cudaStream_t st) {
    if (n)
        split_apsara_sls_size_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_size, d_body_size,
                                                                                   d_counters);
}

void launch_split_apsara_sls_emit(const LcSplitApsaraSlsCfg& c, const SplitApsaraSlsTables& t, uint64_t n,
                                  const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                  cudaStream_t st) {
    if (n)
        split_apsara_sls_emit_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, st>>>(c, t, n, d_rec_off,
                                                                                        d_body_size, d_out);
}

} // namespace lck
