// lc_scan.cuh -- single-pass device-wide prefix scan with decoupled look-back, generic over an
// associative (not necessarily commutative) operator on a 62-bit payload.
//
// Every tile publishes a 64-bit descriptor {flag:2 | payload:62}; a tile first publishes its local
// AGGREGATE, then walks its predecessors (32 descriptors per warp and step) until it meets an
// INCLUSIVE prefix, and finally publishes its own inclusive prefix.  Flag and payload share one
// 8-byte word, so a plain 64-bit store/load is atomic and no fence is needed between them.
// Tiles take their index from an atomic ticket so that a tile can only wait on tiles that are
// already running (forward-progress guarantee independent of block scheduling order).
//
// The look-back serves plain 62-bit sums (output slots).  The other operators serve scans without
// look-back: OpCountMax reads the split's tile prefixes {count:30 | line_start:32}, and OpMlState
// is the multiline state machine -- a 2-state transition function plus the index of the line that
// opened the pending record, per incoming state.
#pragma once
#include <stdint.h>

namespace lcscan {

constexpr uint64_t kPayloadMask = (1ull << 62) - 1;
constexpr uint64_t kFlagAggregate = 1ull << 62;
constexpr uint64_t kFlagInclusive = 2ull << 62;

// ---- operators ---------------------------------------------------------------------------------
struct OpSum {
    static __device__ __forceinline__ uint64_t identity() { return 0; }
    static __device__ __forceinline__ uint64_t combine(uint64_t a, uint64_t b) { return (a + b) & kPayloadMask; }
};

// {count:30 | max:32}
struct OpCountMax {
    static __device__ __forceinline__ uint64_t identity() { return 0; }
    static __device__ __forceinline__ uint64_t make(uint32_t count, uint32_t mx) {
        return ((uint64_t)count << 32) | mx;
    }
    static __device__ __forceinline__ uint32_t count(uint64_t p) { return (uint32_t)(p >> 32); }
    static __device__ __forceinline__ uint32_t maxv(uint64_t p) { return (uint32_t)p; }
    static __device__ __forceinline__ uint64_t combine(uint64_t a, uint64_t b) {
        uint32_t c = (count(a) + count(b)) & 0x3FFFFFFFu;
        uint32_t m = max(maxv(a), maxv(b));
        return make(c, m);
    }
};

// Multiline state machine element.  Incoming state s in {0 = not partial, 1 = partial}.
//   bit 61: out state for s = 0      bit 60: out state for s = 1
//   bits 59..30: lb0 = (index+1) of the last line that opened a record inside the segment when s = 0 (0 = none)
//   bits 29..0 : lb1 = same for s = 1
struct OpMlState {
    static __device__ __forceinline__ uint64_t make(uint32_t f0, uint32_t f1, uint32_t lb0, uint32_t lb1) {
        return ((uint64_t)(f0 & 1) << 61) | ((uint64_t)(f1 & 1) << 60) | ((uint64_t)(lb0 & 0x3FFFFFFFu) << 30) |
               (uint64_t)(lb1 & 0x3FFFFFFFu);
    }
    static __device__ __forceinline__ uint32_t f(uint64_t p, uint32_t s) { return (uint32_t)(p >> (61 - s)) & 1u; }
    static __device__ __forceinline__ uint32_t lb(uint64_t p, uint32_t s) {
        return (uint32_t)(p >> (s ? 0 : 30)) & 0x3FFFFFFFu;
    }
    static __device__ __forceinline__ uint64_t identity() { return make(0, 1, 0, 0); }
    // a happens first, then b
    static __device__ __forceinline__ uint64_t combine(uint64_t a, uint64_t b) {
        uint32_t m0 = f(a, 0), m1 = f(a, 1);
        uint32_t lb0 = lb(b, m0) ? lb(b, m0) : lb(a, 0);
        uint32_t lb1 = lb(b, m1) ? lb(b, m1) : lb(a, 1);
        return make(f(b, m0), f(b, m1), lb0, lb1);
    }
};

__device__ __forceinline__ uint64_t shfl_up64(uint64_t v, int d) {
    uint32_t lo = __shfl_up_sync(0xFFFFFFFFu, (uint32_t)v, d);
    uint32_t hi = __shfl_up_sync(0xFFFFFFFFu, (uint32_t)(v >> 32), d);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl_down64(uint64_t v, int d) {
    uint32_t lo = __shfl_down_sync(0xFFFFFFFFu, (uint32_t)v, d);
    uint32_t hi = __shfl_down_sync(0xFFFFFFFFu, (uint32_t)(v >> 32), d);
    return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
    uint32_t lo = __shfl_sync(0xFFFFFFFFu, (uint32_t)v, src);
    uint32_t hi = __shfl_sync(0xFFFFFFFFu, (uint32_t)(v >> 32), src);
    return ((uint64_t)hi << 32) | lo;
}

// Block-wide exclusive scan in thread order.  smem: THREADS/32 + 1 words.  All threads must call.
template <class Op, int THREADS>
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t& block_total, uint64_t* smem) {
    constexpr int NW = THREADS / 32;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint64_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t t = shfl_up64(inc, d);
        if (lane >= d)
            inc = Op::combine(t, inc);
    }
    __syncthreads(); // protect smem reuse between consecutive calls
    if (lane == 31)
        smem[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint64_t w = lane < NW ? smem[lane] : Op::identity();
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t t = shfl_up64(w, d);
            if (lane >= d)
                w = Op::combine(t, w);
        }
        if (lane < NW)
            smem[lane] = w; // inclusive over warps
    }
    __syncthreads();
    uint64_t warp_prefix = wid ? smem[wid - 1] : Op::identity();
    block_total = smem[NW - 1];
    uint64_t excl = shfl_up64(inc, 1);
    if (lane == 0)
        excl = Op::identity();
    return Op::combine(warp_prefix, excl);
}

__device__ __forceinline__ uint64_t ld_desc(const volatile uint64_t* p) { return *p; }

// Block-cooperative look-back: ALL threads of the block call (uniform control flow); the first WARPS warps poll
// WARPS * 32 predecessors per round.  Why: a tile's walk ends at the nearest predecessor that already holds an
// INCLUSIVE prefix, and every predecessor that is itself still walking only offers its aggregate -- so the faster the
// tiles retire, the more descriptors a walk has to cross.  With one warp (32 descriptors per ~L2 round trip) the scan
// saturates near tile_bytes * 32 / round_trip; WARPS = 4 moves that ceiling 4x out.  Returns the exclusive prefix of
// `tile` to every thread.
// s_part: WARPS words, s_flag: WARPS words of shared memory.
template <class Op, int WARPS>
__device__ __forceinline__ uint64_t lookback_block(volatile uint64_t* desc, uint32_t tile, uint64_t aggregate,
                                                   uint64_t* s_part, uint32_t* s_flag) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (tile == 0) {
        if (threadIdx.x == 0)
            desc[0] = kFlagInclusive | (aggregate & kPayloadMask);
        return Op::identity();
    }
    if (threadIdx.x == 0)
        desc[tile] = kFlagAggregate | (aggregate & kPayloadMask);
    uint64_t prefix = Op::identity();
    int64_t base = (int64_t)tile - 1;
    for (;;) {
        if (wid < WARPS) {
            const int64_t idx = base - (wid * 32 + lane);
            uint64_t d;
            if (idx >= 0) {
                do {
                    d = ld_desc(desc + idx);
                } while ((d >> 62) == 0);
            } else {
                d = kFlagInclusive | Op::identity();
            }
            const unsigned incl = __ballot_sync(0xFFFFFFFFu, (d >> 62) == 2);
            const int stop = incl ? (__ffs(incl) - 1) : 31;
            uint64_t r = (lane <= stop) ? (d & kPayloadMask) : Op::identity();
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) { // ordered reduction: higher lanes are EARLIER tiles
                const uint64_t t = shfl_down64(r, s);
                if (lane + s < 32)
                    r = Op::combine(t, r);
            }
            if (lane == 0) {
                s_part[wid] = r;
                s_flag[wid] = incl != 0;
            }
        }
        __syncthreads();
        uint64_t r = Op::identity();
        bool found = false;
#pragma unroll
        for (int w = 0; w < WARPS; ++w)
            if (!found) {
                r = Op::combine(s_part[w], r); // warp w + 1 holds earlier tiles than warp w
                found = s_flag[w] != 0;
            }
        prefix = Op::combine(r, prefix);
        __syncthreads(); // s_part / s_flag are rewritten in the next round
        if (found)
            break;
        base -= WARPS * 32;
    }
    if (threadIdx.x == 0)
        desc[tile] = kFlagInclusive | (Op::combine(prefix, aggregate) & kPayloadMask);
    return prefix;
}

} // namespace lcscan
