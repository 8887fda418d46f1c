// lc_exec.cuh -- scalar interpretation of a compiled regex blob (lc_tables.h): the semantic core
// that the sm_90a kernels execute once per log line.  Written as __host__ __device__ so that the
// exact same statements can be exercised on the CPU by the test-only emulation library under
// tests/emul/ (which validates the COMPILER's tables against the oracle without a GPU).  The product
// library only ever calls these from device code, apart from the host-side configuration steps of the
// delimiter- and regex-fed SLS serialisers (lc_delim_sls_setup, lc_regex_sls_setup).
#pragma once
#include <stdint.h>
#include <string.h>
#include <time.h>

#include "lc_tables.h"

#if defined(__CUDACC__)
#define LC_HD __host__ __device__ __forceinline__
#else
#define LC_HD inline
#endif

#define LC_SLOT_UNSET 0xFFFFFFFFu

struct LcProgView {
    const LcRegexHeader* h;
    const uint8_t* byte_class;
    const uint8_t* class_pc;
    const uint64_t* actions;
    const uint16_t* pre_next;
    const uint8_t* pre_acc;
    const uint32_t* fwd;
    const uint32_t* fwd_eof;
    const uint16_t* rev_next;
};

LC_HD LcProgView lc_view(const void* blob) {
    const uint8_t* b = (const uint8_t*)blob;
    const LcRegexHeader* h = (const LcRegexHeader*)blob;
    LcProgView v;
    v.h = h;
    v.byte_class = b + h->off_byte_class;
    v.class_pc = b + h->off_class_pc;
    v.actions = (const uint64_t*)(b + h->off_actions);
    v.pre_next = (const uint16_t*)(b + h->off_pre_next);
    v.pre_acc = b + h->off_pre_acc;
    v.fwd = (const uint32_t*)(b + h->off_fwd);
    v.fwd_eof = (const uint32_t*)(b + h->off_fwd_eof);
    v.rev_next = (const uint16_t*)(b + h->off_rev_next);
    return v;
}

// regex_search(..., match_continuous) as a boolean (reference: core/common/StringTools.cpp:263-288).
LC_HD bool lc_prefix_match(const LcProgView& v, const uint8_t* s, uint32_t n) {
    const uint32_t nc = v.h->nclasses;
    uint32_t st = v.h->pre_start;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t e = v.pre_next[st * nc + v.byte_class[s[i]]];
        if (e == LC_PREFIX_ACCEPT)
            return true;
        if (e == LC_PREFIX_DEAD)
            return false;
        st = e;
    }
    return v.pre_acc[st] != 0;
}

LC_HD void lc_apply_action(const LcProgView& v, uint32_t act, uint32_t pos, uint32_t* slots) {
    uint64_t m = v.actions[act];
    while (m) {
#if defined(__CUDA_ARCH__)
        int s = __ffsll((long long)m) - 1;
#else
        int s = __builtin_ctzll(m);
#endif
        slots[s] = pos;
        m &= m - 1;
    }
}

// regex_match with captures, forward-only automaton (mode LC_MODE_FWD1).
// slots: 2*ngroups entries, pre-filled with LC_SLOT_UNSET by the caller.
LC_HD bool lc_full_match_fwd1(const LcProgView& v, const uint8_t* s, uint32_t n, uint32_t* slots) {
    const uint32_t cols = v.h->fwd_cols;
    const uint32_t npc = v.h->npc;
    uint32_t w = 0, pk = 0;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t c = v.byte_class[s[i]];
        uint32_t e = v.fwd[(w * npc + pk) * cols + c];
        if (e == LC_NONE_ENTRY)
            return false;
        uint32_t a = LC_ENTRY_ACT(e);
        if (a)
            lc_apply_action(v, a, i, slots);
        w = LC_ENTRY_NEXT(e);
        if (npc > 1)
            pk = v.class_pc[c];
    }
    uint32_t e = v.fwd_eof[w * npc + pk];
    if (e == LC_NONE_ENTRY)
        return false;
    uint32_t a = LC_ENTRY_ACT(e);
    if (a)
        lc_apply_action(v, a, n, slots);
    return true;
}

// Reverse labelling pass of the two-pass matcher: lab[i] = reverse-DFA state at position i (0..n).
// Returns false early when the state dies (no suffix can reach a full match).
template <class LabT>
LC_HD bool lc_rev_label(const LcProgView& v, const uint8_t* s, uint32_t n, LabT* lab) {
    const uint32_t nc = v.h->nclasses;
    uint32_t d = v.h->rev_start;
    lab[n] = (LabT)d;
    for (uint32_t i = n; i-- > 0;) {
        d = v.rev_next[d * nc + v.byte_class[s[i]]];
        if (d == LC_REV_DEAD)
            return false;
        lab[i] = (LabT)d;
    }
    return true;
}

// Guided forward walk: at every position take the highest-priority transition that stays viable.
template <class LabT>
LC_HD bool lc_fwd_walk(const LcProgView& v, const uint8_t* s, uint32_t n, const LabT* lab, uint32_t* slots) {
    const uint32_t cols = v.h->fwd_cols;
    const uint32_t npc = v.h->npc;
    uint32_t w = 0, pk = 0;
    for (uint32_t i = 0; i <= n; ++i) {
        uint32_t e = v.fwd[(w * npc + pk) * cols + (uint32_t)lab[i]];
        if (e == LC_NONE_ENTRY)
            return false; // only possible at i == 0 (no viable start)
        uint32_t a = LC_ENTRY_ACT(e);
        if (a)
            lc_apply_action(v, a, i, slots);
        w = LC_ENTRY_NEXT(e);
        if (npc > 1 && i < n)
            pk = v.class_pc[v.byte_class[s[i]]];
    }
    return true;
}

// Capture slots -> boost sub_match (offset, length); a group that did not participate reports
// first == second == end of input (SURVEY.md A.1), i.e. (n, 0).
LC_HD void lc_slots_to_cap(const uint32_t* slots, uint32_t g, uint32_t n, uint32_t* off, uint32_t* len) {
    uint32_t b = slots[2 * g], e = slots[2 * g + 1];
    if (b == LC_SLOT_UNSET || e == LC_SLOT_UNSET || e < b) {
        *off = n;
        *len = 0;
    } else {
        *off = b;
        *len = e - b;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Stride-2 two-pass matcher over the fast2 layout (lc_tables.h: LcFast2Header): reference (loop) formulation.
// The kernel's unrolled middle section is a specialisation of exactly these statements.
struct LcFast2View {
    const LcFast2Header* h;
    const uint8_t* cls;
    const uint8_t* t2; // byte addressed (u32 entries)
    const uint8_t* pid;
    const uint8_t* pair_l;
    const uint8_t* rev1;
    const uint32_t* f2;
    const uint32_t* fwd1;
    const uint64_t* masks;
};

LC_HD LcFast2View lc_fast2_view(const void* blob) {
    const uint8_t* b = (const uint8_t*)blob;
    const LcFast2Header* h = (const LcFast2Header*)blob;
    LcFast2View v;
    v.h = h;
    v.cls = b + h->off_cls;
    v.t2 = b + h->off_t2;
    v.pid = b + h->off_pid;
    v.pair_l = b + h->off_pair_l;
    v.rev1 = b + h->off_rev1;
    v.f2 = (const uint32_t*)(b + h->off_f2);
    v.fwd1 = (const uint32_t*)(b + h->off_fwd1);
    v.masks = (const uint64_t*)(b + h->off_masks);
    return v;
}

#define LC_SLOT16_UNSET 0xFFFFu

LC_HD void lc_fast2_apply_mask(const LcFast2View& v, uint32_t act, uint32_t pos, uint16_t* slots) {
    uint64_t m = v.masks[act];
    while (m) {
#if defined(__CUDA_ARCH__)
        int s = __ffsll((long long)m) - 1;
#else
        int s = __builtin_ctzll(m);
#endif
        slots[s] = (uint16_t)pos;
        m &= m - 1;
    }
}

// single forward step of walker w under label L at position pos; returns the next walker
LC_HD uint32_t lc_fast2_single(const LcFast2View& v, uint32_t w, uint32_t L, uint32_t pos, uint16_t* slots) {
    const uint32_t e = v.fwd1[w * v.h->nrev + L];
    const uint32_t a = LC_ENTRY_ACT(e);
    if (a)
        lc_fast2_apply_mask(v, a, pos, slots);
    const uint32_t nx = LC_ENTRY_NEXT(e);
    return nx == 0xFFFFu ? 0u : nx;
}

// slow path of a pair step whose first or second transition sets several slots
LC_HD void lc_fast2_pair_slow(const LcFast2View& v, uint32_t w, uint32_t P, uint32_t pos, uint16_t* slots) {
    const uint32_t La = v.pair_l[2 * P], Lb = v.pair_l[2 * P + 1];
    const uint32_t w1 = lc_fast2_single(v, w, La, pos, slots);
    (void)lc_fast2_single(v, w1, Lb, pos + 1, slots);
}

// s = first byte of the event; `mis` = virtual index of that byte (address & 15 on the device).
// lab[j] receives the pair id of positions (2j, 2j+1) in virtual indexing; needs (n + mis) / 2 + 1 bytes.
// slots: 2 * ngroups u16 entries preset to LC_SLOT16_UNSET.  n must be < 65535.
LC_HD bool lc_fast2_event(const LcFast2View& v, const uint8_t* s, uint32_t mis, uint32_t n, uint8_t* lab,
                          uint16_t* slots) {
    const uint32_t Q = n + mis;
    const uint32_t nrev = v.h->nrev, ncls = v.h->ncls, row_bytes = v.h->row_bytes;
    const uint32_t start = v.h->rev_start;
    // ---- reverse: labels of positions Q (== start) down to mis
    uint32_t d = start;
    uint32_t q = Q;
    if ((q & 1) && q > mis) { // byte q-1 is the first slot of the pair (q-1, q): second slot is the end position
        --q;
        d = v.rev1[d * ncls + v.cls[s[q - mis]]];
        if (!d)
            return false;
        lab[q / 2] = v.pid[d * nrev + start];
    }
    while (q >= mis + 2) { // full byte pair (q-2, q-1)
        q -= 2;
        const uint32_t addr = d * row_bytes + ((uint32_t)v.cls[s[q + 1 - mis]] * ncls + v.cls[s[q - mis]]) * 4;
        const uint32_t e = *(const uint32_t*)(v.t2 + addr);
        lab[q / 2] = (uint8_t)(e >> 16);
        d = (e & 0xFFFFu) / row_bytes;
        if (!d)
            return false;
    }
    if (q > mis) { // one byte left: it sits in the second slot of a pair whose first slot precedes the event
        --q;
        d = v.rev1[d * ncls + v.cls[s[q - mis]]];
        if (!d)
            return false;
    }
    // ---- forward; d == label of position mis
    if (v.fwd1[d] == LC_NONE_ENTRY) // START row
        return false;
    uint32_t w = 0;
    q = mis;
    if (q & 1) {
        w = lc_fast2_single(v, w, d, 0, slots);
        ++q;
    }
    const uint32_t pshift = v.h->pair_shift, f2row = v.h->f2_row;
    while (q + 1 <= Q) {
        const uint32_t P = lab[q / 2] >> pshift; // labels hold pair_id << pair_shift
        const uint32_t e = v.f2[w * f2row + P];
        const uint32_t sa = (e >> 8) & 0x7Fu, sb = (e >> 16) & 0x7Fu;
        if (e & LC_FAST2_ACT_MULTI) {
            lc_fast2_pair_slow(v, w, P, q - mis, slots);
        } else {
            if (sa)
                slots[(sa - 2) / 2] = (uint16_t)(q - mis);
            if (sb)
                slots[(sb - 2) / 2] = (uint16_t)(q + 1 - mis);
        }
        w = e & 0xFFu;
        q += 2;
    }
    if (q == Q)
        (void)lc_fast2_single(v, w, start, q - mis, slots);
    return true;
}

LC_HD void lc_slots16_to_cap(const uint16_t* slots, uint32_t g, uint32_t n, uint32_t* off, uint32_t* len) {
    uint32_t b = slots[2 * g], e = slots[2 * g + 1];
    if (b == LC_SLOT16_UNSET || e == LC_SLOT16_UNSET || e < b) {
        *off = n;
        *len = 0;
    } else {
        *off = b;
        *len = e - b;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Single-pass tagged DFA (lc_tables.h: LcTdfaHeader): reference (loop) formulation; the kernel's unrolled middle
// section is a specialisation of exactly these statements.
struct LcTdfaView {
    const LcTdfaHeader* h;
    const uint8_t* cls;
    const uint8_t* t2; // byte addressed (u32 entries)
    const uint32_t* t1;
    const uint32_t* eof;
    const uint16_t* ops;
    const uint32_t* skip;
};

LC_HD LcTdfaView lc_tdfa_view(const void* blob) {
    const uint8_t* b = (const uint8_t*)blob;
    const LcTdfaHeader* h = (const LcTdfaHeader*)blob;
    LcTdfaView v;
    v.h = h;
    v.cls = b + h->off_cls;
    v.t2 = b + h->off_t2;
    v.t1 = (const uint32_t*)(b + h->off_t1);
    v.eof = (const uint32_t*)(b + h->off_eof);
    v.ops = (const uint16_t*)(b + h->off_ops);
    v.skip = (const uint32_t*)(b + h->off_skip);
    return v;
}

// does the 16-byte chunk w[0..3] hold one of the exit bytes of skip word sk (LC_TDFA_SKIP set)?  Branch-free: both
// exit slots are always tested (a one-exit state repeats its byte in the second, lc_tables.h), a zero-exit state is
// masked at the end.
LC_HD bool lc_tdfa_chunk_has_exit(uint32_t sk, const uint32_t w[4]) {
#ifdef __CUDA_ARCH__
    const uint32_t e0 = __byte_perm(sk, 0, 0x0000), e1 = __byte_perm(sk, 0, 0x1111);
#else
    const uint32_t e0 = (sk & 0xFFu) * 0x01010101u, e1 = ((sk >> 8) & 0xFFu) * 0x01010101u;
#endif
    uint32_t hit = 0;
    for (int j = 0; j < 4; ++j) {
        const uint32_t x0 = w[j] ^ e0, x1 = w[j] ^ e1;
        hit = ((x0 - 0x01010101u) & ~x0) | hit;
        hit = ((x1 - 0x01010101u) & ~x1) | hit;
    }
    // (x - 0x01010101) & ~x & 0x80808080 is nonzero iff some byte of x is zero
    return (hit & 0x80808080u) != 0 && (sk & 0x30000u) != 0;
}

// RegT = uint16_t (events shorter than 65535 bytes: the shared-memory register files of the kernels) or uint32_t
// (the long-event kernel); "unset" is the all-ones value of RegT.
template <class RegT>
LC_HD void lc_tdfa_run_ops(const LcTdfaView& v, uint32_t list, uint32_t pos, RegT* regs) {
    const uint16_t* p = v.ops + list;
    const uint32_t cnt = p[0];
    for (uint32_t k = 1; k <= cnt; ++k) {
        const uint32_t op = p[k], dst = op >> 8, src = op & 0xFFu;
        regs[dst] = src == LC_TDFA_SRC_POS ? (RegT)pos : src == LC_TDFA_SRC_UNSET ? (RegT)~(RegT)0 : regs[src];
    }
}

// one byte from `state` at position pos; returns the next state (0 = dead)
template <class RegT>
LC_HD uint32_t lc_tdfa_single(const LcTdfaView& v, uint32_t state, uint32_t byte, uint32_t pos, RegT* regs) {
    const uint32_t e = v.t1[state * v.h->ncls + v.cls[byte]];
    if (e >> 16)
        lc_tdfa_run_ops(v, e >> 16, pos, regs);
    return e & 0xFFFFu;
}

// s = first byte of the event; `mis` = virtual index of that byte (address & 15 on the device; pairs are aligned
// on even virtual indices).  regs: h->nregs u16 entries, the first 2 * ngroups preset to LC_SLOT16_UNSET; on a
// match they hold the capture boundaries.  n must be < 65535 for RegT = uint16_t.
template <class RegT>
LC_HD bool lc_tdfa_event(const LcTdfaView& v, const uint8_t* s, uint32_t mis, uint32_t n, RegT* regs) {
    const uint32_t ncls = v.h->ncls, row_bytes = v.h->row_bytes;
    uint32_t st = v.h->start;
    uint32_t pos = 0;
    if ((mis & 1) && n) {
        st = lc_tdfa_single(v, st, s[0], 0, regs);
        pos = 1;
    }
    while (pos + 2 <= n) {
        // run skipping exactly as the kernels do it: at a 16-byte boundary of the line's aligned frame, with a whole
        // chunk of input left, a skippable state jumps over a chunk that holds none of its exit bytes
        if (((pos + mis) & 15u) == 0 && pos + 16 <= n && v.skip[st]) {
            uint32_t w[4];
            memcpy(w, s + pos, 16);
            if (!lc_tdfa_chunk_has_exit(v.skip[st], w)) {
                pos += 16;
                continue;
            }
        }
        const uint32_t c0 = v.cls[s[pos]], c1 = v.cls[s[pos + 1]];
        const uint32_t e = *(const uint32_t*)(v.t2 + st * row_bytes + (c0 * ncls + c1) * 4);
        if (e & LC_TDFA_SLOW) {
            const uint32_t s1 = lc_tdfa_single(v, st, s[pos], pos, regs);
            st = lc_tdfa_single(v, s1, s[pos + 1], pos + 1, regs);
        } else {
            const uint32_t sa = (e >> 16) & 0x7Fu, sb = (e >> 24) & 0x7Fu;
            if (sa)
                regs[(sa - 2) / 2] = (RegT)pos;
            if (sb)
                regs[(sb - 2) / 2] = (RegT)(pos + 1);
            st = (e & 0xFFFFu) / row_bytes;
        }
        pos += 2;
    }
    if (pos < n) {
        st = lc_tdfa_single(v, st, s[pos], pos, regs);
        ++pos;
    }
    const uint32_t fin = v.eof[st];
    if (fin == LC_NONE_ENTRY)
        return false;
    lc_tdfa_run_ops(v, fin, n, regs);
    return true;
}

// ------------------------------------------------------------------------------------------------------------
// Delimiter quote FSM (DelimiterModeFsmParser::ParseDelimiterLine, zero-copy variant,
// core/parser/DelimiterModeFsmParser.cpp:260-294) with run skipping: per 16-byte aligned chunk the separator and
// quote positions are found with byte-wise SIMD compares; only those "special" bytes go through the state
// machine, every run of ordinary bytes between them is one step (the ordinary-byte transition is idempotent:
// INITIAL -> DATA, QUOTE / DATA stay, DOUBLE_QUOTE is an error).  Exactly the per-byte machine otherwise.
//   v = line base; [begin, end) = trimmed range; push(field_start, field_len, doubled_quotes) receives every column.
// Reads the aligned 16-byte chunks that contain bytes of [begin, end) (like the kernel's other loaders).
LC_HD uint32_t lc_eq_mask16(const uint32_t w[4], uint32_t splat) {
    uint32_t m = 0;
    for (int k = 0; k < 4; ++k) {
        // bit 0 of every byte of w[k] that equals the splat byte: exact zero-byte test of x (no cross-byte borrows);
        // plain integer ops on both sides (the SIMD-video compare of the GPU is emulated and costs more)
        const uint32_t x = w[k] ^ splat;
        const uint32_t eq = (~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x) & 0x80808080u) >> 7;
        m |= (((eq * 0x01020408u) >> 24) & 0xFu) << (4 * k);
    }
    return m;
}

// Resumable form: the machine's registers + one call per 16-byte aligned chunk, so that a kernel can feed the chunks
// from a staging tile in shared memory stage by stage.  All positions are offsets from the line start `v`; q* are
// positions in the line's 16-byte aligned frame (frame index = offset + mis).
struct LcDelimRun {
    int state; // 0 INITIAL 1 QUOTE 2 DATA 3 DOUBLE_QUOTE
    int dq;
    int fs, fe;
    uint32_t cur; // next unprocessed frame position
};

LC_HD void lc_delim_start(LcDelimRun& r, int32_t begin, uint32_t mis) {
    r.state = 0;
    r.dq = 0;
    r.fs = r.fe = begin;
    r.cur = (uint32_t)begin + mis;
}

// chunk = the 16 bytes at frame positions [q0, q0 + 16), restricted to [qb, qe).  Returns false on a parse error.
//
// Only separators and quotes ("specials") step the machine; the run of ordinary bytes in front of each special is one
// step.  The step itself is table-driven and branch-free apart from the push: on the GPU the 32 lanes of a warp walk
// 32 different lines, and a formulation with one code path per (state, byte kind) made the warp execute most paths for
// every special with few active lanes on the hot instructions.  Entry (state * 2 + kind), kind 0 = separator,
// 1 = quote:  bits 0-1 next state | bits 2-3 fe += | bit 4 push the column first | bit 5 dq-- before the push |
// bit 6 error | bit 7 fs++ | bit 8 dq++.  After a push: dq = 0 and fs = the new fe.
//   INITIAL  sep: push, fe+1 -> INITIAL          quote: fs++ -> QUOTE
//   QUOTE    sep: fe+1 (part of the field)       quote: dq++, fe+1 -> DOUBLE_QUOTE
//   DATA     sep: push, fe+1 -> INITIAL          quote: error
//   DQUOTE   sep: dq--, push, fe+2 -> INITIAL    quote: fe+1 -> QUOTE (it was an escaped quote)
#define LC_DELIM_T(next, dfe, push, dqdec, err, fsinc, dqinc)                                                           \
    ((uint64_t)((next) | (dfe) << 2 | (push) << 4 | (dqdec) << 5 | (err) << 6 | (fsinc) << 7 | (dqinc) << 8))
template <class Push>
LC_HD bool lc_delim_chunk(LcDelimRun& r, const uint32_t w[4], uint32_t q0, uint32_t qb, uint32_t qe, uint32_t sep_splat,
                          uint32_t quote_splat, Push& push) {
    const uint64_t T_LO = LC_DELIM_T(0, 1, 1, 0, 0, 0, 0) | LC_DELIM_T(1, 0, 0, 0, 0, 1, 0) << 16 |
                          LC_DELIM_T(1, 1, 0, 0, 0, 0, 0) << 32 | LC_DELIM_T(3, 1, 0, 0, 0, 0, 1) << 48;
    const uint64_t T_HI = LC_DELIM_T(0, 1, 1, 0, 0, 0, 0) | LC_DELIM_T(2, 0, 0, 0, 1, 0, 0) << 16 |
                          LC_DELIM_T(0, 2, 1, 1, 0, 0, 0) << 32 | LC_DELIM_T(1, 1, 0, 0, 0, 0, 0) << 48;
    const uint32_t ms = lc_eq_mask16(w, sep_splat);
    uint32_t special = ms | lc_eq_mask16(w, quote_splat);
    if (q0 < qb)
        special &= ~((1u << (qb - q0)) - 1u);
    if (qe - q0 < 16)
        special &= (1u << (qe - q0)) - 1u;
    const uint32_t chunk_end = qe - q0 < 16 ? qe : q0 + 16;
    int state = r.state, dq = r.dq, fs = r.fs, fe = r.fe;
    uint32_t cur = r.cur, bad = 0;
    while (special) {
#if defined(__CUDA_ARCH__)
        const int b = __ffs((int)special) - 1;
#else
        const int b = __builtin_ctz(special);
#endif
        special &= special - 1;
        const uint32_t next = q0 + (uint32_t)b;
        const uint32_t gap = next - cur; // run of ordinary bytes in front of the special
        bad |= (gap != 0 && state == 3) ? 1u : 0u;
        state = (gap != 0 && state == 0) ? 2 : state;
        fe += (int)gap;
        cur = next + 1;
        const uint32_t idx = (uint32_t)state * 2u + (((ms >> b) & 1u) ^ 1u); // a byte equal to both counts as separator
        const uint32_t e = (uint32_t)((idx < 4 ? T_LO : T_HI) >> ((idx & 3u) * 16u)) & 0xFFFFu;
        if (e & 0x10u) {
            dq -= (int)((e >> 5) & 1u);
            if (!bad)
                push((uint32_t)fs, (uint32_t)(fe - fs), (uint32_t)dq);
            dq = 0;
        }
        fe += (int)((e >> 2) & 3u);
        dq += (int)((e >> 8) & 1u);
        bad |= (e >> 6) & 1u;
        fs = (e & 0x10u) ? fe : fs + (int)((e >> 7) & 1u);
        state = (int)(e & 3u);
    }
    {
        const uint32_t gap = chunk_end - cur; // ordinary bytes behind the last special of the chunk
        bad |= (gap != 0 && state == 3) ? 1u : 0u;
        state = (gap != 0 && state == 0) ? 2 : state;
        fe += (int)gap;
        cur = chunk_end;
    }
    r.state = state;
    r.dq = dq;
    r.fs = fs;
    r.fe = fe;
    r.cur = cur;
    return bad == 0;
}

// end of line: closes the last column; false = unterminated quote
template <class Push>
LC_HD bool lc_delim_finish(LcDelimRun& r, Push& push) {
    if (r.state == 3)
        r.dq--;
    if (r.state == 1)
        return false;
    push((uint32_t)r.fs, (uint32_t)(r.fe - r.fs), (uint32_t)r.dq);
    return true;
}

template <class Push>
LC_HD bool lc_delim_fsm(const uint8_t* v, int32_t begin, int32_t end, uint8_t sep, uint8_t quote, Push& push) {
    const uint32_t sep_splat = sep * 0x01010101u, quote_splat = quote * 0x01010101u;
    const uint32_t mis = (uint32_t)((uintptr_t)v & 15u);
    const uint8_t* abase = v - mis;
    const uint32_t qb = (uint32_t)begin + mis, qe = (uint32_t)end + mis; // range in the aligned frame
    LcDelimRun r;
    lc_delim_start(r, begin, mis);
    for (uint32_t qc = qb >> 4; end > begin && qc <= ((qe - 1) >> 4); ++qc) {
        uint32_t w[4];
#if defined(__CUDA_ARCH__)
        const uint4 vv = __ldg(reinterpret_cast<const uint4*>(abase) + qc);
        w[0] = vv.x, w[1] = vv.y, w[2] = vv.z, w[3] = vv.w;
#else
        memcpy(w, abase + (size_t)qc * 16, 16);
#endif
        if (!lc_delim_chunk(r, w, qc * 16, qb, qe, sep_splat, quote_splat, push))
            return false;
    }
    return lc_delim_finish(r, push);
}

// ---- bit-parallel form for well-formed records ---------------------------------------------------------------------
// The machine above steps once per separator / quote, and with 32 different lines in a warp the loop over the specials
// of a chunk runs as often as the busiest lane needs.  For a
// record in which every quote sits where the machine accepts one, the columns follow from three masks per chunk:
//   S = separators, Q = quotes, P = inclusive prefix-XOR of Q (with the carry of the chunks before): P is 1 from an
//   opening quote up to the byte before its closing quote, so the REAL separators are S & ~P, an opening quote is
//   Q & P and a closing quote is Q & ~P.
// Well-formed (exactly the paths of the machine that do not end in an error):
//   * an opening quote is the first byte of a column (record start or behind a real separator) or directly follows a
//     closing quote (the escaped quote "" inside a quoted column: DOUBLE_QUOTE -> QUOTE);
//   * a closing quote is followed by a real separator, by another quote, or by the end of the record
//     (DOUBLE_QUOTE + ordinary byte is the machine's error, DATA + quote likewise);
//   * the record does not end inside a quoted column.
// A column with quotes is then `"` content `"`: content = [first + 1, last - 1), doubled quotes = (quotes - 2) / 2.
// Anything else returns false and the caller runs lc_delim_fsm on the record (which also decides about errors).
struct LcDelimFast {
    uint32_t inq;        // 0 / all ones: inside a quoted section where the step starts
    uint32_t prev_rs;    // the byte before the step's first byte was a real separator (or the record starts here)
    uint32_t prev_close; // ... was a closing quote
    uint32_t nq;         // quotes of the open column so far
};

LC_HD void lc_delim_fast_start(LcDelimFast& r) {
    r.inq = 0;
    r.prev_rs = 1;
    r.prev_close = 0;
    r.nq = 0;
}

LC_HD uint32_t lc_popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}
LC_HD uint32_t lc_low_bits(uint32_t n) { return n >= 32 ? 0xFFFFFFFFu : (1u << n) - 1u; } // the n lowest bits

// One step over W (16 or 32) bytes of the record's 16-byte aligned frame, [q0, q0 + W).  ms / mq: masks of the bytes
// equal to the separator / quote.  mark(p, quotes) is called for every real separator: p = its offset from the line
// start, quotes = the number of quotes of the column it closes (a caller that wants columns derives them: the column
// starts behind the previous mark; with quotes it is `"` content `"`, doubled quotes = (quotes - 2) / 2).
template <int W, class Mark>
LC_HD bool lc_delim_fast_step(LcDelimFast& r, uint32_t ms, uint32_t mq, uint32_t q0, uint32_t qb, uint32_t qe,
                              uint32_t mis, Mark& mark) {
    const uint32_t b0 = q0 < qb ? qb - q0 : 0u;              // first byte of the step that belongs to the record
    const uint32_t nb = qe - q0 < (uint32_t)W ? qe - q0 : W; // bytes of the step in front of the record's end
    const uint32_t V = lc_low_bits(nb) & ~lc_low_bits(b0);   // (nb > b0: the caller only passes steps with bytes)
    const uint32_t S = ms & V, Q = mq & V;
    uint32_t P = Q;
    P ^= P << 1;
    P ^= P << 2;
    P ^= P << 4;
    P ^= P << 8;
    if (W > 16)
        P ^= P << 16;
    P = (P ^ r.inq) & lc_low_bits(W);
    const uint32_t RS = S & ~P, open = Q & P, close = Q & ~P;
    const uint32_t first = 1u << b0, last = 1u << (nb - 1);
    const bool ends = qe - q0 <= (uint32_t)W; // the record ends inside this step
    // opening quotes: behind a real separator / at the record start, or behind a closing quote
    uint32_t bad = open & ~(((RS | close) << 1) | ((r.prev_rs | r.prev_close) ? first : 0u));
    // closing quotes: in front of a real separator or a quote; the record's last byte may be one; the successor of
    // the step's last byte is checked with the next step (prev_close)
    bad |= close & (ends ? V : (V & ~last)) & ~(((RS | Q) >> 1) | (ends ? last : 0u));
    if (r.prev_close && !((RS | Q) & first))
        bad |= 1u;
    if (bad)
        return false;
    uint32_t m = RS, cb = b0, nq = r.nq;
    while (m) {
#if defined(__CUDA_ARCH__)
        const uint32_t b = (uint32_t)__ffs((int)m) - 1u;
#else
        const uint32_t b = (uint32_t)__builtin_ctz(m);
#endif
        m &= m - 1;
        mark((uint32_t)(q0 + b - mis), nq + lc_popc32(Q & lc_low_bits(b) & ~lc_low_bits(cb)));
        nq = 0;
        cb = b + 1;
    }
    r.nq = nq + lc_popc32(Q & ~lc_low_bits(cb));
    r.inq = (P & last) ? 0xFFFFFFFFu : 0u;
    r.prev_rs = (RS & last) ? 1u : 0u;
    r.prev_close = (close & last) ? 1u : 0u;
    return true;
}

// end of the record: the mark that closes the last column; false = the record ends inside a quoted column
template <class Mark>
LC_HD bool lc_delim_fast_finish(LcDelimFast& r, int32_t end, Mark& mark) {
    if (r.inq)
        return false;
    mark((uint32_t)end, r.nq);
    return true;
}

// column [start, p) that carries `quotes` quotes -> push(first byte, length, doubled quotes)
template <class Push>
LC_HD void lc_delim_fast_column(uint32_t start, uint32_t p, uint32_t quotes, Push& push) {
    if (quotes)
        push(start + 1, p - start - 2, (quotes - 2) >> 1);
    else
        push(start, p - start, 0u);
}

// whole record, 32 bytes per step as in the kernel (CPU-tier tests).  Returns false when the record is not well-formed
// in the sense above -- columns pushed so far are then to be discarded.
template <class Push>
LC_HD bool lc_delim_fast(const uint8_t* v, int32_t begin, int32_t end, uint8_t sep, uint8_t quote, Push& push) {
    const uint32_t sep_splat = sep * 0x01010101u, quote_splat = quote * 0x01010101u;
    const uint32_t mis = (uint32_t)((uintptr_t)v & 15u);
    const uint8_t* abase = v - mis;
    const uint32_t qb = (uint32_t)begin + mis, qe = (uint32_t)end + mis;
    LcDelimFast r;
    lc_delim_fast_start(r);
    uint32_t start = (uint32_t)begin;
    auto mark = [&](uint32_t p, uint32_t quotes) {
        lc_delim_fast_column(start, p, quotes, push);
        start = p + 1;
    };
    for (uint32_t qc = (qb >> 4) & ~1u; end > begin && qc <= ((qe - 1) >> 4); qc += 2) {
        uint32_t ms = 0, mq = 0;
        for (uint32_t h = 0; h < 2; ++h) {
            if ((qc + h) * 16 >= qe || (qc + h + 1) * 16 <= qb)
                continue; // no byte of the record in this half: not read
            uint32_t w[4];
#if defined(__CUDA_ARCH__)
            const uint4 vv = __ldg(reinterpret_cast<const uint4*>(abase) + qc + h);
            w[0] = vv.x, w[1] = vv.y, w[2] = vv.z, w[3] = vv.w;
#else
            memcpy(w, abase + (size_t)(qc + h) * 16, 16);
#endif
            ms |= lc_eq_mask16(w, sep_splat) << (16 * h);
            mq |= lc_eq_mask16(w, quote_splat) << (16 * h);
        }
        if (!lc_delim_fast_step<32>(r, ms, mq, qc * 16, qb, qe, mis, mark))
            return false;
    }
    return lc_delim_fast_finish(r, end, mark);
}

// ------------------------------------------------------------------------------------------------------------
// SLS wire format of LOG events (next row, SURVEY.md 8f rank 4): the hand-rolled protobuf writer of
// core/protobuf/sls/LogGroupSerializer.cpp:33-143,232-262 as size and emit functions over spans of the arena.
//   Log record = 0x0A varint(body) body ; body = 0x08 varint5(max(time, 2^28)) { 0x12 varint(pair) pair }* [0x25 ns:4]
//   pair       = 0x0A varint(klen) key 0x12 varint(vlen) value
LC_HD uint32_t lc_varint_size(uint32_t v) { return v < (1u << 7) ? 1 : v < (1u << 14) ? 2 : v < (1u << 21) ? 3 : v < (1u << 28) ? 4 : 5; }

LC_HD uint32_t lc_put_varint(uint8_t* p, uint32_t v) {
    uint32_t n = 0;
    while (v >= 0x80u) {
        p[n++] = (uint8_t)(v | 0x80u);
        v >>= 7;
    }
    p[n++] = (uint8_t)v;
    return n;
}

// GetLogContentSize (:232-237) without the tag + length prefix
LC_HD uint32_t lc_sls_pair_inner(uint32_t klen, uint32_t vlen) {
    return 1 + lc_varint_size(klen) + klen + 1 + lc_varint_size(vlen) + vlen;
}

// GetLogSize (:239-253): body = size inside the Logs field, return = with tag and length prefix; 0 entries -> 0, 0
LC_HD uint32_t lc_sls_log_size(const uint32_t* klen, const uint32_t* vlen, uint64_t e0, uint64_t e1, bool has_ns,
                               uint32_t* body_out) {
    if (e0 == e1) {
        *body_out = 0;
        return 0;
    }
    uint32_t body = 1 + 5 + (has_ns ? 1 + 4 : 0);
    for (uint64_t k = e0; k < e1; ++k) {
        const uint32_t in = lc_sls_pair_inner(klen[k], vlen[k]);
        body += 1 + lc_varint_size(in) + in;
    }
    *body_out = body;
    return 1 + lc_varint_size(body) + body;
}

// Writes one Log record at `out` (which has room for lc_sls_log_size bytes).  Called by all `nlanes` cooperating
// lanes with identical arguments except `lane`: lane 0 writes the tags / lengths, every lane copies its share of the
// key and value bytes.
LC_HD void lc_sls_emit_log(uint8_t* out, const uint8_t* base, uint32_t time, bool has_ns, uint32_t ns,
                           const uint32_t* koff, const uint32_t* klen, const uint32_t* voff, const uint32_t* vlen,
                           uint64_t e0, uint64_t e1, uint32_t body, uint32_t lane, uint32_t nlanes) {
    uint32_t at = 0;
    uint8_t hdr[16];
    uint32_t h = 0;
    hdr[h++] = 0x0A;
    h += lc_put_varint(hdr + h, body);
    hdr[h++] = 0x08;
    h += lc_put_varint(hdr + h, time < (1u << 28) ? (1u << 28) : time); // always 5 bytes
    if (lane == 0)
        for (uint32_t j = 0; j < h; ++j)
            out[j] = hdr[j];
    at = h;
    for (uint64_t k = e0; k < e1; ++k) {
        const uint32_t kl = klen[k], vl = vlen[k];
        h = 0;
        hdr[h++] = 0x12;
        h += lc_put_varint(hdr + h, lc_sls_pair_inner(kl, vl));
        hdr[h++] = 0x0A;
        h += lc_put_varint(hdr + h, kl);
        if (lane == 0)
            for (uint32_t j = 0; j < h; ++j)
                out[at + j] = hdr[j];
        at += h;
        for (uint32_t j = lane; j < kl; j += nlanes)
            out[at + j] = base[koff[k] + j];
        at += kl;
        h = 0;
        hdr[h++] = 0x12;
        h += lc_put_varint(hdr + h, vl);
        if (lane == 0)
            for (uint32_t j = 0; j < h; ++j)
                out[at + j] = hdr[j];
        at += h;
        for (uint32_t j = lane; j < vl; j += nlanes)
            out[at + j] = base[voff[k] + j];
        at += vl;
    }
    if (has_ns && lane == 0) {
        out[at] = 0x25;
        out[at + 1] = (uint8_t)ns;
        out[at + 2] = (uint8_t)(ns >> 8);
        out[at + 3] = (uint8_t)(ns >> 16);
        out[at + 4] = (uint8_t)(ns >> 24);
    }
}

// ------------------------------------------------------------------------------------------------------------
// f4, delimiter-fed: the Log record of one event that ProcessorParseDelimiterNative::Process leaves behind, written
// straight from the delimiter stage's result tables (ProcessorParseDelimiterNative.cpp:206-364; the host class's
// ProcessImpl in Processors.cpp).  The event is "flat" on entry: a LogEvent whose only content is SourceKey -> line.
//
// One body function serves both passes: with LcSlsCount it only counts the bytes, with LcSlsWrite it writes them.
// Sink interface: put(p, n) = tag / length bytes (lane 0 writes), copy(p, n) = key / value bytes (all lanes share),
// unquote(p, n, out_n, quote) = a quoted column with its doubled quotes collapsed (AddFieldWithUnQuote, :83-113).

// multi-byte separator (or quote == separator): ProcessorParseDelimiterNative::SplitString (:366-409), the statements
// of the delimiter kernel's split branch; push(field_start, field_len, 0) per column
template <class Push>
LC_HD void lc_delim_split(const uint8_t* v, int32_t begIdx, int32_t endIdx, const uint8_t* sep, uint32_t d,
                          uint32_t nkeys, bool extend, Push& push) {
    const uint32_t size = (uint32_t)(endIdx - begIdx);
    if (d > size) {
        push((uint32_t)begIdx, size, 0u);
        return;
    }
    uint32_t nf = 0, pos = (uint32_t)begIdx;
    const uint32_t top = (uint32_t)endIdx - d;
    bool done = false;
    while (pos <= top && !done) {
        uint32_t pos2 = (uint32_t)endIdx;
        for (uint32_t q = pos; q + d <= (uint32_t)endIdx; ++q) {
            bool eq = true;
            for (uint32_t t = 0; t < d; ++t)
                eq = eq && v[q + t] == sep[t];
            if (eq) {
                pos2 = q;
                break;
            }
        }
        push(pos, pos2 - pos, 0u);
        ++nf;
        if (pos2 == (uint32_t)endIdx) {
            done = true;
            break;
        }
        pos = pos2 + d;
        if (nf >= nkeys && !extend) {
            push(pos2, (uint32_t)endIdx - pos2, 0u);
            ++nf;
            done = true;
        }
    }
    if (!done && pos <= (uint32_t)endIdx)
        push(pos, (uint32_t)endIdx - pos, 0u);
}

#define LC_DELIM_SLS_EXTEND 0u
#define LC_DELIM_SLS_KEEP 1u
#define LC_DELIM_SLS_DISCARD 2u
#define LC_DELIM_SLS_NONE 0xFFFFFFFFu

// Configuration.  Every key string lives in `keys`: key k < nkeys is [key_at[k], key_at[k + 1]), then come SourceKey,
// RenamedSourceKey and "__raw_log__" (key_at has nkeys + 4 entries).
struct LcDelimSlsCfg {
    uint8_t sep[4];
    uint32_t sep_len;
    uint8_t quote;
    uint32_t use_quote;  // sep_len == 1 && quote != sep[0]: the quote state machine parsed the rows
    uint32_t mode;       // LC_DELIM_SLS_EXTEND / KEEP / DISCARD (OverflowedFieldsTreatment)
    uint32_t nkeys;
    uint32_t max_fields; // row width of the tables
    const uint8_t* keys;
    const uint32_t* key_at;
    uint32_t src_overwritten; // SourceKey is one of the keys (mSourceKeyOverwritten)
    uint32_t src_col;         // the column that replaces the source content in place, or NONE
    uint32_t ren_col;         // the column whose key is RenamedSourceKey (not a skipped "_"), or NONE
    uint32_t ren_xcol;        // N when RenamedSourceKey is "__column<N>__", or NONE
    uint32_t ren_is_src;      // RenamedSourceKey == SourceKey
    uint32_t ren_is_raw;      // RenamedSourceKey == "__raw_log__"
    uint32_t keep_fail, keep_succeed, copy_raw;
};

// One event: its line base[eo, eo + elen) and its row of the delimiter tables (f_off holds offsets into base).
struct LcDelimSlsRow {
    uint32_t eo, elen;
    uint32_t status, nf;
    const uint32_t* fo;
    const uint32_t* fl;
    const uint32_t* fd;
    uint32_t time;
    bool has_ns;
    uint32_t ns;
};

struct LcSlsCount {
    uint32_t n;
    LC_HD void put(const uint8_t*, uint32_t k) { n += k; }
    LC_HD void copy(const uint8_t*, uint32_t k) { n += k; }
    LC_HD void unquote(const uint8_t*, uint32_t, uint32_t out_n, uint8_t) { n += out_n; }
};

// writes at out[at...], never at or beyond `lim` (the record's size); nlanes lanes share the copies
struct LcSlsWrite {
    uint8_t* out;
    uint32_t at, lim, lane, nlanes;
    LC_HD void put(const uint8_t* p, uint32_t k) {
        if (lane == 0)
            for (uint32_t j = 0; j < k; ++j)
                if (at + j < lim)
                    out[at + j] = p[j];
        at += k;
    }
    LC_HD void copy(const uint8_t* p, uint32_t k) {
        for (uint32_t j = lane; j < k; j += nlanes)
            if (at + j < lim)
                out[at + j] = p[j];
        at += k;
    }
    LC_HD void unquote(const uint8_t* p, uint32_t k, uint32_t out_n, uint8_t q) {
        if (lane == 0) {
            uint32_t w = 0;
            for (uint32_t i = 0; i < k && w < out_n; ++i) {
                if (p[i] == q) {
                    if (i + 1 < k && p[i + 1] == q) {
                        if (at + w < lim)
                            out[at + w] = q;
                        ++w;
                        ++i;
                    }
                } else {
                    if (at + w < lim)
                        out[at + w] = p[i];
                    ++w;
                }
            }
        }
        at += out_n;
    }
};

// "__column" + decimal(idx) + "__" into k[20]; returns its length
LC_HD uint32_t lc_delim_column_key(uint32_t idx, uint8_t* k) {
    k[0] = '_', k[1] = '_', k[2] = 'c', k[3] = 'o', k[4] = 'l', k[5] = 'u', k[6] = 'm', k[7] = 'n';
    uint32_t digits = 1;
    for (uint32_t t = idx; t >= 10; t /= 10)
        ++digits;
    uint32_t t = idx;
    for (uint32_t d = digits; d-- > 0; t /= 10)
        k[8 + d] = (uint8_t)('0' + t % 10);
    k[8 + digits] = '_';
    k[9 + digits] = '_';
    return 10 + digits;
}

// tag + length prefixes of one Contents entry, its key bytes, then the value's tag + length (the value follows)
template <class S>
LC_HD void lc_sls_pair_open(S& s, const uint8_t* key, uint32_t kl, uint32_t vl) {
    uint8_t h[12];
    uint32_t n = 0;
    h[n++] = 0x12;
    n += lc_put_varint(h + n, lc_sls_pair_inner(kl, vl));
    h[n++] = 0x0A;
    n += lc_put_varint(h + n, kl);
    s.put(h, n);
    s.copy(key, kl);
    n = 0;
    h[n++] = 0x12;
    n += lc_put_varint(h + n, vl);
    s.put(h, n);
}

// Columns j0 <= j < j1 of the row in order: f(j, offset in base, raw length, doubled quotes).  From the table when it
// holds them; a row with more columns than the table holds is walked again from the start of its line with the same
// state machine (or split) that produced the table.  Only such rows, which are rare, pay for the walk.
template <class F>
LC_HD void lc_delim_sls_columns(const LcDelimSlsCfg& c, const uint8_t* base, const LcDelimSlsRow& r, uint32_t j0,
                                uint32_t j1, F& f) {
    if (r.nf <= c.max_fields || j1 <= c.max_fields) {
        for (uint32_t j = j0; j < j1 && j < r.nf; ++j)
            f(j, r.fo[j], r.fl[j], r.fd[j]);
        return;
    }
    const uint8_t* v = base + r.eo;
    int32_t end = (int32_t)r.elen, beg = 0; // the delimiter kernel's trim (:226-238)
    while (end > 0 && (v[end - 1] == ' ' || v[end - 1] == '\r'))
        --end;
    while (beg < end && v[beg] == ' ')
        ++beg;
    uint32_t j = 0;
    auto push = [&](uint32_t o, uint32_t l, uint32_t dq) {
        if (j >= j0 && j < j1)
            f(j, r.eo + o, l, dq);
        ++j;
    };
    if (c.use_quote)
        lc_delim_fsm(v, beg, end, c.sep[0], c.quote, push);
    else
        lc_delim_split(v, beg, end, c.sep, c.sep_len, c.nkeys, c.mode == LC_DELIM_SLS_EXTEND, push);
}

// The body of the event's Log record -- everything inside its Logs field: Time, Contents, Time_ns -- into sink s.
// Returns the number of contents; 0 = the event has none (erased, or LogEvent::Empty) and emits no record.
//   OK:      keys[j] -> column j in column order ("_" skipped and columns >= nkeys dropped in discard mode;
//            __column<j>__ in extend mode; keep mode joins columns nkeys.. into __column<nkeys>__); a column whose key
//            is SourceKey replaces the source content in place (first); then RenamedSourceKey -> line if
//            KeepingSourceWhenParseSucceed and that key is not present yet
//   failed:  RenamedSourceKey -> line [, __raw_log__ -> line] with KeepingSourceWhenParseFail, else erased
//   blank:   untouched: SourceKey -> the whole, untrimmed line
//
// x is the stage chained behind the delimiter (LcDelimNoChain: none).  Before each content the body asks x.own(kid) --
// kid = the key id of the content: key j < nkeys, or nkeys + 0 / 1 / 2 = SourceKey / RenamedSourceKey / "__raw_log__"
// -- and when x owns it, x.in_place(s) is written in its place instead; x.tail(s) runs after the contents, before
// Time_ns.  The count returned is the delimiter stage's, owned content included.
// A content the event holds before the delimiter runs, after SourceKey (the split's offset content), is x's slot: on
// every row that is not erased the body writes column x.slot_col() there when the row parsed and reaches it (that
// column is then not written in column order), else x.slot(s) -- which returns whether it wrote a content.
// x.slot_holds(kid): the slot's key is RenamedSourceKey / "__raw_log__" (kid), which AddLog(..., false) then skips.
struct LcDelimNoChain {
    LC_HD bool own(uint32_t) const { return false; }
    template <class S>
    LC_HD void in_place(S&) {}
    template <class S>
    LC_HD void tail(S&) {}
    LC_HD uint32_t slot_col() const { return LC_DELIM_SLS_NONE; }
    LC_HD bool slot_holds(uint32_t) const { return false; }
    template <class S>
    LC_HD bool slot(S&) {
        return false;
    }
};

template <class S, class X>
LC_HD uint32_t lc_delim_sls_body(const LcDelimSlsCfg& c, const uint8_t* base, const LcDelimSlsRow& r, S& s, X& x) {
    const uint32_t K_SRC = c.nkeys, K_REN = c.nkeys + 1, K_RAW = c.nkeys + 2;
    auto kp = [&](uint32_t k) { return c.keys + c.key_at[k]; };
    auto kl = [&](uint32_t k) { return c.key_at[k + 1] - c.key_at[k]; };
    const uint8_t* line = base + r.eo;
    {
        uint8_t h[6];
        h[0] = 0x08;
        const uint32_t n = 1 + lc_put_varint(h + 1, r.time < (1u << 28) ? (1u << 28) : r.time); // always 5 bytes
        s.put(h, n);
    }
    uint32_t cnt = 0;
    auto whole_line = [&](uint32_t k) {
        ++cnt;
        if (x.own(k)) {
            x.in_place(s);
            return;
        }
        lc_sls_pair_open(s, kp(k), kl(k), r.elen);
        s.copy(line, r.elen);
    };
    auto value = [&](uint32_t off, uint32_t len, uint32_t dq) {
        if (c.use_quote && dq)
            s.unquote(base + off, len, len - dq, c.quote);
        else
            s.copy(base + off, len);
    };
    const uint32_t xcol = x.slot_col();
    auto slot = [&](bool parsed) {
        if (parsed && xcol < r.nf) { // xcol < nkeys < max_fields: always in the table
            const uint32_t dq = c.use_quote ? r.fd[xcol] : 0u;
            lc_sls_pair_open(s, kp(xcol), kl(xcol), r.fl[xcol] - dq);
            value(r.fo[xcol], r.fl[xcol], dq);
            ++cnt;
        } else if (x.slot(s)) {
            ++cnt;
        }
    };
    if (r.status == 2) { // LC_DELIM_BLANK
        whole_line(K_SRC);
        slot(false);
    } else if (r.status != 0) { // LC_DELIM_PARSE_FAIL / LC_DELIM_COLUMNS
        if (c.keep_fail) {
            slot(false);
            if (!x.slot_holds(K_REN))
                whole_line(K_REN);
            if (c.copy_raw && !c.ren_is_raw && !x.slot_holds(K_RAW))
                whole_line(K_RAW);
        }
    } else {
        const uint32_t nf = r.nf, nk = c.nkeys;
        if (c.src_overwritten) {
            if (c.src_col != LC_DELIM_SLS_NONE && c.src_col < nf) {
                const uint32_t j = c.src_col; // < nkeys < max_fields: always in the table
                const uint32_t dq = c.use_quote ? r.fd[j] : 0u;
                if (x.own(K_SRC)) {
                    x.in_place(s);
                } else {
                    lc_sls_pair_open(s, kp(K_SRC), kl(K_SRC), r.fl[j] - dq);
                    value(r.fo[j], r.fl[j], dq);
                }
                ++cnt;
            } else {
                whole_line(K_SRC);
            }
        }
        slot(true);
        const bool joined = c.mode == LC_DELIM_SLS_KEEP && c.use_quote;
        const uint32_t jend = c.mode == LC_DELIM_SLS_EXTEND                 ? 0xFFFFFFFFu
                              : (c.mode == LC_DELIM_SLS_KEEP && !joined) ? nk + 1 // the split's remainder column
                                                                          : nk;
        auto col = [&](uint32_t j, uint32_t off, uint32_t len, uint32_t dq) {
            if (j == c.src_col || j == xcol)
                return;
            if (!c.use_quote)
                dq = 0;
            if (j < nk) {
                if (c.mode == LC_DELIM_SLS_DISCARD && kl(j) == 1 && kp(j)[0] == '_')
                    return;
                if (x.own(j)) {
                    x.in_place(s);
                    ++cnt;
                    return;
                }
                lc_sls_pair_open(s, kp(j), kl(j), len - dq);
            } else {
                uint8_t k[20];
                lc_sls_pair_open(s, k, lc_delim_column_key(j, k), len - dq);
            }
            value(off, len, dq);
            ++cnt;
        };
        lc_delim_sls_columns(c, base, r, 0u, jend, col);
        if (joined && nf > nk) { // sep[0] + unquoted column, for each column from nkeys on
            uint32_t vl = 0;
            auto measure = [&](uint32_t, uint32_t, uint32_t len, uint32_t dq) { vl += 1 + len - dq; };
            lc_delim_sls_columns(c, base, r, nk, 0xFFFFFFFFu, measure);
            uint8_t k[20];
            lc_sls_pair_open(s, k, lc_delim_column_key(nk, k), vl);
            auto piece = [&](uint32_t, uint32_t off, uint32_t len, uint32_t dq) {
                s.put(c.sep, 1);
                value(off, len, dq);
            };
            lc_delim_sls_columns(c, base, r, nk, 0xFFFFFFFFu, piece);
            ++cnt;
        }
        if (c.keep_succeed) { // AddLog(RenamedSourceKey, line, false): only when that key is not present
            const bool present =
                (c.ren_is_src && c.src_overwritten) || (c.ren_col != LC_DELIM_SLS_NONE && c.ren_col < nf) ||
                (c.ren_xcol != LC_DELIM_SLS_NONE && c.ren_xcol >= nk && c.ren_xcol < nf &&
                 (c.mode == LC_DELIM_SLS_EXTEND || (c.mode == LC_DELIM_SLS_KEEP && c.ren_xcol == nk))) ||
                x.slot_holds(K_REN);
            if (!present)
                whole_line(K_REN);
        }
    }
    x.tail(s);
    if (r.has_ns) {
        const uint8_t h[5] = {0x25, (uint8_t)r.ns, (uint8_t)(r.ns >> 8), (uint8_t)(r.ns >> 16), (uint8_t)(r.ns >> 24)};
        s.put(h, 5);
    }
    return cnt;
}

template <class S>
LC_HD uint32_t lc_delim_sls_body(const LcDelimSlsCfg& c, const uint8_t* base, const LcDelimSlsRow& r, S& s) {
    LcDelimNoChain x;
    return lc_delim_sls_body(c, base, r, s, x);
}

// "__column<digits>__": the form of the delimiter's generated overflow keys; *idx = the value when it is canonical
// decimal, else LC_DELIM_SLS_NONE
inline bool lc_delim_column_form(const char* s, uint32_t l, uint32_t* idx) {
    if (l < 11 || memcmp(s, "__column", 8) || s[l - 1] != '_' || s[l - 2] != '_')
        return false;
    uint64_t v = 0;
    for (uint32_t i = 8; i < l - 2; ++i) {
        if (s[i] < '0' || s[i] > '9')
            return false;
        v = v * 10 + (uint64_t)(s[i] - '0');
        if (v >= LC_DELIM_SLS_NONE)
            v = LC_DELIM_SLS_NONE;
    }
    const bool canonical = (l - 10 == 1 || s[8] != '0') && v < LC_DELIM_SLS_NONE;
    *idx = canonical ? (uint32_t)v : LC_DELIM_SLS_NONE;
    return true;
}


// Host side: checks a configuration of the delimiter-fed serialiser and fills `c` and the key strings.  key_bytes
// needs sum(key_lens) + source_len + renamed_len + 11 bytes, key_at nkeys + 4 entries; c.keys / c.key_at are left to
// the caller (device copies).  Returns nullptr, or why the configuration is refused: each refused case would need
// SetContentNoCopy's replace-in-place of an earlier content, which the flat-event model does not describe.
inline const char* lc_delim_sls_setup(const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                                      const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                      const char* source_key, uint32_t source_len, const char* renamed_key,
                                      uint32_t renamed_len, int keep_fail, int keep_succeed, int copy_raw,
                                      uint32_t max_fields, LcDelimSlsCfg* c, uint8_t* key_bytes, uint32_t* key_at) {
    if (sep_len < 1 || sep_len > 4 || (extend && discard))
        return "bad arguments (separator must be 1..4 bytes; extend and discard exclude each other)";
    if (max_fields < nkeys + 1)
        return "max_fields must be at least nkeys + 1";
    const bool disc = discard != 0, overflow_keys = !disc;
    auto eq = [](const char* a, uint32_t la, const char* b, uint32_t lb) { return la == lb && !memcmp(a, b, la); };
    auto is_skip = [&](uint32_t k) { return disc && key_lens[k] == 1 && keys[k][0] == '_'; };
    auto column_form = lc_delim_column_form;
    uint32_t dummy;
    for (uint32_t a = 0; a < nkeys; ++a) {
        if (overflow_keys && column_form(keys[a], key_lens[a], &dummy))
            return "a key of the form __column<digits>__ collides with the generated overflow keys";
        for (uint32_t b = a + 1; b < nkeys; ++b)
            if (eq(keys[a], key_lens[a], keys[b], key_lens[b]) && !is_skip(a))
                return "keys must be distinct (a repeated key overwrites its earlier content)";
    }
    if (overflow_keys && column_form(source_key, source_len, &dummy))
        return "a source key of the form __column<digits>__ collides with the generated overflow keys";
    memset(c, 0, sizeof *c);
    memcpy(c->sep, sep, sep_len);
    c->sep_len = sep_len;
    c->quote = quote;
    c->use_quote = sep_len == 1 && quote != sep[0];
    c->mode = extend ? LC_DELIM_SLS_EXTEND : (disc ? LC_DELIM_SLS_DISCARD : LC_DELIM_SLS_KEEP);
    c->nkeys = nkeys;
    c->max_fields = max_fields;
    c->src_col = c->ren_col = LC_DELIM_SLS_NONE;
    for (uint32_t k = 0; k < nkeys; ++k) {
        if (eq(keys[k], key_lens[k], source_key, source_len)) {
            c->src_overwritten = 1;
            if (!is_skip(k))
                c->src_col = k;
        }
        if (eq(keys[k], key_lens[k], renamed_key, renamed_len) && !is_skip(k))
            c->ren_col = k;
    }
    if (!overflow_keys || !column_form(renamed_key, renamed_len, &c->ren_xcol))
        c->ren_xcol = LC_DELIM_SLS_NONE;
    c->ren_is_src = eq(renamed_key, renamed_len, source_key, source_len);
    c->ren_is_raw = eq(renamed_key, renamed_len, "__raw_log__", 11);
    c->keep_fail = keep_fail != 0;
    c->keep_succeed = keep_succeed != 0;
    c->copy_raw = copy_raw != 0;
    uint32_t at = 0;
    auto add = [&](uint32_t k, const char* s, uint32_t l) {
        key_at[k] = at;
        if (l)
            memcpy(key_bytes + at, s, l);
        at += l;
    };
    for (uint32_t k = 0; k < nkeys; ++k)
        add(k, keys[k], key_lens[k]);
    add(nkeys, source_key, source_len);
    add(nkeys + 1, renamed_key, renamed_len);
    add(nkeys + 2, "__raw_log__", 11);
    key_at[nkeys + 3] = at;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------------------
// f4, regex-fed: the Log record of one event that ProcessorParseRegexNative::Process leaves behind, written straight
// from the regex stage's result tables (ProcessorParseRegexNative.cpp:132-168, CommonParserOptions.cpp:91-117; the
// host class's FinishEvent).  The event is flat on entry: a LogEvent whose only content is SourceKey -> line.  The
// contents Process leaves on such an event depend only on the configuration and the row's status, so the host compiles
// the configuration once into two content plans (lc_regex_sls_setup) and the device walks the plan of each row.  The
// same body function serves the counting and the writing pass (sinks LcSlsCount / LcSlsWrite above).

#define LC_REGEX_SLS_LINE 0xFFFFFFFFu   // value source of a plan entry: the whole line (else capture j)
#define LC_REGEX_SLS_DIGITS 0xFFFFFFFEu // ... the split piece's file offset in decimal (lc_regex_sls_plans only)

// Plan entry e = (plan[2e] = key id, plan[2e + 1] = capture index or LC_REGEX_SLS_LINE), key id k naming the key
// bytes [key_at[k], key_at[k + 1]) of `keys`.  Entries [0, n_ok) are the plan of parsed rows, [n_ok, n_ok + n_fail)
// the plan of failed rows, both in content order.
struct LcRegexSlsCfg {
    const uint32_t* plan;
    const uint32_t* key_at;
    const uint8_t* keys;
    uint32_t n_ok, n_fail;
    uint32_t pitch;      // row pitch of the capture tables
    uint32_t whole_line; // Regex "(.*)": no regex ran, every row is parsed (no status or capture tables)
    uint32_t ok_fits;    // the parsed plan's captures lie inside a row; otherwise no row can be LC_REGEX_OK
    uint32_t keep_fail;  // KeepingSourceWhenParseFail: failed rows are kept, else erased
    uint32_t ok_in_place; // entry 0 of the parsed plan is the source content, overwritten in place (not appended)
};

// One event: its line base[eo, eo + elen) and its row of the capture tables (offsets into base).
struct LcRegexSlsRow {
    uint32_t eo, elen;
    uint32_t status;
    const uint32_t* co;
    const uint32_t* cl;
    uint32_t time;
    bool has_ns;
    uint32_t ns;
};

// The row's verdict: 0 = parsed (LC_REGEX_OK, or whole-line mode), else its failure status.  A row that claims
// LC_REGEX_OK with more keys than the tables have columns cannot come from lc_regex_parse (which reports
// LC_REGEX_KEYS_MISMATCH for it) and is taken as one, so no capture beyond the row is read.
LC_HD uint32_t lc_regex_sls_verdict(const LcRegexSlsCfg& c, uint32_t status) {
    if (c.whole_line)
        return 0u;
    return status == 0u && !c.ok_fits ? 2u : status;
}

// The body of the event's Log record -- Time, the contents of its plan, Time_ns -- into sink s.  Returns the number of
// contents; 0 = the event has none (erased, or LogEvent::Empty) and emits no record.
template <class S>
LC_HD uint32_t lc_regex_sls_body(const LcRegexSlsCfg& c, const uint8_t* base, const LcRegexSlsRow& r, S& s) {
    {
        uint8_t h[6];
        h[0] = 0x08;
        const uint32_t n = 1 + lc_put_varint(h + 1, r.time < (1u << 28) ? (1u << 28) : r.time); // always 5 bytes
        s.put(h, n);
    }
    const bool ok = lc_regex_sls_verdict(c, r.status) == 0u;
    const uint32_t* e = c.plan + (ok ? 0u : 2u * c.n_ok);
    const uint32_t m = ok ? c.n_ok : c.n_fail;
    for (uint32_t k = 0; k < m; ++k) {
        const uint32_t kid = e[2 * k], src = e[2 * k + 1];
        const bool line = src == LC_REGEX_SLS_LINE;
        const uint32_t vo = line ? r.eo : r.co[src];
        const uint32_t vl = line ? r.elen : r.cl[src];
        lc_sls_pair_open(s, c.keys + c.key_at[kid], c.key_at[kid + 1] - c.key_at[kid], vl);
        s.copy(base + vo, vl);
    }
    if (r.has_ns) {
        const uint8_t h[5] = {0x25, (uint8_t)r.ns, (uint8_t)(r.ns >> 8), (uint8_t)(r.ns >> 16), (uint8_t)(r.ns >> 24)};
        s.put(h, 5);
    }
    return m;
}

// Host side: strings[0..count) back to back into key_bytes (sum of lens bytes) with key_at[count + 1] offsets.
inline void lc_sls_key_table(const char* const* strings, const uint32_t* lens, uint32_t count, uint8_t* key_bytes,
                             uint32_t* key_at) {
    uint32_t at = 0;
    for (uint32_t k = 0; k < count; ++k) {
        key_at[k] = at;
        if (lens[k])
            memcpy(key_bytes + at, strings[k], lens[k]);
        at += lens[k];
    }
    key_at[count] = at;
}

// Host side: compiles a configuration of the regex-fed serialiser into its two content plans.  The plans index the key
// table keys[0..nkeys), SourceKey, RenamedSourceKey, "__raw_log__", "content" (ids nkeys .. nkeys + 3; build it with
// lc_sls_key_table).  `plan` needs 3 * nkeys + 12 words (scratch included); c.plan / c.key_at / c.keys are left to the
// caller (device copies).  Returns nullptr, or why the arguments are refused.
//
// Each plan is LogEvent's content algebra (SetContentNoCopy / DelContent, LogEvent.cpp:50-106) run once on symbolic
// values -- "the line" and "capture j" -- starting from the flat event [SourceKey -> line]:
//   parsed: set(keys[j], capture j) for each key in order (whole-line mode: set(keys[0] or "content", line)); a
//           repeated key overwrites the earlier content in place, a key equal to SourceKey replaces the line in place;
//           then delete(SourceKey) unless it is one of the keys; then RenamedSourceKey -> line if
//           KeepingSourceWhenParseSucceed and that key is not live
//   failed: delete(SourceKey); with KeepingSourceWhenParseFail RenamedSourceKey -> line, then "__raw_log__" -> line
//           with CopingRawLog, each only if that key is not live; without it the event is empty and erased
// so the kernels need no branch per quirk.
//
// lc_regex_sls_plans is the same with an optional offset content (has_offset): the event starts as [SourceKey -> line,
// offset_key -> LC_REGEX_SLS_DIGITS] and the key table gains offset_key as id nkeys + 4; `plan` then needs
// 3 * nkeys + 24 words.  A regex key, RenamedSourceKey or "__raw_log__" equal to offset_key lands on that content like
// on any other, and a failed row without KeepingSourceWhenParseFail is erased although the offset content is left
// (ShouldEraseEvent, CommonParserOptions.cpp:107-110).  Without it the plans are lc_regex_sls_setup's.
inline const char* lc_regex_sls_plans(const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                      const char* source_key, uint32_t source_len, const char* renamed_key,
                                      uint32_t renamed_len, int has_offset, const char* offset_key,
                                      uint32_t offset_len, int keep_fail, int keep_succeed, int copy_raw,
                                      int whole_line, uint32_t pitch, LcRegexSlsCfg* c, uint32_t* plan) {
    if ((nkeys && (!keys || !key_lens)) || (source_len && !source_key) || (renamed_len && !renamed_key) ||
        (has_offset && offset_len && !offset_key) || !c || !plan)
        return "bad arguments";
    for (uint32_t k = 0; k < nkeys; ++k)
        if (key_lens[k] && !keys[k])
            return "bad arguments";
    const uint32_t K_SRC = nkeys, K_REN = nkeys + 1, K_RAW = nkeys + 2, K_CONTENT = nkeys + 3, K_OFF = nkeys + 4;
    auto str = [&](uint32_t k, uint32_t* l) -> const char* {
        if (k < nkeys) {
            *l = key_lens[k];
            return keys[k];
        }
        if (k == K_OFF) {
            *l = offset_len;
            return offset_key;
        }
        *l = k == K_SRC ? source_len : k == K_REN ? renamed_len : k == K_RAW ? 11u : 7u;
        return k == K_SRC ? source_key : k == K_REN ? renamed_key : k == K_RAW ? "__raw_log__" : "content";
    };
    auto same = [&](uint32_t a, uint32_t b) {
        uint32_t la, lb;
        const char* pa = str(a, &la);
        const char* pb = str(b, &lb);
        return la == lb && (la == 0 || !memcmp(pa, pb, la));
    };
    // symbolic contents: triples (key id, value source, live) from `list` on; LogEvent::FindContent looks from the back
    uint32_t* list = plan;
    uint32_t len = 0;
    auto find = [&](uint32_t key) -> int64_t {
        for (uint32_t i = len; i-- > 0;)
            if (list[3 * i + 2] && same(list[3 * i], key))
                return (int64_t)i;
        return -1;
    };
    auto set = [&](uint32_t key, uint32_t src) {
        const int64_t i = find(key);
        if (i >= 0) {
            list[3 * i] = key;
            list[3 * i + 1] = src;
        } else {
            list[3 * len] = key, list[3 * len + 1] = src, list[3 * len + 2] = 1u;
            ++len;
        }
    };
    auto add_absent = [&](uint32_t key) { // AddLog(key, line, false)
        if (find(key) < 0)
            set(key, LC_REGEX_SLS_LINE);
    };
    auto del = [&](uint32_t key) {
        const int64_t i = find(key);
        if (i >= 0)
            list[3 * i + 2] = 0u;
    };
    // drops the dead entries, packs the triples into (key id, source) pairs in place; returns the entry count
    auto finish = [&]() {
        uint32_t m = 0;
        for (uint32_t i = 0; i < len; ++i)
            if (list[3 * i + 2]) {
                const uint32_t k = list[3 * i], s = list[3 * i + 1];
                list[2 * m] = k, list[2 * m + 1] = s;
                ++m;
            }
        return m;
    };
    bool src_overwritten = false;
    for (uint32_t k = 0; k < nkeys; ++k)
        src_overwritten = src_overwritten || same(k, K_SRC);
    memset(c, 0, sizeof *c);
    // the event as the processor receives it
    auto start = [&]() {
        list[0] = K_SRC, list[1] = LC_REGEX_SLS_LINE, list[2] = 1u;
        list[3] = K_OFF, list[4] = LC_REGEX_SLS_DIGITS, list[5] = 1u;
        len = has_offset ? 2u : 1u;
    };
    // parsed rows
    start();
    if (whole_line)
        set(nkeys ? 0u : K_CONTENT, LC_REGEX_SLS_LINE);
    else
        for (uint32_t k = 0; k < nkeys; ++k)
            set(k, k);
    if (!src_overwritten)
        del(K_SRC);
    if (keep_succeed)
        add_absent(K_REN);
    c->ok_in_place = list[2];
    c->n_ok = finish();
    // failed rows (none in whole-line mode)
    list = plan + 2 * c->n_ok;
    len = 0;
    if (!whole_line) {
        start();
        del(K_SRC);
        if (keep_fail) {
            add_absent(K_REN);
            if (copy_raw)
                add_absent(K_RAW);
        }
    }
    c->n_fail = keep_fail ? finish() : 0u; // erased: empty, or only the offset content left
    c->pitch = pitch;
    c->whole_line = whole_line != 0;
    c->ok_fits = whole_line || nkeys <= pitch;
    c->keep_fail = keep_fail != 0;
    return nullptr;
}

inline const char* lc_regex_sls_setup(const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                      const char* source_key, uint32_t source_len, const char* renamed_key,
                                      uint32_t renamed_len, int keep_fail, int keep_succeed, int copy_raw,
                                      int whole_line, uint32_t pitch, LcRegexSlsCfg* c, uint32_t* plan) {
    return lc_regex_sls_plans(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len, 0, nullptr, 0u,
                              keep_fail, keep_succeed, copy_raw, whole_line, pitch, c, plan);
}

// ------------------------------------------------------------------------------------------------------------
// f4, delimiter -> regex chain: the Log record of one event that ProcessorParseDelimiterNative::Process followed by
// ProcessorParseRegexNative::Process (regex SourceKey = key k of the delimiter) leaves behind.  The event is flat on
// entry.  The regex stage reads key k's value, which after the delimiter stage is one of
//   column k, unquoted (AddFieldWithUnQuote)   delimiter OK and nfields > k
//   the whole line                             the line stayed under key k: a short row whose SourceKey is key k, a
//                                              short row with KeepingSourceWhenParseSucceed whose RenamedSourceKey is
//                                              key k, a kept failure whose RenamedSourceKey / "__raw_log__" is key k,
//                                              a blank row whose SourceKey is key k
//   absent                                     otherwise: out_key_not_found, the delimiter's record is left as it is
// The value table (lc_delim_regex_tap) is the regex stage's event table; a column with doubled quotes is copied,
// collapsed, into a side region of the line buffer, so captures stay offsets from one base.  The record is then the
// delimiter's body (lc_delim_sls_body) with key k's content deleted -- or overwritten in place by the capture of a
// regex key equal to k -- and the rest of the regex plan (lc_regex_sls_setup, SourceKey = k, "the line" = the value)
// appended.  lc_delim_regex_sls_link refuses the configurations in which a regex content could land on a delimiter
// content other than key k's, so no other in-place overwrite depends on the row.
#define LC_DR_ABSENT 0u
#define LC_DR_COLUMN 1u
#define LC_DR_LINE 2u

struct LcDelimRegexSlsCfg {
    LcDelimSlsCfg d;
    LcRegexSlsCfg x; // the regex plans, over "the line" = the value
    uint32_t col;    // k
    uint32_t src_is_k, ren_is_k, raw_is_k; // the delimiter's SourceKey / RenamedSourceKey / "__raw_log__" is key k
};

LC_HD uint32_t lc_delim_regex_value(const LcDelimRegexSlsCfg& c, uint32_t status, uint32_t nf) {
    if (status == 2) // LC_DELIM_BLANK: untouched
        return c.src_is_k ? LC_DR_LINE : LC_DR_ABSENT;
    if (status != 0) // failed: RenamedSourceKey [, "__raw_log__"] -> line when kept, else erased
        return c.d.keep_fail && (c.ren_is_k || (c.d.copy_raw && c.raw_is_k)) ? LC_DR_LINE : LC_DR_ABSENT;
    if (nf > c.col)
        return LC_DR_COLUMN;
    return c.src_is_k || (c.d.keep_succeed && c.ren_is_k) ? LC_DR_LINE : LC_DR_ABSENT;
}

// The value of one row: base[off, + len) (absent: the empty value at the line), and the bytes of its side copy (0: the
// value lies in the line as it is).
struct LcDrTap {
    uint32_t off, len, copy;
};
LC_HD LcDrTap lc_delim_regex_tap(const LcDelimRegexSlsCfg& c, const LcDelimSlsRow& r) {
    const uint32_t v = lc_delim_regex_value(c, r.status, r.nf);
    if (v == LC_DR_COLUMN) { // k < nkeys < max_fields: always in the table
        const uint32_t dq = c.d.use_quote ? r.fd[c.col] : 0u, n = r.fl[c.col] - dq;
        return {r.fo[c.col], n, dq ? n : 0u};
    }
    return {r.eo, v == LC_DR_LINE ? r.elen : 0u, 0u};
}

// writes the collapsed column of a tap with copy > 0 to dst[0, t.copy)
LC_HD void lc_delim_regex_copy(const LcDelimRegexSlsCfg& c, const uint8_t* base, const LcDelimSlsRow& r, uint8_t* dst,
                               uint32_t copy) {
    LcSlsWrite w{dst, 0u, copy, 0u, 1u};
    w.unquote(base + r.fo[c.col], r.fl[c.col], copy, c.d.quote);
}

// One event: its delimiter row, its value (the tap table) and the regex stage's row over that value.
struct LcDelimRegexSlsRow {
    LcDelimSlsRow d;
    uint32_t vo, vl;
    uint32_t status;
    const uint32_t* co;
    const uint32_t* cl;
};

// the regex stage as the delimiter body's chained stage (LcDelimNoChain's interface; no slot)
struct LcDelimRegexStage : LcDelimNoChain {
    const LcDelimRegexSlsCfg& c;
    const uint8_t* base;
    const LcDelimRegexSlsRow& r;
    bool present, ok;
    uint32_t m; // contents the regex stage wrote
    LC_HD bool own(uint32_t kid) const {
        const uint32_t nk = c.d.nkeys;
        return present && (kid == c.col || (kid == nk && c.src_is_k) || (kid == nk + 1 && c.ren_is_k) ||
                           (kid == nk + 2 && c.raw_is_k));
    }
    template <class S>
    LC_HD void entry(S& s, uint32_t e) { // entry e of the row's plan
        const uint32_t* p = c.x.plan + (ok ? 0u : 2u * c.x.n_ok) + 2 * e;
        const bool line = p[1] == LC_REGEX_SLS_LINE;
        const uint32_t vo = line ? r.vo : r.co[p[1]], vl = line ? r.vl : r.cl[p[1]];
        lc_sls_pair_open(s, c.x.keys + c.x.key_at[p[0]], c.x.key_at[p[0] + 1] - c.x.key_at[p[0]], vl);
        s.copy(base + vo, vl);
        ++m;
    }
    template <class S>
    LC_HD void in_place(S& s) {
        if (ok && c.x.ok_in_place)
            entry(s, 0);
    }
    template <class S>
    LC_HD void tail(S& s) {
        if (!present)
            return;
        const uint32_t n = ok ? c.x.n_ok : c.x.n_fail;
        for (uint32_t e = ok && c.x.ok_in_place ? 1u : 0u; e < n; ++e)
            entry(s, e);
    }
};

// The body of the event's Log record into sink s (LcSlsCount / LcSlsWrite).  Returns the number of contents; 0 = the
// event has none (erased by either stage, or LogEvent::Empty) and emits no record.  A regex failure without
// KeepingSourceWhenParseFail erases the event when key k's content was its only one (ShouldEraseEvent).
template <class S>
LC_HD uint32_t lc_delim_regex_sls_body(const LcDelimRegexSlsCfg& c, const uint8_t* base, const LcDelimRegexSlsRow& r,
                                       S& s) {
    LcDelimRegexStage x{{}, c, base, r, lc_delim_regex_value(c, r.d.status, r.d.nf) != LC_DR_ABSENT,
                        lc_regex_sls_verdict(c.x, r.status) == 0u, 0u};
    const uint32_t n = lc_delim_sls_body(c.d, base, r.d, s, x);
    return x.present ? n - 1 + x.m : n;
}

// The row's counter verdicts (0 / 1): the delimiter stage's successful, failed, discarded, blank, then the regex
// stage's successful, failed (LC_REGEX_NOMATCH), key-not-found, discarded.  cnt = lc_delim_regex_sls_body's result.
// An event the delimiter stage erased never reaches the regex stage.
struct LcDelimRegexVerdict {
    uint32_t ctr[8];
};
LC_HD LcDelimRegexVerdict lc_delim_regex_verdict(const LcDelimRegexSlsCfg& c, const LcDelimRegexSlsRow& r,
                                                 uint32_t cnt) {
    LcDelimRegexVerdict v;
    const uint32_t st = r.d.status;
    v.ctr[0] = st == 0;
    v.ctr[1] = st != 0 && st != 2;
    v.ctr[2] = v.ctr[1] && !c.d.keep_fail;
    v.ctr[3] = st == 2;
    const bool present = lc_delim_regex_value(c, st, r.d.nf) != LC_DR_ABSENT;
    const uint32_t rv = lc_regex_sls_verdict(c.x, r.status);
    v.ctr[5] = present && rv == 1u;
    v.ctr[6] = !present && !v.ctr[2];
    v.ctr[7] = present && rv != 0u && cnt == 0u;
    v.ctr[4] = present && !v.ctr[7];
    return v;
}

// Host side: the chain's own checks and fields, after lc_delim_sls_setup (d) and lc_regex_sls_setup (with the regex
// stage's arguments) accepted their halves.  Returns nullptr (c->col and the *_is_k flags set), or why the chain is
// refused: a regex SourceKey that is not one of the delimiter's keys, or a content the regex stage may write (a key,
// RenamedSourceKey, "__raw_log__") under a name the delimiter stage may leave besides key k -- that overwrite would
// depend on the row's shape.  Likewise ShouldEraseEvent's "_time_" + "_source_" rule on a regex failure.  okey (or
// nullptr): a content the event held before the delimiter stage ran (the split's offset content), which the delimiter
// stage leaves on every row it does not erase.
inline const char* lc_delim_regex_sls_link(const LcDelimSlsCfg& d, const char* const* dkeys, const uint32_t* dkey_lens,
                                           const char* dsrc, uint32_t dsrc_len, const char* dren, uint32_t dren_len,
                                           const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                                           const char* rsrc, uint32_t rsrc_len, const char* rren, uint32_t rren_len,
                                           int rkeep_fail, int rkeep_succeed, int rcopy_raw, int rwhole_line,
                                           LcDelimRegexSlsCfg* c, const char* okey = nullptr, uint32_t okey_len = 0) {
    auto eq = [](const char* a, uint32_t la, const char* b, uint32_t lb) {
        return la == lb && (la == 0 || !memcmp(a, b, la));
    };
    auto is_skip = [&](uint32_t j) {
        return d.mode == LC_DELIM_SLS_DISCARD && dkey_lens[j] == 1 && dkeys[j][0] == '_';
    };
    c->col = LC_DELIM_SLS_NONE;
    for (uint32_t j = 0; j < d.nkeys; ++j)
        if (!is_skip(j) && eq(dkeys[j], dkey_lens[j], rsrc, rsrc_len))
            c->col = j;
    if (c->col == LC_DELIM_SLS_NONE)
        return "the regex SourceKey is not one of the delimiter's keys";
    // a content the delimiter stage may leave under `name`, other than key k's
    auto left = [&](const char* name, uint32_t len) {
        uint32_t idx;
        if (eq(name, len, rsrc, rsrc_len))
            return false;
        for (uint32_t j = 0; j < d.nkeys; ++j)
            if (!is_skip(j) && eq(dkeys[j], dkey_lens[j], name, len))
                return true;
        return eq(name, len, dsrc, dsrc_len) || ((d.keep_fail || d.keep_succeed) && eq(name, len, dren, dren_len)) ||
               (d.keep_fail && d.copy_raw && eq(name, len, "__raw_log__", 11)) ||
               (d.mode != LC_DELIM_SLS_DISCARD && lc_delim_column_form(name, len, &idx)) ||
               (okey && eq(name, len, okey, okey_len));
    };
    bool clash = false;
    if (rwhole_line)
        clash = rnkeys ? left(rkeys[0], rkey_lens[0]) : left("content", 7);
    else
        for (uint32_t j = 0; j < rnkeys; ++j)
            clash = clash || left(rkeys[j], rkey_lens[j]);
    clash = clash || ((rkeep_fail || rkeep_succeed) && left(rren, rren_len)) ||
            (rkeep_fail && rcopy_raw && left("__raw_log__", 11));
    if (clash)
        return "a regex key, RenamedSourceKey or __raw_log__ names a content the delimiter stage may leave besides the "
               "regex SourceKey";
    if (!rkeep_fail && left("_time_", 6) && left("_source_", 8))
        return "_time_ and _source_ may both be left by the delimiter stage (the regex failure's erase rule)";
    c->src_is_k = d.src_col == c->col;
    c->ren_is_k = d.ren_col == c->col;
    c->raw_is_k = eq(dkeys[c->col], dkey_lens[c->col], "__raw_log__", 11);
    return nullptr;
}

// ------------------------------------------------------------------------------------------------------------
// f4, split-fed: the Log records of the events ProcessorSplitLogStringNative / ProcessorSplitMultilineLogStringNative
// cut from one source value (ProcessorSplitLogStringNative.cpp:131-161, ProcessorSplitMultilineLogStringNative.cpp:
// 311-340), written straight from the piece tables of lc_split_lines_dev / lc_multiline_split_dev.  Piece k =
// src[off[k], +len[k]) becomes one record:
//   LC_SPAN_PIECE:        key -> piece                        (RAW events: key = "content")
//   LC_SPAN_PIECE_OFFSET: key -> piece, okey -> decimal(src_pos + off[k])
//   LC_SPAN_OFFSET:       key -> decimal(src_pos + off[k])    (the offset key is the source key: replaced in place)
// A record's size is a closed function of len[k] and the digit count, so the size pass is elementwise.  The emit pass
// is tiled over the OUTPUT: lc_span_sls_tile writes exactly the bytes [t0, t1) of the wire output, whatever records,
// headers or varints the tile cuts through, so one long record never holds up a launch.  Value bytes (almost all the
// output) go out as 16-byte stores aligned on the output, loaded from the misaligned source by funnel-shifting two
// aligned 16-byte loads.
#define LC_SPAN_PIECE 0u
#define LC_SPAN_PIECE_OFFSET 1u
#define LC_SPAN_OFFSET 2u

struct LcSpanSlsCfg {
    const uint8_t* src;  // the source value (the buffer the split ran over)
    uint64_t src_len;
    const uint32_t* off; // piece tables
    const uint32_t* len;
    const uint8_t* key;  // device copies of the keys
    const uint8_t* okey;
    uint32_t klen, oklen;
    uint32_t mode; // LC_SPAN_*
    uint32_t time; // raised to 2^28 already
    uint32_t ns;
    uint32_t has_ns;
    uint64_t src_pos; // the source event's file offset
};

struct LcSpanRec {
    uint64_t num; // src_pos + off (modes with an offset)
    uint32_t nd;  // its decimal digits
    uint32_t va;  // value of the first pair: the piece or the digits
    uint32_t pa;  // inner size of the first pair, of the second (0 = none)
    uint32_t pb;
    uint32_t body;
    uint32_t vat;  // record position of the first pair's value
    uint32_t size; // bytes of the record
};

LC_HD uint32_t lc_dec_digits(uint64_t v) {
    uint32_t d = 1;
    uint64_t p = 10;
    while (d < 20 && v >= p) {
        ++d;
        p *= 10;
    }
    return d;
}

LC_HD LcSpanRec lc_span_sls_rec(const LcSpanSlsCfg& c, uint32_t off, uint32_t len) {
    LcSpanRec r;
    r.num = c.src_pos + off;
    r.nd = c.mode == LC_SPAN_PIECE ? 0u : lc_dec_digits(r.num);
    r.va = c.mode == LC_SPAN_OFFSET ? r.nd : len;
    r.pa = lc_sls_pair_inner(c.klen, r.va);
    r.pb = c.mode == LC_SPAN_PIECE_OFFSET ? lc_sls_pair_inner(c.oklen, r.nd) : 0u;
    r.body = 6 + 1 + lc_varint_size(r.pa) + r.pa + (r.pb ? 1 + lc_varint_size(r.pb) + r.pb : 0u) + (c.has_ns ? 5u : 0u);
    const uint32_t hb = 1 + lc_varint_size(r.body);
    r.vat = hb + 6 + 1 + lc_varint_size(r.pa) + 1 + lc_varint_size(c.klen) + c.klen + 1 + lc_varint_size(r.va);
    r.size = hb + r.body;
    return r;
}

// byte j of the n-byte varint of v
LC_HD uint8_t lc_varint_byte(uint32_t v, uint32_t j, uint32_t n) {
    return (uint8_t)(((v >> (7 * j)) & 0x7Fu) | (j + 1 < n ? 0x80u : 0u));
}

// digit j (from the left) of the nd-digit decimal v
LC_HD uint8_t lc_dec_digit(uint64_t v, uint32_t j, uint32_t nd) {
    for (uint32_t k = j + 1; k < nd; ++k)
        v /= 10;
    return (uint8_t)('0' + v % 10);
}

// byte p of a record outside the source bytes of its value: tags, lengths, keys, digits, the ns trailer
LC_HD uint8_t lc_span_sls_meta(const LcSpanSlsCfg& c, const LcSpanRec& r, uint32_t p) {
    uint32_t n;
    if (p == 0)
        return 0x0A;
    p -= 1;
    if (p < (n = lc_varint_size(r.body)))
        return lc_varint_byte(r.body, p, n);
    p -= n;
    if (p == 0)
        return 0x08;
    p -= 1;
    if (p < 5)
        return lc_varint_byte(c.time, p, 5);
    p -= 5;
    if (p == 0)
        return 0x12;
    p -= 1;
    if (p < (n = lc_varint_size(r.pa)))
        return lc_varint_byte(r.pa, p, n);
    p -= n;
    if (p == 0)
        return 0x0A;
    p -= 1;
    if (p < (n = lc_varint_size(c.klen)))
        return lc_varint_byte(c.klen, p, n);
    p -= n;
    if (p < c.klen)
        return c.key[p];
    p -= c.klen;
    if (p == 0)
        return 0x12;
    p -= 1;
    if (p < (n = lc_varint_size(r.va)))
        return lc_varint_byte(r.va, p, n);
    p -= n;
    if (c.mode == LC_SPAN_OFFSET) {
        if (p < r.nd)
            return lc_dec_digit(r.num, p, r.nd);
        p -= r.nd;
    } else {
        p -= r.va; // (the source bytes are not asked for)
    }
    if (r.pb) {
        if (p == 0)
            return 0x12;
        p -= 1;
        if (p < (n = lc_varint_size(r.pb)))
            return lc_varint_byte(r.pb, p, n);
        p -= n;
        if (p == 0)
            return 0x0A;
        p -= 1;
        if (p < (n = lc_varint_size(c.oklen)))
            return lc_varint_byte(c.oklen, p, n);
        p -= n;
        if (p < c.oklen)
            return c.okey[p];
        p -= c.oklen;
        if (p == 0)
            return 0x12;
        p -= 1;
        if (p == 0)
            return (uint8_t)r.nd; // < 128: one varint byte
        p -= 1;
        if (p < r.nd)
            return lc_dec_digit(r.num, p, r.nd);
        p -= r.nd;
    }
    if (p == 0)
        return 0x25;
    return (uint8_t)(c.ns >> (8 * (p - 1)));
}

struct LcU4 {
    uint32_t x, y, z, w;
};

LC_HD LcU4 lc_ld16(const uint8_t* p) { // p 16-byte aligned
#if defined(__CUDA_ARCH__)
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    return LcU4{v.x, v.y, v.z, v.w};
#else
    LcU4 v;
    memcpy(&v, p, 16);
    return v;
#endif
}

LC_HD void lc_st16(uint8_t* p, const LcU4& v) { // p 16-byte aligned
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<uint4*>(p) = make_uint4(v.x, v.y, v.z, v.w);
#else
    memcpy(p, &v, 16);
#endif
}

LC_HD uint32_t lc_funnel_r(uint32_t lo, uint32_t hi, uint32_t bits) { // bits in [0, 32)
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, bits);
#else
    return bits ? (lo >> bits) | (hi << (32 - bits)) : lo;
#endif
}

// the 16 bytes at s (any alignment).  [lo, hi) = the 16-byte aligned window of the source buffer: two aligned loads
// and a funnel shift when both lie inside it, byte loads at the buffer's ragged ends.
LC_HD LcU4 lc_ld16_any(const uint8_t* s, uintptr_t lo, uintptr_t hi) {
    const uintptr_t a = (uintptr_t)s & ~(uintptr_t)15;
    const uint32_t sh = (uint32_t)((uintptr_t)s & 15);
    if (sh == 0)
        return lc_ld16(s);
    if (a >= lo && a + 32 <= hi) {
        const LcU4 u = lc_ld16(reinterpret_cast<const uint8_t*>(a));
        const LcU4 v = lc_ld16(reinterpret_cast<const uint8_t*>(a + 16));
        const uint32_t q = sh >> 2, b = (sh & 3) * 8;
        // words q .. q+4 of u:v without a dynamically indexed array
        const uint32_t y0 = q == 0 ? u.x : q == 1 ? u.y : q == 2 ? u.z : u.w;
        const uint32_t y1 = q == 0 ? u.y : q == 1 ? u.z : q == 2 ? u.w : v.x;
        const uint32_t y2 = q == 0 ? u.z : q == 1 ? u.w : q == 2 ? v.x : v.y;
        const uint32_t y3 = q == 0 ? u.w : q == 1 ? v.x : q == 2 ? v.y : v.z;
        const uint32_t y4 = q == 0 ? v.x : q == 1 ? v.y : q == 2 ? v.z : v.w;
        return LcU4{lc_funnel_r(y0, y1, b), lc_funnel_r(y1, y2, b), lc_funnel_r(y2, y3, b), lc_funnel_r(y3, y4, b)};
    }
    uint32_t w[4];
    for (uint32_t i = 0; i < 4; ++i)
        w[i] = (uint32_t)s[4 * i] | ((uint32_t)s[4 * i + 1] << 8) | ((uint32_t)s[4 * i + 2] << 16) |
               ((uint32_t)s[4 * i + 3] << 24);
    return LcU4{w[0], w[1], w[2], w[3]};
}

// dst[0, n) = s[0, n): the bytes before dst's first and after its last 16-byte boundary one by one, the words between
// as aligned 16-byte stores; lanes share both
LC_HD void lc_copy_span(uint8_t* dst, const uint8_t* s, uint32_t n, uintptr_t lo, uintptr_t hi, uint32_t lane,
                        uint32_t nlanes) {
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > n)
        head = n;
    const uint32_t nw = (n - head) >> 4, tail = head + nw * 16;
    for (uint32_t j = lane; j < head + (n - tail); j += nlanes) {
        const uint32_t k = j < head ? j : tail + (j - head);
        dst[k] = s[k];
    }
    for (uint32_t w = lane; w < nw; w += nlanes)
        lc_st16(dst + head + 16 * w, lc_ld16_any(s + head + 16 * w, lo, hi));
}

// the record holding output byte t: the last k with rec_off[k] <= t (rec_off[0] == 0, t < total)
LC_HD uint64_t lc_span_sls_find(const uint64_t* rec_off, uint64_t n, uint64_t t) {
    uint64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (rec_off[mid] <= t)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}

// Writes exactly the bytes [t0, t1) of the wire output (records back to back, record k at rec_off[k]), starting at
// record r = lc_span_sls_find(rec_off, n, t0).  Called by `nlanes` cooperating lanes with identical arguments except
// `lane`.
LC_HD void lc_span_sls_tile(const LcSpanSlsCfg& c, const uint64_t* rec_off, uint64_t n, uint64_t r, uint64_t t0,
                            uint64_t t1, uint8_t* out, uint32_t lane, uint32_t nlanes) {
    const uintptr_t lo = ((uintptr_t)c.src + 15) & ~(uintptr_t)15;
    const uintptr_t hi = ((uintptr_t)c.src + c.src_len) & ~(uintptr_t)15;
    for (; r < n && rec_off[r] < t1; ++r) {
        const uint64_t b = rec_off[r];
        const uint32_t off = c.off[r];
        const LcSpanRec R = lc_span_sls_rec(c, off, c.len[r]);
        const uint32_t p0 = t0 > b ? (uint32_t)(t0 - b) : 0u;
        const uint32_t p1 = t1 - b < R.size ? (uint32_t)(t1 - b) : R.size;
        // the source bytes of the value: [vs, ve) of the record (none when the value is the offset)
        const uint32_t vs = R.vat, ve = c.mode == LC_SPAN_OFFSET ? R.vat : R.vat + R.va;
        uint8_t* o = out + b;
        for (uint32_t p = p0 + lane; p < (p1 < vs ? p1 : vs); p += nlanes)
            o[p] = lc_span_sls_meta(c, R, p);
        for (uint32_t p = (p0 > ve ? p0 : ve) + lane; p < p1; p += nlanes)
            o[p] = lc_span_sls_meta(c, R, p);
        const uint32_t a = p0 > vs ? p0 : vs, z = p1 < ve ? p1 : ve;
        if (a < z)
            lc_copy_span(o + a, c.src + off + (a - vs), z - a, lo, hi, lane, nlanes);
    }
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> regex chain: the Log record of piece k that ProcessorSplitLogStringNative /
// ProcessorSplitMultilineLogStringNative followed by ProcessorParseRegexNative (same SourceKey) leave behind, written
// straight from the piece tables of the splitter and the regex tables of lc_regex_parse_dev over those pieces.  The
// piece enters the regex stage as [SourceKey -> piece] or, with log.file.offset metadata, [SourceKey -> piece,
// offset_key -> decimal(src_pos + off[k])]; lc_regex_sls_plans compiles the configuration into the content plans over
// "the piece", "capture j" and "the piece's offset digits", so the rows need no branch per quirk.
struct LcSplitRegexSlsCfg {
    LcRegexSlsCfg x;  // the plans (lc_regex_sls_plans), key table keys..., SourceKey, RenamedSourceKey, "__raw_log__",
                      // "content", offset_key
    uint64_t src_pos; // the source event's file offset
    uint32_t time;    // the source event's time, as the split events inherit it
    uint32_t has_ns, ns;
};

// One piece: src[po, + plen) and its row of the regex tables (offsets into src).
struct LcSplitRegexSlsRow {
    uint32_t po, plen;
    uint32_t status;
    const uint32_t* co;
    const uint32_t* cl;
};

// the nd decimal digits of v into sink s: counting sinks count them, a writing sink's lanes write one digit each
template <class S>
LC_HD void lc_sls_digits(S& s, uint64_t, uint32_t nd) {
    s.put(nullptr, nd);
}
LC_HD void lc_sls_digits(LcSlsWrite& s, uint64_t v, uint32_t nd) {
    for (uint32_t j = s.lane; j < nd; j += s.nlanes)
        if (s.at + j < s.lim)
            s.out[s.at + j] = lc_dec_digit(v, j, nd);
    s.at += nd;
}

// The body of the piece's Log record -- Time, the contents of its plan, Time_ns -- into sink s (LcSlsCount /
// LcSlsWrite / LcSlsCount64), with the record's own time and ns (has_ns = 0: no Time_ns).  Returns the number of
// contents; 0 = erased or empty, no record.
template <class S>
LC_HD uint32_t lc_split_regex_sls_body(const LcSplitRegexSlsCfg& c, const uint8_t* src, const LcSplitRegexSlsRow& r,
                                       uint32_t time, uint32_t has_ns, uint32_t ns, S& s) {
    {
        uint8_t h[6];
        h[0] = 0x08;
        const uint32_t n = 1 + lc_put_varint(h + 1, time < (1u << 28) ? (1u << 28) : time); // always 5 bytes
        s.put(h, n);
    }
    const bool ok = lc_regex_sls_verdict(c.x, r.status) == 0u;
    const uint32_t* e = c.x.plan + (ok ? 0u : 2u * c.x.n_ok);
    const uint32_t m = ok ? c.x.n_ok : c.x.n_fail;
    const uint64_t pos = c.src_pos + r.po;
    const uint32_t nd = lc_dec_digits(pos);
    for (uint32_t k = 0; k < m; ++k) {
        const uint32_t kid = e[2 * k], vs = e[2 * k + 1];
        const uint8_t* key = c.x.keys + c.x.key_at[kid];
        const uint32_t kl = c.x.key_at[kid + 1] - c.x.key_at[kid];
        const bool digits = vs == LC_REGEX_SLS_DIGITS, line = vs == LC_REGEX_SLS_LINE;
        const uint32_t vl = digits ? nd : line ? r.plen : r.cl[vs];
        lc_sls_pair_open(s, key, kl, vl);
        if (digits)
            lc_sls_digits(s, pos, nd);
        else
            s.copy(src + (line ? r.po : r.co[vs]), vl);
    }
    if (has_ns) {
        const uint8_t h[5] = {0x25, (uint8_t)ns, (uint8_t)(ns >> 8), (uint8_t)(ns >> 16), (uint8_t)(ns >> 24)};
        s.put(h, 5);
    }
    return m;
}

// ... with the source event's time and ns, as every split piece inherits them
template <class S>
LC_HD uint32_t lc_split_regex_sls_body(const LcSplitRegexSlsCfg& c, const uint8_t* src, const LcSplitRegexSlsRow& r,
                                       S& s) {
    return lc_split_regex_sls_body(c, src, r, c.time, c.has_ns, c.ns, s);
}

// counting sink of the size pass in 64 bits: a body of 2^32 bytes or more is refused instead of wrapping
struct LcSlsCount64 {
    uint64_t n;
    LC_HD void put(const uint8_t*, uint32_t k) { n += k; }
    LC_HD void copy(const uint8_t*, uint32_t k) { n += k; }
    LC_HD void unquote(const uint8_t*, uint32_t, uint32_t out_n, uint8_t) { n += out_n; }
};

// The piece's counter verdicts (0 / 1): ProcessorParseRegexNative's out_successful (every piece not erased),
// out_failed (LC_REGEX_NOMATCH only) and discarded.  A split event always holds SourceKey, so no key-not-found.
struct LcSplitRegexVerdict {
    uint32_t ok, failed, erased;
};
LC_HD LcSplitRegexVerdict lc_split_regex_verdict(const LcSplitRegexSlsCfg& c, uint32_t status) {
    const uint32_t v = lc_regex_sls_verdict(c.x, status);
    const uint32_t kept = v == 0u || c.x.keep_fail;
    return {kept, v == 1u ? 1u : 0u, kept ? 0u : 1u};
}

// Host side: the configuration of the chain.  offset_key == nullptr: no log.file.offset metadata.  `plan` needs
// 3 * nkeys + 24 words.  Returns nullptr, or why the chain is refused: lc_regex_sls_setup's refusals, and an offset
// key equal to SourceKey (the split would replace the piece by its digits, and the regex would parse those).
inline const char* lc_split_regex_sls_setup(const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                            const char* source_key, uint32_t source_len, const char* renamed_key,
                                            uint32_t renamed_len, const char* offset_key, uint32_t offset_len,
                                            int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                                            uint32_t pitch, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                            LcSplitRegexSlsCfg* c, uint32_t* plan) {
    if (!c)
        return "bad arguments";
    if (offset_key && offset_len == source_len && (offset_len == 0 || (source_key && !memcmp(offset_key, source_key,
                                                                                               offset_len))))
        return "the offset key equals SourceKey";
    memset(c, 0, sizeof *c);
    const char* why = lc_regex_sls_plans(keys, key_lens, nkeys, source_key, source_len, renamed_key, renamed_len,
                                         offset_key != nullptr, offset_key, offset_len, keep_fail, keep_succeed,
                                         copy_raw, whole_line, pitch, &c->x, plan);
    if (why)
        return why;
    c->src_pos = src_pos;
    c->time = time;
    c->has_ns = time_ns != 0xFFFFFFFFu;
    c->ns = c->has_ns ? time_ns : 0u;
    return nullptr;
}

// Host side: the key table the plans of lc_split_regex_sls_setup name, key id k = strings[k] / lens[k]: the regex keys,
// then SourceKey, RenamedSourceKey, "__raw_log__", "content" and the offset key (empty when there is none).  strings
// and lens take nkeys + LC_SPLIT_REGEX_SLS_NSTR entries.  The C-ABI stages this table on the device, and every host
// check of a stage behind the chain (lc_filter_sls_setup, lc_split_regex_ts_setup) resolves its keys against it.
#define LC_SPLIT_REGEX_SLS_NSTR 5
inline void lc_split_regex_sls_strings(const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                       const char* source_key, uint32_t source_len, const char* renamed_key,
                                       uint32_t renamed_len, const char* offset_key, uint32_t offset_len,
                                       const char** strings, uint32_t* lens) {
    for (uint32_t k = 0; k < nkeys; ++k) {
        strings[k] = keys[k];
        lens[k] = key_lens[k];
    }
    const char* const s[LC_SPLIT_REGEX_SLS_NSTR] = {source_key, renamed_key, "__raw_log__", "content", offset_key};
    const uint32_t l[LC_SPLIT_REGEX_SLS_NSTR] = {source_len, renamed_len, 11u, 7u, offset_key ? offset_len : 0u};
    for (uint32_t k = 0; k < LC_SPLIT_REGEX_SLS_NSTR; ++k) {
        strings[nkeys + k] = s[k];
        lens[nkeys + k] = l[k];
    }
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> delimiter chain: the Log record of piece k that ProcessorSplitLogStringNative /
// ProcessorSplitMultilineLogStringNative followed by ProcessorParseDelimiterNative (same SourceKey) leave behind,
// written straight from the piece tables of the splitter and the delimiter tables of lc_delim_parse_dev over those
// pieces.  The piece enters the delimiter stage as [SourceKey -> piece] or, with log.file.offset metadata,
// [SourceKey -> piece, offset_key -> decimal(src_pos + off[k])].  The record is the delimiter's body
// (lc_delim_sls_body) with the offset content as its chained stage's slot: SetContentNoCopy replaces in place, so the
// contents come out as SourceKey's, the offset slot (the column keyed offset_key when the row parsed and reaches it,
// else the digits), the other columns in column order, then RenamedSourceKey / "__raw_log__" unless one of them is the
// offset key.  A blank row is left untouched; a failed row without KeepingSourceWhenParseFail keeps only the offset
// content and is erased (ShouldEraseEvent), so the rows erased and the four counters are those of the delimiter stage
// alone.
struct LcSplitDelimSlsCfg {
    LcDelimSlsCfg d;     // the delimiter stage (lc_delim_sls_setup)
    const uint8_t* okey; // device copy of the offset key
    uint32_t oklen;
    uint32_t has_offset;
    uint32_t off_col;          // the column keyed offset_key (not a skipped "_"), or NONE
    uint32_t ren_is_off;       // RenamedSourceKey == offset_key
    uint32_t raw_is_off;       // "__raw_log__" == offset_key
    uint64_t src_pos;          // the source event's file offset
    uint32_t time;             // the source event's time, as the split events inherit it
    uint32_t has_ns, ns;
};

// the offset content as the delimiter body's chained stage (LcDelimNoChain's interface)
struct LcSplitDelimStage : LcDelimNoChain {
    const LcSplitDelimSlsCfg& c;
    uint64_t pos; // src_pos + the piece's offset
    LC_HD uint32_t slot_col() const { return c.off_col; }
    LC_HD bool slot_holds(uint32_t kid) const {
        return (kid == c.d.nkeys + 1 && c.ren_is_off) || (kid == c.d.nkeys + 2 && c.raw_is_off);
    }
    template <class S>
    LC_HD bool slot(S& s) {
        if (!c.has_offset)
            return false;
        const uint32_t nd = lc_dec_digits(pos);
        lc_sls_pair_open(s, c.okey, c.oklen, nd);
        lc_sls_digits(s, pos, nd);
        return true;
    }
};

// The body of the piece's Log record into sink s (LcSlsCount64 / LcSlsWrite); r = the piece (eo, elen: its offset and
// length in src) and its row of the delimiter tables, with the source event's time and ns.  Returns the number of
// contents; 0 = erased, no record.
template <class S>
LC_HD uint32_t lc_split_delim_sls_body(const LcSplitDelimSlsCfg& c, const uint8_t* src, const LcDelimSlsRow& r,
                                       S& s) {
    LcSplitDelimStage x{{}, c, c.src_pos + r.eo};
    return lc_delim_sls_body(c.d, src, r, s, x);
}

// ... with the record's own time and ns (has_ns = 0: no Time_ns).  It hands the body a copy of the row with that
// time rather than the other way round: forwarding the row's own time through this overload changes the instruction
// schedule of the split -> delimiter emit kernel.
template <class S>
LC_HD uint32_t lc_split_delim_sls_body(const LcSplitDelimSlsCfg& c, const uint8_t* src, const LcDelimSlsRow& r,
                                       uint32_t time, uint32_t has_ns, uint32_t ns, S& s) {
    LcDelimSlsRow q = r;
    q.time = time;
    q.has_ns = has_ns != 0;
    q.ns = ns;
    return lc_split_delim_sls_body(c, src, q, s);
}

// The row's counter verdicts (0 / 1), as lc_delim_parse_sls counts them: successful, failed, discarded, blank.
struct LcDelimSlsVerdict {
    uint32_t ok, failed, erased, blank;
};
LC_HD LcDelimSlsVerdict lc_delim_sls_verdict(const LcDelimSlsCfg& c, uint32_t status) {
    const uint32_t ok = status == 0, blank = status == 2, failed = !ok && !blank;
    return {ok, failed, failed && !c.keep_fail ? 1u : 0u, blank};
}

// Host side: the chain's own checks and fields, after lc_delim_sls_setup accepted the delimiter stage (d, with the
// same keys, SourceKey and RenamedSourceKey).  offset_key == nullptr: no log.file.offset metadata.  Returns nullptr, or
// why the chain is refused: an offset key equal to SourceKey (the split would replace the piece by its digits, and the
// delimiter would parse those), or -- unless overflow columns are discarded -- an offset key of the form
// __column<digits>__, which a generated overflow key could overwrite on some rows and not on others.
inline const char* lc_split_delim_sls_link(const LcDelimSlsCfg& d, const char* const* keys, const uint32_t* key_lens,
                                           const char* source_key, uint32_t source_len, const char* renamed_key,
                                           uint32_t renamed_len, const char* offset_key, uint32_t offset_len,
                                           uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                           LcSplitDelimSlsCfg* c) {
    auto eq = [](const char* a, uint32_t la, const char* b, uint32_t lb) {
        return la == lb && (la == 0 || !memcmp(a, b, la));
    };
    memset(c, 0, sizeof *c);
    c->d = d;
    c->off_col = LC_DELIM_SLS_NONE;
    if (offset_key) {
        uint32_t idx;
        if (eq(offset_key, offset_len, source_key, source_len))
            return "the offset key equals SourceKey";
        if (d.mode != LC_DELIM_SLS_DISCARD && lc_delim_column_form(offset_key, offset_len, &idx))
            return "an offset key of the form __column<digits>__ collides with the generated overflow keys";
        c->has_offset = 1;
        c->oklen = offset_len;
        for (uint32_t k = 0; k < d.nkeys; ++k)
            if (eq(keys[k], key_lens[k], offset_key, offset_len) &&
                !(d.mode == LC_DELIM_SLS_DISCARD && key_lens[k] == 1 && keys[k][0] == '_'))
                c->off_col = k;
        c->ren_is_off = eq(renamed_key, renamed_len, offset_key, offset_len);
        c->raw_is_off = eq("__raw_log__", 11, offset_key, offset_len);
    }
    c->src_pos = src_pos;
    c->time = time;
    c->has_ns = time_ns != 0xFFFFFFFFu;
    c->ns = c->has_ns ? time_ns : 0u;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> delimiter -> regex chain: the Log record of piece k that a splitter, ProcessorParseDelimiterNative (the
// splitter's SourceKey) and ProcessorParseRegexNative (SourceKey = key k of the delimiter) leave behind, written
// straight from the piece tables, the delimiter tables over the pieces, the value table of the tap over those
// (lc_delim_regex_tap, unchanged: the piece tables are its event table) and the regex tables over the values.
//   - The piece enters as [SourceKey -> piece, offset_key -> decimal(src_pos + off[k])], or without the offset content
//     when there is no log.file.offset metadata.
//   - The delimiter stage runs as in the split -> delimiter chain: the offset slot follows SourceKey's content and holds
//     the column keyed offset_key when the row parsed and reaches it, else the digits; a blank piece is left
//     untouched; a failed piece without KeepingSourceWhenParseFail is erased.
//   - The regex stage runs as in the delimiter -> regex chain: it reads key k's value by lc_delim_regex_value's rule,
//     deletes key k's content in place (or overwrites it with a regex key equal to k) and appends the rest of its plan
//     after the delimiter's contents.
//   - ShouldEraseEvent (CommonParserOptions.cpp:99-117): a regex failure without the regex stage's
//     KeepingSourceWhenParseFail erases the event when nothing is left, or when the offset content is all that is left.
// lc_split_delim_regex_sls_link refuses an offset key equal to key k (on a row too short to reach column k the slot
// would hold the digits under key k, and the regex would read them), and any regex content named like the offset key.
struct LcSplitDelimRegexSlsCfg {
    LcDelimRegexSlsCfg r; // the delimiter and regex stages (the tap's configuration)
    LcSplitDelimSlsCfg s; // the offset content and the source event's time (s.d == r.d)
};

// both chained stages at once: the regex stage's own / in_place / tail and the split stage's slot
struct LcSplitDelimRegexStage : LcDelimRegexStage {
    LcSplitDelimStage o;
    LC_HD uint32_t slot_col() const { return o.slot_col(); }
    LC_HD bool slot_holds(uint32_t kid) const { return o.slot_holds(kid); }
    template <class S>
    LC_HD bool slot(S& s) {
        return o.slot(s);
    }
};

// The body of the piece's Log record into sink s (LcSlsCount64 / LcSlsWrite); r.d = the piece and its delimiter row
// (with the source event's time and ns), the rest its value and regex row.  Returns the number of contents; 0 = erased.
template <class S>
LC_HD uint32_t lc_split_delim_regex_sls_body(const LcSplitDelimRegexSlsCfg& c, const uint8_t* src,
                                             const LcDelimRegexSlsRow& r, S& s) {
    LcSplitDelimRegexStage x{{{}, c.r, src, r, lc_delim_regex_value(c.r, r.d.status, r.d.nf) != LC_DR_ABSENT,
                              lc_regex_sls_verdict(c.r.x, r.status) == 0u, 0u},
                             {{}, c.s, c.s.src_pos + r.d.eo}};
    const uint32_t n = lc_delim_sls_body(c.r.d, src, r.d, s, x);
    if (!x.present)
        return n;
    // A present value means the delimiter stage kept the row, so the slot holds the offset content whenever there is
    // one; a failed regex stage without KeepingSourceWhenParseFail appends nothing.
    const uint32_t left = n - 1 + x.m;
    return left == 1 && c.s.has_offset && !x.ok && !c.r.x.keep_fail ? 0u : left;
}

// The piece's counter verdicts: lc_delim_regex_verdict's 8, with cnt = lc_split_delim_regex_sls_body's result.
LC_HD LcDelimRegexVerdict lc_split_delim_regex_verdict(const LcSplitDelimRegexSlsCfg& c, const LcDelimRegexSlsRow& r,
                                                       uint32_t cnt) {
    return lc_delim_regex_verdict(c.r, r, cnt);
}

// Host side: the chain's checks and fields, after lc_delim_sls_setup (c->r.d) and lc_regex_sls_setup (c->r.x, SourceKey
// = rsrc) accepted their halves: lc_split_delim_sls_link, then an offset key equal to the regex SourceKey is refused,
// then lc_delim_regex_sls_link with the offset content as one more content the delimiter stage leaves besides key k
// (which also puts the offset key under its "_time_" / "_source_" rule).  Returns nullptr, or why the chain is refused.
inline const char* lc_split_delim_regex_sls_link(const char* const* dkeys, const uint32_t* dkey_lens,
                                                 const char* dsrc, uint32_t dsrc_len, const char* dren,
                                                 uint32_t dren_len, const char* const* rkeys,
                                                 const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsrc,
                                                 uint32_t rsrc_len, const char* rren, uint32_t rren_len,
                                                 int rkeep_fail, int rkeep_succeed, int rcopy_raw, int rwhole_line,
                                                 const char* offset_key, uint32_t offset_len, uint64_t src_pos,
                                                 uint32_t time, uint32_t time_ns, LcSplitDelimRegexSlsCfg* c) {
    const char* why = lc_split_delim_sls_link(c->r.d, dkeys, dkey_lens, dsrc, dsrc_len, dren, dren_len, offset_key,
                                              offset_len, src_pos, time, time_ns, &c->s);
    if (why)
        return why;
    if (offset_key && offset_len == rsrc_len && (rsrc_len == 0 || !memcmp(offset_key, rsrc, rsrc_len)))
        return "the offset key equals the regex SourceKey";
    return lc_delim_regex_sls_link(c->r.d, dkeys, dkey_lens, dsrc, dsrc_len, dren, dren_len, rkeys, rkey_lens, rnkeys,
                                   rsrc, rsrc_len, rren, rren_len, rkeep_fail, rkeep_succeed, rcopy_raw, rwhole_line,
                                   &c->r, offset_key, offset_len);
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> regex -> filter chain: ProcessorFilterNative (ProcessorFilterNative.cpp:83-117,459-486) behind the
// split -> regex chain.  The filter sees the event the regex stage left behind, so a leaf's key resolves once, on the
// host, through that stage's two content plans to a value source per verdict (parsed / failed): capture j, the piece
// (LC_REGEX_SLS_LINE), the piece's offset digits (LC_REGEX_SLS_DIGITS) or absent.  A leaf is regex_match of that
// value, false when the key is absent; the leaves combine through a postfix program of not / and / or.  In RULE and
// EXPRESSION mode (nprog > 0) an event without contents is removed whatever the leaves say; BYPASS (nprog == 0) keeps
// every event.  The regex stage's counters are not moved: it counted every piece before the filter ran.

#define LC_FILTER_SLS_LEAVES 32        // leaves per filter (lc_b200.h: LC_FILTER_MAX_LEAVES)
#define LC_FILTER_SLS_PROG 128         // program entries per filter (lc_b200.h: LC_FILTER_MAX_PROG)
#define LC_FILTER_SLS_ABSENT 0xFFFFFFFDu // value source of a leaf: its key is not in the event
#define LC_FILTER_SLS_NOT 0xFFFFFFFDu  // program opcodes (lc_b200.h: LC_FILTER_NOT / _AND / _OR)
#define LC_FILTER_SLS_AND 0xFFFFFFFEu
#define LC_FILTER_SLS_OR 0xFFFFFFFFu
#define LC_FILTER_SLS_DIGIT_PITCH 20u  // bytes per row of the digit scratch: the longest decimal u64

struct LcFilterSlsCfg {
    uint32_t nleaves;
    uint32_t nprog;                        // 0: BYPASS mode, every event is kept
    uint32_t src[LC_FILTER_SLS_LEAVES][2]; // value source of leaf l in a parsed [0] / failed [1] row
    uint32_t empty[2];                     // the parsed / failed event has no contents
    uint32_t any_digits;                   // some leaf reads the offset digits
    uint8_t prog[LC_FILTER_SLS_PROG];      // leaf index, or 253 / 254 / 255 = not / and / or
};

// Host side: where `key` (key[0, len)) is in the event the regex stage leaves behind, per verdict: src[0] in a parsed
// event, src[1] in a failed one.  Each is capture j, LC_REGEX_SLS_LINE, LC_REGEX_SLS_DIGITS or LC_FILTER_SLS_ABSENT.
// plan: the chain's plans (lc_regex_sls_plans: entries [0, n_ok) parsed, then n_fail failed; key id k names kstr[k] /
// klen[k]); a plan's keys are unique.
inline void lc_regex_sls_key_src(const uint32_t* plan, uint32_t n_ok, uint32_t n_fail, const char* const* kstr,
                                 const uint32_t* klen, const char* key, uint32_t len, uint32_t src[2]) {
    for (uint32_t v = 0; v < 2; ++v) {
        const uint32_t* e = plan + (v ? 2u * n_ok : 0u);
        uint32_t s = LC_FILTER_SLS_ABSENT;
        for (uint32_t k = 0; k < (v ? n_fail : n_ok); ++k) {
            const uint32_t kid = e[2 * k];
            if (klen[kid] == len && (!len || !memcmp(kstr[kid], key, len))) {
                s = e[2 * k + 1];
                break;
            }
        }
        src[v] = s;
    }
}

// Host side: resolve the leaves against the chain's plans (lc_regex_sls_key_src) and check the program.  Returns nullptr, or why the filter is refused: more
// than LC_FILTER_SLS_LEAVES leaves or LC_FILTER_SLS_PROG entries, an entry that is neither a leaf nor an opcode, a pop
// of an empty stack, a stack deeper than 32, or a program that does not leave exactly one value.
inline const char* lc_filter_sls_setup(const uint32_t* plan, uint32_t n_ok, uint32_t n_fail, const char* const* kstr,
                                       const uint32_t* klen, uint32_t nleaves, const char* const* leaf_keys,
                                       const uint32_t* leaf_lens, uint32_t nprog, const uint32_t* prog,
                                       LcFilterSlsCfg* f) {
    if (!f || !plan || (nleaves && (!leaf_keys || !leaf_lens)) || (nprog && !prog))
        return "bad arguments";
    if (nleaves > LC_FILTER_SLS_LEAVES)
        return "too many filter leaves";
    if (nprog > LC_FILTER_SLS_PROG)
        return "filter program too long";
    memset(f, 0, sizeof *f);
    f->nleaves = nleaves;
    f->nprog = nprog;
    f->empty[0] = n_ok == 0u;
    f->empty[1] = n_fail == 0u;
    uint32_t depth = 0;
    for (uint32_t k = 0; k < nprog; ++k) {
        const uint32_t op = prog[k];
        if (op < nleaves) {
            if (++depth > 32u)
                return "filter program too deep";
            f->prog[k] = (uint8_t)op;
        } else if (op == LC_FILTER_SLS_NOT) {
            if (depth < 1u)
                return "malformed filter program";
            f->prog[k] = 253;
        } else if (op == LC_FILTER_SLS_AND || op == LC_FILTER_SLS_OR) {
            if (depth < 2u)
                return "malformed filter program";
            --depth;
            f->prog[k] = op == LC_FILTER_SLS_AND ? 254 : 255;
        } else {
            return "malformed filter program";
        }
    }
    if (nprog && depth != 1u)
        return "malformed filter program";
    for (uint32_t l = 0; l < nleaves; ++l) {
        if (leaf_lens[l] && !leaf_keys[l])
            return "bad arguments";
        lc_regex_sls_key_src(plan, n_ok, n_fail, kstr, klen, leaf_keys[l], leaf_lens[l], f->src[l]);
        for (uint32_t v = 0; v < 2; ++v)
            f->any_digits |= f->src[l][v] == LC_REGEX_SLS_DIGITS;
    }
    return nullptr;
}

// The row's value source for leaf l: LC_FILTER_SLS_ABSENT, LC_REGEX_SLS_DIGITS, LC_REGEX_SLS_LINE or capture j.  An
// erased row (failed without KeepingSourceWhenParseFail) never reaches the filter; its failed plan is empty.
LC_HD uint32_t lc_filter_leaf_src(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, uint32_t l, uint32_t status) {
    return f.src[l][lc_regex_sls_verdict(c.x, status) == 0u ? 0 : 1];
}

// The leaf's value in row r: *off / *len into the source value (the piece or a capture), or *len = the digit count of
// the piece's offset.  Returns the source (absent: *off = *len = 0).
LC_HD uint32_t lc_filter_leaf(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, uint32_t l,
                              const LcSplitRegexSlsRow& r, uint32_t* off, uint32_t* len) {
    const uint32_t s = lc_filter_leaf_src(c, f, l, r.status);
    *off = 0;
    *len = 0;
    if (s == LC_REGEX_SLS_DIGITS)
        *len = lc_dec_digits(c.src_pos + r.po);
    else if (s == LC_REGEX_SLS_LINE)
        *off = r.po, *len = r.plen;
    else if (s != LC_FILTER_SLS_ABSENT)
        *off = r.co[s], *len = r.cl[s];
    return s;
}

// The filter's verdict on an event that reached it: 1 kept, 0 removed.  bits: bit l = leaf l held (an absent key
// holds no leaf).  empty: the event has no contents.
LC_HD uint32_t lc_filter_eval(const LcFilterSlsCfg& f, uint32_t bits, bool empty) {
    if (f.nprog == 0u)
        return 1u;
    if (empty)
        return 0u;
    uint32_t st = 0, sp = 0; // the stack, bit sp - 1 on top
    for (uint32_t k = 0; k < f.nprog; ++k) {
        const uint32_t op = f.prog[k];
        if (op < LC_FILTER_SLS_LEAVES) {
            st = (st & ~(1u << sp)) | (((bits >> op) & 1u) << sp);
            ++sp;
        } else if (op == 253u) {
            st ^= 1u << (sp - 1);
        } else {
            --sp;
            const uint32_t a = (st >> (sp - 1)) & 1u, b = (st >> sp) & 1u;
            const uint32_t v = op == 254u ? (a & b) : (a | b);
            st = (st & ~(1u << (sp - 1))) | (v << (sp - 1));
        }
    }
    return st & 1u;
}

// The row's verdicts behind the filter: *reached = the regex stage kept it, *empty = it has no contents.
LC_HD void lc_filter_row_state(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, uint32_t status, bool* reached,
                               bool* empty) {
    const bool ok = lc_regex_sls_verdict(c.x, status) == 0u;
    *reached = ok || c.x.keep_fail;
    *empty = f.empty[ok ? 0 : 1] != 0u;
}

// ------------------------------------------------------------------------------------------------------------
// f4, LZ4: one LZ4 *block* (what LZ4_compress_default emits and the SLS server decodes with x-log-bodyrawsize) per
// segment.  A segment is cut into chunks of LC_LZ4_CHUNK bytes; the bytes are a sequential function of the segment:
//   candidate(p)  = the latest q < p with hash(q) == hash(p), kept as q mod 2^16 (so read as the q' = p - d with
//                   d = (p - q) mod 2^16 in [0, 65535]); table entries nothing wrote read as 0 mod 2^16
//   match at p    = p >= the end of the chunk's previous match, d != 0, d <= p, the 4 bytes at p and p - d equal,
//                   p + 12 <= n (the last match starts 12 bytes before the end) and p + 4 <= the chunk's end
//   match length  = the longest run of equal bytes at p and p - d that ends by min(chunk end, n - 5)
// Greedy: the first match in a chunk is taken, the parse resumes at its end.  The table of a chunk is seeded with the
// positions from max(0, c0 - 65535) so that matches reach back into earlier chunks; matches end at the chunk's end, so
// chunks parse independently.  A literal run belongs to the chunk holding the match that ends it (or to the segment's
// last chunk), so a run may span many chunks.  The parse runs W positions at a time: W lanes of a warp on the device
// (W = 32), any W on the host (tests/emul), with the same result, since table updates in a batch are resolved in
// position order.
#define LC_LZ4_CHUNK 65536u
#define LC_LZ4_HASH_LOG 12
#define LC_LZ4_SEQ_CAP (LC_LZ4_CHUNK / 4) // sequences per chunk: matches are >= 4 bytes and end inside the chunk
#define LC_LZ4_MAX_INPUT 0x7E000000u      // LZ4_MAX_INPUT_SIZE
#define LC_LZ4_NOHASH 0xFFFFFFFFu

struct LcLz4Warp { // per-warp scratch (shared memory on the device)
    uint16_t tbl[1u << LC_LZ4_HASH_LOG];
    uint32_t h[32]; // the batch's hashes (LC_LZ4_NOHASH = no position)
    uint32_t d[32]; // candidate distance of each position
    uint32_t v[32]; // per-lane predicate of a ballot
};

struct LcLz4Seq { // one match of a chunk: a = (p - c0) | d << 16, b = length
    uint32_t a, b;
};

struct LcLz4Chunk { // parse pass result of one chunk
    uint32_t nseq;
    uint32_t isize;    // encoded bytes of its sequences, less the first one's token, literal-length bytes and literals
    uint32_t first;    // position of the first match
    uint32_t last_end; // end of the last match
};

LC_HD uint32_t lc_lz4_ext(uint32_t len) { return len >= 15 ? (len - 15) / 255 + 1 : 0u; }
LC_HD uint32_t lc_lz4_rd32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
LC_HD uint32_t lc_lz4_hash(uint32_t v) { return (v * 2654435761u) >> (32 - LC_LZ4_HASH_LOG); }
LC_HD uint32_t lc_lz4_bound(uint32_t n) { return n + n / 255 + 16; } // LZ4_compressBound
LC_HD uint32_t lc_lz4_nchunks(uint32_t n) { return n ? (n + LC_LZ4_CHUNK - 1) / LC_LZ4_CHUNK : 1u; }

LC_HD uint32_t lc_lo_bit(uint32_t m) { // m != 0
#if defined(__CUDA_ARCH__)
    return __ffs(m) - 1;
#else
    return __builtin_ctz(m);
#endif
}
LC_HD uint32_t lc_hi_bit(uint32_t m) { // m != 0
#if defined(__CUDA_ARCH__)
    return 31 - __clz(m);
#else
    return 31 - __builtin_clz(m);
#endif
}

// The lanes of a batch: on the device each lane runs the body once for itself and the warp synchronises between
// phases; the host runs the body for each of the W lanes in turn, which is a valid interleaving of the same phases.
#if defined(__CUDA_ARCH__)
#define LC_LANES(l) for (uint32_t l = lane, l##_once = 1; l##_once; l##_once = 0)
#define LC_WARP_SYNC() __syncwarp()
#else
#define LC_LANES(l) for (uint32_t l = 0; l < W; ++l)
#define LC_WARP_SYNC() ((void)0)
#endif

// bit l = v[l] != 0 for the W lanes (all lanes call it)
LC_HD uint32_t lc_lz4_ballot(const uint32_t* v, uint32_t lane, uint32_t W) {
#if defined(__CUDA_ARCH__)
    (void)W;
    return __ballot_sync(0xFFFFFFFFu, v[lane] != 0);
#else
    (void)lane;
    uint32_t m = 0;
    for (uint32_t j = 0; j < W; ++j)
        m |= (v[j] != 0) << j;
    return m;
#endif
}

// bit j = lane j of the batch has lane l's hash (all lanes call it, each with l = its lane)
LC_HD uint32_t lc_lz4_peers(const uint32_t* h, uint32_t l, uint32_t W) {
#if defined(__CUDA_ARCH__)
    (void)W;
    return __match_any_sync(0xFFFFFFFFu, h[l]);
#else
    uint32_t m = 0;
    for (uint32_t j = 0; j < W; ++j)
        m |= (h[j] == h[l]) << j;
    return m;
#endif
}

// Parse pass of chunk [c0, c1) of the segment s[0, n): its matches go to seq[0, nseq), the summary to *info.
LC_HD void lc_lz4_parse_chunk(const uint8_t* s, uint32_t n, uint32_t c0, uint32_t c1, LcLz4Warp& w, LcLz4Seq* seq,
                              LcLz4Chunk* info, uint32_t lane, uint32_t W) {
    LC_LANES(l) {
        for (uint32_t i = l; i < (1u << LC_LZ4_HASH_LOG); i += W)
            w.tbl[i] = 0;
    }
    LC_WARP_SYNC();
    const uint32_t full = W == 32 ? 0xFFFFFFFFu : (1u << W) - 1u;
    const uint32_t seed = c0 > 65535u ? c0 - 65535u : 0u;
    const uint32_t hend = n >= 4 && c1 > n - 4 ? n - 3 : (n >= 4 ? c1 : 0u); // positions with 4 bytes, < c1
    const uint32_t mend = n >= 12 ? n - 11 : 0u;                              // match starts: p + 12 <= n
    const uint32_t lim = n >= 5 && c1 > n - 5 ? n - 5 : c1;                   // match ends
    uint32_t cur = c0, nseq = 0, isize = 0, first = 0, last_end = 0;
    for (int64_t b = (int64_t)c0 - (int64_t)((c0 - seed + W - 1) / W * W); b < (int64_t)hend; b += W) {
        LC_LANES(l) {
            const int64_t p = b + l;
            w.h[l] = p >= (int64_t)seed && p < (int64_t)hend ? lc_lz4_hash(lc_lz4_rd32(s + p)) : LC_LZ4_NOHASH;
        }
        LC_WARP_SYNC();
        // candidates: the latest earlier lane of the batch with the same hash, else the table
        LC_LANES(l) {
            const uint32_t pr = lc_lz4_peers(w.h, l, W);
            const uint32_t below = pr & ((1u << l) - 1u);
            const uint32_t p = (uint32_t)(b + l);
            w.d[l] = w.h[l] == LC_LZ4_NOHASH ? 0u
                     : below                 ? l - lc_hi_bit(below)
                                             : (uint32_t)(uint16_t)(p - w.tbl[w.h[l]]);
        }
        LC_WARP_SYNC();
        // the table keeps the last lane of each hash
        LC_LANES(l) {
            const uint32_t pr = lc_lz4_peers(w.h, l, W);
            if (w.h[l] != LC_LZ4_NOHASH && !((pr >> l) >> 1))
                w.tbl[w.h[l]] = (uint16_t)(b + l);
        }
        LC_WARP_SYNC();
        if (b + W <= (int64_t)cur)
            continue;
        LC_LANES(l) {
            const int64_t p = b + l;
            const uint32_t d = w.d[l];
            w.v[l] = p >= (int64_t)cur && p < (int64_t)mend && p + 4 <= (int64_t)c1 && w.h[l] != LC_LZ4_NOHASH && d &&
                     d <= p && lc_lz4_rd32(s + p) == lc_lz4_rd32(s + p - d);
        }
        uint32_t m = lc_lz4_ballot(w.v, lane, W);
        LC_WARP_SYNC();
        while (m) {
            const uint32_t j = lc_lo_bit(m);
            const uint32_t p = (uint32_t)(b + j), d = w.d[j];
            uint32_t len = 4;
            for (;;) { // extend W bytes at a time
                LC_LANES(l) {
                    const uint32_t x = p + len + l;
                    w.v[l] = x < lim && s[x] == s[x - d];
                }
                const uint32_t eq = lc_lz4_ballot(w.v, lane, W);
                LC_WARP_SYNC();
                const uint32_t run = eq == full ? W : lc_lo_bit(~eq);
                len += run;
                if (run < W)
                    break;
            }
            if (lane == 0)
                seq[nseq] = LcLz4Seq{(p - c0) | (d << 16), len};
            isize += (nseq ? 1 + lc_lz4_ext(p - last_end) + (p - last_end) : 0u) + 2 + lc_lz4_ext(len - 4);
            if (!nseq)
                first = p;
            ++nseq;
            last_end = cur = p + len;
            m = (int64_t)cur >= b + W ? 0u : m & (full << (uint32_t)(cur - b));
        }
    }
    if (lane == 0)
        *info = LcLz4Chunk{nseq, isize, first, last_end};
}

// Size pass of one segment of n bytes and nch chunks: the block bytes of each chunk and the literal anchor it starts
// from (the end of the latest match in an earlier chunk).  The last chunk ends the block with a literals-only sequence.
LC_HD void lc_lz4_seg_sizes(uint32_t n, uint32_t nch, const LcLz4Chunk* info, uint32_t* csize, uint32_t* anchor) {
    uint32_t a = 0;
    for (uint32_t k = 0; k < nch; ++k) {
        anchor[k] = a;
        uint32_t sz = 0;
        if (info[k].nseq) {
            const uint32_t l0 = info[k].first - a;
            sz = info[k].isize + 1 + lc_lz4_ext(l0) + l0;
            a = info[k].last_end;
        }
        if (k + 1 == nch)
            sz += 1 + lc_lz4_ext(n - a) + (n - a);
        csize[k] = sz;
    }
}

// a length's extension bytes (len >= 15) at o[0, lc_lz4_ext(len)), lanes share them
LC_HD void lc_lz4_put_ext(uint8_t* o, uint32_t len, uint32_t lane, uint32_t W) {
    const uint32_t nb = lc_lz4_ext(len);
    LC_LANES(l) {
        for (uint32_t j = l; j < nb; j += W)
            o[j] = j + 1 < nb ? 255 : (uint8_t)((len - 15) % 255);
    }
}

// one sequence at o: lit literals from s + a, then (mlen != 0) a match of mlen bytes at distance d.  Returns its bytes.
LC_HD uint32_t lc_lz4_put_seq(const uint8_t* s, uint32_t a, uint32_t lit, uint32_t d, uint32_t mlen, uint8_t* o,
                              uint32_t lane, uint32_t W) {
    const uint32_t ml = mlen ? mlen - 4 : 0u;
    if (lane == 0)
        o[0] = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (ml < 15 ? ml : 15));
    uint32_t q = 1;
    lc_lz4_put_ext(o + q, lit, lane, W);
    q += lc_lz4_ext(lit);
    LC_LANES(l) {
        for (uint32_t j = l; j < lit; j += W)
            o[q + j] = s[a + j];
    }
    q += lit;
    if (!mlen)
        return q;
    if (lane == 0) {
        o[q] = (uint8_t)d;
        o[q + 1] = (uint8_t)(d >> 8);
    }
    q += 2;
    lc_lz4_put_ext(o + q, ml, lane, W);
    return q + lc_lz4_ext(ml);
}

// Emit pass of chunk [c0, ..) of the segment s[0, n): its sequences (from its anchor) and, for the segment's last
// chunk, the closing literals, at o.
LC_HD void lc_lz4_emit_chunk(const uint8_t* s, uint32_t n, uint32_t c0, const LcLz4Seq* seq, uint32_t nseq,
                             uint32_t anchor, bool last, uint8_t* o, uint32_t lane, uint32_t W) {
    uint32_t a = anchor;
    for (uint32_t i = 0; i < nseq; ++i) {
        const LcLz4Seq q = seq[i];
        const uint32_t p = c0 + (q.a & 0xFFFFu);
        o += lc_lz4_put_seq(s, a, p - a, q.a >> 16, q.b, o, lane, W);
        a = p + q.b;
    }
    if (last)
        lc_lz4_put_seq(s, a, n - a, 0, 0, o, lane, W);
}

// ------------------------------------------------------------------------------------------------------------
// f4, zstd: one zstd *frame* (RFC 8878) per segment, for FlusherSLS's CompressType "zstd" (ZstdCompressor =
// ZSTD_compress).  The bytes are a sequential function of the segment s[0, n); they need not equal libzstd's.
//   frame      = magic 28 b5 2f fd; a Frame_Header_Descriptor with Single_Segment_Flag = 1, no checksum and no
//                dictionary; Frame_Content_Size in 1 byte (n < 256, FCS flag 0), 2 bytes (n < 65792, flag 1, n - 256) or
//                4 bytes (flag 2); then the blocks.  An empty segment is one empty Raw block: 28 b5 2f fd 20 00 01 00 00.
//   blocks     = LC_ZSTD_BLOCK (128 KiB) bytes of the segment each, the last one shorter.  A block whose compressed
//                body would not be smaller than its bytes is a Raw block; RLE blocks are not used.
//   sequences  = the matches lc_lz4_parse_chunk finds in the block's two LZ4 chunks (they end inside their chunk, so
//                inside the block), each a new offset: Offset_Value = distance + 3, never a repeat offset.
//                Literals_Length = the bytes since the block's previous match (or its start): literal runs are cut at
//                block boundaries, and the bytes after the last match are the block's trailing literals.  LL, OF and ML
//                use the predefined distributions (Symbol_Compression_Modes = 0); each FSE state starts at the lowest
//                decoding state of its symbol.  A block without a match has Number_of_Sequences = 0.
//   literals   = RLE for one distinct byte; Raw for fewer than LC_ZSTD_MIN_HUF literals or when Huffman would not be
//                smaller; else Huffman_Compressed in 4 streams, with the code of lc_zstd_huf_lengths (at most
//                LC_ZSTD_HUF_MAX bits).  Its weights are described with FSE (accuracy log LC_ZSTD_WLOG, counts of
//                lc_zstd_wnorm) or in the direct 4-bit form, whichever is smaller (the direct form on a tie); with
//                neither possible the literals go Raw.
// A block is built by W lanes (lc_zstd_block): a warp on the device (W = 32), any W on the host (tests/emul), with the
// same bytes.  Its literals are gathered behind each chunk's matches in the LZ4 sequence scratch, which has room for
// them: a chunk of c bytes with L literals has at most (c - L) / 4 matches of 8 bytes, and 2 (c - L) + L <= 2 c.
#define LC_ZSTD_BLOCK (2u * LC_LZ4_CHUNK) // segment bytes per block: two LZ4 chunks
#define LC_ZSTD_MIN_HUF 64u               // fewer literals are not Huffman-coded (4 streams need at least 6)
#define LC_ZSTD_HUF_MAX 11u               // longest Huffman code
#define LC_ZSTD_WLOG 6u                   // accuracy log of the FSE weight description
#define LC_ZSTD_RAW 0u                    // literal modes (Literals_Block_Type)
#define LC_ZSTD_RLE 1u
#define LC_ZSTD_HUF 2u

LC_HD uint32_t lc_zstd_nblocks(uint32_t n) { return n ? (n + LC_ZSTD_BLOCK - 1) / LC_ZSTD_BLOCK : 1u; }
LC_HD uint32_t lc_zstd_fcs_bytes(uint32_t n) { return n < 256 ? 1u : n < 65536 + 256 ? 2u : 4u; }
LC_HD uint32_t lc_zstd_hdr(uint32_t n) { return 5 + lc_zstd_fcs_bytes(n); } // magic, descriptor, content size
LC_HD uint64_t lc_zstd_bound(uint64_t n) {                                    // ZSTD_compressBound
    return n + (n >> 8) + (n < (128u << 10) ? ((128u << 10) - n) >> 11 : 0u);
}

LC_HD uint32_t lc_popc(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}
LC_HD uint32_t lc_bits(uint32_t k) { return k >= 32 ? 0xFFFFFFFFu : (1u << k) - 1u; } // the k low bits
LC_HD void lc_or32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
LC_HD void lc_add32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

// OR of v[0, W) (all lanes call it)
LC_HD uint32_t lc_warp_or(const uint32_t* v, uint32_t lane, uint32_t W) {
#if defined(__CUDA_ARCH__)
    (void)W;
    return __reduce_or_sync(0xFFFFFFFFu, v[lane]);
#else
    (void)lane;
    uint32_t m = 0;
    for (uint32_t j = 0; j < W; ++j)
        m |= v[j];
    return m;
#endif
}

// v[0, W) -> its exclusive prefix sums, in place; returns the total (all lanes call it)
LC_HD uint32_t lc_warp_exscan(uint32_t* v, uint32_t lane, uint32_t W) {
#if defined(__CUDA_ARCH__)
    (void)W;
    const uint32_t x = v[lane];
    uint32_t s = x;
    for (uint32_t d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, s, d);
        if (lane >= d)
            s += y;
    }
    v[lane] = s - x;
    return __shfl_sync(0xFFFFFFFFu, s, 31);
#else
    (void)lane;
    uint32_t s = 0;
    for (uint32_t j = 0; j < W; ++j) {
        const uint32_t x = v[j];
        v[j] = s;
        s += x;
    }
    return s;
#endif
}

// Forward bit writer, least significant bit first (every zstd bitstream and the FSE table description).  Bytes at
// and past `cap` are counted in n but not written.
struct LcBitW {
    uint8_t* o;
    uint32_t n, cap, nb;
    uint64_t acc;
};
LC_HD void lc_bw_put(LcBitW& b, uint32_t v, uint32_t nbits) { // nbits <= 24
    b.acc |= (uint64_t)v << b.nb;
    b.nb += nbits;
    while (b.nb >= 8) {
        if (b.n < b.cap)
            b.o[b.n] = (uint8_t)b.acc;
        ++b.n;
        b.acc >>= 8;
        b.nb -= 8;
    }
}
LC_HD void lc_bw_align(LcBitW& b) { // zero bits up to the next byte
    if (b.nb)
        lc_bw_put(b, 0, 8 - b.nb);
}
LC_HD void lc_bw_close(LcBitW& b) { // a backward-read bitstream ends with a 1 bit, then zeros to the byte
    lc_bw_put(b, 1, 1);
    lc_bw_align(b);
}

// An FSE table of accuracy log al: the decoding spread sym[] and, per symbol s, its decoding states in increasing
// order st[cum[s], cum[s + 1]).
struct LcFse {
    uint16_t cum[54];
    uint8_t st[64];
    uint8_t sym[64];
    uint32_t al;
};

// normalised count of symbol s (-1 = "less than 1"): the predefined LL (tab 0), ML (1) and OF (2) distributions
// (RFC 8878 3.1.1.3.2.2), or wn[s] (tab 3)
LC_HD int lc_zstd_norm(uint32_t tab, const int16_t* wn, uint32_t s) {
    if (tab == 0)
        return s == 0 ? 4 : s == 1 ? 3 : s <= 12 ? 2 : s <= 15 ? 1 : s <= 24 ? 2 : s == 25 ? 3 : s == 26 ? 2 : s <= 31 ? 1 : -1;
    if (tab == 1)
        return s == 0 ? 1 : s == 1 ? 4 : s == 2 ? 3 : s <= 8 ? 2 : s <= 45 ? 1 : -1;
    if (tab == 2)
        return s <= 5 ? 1 : s <= 8 ? 2 : s <= 23 ? 1 : -1;
    return wn[s];
}

// one lane builds t for the nsym symbols of table `tab` (FSE_buildDTable's spread)
LC_HD void lc_fse_build(uint32_t tab, const int16_t* wn, uint32_t nsym, uint32_t al, LcFse& t) {
    const uint32_t T = 1u << al, step = (T >> 1) + (T >> 3) + 3;
    uint32_t high = T - 1, pos = 0;
    t.al = al;
    t.cum[0] = 0;
    for (uint32_t s = 0; s < nsym; ++s) {
        const int c = lc_zstd_norm(tab, wn, s);
        if (c == -1)
            t.sym[high--] = (uint8_t)s;
        t.cum[s + 1] = (uint16_t)(t.cum[s] + (c < 0 ? 1 : c));
    }
    for (uint32_t s = 0; s < nsym; ++s)
        for (int i = 0, c = lc_zstd_norm(tab, wn, s); i < c; ++i) {
            t.sym[pos] = (uint8_t)s;
            do
                pos = (pos + step) & (T - 1);
            while (pos > high);
        }
    for (uint32_t u = 0; u < T; ++u) // cum[s] runs to cum[s + 1] ...
        t.st[t.cum[t.sym[u]]++] = (uint8_t)u;
    for (uint32_t s = nsym; s > 0; --s) // ... and is put back
        t.cum[s] = t.cum[s - 1];
    t.cum[0] = 0;
}

// The encoder's first state for symbol s, and one encoding step: from state S (the next symbol's) to a state of s,
// writing the bits the decoder reads to get from there back to S.
LC_HD uint32_t lc_fse_init(const LcFse& t, uint32_t s) { return t.st[t.cum[s]]; }
LC_HD uint32_t lc_fse_enc(const LcFse& t, uint32_t S, uint32_t s, LcBitW& b) {
    const uint32_t c = t.cum[s + 1] - t.cum[s], V = S + (1u << t.al);
    uint32_t nb = lc_hi_bit(V) - lc_hi_bit(2 * c - 1);
    if ((V >> nb) >= 2 * c)
        ++nb;
    lc_bw_put(b, V & lc_bits(nb), nb);
    return t.st[t.cum[s] + (V >> nb) - c];
}

// The FSE table description (FSE_writeNCount) of norm[0, nsym), accuracy log al.
LC_HD void lc_fse_ncount(const int16_t* norm, uint32_t nsym, uint32_t al, LcBitW& b) {
    lc_bw_put(b, al - 5, 4);
    int remaining = (1 << al) + 1, threshold = 1 << al;
    uint32_t nbits = al + 1, s = 0;
    bool prev0 = false;
    while (s < nsym && remaining > 1) {
        if (prev0) {
            uint32_t start = s;
            while (!norm[s])
                ++s;
            for (; s >= start + 24; start += 24)
                lc_bw_put(b, 0xFFFFu, 16);
            for (; s >= start + 3; start += 3)
                lc_bw_put(b, 3, 2);
            lc_bw_put(b, s - start, 2);
        }
        int count = norm[s++];
        const int max = (2 * threshold - 1) - remaining;
        remaining -= count < 0 ? -count : count;
        ++count;
        if (count >= threshold)
            count += max;
        lc_bw_put(b, (uint32_t)count, nbits - (count < max));
        prev0 = count == 1;
        while (remaining < threshold) {
            --nbits;
            threshold >>= 1;
        }
    }
    lc_bw_align(b);
}

// FSE counts of the weight description: c[v] weights of value v < nv among nw, at least 2 distinct values.  Each count
// is at most half the table, so that every decoding state reads at least one bit: the two-state weight decoder then
// stops after exactly nw weights.
LC_HD void lc_zstd_wnorm(const uint32_t* c, uint32_t nv, uint32_t nw, int16_t* norm) {
    const int T = 1 << LC_ZSTD_WLOG;
    int sum = 0;
    for (uint32_t v = 0; v < nv; ++v) {
        int x = (int)((uint64_t)c[v] * T / nw);
        x = c[v] && x < 1 ? 1 : x > T / 2 ? T / 2 : x;
        norm[v] = (int16_t)x;
        sum += x;
    }
    while (sum > T) { // the largest count gives one
        uint32_t best = nv;
        for (uint32_t v = 0; v < nv; ++v)
            if (norm[v] > 1 && (best == nv || norm[v] > norm[best]))
                best = v;
        --norm[best];
        --sum;
    }
    while (sum < T) { // the most frequent value below half the table takes one
        uint32_t best = nv;
        for (uint32_t v = 0; v < nv; ++v)
            if (c[v] && norm[v] < T / 2 && (best == nv || c[v] > c[best]))
                best = v;
        ++norm[best];
        ++sum;
    }
}

struct LcZstdWarp { // per-warp scratch of the block pass (shared memory on the device)
    uint32_t hist[256];         // literal counts
    uint32_t ncnt[512];         // Huffman node counts (leaves in `order`, then internal nodes)
    uint16_t npar[512];         // Huffman node parents, then depths
    uint16_t code[256];         // Huffman code of each byte
    uint8_t len[256];           // its length (0: absent)
    uint8_t order[256];         // the bytes present, by increasing (count, byte)
    uint32_t st[16];            // bit staging of a Huffman stream
    uint32_t v[32], u[32];      // per-lane values
    uint32_t nl[16];            // codes per length, then the next code of each length
    uint32_t res[4];            // lane 0's results for the warp
    uint32_t wc[16];            // weight value counts
    int16_t wn[16];             // their FSE counts
    uint8_t wdesc[128];         // the Huffman tree description
    LcFse ll, ml, of, wf;       // predefined sequence tables, weight table
};

// Huffman code lengths (one lane) of the m >= 2 bytes order[0, m) with counts hist[]: a Huffman tree over the leaves in
// increasing order (a leaf before an internal node of the same count), depths over LC_ZSTD_HUF_MAX cut to it, then the
// Kraft sum repaired: the least frequent codes shorter than the limit grow until the code fits, and the most frequent
// codes shrink while it stays within.  Returns the longest length; the code is complete.
LC_HD uint32_t lc_zstd_huf_lengths(LcZstdWarp& w, uint32_t m) {
    const uint32_t M = LC_ZSTD_HUF_MAX, full = 1u << M;
    for (uint32_t i = 0; i < m; ++i)
        w.ncnt[i] = w.hist[w.order[i]];
    uint32_t li = 0, ii = m;
    for (uint32_t nn = m; nn < 2 * m - 1; ++nn) {
        uint32_t a[2];
        for (uint32_t k = 0; k < 2; ++k)
            a[k] = li < m && (ii >= nn || w.ncnt[li] <= w.ncnt[ii]) ? li++ : ii++;
        w.ncnt[nn] = w.ncnt[a[0]] + w.ncnt[a[1]];
        w.npar[a[0]] = w.npar[a[1]] = (uint16_t)nn;
    }
    w.npar[2 * m - 2] = 0;
    for (uint32_t i = 2 * m - 2; i-- > 0;)
        w.npar[i] = (uint16_t)(w.npar[w.npar[i]] + 1);
    uint32_t K = 0; // Kraft sum in units of 2^-M
    for (uint32_t i = 0; i < m; ++i) {
        const uint32_t d = w.npar[i] < M ? w.npar[i] : M;
        w.len[w.order[i]] = (uint8_t)d;
        K += 1u << (M - d);
    }
    for (uint32_t i = 0; K > full;) {
        uint8_t& L = w.len[w.order[i]];
        if (L >= M) {
            ++i;
            continue;
        }
        K -= 1u << (M - 1 - L);
        ++L;
    }
    while (K < full)
        for (uint32_t i = m; i-- > 0 && K < full;) {
            uint8_t& L = w.len[w.order[i]];
            while (L > 1 && K + (1u << (M - L)) <= full) {
                K += 1u << (M - L);
                --L;
            }
        }
    uint32_t lmax = 0;
    for (uint32_t i = 0; i < m; ++i)
        lmax = w.len[w.order[i]] > lmax ? w.len[w.order[i]] : lmax;
    return lmax;
}

// Canonical codes of the lengths (one lane): by decreasing length, then increasing byte, from code 0 (RFC 8878
// 4.2.1.3).  Then the tree description of the weights of bytes [0, maxs) in w.wdesc (the weight of byte maxs is
// implied); returns its size, or 0 when neither form can hold it.
LC_HD uint32_t lc_zstd_huf_table(LcZstdWarp& w, uint32_t lmax, uint32_t maxs) {
    for (uint32_t L = 0; L < 16; ++L)
        w.nl[L] = 0;
    for (uint32_t s = 0; s <= maxs; ++s)
        ++w.nl[w.len[s]];
    uint32_t next = 0;
    for (uint32_t L = lmax; L >= 1; --L) { // nl[L] becomes the first code of length L
        const uint32_t c = w.nl[L];
        w.nl[L] = next;
        next = (next + c) >> 1;
    }
    for (uint32_t s = 0; s <= maxs; ++s)
        if (w.len[s])
            w.code[s] = (uint16_t)w.nl[w.len[s]]++;
    // weights: lmax + 1 - length (0 for an absent byte)
    const uint32_t N = maxs;
    uint32_t nv = 0, distinct = 0;
    for (uint32_t v = 0; v < 16; ++v)
        w.wc[v] = 0;
    for (uint32_t s = 0; s < N; ++s) {
        const uint32_t wt = w.len[s] ? lmax + 1 - w.len[s] : 0u;
        distinct += !w.wc[wt]++;
        nv = wt + 1 > nv ? wt + 1 : nv;
    }
    const uint32_t direct = N <= 128 ? 1 + (N + 1) / 2 : 0u;
    uint32_t fse = 0;
    if (distinct >= 2) {
        lc_zstd_wnorm(w.wc, nv, N, w.wn);
        lc_fse_build(3, w.wn, nv, LC_ZSTD_WLOG, w.wf);
        LcBitW b{w.wdesc + 1, 0, 127, 0, 0};
        lc_fse_ncount(w.wn, nv, LC_ZSTD_WLOG, b);
        // two interleaved states: even weights on the first, odd on the second, encoded from the end
        uint32_t X[2];
        const auto wt = [&](uint32_t s) { return w.len[s] ? lmax + 1 - w.len[s] : 0u; };
        X[(N - 1) & 1] = lc_fse_init(w.wf, wt(N - 1));
        X[(N - 2) & 1] = lc_fse_init(w.wf, wt(N - 2));
        for (uint32_t i = N - 2; i-- > 0;)
            X[i & 1] = lc_fse_enc(w.wf, X[i & 1], wt(i), b);
        lc_bw_put(b, X[1], LC_ZSTD_WLOG);
        lc_bw_put(b, X[0], LC_ZSTD_WLOG);
        lc_bw_close(b);
        fse = b.n <= 127 ? 1 + b.n : 0u;
    }
    if (fse && (!direct || fse < direct)) {
        w.wdesc[0] = (uint8_t)(fse - 1);
        return fse;
    }
    if (!direct)
        return 0;
    w.wdesc[0] = (uint8_t)(127 + N);
    for (uint32_t j = 0; 2 * j < N; ++j) {
        const uint32_t a = w.len[2 * j] ? lmax + 1 - w.len[2 * j] : 0u;
        const uint32_t c = 2 * j + 1 < N && w.len[2 * j + 1] ? lmax + 1 - w.len[2 * j + 1] : 0u;
        w.wdesc[1 + j] = (uint8_t)(a << 4 | c);
    }
    return direct;
}

// sequence codes (RFC 8878 3.1.1.3.2.1): literal length ll, match length code of mb = ml - 3
LC_HD uint32_t lc_zstd_llc(uint32_t ll) {
    return ll < 16 ? ll : ll < 24 ? 16 + ((ll - 16) >> 1) : ll < 32 ? 20 + ((ll - 24) >> 2) : ll < 48 ? 22 + ((ll - 32) >> 3) : ll < 64 ? 24 : lc_hi_bit(ll) + 19;
}
LC_HD uint32_t lc_zstd_llbase(uint32_t c) {
    return c < 16 ? c : c < 20 ? 16 + 2 * (c - 16) : c < 22 ? 24 + 4 * (c - 20) : c < 24 ? 32 + 8 * (c - 22) : c == 24 ? 48 : 1u << (c - 19);
}
LC_HD uint32_t lc_zstd_llbits(uint32_t c) { return c < 16 ? 0 : c < 20 ? 1 : c < 22 ? 2 : c < 24 ? 3 : c == 24 ? 4 : c - 19; }
LC_HD uint32_t lc_zstd_mlc(uint32_t mb) {
    return mb < 32 ? mb : mb < 40 ? 32 + ((mb - 32) >> 1) : mb < 48 ? 36 + ((mb - 40) >> 2) : mb < 64 ? 38 + ((mb - 48) >> 3) : mb < 96 ? 40 + ((mb - 64) >> 4) : mb < 128 ? 42 : lc_hi_bit(mb) + 36;
}
LC_HD uint32_t lc_zstd_mlbase(uint32_t c) {
    return c < 32 ? c : c < 36 ? 32 + 2 * (c - 32) : c < 38 ? 40 + 4 * (c - 36) : c < 40 ? 48 + 8 * (c - 38) : c < 42 ? 64 + 16 * (c - 40) : c == 42 ? 96 : 1u << (c - 36);
}
LC_HD uint32_t lc_zstd_mlbits(uint32_t c) { return c < 32 ? 0 : c < 36 ? 1 : c < 38 ? 2 : c < 40 ? 3 : c < 42 ? 4 : c == 42 ? 5 : c - 36; }

// One block: segment bytes s[b0, b1) (b1 - b0 <= LC_ZSTD_BLOCK), the matches of its first chunk seq[0][0, nseq[0]) and
// of its second seq[1][0, nseq[1]) (seq[1] == nullptr: one chunk).  Each chunk's literals go to its scratch behind its
// matches.
struct LcZstdBlk {
    const uint8_t* s;
    uint32_t b0, b1;
    LcLz4Seq* seq[2];
    uint32_t nseq[2];
};

// match i of the block: position p, distance d, length ml
LC_HD void lc_zstd_match(const LcZstdBlk& b, uint32_t i, uint32_t& p, uint32_t& d, uint32_t& ml) {
    const uint32_t c = i >= b.nseq[0];
    const LcLz4Seq q = b.seq[c][i - (c ? b.nseq[0] : 0u)];
    p = b.b0 + c * LC_LZ4_CHUNK + (q.a & 0xFFFFu);
    d = q.a >> 16;
    ml = q.b;
}
// literal i of the block (l0 = literals of the first chunk)
LC_HD uint8_t lc_zstd_lit(const LcZstdBlk& b, uint32_t l0, uint32_t i) {
    return i < l0 ? reinterpret_cast<const uint8_t*>(b.seq[0] + b.nseq[0])[i]
                  : reinterpret_cast<const uint8_t*>(b.seq[1] + b.nseq[1])[i - l0];
}

// Literals section header of a Raw / RLE (mode) or Huffman section of r literals (c = compressed size)
LC_HD uint32_t lc_zstd_lhdr(uint32_t mode, uint32_t r, uint32_t c) {
    if (mode != LC_ZSTD_HUF)
        return r < 32 ? 1u : r < 4096 ? 2u : 3u;
    return r < 1024 && c < 1024 ? 3u : r < 16384 && c < 16384 ? 4u : 5u;
}
LC_HD void lc_zstd_put_lhdr(uint8_t* o, uint32_t mode, uint32_t r, uint32_t c) {
    const uint32_t h = lc_zstd_lhdr(mode, r, c);
    uint64_t v;
    if (mode != LC_ZSTD_HUF)
        v = h == 1 ? mode | r << 3 : h == 2 ? mode | 1u << 2 | r << 4 : mode | 3u << 2 | r << 4;
    else
        v = h == 3 ? mode | 1u << 2 | r << 4 | (uint64_t)c << 14
            : h == 4 ? mode | 2u << 2 | r << 4 | (uint64_t)c << 18
                     : mode | 3u << 2 | r << 4 | (uint64_t)c << 22;
    for (uint32_t j = 0; j < h; ++j)
        o[j] = (uint8_t)(v >> (8 * j));
}

// One Huffman stream of literals [a, e) of the block at o: the literals from the last to the first, each code at the
// bit offset its lanes find by a prefix sum, then the closing 1 bit.
LC_HD void lc_zstd_huf_stream(const LcZstdBlk& b, uint32_t l0, uint32_t a, uint32_t e, uint8_t* o, LcZstdWarp& w,
                              uint32_t lane, uint32_t W) {
    uint32_t pos = 0, base = 0; // bits written; bit of w.st[0] (a multiple of 32)
    LC_LANES(l) {
        for (uint32_t j = l; j < 16; j += W)
            w.st[j] = 0;
    }
    LC_WARP_SYNC();
    while (e > a) {
        const uint32_t cnt = e - a < W ? e - a : W;
        LC_LANES(l) {
            const uint32_t ch = l < cnt ? lc_zstd_lit(b, l0, e - 1 - l) : 0u;
            w.u[l] = ch;
            w.v[l] = l < cnt ? w.len[ch] : 0u;
        }
        LC_WARP_SYNC();
        const uint32_t tot = lc_warp_exscan(w.v, lane, W);
        LC_WARP_SYNC();
        LC_LANES(l) {
            if (l < cnt) {
                const uint32_t P = pos - base + w.v[l], ch = w.u[l], c = w.code[ch];
                lc_or32(&w.st[P >> 5], c << (P & 31));
                if ((P & 31) + w.len[ch] > 32)
                    lc_or32(&w.st[(P >> 5) + 1], c >> (32 - (P & 31)));
            }
        }
        LC_WARP_SYNC();
        pos += tot;
        e -= cnt;
        const uint32_t nw = (pos - base) >> 5; // complete words
        LC_LANES(l) {
            for (uint32_t j = l; j < 4 * nw; j += W)
                o[(base >> 3) + j] = (uint8_t)(w.st[j >> 2] >> (8 * (j & 3)));
        }
        const uint32_t carry = w.st[nw];
        LC_WARP_SYNC();
        LC_LANES(l) {
            for (uint32_t j = l; j < 16; j += W)
                w.st[j] = j ? 0u : carry;
        }
        LC_WARP_SYNC();
        base += nw << 5;
    }
    if (lane == 0)
        w.st[(pos - base) >> 5] |= 1u << ((pos - base) & 31);
    LC_WARP_SYNC();
    const uint32_t nbytes = (pos + 8) >> 3;
    LC_LANES(l) {
        for (uint32_t j = (base >> 3) + l; j < nbytes; j += W)
            o[j] = (uint8_t)(w.st[(j - (base >> 3)) >> 2] >> (8 * (j & 3)));
    }
    LC_WARP_SYNC();
}

// One lane: the sequences section of the block's ns matches at b.o[n, cap) (b.n = its start).
LC_HD void lc_zstd_sequences(const LcZstdBlk& b, uint32_t ns, const LcZstdWarp& w, LcBitW& bw) {
    if (ns < 128) {
        lc_bw_put(bw, ns, 8);
    } else if (ns < 0x7F00) {
        lc_bw_put(bw, (ns >> 8) + 128, 8);
        lc_bw_put(bw, ns & 0xFF, 8);
    } else {
        lc_bw_put(bw, 255, 8);
        lc_bw_put(bw, ns - 0x7F00, 16);
    }
    if (!ns)
        return;
    lc_bw_put(bw, 0, 8); // Symbol_Compression_Modes: predefined LL, OF and ML
    uint32_t sll = 0, sof = 0, sml = 0, p, d, ml;
    lc_zstd_match(b, ns - 1, p, d, ml);
    for (uint32_t i = ns; i-- > 0;) {
        uint32_t pp = b.b0, pd = 0, pml = 0;
        if (i) {
            lc_zstd_match(b, i - 1, pp, pd, pml);
            pp += pml;
        }
        const uint32_t ll = p - pp, mb = ml - 3, ov = d + 3;
        const uint32_t llc = lc_zstd_llc(ll), mlc = lc_zstd_mlc(mb), ofc = lc_hi_bit(ov);
        if (i + 1 == ns) {
            sll = lc_fse_init(w.ll, llc);
            sof = lc_fse_init(w.of, ofc);
            sml = lc_fse_init(w.ml, mlc);
        } else {
            sof = lc_fse_enc(w.of, sof, ofc, bw);
            sml = lc_fse_enc(w.ml, sml, mlc, bw);
            sll = lc_fse_enc(w.ll, sll, llc, bw);
        }
        lc_bw_put(bw, ll - lc_zstd_llbase(llc), lc_zstd_llbits(llc));
        lc_bw_put(bw, mb - lc_zstd_mlbase(mlc), lc_zstd_mlbits(mlc));
        lc_bw_put(bw, ov - (1u << ofc), ofc);
        if (i) {
            p = pp - pml;
            d = pd;
            ml = pml;
        }
    }
    lc_bw_put(bw, sml, 6);
    lc_bw_put(bw, sof, 5);
    lc_bw_put(bw, sll, 6);
    lc_bw_close(bw);
}

// Block pass: the compressed body of block b at o[0, b.b1 - b.b0) when it is smaller than the block's bytes; returns
// its size, or 0 for a Raw block (o then holds scratch).
LC_HD uint32_t lc_zstd_block(const LcZstdBlk& b, uint8_t* o, LcZstdWarp& w, uint32_t lane, uint32_t W) {
    const uint32_t raw = b.b1 - b.b0;
    if (raw == 0)
        return 0;
    if (lane == 0) {
        lc_fse_build(0, nullptr, 36, 6, w.ll);
        lc_fse_build(1, nullptr, 53, 6, w.ml);
        lc_fse_build(2, nullptr, 29, 5, w.of);
    }
    LC_LANES(l) {
        for (uint32_t i = l; i < 256; i += W)
            w.hist[i] = 0;
    }
    LC_WARP_SYNC();
    // 1. each chunk's literals behind its matches, W positions at a time, and their histogram
    uint32_t nlit[2] = {0, 0};
    for (uint32_t c = 0; c < 2 && b.seq[c]; ++c) {
        const uint32_t c0 = b.b0 + c * LC_LZ4_CHUNK, c1 = b.b1 - c0 < LC_LZ4_CHUNK ? b.b1 : c0 + LC_LZ4_CHUNK;
        const LcLz4Seq* q = b.seq[c];
        uint8_t* lit = reinterpret_cast<uint8_t*>(b.seq[c] + b.nseq[c]);
        uint32_t m = 0, k = 0; // matches that end before x, literals before x
        for (uint32_t x = c0; x < c1; x += W) {
            const uint32_t x1 = c1 - x < W ? c1 : x + W;
            LC_LANES(l) { // lane l: the coverage of [x, x1) by match m + l, and whether it ends there
                uint32_t cov = 0, end = 0;
                if (m + l < b.nseq[c]) {
                    const LcLz4Seq z = q[m + l];
                    const uint32_t ms = c0 + (z.a & 0xFFFFu), me = ms + z.b;
                    const uint32_t lo = ms > x ? ms : x, hi = me < x1 ? me : x1;
                    cov = lo < hi ? lc_bits(hi - lo) << (lo - x) : 0u;
                    end = me <= x1;
                }
                w.v[l] = cov;
                w.u[l] = end;
            }
            LC_WARP_SYNC();
            const uint32_t litm = ~lc_warp_or(w.v, lane, W) & lc_bits(x1 - x);
            const uint32_t ends = lc_lz4_ballot(w.u, lane, W);
            LC_WARP_SYNC();
            LC_LANES(l) {
                if ((litm >> l) & 1) {
                    const uint8_t ch = b.s[x + l];
                    lit[k + lc_popc(litm & lc_bits(l))] = ch;
                    lc_add32(&w.hist[ch], 1);
                }
            }
            k += lc_popc(litm);
            m += lc_popc(ends);
        }
        nlit[c] = k;
    }
    LC_WARP_SYNC();
    const uint32_t l0 = nlit[0], R = nlit[0] + nlit[1];
    // 2. the bytes present by increasing (count, byte), for the Huffman tree
    if (R >= LC_ZSTD_MIN_HUF) {
        LC_LANES(l) {
            for (uint32_t s = l; s < 256; s += W) {
                const uint32_t cs = w.hist[s];
                if (!cs)
                    continue;
                uint32_t r = 0;
                for (uint32_t t = 0; t < 256; ++t)
                    r += w.hist[t] && (w.hist[t] < cs || (w.hist[t] == cs && t < s));
                w.order[r] = (uint8_t)s;
            }
        }
        LC_WARP_SYNC();
    }
    // 3. one lane: the literal mode, the code and its description
    if (lane == 0) {
        uint32_t m = 0, maxs = 0;
        for (uint32_t s = 0; s < 256; ++s) {
            w.len[s] = 0;
            if (w.hist[s]) {
                ++m;
                maxs = s;
            }
        }
        uint32_t mode = m == 1 ? LC_ZSTD_RLE : LC_ZSTD_RAW, dl = 0;
        if (m >= 2 && R >= LC_ZSTD_MIN_HUF) {
            dl = lc_zstd_huf_table(w, lc_zstd_huf_lengths(w, m), maxs);
            mode = dl ? LC_ZSTD_HUF : mode;
        }
        w.res[0] = mode;
        w.res[1] = dl;
        w.res[2] = maxs;
    }
    LC_WARP_SYNC();
    uint32_t mode = w.res[0];
    const uint32_t dl = w.res[1], q4 = (R + 3) / 4;
    uint32_t sbytes[4] = {0, 0, 0, 0}, csize = 0;
    if (mode == LC_ZSTD_HUF) {
        csize = dl + 6;
        for (uint32_t k = 0; k < 4; ++k) {
            const uint32_t a = k * q4, e = k == 3 ? R : a + q4;
            LC_LANES(l) {
                uint32_t bits = 0;
                for (uint32_t i = a + l; i < e; i += W)
                    bits += w.len[lc_zstd_lit(b, l0, i)];
                w.v[l] = bits;
            }
            LC_WARP_SYNC();
            sbytes[k] = lc_warp_exscan(w.v, lane, W) / 8 + 1;
            LC_WARP_SYNC();
            csize += sbytes[k];
        }
        if (lc_zstd_lhdr(mode, R, csize) + csize >= lc_zstd_lhdr(LC_ZSTD_RAW, R, 0) + R)
            mode = LC_ZSTD_RAW;
    }
    const uint32_t lh = lc_zstd_lhdr(mode, R, csize);
    const uint32_t lsize = lh + (mode == LC_ZSTD_HUF ? csize : mode == LC_ZSTD_RLE ? 1 : R);
    if (lsize + 1 >= raw) // the sequences section takes at least one byte
        return 0;
    // 4. the literals section
    if (lane == 0) {
        lc_zstd_put_lhdr(o, mode, R, csize);
        if (mode == LC_ZSTD_RLE)
            o[lh] = (uint8_t)w.res[2];
        if (mode == LC_ZSTD_HUF)
            for (uint32_t k = 0; k < 3; ++k) {
                o[lh + dl + 2 * k] = (uint8_t)sbytes[k];
                o[lh + dl + 2 * k + 1] = (uint8_t)(sbytes[k] >> 8);
            }
    }
    if (mode == LC_ZSTD_RAW) {
        LC_LANES(l) {
            for (uint32_t i = l; i < R; i += W)
                o[lh + i] = lc_zstd_lit(b, l0, i);
        }
    } else if (mode == LC_ZSTD_HUF) {
        LC_LANES(l) {
            for (uint32_t j = l; j < dl; j += W)
                o[lh + j] = w.wdesc[j];
        }
        uint8_t* so = o + lh + dl + 6;
        for (uint32_t k = 0; k < 4; ++k) {
            lc_zstd_huf_stream(b, l0, k * q4, k == 3 ? R : (k + 1) * q4, so, w, lane, W);
            so += sbytes[k];
        }
    }
    LC_WARP_SYNC();
    // 5. one lane: the sequences section, abandoned when the body reaches the block's size
    if (lane == 0) {
        LcBitW bw{o, lsize, raw - 1, 0, 0};
        lc_zstd_sequences(b, b.nseq[0] + b.nseq[1], w, bw);
        w.res[3] = bw.n <= bw.cap ? bw.n : 0u;
    }
    LC_WARP_SYNC();
    return w.res[3];
}

// frame header of an n-byte segment at o[0, lc_zstd_hdr(n))
LC_HD void lc_zstd_put_hdr(uint32_t n, uint8_t* o) {
    const uint32_t f = lc_zstd_fcs_bytes(n), v = f == 2 ? n - 256 : n;
    o[0] = 0x28;
    o[1] = 0xB5;
    o[2] = 0x2F;
    o[3] = 0xFD;
    o[4] = (uint8_t)((f == 1 ? 0u : f == 2 ? 1u : 2u) << 6 | 0x20);
    for (uint32_t j = 0; j < f; ++j)
        o[5 + j] = (uint8_t)(v >> (8 * j));
}

// bytes of block j of an n-byte segment in its frame (the frame header with block 0), body = lc_zstd_block's result
LC_HD uint32_t lc_zstd_emit_size(uint32_t n, uint32_t j, uint32_t body) {
    const uint32_t b0 = j * LC_ZSTD_BLOCK, b1 = n - b0 < LC_ZSTD_BLOCK ? n : b0 + LC_ZSTD_BLOCK;
    return (j ? 0u : lc_zstd_hdr(n)) + 3 + (body ? body : b1 - b0);
}

// Emit pass of block j of the segment s[0, n) at o: (block 0) the frame header, the block header, then the body from
// the block's slot or (Raw) the segment.
LC_HD void lc_zstd_emit_block(const uint8_t* s, uint32_t n, uint32_t j, const uint8_t* slot, uint32_t body, uint8_t* o,
                              uint32_t lane, uint32_t W) {
    const uint32_t b0 = j * LC_ZSTD_BLOCK, b1 = n - b0 < LC_ZSTD_BLOCK ? n : b0 + LC_ZSTD_BLOCK;
    if (!j) {
        if (lane == 0)
            lc_zstd_put_hdr(n, o);
        o += lc_zstd_hdr(n);
    }
    const uint32_t size = body ? body : b1 - b0, h = (b1 == n) | (body ? 2u : 0u) << 1 | size << 3;
    if (lane == 0) {
        o[0] = (uint8_t)h;
        o[1] = (uint8_t)(h >> 8);
        o[2] = (uint8_t)(h >> 16);
    }
    const uint8_t* src = body ? slot : s + b0;
    LC_LANES(l) {
        for (uint32_t i = l; i < size; i += W)
            o[3 + i] = src[i];
    }
}

// ================================================================================================ timestamp parse
// ProcessorParseTimestampNative (ProcessorParseTimestampNative.cpp:100-235) over Strptime (TimeUtil.cpp:112-160) and
// strptime_ns (Strptime.cpp), in two passes:
//   - lc_ts_full: one lane per event runs the compiled format over the value: the full parse's outcome, Strptime's
//     tv_sec (mktime of the partially filled tm, written even when the parse fails), tv_nsec and the cache key length.
//   - lc_ts_resolve: one warp per group applies ParseLogTime's second-level cache, a sequential state reset at the start
//     of every group, 32 events per step; then the verdict of ProcessEvent.
// The format is compiled on the host (lc_ts_compile) into a short program of LcTsOp.  The strptime_ns directives are
// run as written for the C locale; %c, %x and %X (the "locale's format" conversions) are refused.  %Z with a zone
// name other than GMT / UTC consumes nothing, as strptime_ns does on Linux.
// mktime is restated over a per-year table of the process zone's (standard, daylight) offsets, probed with mktime on
// the host (lc_ts_probe_zone): glibc's mktime honours tm_isdst = 0 / 1 with the zone's standard / daylight offset.
// Bounds: a value is read over [off, off + len) followed by NUL bytes; the reference hands strptime a StringView that
// need not be NUL-terminated, so the two agree whenever the value is terminated.
#define LC_TS_MAX_OPS 96
#define LC_TS_Y0 1800
#define LC_TS_NYEARS 500
#define LC_TS_NO_KEY 0xFFFFFFFFu  // ev_len of an event without SourceKey
#define LC_TS_KFAIL 0xFFFFFFFFu   // LcTsFull::klen of a failed full parse
#define LC_TS_MIN_YEAR (-2147483647 - 1)

#define LC_TS_ST_OK 0
#define LC_TS_ST_NOT_FOUND 1
#define LC_TS_ST_FAILED 2
#define LC_TS_ST_DISCARDED 3

// counters[5]: ProcessorParseTimestampNative's metrics in this order
#define LC_TS_C_KEY_NOT_FOUND 0
#define LC_TS_C_OUT_FAILED 1
#define LC_TS_C_HISTORY_FAILURE 2
#define LC_TS_C_DISCARDED 3
#define LC_TS_C_OUT_SUCCESSFUL 4

enum LcTsOpCode : uint8_t {
    LC_TSO_WS,       // white space in the format, %n, %t: eat isspace
    LC_TSO_LIT,      // literal byte (also %%)
    LC_TSO_FAIL,     // return NULL (unknown conversion, %s inside a format, an alternative modifier not allowed)
    LC_TSO_RESET_NS, // start of %D %F %R %r %T: the recursive strptime_ns call zeroes the nanoseconds
    LC_TSO_WDAY_NAME, LC_TSO_MON_NAME, LC_TSO_CENTURY, LC_TSO_MDAY, LC_TSO_NSEC, LC_TSO_HOUR24, LC_TSO_HOUR12,
    LC_TSO_YDAY, LC_TSO_MIN, LC_TSO_MON, LC_TSO_AMPM, LC_TSO_SEC, LC_TSO_WEEK, LC_TSO_WDAY0, LC_TSO_WDAY1,
    LC_TSO_YEAR2_ISO, LC_TSO_YEAR_ISO, LC_TSO_YEAR, LC_TSO_YEAR2, LC_TSO_ZONE_NAME, LC_TSO_ZONE_OFF,
};
#define LC_TSF_FAIL_AFTER 1u // the conversion runs, then the directive's LEGAL_ALT returns NULL
#define LC_TSF_INNER 2u      // %y inside %D: the recursive call's own split_year

struct LcTsOp {
    uint8_t code, flags, ch, pad;
};

#define LC_TSM_HAVE_F 1u  // strstr(format, "%f")
#define LC_TSM_END_F 2u   // ... and it is the last two bytes
#define LC_TSM_EPOCH 4u   // format == "%s"
#define LC_TSM_F_ONLY 8u  // format == "%f": Strptime returns before mktime

struct LcTsConf {
    LcTsOp ops[LC_TS_MAX_OPS];
    uint32_t nops, mode;
    int32_t source_year;  // SourceYear (-1 unset, 0 deduce from now, > 0 that year)
    int32_t adjust;       // mLogTimeZoneOffsetSecond, subtracted after a successful full parse
    int32_t std_off[LC_TS_NYEARS], dst_off[LC_TS_NYEARS]; // seconds east of UTC, year LC_TS_Y0 + k
};

struct LcTsNow {  // what a call reads of "now"
    int64_t now;  // time(NULL)
    int32_t year, mon, mday; // localtime_r(now): tm_year, tm_mon, tm_mday (DeduceYear)
    int32_t discard_interval; // ilogtail_discard_interval, < 0 = no history discard (flag off, one-time pipeline)
};

// Host: SourceFormat -> program.  Returns 0, or -1 with *err set for a directive the program cannot run.
inline int lc_ts_compile(const char* fmt, size_t len, LcTsConf& c, const char** err) {
    c.nops = 0;
    c.mode = 0;
    if (memchr(fmt, 0, len)) {
        *err = "SourceFormat: a NUL byte inside the format";
        return -1;
    }
    const size_t flen = len;
    for (size_t i = 0; i + 1 < flen; ++i)
        if (fmt[i] == '%' && fmt[i + 1] == 'f') {
            c.mode |= LC_TSM_HAVE_F | (i + 2 == flen ? LC_TSM_END_F : 0u);
            break;
        }
    if (flen == 2 && fmt[0] == '%' && fmt[1] == 's') {
        c.mode |= LC_TSM_EPOCH;
        return 0;
    }
    if (flen == 2 && fmt[0] == '%' && fmt[1] == 'f')
        c.mode |= LC_TSM_F_ONLY;
    auto emit = [&](uint8_t code, uint8_t flags = 0, uint8_t ch = 0) -> bool {
        if (c.nops >= LC_TS_MAX_OPS)
            return false;
        c.ops[c.nops++] = LcTsOp{code, flags, ch, 0};
        return true;
    };
    auto inner = [&](const char* s) -> bool { // the recursive call of %D %F %R %r %T
        bool ok = emit(LC_TSO_RESET_NS);
        for (; *s && ok; ++s) {
            if (*s == ' ')
                ok = emit(LC_TSO_WS);
            else if (*s != '%')
                ok = emit(LC_TSO_LIT, 0, (uint8_t)*s);
            else {
                const char d = *++s;
                const uint8_t code = d == 'm'   ? LC_TSO_MON
                                     : d == 'd' ? LC_TSO_MDAY
                                     : d == 'y' ? LC_TSO_YEAR2
                                     : d == 'Y' ? LC_TSO_YEAR
                                     : d == 'H' ? LC_TSO_HOUR24
                                     : d == 'I' ? LC_TSO_HOUR12
                                     : d == 'M' ? LC_TSO_MIN
                                     : d == 'S' ? LC_TSO_SEC
                                                : LC_TSO_AMPM;
                ok = emit(code, d == 'y' ? LC_TSF_INNER : 0u);
            }
        }
        return ok;
    };
    size_t i = 0;
    while (i < flen) {
        const unsigned char ch = (unsigned char)fmt[i++];
        if (ch == ' ' || (ch >= 9 && ch <= 13)) {
            if (!emit(LC_TSO_WS))
                goto too_long;
            continue;
        }
        if (ch != '%') {
            if (!emit(LC_TSO_LIT, 0, ch))
                goto too_long;
            continue;
        }
        unsigned alt = 0;
        for (;;) {
            const char d = i < flen ? fmt[i++] : '\0';
            // LEGAL_ALT(x) before the conversion fails -> FAIL; after it -> FAIL_AFTER
            auto conv = [&](uint8_t code, unsigned legal) -> bool {
                return emit(code, (alt & ~legal) ? LC_TSF_FAIL_AFTER : 0u);
            };
            bool ok = true;
            switch (d) {
            case '%':
                ok = alt ? emit(LC_TSO_FAIL) : emit(LC_TSO_LIT, 0, '%');
                break;
            case 'E':
            case 'O':
                if (alt) {
                    ok = emit(LC_TSO_FAIL);
                    break;
                }
                alt = d == 'E' ? 1u : 2u;
                continue;
            case 'c':
            case 'x':
            case 'X':
                *err = "SourceFormat: %c, %x and %X (the locale's formats) are not supported on the device";
                return -1;
            case 'D': ok = alt ? emit(LC_TSO_FAIL) : inner("%m/%d/%y"); break;
            case 'F': ok = alt ? emit(LC_TSO_FAIL) : inner("%Y-%m-%d"); break;
            case 'R': ok = alt ? emit(LC_TSO_FAIL) : inner("%H:%M"); break;
            case 'r': ok = alt ? emit(LC_TSO_FAIL) : inner("%I:%M:%S %p"); break;
            case 'T': ok = alt ? emit(LC_TSO_FAIL) : inner("%H:%M:%S"); break;
            case 'A': case 'a': ok = conv(LC_TSO_WDAY_NAME, 0); break;
            case 'B': case 'b': case 'h': ok = conv(LC_TSO_MON_NAME, 0); break;
            case 'C': ok = conv(LC_TSO_CENTURY, 1); break;
            case 'd': case 'e': ok = conv(LC_TSO_MDAY, 2); break;
            case 'f': ok = conv(LC_TSO_NSEC, 2); break;
            case 'k': ok = alt ? emit(LC_TSO_FAIL) : conv(LC_TSO_HOUR24, 2); break;
            case 'H': ok = conv(LC_TSO_HOUR24, 2); break;
            case 'l': ok = alt ? emit(LC_TSO_FAIL) : conv(LC_TSO_HOUR12, 2); break;
            case 'I': ok = conv(LC_TSO_HOUR12, 2); break;
            case 'j': ok = conv(LC_TSO_YDAY, 0); break;
            case 'M': ok = conv(LC_TSO_MIN, 2); break;
            case 'm': ok = conv(LC_TSO_MON, 2); break;
            case 'p': ok = conv(LC_TSO_AMPM, 0); break;
            case 'S': ok = conv(LC_TSO_SEC, 2); break;
            case 'U': case 'W': ok = conv(LC_TSO_WEEK, 2); break;
            case 'V': ok = emit(LC_TSO_WEEK); break;
            case 'w': ok = conv(LC_TSO_WDAY0, 2); break;
            case 'u': ok = conv(LC_TSO_WDAY1, 2); break;
            case 'g': ok = emit(LC_TSO_YEAR2_ISO); break;
            case 'G': ok = emit(LC_TSO_YEAR_ISO); break;
            case 'Y': ok = conv(LC_TSO_YEAR, 1); break;
            case 'y': ok = emit(LC_TSO_YEAR2); break;
            case 'Z': ok = emit(LC_TSO_ZONE_NAME); break;
            case 'z': ok = emit(LC_TSO_ZONE_OFF); break;
            case 'n': case 't': ok = alt ? emit(LC_TSO_FAIL) : emit(LC_TSO_WS); break;
            default: ok = emit(LC_TSO_FAIL); break; // unknown conversion, %s inside a format, a trailing '%'
            }
            if (!ok)
                goto too_long;
            if (d == '\0')
                return 0; // strptime_ns returns NULL before it reads past the format's end
            break;
        }
    }
    return 0;
too_long:
    *err = "SourceFormat: more directives than the device program holds";
    return -1;
}

LC_HD int64_t lc_ts_days_from_civil(int64_t y, uint32_t m, uint32_t d) { // proleptic Gregorian, m 1..12
    y -= m <= 2;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const uint32_t yoe = (uint32_t)(y - era * 400);
    const uint32_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
    const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}

LC_HD int64_t lc_ts_year_of_days(int64_t z) { // civil year of day z since 1970-01-01
    z += 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const uint32_t doe = (uint32_t)(z - era * 146097);
    const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const uint32_t mp = (5 * doy + 2) / 153;
    return (int64_t)yoe + era * 400 + (mp >= 10);
}

struct LcTsTm {
    int sec, min, hour, mday, mon, year, isdst;
};

// mktime of a tm whose fields are in the ranges the parser leaves (mon 0..11, mday 0..31, sec 0..61).  glibc computes
// in 64 bits, so a year that was never set (tm_year = INT_MIN) gives a time far in the past, and -1 only when the
// normalised date leaves the range of tm_year.
LC_HD int64_t lc_ts_mktime(const LcTsConf& c, const LcTsTm& t) {
    const int64_t days = lc_ts_days_from_civil((int64_t)t.year + 1900, (uint32_t)t.mon + 1, 1) + t.mday - 1;
    const int64_t local = days * 86400 + t.hour * 3600 + t.min * 60 + t.sec;
    const int64_t d = local >= 0 ? local / 86400 : (local - 86399) / 86400;
    const int64_t y = lc_ts_year_of_days(d);
    if (y - 1900 < (int64_t)LC_TS_MIN_YEAR)
        return -1; // the normalised tm_year does not fit an int (a never-set year with tm_mday 0): EOVERFLOW
    int64_t k = y - LC_TS_Y0;
    k = k < 0 ? 0 : (k >= LC_TS_NYEARS ? LC_TS_NYEARS - 1 : k);
    return local - (t.isdst ? c.dst_off[k] : c.std_off[k]);
}

struct LcTsIn { // the value: bytes past len read as NUL
    const uint8_t* s;
    uint32_t n;
    LC_HD uint32_t at(uint32_t p) const { return p < n ? s[p] : 0u; }
};

LC_HD bool lc_ts_space(uint32_t ch) { return ch == ' ' || (ch >= 9 && ch <= 13); }
LC_HD bool lc_ts_digit(uint32_t ch) { return ch - '0' < 10u; }

// conv_num: false = NULL (dest untouched)
LC_HD bool lc_ts_num(const LcTsIn& in, uint32_t& p, int& dest, uint32_t llim, uint32_t ulim) {
    uint32_t ch = in.at(p), result = 0, rulim = ulim;
    if (!lc_ts_digit(ch))
        return false;
    do {
        result = result * 10 + (ch - '0');
        rulim /= 10;
        ch = in.at(++p);
    } while (result * 10 <= ulim && rulim && lc_ts_digit(ch));
    if (result < llim || result > ulim)
        return false;
    dest = (int)result;
    return true;
}

// conv_nanosecond: unsigned 32-bit arithmetic, as the reference's
LC_HD bool lc_ts_nsec(const LcTsIn& in, uint32_t& p, uint32_t& dest, int& nlen) {
    uint32_t ch = in.at(p), result = 0;
    if (!lc_ts_digit(ch))
        return false;
    const uint32_t start = p;
    int digits = 0;
    do {
        result = result * 10 + (ch - '0');
        ++digits;
        ch = in.at(++p);
    } while (lc_ts_digit(ch));
    for (int i = 0; i < 9 - digits; i++)
        result *= 10;
    dest = result;
    nlen = (int)(p - start);
    return true;
}

LC_HD const char* lc_ts_name(uint32_t table, uint32_t i) {
    switch (table * 16 + i) {
    case 0: return "Sunday"; case 1: return "Monday"; case 2: return "Tuesday"; case 3: return "Wednesday";
    case 4: return "Thursday"; case 5: return "Friday"; case 6: return "Saturday";
    case 16: return "Sun"; case 17: return "Mon"; case 18: return "Tue"; case 19: return "Wed"; case 20: return "Thu";
    case 21: return "Fri"; case 22: return "Sat";
    case 32: return "January"; case 33: return "February"; case 34: return "March"; case 35: return "April";
    case 36: return "May"; case 37: return "June"; case 38: return "July"; case 39: return "August";
    case 40: return "September"; case 41: return "October"; case 42: return "November"; case 43: return "December";
    case 48: return "Jan"; case 49: return "Feb"; case 50: return "Mar"; case 51: return "Apr"; case 52: return "May";
    case 53: return "Jun"; case 54: return "Jul"; case 55: return "Aug"; case 56: return "Sep"; case 57: return "Oct";
    case 58: return "Nov"; case 59: return "Dec";
    case 64: return "AM"; case 65: return "PM";
    case 80: return "EST"; case 81: return "CST"; case 82: return "MST"; case 83: return "PST";
    case 96: return "EDT"; case 97: return "CDT"; case 98: return "MDT"; case 99: return "PDT";
    case 112: return "GMT"; case 113: return "UTC";
    default: return "";
    }
}

LC_HD uint32_t lc_ts_lower(uint32_t ch) { return ch - 'A' < 26u ? ch + 32 : ch; }

// strncasecmp(name, bp, strlen(name)) == 0
LC_HD bool lc_ts_name_at(const LcTsIn& in, uint32_t p, const char* name, uint32_t& len) {
    uint32_t k = 0;
    for (; name[k]; ++k)
        if (lc_ts_lower((uint8_t)name[k]) != lc_ts_lower(in.at(p + k)))
            return false;
    len = k;
    return true;
}

// find_string over table `full` (and then `abbr` when abbr >= 0) of c names
LC_HD bool lc_ts_find(const LcTsIn& in, uint32_t& p, int& tgt, uint32_t full, int abbr, uint32_t c) {
    for (int t = (int)full; t >= 0; t = t == (int)full ? abbr : -1) {
        for (uint32_t i = 0; i < c; i++) {
            uint32_t len;
            if (lc_ts_name_at(in, p, lc_ts_name((uint32_t)t, i), len)) {
                tgt = (int)i;
                p += len;
                return true;
            }
        }
    }
    return false;
}

struct LcTsFull { // per-event result of the full parse
    int64_t raw;   // Strptime's tv_sec (for a "%f" format: unchanged, 0 here; see lc_ts_resolve)
    uint32_t nsec; // tv_nsec of a successful parse
    uint32_t klen; // cache key length of a successful parse, LC_TS_KFAIL when it failed
};

// %s (Strptime.cpp:85-112): strtoll, at most 10 digits of seconds, the following digits as %f.  end: where strtoll
// stopped (0 when it read no digit), which strptime_ns returns.
LC_HD bool lc_ts_epoch_end(const LcTsIn& in, int64_t& secs, uint32_t& nsec, int& nlen, uint32_t& end) {
    uint32_t p = 0;
    while (lc_ts_space(in.at(p)))
        ++p;
    const bool neg = in.at(p) == '-';
    if (in.at(p) == '-' || in.at(p) == '+')
        ++p;
    uint64_t acc = 0;
    bool over = false;
    const uint64_t lim = neg ? 9223372036854775808ull : 9223372036854775807ull;
    while (lc_ts_digit(in.at(p))) {
        const uint32_t dg = in.at(p++) - '0';
        if (!over && acc > (lim - dg) / 10)
            over = true;
        if (!over)
            acc = acc * 10 + dg;
    }
    if (over)
        acc = lim;
    end = lc_ts_digit(in.at(p - 1)) ? p : 0u;
    int64_t n = neg ? (int64_t)(0 - acc) : (int64_t)acc;
    uint32_t blen = n < 0 ? 1 : 0; // std::to_string(n).length()
    for (uint64_t a = acc;; a /= 10) {
        ++blen;
        if (a < 10)
            break;
    }
    const uint32_t slen = blen >= 10 ? 10 : blen;
    for (uint32_t i = 0; i < blen - slen; ++i)
        n /= 10;
    if (n == 0)
        return false;
    secs = n;
    nsec = 0;
    nlen = 0;
    uint32_t q = slen;
    uint32_t ns;
    int nl;
    if (lc_ts_nsec(in, q, ns, nl)) {
        nsec = ns;
        nlen = nl;
    }
    return true;
}

LC_HD bool lc_ts_epoch(const LcTsIn& in, int64_t& secs, uint32_t& nsec, int& nlen) {
    uint32_t end;
    return lc_ts_epoch_end(in, secs, nsec, nlen, end);
}

// Strptime(value, SourceFormat, &logTime, nanosecondLength, SourceYear) with logTime = {0, 0}
LC_HD LcTsFull lc_ts_full(const LcTsConf& c, const LcTsNow& now, const uint8_t* s, uint32_t n) {
    const LcTsIn in{s, n};
    LcTsTm tm{0, 0, 0, 0, 0, LC_TS_MIN_YEAR, 0};
    uint32_t nsec = 0;
    int nlen = -1;
    bool ok = true;
    int64_t epoch = 0;
    bool have_epoch = false;
    if (c.mode & LC_TSM_EPOCH) {
        ok = lc_ts_epoch(in, epoch, nsec, nlen);
        have_epoch = ok; // localtime_r then mktime gives the seconds back
    } else {
        uint32_t p = 0;
        int split = 0;
        for (uint32_t k = 0; k < c.nops && ok; ++k) {
            const LcTsOp op = c.ops[k];
            int i = 0;
            bool r = true; // bp != NULL after the conversion
            switch (op.code) {
            case LC_TSO_WS:
                while (lc_ts_space(in.at(p)))
                    ++p;
                break;
            case LC_TSO_LIT:
                r = in.at(p++) == op.ch;
                break;
            case LC_TSO_FAIL: r = false; break;
            case LC_TSO_RESET_NS: nsec = 0; break;
            case LC_TSO_WDAY_NAME: { int w; r = lc_ts_find(in, p, w, 0, 1, 7); break; }
            case LC_TSO_MON_NAME: r = lc_ts_find(in, p, tm.mon, 2, 3, 12); break;
            case LC_TSO_CENTURY:
                i = 20;
                r = lc_ts_num(in, p, i, 0, 99);
                i = i * 100 - 1900;
                if (split)
                    i += tm.year % 100;
                split = 1;
                tm.year = i;
                break;
            case LC_TSO_MDAY: r = lc_ts_num(in, p, tm.mday, 1, 31); break;
            case LC_TSO_NSEC: r = lc_ts_nsec(in, p, nsec, nlen); break;
            case LC_TSO_HOUR24: r = lc_ts_num(in, p, tm.hour, 0, 23); break;
            case LC_TSO_HOUR12:
                r = lc_ts_num(in, p, tm.hour, 1, 12);
                if (tm.hour == 12)
                    tm.hour = 0;
                break;
            case LC_TSO_YDAY: i = 1; r = lc_ts_num(in, p, i, 1, 366); break;
            case LC_TSO_MIN: r = lc_ts_num(in, p, tm.min, 0, 59); break;
            case LC_TSO_MON:
                i = 1;
                r = lc_ts_num(in, p, i, 1, 12);
                tm.mon = i - 1;
                break;
            case LC_TSO_AMPM:
                r = lc_ts_find(in, p, i, 4, -1, 2);
                if (tm.hour > 11) {
                    ok = false;
                    continue;
                }
                tm.hour += i * 12;
                break;
            case LC_TSO_SEC: r = lc_ts_num(in, p, tm.sec, 0, 61); break;
            case LC_TSO_WEEK: r = lc_ts_num(in, p, i, 0, 53); break;
            case LC_TSO_WDAY0: r = lc_ts_num(in, p, i, 0, 6); break;
            case LC_TSO_WDAY1: i = 1; r = lc_ts_num(in, p, i, 1, 7); break;
            case LC_TSO_YEAR2_ISO: r = lc_ts_num(in, p, i, 0, 99); break;
            case LC_TSO_YEAR_ISO:
                do
                    ++p;
                while (lc_ts_digit(in.at(p)));
                break;
            case LC_TSO_YEAR:
                i = 1900;
                r = lc_ts_num(in, p, i, 0, 9999);
                tm.year = i - 1900;
                break;
            case LC_TSO_YEAR2:
                r = lc_ts_num(in, p, i, 0, 99);
                if (split && !(op.flags & LC_TSF_INNER))
                    i += (tm.year / 100) * 100;
                else {
                    if (!(op.flags & LC_TSF_INNER))
                        split = 1;
                    i = i <= 68 ? i + 2000 - 1900 : i + 1900 - 1900;
                }
                tm.year = i;
                break;
            case LC_TSO_ZONE_NAME: {
                uint32_t len;
                if (lc_ts_name_at(in, p, "GMT", len) || lc_ts_name_at(in, p, "UTC", len)) {
                    tm.isdst = 0;
                    p += 3;
                }
                break;
            }
            case LC_TSO_ZONE_OFF: {
                while (lc_ts_space(in.at(p)))
                    ++p;
                const uint32_t ch = in.at(p++);
                if (ch == 'G' || ch == 'U' || ch == 'Z') {
                    if ((ch == 'G' && in.at(p++) != 'M') || (ch != 'Z' && in.at(p++) != 'T')) {
                        ok = false;
                        continue;
                    }
                    tm.isdst = 0;
                    break;
                }
                if (ch != '+' && ch != '-') {
                    --p;
                    int z;
                    if (lc_ts_find(in, p, z, 5, -1, 4))
                        break;
                    if (lc_ts_find(in, p, z, 6, -1, 4)) {
                        tm.isdst = 1;
                        break;
                    }
                    const uint32_t b = in.at(p);
                    if ((b >= 'A' && b <= 'I') || (b >= 'L' && b <= 'Y')) {
                        ++p;
                        break;
                    }
                    ok = false;
                    continue;
                }
                int offs = 0, d = 0;
                while (d < 4) {
                    if (lc_ts_digit(in.at(p))) {
                        offs = offs * 10 + (int)(in.at(p++) - '0');
                        d++;
                        continue;
                    }
                    if (d == 2 && in.at(p) == ':') {
                        p++;
                        continue;
                    }
                    break;
                }
                if (d != 2 && (d != 4 || offs % 100 >= 60)) {
                    ok = false;
                    continue;
                }
                tm.isdst = 0;
                break;
            }
            }
            if (!r || (op.flags & LC_TSF_FAIL_AFTER))
                ok = false;
        }
    }
    LcTsFull f{0, nsec, ok ? (nlen < 0 ? n : n - (uint32_t)nlen) : LC_TS_KFAIL};
    if (c.mode & LC_TSM_F_ONLY)
        return f;
    if (have_epoch) {
        f.raw = epoch;
        return f;
    }
    if (c.source_year >= 0 && tm.year == LC_TS_MIN_YEAR) {
        if (c.source_year > 0)
            tm.year = c.source_year - 1900;
        else if (tm.mon == 0 && tm.mday == 1 && now.mon == 11 && now.mday == 31) // DeduceYear
            tm.year = now.year + 1;
        else if (tm.mon == 11 && tm.mday == 31 && now.mon == 0 && now.mday == 1)
            tm.year = now.year - 1;
        else
            tm.year = now.year;
    }
    f.raw = lc_ts_mktime(c, tm);
    return f;
}

LC_HD uint32_t lc_ts_popc(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popc(m);
#else
    return (uint32_t)__builtin_popcount(m);
#endif
}

// Where event i's value is: a dense (off, len) table (len LC_TS_NO_KEY = no SourceKey), or capture column k of a
// regex result (st != NULL: off / len point at column k of [n][pitch] tables; a row not parsed has no value).
struct LcTsSpans {
    const uint32_t* off;
    const uint32_t* len;
    const uint8_t* st;
    uint32_t pitch;
    LC_HD bool get(uint64_t i, uint32_t& o, uint32_t& l) const {
        if (st) {
            if (st[i] != 0)
                return false;
            o = off[i * pitch];
            l = len[i * pitch];
            return true;
        }
        l = len[i];
        if (l == LC_TS_NO_KEY)
            return false;
        o = off[i];
        return true;
    }
};

struct LcTsWarp { // per-warp scratch of the resolution pass (shared memory on the device)
    uint32_t v[32];   // per-lane ballot predicate
    uint32_t off[32]; // the step's values
    uint32_t len[32];
    uint32_t klen[32]; // LcTsFull of the step's events
    uint32_t fns[32];
    int64_t raw[32];
};

// IsPrefixString(value, key): false for an empty key
LC_HD bool lc_ts_prefix(const uint8_t* base, uint32_t a, uint32_t alen, uint32_t k, uint32_t klen) {
    if (klen == 0 || alen < klen)
        return false;
    for (uint32_t i = 0; i < klen; ++i)
        if (base[a + i] != base[k + i])
            return false;
    return true;
}

LC_HD uint32_t lc_ts_below(uint32_t l) { return l >= 32 ? 0xFFFFFFFFu : (1u << l) - 1u; }

// ParseLogTime's second-level cache and ProcessEvent's verdict over the events [e0, e1) of one group, W lanes,
// 32 events per step.  Each lane tests its value against the cache key the step starts with (hx) and against the key
// of the nearest earlier event of the step whose full parse succeeded (hp); the masks then tell which events miss
// (a miss with a successful full parse moves the cache), as far as the step can know them: it ends at the first
// event that hits a key set inside the step and would have to be compared with a key that is not its predecessor's.
// A hit inherits tv_sec from the last full parse of the group, successful or not.  cnt[5] += the counters.
LC_HD void lc_ts_resolve(const LcTsConf& c, const LcTsNow& now, const uint8_t* base, const LcTsSpans& sp, const LcTsFull* full,
                         uint64_t e0, uint64_t e1, int64_t* sec, uint32_t* nsec, uint8_t* status, uint64_t* cnt,
                         LcTsWarp& w, uint32_t lane, uint32_t W) {
    const bool cacheable = !(c.mode & LC_TSM_HAVE_F) || (c.mode & LC_TSM_END_F);
    bool have_key = false;
    uint32_t key_off = 0, key_len = 0;
    int64_t state = 0; // logTime.tv_sec
    for (uint64_t b = e0; b < e1;) {
        const uint32_t nv = e1 - b < W ? (uint32_t)(e1 - b) : W;
        LC_LANES(l) {
            uint32_t o = 0, ln = 0;
            const bool pres = l < nv && sp.get(b + l, o, ln);
            const LcTsFull f = pres ? full[b + l] : LcTsFull{0, 0, LC_TS_KFAIL};
            w.off[l] = o;
            w.len[l] = pres ? ln : LC_TS_NO_KEY;
            w.klen[l] = f.klen;
            w.fns[l] = f.nsec;
            w.raw[l] = f.raw;
        }
        LC_WARP_SYNC();
        LC_LANES(l) { w.v[l] = w.len[l] != LC_TS_NO_KEY; }
        const uint32_t pm = lc_lz4_ballot(w.v, lane, W);
        LC_LANES(l) { w.v[l] = w.len[l] != LC_TS_NO_KEY && w.klen[l] != LC_TS_KFAIL; }
        const uint32_t okm = lc_lz4_ballot(w.v, lane, W);
        LC_LANES(l) {
            w.v[l] = cacheable && have_key && w.len[l] != LC_TS_NO_KEY &&
                     lc_ts_prefix(base, w.off[l], w.len[l], key_off, key_len);
        }
        const uint32_t hxm = lc_lz4_ballot(w.v, lane, W);
        LC_LANES(l) {
            const uint32_t before = okm & lc_ts_below(l);
            const uint32_t p = before ? lc_hi_bit(before) : 0u;
            w.v[l] = cacheable && before && w.len[l] != LC_TS_NO_KEY &&
                     lc_ts_prefix(base, w.off[l], w.len[l], w.off[p], w.klen[p]);
        }
        const uint32_t hpm = lc_lz4_ballot(w.v, lane, W);
        // which events of the step hit, and how far the step can tell
        const uint32_t valid = lc_ts_below(nv);
        uint32_t hitm = 0, pos = 0;
        int owner = -1;
        while (cacheable && pos < nv) {
            const uint32_t rng = valid & ~lc_ts_below(pos);
            if (owner < 0) {
                const uint32_t mv = okm & ~hxm & rng;
                if (!mv) {
                    hitm |= hxm & rng;
                    pos = nv;
                    break;
                }
                const uint32_t m = lc_lo_bit(mv);
                hitm |= hxm & rng & lc_ts_below(m);
                owner = (int)m;
                pos = m + 1;
            } else {
                const uint32_t nx = okm & rng;
                if (!nx) {
                    hitm |= hpm & rng;
                    pos = nv;
                    break;
                }
                const uint32_t m = lc_lo_bit(nx);
                hitm |= hpm & rng & lc_ts_below(m + 1);
                pos = m + 1;
                if ((hpm >> m) & 1u)
                    break; // m hits the owner's key, so the events after it are compared with m's key: next step
                owner = (int)m;
            }
        }
        if (!cacheable)
            pos = nv;
        const uint32_t res = lc_ts_below(pos);
        const uint32_t missm = pm & ~hitm & res, okmiss = okm & missm;
        const int64_t state0 = state;
        // tv_sec left by the full parse of miss lane j
        auto after = [&](uint32_t j) -> int64_t {
            if (c.mode & LC_TSM_F_ONLY)
                return state0 - (int64_t)c.adjust * (int64_t)lc_ts_popc(okmiss & lc_ts_below(j + 1));
            return w.klen[j] != LC_TS_KFAIL ? w.raw[j] - c.adjust : w.raw[j];
        };
        LC_LANES(l) {
            if (l < pos) {
                uint8_t st;
                int64_t s = 0;
                uint32_t ns = 0;
                if (w.len[l] == LC_TS_NO_KEY) {
                    st = LC_TS_ST_NOT_FOUND;
                    cnt[LC_TS_C_KEY_NOT_FOUND]++;
                } else {
                    bool ok;
                    if ((hitm >> l) & 1u) {
                        const uint32_t lm = missm & lc_ts_below(l), lo = okmiss & lc_ts_below(l);
                        s = lm ? after(lc_hi_bit(lm)) : state0;
                        const uint32_t kl = lo ? w.klen[lc_hi_bit(lo)] : key_len;
                        ok = true;
                        if ((c.mode & LC_TSM_END_F) || ((c.mode & LC_TSM_EPOCH) && w.len[l] > kl)) {
                            const LcTsIn in{base + w.off[l] + kl, w.len[l] - kl};
                            uint32_t q = 0;
                            int nl;
                            ok = lc_ts_nsec(in, q, ns, nl);
                            if (!ok)
                                ns = 0;
                        }
                    } else {
                        ok = w.klen[l] != LC_TS_KFAIL;
                        s = after(l);
                        ns = w.fns[l];
                    }
                    if (!ok) {
                        s = 0;
                        ns = 0;
                        st = LC_TS_ST_FAILED;
                        cnt[LC_TS_C_OUT_FAILED]++;
                    } else if (s <= 0 || (now.discard_interval >= 0 && now.now - s > (int64_t)now.discard_interval)) {
                        st = LC_TS_ST_DISCARDED;
                        cnt[LC_TS_C_HISTORY_FAILURE]++;
                        cnt[LC_TS_C_DISCARDED]++;
                    } else {
                        st = LC_TS_ST_OK;
                        cnt[LC_TS_C_OUT_SUCCESSFUL]++;
                    }
                }
                sec[b + l] = s;
                nsec[b + l] = ns;
                status[b + l] = st;
            }
        }
        if (okmiss) {
            const uint32_t j = lc_hi_bit(okmiss);
            have_key = true;
            key_off = w.off[j];
            key_len = w.klen[j];
        }
        if (missm)
            state = after(lc_hi_bit(missm));
        LC_WARP_SYNC();
        b += pos;
    }
}

// Host, at Init: the process zone's offsets for tm_isdst = 0 and 1, per year, as mktime applies them (probed at
// July 1st, 12:00 of each year).
inline void lc_ts_probe_zone(LcTsConf& c) {
    for (int k = 0; k < LC_TS_NYEARS; ++k) {
        const int64_t local = lc_ts_days_from_civil(LC_TS_Y0 + k, 7, 1) * 86400 + 43200;
        for (int d = 0; d < 2; ++d) {
            struct tm t;
            memset(&t, 0, sizeof t);
            t.tm_year = LC_TS_Y0 + k - 1900;
            t.tm_mon = 6;
            t.tm_mday = 1;
            t.tm_hour = 12;
            t.tm_isdst = d;
            const int64_t off = local - (int64_t)mktime(&t);
            (d ? c.dst_off : c.std_off)[k] = (int32_t)off;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> regex -> timestamp chain: ProcessorParseTimestampNative (ProcessorParseTimestampNative.cpp:100-179, the
// SourceKey tkey) behind the split -> regex chain, whose pieces and regex stage are unchanged.
//   - The timestamp stage sees the pieces the regex stage kept, in piece order, as one group: a piece the regex stage
//     erased is not an event of the stage (no counter, no cache step).
//   - Its value is what the regex stage left under tkey: resolved once, on the host, through the chain's two content
//     plans (lc_regex_sls_key_src) to capture j, the piece, or absent (LC_TS_NOT_FOUND).  tkey holding the offset
//     digits is refused.  Both a piece the regex erased and an absent key give the tap's value LC_TS_NO_KEY, which the
//     cache pass skips; the counters come from the size pass, which tells the two apart.
//   - The value is read over [off, off + len) followed by NUL bytes, as every timestamp value is.
//   - LC_TS_OK: Time = the parsed seconds truncated to 32 bits (raised to 2^28 by the body, LogGroupSerializer.cpp:
//     111-119) and, with enable_ns, Time_ns = the parsed nanoseconds (SetTimestamp(t, ns) engages the optional).
//     LC_TS_NOT_FOUND / LC_TS_FAILED: the source event's time and ns.  LC_TS_DISCARDED: no record.
struct LcSplitRegexTsCfg {
    uint32_t src[2];    // value source of tkey in a parsed [0] / failed [1] event: capture j, LC_REGEX_SLS_LINE, or
                        // LC_FILTER_SLS_ABSENT
    uint32_t enable_ns; // mEnableTimestampNanosecond: a parsed time writes Time_ns
};

// counters[8] of the chain: the regex stage's three, then the timestamp stage's five in lc_timestamp_parse's order
#define LC_SRTS_COUNTERS 8

// Host side: whether the source event's Time_ns agrees with enable_ns.  time_ns is the source event's Time_ns as the
// serialiser writes it, so a source Time_ns without enable_ns would give Time_ns to the records that keep the source
// time and not to the parsed ones, a mix no configuration of the reference produces.  Returns nullptr, or why not.
// Cfg: the configuration of the chain in front of the timestamp stage (LcSplitRegexSlsCfg, LcSplitJsonSlsCfg).
template <class Cfg>
inline const char* lc_split_regex_ts_ns_check(const Cfg& c, int enable_ns) {
    return c.has_ns && !enable_ns ? "a source time_ns needs enable_ns" : nullptr;
}

// Host side: resolve tkey (lc_regex_sls_key_src over the plans of lc_split_regex_sls_setup, which accepted c; kstr /
// klen: lc_split_regex_sls_strings' key table) and check the source Time_ns against enable_ns.  Returns nullptr, or
// why the chain is refused.
inline const char* lc_split_regex_ts_setup(const LcSplitRegexSlsCfg& c, const uint32_t* plan, const char* const* kstr,
                                           const uint32_t* klen, const char* tkey, uint32_t tkey_len, int enable_ns,
                                           LcSplitRegexTsCfg* t) {
    if (!t || !plan || (tkey_len && !tkey))
        return "bad arguments";
    const char* why = lc_split_regex_ts_ns_check(c, enable_ns);
    if (why)
        return why;
    lc_regex_sls_key_src(plan, c.x.n_ok, c.x.n_fail, kstr, klen, tkey, tkey_len, t->src);
    if (t->src[0] == LC_REGEX_SLS_DIGITS || t->src[1] == LC_REGEX_SLS_DIGITS)
        return "the timestamp key holds the offset digits (it equals the offset key)";
    t->enable_ns = enable_ns != 0;
    return nullptr;
}

// The tap: row r's value for the timestamp stage, *len = LC_TS_NO_KEY when the regex stage erased the piece or left
// no tkey.
LC_HD void lc_split_regex_ts_value(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& t,
                                   const LcSplitRegexSlsRow& r, uint32_t* off, uint32_t* len) {
    const uint32_t v = lc_regex_sls_verdict(c.x, r.status);
    const uint32_t s = t.src[v == 0u ? 0 : 1];
    *off = 0;
    *len = LC_TS_NO_KEY;
    if ((v != 0u && !c.x.keep_fail) || s == LC_FILTER_SLS_ABSENT)
        return;
    if (s == LC_REGEX_SLS_LINE)
        *off = r.po, *len = r.plen;
    else
        *off = r.co[s], *len = r.cl[s];
}

// The record's time after the timestamp stage (ts: the stage's LC_TS_ST_* of the row, sec / nsec its time).
struct LcSplitRegexTsTime {
    uint32_t keep; // 0: LC_TS_DISCARDED, no record
    uint32_t time, has_ns, ns;
};
LC_HD LcSplitRegexTsTime lc_split_regex_ts_time(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& t, uint32_t ts,
                                                int64_t sec, uint32_t nsec) {
    if (ts == LC_TS_ST_OK)
        return {1u, (uint32_t)sec, t.enable_ns, nsec};
    return {ts != LC_TS_ST_DISCARDED, c.time, c.has_ns, c.ns};
}

// The row's counter verdicts as bits of the LC_SRTS_COUNTERS counters: the regex stage's (lc_split_regex_verdict),
// then -- when the regex stage kept the piece -- the timestamp stage's key_not_found, out_failed, history_failure,
// discarded, out_successful.
// The stage verdicts of a chain's row (lc_split_*_verdict) and, when the stage kept the piece, the timestamp stage's
// key_not_found, out_failed, history_failure, discarded, out_successful as bits 3.. of the LC_SRTS_COUNTERS counters.
LC_HD uint32_t lc_split_ts_verdict_bits(const LcSplitRegexVerdict& v, uint32_t ts) {
    uint32_t bits = v.ok | (v.failed << 1) | (v.erased << 2);
    if (v.erased)
        return bits;
    if (ts == LC_TS_ST_NOT_FOUND)
        bits |= 1u << (3 + LC_TS_C_KEY_NOT_FOUND);
    else if (ts == LC_TS_ST_FAILED)
        bits |= 1u << (3 + LC_TS_C_OUT_FAILED);
    else if (ts == LC_TS_ST_DISCARDED)
        bits |= (1u << (3 + LC_TS_C_HISTORY_FAILURE)) | (1u << (3 + LC_TS_C_DISCARDED));
    else
        bits |= 1u << (3 + LC_TS_C_OUT_SUCCESSFUL);
    return bits;
}

LC_HD uint32_t lc_split_regex_ts_verdict(const LcSplitRegexSlsCfg& c, uint32_t status, uint32_t ts) {
    return lc_split_ts_verdict_bits(lc_split_regex_verdict(c, status), ts);
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> delimiter -> timestamp chain: ProcessorParseTimestampNative (ProcessorParseTimestampNative.cpp:100-235,
// the SourceKey tkey) behind the split -> delimiter chain, whose pieces and delimiter stage are unchanged.
//   - The timestamp stage sees the pieces the delimiter stage did not erase, in piece order, as one group: a failed
//     piece erased without KeepingSourceWhenParseFail is not an event of the stage (no counter, no cache step).  A
//     piece kept without contents is an event: it counts key_not_found.
//   - Its value is what ProcessorParseDelimiterNative::ProcessEvent (ProcessorParseDelimiterNative.cpp:206-364,
//     AddLog :411-419) leaves under tkey.  The keys are distinct (lc_delim_sls_setup), so tkey names at most one
//     column j; a skipped "_" in discard mode names none.
//       blank piece (left untouched):  the piece when tkey is SourceKey, else none
//       parsed piece:                  column j unquoted (AddFieldWithUnQuote) when the row reaches it; else the piece
//                                      when tkey is SourceKey and SourceKey is one of the keys (mSourceKeyOverwritten:
//                                      a short row keeps it), or when tkey is RenamedSourceKey with
//                                      KeepingSourceWhenParseSucceed; else none
//       kept failure:                  the piece when tkey is RenamedSourceKey, or "__raw_log__" with CopingRawLog
//                                      (SourceKey was deleted); else none
//     tkey equal to the offset key is refused, and -- unless overflow columns are discarded -- so is a tkey of the
//     form __column<digits>__, which a generated overflow key would hold on some rows only.
//   - Every value lies inside its own piece, so the tap copies each to its own offset of a value buffer as long as the
//     chunk; a column with doubled quotes is collapsed there in place (never longer than the column).  The value is
//     read over [off, off + len) followed by NUL bytes, as every timestamp value is.
//   - The record's time is lc_split_regex_ts_time's rule: LC_TS_OK sets Time (and Time_ns with enable_ns),
//     LC_TS_NOT_FOUND / LC_TS_FAILED keep the source event's, LC_TS_DISCARDED leaves no record.
struct LcSplitDelimTsCfg {
    uint32_t col;       // the column keyed tkey (not a skipped "_"), or LC_DELIM_SLS_NONE
    uint32_t is_src;    // tkey == SourceKey
    uint32_t is_ren;    // tkey == RenamedSourceKey
    uint32_t is_raw;    // tkey == "__raw_log__"
    uint32_t enable_ns; // mEnableTimestampNanosecond: a parsed time writes Time_ns
};

// counters[9] of the chain: the delimiter stage's four, then the timestamp stage's five in lc_timestamp_parse's order
#define LC_SDTS_COUNTERS 9

// Host side: check tkey and the source Time_ns against the chain's configuration c (lc_split_delim_sls_link accepted
// it with the same keys, SourceKey, RenamedSourceKey and offset key; offset_key == nullptr: no log.file.offset
// metadata) and resolve tkey into *t.  Returns nullptr, or why the chain is refused.
inline const char* lc_split_delim_ts_setup(const LcSplitDelimSlsCfg& c, const char* const* keys,
                                           const uint32_t* key_lens, const char* source_key, uint32_t source_len,
                                           const char* renamed_key, uint32_t renamed_len, const char* offset_key,
                                           uint32_t offset_len, const char* tkey, uint32_t tkey_len, int enable_ns,
                                           LcSplitDelimTsCfg* t) {
    if (!t || (tkey_len && !tkey))
        return "bad arguments";
    auto eq = [](const char* a, uint32_t la, const char* b, uint32_t lb) {
        return la == lb && (la == 0 || !memcmp(a, b, la));
    };
    const char* why = lc_split_regex_ts_ns_check(c, enable_ns);
    if (why)
        return why;
    if (offset_key && eq(tkey, tkey_len, offset_key, offset_len))
        return "the timestamp key equals the offset key";
    uint32_t idx;
    if (c.d.mode != LC_DELIM_SLS_DISCARD && tkey_len && lc_delim_column_form(tkey, tkey_len, &idx))
        return "a timestamp key of the form __column<digits>__ collides with the generated overflow keys";
    memset(t, 0, sizeof *t);
    t->col = LC_DELIM_SLS_NONE;
    for (uint32_t k = 0; k < c.d.nkeys; ++k)
        if (eq(keys[k], key_lens[k], tkey, tkey_len) &&
            !(c.d.mode == LC_DELIM_SLS_DISCARD && key_lens[k] == 1 && keys[k][0] == '_'))
            t->col = k;
    t->is_src = eq(tkey, tkey_len, source_key, source_len);
    t->is_ren = eq(tkey, tkey_len, renamed_key, renamed_len);
    t->is_raw = eq(tkey, tkey_len, "__raw_log__", 11);
    t->enable_ns = enable_ns != 0;
    return nullptr;
}

// The tap's value of one piece: src[off, + n) holding dq doubled quotes, which the value buffer gets collapsed to
// n - dq bytes at off; n = LC_TS_NO_KEY when the delimiter stage erased the piece or left no value under tkey.
struct LcSplitDelimTsValue {
    uint32_t off, n, dq;
};
LC_HD LcSplitDelimTsValue lc_split_delim_ts_value(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& t,
                                                  const LcDelimSlsRow& r) {
    const LcSplitDelimTsValue none{0u, LC_TS_NO_KEY, 0u}, piece{r.eo, r.elen, 0u};
    if (r.status == 2) // LC_DELIM_BLANK: untouched
        return t.is_src ? piece : none;
    if (r.status != 0) // failed: RenamedSourceKey [, "__raw_log__"] -> piece when kept, else erased
        return c.d.keep_fail && (t.is_ren || (c.d.copy_raw && t.is_raw)) ? piece : none;
    if (t.col < r.nf) // col < nkeys < max_fields: always in the table
        return {r.fo[t.col], r.fl[t.col], c.d.use_quote ? r.fd[t.col] : 0u};
    return (t.is_src && c.d.src_overwritten) || (t.is_ren && c.d.keep_succeed) ? piece : none;
}

// The tap's collapse of a column s[0, n) holding doubled quotes q q (a column the state machine parsed holds no lone
// quote) into d[0, n - its pairs), AddFieldWithUnQuote's rule, W lanes taking W bytes per step: a quote is dropped when
// it is the second of its pair, which each lane tells from the run of quotes up to it (odd: the run that reaches the
// step's first byte holds an odd count so far).  v: W words of per-warp scratch (shared memory on the device).  Every
// lane calls it.
LC_HD void lc_split_delim_ts_collapse(uint8_t* d, const uint8_t* s, uint32_t n, uint8_t q, uint32_t* v,
                                      uint32_t lane, uint32_t W) {
    uint32_t w = 0, odd = 0;
    for (uint32_t b = 0; b < n; b += W) {
        const uint32_t nv = n - b < W ? n - b : W;
        LC_LANES(l) { v[l] = l < nv && s[b + l] == q; }
        const uint32_t qm = lc_lz4_ballot(v, lane, W);
        LC_WARP_SYNC();
        LC_LANES(l) {
            uint32_t drop = 0;
            if ((qm >> l) & 1) {
                const uint32_t nq = ~qm & lc_ts_below(l); // the non-quotes below: the run starts after the last
                drop = ((nq ? l - lc_hi_bit(nq) : l + 1 + odd) & 1) == 0;
            }
            v[l] = drop;
        }
        const uint32_t keep = lc_ts_below(nv) & ~lc_lz4_ballot(v, lane, W);
        LC_WARP_SYNC();
        LC_LANES(l) {
            if ((keep >> l) & 1)
                d[w + lc_popc(keep & lc_ts_below(l))] = s[b + l];
        }
        w += lc_popc(keep);
        const uint32_t nq = ~qm & lc_ts_below(nv);
        odd = nq ? (nv - 1 - lc_hi_bit(nq)) & 1 : (odd + nv) & 1;
    }
}

// The record's time after the timestamp stage (ts: the stage's LC_TS_ST_* of the row, sec / nsec its time)
LC_HD LcSplitRegexTsTime lc_split_delim_ts_time(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& t, uint32_t ts,
                                                int64_t sec, uint32_t nsec) {
    if (ts == LC_TS_ST_OK)
        return {1u, (uint32_t)sec, t.enable_ns, nsec};
    return {ts != LC_TS_ST_DISCARDED, c.time, c.has_ns, c.ns};
}

// The row's counter verdicts as bits of the LC_SDTS_COUNTERS counters: the delimiter stage's successful, failed,
// discarded, blank (lc_delim_sls_verdict), then -- when the delimiter stage kept the piece -- the timestamp stage's
// key_not_found, out_failed, history_failure, discarded, out_successful.
LC_HD uint32_t lc_split_delim_ts_verdict(const LcSplitDelimSlsCfg& c, uint32_t status, uint32_t ts) {
    const LcDelimSlsVerdict d = lc_delim_sls_verdict(c.d, status);
    const uint32_t t = lc_split_ts_verdict_bits(LcSplitRegexVerdict{0u, 0u, d.erased}, ts) >> 3;
    return d.ok | (d.failed << 1) | (d.erased << 2) | (d.blank << 3) | (t << 4);
}

// ================================================================================================ Apsara parse
// ProcessorParseApsaraNative (ProcessorParseApsaraNative.cpp: ProcessEvent 116-241, ApsaraEasyReadLogTimeParser
// 251-323, FindBaseFields 342-361, ParseApsaraBaseFields 433-463, AddLog 465-473) in three passes:
//   - lc_ap_scan: one lane per event reads the time's form and, for a date, the full parse (Strptime with
//     "%Y-%m-%d %H:%M:%S" then "%f", mktime over LcTsConf's zone table, minus the Timezone adjustment), the nanoseconds
//     a cache hit would give and the 19-byte cache key; then it counts the event's entries (lc_ap_fields).
//   - lc_ap_resolve: one warp per group applies the time cache in event order, 32 events per step, and gives each
//     event its status, time and counters.
//   - lc_ap_fields again, behind an exclusive sum of the parsed events' entry counts, writes the entries.
// The time cache needs no sequential walk.  A date event whose full parse succeeds leaves the cache key equal to its
// own 19 bytes at value + 1, whether it hit (the key was already those bytes) or missed (it stored them); an event
// whose full parse fails, and every other event, leaves the cache as it was.  So the key an event meets is the key of
// the nearest earlier date event of its group whose full parse succeeded, and the cached seconds are those of the
// nearest earlier one of those that missed.
// The reference's undefined reads, as pinned here (and in the C oracle):
//   - the key is the 19 bytes at value + 1 whatever they are; bytes past the end of the base buffer read as NUL;
//   - a time string (the bytes [1, first ']'] of the value) shorter than the key misses: the comparison reaches its
//     NUL terminator first;
//   - a value shorter than 2 bytes fails the time parse (the reference reads value[1]);
//   - the time string is read as a C string: a NUL byte inside it ends it.
#define LC_AP_NO_KEY 0xFFFFFFFFu
#define LC_AP_KEY_LEN 19
#define LC_AP_MAX_BASE 10

// status: low 3 bits the outcome, LC_AP_ST_OVER set on LC_AP_ST_OK when a key:value key equals SourceKey
#define LC_AP_ST_OK 0
#define LC_AP_ST_NOT_FOUND 1
#define LC_AP_ST_EMPTY 2
#define LC_AP_ST_FAILED 3
#define LC_AP_ST_DISCARDED 4
#define LC_AP_ST_OVER 0x80

// the key of a base-field entry (LcApEntry::key_off; key_len 0)
#define LC_AP_K_LEVEL 0xFFFFFFF0u
#define LC_AP_K_THREAD 0xFFFFFFF1u
#define LC_AP_K_FILE 0xFFFFFFF2u
#define LC_AP_K_LINE 0xFFFFFFF3u

// LcApEv::form
#define LC_AP_F_NONE 0  // no SourceKey
#define LC_AP_F_EMPTY 1 // an empty value
#define LC_AP_F_FAIL 2  // no '[' / ']', shorter than 2 bytes, or an epoch that does not parse
#define LC_AP_F_EPOCH 3 // "[1...]": sec / nsec; the cache is not touched
#define LC_AP_F_DATE 4  // anything else after '['
// LcApEv::flags
#define LC_AP_FULL_OK 1u // DATE: the full parse succeeded (sec / nsec)
#define LC_AP_LONG 2u    // DATE: the time string has at least LC_AP_KEY_LEN bytes, so it can hit
#define LC_AP_OVER 4u    // a key:value key equals SourceKey

struct LcApEntry {
    uint32_t key_off, key_len, val_off, val_len; // offsets into the base buffer; key_off LC_AP_K_*: a base field
};

struct LcApEv { // per-event result of the scan pass
    int64_t sec;     // EPOCH: seconds; DATE with LC_AP_FULL_OK: the full parse's seconds minus the adjustment
    uint32_t nsec;   // EPOCH / DATE full parse: tv_nsec
    uint32_t hnsec;  // DATE: tv_nsec of a cache hit (%f at time string + 20)
    uint32_t key[5]; // DATE: the LC_AP_KEY_LEN bytes at value + 1, little-endian, then a NUL
    uint32_t nent;   // entries of the event if it parses
    uint8_t form, flags;
};

struct LcApWarp { // per-warp scratch of the resolution pass
    uint32_t v[32];
};

LC_HD bool lc_ap_upper(uint32_t ch) { return ch - 'A' < 26u; }

// Strptime(s, "%Y-%m-%d %H:%M:%S"): false = NULL; p = where the parse stopped
LC_HD bool lc_ap_date(const LcTsIn& in, uint32_t& p, LcTsTm& tm) {
    int i = 1900;
    p = 0;
    if (!lc_ts_num(in, p, i, 0, 9999))
        return false;
    tm.year = i - 1900;
    if (in.at(p++) != '-')
        return false;
    i = 1;
    if (!lc_ts_num(in, p, i, 1, 12))
        return false;
    tm.mon = i - 1;
    if (in.at(p++) != '-' || !lc_ts_num(in, p, tm.mday, 1, 31))
        return false;
    while (lc_ts_space(in.at(p)))
        ++p;
    if (!lc_ts_num(in, p, tm.hour, 0, 23) || in.at(p++) != ':' || !lc_ts_num(in, p, tm.min, 0, 59) ||
        in.at(p++) != ':')
        return false;
    return lc_ts_num(in, p, tm.sec, 0, 61);
}

// Strptime(s + q, "%f"): tv_nsec, 0 when it fails
LC_HD uint32_t lc_ap_frac(const LcTsIn& in, uint32_t q) {
    uint32_t ns = 0;
    int nl;
    return lc_ts_nsec(in, q, ns, nl) ? ns : 0u;
}

// ParseApsaraBaseFields then the key:value loop of ProcessEvent over the value s[0, n), in append order:
// out.base(tag, off, len) and out.kv(key_off, key_len, val_off, val_len), offsets relative to s.
// FindBaseFields' slots are classified as they close, which is the order ParseApsaraBaseFields visits them in.
template <class Out> LC_HD void lc_ap_fields(const uint8_t* s, uint32_t n, Out& out) {
    uint32_t nslots = 0, beg = 0, last_end = 0, found = 0; // found: bit 0 level, 1 thread, 2 file
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t ch = s[i];
        if (ch == '[') {
            beg = i + 1;
        } else if (ch == ']') {
            const uint32_t nx = i + 1 < n ? s[i + 1] : 0u;
            if (i + 1 == n || nx == '\t' || nx == '\n') {
                if (nslots >= 1 && found != 7u) {
                    bool lvl = !(found & 1u), thr = !(found & 2u), fil = false;
                    uint32_t colon = i;
                    for (uint32_t k = beg; k < i; ++k) {
                        const uint32_t c = s[k];
                        lvl = lvl && lc_ap_upper(c);
                        thr = thr && lc_ts_digit(c);
                        fil = fil || c == '/' || c == '.';
                        if (c == ':' && colon == i)
                            colon = k;
                    }
                    if (lvl) {
                        found |= 1u;
                        out.base(LC_AP_K_LEVEL, beg, i - beg);
                    } else if (thr) {
                        found |= 2u;
                        out.base(LC_AP_K_THREAD, beg, i - beg);
                    } else if (!(found & 4u) && fil) {
                        found |= 4u;
                        out.base(LC_AP_K_FILE, beg, colon - beg);
                        if (colon < i)
                            out.base(LC_AP_K_LINE, colon + 1, i - colon - 1);
                    }
                }
                last_end = i;
                beg = 0;
                ++nslots;
            }
            if (nslots >= LC_AP_MAX_BASE)
                break;
            if (nx == '\t' && (i + 2 == n || (i + 2 < n && s[i + 2] != '[')))
                break;
        }
    }
    uint32_t kbeg = 0;
    int64_t colon = -1;
    for (uint32_t i = last_end + 1; i <= n; ++i) {
        if (i == n || s[i] == '\t') {
            if (colon >= 0) {
                out.kv(kbeg, (uint32_t)colon - kbeg, (uint32_t)colon + 1, i - (uint32_t)colon - 1);
                colon = -1;
            }
            kbeg = i + 1;
        } else if (s[i] == ':' && colon == -1) {
            colon = i;
        }
    }
}

// counts the entries and tells whether a key:value key equals SourceKey
struct LcApCount {
    const uint8_t* s;
    const uint8_t* skey;
    uint32_t sklen, n, over;
    LC_HD void base(uint32_t, uint32_t, uint32_t) { ++n; }
    LC_HD void kv(uint32_t ko, uint32_t kl, uint32_t, uint32_t) {
        ++n;
        if (kl == sklen && !over) {
            uint32_t k = 0;
            while (k < kl && s[ko + k] == skey[k])
                ++k;
            over = k == kl;
        }
    }
};

// writes the entries from e (value at base offset o)
struct LcApEmit {
    LcApEntry* e;
    uint32_t o;
    LC_HD void base(uint32_t tag, uint32_t off, uint32_t len) { *e++ = LcApEntry{tag, 0u, o + off, len}; }
    LC_HD void kv(uint32_t ko, uint32_t kl, uint32_t vo, uint32_t vl) { *e++ = LcApEntry{o + ko, kl, o + vo, vl}; }
};

// The scan of one event: value base[o, o + len), base_len bytes in the buffer (the key reads NUL past it).
LC_HD LcApEv lc_ap_scan(const LcTsConf& c, const uint8_t* base, uint64_t base_len, uint32_t o, uint32_t len,
                        const uint8_t* skey, uint32_t sklen) {
    LcApEv ev{0, 0, 0, {0, 0, 0, 0, 0}, 0, LC_AP_F_NONE, 0};
    if (len == LC_AP_NO_KEY)
        return ev;
    if (len == 0) {
        ev.form = LC_AP_F_EMPTY;
        return ev;
    }
    const uint8_t* s = base + o;
    ev.form = LC_AP_F_FAIL;
    uint32_t pos = 1;
    while (pos < len && s[pos] != ']')
        ++pos;
    if (len < 2 || s[0] != '[' || pos == len)
        return ev;
    const LcTsIn in{s + 1, pos}; // the time string [1, pos], ']' included
    if (s[1] == '1') {
        int64_t secs;
        uint32_t ns, end;
        int nl;
        if (!lc_ts_epoch_end(in, secs, ns, nl, end) || in.at(end) != ']')
            return ev;
        ev.form = LC_AP_F_EPOCH;
        ev.sec = secs;
        ev.nsec = ns;
    } else {
        ev.form = LC_AP_F_DATE;
        for (uint32_t k = 0; k < LC_AP_KEY_LEN; ++k) {
            const uint64_t at = (uint64_t)o + 1 + k;
            ev.key[k >> 2] |= (uint32_t)(at < base_len ? base[at] : 0u) << ((k & 3u) * 8);
        }
        if (pos >= LC_AP_KEY_LEN) {
            ev.flags |= LC_AP_LONG;
            ev.hnsec = pos > LC_AP_KEY_LEN ? lc_ap_frac(in, LC_AP_KEY_LEN + 1) : 0u;
        }
        LcTsTm tm{0, 0, 0, 0, 0, 0, 0};
        uint32_t p;
        if (lc_ap_date(in, p, tm)) {
            ev.flags |= LC_AP_FULL_OK;
            ev.sec = lc_ts_mktime(c, tm) - c.adjust;
            ev.nsec = in.at(p) ? lc_ap_frac(in, p + 1) : 0u;
        }
    }
    LcApCount cnt{s, skey, sklen, 0, 0};
    lc_ap_fields(s, len, cnt);
    ev.nent = cnt.n;
    ev.flags |= cnt.over ? LC_AP_OVER : 0u;
    return ev;
}

LC_HD bool lc_ap_same_key(const LcApEv& a, const LcApEv& b) {
    return a.key[0] == b.key[0] && a.key[1] == b.key[1] && a.key[2] == b.key[2] && a.key[3] == b.key[3] &&
           a.key[4] == b.key[4];
}

// The time cache and ProcessEvent's verdict over the events [e0, e1) of one group, W lanes, 32 events per step.
// Per event: status, sec, nsec (SetTimestamp's), micro (logTime_in_micro), nent (entries to write: ev.nent for
// LC_AP_ST_OK, else 0).  cnt[5] += key_not_found, out_failed, history_failure, discarded, out_successful (the
// discards of the failure path depend on the event's other contents: the caller adds them).
LC_HD void lc_ap_resolve(const LcTsNow& now, const LcApEv* ev, uint64_t e0, uint64_t e1, uint8_t* status, int64_t* sec,
                         uint32_t* nsec, int64_t* micro, uint32_t* nent, uint64_t* cnt, LcApWarp& w, uint32_t lane,
                         uint32_t W) {
    uint64_t last_ok = ~0ull, last_miss = ~0ull; // the group's nearest earlier full-parsed date / missing date event
    for (uint64_t b = e0; b < e1; b += W) {
        const uint32_t nv = e1 - b < W ? (uint32_t)(e1 - b) : W;
        LC_LANES(l) { w.v[l] = l < nv && ev[b + l].form == LC_AP_F_DATE && (ev[b + l].flags & LC_AP_FULL_OK); }
        const uint32_t okm = lc_lz4_ballot(w.v, lane, W);
        LC_WARP_SYNC();
        LC_LANES(l) {
            bool hit = false;
            if (l < nv && ev[b + l].form == LC_AP_F_DATE && (ev[b + l].flags & LC_AP_LONG)) {
                const uint32_t before = okm & lc_ts_below(l);
                const uint64_t p = before ? b + lc_hi_bit(before) : last_ok;
                hit = p != ~0ull && lc_ap_same_key(ev[b + l], ev[p]);
            }
            w.v[l] = hit;
        }
        const uint32_t hitm = lc_lz4_ballot(w.v, lane, W), missm = okm & ~hitm;
        LC_WARP_SYNC();
        LC_LANES(l) {
            if (l < nv) {
                const uint64_t i = b + l;
                const LcApEv& e = ev[i];
                uint8_t st = LC_AP_ST_FAILED;
                int64_t s = 0, us = 0;
                uint32_t ns = 0;
                if (e.form == LC_AP_F_NONE) {
                    st = LC_AP_ST_NOT_FOUND;
                    cnt[LC_TS_C_KEY_NOT_FOUND]++;
                } else if (e.form == LC_AP_F_EMPTY) {
                    st = LC_AP_ST_EMPTY;
                    cnt[LC_TS_C_OUT_FAILED]++;
                } else {
                    bool ok = e.form == LC_AP_F_EPOCH || (e.form == LC_AP_F_DATE && (e.flags & LC_AP_FULL_OK));
                    uint32_t fns = e.nsec;
                    s = e.sec;
                    if ((hitm >> l) & 1u) {
                        const uint32_t lm = missm & lc_ts_below(l);
                        s = ev[lm ? b + lc_hi_bit(lm) : last_miss].sec;
                        fns = e.hnsec;
                        ok = true;
                    }
                    us = (int64_t)((uint64_t)s * 1000000u + fns / 1000u);
                    if (!ok || s <= 0) {
                        s = us = 0;
                        cnt[LC_TS_C_OUT_FAILED]++;
                    } else {
                        ns = (uint32_t)((int64_t)((uint64_t)us * 1000u) % 1000000000);
                        if (now.discard_interval >= 0 && now.now - s > (int64_t)now.discard_interval) {
                            st = LC_AP_ST_DISCARDED;
                            cnt[LC_TS_C_HISTORY_FAILURE]++;
                            cnt[LC_TS_C_DISCARDED]++;
                        } else {
                            st = LC_AP_ST_OK | ((e.flags & LC_AP_OVER) ? LC_AP_ST_OVER : 0);
                            cnt[LC_TS_C_OUT_SUCCESSFUL]++;
                        }
                    }
                }
                status[i] = st;
                sec[i] = s;
                nsec[i] = ns;
                micro[i] = us;
                nent[i] = (st & 7u) == LC_AP_ST_OK ? e.nent : 0u;
            }
        }
        if (okm)
            last_ok = b + lc_hi_bit(okm);
        if (missm)
            last_miss = b + lc_hi_bit(missm);
        LC_WARP_SYNC();
    }
}

// ================================================================================================ JSON parse
// ProcessorParseJsonNative (ProcessorParseJsonNative.cpp: ProcessEvent, JsonLogLineParserSimdJson,
// OptimizedValueToStringBuffer, ProcessNumberValueOptimized).  The rules are pinned in include/lc_b200.h above
// lc_json_parse.  One thread walks one event: lc_json_walk validates the whole document (strict RFC 8259, root object,
// depth <= 1024, valid UTF-8, paired surrogates, a NUL byte after the root ends the input) and produces its top-level
// members.  The count pass and the emit pass run the same walk (EMIT false / true), so their sizes agree.
//
// SLOW = false is the fast instantiation: nesting up to LC_JSON_FAST_DEPTH in a 64-bit register, floats of at most
// 19 significant digits through one exact operation (mantissa <= 2^53, |decimal exponent| <= 22) or else the
// Eisel-Lemire step over a 128-bit power-of-five table in global memory, "%f" of |x| < 2^64 in 64/128-bit integers.  Anything else returns LC_JSON_W_SLOW and the event goes to the SLOW = true
// instantiation: nesting up to 1024 on a bit stack in local memory, exact decimal-to-double conversion of any length
// (800 significant digits and a sticky digit, decided by big-integer comparison with the halfway points), "%f" of
// integer parts of any size.  Reads stay inside the event; writes go only to the event's entry and arena ranges, and
// a write past either sets `over` instead.
#include "lc_json_pow5.h" // the Eisel-Lemire table; the device walks read the engine's copy through LcJsonOut::pow5

#define LC_JSON_NO_KEY 0xFFFFFFFFu
#define LC_JSON_ST_OK 0u
#define LC_JSON_ST_NOT_FOUND 1u
#define LC_JSON_ST_EMPTY 2u
#define LC_JSON_ST_FAILED 3u
#define LC_JSON_ST_OVER 0x80u
#define LC_JSON_ARENA 0x80000000u // tag bit of an offset into the arena (otherwise an offset into base)
#define LC_JSON_FAST_DEPTH 64u
#define LC_JSON_MAX_DEPTH 1024u
#define LC_JSON_MAX_DIGITS 800
#define LC_JSON_BIG_LIMBS 144 // 4608 bits: both sides of a halfway-point comparison fit (< 3800 bits)

enum : uint32_t { LC_JSON_W_OK = 0, LC_JSON_W_FAIL = 1, LC_JSON_W_SLOW = 2 };

struct LcJsonEntry {
    uint32_t key_off, key_len, val_off, val_len;
};

// Where a walk's output goes.  The count pass (EMIT false) only sums nent and narena; the emit pass writes entry k to
// ent[k] and arena byte j to arena[j] when they are inside [0, ent_cap) / [0, arena_cap), and sets over otherwise.
template <bool EMIT>
struct LcJsonOut {
    const uint64_t* pow5; // lc_json_pow5 (host) or its device copy
    LcJsonEntry* ent;
    uint8_t* arena;
    uint32_t ent_cap, arena_cap;
    uint32_t base_off;  // the event's offset in base
    uint32_t arena_off; // the event's first arena byte in the arena
    uint32_t nent, narena;
    bool over, skey_hit;
    LC_HD void put(uint32_t j, uint32_t c) {
        if constexpr (EMIT) {
            if (j < arena_cap)
                arena[j] = (uint8_t)c;
            else
                over = true;
        }
    }
    LC_HD void entry(uint32_t ko, uint32_t kl, uint32_t vo, uint32_t vl) {
        if constexpr (EMIT) {
            if (nent < ent_cap)
                ent[nent] = LcJsonEntry{ko, kl, vo, vl};
            else
                over = true;
        }
        ++nent;
    }
    LC_HD void grow(uint32_t k) { // narena stays <= 2^31 (the call refuses totals that reach the tag bit)
        narena += k;
        if (narena > LC_JSON_ARENA)
            narena = LC_JSON_ARENA;
    }
};

LC_HD uint64_t lc_js_bits(double x) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t u;
    memcpy(&u, &x, 8);
    return u;
#endif
}

LC_HD double lc_js_dbl(uint64_t u) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double x;
    memcpy(&x, &u, 8);
    return x;
#endif
}

LC_HD uint32_t lc_js_ws(const uint8_t* s, uint32_t n, uint32_t p) {
    while (p < n && (s[p] == ' ' || s[p] == '\t' || s[p] == '\n' || s[p] == '\r'))
        ++p;
    return p;
}

LC_HD bool lc_js_digit(const uint8_t* s, uint32_t n, uint32_t p) { return p < n && s[p] >= '0' && s[p] <= '9'; }

// the 4 hex digits at s[p..p+4) as a value, -1 when they are not 4 hex digits inside the event
LC_HD int32_t lc_js_hex4(const uint8_t* s, uint32_t n, uint32_t p) {
    if (p > n || n - p < 4)
        return -1;
    int32_t v = 0;
    for (uint32_t k = 0; k < 4; ++k) {
        const uint32_t c = s[p + k];
        uint32_t d;
        if (c >= '0' && c <= '9')
            d = c - '0';
        else if ((c | 0x20u) >= 'a' && (c | 0x20u) <= 'f')
            d = (c | 0x20u) - 'a' + 10;
        else
            return -1;
        v = v * 16 + (int32_t)d;
    }
    return v;
}

// length of the valid UTF-8 sequence (2..4 bytes) that starts with the byte >= 0x80 at s[p], 0 when it is not valid
// (overlong forms, surrogates and code points past U+10FFFF are not valid)
LC_HD uint32_t lc_js_utf8_len(const uint8_t* s, uint32_t n, uint32_t p) {
    const uint32_t c = s[p];
    uint32_t k, lo = 0x80, hi = 0xBF;
    if (c < 0xC2)
        return 0;
    if (c < 0xE0) {
        k = 2;
    } else if (c < 0xF0) {
        k = 3;
        if (c == 0xE0)
            lo = 0xA0;
        if (c == 0xED)
            hi = 0x9F;
    } else if (c < 0xF5) {
        k = 4;
        if (c == 0xF0)
            lo = 0x90;
        if (c == 0xF4)
            hi = 0x8F;
    } else {
        return 0;
    }
    if (n - p < k)
        return 0;
    if (s[p + 1] < lo || s[p + 1] > hi)
        return 0;
    for (uint32_t j = 2; j < k; ++j)
        if ((s[p + j] & 0xC0u) != 0x80u)
            return 0;
    return k;
}

struct LcJsPutNone {
    LC_HD void operator()(uint32_t, uint32_t) {}
};

// compares the unescaped bytes with SourceKey
struct LcJsPutCmp {
    const uint8_t* k;
    uint32_t kl;
    bool eq;
    LC_HD void operator()(uint32_t j, uint32_t c) { eq = eq && j < kl && k[j] == c; }
};

// writes the unescaped bytes to the arena at `at`
template <bool EMIT>
struct LcJsPutArena {
    LcJsonOut<EMIT>* o;
    uint32_t at;
    LC_HD void operator()(uint32_t j, uint32_t c) { o->put(at + j, c); }
};

// The string whose opening quote is s[p - 1]: returns the position after its closing quote, 0 when it is not valid.
// *ulen is its unescaped length, *esc whether it has an escape; put(j, byte) receives unescaped byte j.
template <class Put>
LC_HD uint32_t lc_js_str(const uint8_t* s, uint32_t n, uint32_t p, uint32_t* ulen, bool* esc, Put& put) {
    uint32_t u = 0;
    bool e = false;
    while (p < n) {
        const uint32_t c = s[p];
        if (c == '"') {
            *ulen = u;
            *esc = e;
            return p + 1;
        }
        if (c < 0x20)
            return 0;
        if (c == '\\') {
            e = true;
            if (p + 1 >= n)
                return 0;
            uint32_t o;
            switch (s[p + 1]) {
            case '"': o = '"'; break;
            case '\\': o = '\\'; break;
            case '/': o = '/'; break;
            case 'b': o = 8; break;
            case 'f': o = 12; break;
            case 'n': o = 10; break;
            case 'r': o = 13; break;
            case 't': o = 9; break;
            case 'u': {
                int32_t cp = lc_js_hex4(s, n, p + 2);
                if (cp < 0 || (cp >= 0xDC00 && cp <= 0xDFFF))
                    return 0;
                p += 6;
                if (cp >= 0xD800 && cp <= 0xDBFF) {
                    if (p + 1 >= n || s[p] != '\\' || s[p + 1] != 'u')
                        return 0;
                    const int32_t lo = lc_js_hex4(s, n, p + 2);
                    if (lo < 0xDC00 || lo > 0xDFFF)
                        return 0;
                    p += 6;
                    cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
                }
                const uint32_t v = (uint32_t)cp;
                if (v < 0x80) {
                    put(u++, v);
                } else if (v < 0x800) {
                    put(u++, 0xC0 | (v >> 6));
                    put(u++, 0x80 | (v & 0x3F));
                } else if (v < 0x10000) {
                    put(u++, 0xE0 | (v >> 12));
                    put(u++, 0x80 | ((v >> 6) & 0x3F));
                    put(u++, 0x80 | (v & 0x3F));
                } else {
                    put(u++, 0xF0 | (v >> 18));
                    put(u++, 0x80 | ((v >> 12) & 0x3F));
                    put(u++, 0x80 | ((v >> 6) & 0x3F));
                    put(u++, 0x80 | (v & 0x3F));
                }
                continue;
            }
            default:
                return 0;
            }
            put(u++, o);
            p += 2;
            continue;
        }
        if (c < 0x80) {
            put(u++, c);
            ++p;
            continue;
        }
        const uint32_t k = lc_js_utf8_len(s, n, p);
        if (!k)
            return 0;
        for (uint32_t j = 0; j < k; ++j)
            put(u++, s[p + j]);
        p += k;
    }
    return 0;
}

// The number at s[p] ('-' or a digit): returns the position after it, 0 when it does not follow the JSON grammar.
// *isint: no fraction and no exponent.
LC_HD uint32_t lc_js_num(const uint8_t* s, uint32_t n, uint32_t p, bool* isint) {
    if (s[p] == '-')
        ++p;
    if (!lc_js_digit(s, n, p))
        return 0;
    if (s[p] == '0')
        ++p;
    else
        while (lc_js_digit(s, n, p))
            ++p;
    bool in = true;
    if (p < n && s[p] == '.') {
        const uint32_t q = ++p;
        while (lc_js_digit(s, n, p))
            ++p;
        if (p == q)
            return 0;
        in = false;
    }
    if (p < n && (s[p] | 0x20u) == 'e') {
        ++p;
        if (p < n && (s[p] == '+' || s[p] == '-'))
            ++p;
        const uint32_t q = p;
        while (lc_js_digit(s, n, p))
            ++p;
        if (p == q)
            return 0;
        in = false;
    }
    *isint = in;
    return p;
}

// true when the nd digits at s[p] are <= the nd digits of lim (same length)
LC_HD bool lc_js_digits_le(const uint8_t* s, uint32_t p, const char* lim, uint32_t nd) {
    for (uint32_t k = 0; k < nd; ++k)
        if (s[p + k] != (uint8_t)lim[k])
            return s[p + k] < (uint8_t)lim[k];
    return true;
}

LC_HD void lc_js_mul128(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#if defined(__CUDA_ARCH__)
    *hi = __umul64hi(a, b);
    *lo = a * b;
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    *hi = (uint64_t)(p >> 64);
    *lo = (uint64_t)p;
#endif
}

LC_HD uint32_t lc_js_clz64(uint64_t x) { // x != 0
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clzll((long long)x);
#else
    return (uint32_t)__builtin_clzll(x);
#endif
}

// The Eisel-Lemire step (Lemire, "Number Parsing at a Gigabyte per Second", 2021): the correctly rounded double of
// w * 10^q (w != 0, exact) from one or two 64 x 128-bit products with the table of lc_json_pow5.h.  false when it
// cannot decide (q outside the table, a subnormal result, or a product whose dropped bits might carry), which sends
// the event to the slow walk.
LC_HD bool lc_js_eisel_lemire(uint64_t w, int32_t q, bool neg, const uint64_t* pow5, double* out) {
    if (q < LC_JSON_POW5_QMIN || q > LC_JSON_POW5_QMAX)
        return false;
    const uint64_t* t = pow5 + 2 * (q - LC_JSON_POW5_QMIN);
    const uint32_t lz = lc_js_clz64(w);
    w <<= lz;
    uint64_t hi, lo;
    lc_js_mul128(w, t[0], &hi, &lo);
    if ((hi & 0x1FFull) == 0x1FFull) { // the 9 bits below the 55 kept ones may carry: add the second product
        uint64_t hi2, lo2;
        lc_js_mul128(w, t[1], &hi2, &lo2);
        lo += hi2;
        if (hi2 > lo)
            ++hi;
    }
    if (lo == 0xFFFFFFFFFFFFFFFFull && (q < -27 || q > 55))
        return false;
    const uint32_t upper = (uint32_t)(hi >> 63);
    uint64_t m = hi >> (upper + 9);
    int32_t p2 = (((152170 + 65536) * q) >> 16) + 63 + (int32_t)upper - (int32_t)lz + 1023;
    if (p2 <= 0)
        return false; // subnormal
    if (lo <= 1 && q >= -4 && q <= 23 && (m & 3) == 1 && (m << (upper + 9)) == hi)
        m &= ~1ull; // an exact halfway case: round to even (down)
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << 52)) {
        m = 1ull << 52;
        ++p2;
    }
    if (p2 >= 0x7FF)
        return false; // overflow: the slow walk renders it
    *out = lc_js_dbl(((uint64_t)p2 << 52) | (m & ~(1ull << 52)) | (neg ? 0x8000000000000000ull : 0ull));
    return true;
}

// The double of the number [a, b) when the fast instantiation can decide it: at most 19 significant digits, then
// one correctly rounded multiplication or division by an exact power of ten (mantissa <= 2^53, decimal exponent in
// [-22, 22]) or the Eisel-Lemire step.
LC_HD bool lc_js_dec_fast(const uint8_t* s, uint32_t a, uint32_t b, const uint64_t* pow5, double* out) {
    const bool neg = s[a] == '-';
    uint32_t p = a + (neg ? 1u : 0u), nsig = 0;
    uint64_t w = 0;
    int32_t e10 = 0;
    bool frac = false;
    for (; p < b; ++p) {
        const uint32_t c = s[p];
        if (c == '.') {
            frac = true;
            continue;
        }
        if (c < '0' || c > '9')
            break;
        if (nsig || c != '0') {
            if (nsig == 19)
                return false;
            w = w * 10 + (c - '0');
            ++nsig;
        }
        if (frac)
            --e10;
    }
    if (p < b) { // exponent
        ++p;
        bool eneg = false;
        if (s[p] == '+' || s[p] == '-')
            eneg = s[p++] == '-';
        int32_t ev = 0;
        for (; p < b; ++p)
            if (ev < 100000)
                ev = ev * 10 + (int32_t)(s[p] - '0');
        e10 += eneg ? -ev : ev;
    }
    if (w == 0) {
        *out = neg ? -0.0 : 0.0;
        return true;
    }
    if (w > (1ull << 53) || e10 < -22 || e10 > 22)
        return lc_js_eisel_lemire(w, e10, neg, pow5, out);
    double pw = 1.0;
    for (int32_t k = e10 < 0 ? -e10 : e10; k > 0; --k)
        pw *= 10.0; // exact up to 1e22
    double x = (double)w;
    if (e10 >= 0) {
        x *= pw;
    } else {
#if defined(__CUDA_ARCH__)
        // x / pw without the division routine's call: the correctly rounded reciprocal, a quotient within one ulp
        // and one residual step give the correctly rounded quotient (Markstein); x and pw are far from the
        // subnormal and overflow ranges here
        const double r = __drcp_rn(pw), q = x * r;
        x = __fma_rn(__fma_rn(-q, pw, x), r, q);
#else
        x /= pw;
#endif
    }
    *out = neg ? -x : x;
    return true;
}

// ---- big integers of the slow path (little-endian 32-bit limbs)
struct LcJsBig {
    uint32_t n;
    uint32_t w[LC_JSON_BIG_LIMBS];
};

LC_HD void lc_big_set(LcJsBig& x, uint64_t v) {
    x.n = 0;
    while (v) {
        x.w[x.n++] = (uint32_t)v;
        v >>= 32;
    }
}

LC_HD void lc_big_muladd(LcJsBig& x, uint32_t m, uint32_t add) {
    uint64_t carry = add;
    for (uint32_t k = 0; k < x.n; ++k) {
        const uint64_t t = (uint64_t)x.w[k] * m + carry;
        x.w[k] = (uint32_t)t;
        carry = t >> 32;
    }
    if (carry && x.n < LC_JSON_BIG_LIMBS)
        x.w[x.n++] = (uint32_t)carry;
}

LC_HD void lc_big_mulpow10(LcJsBig& x, uint32_t e) {
    for (; e >= 9; e -= 9)
        lc_big_muladd(x, 1000000000u, 0);
    uint32_t m = 1;
    for (; e; --e)
        m *= 10;
    if (m > 1)
        lc_big_muladd(x, m, 0);
}

LC_HD void lc_big_shl(LcJsBig& x, uint32_t bits) {
    if (!x.n)
        return;
    const uint32_t lw = bits >> 5, b = bits & 31;
    uint32_t nn = x.n + lw + 1;
    if (nn > LC_JSON_BIG_LIMBS)
        nn = LC_JSON_BIG_LIMBS;
    for (uint32_t k = nn; k-- > 0;) {
        const uint32_t hi = k >= lw && k - lw < x.n ? x.w[k - lw] : 0u;
        const uint32_t lo = b && k >= lw + 1 && k - lw - 1 < x.n ? x.w[k - lw - 1] : 0u;
        x.w[k] = b ? (hi << b) | (lo >> (32 - b)) : hi;
    }
    x.n = nn;
    while (x.n && !x.w[x.n - 1])
        --x.n;
}

LC_HD int lc_big_cmp(const LcJsBig& x, const LcJsBig& y) {
    if (x.n != y.n)
        return x.n < y.n ? -1 : 1;
    for (uint32_t k = x.n; k-- > 0;)
        if (x.w[k] != y.w[k])
            return x.w[k] < y.w[k] ? -1 : 1;
    return 0;
}

// x = divided by 10^9, returns the remainder
LC_HD uint32_t lc_big_div1e9(LcJsBig& x) {
    uint64_t r = 0;
    for (uint32_t k = x.n; k-- > 0;) {
        const uint64_t t = (r << 32) | x.w[k];
        x.w[k] = (uint32_t)(t / 1000000000u);
        r = t % 1000000000u;
    }
    while (x.n && !x.w[x.n - 1])
        --x.n;
    return (uint32_t)r;
}

// sign of D * 10^E - M * 2^t
LC_HD int lc_js_cmp_mid(const LcJsBig& D, int32_t E, uint64_t M, int32_t t, LcJsBig& L, LcJsBig& R) {
    L = D;
    lc_big_set(R, M);
    if (E >= 0)
        lc_big_mulpow10(L, (uint32_t)E);
    else
        lc_big_mulpow10(R, (uint32_t)-E);
    if (t >= 0)
        lc_big_shl(R, (uint32_t)t);
    else
        lc_big_shl(L, (uint32_t)-t);
    return lc_big_cmp(L, R);
}

// The correctly rounded double (round half to even) of the number [a, b), any number of digits: the first 800
// significant digits and a sticky digit for the rest, a first estimate from 19 digits, then steps to the neighbour
// while the value lies past a halfway point.  Overflow gives infinity, underflow a signed zero.
LC_HD double lc_js_dec_slow(const uint8_t* s, uint32_t a, uint32_t b) {
    LcJsBig D, L, R;
    const bool neg = s[a] == '-';
    uint32_t p = a + (neg ? 1u : 0u), nd = 0, k19 = 0;
    uint64_t w19 = 0;
    int64_t E = 0;
    bool frac = false, sticky = false;
    lc_big_set(D, 0);
    uint32_t chunk = 0, clen = 0;
    for (; p < b; ++p) {
        const uint32_t c = s[p];
        if (c == '.') {
            frac = true;
            continue;
        }
        if (c < '0' || c > '9')
            break;
        const uint32_t d = c - '0';
        if (nd == 0 && d == 0) {
            if (frac)
                --E;
        } else if (nd < LC_JSON_MAX_DIGITS) {
            chunk = chunk * 10 + d;
            if (++clen == 9) {
                lc_big_muladd(D, 1000000000u, chunk);
                chunk = clen = 0;
            }
            if (k19 < 19) {
                w19 = w19 * 10 + d;
                ++k19;
            }
            ++nd;
            if (frac)
                --E;
        } else {
            sticky = sticky || d != 0;
            if (!frac)
                ++E;
        }
    }
    if (sticky) {
        chunk = chunk * 10 + 1;
        ++clen;
        ++nd;
        --E;
    }
    if (clen) {
        uint32_t m = 1;
        for (uint32_t j = 0; j < clen; ++j)
            m *= 10;
        lc_big_muladd(D, m, chunk);
    }
    if (p < b) {
        ++p;
        bool eneg = false;
        if (s[p] == '+' || s[p] == '-')
            eneg = s[p++] == '-';
        int64_t ev = 0;
        for (; p < b; ++p)
            if (ev < 100000000)
                ev = ev * 10 + (s[p] - '0');
        E += eneg ? -ev : ev;
    }
    const double zero = neg ? -0.0 : 0.0;
    if (nd == 0)
        return zero;
    const int64_t dexp = (int64_t)nd + E; // the value lies in [10^(dexp-1), 10^dexp)
    if (dexp > 310)
        return neg ? -lc_js_dbl(0x7FF0000000000000ull) : lc_js_dbl(0x7FF0000000000000ull);
    if (dexp < -323)
        return zero;
    // estimate: the first 19 digits times a power of ten, a few ulps off
    double x = (double)w19;
    for (int64_t e = E + (int64_t)nd - k19; e != 0;) {
        const int64_t st = e > 22 ? 22 : e < -22 ? -22 : e;
        double pw = 1.0;
        for (int64_t j = st < 0 ? -st : st; j > 0; --j)
            pw *= 10.0;
        x = st < 0 ? x / pw : x * pw;
        e -= st;
    }
    uint64_t u = lc_js_bits(x) & 0x7FFFFFFFFFFFFFFFull;
    if (u >= 0x7FF0000000000000ull)
        u = 0x7FEFFFFFFFFFFFFFull;
    const int32_t Ei = (int32_t)E;
    for (int it = 0; it < 4096; ++it) {
        const uint32_t be = (uint32_t)(u >> 52);
        const uint64_t m = be ? (u & 0xFFFFFFFFFFFFFull) | (1ull << 52) : u;
        const int32_t q = be ? (int32_t)be - 1075 : -1074;
        // the halfway point above: (2m + 1) * 2^(q - 1)
        int c = lc_js_cmp_mid(D, Ei, 2 * m + 1, q - 1, L, R);
        if (c > 0 || (c == 0 && (m & 1))) {
            if (u == 0x7FEFFFFFFFFFFFFFull) {
                u = 0x7FF0000000000000ull;
                break;
            }
            ++u;
            continue;
        }
        if (u == 0)
            break;
        // the halfway point below; the gap below a power of two is half as wide (except at the smallest normal)
        c = (m == (1ull << 52) && be > 1) ? lc_js_cmp_mid(D, Ei, 4 * m - 1, q - 2, L, R)
                                          : lc_js_cmp_mid(D, Ei, 2 * m - 1, q - 1, L, R);
        if (c < 0 || (c == 0 && (m & 1))) {
            --u;
            continue;
        }
        break;
    }
    return lc_js_dbl(u | (neg ? 0x8000000000000000ull : 0ull));
}

// Appends "%f" of the finite x to the arena at `at` (EMIT) and returns its length; LC_JSON_W_SLOW in *slow when the
// fast instantiation cannot print it (|x| >= 2^64).
template <bool SLOW, bool EMIT>
LC_HD uint32_t lc_js_printf(double x, LcJsonOut<EMIT>& o, uint32_t at, bool* slow) {
    const uint64_t bits = lc_js_bits(x);
    const bool neg = bits >> 63;
    const uint64_t u = bits & 0x7FFFFFFFFFFFFFFFull;
    const uint32_t be = (uint32_t)(u >> 52);
    uint32_t len = 0;
    if (neg)
        o.put(at + len++, '-');
    if (be >= 1023 + 64) { // |x| >= 2^64: an integer m << q with q >= 12
        if constexpr (!SLOW) {
            *slow = true;
            return 0;
        } else {
            LcJsBig B;
            lc_big_set(B, (u & 0xFFFFFFFFFFFFFull) | (1ull << 52));
            lc_big_shl(B, be - 1075);
            uint32_t ch[40], nc = 0;
            while (B.n && nc < 40)
                ch[nc++] = lc_big_div1e9(B);
            uint32_t nd = 1;
            for (uint32_t t = ch[nc - 1]; t >= 10; t /= 10)
                ++nd;
            for (uint32_t j = nd, t = ch[nc - 1]; j-- > 0; t /= 10)
                o.put(at + len + j, '0' + t % 10);
            len += nd;
            for (uint32_t c = nc - 1; c-- > 0;) {
                for (uint32_t j = 9, t = ch[c]; j-- > 0; t /= 10)
                    o.put(at + len + j, '0' + t % 10);
                len += 9;
            }
            for (uint32_t j = 0; j < 7; ++j)
                o.put(at + len++, j ? '0' : '.');
            return len;
        }
    }
    uint64_t ip = 0;
    uint32_t f6 = 0;
    if (u) {
        const uint64_t m = be ? (u & 0xFFFFFFFFFFFFFull) | (1ull << 52) : u;
        const int32_t q = be ? (int32_t)be - 1075 : -1074;
        if (q >= 0) {
            ip = m << q;
        } else {
            const uint32_t k = (uint32_t)-q;
            const uint64_t fr = k >= 64 ? m : m & ((1ull << k) - 1);
            ip = k >= 64 ? 0 : m >> k;
            if (k < 75) { // fr * 10^6 < 2^73: below 2^(k-1) from k = 75 on, so it rounds to 0
                const unsigned __int128 P = (unsigned __int128)fr * 1000000u;
                const unsigned __int128 half = (unsigned __int128)1 << (k - 1);
                f6 = (uint32_t)(P >> k);
                const unsigned __int128 rem = P & ((half << 1) - 1);
                if (rem > half || (rem == half && (f6 & 1)))
                    ++f6;
                if (f6 == 1000000) {
                    f6 = 0;
                    ++ip;
                }
            }
        }
    }
    uint32_t nd = 1;
    for (uint64_t t = ip; t >= 10; t /= 10)
        ++nd;
    uint64_t t = ip;
    for (uint32_t j = nd; j-- > 0; t /= 10)
        o.put(at + len + j, '0' + (uint32_t)(t % 10));
    len += nd;
    o.put(at + len++, '.');
    uint32_t f = f6;
    for (uint32_t j = 6; j-- > 0; f /= 10)
        o.put(at + len + j, '0' + f % 10);
    return len + 6;
}

// The bracket types of the open containers: bit k set for an object at depth k + 1 (the root object is bit 0).  The
// fast instantiation keeps LC_JSON_FAST_DEPTH bits in a register, the slow one LC_JSON_MAX_DEPTH in local memory.
template <bool SLOW>
struct LcJsStack {
    uint64_t b = 1;
    LC_HD void set(uint32_t k, bool obj) { b = (b & ~(1ull << k)) | ((uint64_t)obj << k); }
    LC_HD bool get(uint32_t k) const { return (b >> k) & 1u; }
};
template <>
struct LcJsStack<true> {
    uint32_t w[LC_JSON_MAX_DEPTH / 32] = {1};
    LC_HD void set(uint32_t k, bool obj) { w[k >> 5] = (w[k >> 5] & ~(1u << (k & 31))) | ((uint32_t)obj << (k & 31)); }
    LC_HD bool get(uint32_t k) const { return (w[k >> 5] >> (k & 31)) & 1u; }
};

// Skips the nested object or array whose opening bracket is s[p] (a member value of the root object, depth 2):
// *end receives the position after its closing bracket.  Bit d - 1 of the stack is set for an object at depth d.
template <bool SLOW>
LC_HD uint32_t lc_js_skip(const uint8_t* s, uint32_t n, uint32_t p, uint32_t* end) {
    constexpr uint32_t kMax = SLOW ? LC_JSON_MAX_DEPTH : LC_JSON_FAST_DEPTH;
    LcJsStack<SLOW> stk;
    uint32_t d = 1;
    bool need = true;
    LcJsPutNone none;
    for (;;) {
        if (need) {
            p = lc_js_ws(s, n, p);
            if (p >= n)
                return LC_JSON_W_FAIL;
            const uint32_t c = s[p];
            uint32_t ul;
            bool esc, isint;
            if (c == '{' || c == '[') {
                if (d == kMax)
                    return SLOW ? LC_JSON_W_FAIL : LC_JSON_W_SLOW;
                const bool obj = c == '{';
                stk.set(d, obj);
                ++d;
                p = lc_js_ws(s, n, p + 1);
                if (p >= n)
                    return LC_JSON_W_FAIL;
                if (s[p] == (obj ? '}' : ']')) {
                    ++p;
                    --d;
                    need = false;
                    continue;
                }
                if (obj) {
                    if (s[p] != '"' || !(p = lc_js_str(s, n, p + 1, &ul, &esc, none)))
                        return LC_JSON_W_FAIL;
                    p = lc_js_ws(s, n, p);
                    if (p >= n || s[p] != ':')
                        return LC_JSON_W_FAIL;
                    ++p;
                }
                continue;
            }
            if (c == '"') {
                if (!(p = lc_js_str(s, n, p + 1, &ul, &esc, none)))
                    return LC_JSON_W_FAIL;
            } else if (c == 't') {
                if (n - p < 4 || s[p + 1] != 'r' || s[p + 2] != 'u' || s[p + 3] != 'e')
                    return LC_JSON_W_FAIL;
                p += 4;
            } else if (c == 'f') {
                if (n - p < 5 || s[p + 1] != 'a' || s[p + 2] != 'l' || s[p + 3] != 's' || s[p + 4] != 'e')
                    return LC_JSON_W_FAIL;
                p += 5;
            } else if (c == 'n') {
                if (n - p < 4 || s[p + 1] != 'u' || s[p + 2] != 'l' || s[p + 3] != 'l')
                    return LC_JSON_W_FAIL;
                p += 4;
            } else if (c == '-' || (c >= '0' && c <= '9')) {
                if (!(p = lc_js_num(s, n, p, &isint)))
                    return LC_JSON_W_FAIL;
            } else {
                return LC_JSON_W_FAIL;
            }
        }
        // after a value inside the container at depth d
        if (d == 1) {
            *end = p;
            return LC_JSON_W_OK;
        }
        need = true;
        p = lc_js_ws(s, n, p);
        if (p >= n)
            return LC_JSON_W_FAIL;
        const bool obj = stk.get(d - 1);
        if (s[p] == ',') {
            ++p;
            if (obj) {
                uint32_t ul;
                bool esc;
                p = lc_js_ws(s, n, p);
                if (p >= n || s[p] != '"' || !(p = lc_js_str(s, n, p + 1, &ul, &esc, none)))
                    return LC_JSON_W_FAIL;
                p = lc_js_ws(s, n, p);
                if (p >= n || s[p] != ':')
                    return LC_JSON_W_FAIL;
                ++p;
            }
            continue;
        }
        if (s[p] == (obj ? '}' : ']')) {
            ++p;
            --d;
            need = false;
            continue;
        }
        return LC_JSON_W_FAIL;
    }
}

// The walk over one event's value s[0, n) (n > 0): LC_JSON_W_OK with o.nent members and o.narena arena bytes,
// LC_JSON_W_FAIL, or LC_JSON_W_SLOW (fast instantiation only: the event needs the slow one).
template <bool SLOW, bool EMIT>
LC_HD uint32_t lc_json_walk(const uint8_t* s, uint32_t n, const uint8_t* skey, uint32_t sklen, LcJsonOut<EMIT>& o) {
    LcJsPutNone none;
    uint32_t p = lc_js_ws(s, n, 0);
    if (p >= n || s[p] != '{')
        return LC_JSON_W_FAIL;
    p = lc_js_ws(s, n, p + 1);
    if (p < n && s[p] == '}') {
        ++p;
    } else {
        for (;;) {
            if (p >= n || s[p] != '"')
                return LC_JSON_W_FAIL;
            // the key
            const uint32_t k0 = p + 1;
            uint32_t kl, vl = 0, vo;
            bool kesc, vesc, isint;
            LcJsPutCmp cmp{skey, sklen, true};
            if (!(p = lc_js_str(s, n, k0, &kl, &kesc, cmp)))
                return LC_JSON_W_FAIL;
            if (cmp.eq && kl == sklen)
                o.skey_hit = true;
            uint32_t ko = o.base_off + k0;
            if (kesc) {
                ko = LC_JSON_ARENA | (o.arena_off + o.narena);
                if constexpr (EMIT) {
                    LcJsPutArena<EMIT> put{&o, o.narena};
                    lc_js_str(s, n, k0, &kl, &kesc, put);
                }
                o.grow(kl);
            }
            p = lc_js_ws(s, n, p);
            if (p >= n || s[p] != ':')
                return LC_JSON_W_FAIL;
            p = lc_js_ws(s, n, p + 1);
            if (p >= n)
                return LC_JSON_W_FAIL;
            // the value
            const uint32_t c = s[p], v0 = p;
            vo = o.base_off + v0;
            if (c == '"') {
                if (!(p = lc_js_str(s, n, v0 + 1, &vl, &vesc, none)))
                    return LC_JSON_W_FAIL;
                vo = o.base_off + v0 + 1;
                if (vesc) {
                    vo = LC_JSON_ARENA | (o.arena_off + o.narena);
                    if constexpr (EMIT) {
                        LcJsPutArena<EMIT> put{&o, o.narena};
                        lc_js_str(s, n, v0 + 1, &vl, &vesc, put);
                    }
                    o.grow(vl);
                }
            } else if (c == '{' || c == '[') {
                const uint32_t r = lc_js_skip<SLOW>(s, n, p, &p);
                if (r != LC_JSON_W_OK)
                    return r;
                vl = p - v0;
            } else if (c == 't') {
                if (n - p < 4 || s[p + 1] != 'r' || s[p + 2] != 'u' || s[p + 3] != 'e')
                    return LC_JSON_W_FAIL;
                p += 4;
                vl = 4;
            } else if (c == 'f') {
                if (n - p < 5 || s[p + 1] != 'a' || s[p + 2] != 'l' || s[p + 3] != 's' || s[p + 4] != 'e')
                    return LC_JSON_W_FAIL;
                p += 5;
                vl = 5;
            } else if (c == 'n') {
                if (n - p < 4 || s[p + 1] != 'u' || s[p + 2] != 'l' || s[p + 3] != 'l')
                    return LC_JSON_W_FAIL;
                p += 4;
            } else if (c == '-' || (c >= '0' && c <= '9')) {
                if (!(p = lc_js_num(s, n, p, &isint)))
                    return LC_JSON_W_FAIL;
                if (isint) {
                    // "%" PRId64 / "%" PRIu64 of an integer in range is its own text, but for "-0"; else empty
                    const bool neg = c == '-';
                    const uint32_t d0 = v0 + (neg ? 1u : 0u), nd = p - d0;
                    if (neg ? (nd < 19 || (nd == 19 && lc_js_digits_le(s, d0, "9223372036854775808", 19)))
                            : (nd < 20 || (nd == 20 && lc_js_digits_le(s, d0, "18446744073709551615", 20)))) {
                        if (neg && nd == 1 && s[d0] == '0') {
                            vo = o.base_off + d0;
                            vl = 1;
                        } else {
                            vl = p - v0;
                        }
                    }
                } else {
                    double x;
                    if (!lc_js_dec_fast(s, v0, p, o.pow5, &x)) {
                        if constexpr (!SLOW)
                            return LC_JSON_W_SLOW;
                        else
                            x = lc_js_dec_slow(s, v0, p);
                    }
                    if ((lc_js_bits(x) & 0x7FFFFFFFFFFFFFFFull) < 0x7FF0000000000000ull) { // infinity renders empty
                        bool slow = false;
                        vl = lc_js_printf<SLOW, EMIT>(x, o, o.narena, &slow);
                        if (slow)
                            return LC_JSON_W_SLOW;
                        vo = LC_JSON_ARENA | (o.arena_off + o.narena);
                        o.grow(vl);
                    }
                }
            } else {
                return LC_JSON_W_FAIL;
            }
            o.entry(ko, kl, vo, vl);
            p = lc_js_ws(s, n, p);
            if (p < n && s[p] == ',') {
                p = lc_js_ws(s, n, p + 1);
                continue;
            }
            if (p < n && s[p] == '}') {
                ++p;
                break;
            }
            return LC_JSON_W_FAIL;
        }
    }
    p = lc_js_ws(s, n, p);
    return p < n && s[p] != 0 ? LC_JSON_W_FAIL : LC_JSON_W_OK;
}

// One event of the count pass: its status, entry count and arena bytes; *slow when the fast instantiation gave up.
// len == LC_JSON_NO_KEY: no SourceKey; an empty value is LC_JSON_ST_EMPTY.  The caller has checked the range.
template <bool SLOW>
LC_HD uint32_t lc_json_count(const uint8_t* base, uint32_t off, uint32_t len, const uint8_t* skey, uint32_t sklen,
                             const uint64_t* pow5, uint32_t* nent, uint32_t* narena, bool* slow) {
    *nent = *narena = 0;
    *slow = false;
    if (len == LC_JSON_NO_KEY)
        return LC_JSON_ST_NOT_FOUND;
    if (len == 0)
        return LC_JSON_ST_EMPTY;
    LcJsonOut<false> o{pow5, nullptr, nullptr, 0, 0, off, 0, 0, 0, false, false};
    const uint32_t r = lc_json_walk<SLOW, false>(base + off, len, skey, sklen, o);
    if (r == LC_JSON_W_SLOW) {
        *slow = true;
        return LC_JSON_ST_FAILED;
    }
    if (r != LC_JSON_W_OK)
        return LC_JSON_ST_FAILED;
    *nent = o.nent;
    *narena = o.narena;
    return LC_JSON_ST_OK | (o.skey_hit ? LC_JSON_ST_OVER : 0u);
}

// One event of the emit pass into its ranges ent[0, ent_cap) and arena[0, arena_cap) (arena_off: the range's start in
// the arena); false when the walk does not fill them exactly (nothing is written past them).
template <bool SLOW>
LC_HD bool lc_json_emit(const uint8_t* base, uint32_t off, uint32_t len, const uint8_t* skey, uint32_t sklen,
                        const uint64_t* pow5, LcJsonEntry* ent, uint32_t ent_cap, uint8_t* arena, uint32_t arena_off, uint32_t arena_cap) {
    LcJsonOut<true> o{pow5, ent, arena, ent_cap, arena_cap, off, arena_off, 0, 0, false, false};
    const uint32_t r = lc_json_walk<SLOW, true>(base + off, len, skey, sklen, o);
    return r == LC_JSON_W_OK && !o.over && o.nent == ent_cap && o.narena == arena_cap;
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> JSON chain: the Log record of piece k that ProcessorSplitLogStringNative /
// ProcessorSplitMultilineLogStringNative followed by ProcessorParseJsonNative (same SourceKey) leave behind, written
// straight from the piece tables of the splitter and the tables of lc_json_parse_dev over those pieces.  The piece
// enters the JSON stage as [SourceKey -> piece] or, with log.file.offset metadata, [SourceKey -> piece, offset_key ->
// decimal(src_pos + off[k])], and AddLog overwrites in place, so the record of a parsed piece is: SourceKey (when a
// member has it), the offset content, then every other distinct member key in order of its first occurrence, each
// with the value of its last occurrence, then RenamedSourceKey unless that key is present.  The keys come from the
// data, so a resolve pass finds, per event, which member emits and which value it takes (lc_json_resolve_*).
#define LC_JSON_SLS_NONE 0xFFFFFFFFu
#define LC_JSON_SLS_WARP 32u // events of at most this many members resolve in one warp, larger ones by sorting

struct LcSplitJsonSlsCfg {
    const uint8_t* skey; // SourceKey, RenamedSourceKey, the offset key and "__raw_log__" (device copies on the
    const uint8_t* rkey; // device: a string literal here would add a module global and move the existing kernels'
    const uint8_t* okey; // constant-bank address slots)
    const uint8_t* raw;
    uint32_t sklen, rklen, oklen;
    uint32_t has_offset;
    uint32_t keep_fail, keep_succeed, copy_raw;
    uint32_t ren_is_off; // RenamedSourceKey == offset key (with offset metadata: always present)
    uint32_t raw_is_off; // "__raw_log__" == offset key
    uint32_t ren_is_raw; // RenamedSourceKey == "__raw_log__"
    uint64_t src_pos;    // the source event's file offset
    uint32_t time;       // the source event's time, as the split events inherit it
    uint32_t has_ns, ns;
};

// What the resolve pass found about one event's members: the entry (index in the event) whose value SourceKey and the
// offset key take (LC_JSON_SLS_NONE: no member has that key), and whether a member is keyed RenamedSourceKey.
// "__raw_log__" is only added to failed pieces, which have no members, so it needs no flag.
struct LcJsonSlsEv {
    uint32_t src_win, off_win, has_ren;
};

// FNV-1a of a rendered key: the resolve compares keys only inside runs of equal hashes
struct LcJsonKeyHash {
    LC_HD uint32_t operator()(const uint8_t* p, uint32_t n) const {
        uint32_t h = 2166136261u;
        for (uint32_t i = 0; i < n; ++i)
            h = (h ^ p[i]) * 16777619u;
        return h;
    }
};

// the bytes an entry offset names: the source, or (LC_JSON_ARENA) the arena
LC_HD const uint8_t* lc_json_span(const uint8_t* src, const uint8_t* arena, uint32_t o) {
    return o & LC_JSON_ARENA ? arena + (o & ~LC_JSON_ARENA) : src + o;
}

// <0, 0, >0: byte order, then length
LC_HD int lc_json_key_cmp(const uint8_t* a, uint32_t al, const uint8_t* b, uint32_t bl) {
    const uint32_t n = al < bl ? al : bl;
    for (uint32_t i = 0; i < n; ++i)
        if (a[i] != b[i])
            return a[i] < b[i] ? -1 : 1;
    return al == bl ? 0 : (al < bl ? -1 : 1);
}

// bit 0: SourceKey, bit 1: the offset key (with offset metadata), bit 2: RenamedSourceKey
LC_HD uint32_t lc_json_sls_special(const LcSplitJsonSlsCfg& c, const uint8_t* k, uint32_t kl) {
    return (lc_json_key_cmp(k, kl, c.skey, c.sklen) == 0 ? 1u : 0u) |
           (c.has_offset && lc_json_key_cmp(k, kl, c.okey, c.oklen) == 0 ? 2u : 0u) |
           (lc_json_key_cmp(k, kl, c.rkey, c.rklen) == 0 ? 4u : 0u);
}

// Per-warp workspace of lc_json_resolve_warp (shared memory on the device)
struct LcJsonResolveWarp {
    uint32_t h[32], lead[32], win[32], sp[32];
};

// Resolve one event of m <= 32 members e[0, m) in one warp, lane l holding member l: __match_any_sync on the key hash
// gives each lane its candidates, and a byte compare with the earlier ones finds the first member of its key (its
// leader); a second match on the leader gives the key's members, the last of which holds the value.  win[l] = that
// last member at the leader of every key other than SourceKey and the offset key, else LC_JSON_SLS_NONE; *ev as
// LcJsonSlsEv says.  Every lane calls it (the host runs the 32 lanes in turn, lc_lz4_peers standing in for the match).
template <class H>
LC_HD void lc_json_resolve_warp(const LcSplitJsonSlsCfg& c, const uint8_t* src, const uint8_t* arena,
                                const LcJsonEntry* e, uint32_t m, uint32_t* win, LcJsonSlsEv* ev, LcJsonResolveWarp& w,
                                uint32_t lane) {
    const uint32_t W = 32;
    (void)lane;
    const uint32_t valid = lc_low_bits(m);
    LC_LANES(l) {
        w.h[l] = l < m ? H()(lc_json_span(src, arena, e[l].key_off), e[l].key_len) : 0u;
    }
    LC_WARP_SYNC();
    LC_LANES(l) {
        const uint32_t below = lc_lz4_peers(w.h, l, W) & valid & lc_low_bits(l);
        uint32_t lead = l;
        if (l < m) {
            const uint8_t* k = lc_json_span(src, arena, e[l].key_off);
            for (uint32_t b = below; b; b &= b - 1) {
                const uint32_t j = lc_lo_bit(b);
                if (lc_json_key_cmp(k, e[l].key_len, lc_json_span(src, arena, e[j].key_off), e[j].key_len) == 0) {
                    lead = j;
                    break;
                }
            }
        }
        w.lead[l] = lead;
    }
    LC_WARP_SYNC();
    LC_LANES(l) {
        const uint32_t grp = lc_lz4_peers(w.lead, l, W) & valid;
        uint32_t wn = LC_JSON_SLS_NONE, sp = 0;
        if (l < m && w.lead[l] == l) {
            wn = lc_hi_bit(grp);
            sp = lc_json_sls_special(c, lc_json_span(src, arena, e[l].key_off), e[l].key_len);
        }
        w.win[l] = wn;
        w.sp[l] = sp;
        if (l < m)
            win[l] = sp & 3u ? LC_JSON_SLS_NONE : wn;
    }
    LC_WARP_SYNC();
    LC_LANES(l) {
        if (l == 0) {
            LcJsonSlsEv r{LC_JSON_SLS_NONE, LC_JSON_SLS_NONE, 0u};
            for (uint32_t j = 0; j < m; ++j) {
                if (w.sp[j] & 1u)
                    r.src_win = w.win[j];
                if (w.sp[j] & 2u)
                    r.off_win = w.win[j];
                if (w.sp[j] & 4u)
                    r.has_ren = 1u;
            }
            *ev = r;
        }
    }
}

// member x before member y: by key hash, then key bytes, then position
LC_HD bool lc_json_resolve_less(const uint8_t* src, const uint8_t* arena, const LcJsonEntry* e, const uint32_t* h,
                                uint32_t x, uint32_t y) {
    if (h[x] != h[y])
        return h[x] < h[y];
    const int k = lc_json_key_cmp(lc_json_span(src, arena, e[x].key_off), e[x].key_len,
                                  lc_json_span(src, arena, e[y].key_off), e[y].key_len);
    return k ? k < 0 : x < y;
}

// Resolve one event of any member count in one thread, with the outputs of lc_json_resolve_warp: a bottom-up merge
// sort of the member indices by (hash, key bytes, index) puts each key's members next to each other in document order,
// so the first of a run is the leader and the last holds the value.  O(m log m) key comparisons whatever the hashes
// (equal hashes only fall through to the byte compare); h, a, b: m words of scratch each.
template <class H>
LC_HD void lc_json_resolve_sort(const LcSplitJsonSlsCfg& c, const uint8_t* src, const uint8_t* arena,
                                const LcJsonEntry* e, uint32_t m, uint32_t* win, LcJsonSlsEv* ev, uint32_t* h,
                                uint32_t* a, uint32_t* b) {
    for (uint32_t j = 0; j < m; ++j) {
        h[j] = H()(lc_json_span(src, arena, e[j].key_off), e[j].key_len);
        a[j] = j;
    }
    for (uint32_t run = 1; run < m; run *= 2) {
        for (uint32_t lo = 0; lo < m; lo += 2 * run) {
            const uint32_t mid = lo + run < m ? lo + run : m, hi = mid + run < m ? mid + run : m;
            uint32_t p = lo, q = mid, o = lo;
            while (p < mid && q < hi)
                b[o++] = lc_json_resolve_less(src, arena, e, h, a[q], a[p]) ? a[q++] : a[p++];
            while (p < mid)
                b[o++] = a[p++];
            while (q < hi)
                b[o++] = a[q++];
        }
        uint32_t* t = a;
        a = b;
        b = t;
    }
    LcJsonSlsEv r{LC_JSON_SLS_NONE, LC_JSON_SLS_NONE, 0u};
    for (uint32_t s = 0, t; s < m; s = t) {
        const uint32_t lead = a[s];
        const uint8_t* k = lc_json_span(src, arena, e[lead].key_off);
        for (t = s + 1; t < m && h[a[t]] == h[lead] &&
                        lc_json_key_cmp(lc_json_span(src, arena, e[a[t]].key_off), e[a[t]].key_len, k,
                                        e[lead].key_len) == 0;
             ++t)
            win[a[t]] = LC_JSON_SLS_NONE;
        const uint32_t wn = a[t - 1], sp = lc_json_sls_special(c, k, e[lead].key_len);
        win[lead] = sp & 3u ? LC_JSON_SLS_NONE : wn;
        if (sp & 1u)
            r.src_win = wn;
        if (sp & 2u)
            r.off_win = wn;
        if (sp & 4u)
            r.has_ren = 1u;
    }
    *ev = r;
}

// One piece: src[po, + plen), its JSON status, its m entries e (offsets into src or the arena), the resolve's win[m]
// and event record.
struct LcSplitJsonSlsRow {
    uint32_t po, plen;
    uint32_t status;
    const LcJsonEntry* e;
    const uint32_t* win;
    uint32_t m;
    LcJsonSlsEv ev;
};

// The body of the piece's Log record -- Time, its contents, Time_ns -- into sink s (LcSlsCount64 / LcSlsWrite), with
// the record's own time and ns (has_ns = 0: no Time_ns).  Returns the number of contents; 0 = erased or empty, no
// record.
template <class S>
LC_HD uint32_t lc_split_json_sls_body(const LcSplitJsonSlsCfg& c, const uint8_t* src, const uint8_t* arena,
                                      const LcSplitJsonSlsRow& r, uint32_t time, uint32_t has_ns, uint32_t ns, S& s) {
    {
        uint8_t h[6];
        h[0] = 0x08;
        const uint32_t n = 1 + lc_put_varint(h + 1, time < (1u << 28) ? (1u << 28) : time); // always 5 bytes
        s.put(h, n);
    }
    const uint64_t pos = c.src_pos + r.po;
    const uint32_t nd = lc_dec_digits(pos);
    uint32_t k = 0;
    auto member = [&](const uint8_t* key, uint32_t kl, const LcJsonEntry& v) {
        lc_sls_pair_open(s, key, kl, v.val_len);
        s.copy(lc_json_span(src, arena, v.val_off), v.val_len);
        ++k;
    };
    auto digits = [&]() {
        lc_sls_pair_open(s, c.okey, c.oklen, nd);
        lc_sls_digits(s, pos, nd);
        ++k;
    };
    auto piece = [&](const uint8_t* key, uint32_t kl) {
        lc_sls_pair_open(s, key, kl, r.plen);
        s.copy(src + r.po, r.plen);
        ++k;
    };
    if ((r.status & 0x7Fu) == LC_JSON_ST_OK) {
        if (r.ev.src_win != LC_JSON_SLS_NONE)
            member(c.skey, c.sklen, r.e[r.ev.src_win]);
        if (c.has_offset) {
            if (r.ev.off_win != LC_JSON_SLS_NONE)
                member(c.okey, c.oklen, r.e[r.ev.off_win]);
            else
                digits();
        }
        for (uint32_t j = 0; j < r.m; ++j)
            if (r.win[j] != LC_JSON_SLS_NONE)
                member(lc_json_span(src, arena, r.e[j].key_off), r.e[j].key_len, r.e[r.win[j]]);
        if (c.keep_succeed && !r.ev.has_ren && !(c.has_offset && c.ren_is_off))
            piece(c.rkey, c.rklen);
    } else {
        if (!c.keep_fail)
            return 0u; // ShouldEraseEvent: nothing but the offset content is left
        if (c.has_offset)
            digits();
        if (!(c.has_offset && c.ren_is_off))
            piece(c.rkey, c.rklen);
        if (c.copy_raw && !(c.has_offset && c.raw_is_off) && !c.ren_is_raw)
            piece(c.raw, 11u);
    }
    if (has_ns) {
        const uint8_t h[5] = {0x25, (uint8_t)ns, (uint8_t)(ns >> 8), (uint8_t)(ns >> 16), (uint8_t)(ns >> 24)};
        s.put(h, 5);
    }
    return k;
}

// ... with the source event's time and ns, as every split piece inherits them
template <class S>
LC_HD uint32_t lc_split_json_sls_body(const LcSplitJsonSlsCfg& c, const uint8_t* src, const uint8_t* arena,
                                      const LcSplitJsonSlsRow& r, S& s) {
    return lc_split_json_sls_body(c, src, arena, r, c.time, c.has_ns, c.ns, s);
}

// The piece's counter verdicts (0 / 1): ProcessorParseJsonNative's out_successful (every piece not erased),
// out_failed (LC_JSON_FAILED only) and discarded.  A split event always holds SourceKey, so no key-not-found.
LC_HD LcSplitRegexVerdict lc_split_json_verdict(const LcSplitJsonSlsCfg& c, uint32_t status) {
    const uint32_t st = status & 0x7Fu, kept = st == LC_JSON_ST_OK || c.keep_fail;
    return {kept, st == LC_JSON_ST_FAILED ? 1u : 0u, kept ? 0u : 1u};
}

// Host side: the configuration of the chain, with the key pointers as given and `raw` at a host "__raw_log__" (the
// device caller points them at its copies).
// offset_key == nullptr: no log.file.offset metadata.  Returns nullptr, or why the chain is refused: an offset key
// equal to SourceKey (the split would replace the piece by its digits, and the JSON stage would parse those).
inline const char* lc_split_json_sls_setup(const char* source_key, uint32_t source_len, const char* renamed_key,
                                           uint32_t renamed_len, const char* offset_key, uint32_t offset_len,
                                           int keep_fail, int keep_succeed, int copy_raw, uint64_t src_pos,
                                           uint32_t time, uint32_t time_ns, LcSplitJsonSlsCfg* c) {
    auto eq = [](const char* a, uint32_t al, const char* b, uint32_t bl) {
        return al == bl && (al == 0 || !memcmp(a, b, al));
    };
    if (!c)
        return "bad arguments";
    if (offset_key && eq(offset_key, offset_len, source_key, source_len))
        return "the offset key equals SourceKey";
    memset(c, 0, sizeof *c);
    c->skey = reinterpret_cast<const uint8_t*>(source_key);
    c->rkey = reinterpret_cast<const uint8_t*>(renamed_key);
    c->okey = reinterpret_cast<const uint8_t*>(offset_key);
    c->raw = reinterpret_cast<const uint8_t*>("__raw_log__");
    c->sklen = source_len;
    c->rklen = renamed_len;
    c->oklen = offset_key ? offset_len : 0u;
    c->has_offset = offset_key != nullptr;
    c->keep_fail = keep_fail != 0;
    c->keep_succeed = keep_succeed != 0;
    c->copy_raw = copy_raw != 0;
    c->ren_is_off = offset_key && eq(renamed_key, renamed_len, offset_key, offset_len);
    c->raw_is_off = offset_key && eq("__raw_log__", 11, offset_key, offset_len);
    c->ren_is_raw = eq(renamed_key, renamed_len, "__raw_log__", 11);
    c->src_pos = src_pos;
    c->time = time;
    c->has_ns = time_ns != 0xFFFFFFFFu;
    c->ns = c->has_ns ? time_ns : 0u;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> JSON -> timestamp chain: ProcessorParseTimestampNative (ProcessorParseTimestampNative.cpp:100-235, the
// SourceKey tkey) behind the split -> JSON chain, whose pieces and JSON stage are unchanged.
//   - The timestamp stage sees the pieces the JSON stage kept, in piece order, as one group: a piece the JSON stage
//     erased is not an event of the stage (no counter, no cache step).
//   - Its value under tkey (keys compare by their rendered bytes): in a parsed piece, the rendered value of the LAST
//     member keyed tkey, else the piece when tkey is RenamedSourceKey with keep_succeed, else none; in a kept failure,
//     the piece when tkey is RenamedSourceKey, or "__raw_log__" with copy_raw, else none.  tkey equal to the offset key
//     is refused.  Both an erased piece and no value give the tap's LC_TS_NO_KEY; the counters come from the size
//     pass, which tells the two apart.
//   - A value lies in the chunk (a member span or the piece) or in the arena (escaped strings, %f renderings), and the
//     timestamp passes read one base: the tap copies each value into a buffer of src_len + arena bytes, a chunk value
//     to its own offset and an arena value to src_len + its arena offset.  Pieces and arena spans are disjoint, so no
//     two values share bytes.  The value is read over [off, off + len) followed by NUL bytes, as every timestamp value
//     is.
//   - The record's time is lc_split_regex_ts_time's rule: LC_TS_OK sets Time (and Time_ns with enable_ns),
//     LC_TS_NOT_FOUND / LC_TS_FAILED keep the source event's, LC_TS_DISCARDED leaves no record.
struct LcSplitJsonTsCfg {
    const uint8_t* tkey; // the timestamp stage's SourceKey (a device copy on the device, as LcSplitJsonSlsCfg's keys)
    uint32_t tklen;
    uint32_t piece_ok;   // a parsed piece without a member keyed tkey holds the piece under tkey
    uint32_t piece_fail; // a kept failure holds the piece under tkey
    uint32_t enable_ns;  // mEnableTimestampNanosecond: a parsed time writes Time_ns
    uint64_t arena_at;   // where the arena's bytes start in the value buffer (src_len)
    uint64_t val_cap;    // the value buffer's size: a value that would not fit gets no value
};

// Host side: check tkey and the source Time_ns against the chain's configuration c, as lc_split_json_sls_setup left
// it (key pointers on the host).  Returns nullptr, or why the chain is refused: tkey equal to the offset key (the
// value would be the offset digits or an offset member), or a source Time_ns without enable_ns.
inline const char* lc_split_json_ts_setup(const LcSplitJsonSlsCfg& c, const char* tkey, uint32_t tkey_len,
                                          int enable_ns, LcSplitJsonTsCfg* t) {
    if (!t || (tkey_len && !tkey))
        return "bad arguments";
    const char* why = lc_split_regex_ts_ns_check(c, enable_ns);
    if (why)
        return why;
    const uint8_t* k = reinterpret_cast<const uint8_t*>(tkey);
    if (c.has_offset && lc_json_key_cmp(k, tkey_len, c.okey, c.oklen) == 0)
        return "the timestamp key equals the offset key";
    memset(t, 0, sizeof *t);
    t->tkey = k;
    t->tklen = tkey_len;
    const bool ren = lc_json_key_cmp(k, tkey_len, c.rkey, c.rklen) == 0;
    t->piece_ok = ren && c.keep_succeed;
    t->piece_fail = ren || (c.copy_raw && lc_json_key_cmp(k, tkey_len, c.raw, 11u) == 0);
    t->enable_ns = enable_ns != 0;
    return nullptr;
}

// The last of a parsed piece's m members e[0, m) whose key is tkey (LC_JSON_SLS_NONE: none), W lanes scanning W
// members per step from the last one backward; v: W words of per-warp scratch (shared memory on the device).  Every
// lane calls it and gets the same answer.
LC_HD uint32_t lc_json_ts_last_member(const LcSplitJsonTsCfg& t, const uint8_t* src, const uint8_t* arena,
                                      const LcJsonEntry* e, uint32_t m, uint32_t* v, uint32_t lane, uint32_t W) {
    for (uint32_t top = m; top > 0;) {
        const uint32_t nv = top < W ? top : W;
        LC_LANES(l) {
            uint32_t hit = 0;
            if (l < nv) {
                const LcJsonEntry& x = e[top - 1 - l];
                hit = x.key_len == t.tklen &&
                      lc_json_key_cmp(lc_json_span(src, arena, x.key_off), x.key_len, t.tkey, t.tklen) == 0;
            }
            v[l] = hit;
        }
        const uint32_t b = lc_lz4_ballot(v, lane, W);
        LC_WARP_SYNC();
        if (b)
            return top - 1 - lc_lo_bit(b);
        top -= nv;
    }
    return LC_JSON_SLS_NONE;
}

// The tap's value of one piece (its JSON status, the piece src[po, + plen), its entries e and lc_json_ts_last_member's
// answer w): *from = where its bytes are (an entry offset: LC_JSON_ARENA tags the arena), *off / *len = where the
// timestamp passes read it in the value buffer; *len = LC_TS_NO_KEY when the JSON stage erased the piece or left no
// value under tkey.
LC_HD void lc_split_json_ts_value(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& t, uint32_t status, uint32_t po,
                                  uint32_t plen, const LcJsonEntry* e, uint32_t w, uint32_t* from, uint32_t* off,
                                  uint32_t* len) {
    const bool ok = (status & 0x7Fu) == LC_JSON_ST_OK;
    *from = *off = 0;
    *len = LC_TS_NO_KEY;
    uint32_t vo, vl;
    if (!ok && !c.keep_fail)
        return; // erased: no event of the stage
    if (ok && w != LC_JSON_SLS_NONE)
        vo = e[w].val_off, vl = e[w].val_len;
    else if (ok ? t.piece_ok : t.piece_fail)
        vo = po, vl = plen;
    else
        return;
    const uint64_t at = vo & LC_JSON_ARENA ? t.arena_at + (vo & ~LC_JSON_ARENA) : (uint64_t)vo;
    if (at + vl > t.val_cap)
        return;
    *from = vo;
    *off = (uint32_t)at;
    *len = vl;
}

// The record's time after the timestamp stage (ts: the stage's LC_TS_ST_* of the row, sec / nsec its time)
LC_HD LcSplitRegexTsTime lc_split_json_ts_time(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& t, uint32_t ts,
                                               int64_t sec, uint32_t nsec) {
    if (ts == LC_TS_ST_OK)
        return {1u, (uint32_t)sec, t.enable_ns, nsec};
    return {ts != LC_TS_ST_DISCARDED, c.time, c.has_ns, c.ns};
}

// The row's counter verdicts as bits of the LC_SRTS_COUNTERS counters: the JSON stage's (lc_split_json_verdict), then
// -- when the JSON stage kept the piece -- the timestamp stage's five.
LC_HD uint32_t lc_split_json_ts_verdict(const LcSplitJsonSlsCfg& c, uint32_t status, uint32_t ts) {
    return lc_split_ts_verdict_bits(lc_split_json_verdict(c, status), ts);
}

// ------------------------------------------------------------------------------------------------------------
// f4, split -> Apsara chain: the Log record of piece k that ProcessorSplitLogStringNative /
// ProcessorSplitMultilineLogStringNative followed by ProcessorParseApsaraNative (same SourceKey) leave behind, written
// straight from the piece tables of the splitter and the tables of lc_apsara_parse_dev over those pieces (the chunk as
// its base, one group).  The piece enters the Apsara stage as [SourceKey -> piece] or, with log.file.offset metadata,
// [SourceKey -> piece, offset_key -> decimal(src_pos + off[k])].  AppendContentNoCopy never removes a duplicate, so the
// record of a parsed piece is those two, the base fields, the key:value fields and "microtime" in append order, less
// the one entry DelContent(SourceKey) removes (the newest live one with that key), plus RenamedSourceKey unless some
// live content has that key.  The rule is pinned in include/lc_b200.h above lc_sls_serialize_split_apsara_dev.
//
// The fixed key names, back to back: "__raw_log__" (0, 11), "microtime" (11, 9), then the base fields' names in
// LC_AP_K_* order.  The device reads the engine's copy through LcSplitApsaraSlsCfg::names: a string literal in device
// code would add a module global and move the existing kernels' constant-bank address slots.
#define LC_AP_SLS_NAMES "__raw_log__microtime__LEVEL____THREAD____FILE____LINE__"
#define LC_AP_SLS_NAMES_LEN 55u
#define LC_AP_SLS_NONE 0xFFu // no base field has that name
#define LC_AP_SLS_COUNTERS 5 // lc_apsara_parse's order: key_not_found, out_failed, history_failure, discarded, ok

// offset and length in LC_AP_SLS_NAMES of base field t (key_off - LC_AP_K_LEVEL)
LC_HD uint32_t lc_ap_sls_base_at(uint32_t t) { return t == 0u ? 20u : t == 1u ? 29u : t == 2u ? 39u : 47u; }
LC_HD uint32_t lc_ap_sls_base_len(uint32_t t) { return t == 0u ? 9u : t == 1u ? 10u : 8u; }

struct LcSplitApsaraSlsCfg {
    const uint8_t* skey;  // SourceKey, RenamedSourceKey, the offset key and LC_AP_SLS_NAMES (device copies on the
    const uint8_t* rkey;  // device, see above)
    const uint8_t* okey;
    const uint8_t* names;
    uint32_t sklen, rklen, oklen;
    uint32_t has_offset;
    uint32_t keep_fail, keep_succeed, copy_raw;
    uint32_t enable_ns;  // mEnableTimestampNanosecond: a parsed piece writes its Time_ns
    uint32_t sk_base;    // the base field named SourceKey (0..3), else LC_AP_SLS_NONE
    uint32_t sk_micro;   // SourceKey == "microtime"
    uint32_t rk_base;    // the base field named RenamedSourceKey, else LC_AP_SLS_NONE
    uint32_t rk_sk;      // RenamedSourceKey == SourceKey
    uint32_t rk_off;     // RenamedSourceKey == the offset key (with offset metadata)
    uint32_t rk_micro;   // RenamedSourceKey == "microtime"
    uint32_t rk_raw;     // RenamedSourceKey == "__raw_log__"
    uint32_t raw_off;    // "__raw_log__" == the offset key (with offset metadata)
    uint64_t src_pos;    // the source event's file offset
    uint32_t time;       // the source event's time, as the split events inherit it
    uint32_t has_ns, ns; // ... and its Time_ns as the serialiser writes it
};

// One piece: src[po, + plen), lc_apsara_parse_dev's status / sec / nsec / micro of it, and its m entries e (offsets
// into src; only a parsed piece has any).
struct LcSplitApsaraSlsRow {
    uint32_t po, plen;
    uint32_t status;
    int64_t sec;
    uint32_t nsec;
    int64_t micro;
    const LcApEntry* e;
    uint32_t m;
};

// whether a base field of the piece has tag t (the base fields come first, at most four)
LC_HD bool lc_ap_sls_has_base(const LcSplitApsaraSlsRow& r, uint32_t t) {
    for (uint32_t j = 0; j < r.m && r.e[j].key_off >= LC_AP_K_LEVEL; ++j)
        if (r.e[j].key_off - LC_AP_K_LEVEL == t)
            return true;
    return false;
}

// The body of the piece's Log record -- Time, its contents, Time_ns -- into sink s (LcSlsCount64 / LcSlsWrite).
// Returns the number of contents; 0 = erased, no record.
template <class S>
LC_HD uint32_t lc_split_apsara_sls_body(const LcSplitApsaraSlsCfg& c, const uint8_t* src, const LcSplitApsaraSlsRow& r,
                                        S& s) {
    const uint32_t st = r.status & 7u;
    const bool ok = st == LC_AP_ST_OK, kept = ok || st == LC_AP_ST_EMPTY || st == LC_AP_ST_NOT_FOUND;
    if (st == LC_AP_ST_DISCARDED || (!kept && !c.keep_fail))
        return 0u; // too old, or ShouldEraseEvent: nothing but the offset content is left
    {
        const uint32_t t = ok ? (uint32_t)r.sec : c.time;
        uint8_t h[6];
        h[0] = 0x08;
        const uint32_t n = 1 + lc_put_varint(h + 1, t < (1u << 28) ? (1u << 28) : t); // always 5 bytes
        s.put(h, n);
    }
    const uint64_t pos = c.src_pos + r.po;
    const uint32_t nd = lc_dec_digits(pos);
    uint32_t k = 0;
    auto piece = [&](const uint8_t* key, uint32_t kl) {
        lc_sls_pair_open(s, key, kl, r.plen);
        s.copy(src + r.po, r.plen);
        ++k;
    };
    auto digits = [&]() {
        lc_sls_pair_open(s, c.okey, c.oklen, nd);
        lc_sls_digits(s, pos, nd);
        ++k;
    };
    if (ok) {
        // DelContent(SourceKey) unless a key:value key is SourceKey: "microtime", else a base field, else the piece
        enum : uint32_t { DEL_NONE, DEL_PIECE, DEL_MICRO, DEL_BASE };
        uint32_t del = DEL_NONE;
        if (!(r.status & LC_AP_ST_OVER)) {
            if (c.sk_micro)
                del = DEL_MICRO;
            else if (c.sk_base != LC_AP_SLS_NONE && lc_ap_sls_has_base(r, c.sk_base))
                del = DEL_BASE;
            else
                del = DEL_PIECE;
        }
        if (del != DEL_PIECE)
            piece(c.skey, c.sklen);
        if (c.has_offset)
            digits();
        for (uint32_t j = 0; j < r.m; ++j) {
            const LcApEntry& x = r.e[j];
            if (x.key_off >= LC_AP_K_LEVEL) {
                const uint32_t t = x.key_off - LC_AP_K_LEVEL;
                if (del == DEL_BASE && t == c.sk_base)
                    continue;
                lc_sls_pair_open(s, c.names + lc_ap_sls_base_at(t), lc_ap_sls_base_len(t), x.val_len);
            } else {
                lc_sls_pair_open(s, src + x.key_off, x.key_len, x.val_len);
            }
            s.copy(src + x.val_off, x.val_len);
            ++k;
        }
        if (del != DEL_MICRO) {
            const bool neg = r.micro < 0; // "%ld": a wrapped logTime_in_micro renders negative
            const uint64_t mag = neg ? 0u - (uint64_t)r.micro : (uint64_t)r.micro;
            const uint32_t md = lc_dec_digits(mag);
            lc_sls_pair_open(s, c.names + 11, 9u, md + (neg ? 1u : 0u));
            if (neg) {
                const uint8_t minus = '-';
                s.put(&minus, 1);
            }
            lc_sls_digits(s, mag, md);
            ++k;
        }
        if (c.keep_succeed) {
            bool present = (c.rk_sk && del != DEL_PIECE) || (c.has_offset && c.rk_off) ||
                           (c.rk_micro && del != DEL_MICRO) ||
                           (c.rk_base != LC_AP_SLS_NONE && lc_ap_sls_has_base(r, c.rk_base) &&
                            !(del == DEL_BASE && c.rk_base == c.sk_base));
            for (uint32_t j = 0; j < r.m && !present; ++j) {
                const LcApEntry& x = r.e[j];
                if (x.key_off < LC_AP_K_LEVEL && x.key_len == c.rklen) {
                    uint32_t b = 0;
                    while (b < x.key_len && src[x.key_off + b] == c.rkey[b])
                        ++b;
                    present = b == x.key_len;
                }
            }
            if (!present)
                piece(c.rkey, c.rklen);
        }
    } else if (kept) {
        piece(c.skey, c.sklen); // an empty value: the piece is kept untouched
        if (c.has_offset)
            digits();
    } else {
        if (c.has_offset)
            digits();
        if (!(c.has_offset && c.rk_off))
            piece(c.rkey, c.rklen);
        if (c.copy_raw && !(c.has_offset && c.raw_off) && !c.rk_raw)
            piece(c.names, 11u);
    }
    const bool has_ns = ok ? c.enable_ns != 0 : c.has_ns != 0;
    if (has_ns) {
        const uint32_t ns = ok ? r.nsec : c.ns;
        const uint8_t h[5] = {0x25, (uint8_t)ns, (uint8_t)(ns >> 8), (uint8_t)(ns >> 16), (uint8_t)(ns >> 24)};
        s.put(h, 5);
    }
    return k;
}

// The piece's counter verdicts as bits of ProcessorParseApsaraNative's counters in lc_apsara_parse's order
// (LC_TS_C_*): discarded also counts a failed piece ShouldEraseEvent erases.
LC_HD uint32_t lc_split_apsara_verdict(const LcSplitApsaraSlsCfg& c, uint32_t status) {
    const uint32_t st = status & 7u;
    if (st == LC_AP_ST_OK)
        return 1u << LC_TS_C_OUT_SUCCESSFUL;
    if (st == LC_AP_ST_NOT_FOUND)
        return 1u << LC_TS_C_KEY_NOT_FOUND;
    if (st == LC_AP_ST_EMPTY)
        return 1u << LC_TS_C_OUT_FAILED;
    if (st == LC_AP_ST_DISCARDED)
        return (1u << LC_TS_C_HISTORY_FAILURE) | (1u << LC_TS_C_DISCARDED);
    return (1u << LC_TS_C_OUT_FAILED) | (c.keep_fail ? 0u : 1u << LC_TS_C_DISCARDED);
}

// Host side: the configuration of the chain, with the key pointers as given and `names` at a host LC_AP_SLS_NAMES (the
// device caller points them at its copies).  offset_key == nullptr: no log.file.offset metadata; time_ns 0xFFFFFFFF:
// the source event writes no Time_ns.  Returns nullptr, or why the chain is refused: an offset key equal to SourceKey
// (the split would replace the piece by its digits, and the Apsara stage would parse those), and a source Time_ns
// without enable_ns (the pieces that keep the source time would write Time_ns and the parsed ones would not, a mix no
// configuration of the reference produces).
inline const char* lc_split_apsara_sls_setup(const char* source_key, uint32_t source_len, const char* renamed_key,
                                             uint32_t renamed_len, const char* offset_key, uint32_t offset_len,
                                             int keep_fail, int keep_succeed, int copy_raw, uint64_t src_pos,
                                             uint32_t time, uint32_t time_ns, int enable_ns,
                                             LcSplitApsaraSlsCfg* c) {
    auto eq = [](const char* a, uint32_t al, const char* b, uint32_t bl) {
        return al == bl && (al == 0 || !memcmp(a, b, al));
    };
    static const char* const kNames = LC_AP_SLS_NAMES;
    auto base_of = [&](const char* k, uint32_t kl) {
        for (uint32_t t = 0; t < 4; ++t)
            if (eq(k, kl, kNames + lc_ap_sls_base_at(t), lc_ap_sls_base_len(t)))
                return t;
        return (uint32_t)LC_AP_SLS_NONE;
    };
    if (!c)
        return "bad arguments";
    if (offset_key && eq(offset_key, offset_len, source_key, source_len))
        return "the offset key equals SourceKey";
    if (time_ns != 0xFFFFFFFFu && !enable_ns)
        return "a source time_ns needs enable_ns";
    memset(c, 0, sizeof *c);
    c->skey = reinterpret_cast<const uint8_t*>(source_key);
    c->rkey = reinterpret_cast<const uint8_t*>(renamed_key);
    c->okey = reinterpret_cast<const uint8_t*>(offset_key);
    c->names = reinterpret_cast<const uint8_t*>(kNames);
    c->sklen = source_len;
    c->rklen = renamed_len;
    c->oklen = offset_key ? offset_len : 0u;
    c->has_offset = offset_key != nullptr;
    c->keep_fail = keep_fail != 0;
    c->keep_succeed = keep_succeed != 0;
    c->copy_raw = copy_raw != 0;
    c->enable_ns = enable_ns != 0;
    c->sk_base = base_of(source_key, source_len);
    c->sk_micro = eq(source_key, source_len, kNames + 11, 9);
    c->rk_base = base_of(renamed_key, renamed_len);
    c->rk_sk = eq(renamed_key, renamed_len, source_key, source_len);
    c->rk_off = offset_key && eq(renamed_key, renamed_len, offset_key, offset_len);
    c->rk_micro = eq(renamed_key, renamed_len, kNames + 11, 9);
    c->rk_raw = eq(renamed_key, renamed_len, kNames, 11);
    c->raw_off = offset_key && eq(kNames, 11, offset_key, offset_len);
    c->src_pos = src_pos;
    c->time = time;
    c->has_ns = time_ns != 0xFFFFFFFFu;
    c->ns = c->has_ns ? time_ns : 0u;
    return nullptr;
}
