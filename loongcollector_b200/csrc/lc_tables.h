// lc_tables.h -- POD layout of a compiled regex ("program blob") shared by the host compiler
// (regex_compiler.cpp) and the sm_90a kernels (kernels_regex.cu).
//
// A compiled pattern is ONE contiguous blob: a fixed header followed by 16-byte aligned arrays
// addressed by byte offsets from the blob start, so the same bytes can live in host memory,
// in HBM and be staged into shared memory by a kernel without any pointer fix-up.
//
// Three automata are derived from one prioritised (Perl leftmost-first) Thompson NFA:
//   * PREFIX   boolean DFA: "does some prefix of the line match" == boost::regex_search(...,
//              match_continuous) (reference: core/common/StringTools.cpp:263-288).  Used by the
//              multiline splitter.
//   * FWD1     forward-only tagged automaton over NFA "walker" states.  Exact for patterns whose
//              highest-priority viable transition never depends on look-ahead (checked at compile
//              time against the reverse DFA).  One table look-up per input byte.
//   * REV+FWD2 general case: a reverse DFA pass labels every position with the set of NFA
//              transitions that can still reach a full match; the forward walk then takes, at
//              every byte, the highest-priority viable transition -- which is exactly the path a
//              backtracking matcher (boost perl_matcher, regex_match) returns first.
#pragma once
#include <stdint.h>

#define LC_REGEX_MAGIC 0x4C435258u /* 'LCRX' */
#define LC_MAX_GROUPS 32u
#define LC_NONE_ENTRY 0xFFFFFFFFu
#define LC_PREFIX_DEAD 0u
#define LC_PREFIX_ACCEPT 0xFFFFu
#define LC_REV_DEAD 0u

enum LcRegexMode {
    LC_MODE_FWD1 = 0,   // forward-only tagged automaton
    LC_MODE_TWOPASS = 1 // reverse DFA + guided forward walk
};

// Entry of the forward tables: bits 0..15 next walker state, bits 16..31 action id
// (index into the save-mask list; action 0 == no capture boundary crossed).
// LC_NONE_ENTRY == no viable transition (the line does not match).
#define LC_ENTRY_NEXT(e) ((e) & 0xFFFFu)
#define LC_ENTRY_ACT(e) ((e) >> 16)

struct LcRegexHeader {
    uint32_t magic;
    uint32_t total_bytes;
    uint32_t ngroups;  // capture groups (what.size() - 1)
    uint32_t nclasses; // byte equivalence classes
    uint32_t mode;     // LcRegexMode
    uint32_t npc;      // number of "previous byte" context kinds (1 when no context assertions)
    uint32_t nw;       // walker states (0 == START)
    uint32_t nact;     // actions (save masks)
    // PREFIX dfa
    uint32_t pre_nstates;
    uint32_t pre_start;
    // reverse dfa (TWOPASS)
    uint32_t rev_nstates;
    uint32_t rev_start; // state at position n (end of input)
    // byte offsets of the arrays inside the blob
    uint32_t off_byte_class; // u8  [256]
    uint32_t off_class_pc;   // u8  [nclasses]   class -> prev-context kind
    uint32_t off_actions;    // u64 [nact]       bit s set => capture slot s := current position
    uint32_t off_pre_next;   // u16 [pre_nstates][nclasses]  (0 dead, 0xFFFF accept before this byte)
    uint32_t off_pre_acc;    // u8  [pre_nstates]            accept at end of input
    uint32_t off_fwd;        // u32 FWD1: [nw*npc][nclasses]   TWOPASS: [nw*npc][rev_nstates]
    uint32_t off_fwd_eof;    // u32 FWD1: [nw*npc]  entry taken at end of input (next ignored)
    uint32_t off_rev_next;   // u16 [rev_nstates][nclasses]
    uint32_t fwd_cols;       // row length of the fwd table
    uint32_t flags;          // unused
    uint32_t off_rev_byte;   // TWOPASS: LabT [rev_nstates][256] reverse transition indexed by raw byte
    uint32_t rev_label_bytes; // 1 when rev_nstates <= 256 (LabT = u8) else 2 (u16)
    uint32_t off_fwd_byte;   // FWD1 (npc == 1 only): u32 [nw][256] forward entry indexed by raw byte, else 0
    uint32_t reserved[7];
};

// ---- "fast blob": kernel-ready re-layout of a TWOPASS automaton without context kinds, with <= 63 reverse
// states, <= 255 walkers and <= 31 capture groups (the common case for log patterns).  Built once per pattern
// on the host; the kernel copies it verbatim into shared memory.
//   rev   u8  [rev_nstates][260]   reverse transition by raw byte, value = next_state * 4 (labels are stored
//                                  pre-multiplied so that they index 32-bit forward entries directly).  The 260-byte
//                                  row pitch skews rows across shared-memory banks: bank = (state + byte/4) mod 32.
//   fwd   u32 [nw][64]             256-byte rows.  entry = slot_byte | next_row_index << 8 | multi << 31 where
//                                  slot_byte: 0 = no capture boundary, 4*slot+4 = set that one slot;
//                                  multi = several slots are set (action id in cx; reserved[0] = has_multi).
//                                  address of the next look-up = (entry & 0x00FFFF00) | label  -- one PRMT.
//   cx    u8  [nw][64]             action id of multi-slot entries (0 elsewhere)
//   masks u64 [nact]               save masks of the actions
#define LC_FAST_MAGIC 0x4C434658u /* 'LCFX' */
#define LC_FAST_REV_PITCH 260u
#define LC_FAST_MAX_REV 63u
#define LC_FAST_MAX_WALKERS 255u
#define LC_FAST_MAX_GROUPS 31u
struct LcFastHeader {
    uint32_t magic;
    uint32_t total_bytes;
    uint32_t ngroups;
    uint32_t rev_start4; // start state * 4
    uint32_t nrev;
    uint32_t nw;
    uint32_t nact;
    uint32_t off_rev;
    uint32_t off_fwd;
    uint32_t off_cx;
    uint32_t off_masks;
    uint32_t reserved[5];
};

// ---- "fast2 blob": stride-2 layout of the same two-pass automaton.  Two input bytes are consumed per dependent
// look-up and ONE label byte is stored per byte pair, which halves both the dependency chain and the
// shared-memory footprint per in-flight line.  Pairs are aligned on even addresses.
//   cls    u8  [256]                  byte -> class.  64 words: ASCII text never bank-conflicts (bytes b, b+128 share
//                                     a bank); the row offset (c1 * ncls + c0) * 4 is computed arithmetically.
//   t2     u32 [nrev][ncls*ncls]      reverse pair step from state D over bytes (b1 = later, b0 = earlier):
//                                     entry = next_state * row_bytes (bits 0..15, the byte offset of its row,
//                                     row_bytes = ncls*ncls*4) | (pair_id << pair_shift) << 16.
//   pid    u8  [nrev][nrev]           (pair id << pair_shift) of (label(q), label(q+1)); 0 = impossible
//   pair_l u8  [npairs][2]            inverse of pid (indexed by the plain pair id)
//   rev1   u8  [nrev][ncls]           single reverse step by class (peeled first / last byte)
//   f2     u32 [nw][f2_row]           forward pair step: byte0 = next walker after both steps, byte1 = slot set by
//                                     the 1st step, byte2 = slot set by the 2nd step (2*slot + 2, 0 = none; bit 7 of
//                                     byte1 = some step sets several slots -> slow path via pair_l + fwd1 + masks),
//                                     byte3 = 0.
//                                     compact layout (npairs <= 63: pair_shift = 2, f2_row = 64): labels hold
//                                     pair_id * 4 and PRMT(entry, labels) = walker << 8 | pair_id * 4 is directly the
//                                     BYTE offset of the next entry (256-byte rows);
//                                     wide layout (pair_shift = 0, f2_row = 256): PRMT gives the entry INDEX.
//   fwd1   u32 [nw][nrev]             single forward step: next walker | action id << 16 (LC_NONE_ENTRY = no path)
//   masks  u64 [nact]
#define LC_FAST2_MAGIC 0x4C434632u /* 'LCF2' */
#define LC_FAST2_ACT_MULTI 0x8000u /* bit 7 of byte1 of an f2 entry */
struct LcFast2Header {
    uint32_t magic;
    uint32_t total_bytes;
    uint32_t ngroups;
    uint32_t rev_start;
    uint32_t nrev;
    uint32_t ncls;
    uint32_t nw;
    uint32_t npairs;
    uint32_t nact;
    uint32_t row_bytes; // ncls * ncls * 4
    uint32_t off_cls;
    uint32_t pair_shift; // 2 = compact f2 layout, 0 = wide
    uint32_t off_t2;
    uint32_t off_pid;
    uint32_t off_pair_l;
    uint32_t off_rev1;
    uint32_t off_f2;
    uint32_t off_fwd1;
    uint32_t off_masks;
    uint32_t has_multi;
    uint32_t f2_row; // entries per f2 row (64 or 256)
    uint32_t reserved[3];
};

// ---- "tdfa blob": single forward pass, stride 2.  The priority-ordered NFA thread list is determinised together
// with the capture bookkeeping (a tagged DFA with leftmost-first / Perl disambiguation): a state is the ordered list
// of live threads, each with a map tag -> register; a transition may set registers to the current position.  The
// scheme never needs register copies while scanning: an inherited value keeps its register, a new value takes the
// tag's home register (= the tag index) when no live thread still refers to it, else a spare.  Only the end-of-input
// action moves the winner's values to the home registers.  No reverse pass, no labels: half the look-ups of the
// two-pass layouts and a per-line footprint of just the register file.
//   cls   u8  [256]                byte -> class
//   t2    u32 [nstates+1][row_bytes/4] pair step over bytes (b0 = earlier, b1 = later), indexed (c0 * ncls + c1):
//                                  bits 0..15 = next_state * row_bytes (row_bytes = (ncls*ncls | 1) * 4: an odd word
//                                  pitch spreads the states over the shared-memory banks; state 0 = dead),
//                                  bits 16..22 = register set by the 1st step at position p   (2*reg + 2, 0 = none),
//                                  bit  23     = slow path (some step sets more than one register): such entries
//                                                lead to the absorbing SINK row (index nstates) instead of the real
//                                                next state, which only the single-step tables can produce,
//                                  bits 24..30 = register set by the 2nd step at position p+1 (2*reg + 2, 0 = none).
//   t1    u32 [nstates][ncls]      single step: next state | op-list index << 16 (peeled bytes and the slow path)
//   eof   u32 [nstates]            end of input: op-list index of the winning thread, LC_NONE_ENTRY = no match
//   ops   u16 []                   op lists: [count, op...], op = dst << 8 | src ; src 0xFF = current position,
//                                  0xFE = unset, else a register (copy).  List 0 is empty.
//   skip  u32 [nstates+1]          run skipping: a state that every byte except at most two "exit" bytes maps back to
//                                  itself without touching a register (the inside of [^"]*, .*, the dead state) can
//                                  jump over a whole 16-byte chunk that holds none of its exit bytes.
//                                  0 = not skippable; else LC_TDFA_SKIP | nexits << 16 | exit2 << 8 | exit1, with
//                                  exit2 = exit1 when nexits = 1.
#define LC_TDFA_MAGIC 0x4C435444u /* 'LCTD' */
#define LC_TDFA_SLOW 0x00800000u
#define LC_TDFA_SRC_POS 0xFFu
#define LC_TDFA_SRC_UNSET 0xFEu
#define LC_TDFA_MAX_REGS 62u
#define LC_TDFA_SKIP 0x80000000u
#define LC_TDFA_REBASE_ROOM 2048u /* window base + class table + blob header precede the (row-aligned) pair table */
struct LcTdfaHeader {
    uint32_t magic;
    uint32_t total_bytes;
    uint32_t ngroups;
    uint32_t nstates;
    uint32_t ncls;
    uint32_t nregs; // 2 * ngroups home registers + spares
    uint32_t start;
    uint32_t row_bytes;
    uint32_t off_cls;
    uint32_t off_t2;
    uint32_t off_t1;
    uint32_t off_eof;
    uint32_t off_ops;
    uint32_t has_slow;
    uint32_t max_threads; // diagnostics
    uint32_t sink;        // index of the slow-path sink row (= nstates; t2 has nstates + 1 rows)
    uint32_t off_skip;
    uint32_t reserved2[3];
};

#ifdef __cplusplus
static_assert(sizeof(LcFast2Header) % 16 == 0, "fast2 header must keep 16B alignment");
static_assert(sizeof(LcTdfaHeader) % 16 == 0, "tdfa header must keep 16B alignment");
static_assert(sizeof(LcFastHeader) % 16 == 0, "fast header must keep 16B alignment");
static_assert(sizeof(LcRegexHeader) % 16 == 0, "header must keep 16B alignment of what follows");
#endif
