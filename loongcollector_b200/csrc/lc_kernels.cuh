// lc_kernels.cuh -- launch interface between the C-ABI layer (lc_capi.cu) and the sm_90a kernels
// (lc_kernels.cu).  Device pointers + stream in, nothing else.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct LcDelimSlsCfg; // lc_exec.cuh
struct LcRegexSlsCfg;
struct LcDelimRegexSlsCfg;
struct LcSpanSlsCfg;
struct LcSplitRegexSlsCfg;
struct LcSplitDelimSlsCfg;
struct LcSplitDelimRegexSlsCfg;
struct LcSplitDelimTsCfg;
struct LcFilterSlsCfg;
struct LcSplitRegexTsCfg;
struct LcLz4Seq;
struct LcTsConf;
struct LcTsNow;
struct LcTsSpans;
struct LcTsFull;
struct LcApEv;
struct LcApEntry;
struct LcJsonEntry;
struct LcSplitJsonSlsCfg;
struct LcSplitJsonTsCfg;
struct LcJsonSlsEv;
struct LcSplitApsaraSlsCfg;
struct LcLz4Chunk;

namespace lck {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 4;
constexpr uint32_t kScanTile = kScanThreads * kScanItems;

inline uint32_t scan_tiles(uint64_t n) { return (uint32_t)((n + kScanTile - 1) / kScanTile); }

// a1: newline split in three passes (masks, tile scan, emission).  n_out: u32 device counter.
// d_total: u64 device counter (zeroed) that receives the un-truncated number of split chars (the line numbers keep
// 30 bits of count: the caller reports LC_ERR_TOO_LARGE beyond that).
// d_scratch: split_scratch_bytes(len, probe) bytes (not initialised): masks, per-tile counts and prefixes.
// Returns the number of kernels launched.
uint64_t split_scratch_bytes(uint64_t len, bool probe);
int launch_split(const uint8_t* d_buf, uint32_t len, uint8_t split_char, uint32_t* d_off, uint32_t* d_len,
                 uint32_t cap, uint32_t* d_n_out, unsigned long long* d_total, uint64_t* d_scratch, cudaStream_t st);

// exclusive sum of u32 -> u64 (out has n entries; *d_total receives the grand total)
void launch_exclusive_sum(const uint32_t* d_in, uint64_t n, uint64_t* d_out, uint64_t* d_total, uint64_t* d_desc,
                          uint32_t* d_ticket, cudaStream_t st);

// a3: regex_match + capture groups, one thread per event (baseline kernel, tables read from global memory)
// d_lab_off: per-event byte offset into d_lab (two-pass label scratch, u16 labels); unused for forward-only.
void launch_regex_parse_basic(const void* d_blob, uint32_t mode, uint32_t ngroups, const uint8_t* d_base,
                              const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                              uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len, const uint64_t* d_lab_off,
                              uint16_t* d_lab, cudaStream_t st);
// per-event scratch need of the two-pass matcher: len + 1 labels, rounded up to 8 labels (16 B)
void launch_label_sizes(const uint32_t* d_ev_len, uint64_t n, uint32_t* d_sizes, cudaStream_t st);

// d_out[0] = max(ev_len), d_out[1] = sum(ev_len); d_out must be zeroed by the caller
void launch_len_stats(const uint32_t* d_ev_len, uint64_t n, unsigned long long* d_out, cudaStream_t st);

// order[] = event indices sorted by descending length bucket (d_hist64: 64-word scratch + 1 flag word); 3 launches.
// d_hist64[64] = 1 when the lengths span more than two adjacent buckets (a ragged batch: use the order), else 0.
void launch_length_order(const uint32_t* d_ev_len, uint64_t n, uint32_t* d_hist64, uint32_t* d_order,
                         cudaStream_t st);

// a3 fast path: persistent kernel, automaton staged in shared memory.  Labels of events needing
// <= lab_words 32-bit words stay in shared memory, longer events bump-allocate from d_scratch.
// d_bump, d_overflow and d_next_batch must be zeroed by the caller.  Dynamic shared memory =
// blob_bytes + (threads / 32) * lab_words * 128.  Returns a cudaError_t value (0 on success).
int launch_regex_parse_fast(const void* d_blob, uint32_t blob_bytes, uint32_t rev_label_bytes, uint32_t ngroups,
                            const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                            uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                            uint32_t lab_words, uint32_t threads, uint32_t grid, uint32_t* d_scratch,
                            uint64_t scratch_words, unsigned long long* d_bump, uint32_t* d_overflow,
                            unsigned long long* d_next_batch, const uint32_t* d_order, cudaStream_t st);

// a3 fastest path: two-pass automaton in the host-built fast layout (LcFastHeader).  Shared memory per block =
// blob + labels (threads/32 * lab_words * 128 B) + capture slots (threads * slot_pitch * 4 B).
inline uint32_t fast_slot_pitch(uint32_t ngroups) { return (2 * ngroups + 1) | 1u; } // odd word pitch
inline size_t fast_smem_bytes(uint32_t blob_bytes, uint32_t ngroups, uint32_t lab_words, uint32_t threads) {
    return (size_t)blob_bytes + (size_t)(threads / 32) * lab_words * 128 + (size_t)threads * fast_slot_pitch(ngroups) * 4;
}
int launch_regex_twopass_fast(const void* d_fast_blob, uint32_t blob_bytes, bool multi, uint32_t ngroups,
                              const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                              uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                              uint32_t lab_words, uint32_t threads, uint32_t grid, uint32_t* d_scratch,
                              uint64_t scratch_words, unsigned long long* d_bump, uint32_t* d_overflow,
                              unsigned long long* d_next_batch, const uint32_t* d_order, cudaStream_t st);

// a3 stride-2 path (LcFast2Header): labels take (len + 15) / 8 + 1 words, capture slots are u16.
// Only valid when every event is shorter than 65535 bytes.
inline uint32_t fast2_slot_pitch(uint32_t ngroups) { return ((ngroups + 1) | 1u) * 2; } // halfwords; odd WORD pitch
inline size_t fast2_smem_bytes(uint32_t blob_bytes, uint32_t ngroups, uint32_t lab_words, uint32_t threads) {
    return (size_t)blob_bytes + (size_t)(threads / 32) * lab_words * 128 + (size_t)threads * fast2_slot_pitch(ngroups) * 2;
}
int launch_regex_fast2(const void* d_blob, uint32_t blob_bytes, bool multi, bool compact, uint32_t ngroups,
                       const uint8_t* d_base,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                       uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len, uint32_t lab_words,
                       uint32_t threads, uint32_t grid, uint32_t* d_scratch, uint64_t scratch_words,
                       unsigned long long* d_bump, uint32_t* d_overflow, unsigned long long* d_next_batch,
                       const uint32_t* d_order, cudaStream_t st);

// a3 single-pass tagged-DFA path (LcTdfaHeader): no labels; per thread only nregs u16 registers in shared memory.
// Events of 65535 bytes or more raise *d_overflow and are left to launch_regex_tdfa_long (32-bit slots).
// Lines are fetched cooperatively (cp.async, 4 full 128-byte lines per instruction) into a per-warp 4 KB tile;
// carve-out = 512 B (aligned class table) + blob + register files + 128 B (alignment of the tiles) + 256 B line
// info and 4 KB tile per warp
inline uint32_t tdfa_reg_pitch(uint32_t nregs) { return (((nregs + 1) / 2) | 1u) * 2; } // halfwords; odd WORD pitch
inline size_t tdfa_staged_smem_bytes(uint32_t blob_bytes, uint32_t nregs, uint32_t threads) {
    return 512 + (size_t)blob_bytes + 16 + (size_t)threads * tdfa_reg_pitch(nregs) * 2 + 128 +
           (size_t)(threads / 32) * (256 + 4096);
}
int launch_regex_tdfa_staged(const void* d_blob, uint32_t blob_bytes, bool slow, uint32_t nregs, const uint8_t* d_base,
                             const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint32_t ev_stride /* elements */,
                             uint64_t n, uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                             uint32_t threads, uint32_t grid, unsigned long long* d_next_batch, uint32_t* d_overflow,
                             const uint32_t* d_order /* or nullptr */, const uint32_t* d_order_flag /* or nullptr */,
                             cudaStream_t st);

// several patterns in one grid: all tagged-DFA blobs co-resident in shared memory, tried per line in array order
constexpr uint32_t LC_MULTI_MAX = 8;
struct TdfaMultiArgs {
    const void* blob[LC_MULTI_MAX]; // device tdfa blobs
    uint32_t blob_bytes[LC_MULTI_MAX];
    uint32_t nkeys[LC_MULTI_MAX];
    uint32_t npat;
};
inline size_t tdfa_multi_table_bytes(const TdfaMultiArgs& a) {
    size_t t = 256;
    for (uint32_t p = 0; p < a.npat; ++p)
        t += 256 + ((a.blob_bytes[p] + 255u) & ~255u);
    return t;
}
inline size_t tdfa_multi_smem_bytes(const TdfaMultiArgs& a, uint32_t max_nregs, uint32_t threads) {
    return tdfa_multi_table_bytes(a) + 16 + (size_t)threads * tdfa_reg_pitch(max_nregs) * 2 + 128 +
           (size_t)(threads / 32) * (256 + 4096);
}
int launch_regex_tdfa_multi(const TdfaMultiArgs& a, uint32_t p_base, bool resume, bool slow, uint32_t max_nregs,
                            const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                            const uint8_t* d_sel, uint8_t* d_which, uint8_t* d_status, uint32_t* d_cap_off,
                            uint32_t* d_cap_len, uint32_t gpitch, uint32_t threads, uint32_t grid,
                            unsigned long long* d_next_batch, uint32_t* d_overflow, const uint32_t* d_order,
                            const uint32_t* d_order_flag, cudaStream_t st);
// events >= 65535 bytes (skipped by the staged kernels, which raise *d_overflow): 32-bit registers, no-op otherwise
void launch_regex_tdfa_long(const TdfaMultiArgs& a, const uint8_t* d_base, const uint32_t* d_ev_off,
                            const uint32_t* d_ev_len, uint32_t ev_stride, uint64_t n, const uint8_t* d_sel,
                            uint8_t* d_which, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len,
                            uint32_t gpitch, const uint32_t* d_overflow, bool bool_only, cudaStream_t st);

// parse status -> boolean (1 = the whole value matched)
void launch_status_to_bool(uint8_t* d_status, uint64_t n, cudaStream_t st);

// anchored prefix probe, one bool per event
void launch_prefix_match(const void* d_blob, const uint8_t* d_base, const uint32_t* d_ev_off,
                         const uint32_t* d_ev_len, uint64_t n, uint8_t* d_out, cudaStream_t st);

// a2: multiline.  Lines (d_off, d_len) and per-line flags come from launch_split_probe over the same buffer.
struct MlConfig {
    const void* blob_start; // device blobs or nullptr
    const void* blob_cont;
    const void* blob_end;
    int discard;
    // split + probe pass only (host-built from the prefix DFAs): first[p] bit b = a line starting with byte b can
    // match pattern p; empty_flags = flag bits of an empty line
    uint32_t first[3][8];
    uint32_t empty_flags;
};
// split + per-line probes in one formulation (the three split passes): d_flags[i] bit0/1/2 = start/continue/end
// pattern matches a prefix of line i.  Other arguments and the result as for launch_split.
int launch_split_probe(const MlConfig& cfg, const uint8_t* d_buf, uint32_t len, uint32_t* d_off, uint32_t* d_len,
                       uint8_t* d_flags, uint32_t cap, uint32_t* d_n_out, unsigned long long* d_total,
                       uint64_t* d_scratch, cudaStream_t st);
// state scan + counts + slots + emission over the split's line table; reads the line count from d_n_lines (no host
// round trip in between).  Five launches; d_scratch: ml_pass_scratch_bytes(line_cap), not initialised.
// d_counters[0..1] += matched_events, unmatch_lines; *d_total = number of output events.
uint32_t ml_pass_tiles(uint64_t line_cap);
uint64_t ml_pass_scratch_bytes(uint64_t line_cap);
int launch_ml_passes(const MlConfig& cfg, const uint8_t* d_flags, const uint32_t* d_off, const uint32_t* d_len,
                     const uint32_t* d_n_lines, uint32_t line_cap, uint32_t total_len, uint32_t* d_out_off,
                     uint32_t* d_out_len, uint8_t* d_out_flags, uint64_t cap, uint64_t* d_scratch,
                     unsigned long long* d_counters, uint64_t* d_total, cudaStream_t st);

// f3: last complete record of a chunk from the split pass's line table + flags; d_out[0] = keep bytes, [1] = rollback
void launch_last_record(const uint8_t* d_flags, const uint32_t* d_off, const uint32_t* d_len, const uint32_t* d_n_lines,
                        uint32_t line_cap, uint32_t size, bool has_start, bool has_end, unsigned long long* d_out,
                        cudaStream_t st);

// a4: delimiter
struct DelimConfig {
    uint8_t sep[4];
    uint32_t sep_len;
    uint8_t quote;
    uint32_t nkeys;
    int extend;
    int allow_short;
    uint32_t max_fields;
    // optional column tap: the (off, len) of column tap_col of every line also leave as two DENSE tables (the event
    // table of a processor chained on that column); tap_col >= max_fields or null pointers = no tap
    uint32_t tap_col;
    uint32_t* tap_off;
    uint32_t* tap_len;
};
// d_next_batch: zeroed u64 batch counter of the persistent tiled kernel (quote-FSM mode); nullptr = thread-per-line
void launch_delim(const DelimConfig& cfg, const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len,
                  uint64_t n, uint8_t* d_status, uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len,
                  uint32_t* d_f_dq, unsigned long long* d_next_batch, cudaStream_t st);

// next row (rank 4): SLS wire format of LOG events.  ev_ns may be null; 0xFFFFFFFF = no nanosecond part.
// rec_size[i] = bytes of event i's Log record (0 = empty event, skipped); body_size[i] = bytes inside its Logs field.
void launch_sls_sizes(const uint64_t* d_ent_begin, const uint32_t* d_klen, const uint32_t* d_vlen,
                      const uint32_t* d_ev_ns, uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                      cudaStream_t st);
void launch_sls_emit(const uint8_t* d_base, const uint32_t* d_ev_time, const uint32_t* d_ev_ns,
                     const uint64_t* d_ent_begin, const uint32_t* d_koff, const uint32_t* d_klen,
                     const uint32_t* d_voff, const uint32_t* d_vlen, uint64_t n, const uint64_t* d_rec_off,
                     const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st);

// f4, regex-fed: Log records from the regex stage's result tables (lc_regex_parse_dev) + the content plans of
// lc_exec.cuh (LcRegexSlsCfg, plans and key strings on the device).  Sizes as for launch_sls_sizes; d_counters (or
// nullptr): u64 [3] += successful, failed (LC_REGEX_NOMATCH), discarded events.
struct RegexSlsTables {
    const uint8_t* base;
    const uint32_t* ev_off;
    const uint32_t* ev_len;
    const uint8_t* status;  // nullptr in whole-line mode
    const uint32_t* cap_off; // [n][pitch], or nullptr when no plan reads a capture
    const uint32_t* cap_len;
};
void launch_regex_sls_sizes(const LcRegexSlsCfg& c, const RegexSlsTables& t, const uint32_t* d_ev_ns, uint64_t n,
                            uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                            cudaStream_t st);
void launch_regex_sls_emit(const LcRegexSlsCfg& c, const RegexSlsTables& t, const uint32_t* d_ev_time,
                           const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off, const uint32_t* d_body_size,
                           uint8_t* d_out, cudaStream_t st);

// f4, split -> regex chain: Log records of the pieces t.ev_off / t.ev_len of the source value t.base, parsed into the
// regex tables of t (lc_exec.cuh: LcSplitRegexSlsCfg, plans and key strings on the device).  Sizes as for
// launch_sls_sizes; d_counters: u64 [4] += successful, failed (LC_REGEX_NOMATCH), discarded pieces, and pieces whose
// record would reach 4 GiB.  d_keep (or nullptr): a filter's verdict per piece (launch_filter_eval); a removed piece
// has no record.
void launch_split_regex_sls_sizes(const LcSplitRegexSlsCfg& c, const RegexSlsTables& t, uint64_t n,
                                  const uint8_t* d_keep, uint32_t* d_rec_size, uint32_t* d_body_size,
                                  unsigned long long* d_counters, cudaStream_t st);
// f4, split -> regex -> filter chain (lc_exec.cuh: LcFilterSlsCfg).  launch_filter_tap: leaf's values as a dense
// (d_off, d_len) table over t.base and, with d_doff, a (d_doff, d_dlen) table over the digit scratch d_dig (20 bytes
// per piece).  launch_filter_eval: d_keep[i] = the filter's verdict from the match bytes d_match (lc_regex_match_dev
// over those tables, [l * n + i] and, with digits, [(nleaves + l) * n + i]); d_counters: u64 [1] += removed pieces.
void launch_filter_tap(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, uint32_t leaf, const RegexSlsTables& t,
                       uint64_t n, uint32_t* d_off, uint32_t* d_len, uint32_t* d_doff, uint32_t* d_dlen,
                       uint8_t* d_dig, cudaStream_t st);
void launch_filter_eval(const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f, const uint8_t* d_status, uint64_t n,
                        const uint8_t* d_match, uint8_t* d_keep, unsigned long long* d_counters, cudaStream_t st);
void launch_split_regex_sls_emit(const LcSplitRegexSlsCfg& c, const RegexSlsTables& t, uint64_t n,
                                 const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                 cudaStream_t st);
// f4, split -> regex -> timestamp chain (lc_exec.cuh: LcSplitRegexTsCfg).  launch_split_regex_ts_tap: the dense value
// table (d_off, d_len) over t.base that the timestamp passes take (LC_TS_NO_KEY: erased by the regex stage, or no
// tkey).  The size and emit passes are launch_split_regex_sls_*'s with each record's time from the timestamp tables ts
// (a discarded piece has no record); d_counters: u64 [9] += the chain's 8 counters (LC_SRTS_COUNTERS), then pieces
// whose record would reach 4 GiB.
struct TsRowTables {
    const uint8_t* status; // LC_TS_* per piece
    const int64_t* sec;
    const uint32_t* nsec;
};
void launch_split_regex_ts_tap(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                               uint64_t n, uint32_t* d_off, uint32_t* d_len, cudaStream_t st);
void launch_split_regex_ts_sls_sizes(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                                     const TsRowTables& ts, uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                                     unsigned long long* d_counters, cudaStream_t st);
void launch_split_regex_ts_sls_emit(const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const RegexSlsTables& t,
                                    const TsRowTables& ts, uint64_t n, const uint64_t* d_rec_off,
                                    const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st);

// f4, delimiter-fed: Log records from the delimiter stage's result tables (launch_delim) + the configuration of
// lc_exec.cuh (LcDelimSlsCfg, key strings on the device).  Sizes as for launch_sls_sizes; d_counters (or nullptr):
// u64 [4] += successful, failed, discarded, blank events.
struct DelimSlsTables {
    const uint8_t* base;
    const uint32_t* ev_off;
    const uint32_t* ev_len;
    const uint8_t* status;
    const uint32_t* nfields;
    const uint32_t* f_off; // [n][max_fields]
    const uint32_t* f_len;
    const uint32_t* f_dq;
};
void launch_delim_sls_sizes(const LcDelimSlsCfg& c, const DelimSlsTables& t, const uint32_t* d_ev_ns, uint64_t n,
                            uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                            cudaStream_t st);
void launch_delim_sls_emit(const LcDelimSlsCfg& c, const DelimSlsTables& t, const uint32_t* d_ev_time,
                           const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off, const uint32_t* d_body_size,
                           uint8_t* d_out, cudaStream_t st);

// f4, delimiter -> regex chain (lc_exec.cuh: LcDelimRegexSlsCfg).  launch_delim_regex_tap_sizes: d_copy[i] = bytes of
// row i's side copy (0 = none).  launch_delim_regex_tap: the value table (d_val_off, d_val_len) of every row; a row
// with a copy gets it at d_base[side_at + d_slot[i], + d_copy[i]) (d_slot = exclusive sum of d_copy).  The sizes and
// emit passes as for launch_sls_sizes over the delimiter tables, the value table and the regex tables over it
// (status / captures nullptr in whole-line mode); d_counters (or nullptr): u64 [8] += lc_delim_regex_verdict.
struct DelimRegexSlsTables {
    DelimSlsTables d;
    const uint32_t* val_off;
    const uint32_t* val_len;
    const uint8_t* status;
    const uint32_t* cap_off; // [n][pitch]
    const uint32_t* cap_len;
};
void launch_delim_regex_tap_sizes(const LcDelimRegexSlsCfg& c, const DelimSlsTables& t, uint64_t n, uint32_t* d_copy,
                                  cudaStream_t st);
void launch_delim_regex_tap(const LcDelimRegexSlsCfg& c, const DelimSlsTables& t, uint64_t n, const uint64_t* d_slot,
                            uint64_t side_at, uint8_t* d_base, uint32_t* d_val_off, uint32_t* d_val_len,
                            cudaStream_t st);
void launch_delim_regex_sls_sizes(const LcDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, const uint32_t* d_ev_ns,
                                  uint64_t n, uint32_t* d_rec_size, uint32_t* d_body_size,
                                  unsigned long long* d_counters, cudaStream_t st);
void launch_delim_regex_sls_emit(const LcDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, const uint32_t* d_ev_time,
                                 const uint32_t* d_ev_ns, uint64_t n, const uint64_t* d_rec_off,
                                 const uint32_t* d_body_size, uint8_t* d_out, cudaStream_t st);

// f4, split -> delimiter chain (lc_exec.cuh: LcSplitDelimSlsCfg): the sizes and emit passes as for launch_sls_sizes
// over the piece tables (t.ev_off / t.ev_len over t.base = the source value) and the delimiter tables over them;
// d_counters: u64 [5] += successful, failed, discarded, blank, pieces whose record would reach 4 GiB.
void launch_split_delim_sls_sizes(const LcSplitDelimSlsCfg& c, const DelimSlsTables& t, uint64_t n,
                                  uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                  cudaStream_t st);
void launch_split_delim_sls_emit(const LcSplitDelimSlsCfg& c, const DelimSlsTables& t, uint64_t n,
                                 const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                 cudaStream_t st);

// f4, split -> delimiter -> regex chain (lc_exec.cuh: LcSplitDelimRegexSlsCfg): the sizes and emit passes over the
// piece tables (t.d.ev_off / t.d.ev_len over t.d.base = the source value, with its side copies), the delimiter tables
// over them, the value table of the tap and the regex tables over the values; d_counters: u64 [9] +=
// lc_delim_regex_verdict's 8, pieces whose record would reach 4 GiB.
void launch_split_delim_regex_sls_sizes(const LcSplitDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, uint64_t n,
                                        uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                        cudaStream_t st);
void launch_split_delim_regex_sls_emit(const LcSplitDelimRegexSlsCfg& c, const DelimRegexSlsTables& t, uint64_t n,
                                       const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                       cudaStream_t st);

// f4, split -> delimiter -> timestamp chain (lc_exec.cuh: LcSplitDelimTsCfg).  launch_split_delim_ts_tap: the value
// table (d_off, d_len) over d_val that the timestamp passes take, with each value copied into d_val (at least as long
// as the source value) at its own offset, a column with doubled quotes collapsed; LC_TS_NO_KEY: erased by the
// delimiter stage, or no value.  The size and emit passes are launch_split_delim_sls_*'s with each record's time from
// the timestamp tables ts; d_counters: u64 [10] += the chain's 9 counters (LC_SDTS_COUNTERS), then pieces whose
// record would reach 4 GiB.
void launch_split_delim_ts_tap(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc, const DelimSlsTables& t,
                               uint64_t n, uint8_t* d_val, uint32_t* d_off, uint32_t* d_len, cudaStream_t st);
void launch_split_delim_ts_sls_sizes(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc,
                                     const DelimSlsTables& t, const TsRowTables& ts, uint64_t n,
                                     uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                     cudaStream_t st);
void launch_split_delim_ts_sls_emit(const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc,
                                    const DelimSlsTables& t, const TsRowTables& ts, uint64_t n,
                                    const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                    cudaStream_t st);

// f4, split-fed: Log records of the pieces of one source value (lc_exec.cuh: LcSpanSlsCfg, keys on the device).
// rec_size[k] = bytes of piece k's record (never 0); the emit pass writes the `total` bytes from the record offsets,
// one warp per kSpanTile bytes of output.
constexpr uint32_t kSpanTile = 1024;
void launch_span_sls_sizes(const LcSpanSlsCfg& c, uint64_t n, uint32_t* d_rec_size, cudaStream_t st);
void launch_span_sls_emit(const LcSpanSlsCfg& c, const uint64_t* d_rec_off, uint64_t n, uint64_t total, uint8_t* d_out,
                          cudaStream_t st);

// f4, LZ4: one LZ4 block per segment g = in[seg_off[g], + seg_len[g]) (lc_exec.cuh).  Chunk k of LC_LZ4_CHUNK bytes
// belongs to the segment g with first[g] <= k < first[g + 1] (first = exclusive sum of lc_lz4_nchunks per segment).
// launch_lz4_chunks: nch[g] = chunks of segment g; *d_too_large |= 1 for a segment over LC_LZ4_MAX_INPUT.
// launch_lz4_parse: the matches of chunks [k0, k1) (seq: LC_LZ4_SEQ_CAP entries per chunk).
// launch_lz4_sizes: block bytes per chunk and its literal anchor.  After an exclusive sum of d_csize (d_choff,
// *d_total), launch_lz4_emit writes the blocks and the per-segment table (blk_off, blk_len).
struct Lz4Segs {
    const uint8_t* in;
    const uint64_t* seg_off;
    const uint32_t* seg_len;
    const uint64_t* first;
    uint64_t nseg, nchunks;
};
void launch_lz4_chunks(const uint32_t* d_seg_len, uint64_t nseg, uint32_t* d_nch, uint32_t* d_too_large,
                       cudaStream_t st);
void launch_lz4_parse(const Lz4Segs& g, uint64_t k0, uint64_t k1, LcLz4Seq* d_seq, LcLz4Chunk* d_info,
                      cudaStream_t st);
void launch_lz4_sizes(const Lz4Segs& g, const LcLz4Chunk* d_info, uint32_t* d_csize, uint32_t* d_anchor,
                      cudaStream_t st);
void launch_lz4_emit(const Lz4Segs& g, const LcLz4Seq* d_seq, const LcLz4Chunk* d_info, const uint32_t* d_anchor,
                     const uint64_t* d_choff, const uint64_t* d_total, uint8_t* d_out, uint64_t* d_blk_off,
                     uint32_t* d_blk_len, cudaStream_t st);

// f4, zstd: one zstd frame per segment (lc_exec.cuh), over the matches launch_lz4_parse left in d_seq (every chunk of
// the segments in g).  Block k of LC_ZSTD_BLOCK bytes belongs to the segment g with bfirst[g] <= k < bfirst[g + 1]
// (bfirst = exclusive sum of lc_zstd_nblocks per segment, which launch_zstd_nblocks writes).
// launch_zstd_blocks: the compressed body of each block in its slot (d_slot + k * LC_ZSTD_BLOCK), d_body[k] = its size
// or 0 (Raw), d_esz[k] = the block's bytes in its frame; its literals go to the scratch behind each chunk's matches.
// After an exclusive sum of d_esz (d_boff, *d_total), launch_zstd_emit writes the frames and the per-segment table.
void launch_zstd_nblocks(const uint32_t* d_seg_len, uint64_t nseg, uint32_t* d_nblk, cudaStream_t st);
void launch_zstd_blocks(const Lz4Segs& g, const uint64_t* d_bfirst, uint64_t nblocks, LcLz4Seq* d_seq,
                        const LcLz4Chunk* d_info, uint8_t* d_slot, uint32_t* d_body, uint32_t* d_esz, cudaStream_t st);
void launch_zstd_emit(const Lz4Segs& g, const uint64_t* d_bfirst, uint64_t nblocks, const uint8_t* d_slot,
                      const uint32_t* d_body, const uint64_t* d_boff, const uint64_t* d_total, uint8_t* d_out,
                      uint64_t* d_frm_off, uint32_t* d_frm_len, cudaStream_t st);

// ProcessorParseTimestampNative (lc_exec.cuh): launch_ts_full runs the compiled format over every event with a value
// (one thread per event, d_full[i]); launch_ts_resolve applies the second-level cache and the verdict, one warp per
// group (events [d_grp[g], d_grp[g + 1])), and adds the five counters to d_counters (u64, zeroed by the caller).
void launch_ts_full(const LcTsConf* d_conf, const LcTsNow& now, const uint8_t* d_base, const LcTsSpans& sp, uint64_t n,
                    LcTsFull* d_full, cudaStream_t st);
void launch_ts_resolve(const LcTsConf* d_conf, const LcTsNow& now, const uint8_t* d_base, const LcTsSpans& sp, const LcTsFull* d_full,
                       const uint32_t* d_grp, uint64_t ngroups, int64_t* d_sec, uint32_t* d_nsec, uint8_t* d_status,
                       unsigned long long* d_counters, cudaStream_t st);

// ProcessorParseApsaraNative (lc_exec.cuh): launch_ap_scan reads each event's time form, full parse, hit
// nanoseconds, cache key and entry count (one thread per event; *d_bad |= 1 for an event past base_len, which is not
// read); launch_ap_resolve applies the time cache and the verdicts, one warp per group, and writes each event's entry
// count (0 unless parsed); after an exclusive sum of those counts (d_first), launch_ap_emit writes the entries.
void launch_ap_scan(const LcTsConf* d_conf, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_off,
                    const uint32_t* d_len, uint64_t n, const uint8_t* d_skey, uint32_t sklen, LcApEv* d_ev,
                    uint32_t* d_bad, cudaStream_t st);
void launch_ap_resolve(const LcTsNow& now, const LcApEv* d_ev, const uint32_t* d_grp, uint64_t ngroups,
                       uint8_t* d_status, int64_t* d_sec, uint32_t* d_nsec, int64_t* d_micro, uint32_t* d_nent,
                       unsigned long long* d_counters, cudaStream_t st);
void launch_ap_emit(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len, const uint8_t* d_status,
                    uint64_t n, const uint64_t* d_first, LcApEntry* d_entries, cudaStream_t st);

// ProcessorParseJsonNative (lc_exec.cuh): launch_json_count runs the fast walk, one thread per event, and writes each
// event's status, entry count, arena bytes and slow flag; an event the fast walk gives up on is appended to d_slow_list
// (*d_nslow) and launch_json_count_slow finishes it over that list.  *d_bad |= 1 for an event past base_len, which is
// not read.  counters[3] += key_not_found, out_failed, ok.  After exclusive sums of both counts (d_first, d_afirst),
// launch_json_emit and launch_json_emit_slow write the entries and arena bytes; *d_bad |= 2 when an event would not
// fill its ranges exactly (nothing is written past them).
void launch_json_count(const uint8_t* d_base, uint64_t base_len, const uint32_t* d_off, const uint32_t* d_len,
                       uint64_t n, const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, uint8_t* d_status, uint32_t* d_nent,
                       uint32_t* d_narena, uint8_t* d_slow, uint32_t* d_slow_list, uint32_t* d_nslow, uint32_t* d_bad,
                       unsigned long long* d_counters, cudaStream_t st);
void launch_json_count_slow(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len,
                            const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint32_t* d_slow_list, const uint32_t* d_nslow,
                            uint8_t* d_status, uint32_t* d_nent, uint32_t* d_narena, unsigned long long* d_counters,
                            cudaStream_t st);
void launch_json_emit(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                      const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint8_t* d_status, const uint8_t* d_slow,
                      const uint64_t* d_first, const uint64_t* d_afirst, LcJsonEntry* d_entries, uint8_t* d_arena,
                      uint32_t* d_bad, cudaStream_t st);
void launch_json_emit_slow(const uint8_t* d_base, const uint32_t* d_off, const uint32_t* d_len,
                           const uint8_t* d_skey, uint32_t sklen, const uint64_t* d_pow5, const uint8_t* d_status,
                           const uint32_t* d_slow_list, const uint32_t* d_nslow, const uint64_t* d_first,
                           const uint64_t* d_afirst, LcJsonEntry* d_entries, uint8_t* d_arena, uint32_t* d_bad,
                           cudaStream_t st);

// f4, split -> JSON chain (lc_exec.cuh: LcSplitJsonSlsCfg, keys on the device): the pieces off / len of the source
// value src, parsed by lc_json_parse_dev into status / first / ent / arena; win (one word per entry) and ev (one record
// per piece) are the resolve pass's output.  launch_json_resolve: d_list / d_nlist take the pieces of more than
// LC_JSON_SLS_WARP members (*d_nlist zeroed by the caller), d_scratch 3 * n_entries words.  Sizes as for
// launch_sls_sizes; d_counters: u64 [4] += successful, failed (LC_JSON_FAILED), discarded pieces, and pieces whose
// record would reach 4 GiB.
struct SplitJsonSlsTables {
    const uint8_t* src;
    const uint32_t* off;
    const uint32_t* len;
    const uint8_t* status;
    const uint64_t* first;
    const LcJsonEntry* ent;
    const uint8_t* arena;
    uint32_t* win;
    LcJsonSlsEv* ev;
};
void launch_json_resolve(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n, uint64_t n_entries,
                         uint32_t* d_list, uint32_t* d_nlist, uint32_t* d_scratch, cudaStream_t st);
void launch_split_json_sls_sizes(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n,
                                 uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                 cudaStream_t st);
void launch_split_json_sls_emit(const LcSplitJsonSlsCfg& c, const SplitJsonSlsTables& t, uint64_t n,
                                const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                cudaStream_t st);
// f4, split -> JSON -> timestamp chain (lc_exec.cuh: LcSplitJsonTsCfg).  launch_split_json_ts_tap: the dense value
// table (d_off, d_len) over d_val that the timestamp passes take, with each value copied into d_val (tc.val_cap bytes:
// the chunk's bytes at their own offsets, the arena's from tc.arena_at); LC_TS_NO_KEY: erased by the JSON stage, or no
// value.  It needs no resolve pass.  The size and emit passes are launch_split_json_sls_*'s (t.win / t.ev set) with
// each record's time from the timestamp tables ts; d_counters: u64 [9] += the chain's 8 counters (LC_SRTS_COUNTERS),
// then pieces whose record would reach 4 GiB.
void launch_split_json_ts_tap(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc, const SplitJsonSlsTables& t,
                              uint64_t n, uint8_t* d_val, uint32_t* d_off, uint32_t* d_len, cudaStream_t st);
void launch_split_json_ts_sls_sizes(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc,
                                    const SplitJsonSlsTables& t, const TsRowTables& ts, uint64_t n,
                                    uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                    cudaStream_t st);
void launch_split_json_ts_sls_emit(const LcSplitJsonSlsCfg& c, const LcSplitJsonTsCfg& tc,
                                   const SplitJsonSlsTables& t, const TsRowTables& ts, uint64_t n,
                                   const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                   cudaStream_t st);

// f4, split -> Apsara chain (lc_exec.cuh: LcSplitApsaraSlsCfg, keys on the device): the pieces off / len of the source
// value src, parsed by lc_apsara_parse_dev (src as its base) into status / sec / nsec / micro / first / ent.  Sizes as
// for launch_sls_sizes; d_counters: u64 [6] += lc_apsara_parse's five (discarded with the failed pieces erased), then
// the pieces whose record would reach 4 GiB.
struct SplitApsaraSlsTables {
    const uint8_t* src;
    const uint32_t* off;
    const uint32_t* len;
    const uint8_t* status;
    const int64_t* sec;
    const uint32_t* nsec;
    const int64_t* micro;
    const uint64_t* first;
    const LcApEntry* ent;
};
void launch_split_apsara_sls_sizes(const LcSplitApsaraSlsCfg& c, const SplitApsaraSlsTables& t, uint64_t n,
                                   uint32_t* d_rec_size, uint32_t* d_body_size, unsigned long long* d_counters,
                                   cudaStream_t st);
void launch_split_apsara_sls_emit(const LcSplitApsaraSlsCfg& c, const SplitApsaraSlsTables& t, uint64_t n,
                                  const uint64_t* d_rec_off, const uint32_t* d_body_size, uint8_t* d_out,
                                  cudaStream_t st);

} // namespace lck
