/*
 * lc_b200.h -- C-ABI of the H100-native log-parsing engine (libloongcollector_b200.so).
 *
 * POD only: plain pointers and sizes, int return codes, no exceptions, no C++/torch types.
 * These are the entry points a LoongCollector build binds to replace the CPU arithmetic inside
 *   Processor::Process(PipelineEventGroup&)      core/collection_pipeline/plugin/interface/Processor.h:27-37
 * for the four native processors on the hot path; each function cites the reference code whose
 * RESULT it reproduces bit-exactly.  The reference-side binding is shown in INTEGRATION.md.
 *
 * Conventions
 *  - "base" is the contiguous SourceBuffer allocation holding the group's bytes
 *    (core/common/memory/SourceBuffer.h:98-131,156-181); every offset is u32 relative to base.
 *  - Host-pointer entry points (no suffix) validate the event table against base_len (LC_ERR_INVALID_ARG), copy
 *    base + the event table to the GPU, run the kernels and copy the results back before returning.
 *    *_dev entry points take DEVICE pointers (arena already resident in HBM) and queue their kernels on the
 *    engine's current stream -- lc_engine_stream(), replaceable with lc_engine_set_stream().  The regex / delimiter
 *    *_dev calls never wait for the device (results are valid once the stream has drained: lc_engine_sync or the
 *    caller's own event); the split / multiline *_dev calls return a count and therefore synchronise.  *_dev
 *    callers guarantee ev_off[i] + ev_len[i] <= base_len (device tables are not re-read on the host).
 *  - One lc_engine per (GPU, host thread): mirrors the reference's per-thread regex copies
 *    (ProcessorParseRegexNative.cpp:64-67,255-257).  An engine is not thread-safe; regexes are immutable
 *    after compilation and may be shared between engines.
 *  - There is NO CPU fallback: if no CUDA device is usable every compute call fails with LC_ERR_CUDA.
 */
#ifndef LC_B200_H
#define LC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LC_OK 0
#define LC_ERR_INVALID_ARG 1
#define LC_ERR_CUDA 2          /* no device / CUDA runtime failure (message in lc_last_error) */
#define LC_ERR_REGEX_INVALID 3 /* pattern does not parse (reference: Init returns false, ParamExtractor.cpp:199-209) */
#define LC_ERR_REGEX_UNSUPPORTED 4 /* valid for boost but outside the automaton subset (back-refs, look-behind, multi-byte look-ahead...) */
#define LC_ERR_CAPACITY 5      /* caller-provided output capacity too small; *n_out holds the needed count */
#define LC_ERR_TOO_LARGE 6     /* buffer >= 4 GiB or >= 2^30 lines in one call */
#define LC_ERR_INTERNAL 7      /* a device pass would have written past its own output range; nothing was */

/* per-event status of lc_regex_parse (ProcessorParseRegexNative.cpp:186-253) */
#define LC_REGEX_OK 0
#define LC_REGEX_NOMATCH 1       /* regex_match false            -> out_failed++ (:225) */
#define LC_REGEX_KEYS_MISMATCH 2 /* what.size() <= keys.size()   -> fail, out_failed NOT incremented (:227-244) */

/* per-event status of lc_delim_parse (ProcessorParseDelimiterNative.cpp:206-364) */
#define LC_DELIM_OK 0
#define LC_DELIM_PARSE_FAIL 1 /* FSM error (DelimiterModeFsmParser.cpp:260-294) or SplitString false */
#define LC_DELIM_BLANK 2      /* empty / all-blank value: out_failed++, event left untouched (:220-242) */
#define LC_DELIM_COLUMNS 3    /* column-count rule failed (:285) */

/* flag bits of lc_multiline_split output events */
#define LC_ML_IS_LAST 1u /* isLastLog flag the reference passes to CreateNewEvent (rawSize rule, :329-332) */
#define LC_ML_MATCHED 2u /* emitted as a matched record (matched_events++), else an unmatched single line */

typedef struct lc_engine lc_engine_t;
typedef struct lc_regex lc_regex_t;

/* ---- library / engine ---------------------------------------------------------------------- */
const char* lc_version(void);
/* Thread-local message of the last failing call on this thread. */
const char* lc_last_error(void);
/* Number of visible CUDA devices (0 if none / runtime unusable). */
int lc_device_count(void);
/* Creates an engine bound to CUDA device `device` with its own stream, workspace and pinned staging.  The own stream
 * is a blocking stream: it is ordered with the legacy default stream (PyTorch's default stream), so device buffers
 * filled there before a *_dev call are complete when its kernels read them, and work queued there afterwards waits
 * for the engine's. */
int lc_engine_create(int device, lc_engine_t** out);
void lc_engine_destroy(lc_engine_t* e);
/* Blocks until all work queued on the engine's stream is complete. */
int lc_engine_sync(lc_engine_t* e);
/* CUDA stream (cudaStream_t) the engine queues its work on, for callers that enqueue their own work. */
void* lc_engine_stream(lc_engine_t* e);
/* Makes the engine queue on the caller's stream (cudaStream_t; NULL = back to the engine's own).  Drains the
 * previous stream first: the engine's workspace is re-used from call to call and ordered by the stream. */
int lc_engine_set_stream(lc_engine_t* e, void* stream);
/* Number of kernel launches issued by this engine so far (bench.py's gpu_launches). */
uint64_t lc_engine_launch_count(const lc_engine_t* e);
/* Pinned host memory helpers (a SourceBuffer arena allocated here is DMA-able without staging). */
void* lc_host_alloc(size_t bytes);
void lc_host_free(void* p);

/* ---- regex compilation (host only, no GPU needed) -------------------------------------------
 * Replaces boost::regex(pattern) at ProcessorParseRegexNative.cpp:66 and
 * ProcessorSplitMultilineLogStringNative.cpp:72-78.  *out is set (and must be freed) whenever the
 * return code is LC_OK or LC_ERR_REGEX_UNSUPPORTED/INVALID so that lc_regex_error() can be read. */
int lc_regex_compile(const char* pattern, size_t len, lc_regex_t** out);
void lc_regex_free(lc_regex_t* r);
const char* lc_regex_error(const lc_regex_t* r);
uint32_t lc_regex_ngroups(const lc_regex_t* r);
/* info[0..7] = mode (0 forward-only, 1 two-pass), byte classes, NFA walker states, context kinds,
 * reverse-DFA states, prefix-DFA states, table bytes, NFA instructions. */
void lc_regex_info(const lc_regex_t* r, uint32_t info[8]);

/* ---- a1: ProcessorSplitLogStringNative::ProcessEvent (inner/ProcessorSplitLogStringNative.cpp:101-174)
 * Cuts buf[0,len) on split_char.  Piece k = (out_off[k], out_len[k]); empty pieces kept; a trailing
 * split char yields no extra empty piece.  *n_out = number of pieces (even when > cap => LC_ERR_CAPACITY). */
int lc_split_lines(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, uint32_t* out_off,
                   uint32_t* out_len, uint64_t cap, uint64_t* n_out);
int lc_split_lines_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, uint8_t split_char, uint32_t* d_out_off,
                       uint32_t* d_out_len, uint64_t cap, uint64_t* n_out /* host */);

/* ---- a3: ProcessorParseRegexNative::RegexLogLineParser (ProcessorParseRegexNative.cpp:186-253)
 * For each event i (value = base[ev_off[i], +ev_len[i])): boost::regex_match over the whole value
 * (StringTools.cpp:183-211).  status[i] as LC_REGEX_*; on LC_REGEX_OK row i of cap_off/cap_len
 * ([n][ngroups], offsets relative to base) holds what[g+1] = (begin, length); groups that did not
 * participate report (end of value, 0).  Rows of failed events are zero-filled. */
int lc_regex_parse(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                   const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint32_t nkeys, uint8_t* status,
                   uint32_t* cap_off, uint32_t* cap_len);
int lc_regex_parse_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                       uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len);

/* Batched event groups -- Processor::Process(std::vector<PipelineEventGroup>&) (Processor.h:31): the arenas of many
 * groups (<= 512 KB each, LogFileReader.cpp:97) go up back to back into ONE packed device arena and are parsed by one
 * launch sequence, instead of one launch + six copies + one sync per group.  Span k = the bytes
 * [span_ptr[k], + span_len[k]) of one group's SourceBuffer chunk (DMA-able without staging when it was allocated
 * with lc_host_alloc); it lands at [span_dst[k], + span_len[k]) of the packed arena (16-byte aligned, ascending,
 * non-overlapping, below packed_len).  Events [span_first_ev[k], span_first_ev[k+1]) belong to span k; ev_off[] and
 * the returned cap_off[] are relative to the PACKED arena (host address = span_ptr[k] + (off - span_dst[k])). */
int lc_regex_parse_packed(lc_engine_t* e, const lc_regex_t* re, uint64_t nspans, const uint8_t* const* span_ptr,
                          const uint32_t* span_len, const uint32_t* span_dst, const uint64_t* span_first_ev,
                          uint64_t packed_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                          uint32_t nkeys, uint8_t* status, uint32_t* cap_off, uint32_t* cap_len);

/* Same, handing the spans back as they finish: on_done(ctx, first_span, span_count) is called on the calling thread, in
 * span order, once the result rows of those spans' events have landed in status / cap_off / cap_len -- later spans are
 * still being uploaded and parsed meanwhile, so the caller's per-event epilogue overlaps the GPU pipeline. */
typedef void (*lc_spans_done_fn)(void* ctx, uint64_t first_span, uint64_t span_count);
int lc_regex_parse_packed_cb(lc_engine_t* e, const lc_regex_t* re, uint64_t nspans, const uint8_t* const* span_ptr,
                             const uint32_t* span_len, const uint32_t* span_dst, const uint64_t* span_first_ev,
                             uint64_t packed_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                             uint32_t nkeys, uint8_t* status, uint32_t* cap_off, uint32_t* cap_len,
                             lc_spans_done_fn on_done, void* ctx);

/* Same, with the event table read in place from a strided table: event i = (d_ev_off[i * ev_stride],
 * d_ev_len[i * ev_stride]).  Lets one processor's output feed the next without a gather -- e.g. column k of
 * lc_delim_parse_dev's [n][max_fields] tables (d_f_off + k, d_f_len + k, stride max_fields) is the event table of
 * the regex that parses that column (the delimiter -> regex chain of a pipeline, BASELINE config C4). */
int lc_regex_parse_strided_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                               const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint32_t ev_stride, uint64_t n,
                               uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len);

/* Several patterns evaluated in ONE grid (BASELINE config C5 "multi-pattern"; north_star: "evaluate every log line
 * in the batch in one grid").  The reference runs one ProcessorParseRegexNative per pattern, each holding its own
 * boost::regex (ProcessorParseRegexNative.cpp:64-67), and a line parsed by pattern p sees exactly RegexLogLineParser
 * of that instance (:186-253).  Here all automata are resident in shared memory together and every line is tried on
 * the patterns in array order until one matches (== regex_match of `(?:p0)|(?:p1)|...`, groups numbered per
 * pattern); with sel != NULL line i is tried on pattern sel[i] only (LC_MULTI_ANY = on all, in order).
 * which[i] = index of the pattern that matched or LC_MULTI_NONE; status[i] as LC_REGEX_* for that pattern's nkeys;
 * rows of cap_off / cap_len are [n][row_pitch] (row_pitch >= the largest group count), columns beyond the matching
 * pattern's groups and rows of unmatched lines are zero.  1..8 patterns. */
#define LC_MULTI_NONE 0xFFu
#define LC_MULTI_ANY 0xFFu
int lc_regex_parse_multi(lc_engine_t* e, const lc_regex_t* const* res, uint32_t npat, const uint32_t* nkeys,
                         const uint8_t* base, uint64_t base_len, const uint32_t* ev_off, const uint32_t* ev_len,
                         uint64_t n, const uint8_t* sel, uint8_t* which, uint8_t* status, uint32_t row_pitch,
                         uint32_t* cap_off, uint32_t* cap_len);
int lc_regex_parse_multi_dev(lc_engine_t* e, const lc_regex_t* const* res, uint32_t npat, const uint32_t* nkeys,
                             const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                             const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_sel, uint8_t* d_which,
                             uint8_t* d_status, uint32_t row_pitch, uint32_t* d_cap_off, uint32_t* d_cap_len);

/* Boolean whole-value match == BoostRegexMatch(buf, size, reg, exception) without captures
 * (core/common/StringTools.cpp:213-236), the arithmetic of ProcessorFilterNative::IsMatched
 * (core/plugin/processor/ProcessorFilterNative.cpp:258-275): out_match[i] = 1 iff regex_match holds.
 * Only the reverse pass of the automaton runs. */
int lc_regex_match(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                   const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint8_t* out_match);
int lc_regex_match_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint8_t* d_out_match);

/* Anchored prefix probe == BoostRegexSearch / regex_search(match_continuous) (StringTools.cpp:263-288),
 * one boolean per event. */
int lc_regex_prefix_match(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                          const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint8_t* out_match);

/* ---- a2: ProcessorSplitMultilineLogStringNative::ProcessEvent (inner/...Multiline...cpp:127-393)
 * One source value buf[0,len).  start/cont/end: compiled pattern or NULL (pattern string empty, :68-70).
 * Output event k = (out_off[k], out_len[k], out_flags[k] = LC_ML_*) in reference emission order.
 * counters[0..2] += matched_events, input_lines, unmatched_lines (:82-84,106-107). */
int lc_multiline_split(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                       const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, uint32_t* out_off,
                       uint32_t* out_len, uint8_t* out_flags, uint64_t cap, uint64_t* n_out, uint64_t counters[3]);
int lc_multiline_split_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, const lc_regex_t* start,
                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, uint32_t* d_out_off,
                           uint32_t* d_out_len, uint8_t* d_out_flags, uint64_t cap, uint64_t* n_out /* host */,
                           uint64_t counters[3] /* host */);

/* ---- f3 (next row): LogFileReader::RemoveLastIncompleteLog (core/file_server/reader/LogFileReader.cpp:1997-2064) for
 * raw text (RawTextParser::GetLastLine, :2186-2204): how many leading bytes of a freshly read chunk form complete logs.
 * start / end: MultilineOptions::GetStartPatternReg / GetEndPatternReg or NULL (multiline mode iff one is set).
 * *keep_bytes = the function's return value ("the number of bytes left, including \n"); *rollback_line_feeds =
 * rollbackLineFeedCount (left untouched when allow_rollback == 0 or len == 0, like the reference).  The walk back
 * over the chunk's lines becomes "the last line whose probe flag is set" over the split pass's line table, so a raw
 * file chunk can go to the GPU before the reader knows where its last complete record ends. */
int lc_remove_last_incomplete_log(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                  const lc_regex_t* end, int allow_rollback, uint64_t* keep_bytes,
                                  int32_t* rollback_line_feeds);
int lc_remove_last_incomplete_log_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, const lc_regex_t* start,
                                      const lc_regex_t* end, int allow_rollback, uint64_t* keep_bytes /* host */,
                                      int32_t* rollback_line_feeds /* host */);

/* ---- a4: ProcessorParseDelimiterNative::ProcessEvent (ProcessorParseDelimiterNative.cpp:206-409)
 *          + DelimiterModeFsmParser::ParseDelimiterLine (core/parser/DelimiterModeFsmParser.cpp:260-294)
 * Per event: trim (:226-238), then the quote FSM (sep_len == 1 && quote != sep[0]) or the multi-char
 * SplitString (:366-409).  status[i] as LC_DELIM_*; nfields[i] = parsed column count; rows of
 * f_off/f_len/f_dq are [n][max_fields]: raw span of column j and, for the FSM path, the number of doubled
 * quotes inside it (the un-escaped value has f_len - f_dq bytes; the host shim materialises it in the
 * arena exactly as AddFieldWithUnQuote does, :83-113).  Columns beyond max_fields are counted, not stored. */
int lc_delim_parse(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                   const uint32_t* ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                   uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* status,
                   uint32_t* nfields, uint32_t* f_off, uint32_t* f_len, uint32_t* f_dq);
int lc_delim_parse_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                       const uint32_t* d_ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                       uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* d_status,
                       uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len, uint32_t* d_f_dq);

/* Same, with a column tap for processor chains (ProcessorParseDelimiterNative -> ProcessorParseRegexNative on one
 * column, BASELINE config C4): the (offset, length) of column tap_col of every line are ALSO written to the dense
 * tables d_tap_off / d_tap_len -- exactly the event table lc_regex_parse_dev needs for that column, so the next stage
 * reads 8 bytes per line instead of striding through the [n][max_fields] tables (rows of failed lines are (0, 0)). */
int lc_delim_parse_tap_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                           const uint32_t* d_ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                           uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* d_status,
                           uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len, uint32_t* d_f_dq,
                           uint32_t tap_col, uint32_t* d_tap_off, uint32_t* d_tap_len);

/* The same chain with HOST buffers (pinned memory recommended: lc_host_alloc): the arena is uploaded ONCE, in chunks of
 * whole events; per chunk the delimiter stage runs with the column tap and the regex stage on the tapped column, and both
 * stages' tables travel back while later chunks are still being uploaded (three streams, as in lc_regex_parse).
 * Outputs: the delimiter tables of lc_delim_parse ([n], [n][max_fields]) and the regex tables of lc_regex_parse for
 * column `column` ([n], [n][regex_nkeys groups]; a line whose delimiter stage failed or that has no such column is
 * parsed as the empty value).  Replaces: ProcessorParseDelimiterNative::Process followed by
 * ProcessorParseRegexNative::Process on one of its keys (core/plugin/processor/ProcessorParseDelimiterNative.cpp:206-364,
 * ProcessorParseRegexNative.cpp:132-168) -- a pipeline's `processors` list, collection_pipeline/CollectionPipeline.cpp. */
int lc_delim_regex_chain(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                         const uint32_t* ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                         uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* status,
                         uint32_t* nfields, uint32_t* f_off, uint32_t* f_len, uint32_t* f_dq, uint32_t column,
                         const lc_regex_t* re, uint32_t regex_nkeys, uint8_t* re_status, uint32_t* cap_off,
                         uint32_t* cap_len);

/* ---- f4 (next row): SLSEventGroupSerializer::Serialize for LOG events
 *          (core/collection_pipeline/serializer/SLSSerializer.cpp:254-269,377-395 over the writer of
 *           core/protobuf/sls/LogGroupSerializer.cpp:33-143,232-262)
 * Emits the `Logs` fields (field 1 of sls_logs::LogGroup), concatenated in event order.  Event i owns the contents
 * entries [ent_begin[i], ent_begin[i+1]) (m = ent_begin[n] entries in all); entry k is the key
 * base[ent_koff[k], +ent_klen[k]) and the value base[ent_voff[k], +ent_vlen[k]).  Events without entries are skipped
 * (LogEvent::Empty); Time below 2^28 is raised to 2^28 (the reference keeps the varint at 5 bytes);
 * ev_time_ns may be NULL, and ev_time_ns[i] == LC_SLS_NO_NS means "no Time_ns field" (nanoseconds disabled or not
 * set).  *out_len receives the total size; if it exceeds out_cap nothing is written and LC_ERR_CAPACITY is returned.
 * The group-level fields (Topic, Source, MachineUUID, LogTags) are a few bytes appended by the caller. */
#define LC_SLS_NO_NS 0xFFFFFFFFu
int lc_sls_serialize_logs(lc_engine_t* e, const uint8_t* base, uint64_t base_len, uint64_t n, const uint32_t* ev_time,
                          const uint32_t* ev_time_ns, const uint64_t* ent_begin, const uint32_t* ent_koff,
                          const uint32_t* ent_klen, const uint32_t* ent_voff, const uint32_t* ent_vlen, uint8_t* out,
                          uint64_t out_cap, uint64_t* out_len);

/* Device-fed variant for the regex -> serialise hand-over: the `Logs` fields of the events a ProcessorParseRegexNative
 * leaves behind, written straight from its DEVICE result tables (status / cap_off / cap_len of lc_regex_parse_dev,
 * rows of row_pitch entries) and the constant key strings -- no host-side (key, value) span lists, the bytes never
 * leave the GPU between parsing and the wire format.  Event i with LC_REGEX_OK carries keys[k] -> capture k for
 * k < nkeys in key order (AddLog per capture, ProcessorParseRegexNative.cpp:249-251; the source key is deleted,
 * :153-155); a failed event carries the one content fail_key -> the whole line when fail_key != NULL
 * (KeepingSourceWhenParseFail with RenamedSourceKey, :156-158) and is skipped otherwise (erased,
 * CommonParserOptions.cpp:99-117).  keys must be distinct.  d_ev_time_ns may be NULL; LC_SLS_NO_NS per event = no
 * Time_ns.  d_out receives the bytes on the device; *out_len (host) their count; LC_ERR_CAPACITY if > out_cap.
 * The fixed configuration of lc_sls_serialize_regex_dev below, which this calls with its own two content plans. */
int lc_sls_serialize_parsed_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                                const uint32_t* d_ev_len, const uint8_t* d_status, const uint32_t* d_cap_off,
                                const uint32_t* d_cap_len, uint32_t row_pitch, uint64_t n, const char* const* keys,
                                const uint32_t* key_lens, uint32_t nkeys, const char* fail_key, uint32_t fail_key_len,
                                const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                                uint64_t out_cap, uint64_t* out_len);

/* The full regex -> serialise hand-over: the `Logs` fields of the events ProcessorParseRegexNative::Process leaves
 * behind (ProcessorParseRegexNative.cpp:132-168, CommonParserOptions.cpp:91-117), written straight from the DEVICE
 * tables of one lc_regex_parse_dev call (d_status, [n][row_pitch] d_cap_off / d_cap_len, parsed with nkeys keys) and
 * the processor's configuration.  Every event is taken to be flat: a LogEvent whose only content is source_key -> its
 * line.  The contents such an event ends with depend only on the configuration and its status, so the configuration is
 * compiled once into two content plans -- LogEvent's SetContentNoCopy / DelContent applied to "the line" and
 * "capture j" -- which the kernels walk per event:
 *   LC_REGEX_OK: keys[j] -> capture j in key order; a repeated key overwrites the earlier content in place; a key
 *     equal to source_key replaces the line in place and the source is not deleted, else it is; then renamed_key ->
 *     line if keep_succeed and that key is not present.
 *   LC_REGEX_NOMATCH / LC_REGEX_KEYS_MISMATCH: the source is deleted; with keep_fail renamed_key -> line, then
 *     "__raw_log__" -> line if copy_raw, each unless that key is present; without keep_fail the event is erased.
 *   whole_line != 0 (Regex "(.*)", :147-148): no regex ran and d_status / d_cap_off / d_cap_len may be NULL; every
 *     event gets keys[0] (or "content" when nkeys == 0) -> line, and the source is deleted unless it is one of the keys.
 * renamed_key is CommonParserOptions' RenamedSourceKey (source_key when not configured).  Events without contents
 * emit nothing.  counters[3] (host, may be NULL) = ProcessorParseRegexNative's out_successful (every event not
 * erased), out_failed (LC_REGEX_NOMATCH only, :227-244) and discarded.  d_ev_time_ns may be NULL; LC_SLS_NO_NS per
 * event = no Time_ns.  d_out receives the bytes on the device; *out_len (host) their count; LC_ERR_CAPACITY if
 * > out_cap (nothing written, *out_len and counters set). */
int lc_sls_serialize_regex_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                               const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status, const uint32_t* d_cap_off,
                               const uint32_t* d_cap_len, uint32_t row_pitch, const char* const* keys,
                               const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                               uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                               int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                               const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                               uint64_t out_cap, uint64_t* out_len, uint64_t counters[3]);

/* The same with HOST buffers: parse (lc_regex_parse with nkeys keys; re may be NULL in whole-line mode) and serialise
 * in one call.  The arena goes up once, in chunks of whole events on a copy stream while earlier chunks are parsed and
 * sized; the capture tables stay on the device and only the wire bytes (out, in event order) and counters[3] come
 * back.  *out_len and counters are set on LC_OK and on LC_ERR_CAPACITY. */
int lc_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                       const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                       const uint32_t* ev_time_ns, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                       const char* source_key, uint32_t source_key_len, const char* renamed_key,
                       uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[3]);

/* Device-fed variant for the delimiter -> serialise hand-over: the `Logs` fields of the events a
 * ProcessorParseDelimiterNative leaves behind (ProcessorParseDelimiterNative.cpp:206-364), written straight from the
 * DEVICE tables of one lc_delim_parse_dev call (d_status, d_nfields, [n][max_fields] d_f_off / d_f_len / d_f_dq) and
 * the configuration the parse ran with.  Every event is taken to be flat: a LogEvent whose only content is
 * source_key -> its line.  Per event:
 *   LC_DELIM_OK: keys[j] -> column j in column order, doubled quotes collapsed (AddFieldWithUnQuote); in discard mode
 *     keys "_" and columns >= nkeys are skipped; in extend mode (extend != 0) column j >= nkeys gets "__column<j>__";
 *     in keep mode (neither flag) columns nkeys.. are re-joined as sep[0] + column each under "__column<nkeys>__"
 *     (the multi-byte split's remainder column already holds its separator).  A key equal to source_key replaces the
 *     source content in place (it comes first; a row too short to reach it keeps the line there).  keep_succeed adds
 *     renamed_key -> line unless that key is present.  A row with more columns than max_fields is walked again on the
 *     device from the start of its line.
 *   LC_DELIM_PARSE_FAIL / LC_DELIM_COLUMNS: with keep_fail, renamed_key -> line, then "__raw_log__" -> line if copy_raw
 *     and renamed_key is another key; without keep_fail the event is erased.
 *   LC_DELIM_BLANK: untouched, source_key -> the untrimmed line.
 * renamed_key is CommonParserOptions' RenamedSourceKey (source_key when not configured).  Events without contents
 * emit nothing.  Refused with LC_ERR_INVALID_ARG: repeated keys (except "_" in discard mode), keys or a source_key of
 * the form "__column<digits>__" in extend or keep mode, max_fields < nkeys + 1.  d_ev_time_ns may be NULL;
 * LC_SLS_NO_NS per event = no Time_ns.  d_out receives the bytes on the device; *out_len (host) their count;
 * LC_ERR_CAPACITY if > out_cap (nothing written). */
int lc_sls_serialize_delim_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                               const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status, const uint32_t* d_nfields,
                               const uint32_t* d_f_off, const uint32_t* d_f_len, const uint32_t* d_f_dq,
                               uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
                               int discard, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                               const char* source_key, uint32_t source_key_len, const char* renamed_key,
                               uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                               const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                               uint64_t out_cap, uint64_t* out_len);

/* The same with HOST buffers: parse (lc_delim_parse with allow_short, tables max_fields wide) and serialise in one
 * call.  The arena goes up once, in chunks of whole events on a copy stream while earlier chunks are parsed; the
 * tables stay on the device and only the wire bytes come back (out, in event order).  counters[4] = successful,
 * failed (parse failures), discarded (erased failures), blank events -- ProcessorParseDelimiterNative's out_successful,
 * discarded, and out_failed = failed + blank.  *out_len and counters are set on LC_OK and on LC_ERR_CAPACITY. */
int lc_delim_parse_sls(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                       const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time, const uint32_t* ev_time_ns,
                       const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard, int allow_short,
                       uint32_t max_fields, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                       const char* source_key, uint32_t source_key_len, const char* renamed_key,
                       uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, uint8_t* out,
                       uint64_t out_cap, uint64_t* out_len, uint64_t counters[4]);

/* Device-fed variant for the split -> serialise hand-over: the `Logs` fields of the events ProcessorSplitLogStringNative
 * or ProcessorSplitMultilineLogStringNative cut from ONE source value (ProcessorSplitLogStringNative.cpp:131-161,
 * ProcessorSplitMultilineLogStringNative.cpp:311-340), written straight from the DEVICE piece tables of one
 * lc_split_lines_dev or lc_multiline_split_dev call over d_src[0, src_len).  Piece k = d_src[d_off[k], +d_len[k])
 * becomes one record with the source event's time / time_ns (LC_SLS_NO_NS = no Time_ns):
 *   offset_key == NULL:      key -> piece  (a RAW event: pass key "content")
 *   offset_key != key:       key -> piece, offset_key -> decimal(src_pos + d_off[k])  (log.file.offset metadata)
 *   offset_key == key:       key -> decimal(src_pos + d_off[k])  (SetContentNoCopy replaces the piece in place)
 * Records are never empty.  d_out receives the bytes on the device; *out_len (host) their count; LC_ERR_CAPACITY if
 * > out_cap (nothing written).  LC_ERR_TOO_LARGE when src_len + key_len + offset_key_len + 96 >= 2^32. */
int lc_sls_serialize_spans_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                               const uint32_t* d_len, uint64_t n, const char* key, uint32_t key_len,
                               const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                               uint32_t time_ns, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len);

/* The same with a HOST source value: upload it once, split it on the device (lc_split_lines / lc_multiline_split
 * rules), serialise the pieces as above and bring back only the wire bytes.  *n_events (may be NULL) = number of
 * pieces; the multiline call adds to counters[3] as lc_multiline_split does.  *out_len, *n_events and counters are
 * set on LC_OK and on LC_ERR_CAPACITY. */
int lc_split_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, const char* key,
                 uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                 uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events);
int lc_multiline_split_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* key,
                           uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                           uint32_t time, uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* n_events, uint64_t counters[3]);

/* ---- f4: the split -> regex chain (ProcessorSplitLogStringNative or ProcessorSplitMultilineLogStringNative, then
 * ProcessorParseRegexNative with the same SourceKey -- BASELINE configs C2 / C3 on file input) to the SLS wire format.
 * The source event is flat: source_key -> the value, with its position src_pos, time and time_ns (LC_SLS_NO_NS = no
 * Time_ns).  Piece k enters the regex stage as [source_key -> piece] or, when offset_key != NULL (log.file.offset
 * metadata; an empty key is still a key), [source_key -> piece, offset_key -> decimal(src_pos + off[k])].  The regex
 * stage then runs as for lc_sls_serialize_regex_dev (keys .. whole_line), on that event: a regex key equal to
 * offset_key overwrites the digits in place; renamed_key or "__raw_log__" equal to offset_key is not added (the key is
 * present); a failed piece without keep_fail is erased (ShouldEraseEvent, CommonParserOptions.cpp:107-110).
 * counters[3] (may be NULL) = ProcessorParseRegexNative's out_successful, out_failed (LC_REGEX_NOMATCH) and discarded.
 * Refused with LC_ERR_INVALID_ARG: offset_key equal to source_key, and lc_sls_serialize_regex_dev's refusals.
 * LC_ERR_TOO_LARGE when src_len plus the key bytes reach 4 GiB, or a record would.
 *
 * lc_sls_serialize_split_regex_dev: from the DEVICE piece tables of one lc_split_lines_dev / lc_multiline_split_dev
 * call over d_src[0, src_len) and the DEVICE tables of lc_regex_parse_dev over those pieces (d_status, [n][row_pitch]
 * d_cap_off / d_cap_len; NULL in whole-line mode).  d_out receives the bytes; *out_len (host) their count;
 * LC_ERR_CAPACITY if > out_cap (nothing written, *out_len and counters set). */
int lc_sls_serialize_split_regex_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
                                     const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                     const char* source_key, uint32_t source_key_len, const char* renamed_key,
                                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                     int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                                     uint32_t time, uint32_t time_ns, uint8_t* d_out, uint64_t out_cap,
                                     uint64_t* out_len, uint64_t counters[3]);

/* The same with a HOST source value: upload it once, split it on the device (lc_split_lines / lc_multiline_split
 * rules), run lc_regex_parse_dev over the pieces (re may be NULL in whole-line mode), serialise, and bring back only
 * the wire bytes.  *n_events (may be NULL) = number of pieces; the multiline calls add the splitter's counters to
 * ml_counters[3] (may be NULL) as lc_multiline_split does.  *out_len, *n_events and the counters are set on LC_OK and
 * on LC_ERR_CAPACITY.  The _lz4 variants put tail[0, tail_len) behind the records and return ONE LZ4 block, as
 * lc_regex_parse_sls_lz4 does (*raw_len = records + tail bytes). */
int lc_split_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                             uint8_t split_char, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                             const char* source_key, uint32_t source_key_len, const char* renamed_key,
                             uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                             const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                             uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                             uint64_t counters[3]);
int lc_split_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                 uint8_t split_char, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                 const char* source_key, uint32_t source_key_len, const char* renamed_key,
                                 uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                 int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                                 uint32_t time, uint32_t time_ns, const uint8_t* tail, uint64_t tail_len,
                                 uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                 uint64_t* n_events, uint64_t counters[3]);
int lc_multiline_split_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                       const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                       int discard_unmatched, const char* const* keys, const uint32_t* key_lens,
                                       uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                                       const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                       int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
                                       uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                       uint64_t counters[3], uint64_t ml_counters[3]);
int lc_multiline_split_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                           const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                           int discard_unmatched, const char* const* keys, const uint32_t* key_lens,
                                           uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                                           const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                           int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
                                           uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                           uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                           uint64_t counters[3], uint64_t ml_counters[3]);

/* ---- f4: the split -> delimiter chain (ProcessorSplitLogStringNative or ProcessorSplitMultilineLogStringNative, then
 * ProcessorParseDelimiterNative with the same SourceKey -- BASELINE config C4 on file input) to the SLS wire format.
 * The source event is flat, as for the split -> regex chain, and piece k enters the delimiter stage as [source_key ->
 * piece] or, when offset_key != NULL, [source_key -> piece, offset_key -> decimal(src_pos + off[k])].  The delimiter
 * stage then runs as for lc_sls_serialize_delim_dev (sep .. copy_raw) on that event, and SetContentNoCopy replaces in
 * place, so a record's contents are: source_key's (the column keyed source_key, or deleted), the offset content (the
 * column keyed offset_key -- not written again in column order -- or the digits when the row failed, is too short to
 * reach it, or skips it as a discarded "_"), the other columns in column order, then renamed_key / "__raw_log__"
 * unless one of them is offset_key (the key is present).  A blank or empty piece is left untouched; a failed piece
 * without keep_fail keeps only the offset content and is erased (ShouldEraseEvent).  counters[4] (may be NULL) =
 * successful, failed, discarded, blank, as lc_delim_parse_sls counts them (out_failed = failed + blank).  Refused with
 * LC_ERR_INVALID_ARG: offset_key equal to source_key; unless discard, an offset_key of the form __column<digits>__
 * (a generated overflow key could collide with it on some rows); and lc_sls_serialize_delim_dev's refusals.
 * LC_ERR_TOO_LARGE when src_len reaches 0xFFFFFFF0, n reaches 2^30 or n * max_fields 2^32, or a record would reach
 * 4 GiB.
 *
 * lc_sls_serialize_split_delim_dev: from the DEVICE piece tables of one lc_split_lines_dev / lc_multiline_split_dev
 * call over d_src[0, src_len) and the DEVICE tables of lc_delim_parse_dev over those pieces (d_status, d_nfields,
 * [n][max_fields] d_f_off / d_f_len / d_f_dq).  d_out receives the bytes; *out_len (host) their count;
 * LC_ERR_CAPACITY if > out_cap (nothing written, *out_len and counters set). */
int lc_sls_serialize_split_delim_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                                     const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                                     uint8_t quote, int extend, int discard, const char* const* keys,
                                     const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                     uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                     int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                     uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                     uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[4]);

/* The same with a HOST source value: upload it once, split it on the device, run lc_delim_parse_dev over the pieces
 * (allow_short, max_fields as for lc_delim_parse_sls), serialise, and bring back only the wire bytes; *n_events,
 * ml_counters, the _lz4 variants and which outputs are set on LC_ERR_CAPACITY as for lc_split_regex_parse_sls. */
int lc_split_delim_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, const uint8_t* sep,
                             uint32_t sep_len, uint8_t quote, int extend, int discard, int allow_short,
                             uint32_t max_fields, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                             const char* source_key, uint32_t source_key_len, const char* renamed_key,
                             uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                             const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                             uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                             uint64_t counters[4]);
int lc_split_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char,
                                 const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                                 int allow_short, uint32_t max_fields, const char* const* keys,
                                 const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                 uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                 int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                 uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                 const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events, uint64_t counters[4]);
int lc_multiline_split_delim_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                       const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched,
                                       const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                                       int allow_short, uint32_t max_fields, const char* const* keys,
                                       const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                       uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                       int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                       uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                       uint64_t counters[4], uint64_t ml_counters[3]);
int lc_multiline_split_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched,
                                           const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
                                           int discard, int allow_short, uint32_t max_fields, const char* const* keys,
                                           const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                           uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                           int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                           uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                           uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                           uint64_t counters[4], uint64_t ml_counters[3]);

/* ---- f4: the split -> regex -> filter chain (the split -> regex chain, then ProcessorFilterNative /
 * processor_filter_regex_native; the pipeline of the reference's file-to-blackhole benchmark) to the SLS wire format.
 * The filter sees the event the
 * regex stage left behind: a leaf is regex_match of its key's value there, false when the key is absent
 * (ProcessorFilterNative.cpp:459-486); keys are compared as bytes.  prog is a postfix program: an entry < nleaves
 * pushes that leaf, LC_FILTER_NOT pops one value and pushes its negation, LC_FILTER_AND / LC_FILTER_OR pop two and
 * push the result; it must leave exactly one value.  nprog == 0 is BYPASS mode (every event kept; regs may be NULL).
 * Otherwise (RULE / EXPRESSION mode) an event without contents is removed whatever the leaves say (:83-117).  The
 * filter keeps event order and moves none of the regex stage's counters.  DiscardingNonUTF8 is not supported.
 * Refused with LC_ERR_INVALID_ARG: more than LC_FILTER_MAX_LEAVES leaves or LC_FILTER_MAX_PROG entries, a malformed
 * program (an unknown entry, a pop of an empty stack, more than 32 values on the stack, not one value at the end), a
 * NULL leaf regex in RULE / EXPRESSION mode.  LC_ERR_TOO_LARGE also when some leaf reads the offset digits and the
 * chunk has 2^32 / 20 pieces or more. */
#define LC_FILTER_MAX_LEAVES 32
#define LC_FILTER_MAX_PROG 128
#define LC_FILTER_NOT 0xFFFFFFFDu
#define LC_FILTER_AND 0xFFFFFFFEu
#define LC_FILTER_OR 0xFFFFFFFFu
typedef struct lc_filter_desc {
    uint32_t nleaves;
    const char* const* keys; /* key of leaf l: keys[l][0, key_lens[l]) */
    const uint32_t* key_lens;
    const lc_regex_t* const* regs; /* regex of leaf l, matched against the whole value */
    uint32_t nprog;
    const uint32_t* prog;
} lc_filter_desc_t;

/* Each takes its unfiltered sibling's arguments plus the filter, and counters[4] (may be NULL) = the regex stage's
 * three, then the events the filter removed.  Sizing, capacity, 4 GiB, LZ4 and tail rules are the siblings'; a chunk
 * whose pieces are all removed gives 0 bytes (the LZ4 calls: the block of the tail alone). */
int lc_sls_serialize_split_regex_filter_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len,
                                            const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                            const uint8_t* d_status, const uint32_t* d_cap_off,
                                            const uint32_t* d_cap_len, uint32_t row_pitch, const char* const* keys,
                                            const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                            uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                            int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                                            const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                                            uint32_t time, uint32_t time_ns, const lc_filter_desc_t* filter,
                                            uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
                                            uint64_t counters[4]);
int lc_split_regex_filter_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                    uint8_t split_char, const char* const* keys, const uint32_t* key_lens,
                                    uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                                    const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
                                    int copy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len,
                                    uint64_t src_pos, uint32_t time, uint32_t time_ns, const lc_filter_desc_t* filter,
                                    uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                    uint64_t counters[4]);
int lc_split_regex_filter_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                        uint8_t split_char, const char* const* keys, const uint32_t* key_lens,
                                        uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                                        const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                        int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
                                        uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                        const lc_filter_desc_t* filter, const uint8_t* tail, uint64_t tail_len,
                                        uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                        uint64_t* n_events, uint64_t counters[4]);
int lc_multiline_split_regex_filter_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                              const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                              int discard_unmatched, const char* const* keys, const uint32_t* key_lens,
                                              uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                                              const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                              int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
                                              uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                                              uint32_t time_ns, const lc_filter_desc_t* filter, uint8_t* out,
                                              uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                              uint64_t counters[4], uint64_t ml_counters[3]);
int lc_multiline_split_regex_filter_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const lc_filter_desc_t* filter,
    const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
    uint64_t* n_events, uint64_t counters[4], uint64_t ml_counters[3]);

/* ---- f4: the split -> regex -> timestamp chain (the split -> regex chain, then ProcessorParseTimestampNative with
 * SourceKey tkey, ProcessorParseTimestampNative.cpp:100-179; the processor documentation's nginx pipeline) to the SLS
 * wire format.  Pieces and the regex stage are exactly the split -> regex chain's (same arguments, offset metadata,
 * refusals and erase rule).  The row rule:
 *   - The timestamp stage sees the pieces the regex stage kept, in piece order, as ONE group (the second-level cache
 *     starts empty per call).  A piece the regex stage erased is no event of the stage: no counter, no cache step.
 *   - Its value is what the regex stage left under tkey: a capture (with repeated keys the plan's winner), the piece
 *     (KeepingSourceWhenParseSucceed, or a kept failure under SourceKey / RenamedSourceKey / "__raw_log__"), or
 *     nothing (LC_TS_NOT_FOUND).  A tkey that holds the offset digits (tkey equal to offset_key) is refused with
 *     LC_ERR_INVALID_ARG.  The value is read over [off, off + len) followed by NUL bytes, as lc_timestamp_parse reads.
 *   - LC_TS_OK: the record's Time is the parsed seconds truncated to 32 bits (raised to at least 2^28 as every
 *     record's); with enable_ns (mEnableTimestampNanosecond) Time_ns is the parsed nanoseconds, even 0 and even when
 *     the source event had none.  LC_TS_NOT_FOUND, LC_TS_FAILED: the source event's time / time_ns.  LC_TS_DISCARDED:
 *     no record.
 *   - time_ns is the source event's Time_ns as the serialiser writes it, so it must agree with enable_ns: a time_ns
 *     other than LC_SLS_NO_NS with enable_ns == 0 is refused with LC_ERR_INVALID_ARG (the records that keep the source
 *     time would carry Time_ns and the parsed ones would not).
 *   - counters[8] (may be NULL) = the regex stage's out_successful, out_failed, discarded, then the timestamp stage's
 *     key_not_found, out_failed, history_failure, discarded, out_successful.
 *
 * lc_split_regex_timestamp_tap_dev: from the DEVICE piece and regex tables (as for lc_sls_serialize_split_regex_dev)
 * and the regex stage's configuration, writes the DEVICE value table d_val_off / d_val_len[n] over d_src that
 * lc_timestamp_parse_dev takes with one group (ev_len LC_TS_NO_KEY: erased by the regex stage, or no tkey).  It
 * queues the work on the engine's stream and returns without waiting.
 * lc_sls_serialize_split_regex_timestamp_dev: lc_sls_serialize_split_regex_dev's arguments plus the DEVICE results
 * of that lc_timestamp_parse_dev call (d_ts_status, d_ts_sec, d_ts_nsec) and enable_ns.  Sizing query, capacity and
 * 4 GiB rules are the sibling's. */
struct lc_timestamp; /* lc_timestamp_t, compiled by lc_timestamp_compile below */
int lc_split_regex_timestamp_tap_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
                                     const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                     const char* source_key, uint32_t source_key_len, const char* renamed_key,
                                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                     int whole_line, const char* offset_key, uint32_t offset_key_len,
                                     const char* tkey, uint32_t tkey_len, uint32_t* d_val_off, uint32_t* d_val_len);
int lc_sls_serialize_split_regex_timestamp_dev(
    lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
    const uint8_t* d_status, const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
    const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
    uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
    int copy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, const uint8_t* d_ts_status, const int64_t* d_ts_sec, const uint32_t* d_ts_nsec, int enable_ns,
    uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]);

/* The same with a HOST source value: upload it once, split, regex, tap, both timestamp passes (ts compiled by
 * lc_timestamp_compile; now = time(NULL) of the call, discard_interval as for lc_timestamp_parse, -1 = no history
 * discard), size and emit (and LZ4), and bring back only the bytes.  *n_events, ml_counters, LZ4, the tail and the
 * capacity as for lc_split_regex_parse_sls.  A chunk whose pieces are all erased or discarded gives 0 bytes (the LZ4
 * calls: the block of the tail alone). */
int lc_split_regex_timestamp_parse_sls(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, uint8_t split_char,
    const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
    uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
    int copy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now,
    int32_t discard_interval, int enable_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
    uint64_t counters[8]);
int lc_split_regex_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, uint8_t split_char,
    const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
    uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
    int copy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now,
    int32_t discard_interval, int enable_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
    uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events, uint64_t counters[8]);
int lc_multiline_split_regex_timestamp_parse_sls(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out, uint64_t out_cap,
    uint64_t* out_len, uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]);
int lc_multiline_split_regex_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, const uint8_t* tail,
    uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
    uint64_t counters[8], uint64_t ml_counters[3]);

/* lc_regex_parse_sls / lc_delim_parse_sls finished as the SLS flusher finishes a group: the records, followed by
 * tail[0, tail_len) (the group-level fields: topic, source, machine uuid, tags), become ONE LZ4 block (the block format
 * of lc_lz4_compress_dev) and only the block comes back.  *raw_len = records + tail bytes (x-log-bodyrawsize),
 * *out_len = the block's size; if it exceeds out_cap, LC_ERR_CAPACITY and nothing is written to out.  *raw_len,
 * *out_len and counters are set on LC_OK and on LC_ERR_CAPACITY; the counters are those of the sibling call. */
int lc_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                           const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                           const uint32_t* ev_time_ns, const char* const* keys, const uint32_t* key_lens,
                           uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                           uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* raw_len, uint64_t counters[3]);
int lc_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                           const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time, const uint32_t* ev_time_ns,
                           const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                           int allow_short, uint32_t max_fields, const char* const* keys, const uint32_t* key_lens,
                           uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                           uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* raw_len, uint64_t counters[4]);

/* ---- f4: the delimiter -> regex chain (ProcessorParseDelimiterNative::Process, then ProcessorParseRegexNative::Process
 * whose SourceKey is one of the delimiter's keys -- BASELINE config C4) to the SLS wire format.  Every event is taken
 * to be flat: a LogEvent whose only content is source_key -> its line.  The chain's configuration is both stages'
 * arguments: the delimiter's (sep .. copy_raw, as for lc_sls_serialize_delim_dev) and the regex stage's (rkeys ..
 * rcopy_raw, whole_line, as for lc_sls_serialize_regex_dev; rsource_key = key k of the delimiter).
 * The regex stage reads key k's value: column k with its doubled quotes collapsed (AddFieldWithUnQuote) when the row
 * parsed and has the column; the whole line when the line stayed under key k (a short row whose source_key is key k,
 * a short row with keep_succeed whose renamed_key is key k, a kept failure whose renamed_key or "__raw_log__" is key
 * k, a blank row whose source_key is key k); otherwise no value (out_key_not_found; the delimiter's record is left as
 * it is).  With a value, key k's content is deleted in place -- or overwritten in place by the capture of a regex key
 * equal to k -- and the regex stage's other contents follow the delimiter's (ProcessorParseRegexNative.cpp:132-168).
 * Refused with LC_ERR_INVALID_ARG, besides each stage's own refusals: an rsource_key that is not one of the
 * delimiter's keys ("_" in discard mode is none), and a regex key, rrenamed_key or (rkeep_fail + rcopy_raw)
 * "__raw_log__" equal to a content the delimiter stage may leave besides key k's: another key, source_key,
 * renamed_key, "__raw_log__", "__column<digits>__" in extend or keep mode; also "_time_" and "_source_" both among
 * those without rkeep_fail (ShouldEraseEvent's rule would depend on the row).
 *
 * lc_delim_regex_tap_dev: the regex stage's event table from the DEVICE tables of one lc_delim_parse_dev call: value
 * i = d_base[d_val_off[i], + d_val_len[i]); a row without a value gets (its line's offset, 0).  A column with doubled
 * quotes is copied, collapsed, into d_base's side region [align16(base_len), base_cap), one slot per row in row order,
 * so captures stay offsets from d_base; *side_len = the bytes the copies take.  If they do not fit, LC_ERR_CAPACITY
 * and nothing is written (a sizing query); LC_ERR_TOO_LARGE when align16(base_len) + *side_len reaches 4 GiB.
 * Queued on the engine stream after one synchronise (the side size). */
int lc_delim_regex_tap_dev(lc_engine_t* e, uint8_t* d_base, uint64_t base_len, uint64_t base_cap,
                           const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status,
                           const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                           const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                           uint8_t quote, int extend, int discard, const char* const* keys, const uint32_t* key_lens,
                           uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                           uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                           const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                           const char* rsource_key, uint32_t rsource_key_len, const char* rrenamed_key,
                           uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed, int rcopy_raw, int whole_line,
                           uint32_t* d_val_off, uint32_t* d_val_len, uint64_t* side_len /* host */);

/* The `Logs` fields of the events the chain leaves behind, from the delimiter tables, the value table of
 * lc_delim_regex_tap_dev and the DEVICE tables of lc_regex_parse_dev over it (d_re_status, [n][row_pitch]
 * d_cap_off / d_cap_len, parsed with rnkeys keys; NULL in whole-line mode).  base_len covers the side copies.
 * counters[8] (host, may be NULL) = the delimiter's successful, failed, discarded, blank events (as lc_delim_parse_sls)
 * and the regex stage's out_successful, out_failed (LC_REGEX_NOMATCH), out_key_not_found and discarded events.
 * d_ev_time_ns may be NULL; LC_SLS_NO_NS per event = no Time_ns.  d_out receives the bytes on the device; *out_len
 * (host) their count; LC_ERR_CAPACITY if > out_cap (nothing written, *out_len and counters set). */
int lc_sls_serialize_delim_regex_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len,
                                     const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                                     const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off,
                                     const uint32_t* d_f_len, const uint32_t* d_f_dq, uint32_t max_fields,
                                     const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                                     const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                     const char* source_key, uint32_t source_key_len, const char* renamed_key,
                                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                     const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                                     const char* rsource_key, uint32_t rsource_key_len, const char* rrenamed_key,
                                     uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed, int rcopy_raw,
                                     int whole_line, const uint32_t* d_val_off, const uint32_t* d_val_len,
                                     const uint8_t* d_re_status, const uint32_t* d_cap_off, const uint32_t* d_cap_len,
                                     uint32_t row_pitch, const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns,
                                     uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]);

/* The same with HOST buffers: the arena goes up once, in chunks of whole events; per chunk the delimiter stage
 * (lc_delim_parse with allow_short, tables max_fields wide), the value tap, the regex stage over the values (re may be
 * NULL in whole-line mode) and the size pass run on the device, and only the wire bytes (out, in event order) and
 * counters[8] come back.  The device holds the lines plus at most their total length of side copies, which must stay
 * below 4 GiB (LC_ERR_TOO_LARGE).  *out_len and counters are set on LC_OK and on LC_ERR_CAPACITY.  The _lz4 variant
 * puts tail[0, tail_len) behind the records and returns ONE LZ4 block, as lc_delim_parse_sls_lz4 does. */
int lc_delim_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                             const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                             const uint32_t* ev_time_ns, int allow_short, uint32_t max_fields, const uint8_t* sep,
                             uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                             const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len,
                             const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
                             int copy_raw, const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys,
                             const char* rsource_key, uint32_t rsource_key_len, const char* rrenamed_key,
                             uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed, int rcopy_raw,
                             int whole_line, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]);
int lc_delim_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                                 const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                                 const uint32_t* ev_time_ns, int allow_short, uint32_t max_fields, const uint8_t* sep,
                                 uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
                                 const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                 uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                 int keep_fail, int keep_succeed, int copy_raw, const char* const* rkeys,
                                 const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key,
                                 uint32_t rsource_key_len, const char* rrenamed_key, uint32_t rrenamed_key_len,
                                 int rkeep_fail, int rkeep_succeed, int rcopy_raw, int whole_line, const uint8_t* tail,
                                 uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                 uint64_t* raw_len, uint64_t counters[8]);

/* ---- f4: the split -> delimiter -> regex chain (ProcessorSplitLogStringNative or
 * ProcessorSplitMultilineLogStringNative, then ProcessorParseDelimiterNative with the same SourceKey, then
 * ProcessorParseRegexNative reading one of the delimiter's keys -- BASELINE config C4 on file input) to the SLS wire
 * format.  The source event is flat, and piece k enters the chain as [source_key -> piece] or, when offset_key !=
 * NULL, [source_key -> piece, offset_key -> decimal(src_pos + off[k])].
 *   - The delimiter stage (sep .. copy_raw) runs as for lc_sls_serialize_split_delim_dev: the offset content follows
 *     source_key's and holds the column keyed offset_key when the row parsed and reaches it, else the digits; a blank
 *     piece is left untouched; a failed piece without keep_fail is erased.
 *   - The regex stage (rkeys .. whole_line) then runs as for lc_sls_serialize_delim_regex_dev: it reads key k's value
 *     (column k unquoted, the whole line, or none), deletes key k's content in place or overwrites it by a regex key
 *     equal to k, and its other contents follow the delimiter's.
 *   - A regex failure without rkeep_fail erases the piece when no content is left, or only the offset content
 *     (ShouldEraseEvent); the regex stage's discarded counter counts it.
 * counters[8] (may be NULL) as lc_sls_serialize_delim_regex_dev's.  Refused with LC_ERR_INVALID_ARG: what
 * lc_sls_serialize_split_delim_dev or lc_sls_serialize_delim_regex_dev refuses; an offset_key equal to rsource_key;
 * a regex key, rrenamed_key or "__raw_log__" equal to offset_key (the offset content counts as one more content the
 * delimiter stage leaves besides key k's, also for the "_time_" / "_source_" rule).
 *
 * lc_sls_serialize_split_delim_regex_dev: from the DEVICE piece tables of one lc_split_lines_dev /
 * lc_multiline_split_dev call over d_src[0, src_len), the delimiter tables of lc_delim_parse_dev over those pieces,
 * the value table of lc_delim_regex_tap_dev over the same tables (its side copies behind src_len in d_src) and the
 * regex tables of lc_regex_parse_dev over the values (NULL in whole-line mode).  d_out receives the bytes; *out_len
 * (host) their count; LC_ERR_CAPACITY if > out_cap (nothing written, *out_len and counters set).  LC_ERR_TOO_LARGE
 * when src_len reaches 0xFFFFFFF0, n reaches 2^30, n * max_fields or n * row_pitch 2^32, or a record would reach
 * 4 GiB. */
int lc_sls_serialize_split_delim_regex_dev(
    lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
    const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
    const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
    int discard, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
    uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
    int copy_raw, const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key,
    uint32_t rsource_key_len, const char* rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed,
    int rcopy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, const uint32_t* d_val_off, const uint32_t* d_val_len, const uint8_t* d_re_status,
    const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch, uint8_t* d_out, uint64_t out_cap,
    uint64_t* out_len, uint64_t counters[8]);

/* The same with a HOST source value: upload it once, split it on the device, run lc_delim_parse_dev over the pieces
 * (allow_short, max_fields as for lc_delim_parse_sls), the value tap, the regex stage over the values (re may be NULL
 * in whole-line mode), serialise, and bring back only the wire bytes; *n_events, ml_counters, the _lz4 variants and
 * which outputs are set on LC_ERR_CAPACITY as for lc_split_regex_parse_sls.  The side copies go behind the source on
 * the device: LC_ERR_TOO_LARGE, before anything is allocated, when align16(len) + len reaches 4 GiB; and past the
 * piece, column and capture limits of lc_split_delim_parse_sls / lc_split_regex_parse_sls. */
int lc_split_delim_regex_parse_sls(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, uint8_t split_char, int allow_short,
    uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
    const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len,
    const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
    const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key,
    uint32_t rsource_key_len, const char* rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed,
    int rcopy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t counters[8]);
int lc_split_delim_regex_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, uint8_t split_char, int allow_short,
    uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
    const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len,
    const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
    const char* const* rkeys, const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key,
    uint32_t rsource_key_len, const char* rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed,
    int rcopy_raw, int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
    uint32_t time_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
    uint64_t* raw_len, uint64_t* n_events, uint64_t counters[8]);
int lc_multiline_split_delim_regex_parse_sls(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, int allow_short, uint32_t max_fields,
    const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* const* rkeys,
    const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key, uint32_t rsource_key_len,
    const char* rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed, int rcopy_raw,
    int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
    uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t counters[8],
    uint64_t ml_counters[3]);
int lc_multiline_split_delim_regex_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, int allow_short, uint32_t max_fields,
    const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* const* rkeys,
    const uint32_t* rkey_lens, uint32_t rnkeys, const char* rsource_key, uint32_t rsource_key_len,
    const char* rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail, int rkeep_succeed, int rcopy_raw,
    int whole_line, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
    const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
    uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]);

/* ---- f4: the split -> delimiter -> timestamp chain (the split -> delimiter chain, then ProcessorParseTimestampNative
 * with SourceKey tkey, ProcessorParseTimestampNative.cpp:100-235; a CSV / TSV file whose logs take their time from
 * one of their columns) to the SLS wire format.  Pieces and the delimiter stage are exactly the split -> delimiter
 * chain's (same arguments, offset metadata, refusals, record layout, empty-record handling and erase rule).  The row
 * rule:
 *   - The timestamp stage sees the pieces the delimiter stage did not erase, in piece order, as ONE group (the
 *     second-level cache starts empty per call).  A failed piece erased without keep_fail is no event of the stage: no
 *     counter, no cache step.  A piece kept without a record (no contents left) is an event: it counts key_not_found.
 *   - Its value under tkey is what ProcessorParseDelimiterNative::ProcessEvent (:206-364, AddLog :411-419) leaves
 *     there.  The keys are distinct, so tkey names at most one column j; a "_" in discard mode names none.
 *       blank or empty piece (LC_DELIM_BLANK, left untouched): the piece when tkey is source_key, else none;
 *       parsed piece (LC_DELIM_OK), the first rule that applies: column j when the row reaches it (nf > j), with
 *       doubled quotes collapsed as AddFieldWithUnQuote does; the piece when tkey is source_key and source_key is one
 *       of the keys (a short row keeps it); the piece when keep_succeed is set and tkey is renamed_key; else none;
 *       kept failure (LC_DELIM_PARSE_FAIL, LC_DELIM_COLUMNS with keep_fail; source_key was deleted): the piece when tkey
 *       is renamed_key, or when tkey is "__raw_log__" and copy_raw is set, else none.
 *     A value is read over [off, off + len) followed by NUL bytes, as lc_timestamp_parse reads every value.
 *   - LC_TS_OK: the record's Time is the parsed seconds truncated to 32 bits (raised to at least 2^28 as every
 *     record's); with enable_ns Time_ns is the parsed nanoseconds.  LC_TS_NOT_FOUND, LC_TS_FAILED: the source event's
 *     time / time_ns.  LC_TS_DISCARDED: no record.
 *   - Refused with LC_ERR_INVALID_ARG beyond the split -> delimiter chain's refusals: tkey equal to offset_key; unless
 *     discard, a tkey of the form __column<digits>__ (a generated overflow key could hold it on some rows only); and a
 *     time_ns other than LC_SLS_NO_NS with enable_ns == 0 (some records would carry Time_ns and others not).
 *   - counters[9] (may be NULL) = the delimiter stage's successful, failed, discarded, blank (as
 *     lc_split_delim_parse_sls counts them), then the timestamp stage's key_not_found, out_failed, history_failure,
 *     discarded, out_successful.
 *
 * lc_split_delim_timestamp_tap_dev: from the DEVICE piece and delimiter tables (as for
 * lc_sls_serialize_split_delim_dev) and the delimiter stage's configuration, writes the value table d_val_off /
 * d_val_len[n] that lc_timestamp_parse_dev takes with one group over d_val (d_val_len LC_TS_NO_KEY: erased by the
 * delimiter stage, or no value), and copies each value into d_val at its own offset in d_src; a column with doubled
 * quotes is collapsed there.  val_cap must be at least src_len.  Only the tkey values are copied; the other bytes of
 * d_val are left as they are.  It queues the work on the engine's stream and returns without waiting.
 * lc_sls_serialize_split_delim_timestamp_dev: lc_sls_serialize_split_delim_dev's arguments plus the DEVICE results of
 * that lc_timestamp_parse_dev call (d_ts_status, d_ts_sec, d_ts_nsec) and enable_ns.  Sizing query, capacity and the
 * 4 GiB / 2^30 rules are the sibling's. */
int lc_split_delim_timestamp_tap_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                                     const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                                     uint8_t quote, int extend, int discard, const char* const* keys,
                                     const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                     uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                     int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                     uint32_t offset_key_len, const char* tkey, uint32_t tkey_len, uint8_t* d_val,
                                     uint64_t val_cap, uint32_t* d_val_off, uint32_t* d_val_len);
int lc_sls_serialize_split_delim_timestamp_dev(
    lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
    const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
    const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
    int discard, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
    uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
    int copy_raw, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
    const uint8_t* d_ts_status, const int64_t* d_ts_sec, const uint32_t* d_ts_nsec, int enable_ns, uint8_t* d_out,
    uint64_t out_cap, uint64_t* out_len, uint64_t counters[9]);

/* The same with a HOST source value: upload it once, split, run lc_delim_parse_dev (allow_short, max_fields as for
 * lc_split_delim_parse_sls), the tap, both timestamp passes (ts compiled by lc_timestamp_compile; now = time(NULL) of
 * the call, discard_interval as for lc_timestamp_parse, -1 = no history discard), size and emit (and LZ4), and bring
 * back only the bytes.  The value and timestamp tables stay in the engine's buffers.  *n_events, ml_counters, the
 * tail, raw_len and the behaviour on LC_ERR_CAPACITY are as for lc_split_delim_parse_sls.  A chunk whose pieces are
 * all erased or discarded gives 0 bytes (the LZ4 calls: the block of the tail alone). */
int lc_split_delim_timestamp_parse_sls(
    lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, const uint8_t* sep, uint32_t sep_len,
    uint8_t quote, int extend, int discard, int allow_short, uint32_t max_fields, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out,
    uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t counters[9]);
int lc_split_delim_timestamp_parse_sls_lz4(
    lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, const uint8_t* sep, uint32_t sep_len,
    uint8_t quote, int extend, int discard, int allow_short, uint32_t max_fields, const char* const* keys,
    const uint32_t* key_lens, uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, const uint8_t* tail,
    uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
    uint64_t counters[9]);
int lc_multiline_split_delim_timestamp_parse_sls(
    lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
    const lc_regex_t* end, int discard_unmatched, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
    int discard, int allow_short, uint32_t max_fields, const char* const* keys, const uint32_t* key_lens,
    uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
    int keep_fail, int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
    uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now,
    int32_t discard_interval, int enable_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
    uint64_t counters[9], uint64_t ml_counters[3]);
int lc_multiline_split_delim_timestamp_parse_sls_lz4(
    lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
    const lc_regex_t* end, int discard_unmatched, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
    int discard, int allow_short, uint32_t max_fields, const char* const* keys, const uint32_t* key_lens,
    uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
    int keep_fail, int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
    uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now,
    int32_t discard_interval, int enable_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
    uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events, uint64_t counters[9], uint64_t ml_counters[3]);

/* LZ4 compression of serialised groups (FlusherSLS's default compressor, LZ4Compressor::Compress =
 * LZ4_compress_default): segment g = d_in[d_seg_off[g], + d_seg_len[g]) becomes one LZ4 *block* (not a frame), the
 * blocks packed back to back in d_out: block g = d_out[d_blk_off[g], + d_blk_len[g]).  The bytes are deterministic;
 * they need not equal liblz4's.  A block is never larger than LZ4_compressBound(n) = n + n / 255 + 16, and an empty
 * segment is the single byte 0x00.  *out_len (host) = the total; if it exceeds out_cap, LC_ERR_CAPACITY and nothing is
 * written.  A segment over LZ4_MAX_INPUT_SIZE (0x7E000000) is refused with LC_ERR_TOO_LARGE. */
int lc_lz4_compress_dev(lc_engine_t* e, const uint8_t* d_in, uint64_t nseg, const uint64_t* d_seg_off,
                        const uint32_t* d_seg_len, uint8_t* d_out, uint64_t out_cap, uint64_t* d_blk_off,
                        uint32_t* d_blk_len, uint64_t* out_len);

/* The same with HOST segments seg_ptr[g][0, seg_len[g]): they go up in groups of whole segments while earlier groups
 * are parsed, and only the blocks come back (out, blk_off, blk_len on the host).  *out_len is set on LC_OK and on
 * LC_ERR_CAPACITY. */
int lc_lz4_compress(lc_engine_t* e, uint64_t nseg, const uint8_t* const* seg_ptr, const uint32_t* seg_len,
                    uint8_t* out, uint64_t out_cap, uint64_t* blk_off, uint32_t* blk_len, uint64_t* out_len);

/* zstd compression of serialised groups (FlusherSLS's CompressType "zstd", ZstdCompressor::Compress = ZSTD_compress
 * at level 1): segment g = d_in[d_seg_off[g], + d_seg_len[g]) becomes one complete zstd *frame* (RFC 8878), the frames
 * packed back to back in d_out: frame g = d_out[d_frm_off[g], + d_frm_len[g]).  The bytes are deterministic; they
 * need not equal libzstd's.  Frame header: Single_Segment_Flag set, Frame_Content_Size present, no checksum, no
 * dictionary; an empty segment is exactly 28 b5 2f fd 20 00 01 00 00.  Blocks hold at most 128 KiB of the segment,
 * and a block that would not shrink is stored Raw, so a frame is never larger than ZSTD_compressBound(n).  Matches are
 * those of the LZ4 compressor's parse pass (offsets up to 65 535); literals are Huffman-coded, sequences use the
 * predefined FSE tables (the layout is pinned in lc_exec.cuh).  *out_len (host) = the total; if it exceeds out_cap,
 * LC_ERR_CAPACITY and nothing is written.  A segment over LZ4_MAX_INPUT_SIZE (0x7E000000, the limit of the shared
 * parse pass) is refused with LC_ERR_TOO_LARGE.  Workspace: the LZ4 call's, plus 128 KiB per block of 128 KiB. */
int lc_zstd_compress_dev(lc_engine_t* e, const uint8_t* d_in, uint64_t nseg, const uint64_t* d_seg_off,
                         const uint32_t* d_seg_len, uint8_t* d_out, uint64_t out_cap, uint64_t* d_frm_off,
                         uint32_t* d_frm_len, uint64_t* out_len);

/* The same with HOST segments seg_ptr[g][0, seg_len[g]): they go up in groups of whole segments while earlier groups
 * are parsed, and only the frames come back (out, frm_off, frm_len on the host).  *out_len is set on LC_OK and on
 * LC_ERR_CAPACITY. */
int lc_zstd_compress(lc_engine_t* e, uint64_t nseg, const uint8_t* const* seg_ptr, const uint32_t* seg_len,
                     uint8_t* out, uint64_t out_cap, uint64_t* frm_off, uint32_t* frm_len, uint64_t* out_len);

/* ---- ProcessorParseTimestampNative (ProcessorParseTimestampNative.cpp:100-235, Strptime TimeUtil.cpp:112-160,
 *      strptime_ns Strptime.cpp)
 * lc_timestamp_compile is Init: SourceFormat becomes a device program; source_year is SourceYear (-1 unset, 0 deduce
 * the year from "now" as DeduceYear does, > 0 that year); tz_adjust is mLogTimeZoneOffsetSecond (SourceTimezone's
 * offset minus the local one, ParseLogTimeZoneOffsetSecond), subtracted after every successful full parse.  The
 * process's local zone is probed with mktime here (a per-year table of its standard and daylight offsets), so the
 * kernels need no tzdata; compile again after the zone changes.  Refused with LC_ERR_INVALID_ARG (message in
 * lc_last_error): %c, %x and %X (the locale's formats), a NUL byte inside the format, and a format of more than 96
 * directives and literal bytes.  Every other strptime_ns directive runs as the reference runs it: %Z consumes GMT or
 * UTC and nothing else; unknown conversions and %s inside a longer format fail every value.
 *
 * lc_timestamp_parse[_dev]: event i's value is base[ev_off[i], + ev_len[i]); ev_len[i] == LC_TS_NO_KEY means the
 * event has no SourceKey.  Events [grp[g], grp[g + 1]) form group g (grp has ngroups + 1 entries, grp[0] = 0 and
 * grp[ngroups] = n); ParseLogTime's second-level cache starts empty in every group and events keep their order in it.
 * now is time(NULL) of the call (the reference reads it per event); discard_interval >= 0 discards an event whose time
 * is more than that many seconds behind now (ilogtail_discard_old_data with ilogtail_discard_interval, 43200 by default;
 * pass -1 for one-time pipelines or with the flag off); a time <= 0 is always discarded.
 * Per event: status[i] as LC_TS_*; sec[i] / nsec[i] the time the event gets (SetTimestamp) for LC_TS_OK and the one
 * it would have got for LC_TS_DISCARDED, 0 for the other statuses.  counters[5] = key_not_found, out_failed, history_failure, discarded,
 * out_successful.  A value is read over [off, off + len) followed by NUL bytes: the reference hands strptime a
 * StringView that need not be terminated, so the two agree whenever the value is terminated.
 * The _dev calls take device tables and write d_counters (u64[5], device) without waiting for the device; the first
 * call of a compiled format on an engine also uploads its program from host memory. */
#define LC_TS_OK 0
#define LC_TS_NOT_FOUND 1  /* no SourceKey: out_key_not_found++, event kept */
#define LC_TS_FAILED 2     /* parse failure: out_failed++, event kept with its time unchanged */
#define LC_TS_DISCARDED 3  /* time <= 0 or too old: history_failure++, discarded++, event erased */
#define LC_TS_NO_KEY 0xFFFFFFFFu
typedef struct lc_timestamp lc_timestamp_t;
int lc_timestamp_compile(const char* format, size_t len, int32_t source_year, int32_t tz_adjust,
                         lc_timestamp_t** out);
void lc_timestamp_free(lc_timestamp_t* t);
int lc_timestamp_parse(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* base, uint64_t base_len,
                       const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* grp,
                       uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* sec, uint32_t* nsec,
                       uint8_t* status, uint64_t* counters);
int lc_timestamp_parse_dev(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, uint64_t base_len,
                           const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint32_t* d_grp,
                           uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec, uint32_t* d_nsec,
                           uint8_t* d_status, uint64_t* d_counters);
/* The same over capture column k of one lc_regex_parse_dev result (d_rx_status, [n][row_pitch] d_cap_off / d_cap_len),
 * read in place: a row the regex did not parse (status != LC_REGEX_OK) has no value (LC_TS_NOT_FOUND). */
int lc_timestamp_parse_capture_dev(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, uint64_t base_len,
                                   const uint8_t* d_rx_status, const uint32_t* d_cap_off, const uint32_t* d_cap_len,
                                   uint32_t row_pitch, uint32_t k, uint64_t n, const uint32_t* d_grp,
                                   uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec,
                                   uint32_t* d_nsec, uint8_t* d_status, uint64_t* d_counters);

/* ---- ProcessorParseApsaraNative (ProcessorParseApsaraNative.cpp: ProcessEvent 116-241, ApsaraEasyReadLogTimeParser
 *      251-323, FindBaseFields 342-361, ParseApsaraBaseFields 433-463)
 * lc_apsara_compile is Init: source_key is SourceKey; tz_adjust is mLogTimeZoneOffsetSecond (Timezone's offset minus
 * the local one, ParseLogTimeZoneOffsetSecond; 0 without a valid Timezone), subtracted from every parsed
 * "%Y-%m-%d %H:%M:%S" time and never from an epoch ("[1...]") time.  The process's local zone is probed here as
 * lc_timestamp_compile probes it; compile again after the zone changes.
 *
 * lc_apsara_parse[_dev]: event i's value is base[ev_off[i], + ev_len[i]); ev_len[i] == LC_TS_NO_KEY means the event
 * has no SourceKey.  Events [grp[g], grp[g + 1]) form group g (grp[0] = 0, grp[ngroups] = n, not decreasing); the time
 * cache starts empty in every group and follows event order.  now is time(NULL) of the call; discard_interval >= 0
 * discards an event whose time is more than that many seconds behind now, -1 = no such rule.
 * Per event:
 *   - status[i]: LC_APSARA_* in the low 3 bits; LC_APSARA_OVERWRITTEN is set on LC_APSARA_OK when a key:value key
 *     equals SourceKey (the event keeps its SourceKey content).
 *   - sec[i], nsec[i]: SetTimestamp's seconds and nanoseconds (micro * 1000 % 10^9) for LC_APSARA_OK, and the ones
 *     the event would have got for LC_APSARA_DISCARDED; micro[i] is logTime_in_micro (the "microtime" content is its
 *     "%ld" digits).  All three are 0 for the other statuses.
 *   - first[i] .. first[i + 1]: its entries (first has n + 1 entries; only LC_APSARA_OK events have any), in append
 *     order: the base fields (key_off one of LC_APSARA_KEY_*, key_len 0), then the key:value fields (key and value
 *     as offsets into base).  The "microtime" content follows them and is not an entry.
 * counters[5] = key_not_found, out_failed, history_failure, discarded, out_successful.  out_failed counts empty values
 * and failed time parses; discarded counts only the history discards: whether a failed event is erased depends on
 * its other contents (CommonParserOptions::ShouldEraseEvent), which the caller adds.
 * *n_entries is the number of entries; when it exceeds entry_cap the call returns LC_ERR_CAPACITY and writes no entry
 * (the other outputs are written), so entry_cap 0 makes a sizing query.  An event past base_len is refused with
 * LC_ERR_INVALID_ARG (the _dev call finds it on the device, without reading it).  The time string is read as a C
 * string and the 19-byte cache key past the end of base reads as NUL bytes (see lc_exec.cuh).
 * The _dev call takes device tables (d_grp as above, not checked).  Unlike the other _dev calls it waits for the
 * device before it returns: it reads the entry total on the host, and every output, the entries included, is written
 * when it returns, so it can be read from any stream.  The host call sizes its device copy of the entries from the
 * total, not from entry_cap. */
#define LC_APSARA_OK 0
#define LC_APSARA_NOT_FOUND 1 /* no SourceKey: out_key_not_found++, event kept */
#define LC_APSARA_EMPTY 2     /* empty value: out_failed++, event kept untouched */
#define LC_APSARA_FAILED 3    /* time parse failed or gave <= 0: out_failed++, the failure path */
#define LC_APSARA_DISCARDED 4 /* too old: history_failure++, discarded++, event erased */
#define LC_APSARA_OVERWRITTEN 0x80
#define LC_APSARA_KEY_LEVEL 0xFFFFFFF0u  /* __LEVEL__ */
#define LC_APSARA_KEY_THREAD 0xFFFFFFF1u /* __THREAD__ */
#define LC_APSARA_KEY_FILE 0xFFFFFFF2u   /* __FILE__ */
#define LC_APSARA_KEY_LINE 0xFFFFFFF3u   /* __LINE__ */
typedef struct lc_apsara lc_apsara_t;
typedef struct {
    uint32_t key_off, key_len, val_off, val_len;
} lc_apsara_entry_t;
int lc_apsara_compile(const char* source_key, size_t key_len, int32_t tz_adjust, lc_apsara_t** out);
void lc_apsara_free(lc_apsara_t* a);
int lc_apsara_parse(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* base, uint64_t base_len,
                    const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* grp, uint64_t ngroups,
                    int64_t now, int32_t discard_interval, uint8_t* status, int64_t* sec, uint32_t* nsec,
                    int64_t* micro, uint64_t* first, lc_apsara_entry_t* entries, uint64_t entry_cap,
                    uint64_t* n_entries, uint64_t* counters);
int lc_apsara_parse_dev(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* d_base, uint64_t base_len,
                        const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint32_t* d_grp,
                        uint64_t ngroups, int64_t now, int32_t discard_interval, uint8_t* d_status, int64_t* d_sec,
                        uint32_t* d_nsec, int64_t* d_micro, uint64_t* d_first, lc_apsara_entry_t* d_entries,
                        uint64_t entry_cap, uint64_t* n_entries, uint64_t* d_counters);

/* ---- ProcessorParseJsonNative (ProcessorParseJsonNative.cpp: ProcessEvent, JsonLogLineParserSimdJson,
 *      OptimizedValueToStringBuffer, ProcessNumberValueOptimized)
 * lc_json_compile is Init: source_key is SourceKey.  lc_json_parse[_dev]: event i's value is base[ev_off[i], +
 * ev_len[i]); ev_len[i] == LC_TS_NO_KEY means the event has no SourceKey.  No state crosses events, so there is no
 * group table.
 *
 * Verdict (pinned; the reference's default build parses with simdjson's on-demand API, the other build with
 * rapidjson, neither of which is linked here).  An event parses when its value is strict RFC 8259 JSON whose root is
 * an object: valid UTF-8 everywhere, no raw control bytes in strings, only valid escapes, \u surrogates in pairs,
 * numbers of the JSON grammar (no leading zeros, no '+', no NaN / Infinity), nesting depth (the root object is depth
 * 1) at most 1024 as simdjson's default limit, whitespace around the root object.  The document ends at the root's
 * closing brace; after it (and whitespace) a NUL byte ends the input and what follows it is ignored, as in both
 * reference paths (the reference's TestMultipleLines depends on it); any other byte fails the event.  Where
 * simdjson's lazy on-demand API accepts input this rule rejects -- malformed nested values such as {"a":[1,,2]},
 * trailing garbage, "tru" atoms -- the event fails here; rapidjson fails these inputs too.
 *
 * Rendering (pinned to the simdjson path):
 *   string          its unescaped bytes (\u0000 is a NUL byte, a surrogate pair 4 bytes of UTF-8)
 *   true / false    verbatim;  null: empty
 *   object / array  the source text from its opening to its matching closing bracket, inner whitespace kept
 *   integer         (no '.', no exponent) with '-': "%" PRId64 when it fits int64 ("-0" is "0"), else empty;
 *                   without '-': "%" PRIu64 when it fits uint64, else empty
 *   other numbers   std::to_string(double) = "%f" of the correctly rounded double (round half to even on the
 *                   sixth decimal); a double that overflows renders empty, one that underflows "0.000000" with its
 *                   sign
 * The empty renderings of out-of-range integers and overflowing doubles follow from the reference code and
 * simdjson's documented range errors; they are not confirmed by a run.  An empty rendering keeps the member.
 * Keys are unescaped; a key equal to SourceKey sets LC_JSON_OVERWRITTEN.
 *
 * Outputs:
 *   - status[i]: LC_JSON_* in the low bits, LC_JSON_OVERWRITTEN with LC_JSON_OK.
 *   - first[i] .. first[i + 1]: event i's entries (first has n + 1 words; only LC_JSON_OK events have any): the
 *     top-level members in document order, duplicates included (the caller applies them with overwrite, as
 *     AddLog(key, value, event) does).  An entry's key_off / val_off is an offset into base, or, with LC_JSON_ARENA
 *     set, (offset | LC_JSON_ARENA) into the arena.  The arena holds only bytes that are not in base: keys and
 *     strings with escapes, and every "%f" rendering, in document order, event after event.  Everything else is a
 *     span of base: strings without escapes (without their quotes), integers ("-0" points at its "0"), true /
 *     false, nested values.  An empty rendering is val_len 0 with val_off at the value's first byte.
 *   - counters[3] = key_not_found, out_failed, ok (events that parsed).  out_failed counts parse failures, not
 *     empty values (LC_JSON_EMPTY takes the failure path uncounted, as the reference does).
 * *n_entries and *arena_bytes are the totals; when either exceeds its cap the call returns LC_ERR_CAPACITY and writes
 * no entry and no arena byte (the other outputs are written), so caps of 0 make a sizing query.  An event past
 * base_len (ev_off + ev_len computed in 64 bits) is refused with LC_ERR_INVALID_ARG; the _dev call finds it on the
 * device without reading it.  base_len or an arena total of 2^31 or more is refused with LC_ERR_TOO_LARGE.
 * LC_ERR_INTERNAL reports an emit pass that would have left its event's ranges (nothing was written past them).
 * The _dev call takes device tables and, like lc_apsara_parse_dev, waits for the device before it returns. */
#define LC_JSON_OK 0
#define LC_JSON_NOT_FOUND 1 /* no SourceKey: out_key_not_found++, event kept */
#define LC_JSON_EMPTY 2     /* empty value: the failure path, not counted */
#define LC_JSON_FAILED 3    /* not a JSON object by the rule above: out_failed++, the failure path */
#define LC_JSON_OVERWRITTEN 0x80
#define LC_JSON_ARENA 0x80000000u
typedef struct lc_json lc_json_t;
typedef struct {
    uint32_t key_off, key_len, val_off, val_len;
} lc_json_entry_t;
int lc_json_compile(const char* source_key, size_t key_len, lc_json_t** out);
void lc_json_free(lc_json_t* js);
int lc_json_parse(lc_engine_t* e, const lc_json_t* js, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                  const uint32_t* ev_len, uint64_t n, uint8_t* status, uint64_t* first, lc_json_entry_t* entries,
                  uint64_t entry_cap, uint64_t* n_entries, uint8_t* arena, uint64_t arena_cap, uint64_t* arena_bytes,
                  uint64_t* counters);
int lc_json_parse_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_base, uint64_t base_len,
                      const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint8_t* d_status,
                      uint64_t* d_first, lc_json_entry_t* d_entries, uint64_t entry_cap, uint64_t* n_entries,
                      uint8_t* d_arena, uint64_t arena_cap, uint64_t* arena_bytes, uint64_t* d_counters);

/* ---- f4: the split -> JSON chain (ProcessorSplitLogStringNative or ProcessorSplitMultilineLogStringNative, then
 * ProcessorParseJsonNative with the same SourceKey -- the reference's documented pipeline for JSON-lines files) to
 * the SLS wire format.  The source event is flat, as for the split -> regex chain: SourceKey (js's) -> the value, with
 * its position src_pos, time and time_ns (LC_SLS_NO_NS = no Time_ns).  Piece k enters the JSON stage as [SourceKey ->
 * piece] or, when offset_key != NULL, [SourceKey -> piece, offset_key -> decimal(src_pos + off[k])], and the stage does
 * what ProcessorParseJsonNative::ProcessEvent does (oracle/json_parse.py restates it).  AddLog overwrites in place, so
 * a repeated key keeps its FIRST position and takes its LAST value; keys are equal when their rendered bytes are
 * ("a" and "\u0061" are one key).
 *   A piece that parses (LC_JSON_OK), contents in this order: SourceKey, only when a member has that key
 *   (LC_JSON_OVERWRITTEN), with the last such member's value (else SourceKey is deleted); the offset content, with the
 *   last member keyed offset_key if there is one, else the digits; every other distinct member key in order of first
 *   occurrence, with the value of its last occurrence; with keep_succeed, renamed_key -> piece unless that key is
 *   present (a member key, the offset key, or SourceKey while overwritten -- AddLog(..., false)).
 *   A piece that fails (LC_JSON_FAILED, or LC_JSON_EMPTY for an empty piece): SourceKey is deleted and the offset
 *   content stays; with keep_fail, renamed_key -> piece, and with copy_raw as well "__raw_log__" -> piece, neither
 *   added when already present; without keep_fail the piece is erased (ShouldEraseEvent).
 *   A piece left without contents (e.g. {} without an offset key) has no record and still counts as successful.
 *   Every record carries the source event's time and time_ns.  renamed_key is the effective RenamedSourceKey
 *   (SourceKey when the configuration leaves it empty).
 * counters[3] (may be NULL) = out_successful, out_failed (LC_JSON_FAILED only) and discarded, in the split -> regex
 * chain's order; a piece always holds SourceKey, so there is no key-not-found.  Refused with LC_ERR_INVALID_ARG: an
 * offset_key equal to SourceKey, bad arguments.  LC_ERR_TOO_LARGE: src_len >= 2^31 (the arena bit of the entries),
 * n >= 2^30, or a record that would reach 4 GiB.
 *
 * lc_sls_serialize_split_json_dev: from the DEVICE piece tables of one lc_split_lines_dev / lc_multiline_split_dev
 * call over d_src[0, src_len) and the DEVICE tables of lc_json_parse_dev over those pieces with js (d_status, d_first,
 * d_entries, d_arena).  d_out receives the bytes; *out_len (host) their count; LC_ERR_CAPACITY if > out_cap (nothing
 * written, *out_len and counters set). */
int lc_sls_serialize_split_json_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len,
                                    const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                    const uint64_t* d_first, const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                                    const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                    int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                                    uint64_t src_pos, uint32_t time, uint32_t time_ns, uint8_t* d_out,
                                    uint64_t out_cap, uint64_t* out_len, uint64_t counters[3]);

/* The same with a HOST source value: upload it once, split it on the device, run lc_json_parse_dev's passes over the
 * pieces, serialise, and bring back only the wire bytes; *n_events, ml_counters, the _lz4 variants and which outputs
 * are set on LC_ERR_CAPACITY as for lc_split_regex_parse_sls.  A chunk whose pieces are all erased or empty gives 0
 * bytes (the _lz4 calls then return the block of the tail alone). */
int lc_split_json_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, uint8_t split_char,
                            const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,
                            int copy_raw, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                            uint32_t time, uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                            uint64_t* n_events, uint64_t counters[3]);
int lc_split_json_parse_sls_lz4(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                uint8_t split_char, const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                                uint64_t src_pos, uint32_t time, uint32_t time_ns, const uint8_t* tail,
                                uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                uint64_t* raw_len, uint64_t* n_events, uint64_t counters[3]);
int lc_multiline_split_json_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                      const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                      int discard_unmatched, const char* renamed_key, uint32_t renamed_key_len,
                                      int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                      uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                      uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                      uint64_t counters[3], uint64_t ml_counters[3]);
int lc_multiline_split_json_parse_sls_lz4(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                          const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                          int discard_unmatched, const char* renamed_key, uint32_t renamed_key_len,
                                          int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                          uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                          const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                          uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                          uint64_t counters[3], uint64_t ml_counters[3]);

/* ---- f4: the split -> JSON -> timestamp chain (the split -> JSON chain, then ProcessorParseTimestampNative with
 * SourceKey tkey, ProcessorParseTimestampNative.cpp:100-235; a JSON-lines file whose logs take their time from one of
 * their members) to the SLS wire format.  Pieces and the JSON stage are exactly the split -> JSON chain's (same
 * arguments, offset metadata, refusals, record layout and erase rule).  The row rule:
 *   - The timestamp stage sees the pieces the JSON stage kept, in piece order, as ONE group (the second-level cache
 *     starts empty per call).  A piece the JSON stage erased (failed, without keep_fail) is no event of the stage: no
 *     counter, no cache step.  A parsed piece left without contents ({} without an offset key or keep_succeed) is an
 *     event: it counts key_not_found and still has no record.
 *   - Its value under tkey, keys comparing by their rendered bytes ("time" and "\u0074ime" are one key):
 *       a parsed piece (LC_JSON_OK): the rendered value of the LAST member keyed tkey (so tkey == SourceKey finds a
 *       member that overwrote it), else the piece when tkey is renamed_key and keep_succeed is set, else none
 *       (LC_TS_NOT_FOUND; tkey == SourceKey without such a member included: the stage deleted SourceKey);
 *       a kept failure (LC_JSON_FAILED, LC_JSON_EMPTY): the piece when tkey is renamed_key, or when tkey is
 *       "__raw_log__" and copy_raw is set, else none.
 *     A value is read over [off, off + len) followed by NUL bytes, as lc_timestamp_parse reads every value: an
 *     integer member is its digit span ("ts":1700000000), -0 is "0", and a non-integer number is its %f rendering.
 *   - LC_TS_OK: the record's Time is the parsed seconds truncated to 32 bits (raised to at least 2^28 as every
 *     record's); with enable_ns Time_ns is the parsed nanoseconds.  LC_TS_NOT_FOUND, LC_TS_FAILED: the source event's
 *     time / time_ns.  LC_TS_DISCARDED: no record.
 *   - Refused with LC_ERR_INVALID_ARG beyond the split -> JSON chain's refusals: tkey equal to offset_key, and a
 *     time_ns other than LC_SLS_NO_NS with enable_ns == 0 (some records would carry Time_ns and others not).
 *   - counters[8] (may be NULL) = the JSON stage's out_successful, out_failed, discarded, then the timestamp stage's
 *     key_not_found, out_failed, history_failure, discarded, out_successful.
 *
 * lc_split_json_timestamp_tap_dev: from the DEVICE piece and JSON tables (as for lc_sls_serialize_split_json_dev) and
 * the JSON stage's configuration, writes the value table d_val_off / d_val_len[n] that lc_timestamp_parse_dev takes
 * with one group over d_val (ev_len LC_TS_NO_KEY: erased by the JSON stage, or no value), and copies each value into
 * d_val: a value in the chunk to its own offset, a value in the arena to src_len + its arena offset.  val_cap must be
 * at least src_len + the arena's bytes (lc_json_parse_dev's *arena_bytes); a value that would end past val_cap gets
 * no value.  Only the tkey values are copied; the other bytes of d_val are left as they are.  It queues the work on
 * the engine's stream and returns without waiting.
 * lc_sls_serialize_split_json_timestamp_dev: lc_sls_serialize_split_json_dev's arguments plus the DEVICE results of
 * that lc_timestamp_parse_dev call (d_ts_status, d_ts_sec, d_ts_nsec) and enable_ns.  Sizing query, capacity and the
 * 2 GiB / 2^30 / 4 GiB rules are the sibling's. */
int lc_split_json_timestamp_tap_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len,
                                    const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                    const uint64_t* d_first, const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                                    const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                    int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                                    const char* tkey, uint32_t tkey_len, uint8_t* d_val, uint64_t val_cap,
                                    uint32_t* d_val_off, uint32_t* d_val_len);
int lc_sls_serialize_split_json_timestamp_dev(
    lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
    const uint32_t* d_len, uint64_t n, const uint8_t* d_status, const uint64_t* d_first,
    const lc_json_entry_t* d_entries, const uint8_t* d_arena, const char* renamed_key, uint32_t renamed_key_len,
    int keep_fail, int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
    uint32_t time, uint32_t time_ns, const uint8_t* d_ts_status, const int64_t* d_ts_sec, const uint32_t* d_ts_nsec,
    int enable_ns, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]);

/* The same with a HOST source value: upload it once, split, run the JSON passes, the tap, both timestamp passes (ts
 * compiled by lc_timestamp_compile; now = time(NULL) of the call, discard_interval as for lc_timestamp_parse, -1 = no
 * history discard), size and emit (and LZ4), and bring back only the bytes.  The value and timestamp tables stay in
 * the engine's buffers.  *n_events, ml_counters, the tail, raw_len and the behaviour on LC_ERR_CAPACITY are as for
 * lc_split_json_parse_sls.  A chunk whose pieces are all erased or discarded gives 0 bytes (the LZ4 calls: the block
 * of the tail alone). */
int lc_split_json_timestamp_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                      uint8_t split_char, const char* renamed_key, uint32_t renamed_key_len,
                                      int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                      uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                      const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now,
                                      int32_t discard_interval, int enable_ns, uint8_t* out, uint64_t out_cap,
                                      uint64_t* out_len, uint64_t* n_events, uint64_t counters[8]);
int lc_split_json_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, uint8_t split_char,
    const char* renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
    const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
    const char* tkey, uint32_t tkey_len, const struct lc_timestamp* ts, int64_t now, int32_t discard_interval,
    int enable_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
    uint64_t* raw_len, uint64_t* n_events, uint64_t counters[8]);
int lc_multiline_split_json_timestamp_parse_sls(
    lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out,
    uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]);
int lc_multiline_split_json_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* renamed_key,
    uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
    uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns, const char* tkey, uint32_t tkey_len,
    const struct lc_timestamp* ts, int64_t now, int32_t discard_interval, int enable_ns, const uint8_t* tail,
    uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
    uint64_t counters[8], uint64_t ml_counters[3]);

/* ---- f4: the split -> Apsara chain (ProcessorSplitLogStringNative or ProcessorSplitMultilineLogStringNative, then
 * ProcessorParseApsaraNative with the same SourceKey -- input_file, processor_parse_apsara_native, a flusher) to the
 * SLS wire format.  The source event is flat, as for the split -> JSON chain: SourceKey (ap's) -> the value, with its
 * position src_pos, time and time_ns (LC_SLS_NO_NS = no Time_ns).  Piece k enters the Apsara stage as [SourceKey ->
 * piece] or, when offset_key != NULL, [SourceKey -> piece, offset_key -> decimal(src_pos + off[k])], and the stage does
 * what ProcessorParseApsaraNative::ProcessEvent does (oracle/apsara.py restates it) with the time cache over the
 * pieces in order, the chunk as lc_apsara_parse_dev's base.  AppendContentNoCopy never removes a duplicate, so every
 * field is appended, duplicates included.
 *   A piece that parses (LC_APSARA_OK): its own time and, with enable_ns, Time_ns = its nanoseconds; contents in this
 *   order: the piece (key SourceKey); the offset content; the base fields as found (__LEVEL__, __THREAD__, __FILE__,
 *   __LINE__); the key:value fields in order, duplicates kept, keys equal to the offset key, a base-field name or
 *   "microtime" included; "microtime" -> the "%ld" digits of logTime_in_micro.  Then DelContent(SourceKey) removes
 *   the NEWEST entry keyed SourceKey -- "microtime" when SourceKey is "microtime", else the base field of that name
 *   when there is one, else the piece -- unless a key:value key equals SourceKey (LC_APSARA_OVERWRITTEN: every
 *   SourceKey entry stays).  With keep_succeed, renamed_key -> piece unless a content left has that key.
 *   An empty piece (LC_APSARA_EMPTY): kept untouched, [SourceKey -> "", the offset content], the source event's time.
 *   A piece that fails (LC_APSARA_FAILED): SourceKey is deleted and the offset content stays; with keep_fail,
 *   renamed_key -> piece, and with copy_raw as well "__raw_log__" -> piece, neither added when already present;
 *   without keep_fail the piece is erased (ShouldEraseEvent: nothing but the offset content is left).  The source
 *   event's time and time_ns.
 *   A piece too old for discard_interval (LC_APSARA_DISCARDED) is erased.
 *   renamed_key is the effective RenamedSourceKey (SourceKey when the configuration leaves it empty).
 * counters[5] (may be NULL) in lc_apsara_parse's order: key_not_found (0: a piece always holds SourceKey), out_failed
 * (empty and failed pieces), history_failure, discarded (the too-old pieces and the failed pieces erased), and
 * out_successful -- the counters ProcessorParseApsaraNative::Process moves.  Refused with LC_ERR_INVALID_ARG: an
 * offset_key equal to SourceKey, a time_ns other than LC_SLS_NO_NS without enable_ns (the kept pieces would write
 * Time_ns and the parsed ones not), bad arguments.  LC_ERR_TOO_LARGE: src_len >= 0xFFFFFFF0 (lc_apsara_parse_dev's
 * offsets stay below its LC_APSARA_KEY_* tags), n >= 2^30, or a record that would reach 4 GiB.
 *
 * lc_sls_serialize_split_apsara_dev: from the DEVICE piece tables of one lc_split_lines_dev / lc_multiline_split_dev
 * call over d_src[0, src_len) and the DEVICE tables of lc_apsara_parse_dev over those pieces with ap, d_src as base
 * and one group (d_status, d_sec, d_nsec, d_micro, d_first, d_entries).  d_out receives the bytes; *out_len (host)
 * their count; LC_ERR_CAPACITY if > out_cap (nothing written, *out_len and counters set). */
int lc_sls_serialize_split_apsara_dev(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* d_src, uint64_t src_len,
                                      const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                      const uint8_t* d_status, const int64_t* d_sec, const uint32_t* d_nsec,
                                      const int64_t* d_micro, const uint64_t* d_first,
                                      const lc_apsara_entry_t* d_entries, const char* renamed_key,
                                      uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                      const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                                      uint32_t time_ns, int enable_ns, uint8_t* d_out, uint64_t out_cap,
                                      uint64_t* out_len, uint64_t counters[5]);

/* The same with a HOST source value: upload it once, split it on the device, run lc_apsara_parse_dev's passes over the
 * pieces (the chunk as one group; now = time(NULL) of the caller, discard_interval as for lc_apsara_parse, -1 = no
 * history discard), serialise, and bring back only the wire bytes; *n_events, ml_counters, the _lz4 variants and which
 * outputs are set on LC_ERR_CAPACITY as for lc_split_regex_parse_sls.  A chunk whose pieces are all erased gives 0
 * bytes (the _lz4 calls then return the block of the tail alone). */
int lc_split_apsara_parse_sls(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                              uint8_t split_char, const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                              int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                              uint64_t src_pos, uint32_t time, uint32_t time_ns, int enable_ns, int64_t now,
                              int32_t discard_interval, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                              uint64_t* n_events, uint64_t counters[5]);
int lc_split_apsara_parse_sls_lz4(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                  uint8_t split_char, const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                  int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                                  uint64_t src_pos, uint32_t time, uint32_t time_ns, int enable_ns, int64_t now,
                                  int32_t discard_interval, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                                  uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                  uint64_t counters[5]);
int lc_multiline_split_apsara_parse_sls(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                        const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                        int discard_unmatched, const char* renamed_key, uint32_t renamed_key_len,
                                        int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                        uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,
                                        int enable_ns, int64_t now, int32_t discard_interval, uint8_t* out,
                                        uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t counters[5],
                                        uint64_t ml_counters[3]);
int lc_multiline_split_apsara_parse_sls_lz4(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                            const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                            int discard_unmatched, const char* renamed_key, uint32_t renamed_key_len,
                                            int keep_fail, int keep_succeed, int copy_raw, const char* offset_key,
                                            uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                                            uint32_t time_ns, int enable_ns, int64_t now, int32_t discard_interval,
                                            const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                            uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                            uint64_t counters[5], uint64_t ml_counters[3]);

#ifdef __cplusplus
}
#endif
#endif /* LC_B200_H */
