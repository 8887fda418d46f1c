/*
 * lc_b200_host.h -- C entry points of the C++ host layer (loongcollector_b200/host): the GPU-backed
 * replacements of the reference's Processor subclasses, driven through JSON event groups exactly like the
 * reference's unit tests drive them (PipelineEventGroup::FromJsonString / ToJsonString,
 * core/models/PipelineEventGroup.cpp:432-483).  A LoongCollector build links the C++ classes directly
 * (INTEGRATION.md); these functions exist so that tests in any language can replay the reference fixtures.
 */
#ifndef LC_B200_HOST_H
#define LC_B200_HOST_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct lc_host_processor lc_host_processor_t;

/* type: "processor_split_string_native" | "processor_split_multiline_log_string_native" |
 *       "processor_parse_regex_native" | "processor_parse_delimiter_native" (the reference's plugin names).
 * Returns NULL when Init(config) fails; *err_out (if not NULL) then holds a malloc'd message. */
lc_host_processor_t* lc_host_processor_create(const char* type, const char* config_json, char** err_out);
void lc_host_processor_destroy(lc_host_processor_t* p);
/* Runs Processor::Process(PipelineEventGroup&) on the group described by group_json and returns the group's
 * ToJsonString(enable_event_meta) ("null" for an empty group) as a malloc'd string; NULL + *err_out on error. */
char* lc_host_processor_process(lc_host_processor_t* p, const char* group_json, int enable_event_meta, char** err_out);
/* Runs Processor::Process(std::vector<PipelineEventGroup>&) -- one call for all groups, as a pipeline hands them over
 * -- on the JSON array of groups groups_json and returns the array of their ToJson(enable_event_meta) as a malloc'd
 * string; NULL + *err_out on error. */
char* lc_host_processor_process_groups(lc_host_processor_t* p, const char* groups_json, int enable_event_meta,
                                       char** err_out);
/* {"counter": value, ...} with the reference's counter meanings. */
char* lc_host_processor_counters(const lc_host_processor_t* p);
/* The process-wide flags ilogtail_discard_old_data / ilogtail_discard_interval as the time-parsing processors
 * (processor_parse_timestamp_native, processor_parse_apsara_native) read them: on with 43200 s by default, off for
 * one-time pipelines.  Returns 0, or -1 for another processor. */
int lc_host_processor_set_discard_old_data(lc_host_processor_t* p, int enabled, int32_t interval);
void lc_host_string_free(char* s);

/* SLSEventGroupSerializer::Serialize (core/collection_pipeline/serializer/SLSSerializer.cpp:162-252) of the LOG or RAW
 * group described by group_json; enable_ns = GlobalConfig::mEnableTimestampNanosecond.  Returns the malloc'd wire
 * bytes (free with lc_host_string_free) and their length, or NULL + *err_out = the reference's error message. */
char* lc_host_sls_serialize(const char* group_json, int enable_ns, unsigned long long* len_out, char** err_out);

/* SerializeSls of the processor p on the group described by group_json (p must be a
 * "processor_parse_delimiter_native", a "processor_parse_regex_native", a "processor_split_string_native" or a
 * "processor_split_multiline_log_string_native"): the malloc'd wire bytes and their length,
 * or NULL + *err_out = the serializer's error message.  With process_then_serialize != 0 it runs Process(group) + SLSEventGroupSerializer::Serialize on the
 * same in-memory group instead -- the result SerializeSls must equal byte for byte.  (lc_host_processor_process +
 * lc_host_sls_serialize differ from both in content order: a JSON round trip lists the contents by key.)  An engine
 * failure or a bad group returns NULL + *fail_out instead. */
char* lc_host_processor_serialize_sls(lc_host_processor_t* p, const char* group_json, int enable_ns,
                                      int process_then_serialize, unsigned long long* len_out, char** err_out,
                                      char** fail_out);

/* SerializeSlsLz4 of p (a "processor_parse_delimiter_native" or a "processor_parse_regex_native") on the group
 * described by group_json: the malloc'd LZ4 block and its length, *raw_len_out = the size of the wire bytes it
 * decompresses to; or NULL + *err_out = the serializer's error message; NULL + *fail_out on an engine failure or a bad
 * group. */
char* lc_host_processor_serialize_sls_lz4(lc_host_processor_t* p, const char* group_json, int enable_ns,
                                          unsigned long long* len_out, unsigned long long* raw_len_out, char** err_out,
                                          char** fail_out);

/* The delimiter -> regex, split -> regex or split -> delimiter chain of a pipeline on the group described by
 * group_json: delim (a "processor_parse_delimiter_native", "processor_split_string_native" or
 * "processor_split_multiline_log_string_native") followed by regex (a "processor_parse_regex_native" reading one of
 * delim's keys, or the splitter's SourceKey; behind a splitter, also a "processor_parse_delimiter_native", a
 * "processor_parse_json_native" or a "processor_parse_apsara_native" reading its SourceKey).  mode 0: delim's
 * SerializeSls(group, regex); mode 1: Process + Process + SLSEventGroupSerializer::Serialize on the same in-memory group (the result mode 0 must equal byte for byte); mode 2:
 * SerializeSlsLz4(group, regex), the LZ4 block with *raw_len_out = the size it decompresses to.  Returns the malloc'd
 * bytes and their length, or NULL + *err_out = the serializer's error message; NULL + *fail_out on an engine failure or
 * a bad group. */
char* lc_host_chain_serialize_sls(lc_host_processor_t* delim, lc_host_processor_t* regex, const char* group_json,
                                  int enable_ns, int mode, unsigned long long* len_out, unsigned long long* raw_len_out,
                                  char** err_out, char** fail_out);

/* The split -> regex -> filter chain on the group described by group_json: split (either splitter), then regex (a
 * "processor_parse_regex_native" reading the splitter's SourceKey), then filter (a "processor_filter_regex_native").
 * mode 0: split's SerializeSls(group, regex, filter); mode 1: Process x 3 + SLSEventGroupSerializer::Serialize on the
 * same in-memory group; mode 2: SerializeSlsLz4(group, regex, filter).  Returns as lc_host_chain_serialize_sls.
 * The split -> delimiter -> regex chain goes through the same call: regex is then a
 * "processor_parse_delimiter_native" reading the splitter's SourceKey and filter a "processor_parse_regex_native"
 * reading one of its keys, and modes 0 and 2 are split's SerializeSls / SerializeSlsLz4(group, delimiter, regex).
 * So does the split -> regex -> timestamp chain: filter is then a "processor_parse_timestamp_native", and modes 0 and
 * 2 are split's SerializeSls / SerializeSlsLz4(group, regex, timestamp).  And the split -> JSON -> timestamp chain:
 * regex is then a "processor_parse_json_native" reading the splitter's SourceKey and filter a
 * "processor_parse_timestamp_native", and modes 0 and 2 are split's SerializeSls / SerializeSlsLz4(group, json,
 * timestamp).  Likewise the split -> delimiter -> timestamp chain: regex is then a "processor_parse_delimiter_native"
 * reading the splitter's SourceKey and filter a "processor_parse_timestamp_native", and modes 0 and 2 are split's
 * SerializeSls / SerializeSlsLz4(group, delimiter, timestamp). */
char* lc_host_chain3_serialize_sls(lc_host_processor_t* split, lc_host_processor_t* regex, lc_host_processor_t* filter,
                                   const char* group_json, int enable_ns, int mode, unsigned long long* len_out,
                                   unsigned long long* raw_len_out, char** err_out, char** fail_out);

/* LZ4Compressor::Compress (core/common/compression/LZ4Compressor.cpp:25-44), GPU-backed: the n inputs
 * (data[k], len[k]) in one device call, one LZ4 block each.  Returns the malloc'd blocks back to back, their total
 * length and blk_len[k]; or NULL + *err_out = the compressor's error message ("input size is incorrect") or an engine
 * failure. */
char* lc_host_lz4_compress(const char* const* data, const unsigned long long* len, unsigned long long n,
                           unsigned long long* len_out, unsigned long long* blk_len, char** err_out);

/* ZstdCompressor::Compress (core/common/compression/ZstdCompressor.cpp), GPU-backed, the twin of lc_host_lz4_compress:
 * the n inputs in one device call, one zstd frame each, back to back (frm_len[k]); or NULL + *err_out. */
char* lc_host_zstd_compress(const char* const* data, const unsigned long long* len, unsigned long long n,
                            unsigned long long* len_out, unsigned long long* frm_len, char** err_out);

/* Loads a dynamic plugin the way the agent does (dlopen, dlsym("processor_interface"), version == 100 --
 * PluginRegistry.cpp:255-275) and drives it like DynamicCProcessorProxy (.cpp:21-36): init(ins, &config, &context),
 * process(plugin_state, &group), finalize(plugin_state).  Returns the processed group's JSON ("null" when group_json
 * is NULL: init / finalize only); NULL + *err_out on any failure.  *version_out / *name_out (malloc'd) report the
 * interface fields as soon as the symbol resolves. */
char* lc_host_dynamic_plugin_roundtrip(const char* so_path, const char* config_json, const char* group_json,
                                       int enable_event_meta, int* version_out, char** name_out, char** err_out);

/* Makes every SourceBuffer chunk created from now on pinned (lc_host_alloc): a group's arena is then DMA-able in
 * place -- the integration's replacement of SourceBuffer's `new char[]` (core/common/memory/SourceBuffer.h:98-131). */
void lc_host_use_pinned_arenas(int on);

/* End-to-end run at the plugin boundary (bench.py's `e2e`).  Builds event groups of <= group_bytes from the line
 * table (one arena chunk per group, one LogEvent {"content": line} per line: the state the reader + split processor
 * leave, LogFileReader.cpp:97) and times `reps` repetitions of
 *   mode 0: ProcessorInstance::Process with ONE group per call (a ProcessorRunner thread popping groups),
 *   mode 1: ProcessorInstance::Process(std::vector<PipelineEventGroup>&) with ALL groups (batched override).
 * data[line_off[i] + line_len[i]] must be readable (the separator byte travels with the line).  Groups are rebuilt,
 * untimed, before every repetition.  seconds_out[reps] = wall time of the Process calls of each repetition.
 * stats_out[12] = groups, in events, out events, live contents, content checksum (sum of key.size*131 +
 * value.size*31 + first value byte), arena bytes, then ProcessorInstance's counters: in events, out events, in
 * bytes, out bytes, process ns, process ms, then the plugin's own phase timers (gather ns, engine-call ns, epilogue ns;
 * 0 when it has none), one spare -- all summed over the repetitions.  Returns 0, or 1 + *err_out. */
int lc_host_bench_plugin(const char* type, const char* config_json, const uint8_t* data, const uint32_t* line_off,
                         const uint32_t* line_len, uint64_t n_lines, uint32_t group_bytes, int mode, int reps,
                         double* seconds_out, uint64_t stats_out[16], char** err_out);

#ifdef __cplusplus
}
#endif
#endif
