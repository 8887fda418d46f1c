// Processors.h -- GPU-backed replacements of LoongCollector's four native log-parsing processors behind the
// reference's own plugin API: same class names, Init(const Json::Value&) parameters, Process(PipelineEventGroup&)
// side effects and counters.  The per-byte work (newline scan, regex automata, delimiter FSM) happens on the
// GPU through include/lc_b200.h; this file keeps only the host-side policy that needs the event object graph.
//   Processor interface ............ core/collection_pipeline/plugin/interface/Processor.h:27-37
//   CommonParserOptions ............ core/plugin/processor/CommonParserOptions.cpp:28-117
//   MultilineOptions ............... core/file_server/MultilineOptions.cpp:22-222
//   processors ..................... core/plugin/processor/{ProcessorParseRegexNative,ProcessorParseDelimiterNative}.cpp,
//                                    core/plugin/processor/inner/{ProcessorSplitLogStringNative,ProcessorSplitMultilineLogStringNative}.cpp
#pragma once
#include <atomic>
#include <chrono>
#include <memory>
#include <string>
#include <vector>

#include "../../include/lc_b200.h"
#include "Models.h"

namespace logtail {

struct ThreadScratch; // pinned per-thread tables of the batched paths (Processors.cpp)

// Process() runs concurrently on the same instance from every ProcessorRunner thread (ProcessorRunner.cpp:48-53):
// counters are atomic like the reference's (monitor/metric_models/MetricTypes.h, relaxed adds).
struct Counter {
    std::atomic<uint64_t> v{0};
    uint64_t GetValue() const { return v.load(std::memory_order_relaxed); }
    void Add(uint64_t d) { v.fetch_add(d, std::memory_order_relaxed); }
};

class Processor {
public:
    virtual ~Processor() = default;
    virtual const std::string& Name() const = 0;
    virtual bool Init(const Json::Value& config) = 0;
    virtual void Process(std::vector<PipelineEventGroup>& groups) {
        for (auto& g : groups)
            Process(g);
    }
    virtual void Process(PipelineEventGroup& group) = 0;
    const std::string& LastError() const { return mError; }
    // The reference's Process never throws (per-event failure = counters + policy): an engine failure (CUDA error,
    // out of memory) leaves the affected groups untouched, is counted here and its text kept in LastError().
    uint64_t EngineErrors() const { return mEngineErrors.GetValue(); }
    // name -> value of every counter the reference registers for this plugin
    virtual std::vector<std::pair<std::string, uint64_t>> Counters() const { return {}; }

protected:
    virtual bool IsSupportedEvent(const PipelineEventPtr& e) const = 0;
    bool Fail(const std::string& msg) {
        mError = msg;
        return false;
    }
    void EngineFailed(const char* what) {
        mEngineErrors.Add(1);
        mError = what;
    }
    std::string mError;
    Counter mEngineErrors;
};

// ProcessorInstance (core/collection_pipeline/plugin/instance/ProcessorInstance.cpp:29-63): the wrapper the pipeline
// calls -- in / out event and byte counters (two DataSize() sweeps per call) and the wall time spent in the plugin.
class ProcessorInstance {
public:
    explicit ProcessorInstance(Processor* plugin) : mPlugin(plugin) {}
    const std::string& Name() const { return mPlugin->Name(); }
    Processor* GetPlugin() { return mPlugin.get(); }
    bool Init(const Json::Value& config) { return mPlugin->Init(config); }
    void Process(std::vector<PipelineEventGroup>& eventGroupList);
    Counter mInEventsTotal, mOutEventsTotal, mInSizeBytes, mOutSizeBytes, mTotalProcessTimeMs;
    // finer-grained than the reference's millisecond counter (kept in addition to it)
    Counter mTotalProcessTimeNs;

private:
    std::unique_ptr<Processor> mPlugin;
};

struct CommonParserOptions {
    bool mKeepingSourceWhenParseFail = false;
    bool mKeepingSourceWhenParseSucceed = false;
    std::string mRenamedSourceKey;
    bool mCopingRawLog = false;
    static const std::string legacyUnmatchedRawLogKey;
    bool Init(const Json::Value& config);
    bool ShouldAddSourceContent(bool parseSuccess) const;
    bool ShouldAddLegacyUnmatchedRawLog(bool parseSuccess) const;
    bool ShouldEraseEvent(bool parseSuccess, const LogEvent& sourceEvent, const GroupMetadata& metadata) const;
};

struct MultilineOptions {
    enum class UnmatchedContentTreatment { DISCARD, SINGLE_LINE };
    std::string mStartPattern, mContinuePattern, mEndPattern;
    UnmatchedContentTreatment mUnmatchedContentTreatment = UnmatchedContentTreatment::SINGLE_LINE;
    bool mIgnoringUnmatchWarning = false;
    bool mIsMultiline = false;
    bool Init(const Json::Value& config, std::string& err);
};

class CompiledRegex {
public:
    CompiledRegex() = default;
    ~CompiledRegex();
    CompiledRegex(const CompiledRegex&) = delete;
    CompiledRegex& operator=(const CompiledRegex&) = delete;
    bool Compile(const std::string& pattern, std::string& err);
    lc_regex_t* get() const { return mRe; }
    uint32_t groups() const { return mRe ? lc_regex_ngroups(mRe) : 0; }

private:
    lc_regex_t* mRe = nullptr;
};

class ProcessorParseRegexNative;
class ProcessorParseDelimiterNative;
class ProcessorFilterNative;
class ProcessorParseTimestampNative;
class ProcessorParseApsaraNative;
class ProcessorParseJsonNative;

class ProcessorSplitLogStringNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void ProcessImpl(PipelineEventGroup& group);
    using Processor::Process;
    std::string mSourceKey = "content";
    char mSplitChar = '\n';
    bool mEnableRawContent = false;
    // SLSEventGroupSerializer::Serialize after Process(group): the same bytes or error message and the same counters.
    // A group whose events are all LogEvents {SourceKey -> value} is split and serialised on the device, one source
    // event per call, and only the wire bytes come back; any other group runs Process + Serialize.
    bool SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out, std::string& err);
    // Process(group), then next.Process(group) (next: the regex processor behind this one, reading SourceKey), then
    // SLSEventGroupSerializer::Serialize: the same bytes or error message, and the same counter updates on both
    // processors.  On a flat group without EnableRawContent, whose regex SourceKey is this SourceKey and whose
    // configuration lc_split_regex_parse_sls accepts, each source event is split, parsed and serialised in one device
    // pass (log.file.offset metadata included) and only the wire bytes come back; the group's events are left as they
    // were.  Otherwise the three calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& out,
                      std::string& err);
    // The same followed by LZ4Compressor::Compress.  A device-path group of one source event is compressed on the
    // device (lc_split_regex_parse_sls_lz4); other groups compress SerializeSls's bytes.
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // Process(group), next.Process(group), filter.Process(group) (filter: the processor_filter_regex_native behind
    // next), then SLSEventGroupSerializer::Serialize: the same bytes or error message, and the same counter updates.
    // The device path (lc_split_regex_filter_parse_sls[_lz4]) applies under SerializeSls(group, next)'s conditions when
    // filter.DeviceFilter accepts the rule; otherwise the four calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative& filter,
                      bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative& filter,
                         bool enableNs, std::string& block, uint64_t& rawSize, std::string& err);
    // Process(group), then next.Process(group) (next: the delimiter processor behind this one, reading SourceKey), then
    // SLSEventGroupSerializer::Serialize: the same bytes or error message, and the same counter updates on both
    // processors.  On a flat group without EnableRawContent, whose delimiter SourceKey is this SourceKey and whose
    // configuration lc_split_delim_parse_sls accepts, each source event is split, parsed and serialised in one device
    // pass (log.file.offset metadata included) and only the wire bytes come back; the group's events are left as they
    // were.  Otherwise the three calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs, std::string& out,
                      std::string& err);
    // The same followed by LZ4Compressor::Compress.  A device-path group of one source event is compressed on the
    // device (lc_split_delim_parse_sls_lz4); other groups compress SerializeSls's bytes.
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs,
                         std::string& block, uint64_t& rawSize, std::string& err);
    // The split -> delimiter -> regex chain: Process(group), next.Process(group), regex.Process(group) (regex reading
    // one of next's keys), then SLSEventGroupSerializer::Serialize: the same bytes or error message, and the same
    // counter updates on all three processors.  On a flat group without EnableRawContent, whose delimiter SourceKey is
    // this SourceKey, whose regex SourceKey is one of the delimiter's keys and whose configuration
    // lc_split_delim_regex_parse_sls accepts, each source event is split, parsed by both stages and serialised in one
    // device pass (log.file.offset metadata included) and only the wire bytes come back; the group's events are left as
    // they were.  Otherwise the four calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, ProcessorParseRegexNative& regex,
                      bool enableNs, std::string& out, std::string& err);
    // The same followed by LZ4Compressor::Compress.  A device-path group of one source event is compressed on the
    // device (lc_split_delim_regex_parse_sls_lz4); other groups compress SerializeSls's bytes.
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                         ProcessorParseRegexNative& regex, bool enableNs, std::string& block, uint64_t& rawSize,
                         std::string& err);
    // The split -> regex -> timestamp chain: Process(group), next.Process(group), timestamp.Process(group)
    // (timestamp: the processor_parse_timestamp_native behind next), then SLSEventGroupSerializer::Serialize: the
    // same bytes or error message, and the same counter updates on all three processors.  The device path
    // (lc_split_regex_timestamp_parse_sls[_lz4]) applies under SerializeSls(group, next)'s conditions when the group
    // holds exactly one source event (the reader's shape: the second-level cache then never has to carry across
    // calls) and the chain accepts timestamp's SourceKey; "now" is read once per call.  Otherwise the four calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);

    // The split -> JSON chain: Process(group), then next.Process(group) (next: the processor_parse_json_native behind
    // this one, reading SourceKey), then SLSEventGroupSerializer::Serialize: the same bytes or error message, and the
    // same counter updates on both processors.  On a flat group without EnableRawContent, whose JSON SourceKey is this
    // SourceKey and whose configuration lc_split_json_parse_sls accepts, each source event is split, parsed and
    // serialised in one device pass (log.file.offset metadata included) and only the wire bytes come back; the
    // group's events are left as they were.  Otherwise the three calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& out,
                      std::string& err);
    // The same followed by LZ4Compressor::Compress.  A device-path group of one source event is compressed on the
    // device (lc_split_json_parse_sls_lz4); other groups compress SerializeSls's bytes.
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // The split -> Apsara chain: Process(group), then next.Process(group) (next: the processor_parse_apsara_native
    // behind this one, reading SourceKey), then SLSEventGroupSerializer::Serialize: the same bytes or error message, and
    // the same counter updates on both processors.  On a flat group of ONE source event without EnableRawContent (a
    // reader chunk: the time cache runs over the whole group), whose Apsara SourceKey is this SourceKey and whose
    // configuration lc_split_apsara_parse_sls accepts, the event is split, parsed and serialised in one device pass
    // (log.file.offset metadata included; now = time(NULL), the history discard as next has it) and only the wire
    // bytes come back; the group's events are left as they were.  Otherwise the three calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs, std::string& out,
                      std::string& err);
    // The same followed by LZ4Compressor::Compress; a device-path group is compressed on the device
    // (lc_split_apsara_parse_sls_lz4).
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs,
                         std::string& block, uint64_t& rawSize, std::string& err);
    // The split -> JSON -> timestamp chain: Process(group), next.Process(group), timestamp.Process(group)
    // (timestamp: the processor_parse_timestamp_native behind next), then SLSEventGroupSerializer::Serialize: the
    // same bytes or error message, and the same counter updates on all three processors.  The device path
    // (lc_split_json_timestamp_parse_sls[_lz4]) applies under SerializeSls(group, next)'s conditions when the group
    // holds exactly one source event (the reader's shape: the second-level cache then spans the group) and the chain
    // accepts timestamp's SourceKey; "now" is read once per call.  Otherwise the four calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // The split -> delimiter -> timestamp chain: Process(group), next.Process(group), timestamp.Process(group)
    // (timestamp: the processor_parse_timestamp_native behind next), then SLSEventGroupSerializer::Serialize: the
    // same bytes or error message, and the same counter updates on all three processors.  The device path
    // (lc_split_delim_timestamp_parse_sls[_lz4]) applies under SerializeSls(group, next)'s conditions when the group
    // holds exactly one source event (the reader's shape: the second-level cache then spans the group) and the chain
    // accepts timestamp's SourceKey; "now" is read once per call.  Otherwise the four calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs,
                           std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative* filter,
                           bool enableNs, std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs,
                           std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                           ProcessorParseRegexNative& regex, bool enableNs, std::string& out, uint64_t* rawSize,
                           std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
};

class ProcessorSplitMultilineLogStringNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void ProcessImpl(PipelineEventGroup& group);
    using Processor::Process;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey = "content";
    MultilineOptions mMultiline;
    bool mEnableRawContent = false;
    // SLSEventGroupSerializer::Serialize after Process(group): the same bytes or error message and the same counters.
    // A group whose events are all LogEvents {SourceKey -> value} is split and serialised on the device, one source
    // event per call, and only the wire bytes come back; any other group runs Process + Serialize.
    bool SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out, std::string& err);
    // The split -> regex chain, as ProcessorSplitLogStringNative's (lc_multiline_split_regex_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& out,
                      std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // The split -> regex -> filter chain, as ProcessorSplitLogStringNative's
    // (lc_multiline_split_regex_filter_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative& filter,
                      bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative& filter,
                         bool enableNs, std::string& block, uint64_t& rawSize, std::string& err);
    // The split -> delimiter chain, as ProcessorSplitLogStringNative's (lc_multiline_split_delim_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs, std::string& out,
                      std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs,
                         std::string& block, uint64_t& rawSize, std::string& err);
    // The split -> delimiter -> regex chain, as ProcessorSplitLogStringNative's
    // (lc_multiline_split_delim_regex_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, ProcessorParseRegexNative& regex,
                      bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                         ProcessorParseRegexNative& regex, bool enableNs, std::string& block, uint64_t& rawSize,
                         std::string& err);
    // The split -> regex -> timestamp chain, as ProcessorSplitLogStringNative's
    // (lc_multiline_split_regex_timestamp_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    Counter mMatchedEventsTotal, mMatchedLinesTotal, mUnmatchedLinesTotal;

    // The split -> JSON chain, as ProcessorSplitLogStringNative's (lc_multiline_split_json_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& out,
                      std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // The split -> Apsara chain, as ProcessorSplitLogStringNative's (lc_multiline_split_apsara_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs, std::string& out,
                      std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs,
                         std::string& block, uint64_t& rawSize, std::string& err);
    // The split -> JSON -> timestamp chain, as ProcessorSplitLogStringNative's
    // (lc_multiline_split_json_timestamp_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
    // The split -> delimiter -> timestamp chain, as ProcessorSplitLogStringNative's
    // (lc_multiline_split_delim_timestamp_parse_sls[_lz4]).
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                      ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out, std::string& err);
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                         ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);
protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next, bool enableNs,
                           std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, ProcessorFilterNative* filter,
                           bool enableNs, std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next, bool enableNs,
                           std::string& out, uint64_t* rawSize, std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                           ProcessorParseRegexNative& regex, bool enableNs, std::string& out, uint64_t* rawSize,
                           std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                           ProcessorParseTimestampNative& timestamp, bool enableNs, std::string& out,
                           uint64_t* rawSize, std::string& err);
    CompiledRegex mStart, mContinue, mEnd;
};

class ProcessorParseRegexNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    // Batched override of Processor.h:31: the arenas of all groups are packed into one device arena and parsed by
    // one launch sequence (lc_regex_parse_packed); gather and per-event epilogue run on a few host threads.
    void Process(std::vector<PipelineEventGroup>& groups) override;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey, mRegex;
    std::vector<std::string> mKeys;
    CommonParserOptions mCommonParserOptions;
    Counter mDiscardedEventsTotal, mOutFailedEventsTotal, mOutKeyNotFoundEventsTotal, mOutSuccessfulEventsTotal;
    // Process(group) followed by SLSEventGroupSerializer::Serialize (enableNs = its mEnableTimestampNanosecond): the
    // same bytes or error message, and the same counter updates.  When every event is flat (a LogEvent whose only
    // content is SourceKey -> line) and the group carries no log.file.offset metadata, the group is parsed and
    // serialised in one device pass (lc_regex_parse_sls): the capture tables never leave the GPU, no LogEvent is
    // touched and the group's events are left as they were.  Otherwise Process runs.
    bool SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out, std::string& err);
    // SerializeSls followed by LZ4Compressor::Compress: on success `block` is one LZ4 block that decompresses to exactly
    // SerializeSls's bytes, and rawSize is their size.  Errors and counters are SerializeSls's.  The one-pass path
    // compresses on the device (lc_regex_parse_sls_lz4): only the block comes back.
    bool SerializeSlsLz4(PipelineEventGroup& group, bool enableNs, std::string& block, uint64_t& rawSize,
                         std::string& err);

private:
    bool SerializeSlsImpl(PipelineEventGroup& group, bool enableNs, std::string& out, uint64_t* rawSize,
                          std::string& err);

public:

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    struct EventResult {
        uint8_t status;
        const uint32_t* capOff; // row of the capture tables (offsets relative to `origin - originOff`)
        const uint32_t* capLen;
        const char* origin;     // first byte of the source value
        uint32_t originOff;     // its offset in the table's coordinate system
    };
    struct LocalCounters {
        uint64_t discarded = 0, failed = 0, keyNotFound = 0, successful = 0;
    };
    // ProcessEvent epilogue (:135-167) of one event; returns false when the event is to be erased
    bool FinishEvent(PipelineEventGroup& group, PipelineEventPtr& e, const LogEvent::Content* src, const EventResult* r,
                     LocalCounters& c) const;
    void ProcessBatch(PipelineEventGroup* groups, size_t ngroups);
    void EpilogueGroup(PipelineEventGroup& group, uint64_t firstEv, const struct ThreadScratch& sc, uint32_t G,
                       LocalCounters& c) const;
    void AddCounters(const LocalCounters& c);
    friend class ProcessorParseDelimiterNative; // the delimiter -> regex chain's SerializeSls
    friend struct SplitRegexStage;              // the split -> regex chain's
    friend struct SplitDelimRegexStage;         // the split -> delimiter -> regex chain's
    bool mSourceKeyOverwritten = false;
    bool mIsWholeLineMode = false;
    bool mKeysDistinct = false; // no key repeats: an event that holds only the source key takes the parsed fields as
                                // plain appends (AppendContentNoCopy) instead of one look-up per key
    CompiledRegex mReg;

public:
    // wall time of the three phases of the batched path, summed over calls (ns): gather, engine call, epilogue
    Counter mGatherNs, mEngineNs, mEpilogueNs;
};

class ProcessorParseDelimiterNative : public Processor {
public:
    enum class OverflowedFieldsTreatment { EXTEND, KEEP, DISCARD };
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void ProcessImpl(PipelineEventGroup& group);
    using Processor::Process;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey, mSeparator;
    char mQuote = '"';
    std::vector<std::string> mKeys;
    bool mAllowingShortenedFields = true;
    OverflowedFieldsTreatment mOverflowedFieldsTreatment = OverflowedFieldsTreatment::EXTEND;
    bool mExtractingPartialFields = false;
    CommonParserOptions mCommonParserOptions;
    Counter mDiscardedEventsTotal, mOutFailedEventsTotal, mOutKeyNotFoundEventsTotal, mOutSuccessfulEventsTotal;
    // Process(group) followed by SLSEventGroupSerializer::Serialize (enableNs = its mEnableTimestampNanosecond): the
    // same bytes or error message, and the same counter updates.  When every event is flat (a LogEvent whose only
    // content is SourceKey -> line), the group carries no log.file.offset metadata and the configuration is one
    // lc_delim_parse_sls accepts, the group is parsed and serialised in one device pass (lc_delim_parse_sls): the
    // delimiter tables never leave the GPU and the group's events are left as they were.  Otherwise Process runs.
    bool SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out, std::string& err);
    // SerializeSls followed by LZ4Compressor::Compress, as for ProcessorParseRegexNative (lc_delim_parse_sls_lz4).
    bool SerializeSlsLz4(PipelineEventGroup& group, bool enableNs, std::string& block, uint64_t& rawSize,
                         std::string& err);
    // Process(group), then next.Process(group) (next: the regex processor behind this one in the pipeline, parsing one
    // of this processor's keys), then SLSEventGroupSerializer::Serialize: the same bytes or error message, and the same
    // counter updates on both processors.  On a flat group without log.file.offset metadata and a chain
    // lc_delim_regex_parse_sls accepts, both stages run in one device pass and only the wire bytes come back; the
    // group's events are left as they were.  Otherwise the three calls run.
    bool SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& out,
                      std::string& err);
    // The same followed by LZ4Compressor::Compress, as SerializeSlsLz4 (lc_delim_regex_parse_sls_lz4).
    bool SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs, std::string& block,
                         uint64_t& rawSize, std::string& err);

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    bool SerializeSlsImpl(PipelineEventGroup& group, bool enableNs, std::string& out, uint64_t* rawSize,
                          std::string& err);
    bool ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next, bool enableNs,
                           std::string& out, uint64_t* rawSize, std::string& err);
    friend struct SplitDelimStage;      // the split -> delimiter chain's SerializeSls
    friend struct SplitDelimRegexStage; // the split -> delimiter -> regex chain's
    bool mSourceKeyOverwritten = false;
    bool mDeviceSls = false; // the configuration passes lc_delim_parse_sls's checks
};

// First "next" row (SURVEY.md 8f): regex include / exclude filter.  Every regex leaf of the rule / expression is
// evaluated for the whole group with one batched boolean regex_match on the GPU; the and/or/not tree and the
// non-UTF8 blanking stay on the host.  core/plugin/processor/ProcessorFilterNative.cpp:30-275,380-488
// processor_parse_timestamp_native (ProcessorParseTimestampNative.cpp:30-235): the groups of one call go to the device
// in one lc_timestamp_parse call (the full parse and the second-level cache run there, the cache starting empty in
// every group); the host sets the times, erases the discarded events (rIdx / wIdx) and adds the counters.
// Init also fails where the device program refuses SourceFormat (%c, %x, %X: LastError() says so); there is no CPU
// fallback.  "now" is read once per call, where the reference calls time(NULL) per event.
class ProcessorParseTimestampNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    ~ProcessorParseTimestampNative() override { lc_timestamp_free(mProgram); }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void Process(std::vector<PipelineEventGroup>& groups) override;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey, mSourceFormat, mSourceTimezone;
    int32_t mSourceYear = -1;
    int32_t mLogTimeZoneOffsetSecond = 0;
    // ilogtail_discard_old_data (on by default; off for one-time pipelines) and ilogtail_discard_interval
    bool mDiscardOldData = true;
    int32_t mDiscardInterval = 43200;
    std::vector<std::string> mWarnings; // the reference's PARAM_WARNING_* messages of the last Init
    Counter mDiscardedEventsTotal, mOutFailedEventsTotal, mOutKeyNotFoundEventsTotal, mOutSuccessfulEventsTotal,
        mHistoryFailureTotal;

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    friend struct SplitRegexTsStage; // the split -> regex -> timestamp chain's SerializeSls
    friend struct SplitJsonTsStage;  // the split -> JSON -> timestamp chain's
    friend struct SplitDelimTsStage; // the split -> delimiter -> timestamp chain's
    lc_timestamp_t* mProgram = nullptr;
};

// processor_parse_apsara_native (ProcessorParseApsaraNative.cpp:37-473): the groups of one call go to the device in
// one lc_apsara_parse call (the time parse, the time cache, the base and key:value field scans run there, the cache
// starting empty in every group); the host appends the entries and "microtime" (AppendContentNoCopy, no
// de-duplication), applies CommonParserOptions, erases events and adds the counters.  "now" is read once per call,
// where the reference calls time(NULL) per event.
class ProcessorParseApsaraNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    ~ProcessorParseApsaraNative() override { lc_apsara_free(mProgram); }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void Process(std::vector<PipelineEventGroup>& groups) override;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey, mTimezone;
    int32_t mLogTimeZoneOffsetSecond = 0;
    CommonParserOptions mCommonParserOptions;
    // ilogtail_discard_old_data (on by default; off for one-time pipelines) and ilogtail_discard_interval
    bool mDiscardOldData = true;
    int32_t mDiscardInterval = 43200;
    std::vector<std::string> mWarnings; // the reference's PARAM_WARNING_* messages of the last Init
    Counter mDiscardedEventsTotal, mOutFailedEventsTotal, mOutKeyNotFoundEventsTotal, mOutSuccessfulEventsTotal,
        mHistoryFailureTotal;

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    lc_apsara_t* mProgram = nullptr;
    friend struct SplitApsaraStage; // the split -> Apsara chain's SerializeSls
};

// processor_parse_json_native (ProcessorParseJsonNative.cpp: ProcessEvent, JsonLogLineParserSimdJson): the groups of
// one call go to the device in one lc_json_parse call (cut where the values or the arena would reach 2 GiB);
// the validation and the rendering of every member run there.  The host applies the members with overwrite
// (SetContentNoCopy, as AddLog(key, value, event) does), copies the arena bytes into the group's SourceBuffer,
// applies CommonParserOptions, erases events and adds the counters.
class ProcessorParseJsonNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    ~ProcessorParseJsonNative() override { lc_json_free(mProgram); }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void Process(std::vector<PipelineEventGroup>& groups) override;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey;
    CommonParserOptions mCommonParserOptions;
    Counter mDiscardedEventsTotal, mOutFailedEventsTotal, mOutKeyNotFoundEventsTotal, mOutSuccessfulEventsTotal;

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    void ProcessBatch(std::vector<PipelineEventGroup>& groups, size_t g0, size_t g1);
    lc_json_t* mProgram = nullptr;
    friend struct SplitJsonStage; // the split -> JSON chain's SerializeSls
};

class ProcessorFilterNative : public Processor {
public:
    static const std::string sName;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void ProcessImpl(PipelineEventGroup& group);
    using Processor::Process;
    bool mDiscardingNonUTF8 = false;
    ~ProcessorFilterNative() override;
    // The rule as the split -> regex -> filter device calls take it: RULE and Include mode the leaves ANDed in their
    // evaluation order, EXPRESSION mode the postfix program of the tree, BYPASS the empty program.  *d points into
    // this object.  False when the device calls cannot reproduce the rule: DiscardingNonUTF8, more leaves or program
    // entries than lc_b200.h allows, or a stack deeper than 32.
    bool DeviceFilter(lc_filter_desc_t* d) const;

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    enum class Mode { BYPASS_MODE, EXPRESSION_MODE, RULE_MODE };
    struct Leaf {
        std::string key;
        CompiledRegex* reg;
    };
    struct Node { // expression tree; leaf >= 0 indexes mLeaves
        int op = 0; // 0 leaf, 1 not, 2 and, 3 or
        int leaf = -1;
        int left = -1, right = -1;
    };
    int ParseExpression(const Json::Value& v, std::string& err);
    bool Eval(int node, const std::vector<std::vector<uint8_t>>& leafResult, size_t ev) const;
    Mode mFilterMode = Mode::BYPASS_MODE;
    std::vector<Leaf> mLeaves;
    std::vector<Node> mNodes;
    int mRoot = -1;
    // DeviceFilter's description, built by Init
    void BuildDeviceFilter();
    bool mDeviceOk = false;
    std::vector<const char*> mDevKeys;
    std::vector<uint32_t> mDevKeyLens;
    std::vector<const lc_regex_t*> mDevRegs;
    std::vector<uint32_t> mDevProg;
};

// Second "next" row (SURVEY.md 8f): merges already-split LogEvents of a group back into records -- by the docker
// partial-log flag or by start / continue / end patterns.  The anchored prefix probes of every event are evaluated for
// the whole group with one batched lc_regex_prefix_match per pattern; the sequential merge walk (which needs the
// event objects and joins the values in place in the arena) stays on the host.
// core/plugin/processor/inner/ProcessorMergeMultilineLogNative.cpp:33-420
class ProcessorMergeMultilineLogNative : public Processor {
public:
    enum class MergeType { BY_REGEX, BY_FLAG };
    static const std::string sName;
    static const std::string PartLogFlag;
    const std::string& Name() const override { return sName; }
    bool Init(const Json::Value& config) override;
    void Process(PipelineEventGroup& group) override;
    void ProcessImpl(PipelineEventGroup& group);
    using Processor::Process;
    std::vector<std::pair<std::string, uint64_t>> Counters() const override;
    std::string mSourceKey = "content";
    MergeType mMergeType = MergeType::BY_REGEX;
    MultilineOptions mMultiline;
    Counter mMergedEventsTotal, mUnmatchedEventsTotal;

protected:
    bool IsSupportedEvent(const PipelineEventPtr& e) const override { return e.Is<LogEvent>(); }

private:
    void MergeLogsByFlag(PipelineEventGroup& group);
    void MergeLogsByRegex(PipelineEventGroup& group);
    void MergeEvents(PipelineEventGroup& group, std::vector<LogEvent*>& logEvents, bool insertLineBreak);
    void HandleUnmatchLogs(EventsContainer& logEvents, size_t& newSize, size_t begin, size_t end);
    // the *RegPtr members of MultilineOptions (MultilineOptions.cpp:125-160,196-215): compiled from the pattern
    // with its trailing '$' / ".*" removed; unset when that is empty or dropped by the combination rules
    CompiledRegex mStartReg, mContinueReg, mEndReg;
    bool mHasStart = false, mHasContinue = false, mHasEnd = false;
};

// Fourth "next" row (SURVEY.md 8f): the SLS wire format of a group of LOG events.  Mirrors
// SLSEventGroupSerializer::Serialize (core/collection_pipeline/serializer/SLSSerializer.cpp:162-252): the `Logs`
// fields -- all the bytes that scale with the data -- are written on the GPU straight from the arena spans of the
// events' contents (lc_sls_serialize_logs); Topic / Source / MachineUUID / LogTags are appended here.
class SLSEventGroupSerializer {
public:
    bool mEnableTimestampNanosecond = false;      // GlobalConfig::mEnableTimestampNanosecond
    int32_t mMaxSendLogGroupSize = 10 * 1024 * 1024; // flag max_send_log_group_size (FlusherSLS.cpp:61)
    bool Serialize(PipelineEventGroup& group, std::string& res, std::string& errorMsg) const;
};

// FlusherSLS's default compressor (core/common/compression/LZ4Compressor.cpp:25-44) on the GPU: one LZ4 block per
// input (lc_lz4_compress).  The blocks are valid LZ4 blocks of the input, not liblz4's exact bytes.  The batched
// overload compresses many serialised groups in one device call, as the flusher holds many queue items
// (FlusherSLS.cpp:1065-1144); a lone small group is faster through liblz4 on the CPU (DESIGN.md §5), so callers with
// one group at a time should batch them.
class LZ4Compressor {
public:
    bool Compress(const std::string& input, std::string& output, std::string& errorMsg);
    bool Compress(const std::vector<std::string>& inputs, std::vector<std::string>& outputs, std::string& errorMsg);
};

// core/common/compression/CompressType.h
enum class CompressType { NONE, LZ4, ZSTD };

// FlusherSLS's other compressor, CompressType "zstd" (core/common/compression/ZstdCompressor.cpp: ZSTD_compress at
// the configured level) on the GPU: one zstd frame per input (lc_zstd_compress).  The frames are valid zstd frames of
// the input, not libzstd's exact bytes.  The level is accepted for the reference's constructor and does not change the
// bytes: there is one device encoder, whose ratio lies between libzstd's levels -1 and 1 (DESIGN.md §5).  As for
// LZ4Compressor, the batched overload compresses many serialised groups in one device call.
class ZstdCompressor {
public:
    explicit ZstdCompressor(CompressType type, int32_t level = 1) : mType(type), mCompressionLevel(level) {}
    bool Compress(const std::string& input, std::string& output, std::string& errorMsg);
    bool Compress(const std::vector<std::string>& inputs, std::vector<std::string>& outputs, std::string& errorMsg);
    CompressType GetCompressType() const { return mType; }

private:
    CompressType mType;
    int32_t mCompressionLevel;
};

// Factory by plugin type name (the names the reference registers, PluginRegistry.cpp:183-200).
Processor* CreateProcessor(const std::string& type);

} // namespace logtail
