#include "Processors.h"

#include "../csrc/lc_exec.cuh" // lc_delim_sls_setup: the configuration checks of lc_delim_parse_sls

#include <stdlib.h>
#include <string.h>

#include <sched.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <stdexcept>
#include <thread>

namespace logtail {

// ------------------------------------------------------------------------------------------------ engine per thread
namespace {

// One engine per (GPU, host thread): the reference keeps one regex copy per ProcessorRunner thread
// (ProcessorParseRegexNative.cpp:64-67); here the per-thread state is the engine's stream and workspace.
struct ThreadEngine {
    lc_engine_t* e = nullptr;
    ~ThreadEngine() {
        if (e)
            lc_engine_destroy(e);
    }
};

lc_engine_t* Engine() {
    static thread_local ThreadEngine t;
    if (!t.e) {
        const char* d = getenv("LC_B200_DEVICE");
        int dev = d ? atoi(d) : 0;
        if (lc_engine_create(dev, &t.e) != LC_OK)
            throw std::runtime_error(std::string("loongcollector_b200: ") + lc_last_error());
    }
    return t.e;
}

void Check(int rc, const char* what) {
    if (rc != LC_OK)
        throw std::runtime_error(std::string(what) + ": " + lc_last_error());
}

// Grow-only pinned host table (lc_host_alloc): result tables land here by DMA without a staging copy.
template <class T>
struct PinnedVec {
    T* p = nullptr;
    size_t cap = 0;
    ~PinnedVec() { lc_host_free(p); }
    T* ensure(size_t n) {
        if (n > cap) {
            lc_host_free(p);
            cap = n + n / 4 + 64;
            p = static_cast<T*>(lc_host_alloc(cap * sizeof(T)));
            if (!p) {
                cap = 0;
                throw std::runtime_error(std::string("loongcollector_b200: ") + lc_last_error());
            }
        }
        return p;
    }
};

} // namespace

struct ThreadScratch {
    PinnedVec<uint32_t> off, len, capOff, capLen;
    PinnedVec<uint8_t> status, staging;
};

namespace {
ThreadScratch& Scratch() {
    static thread_local ThreadScratch s;
    return s;
}

// Host threads used for the gather / epilogue of a batched Process call (env LC_B200_HOST_THREADS; default: the CPUs of
// the process's affinity mask, at most 64).  The reference spends this work on its process_thread_count ProcessorRunner threads.
unsigned HostThreads() {
    static const unsigned n = [] {
        const char* e = getenv("LC_B200_HOST_THREADS");
        unsigned hw = std::thread::hardware_concurrency();
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof set, &set) == 0 && CPU_COUNT(&set) > 0)
            hw = (unsigned)CPU_COUNT(&set); // the CPUs this process may use (e.g. the GPU's NUMA node)
        unsigned want = e ? (unsigned)atoi(e) : 64u;
        if (want < 1)
            want = 1;
        if (hw && want > hw)
            want = hw;
        return want;
    }();
    return n;
}

// Persistent worker pool: a batched Process call runs several short parallel regions (gather, one epilogue per engine
// chunk), so the threads are created once per process, not per region.  One region at a time; a caller that finds the
// pool busy (another ProcessorRunner thread inside its own batch) simply runs its region on its own thread.
class HostPool {
public:
    using Fn = std::function<void(size_t, size_t, unsigned)>;
    static HostPool& Get() {
        static HostPool p(HostThreads());
        return p;
    }
    unsigned Size() const { return mN; }
    void Run(size_t n, size_t minPerThread, const Fn& fn) {
        unsigned t = mN;
        if (minPerThread && n / minPerThread < t)
            t = (unsigned)std::max<size_t>(1, n / minPerThread);
        std::unique_lock<std::mutex> busy(mBusy, std::try_to_lock);
        if (t <= 1 || !busy.owns_lock()) {
            fn(0, n, 0u);
            return;
        }
        {
            std::lock_guard<std::mutex> lk(mMu);
            mFn = &fn;
            mTotal = n;
            mParts = t;
            mPending = t - 1;
            ++mGen;
        }
        mCv.notify_all();
        fn(0, n / t, 0u);
        std::unique_lock<std::mutex> lk(mMu);
        mDone.wait(lk, [&] { return mPending == 0; });
        mFn = nullptr;
    }

private:
    explicit HostPool(unsigned n) : mN(n ? n : 1) {
        for (unsigned k = 1; k < mN; ++k)
            mThreads.emplace_back([this, k] { Work(k); });
    }
    ~HostPool() {
        {
            std::lock_guard<std::mutex> lk(mMu);
            mStop = true;
            ++mGen;
        }
        mCv.notify_all();
        for (auto& t : mThreads)
            t.join();
    }
    void Work(unsigned k) {
        uint64_t seen = 0;
        for (;;) {
            const Fn* fn;
            size_t total;
            unsigned parts;
            {
                std::unique_lock<std::mutex> lk(mMu);
                mCv.wait(lk, [&] { return mGen != seen; });
                seen = mGen;
                if (mStop)
                    return;
                fn = mFn;
                total = mTotal;
                parts = mParts;
            }
            if (k < parts && fn)
                (*fn)(total * k / parts, total * (k + 1) / parts, k);
            if (k < parts) {
                std::lock_guard<std::mutex> lk(mMu);
                if (--mPending == 0)
                    mDone.notify_one();
            }
        }
    }
    unsigned mN;
    std::vector<std::thread> mThreads;
    std::mutex mMu, mBusy;
    std::condition_variable mCv, mDone;
    const Fn* mFn = nullptr;
    size_t mTotal = 0;
    unsigned mParts = 0, mPending = 0;
    uint64_t mGen = 0;
    bool mStop = false;
};

// fn(begin, end, thread) over [0, n) in contiguous slices
template <class Fn>
void ParallelFor(size_t n, size_t minPerThread, Fn fn) {
    HostPool::Get().Run(n, minPerThread, fn);
}

// Flattens the source values of the events to be parsed into (base, off[], len[]).  If every value lies
// inside ONE arena chunk (the production shape: all lines alias the file read buffer) the span is handed to
// the engine as is; otherwise the values are packed into a staging buffer.
struct FlatBatch {
    std::vector<uint32_t> off, len;
    std::vector<size_t> eventIndex;
    std::vector<const char*> origin; // original data pointer of each value
    const uint8_t* base = nullptr;
    uint64_t baseLen = 0;
    std::vector<uint8_t> packed;

    void Add(size_t idx, StringView v) {
        eventIndex.push_back(idx);
        origin.push_back(v.data());
        len.push_back((uint32_t)v.size());
    }
    void Finish(SourceBuffer& sb) {
        size_t n = origin.size();
        off.resize(n);
        if (!n)
            return;
        const char* lo = origin[0];
        const char* hi = origin[0] + len[0];
        for (size_t i = 1; i < n; ++i) {
            lo = std::min(lo, origin[i]);
            hi = std::max(hi, origin[i] + len[i]);
        }
        size_t chunkSize = 0;
        if ((uint64_t)(hi - lo) < 0xFFFFFFF0ull && sb.ChunkContaining(lo, (size_t)(hi - lo), &chunkSize)) {
            base = reinterpret_cast<const uint8_t*>(lo);
            baseLen = (uint64_t)(hi - lo);
            for (size_t i = 0; i < n; ++i)
                off[i] = (uint32_t)(origin[i] - lo);
            return;
        }
        size_t total = 0;
        for (size_t i = 0; i < n; ++i)
            total += len[i];
        packed.resize(total + 1);
        size_t at = 0;
        for (size_t i = 0; i < n; ++i) {
            off[i] = (uint32_t)at;
            if (len[i])
                memcpy(packed.data() + at, origin[i], len[i]);
            at += len[i];
        }
        base = packed.data();
        baseLen = total;
    }
    // view of [o, o + l) (offsets relative to base) for event i, mapped back onto the original bytes
    StringView View(size_t i, uint32_t o, uint32_t l) const { return StringView(origin[i] + (o - off[i]), l); }
};

bool GetString(const Json::Value& cfg, const char* key, std::string& out) {
    if (cfg.isMember(key) && cfg[key].isString()) {
        out = cfg[key].asString();
        return true;
    }
    return false;
}
void GetBool(const Json::Value& cfg, const char* key, bool& out) {
    if (cfg.isMember(key) && cfg[key].isBool())
        out = cfg[key].asBool();
}

void AddLog(LogEvent& ev, StringView key, StringView value, bool overwritten = true) {
    if (!overwritten && ev.HasContent(key))
        return;
    ev.SetContentNoCopy(key, value);
}

std::string ToString(uint64_t v) {
    return std::to_string(v);
}

// CreateNewEvent of both splitters (ProcessorSplitLogStringNative.cpp:135-157,
// ProcessorSplitMultilineLogStringNative.cpp:311-340)
void EmitSplitEvent(PipelineEventGroup& group, const LogEvent& src, StringView sourceVal, const StringBuffer& sourceKey,
                    StringView content, bool isLast, bool raw, EventsContainer& out) {
    if (raw) {
        auto t = group.CreateRawEvent(true);
        t->SetContentNoCopy(content);
        t->SetTimestamp(src.GetTimestamp(), src.GetTimestampNanosecond());
        out.emplace_back(std::move(t), true, nullptr);
        return;
    }
    auto t = group.CreateLogEvent(true);
    t->SetContentNoCopy(StringView(sourceKey.data, sourceKey.size), content);
    t->SetTimestamp(src.GetTimestamp(), src.GetTimestampNanosecond());
    uint64_t rel = (uint64_t)(content.data() - sourceVal.data());
    uint64_t offset = src.GetPosition().first + rel;
    uint64_t length = isLast ? src.GetPosition().second - rel : content.size() + 1;
    t->SetPosition(offset, length);
    if (group.HasMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY)) {
        StringBuffer offStr = group.GetSourceBuffer()->CopyString(ToString(offset));
        t->SetContentNoCopy(group.GetMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY),
                            StringView(offStr.data, offStr.size));
    }
    out.emplace_back(std::move(t), true, nullptr);
}

} // namespace

// ------------------------------------------------------------------------------------------------ options
const std::string CommonParserOptions::legacyUnmatchedRawLogKey = "__raw_log__";

bool CommonParserOptions::Init(const Json::Value& config) {
    GetBool(config, "KeepingSourceWhenParseFail", mKeepingSourceWhenParseFail);
    GetBool(config, "KeepingSourceWhenParseSucceed", mKeepingSourceWhenParseSucceed);
    GetString(config, "RenamedSourceKey", mRenamedSourceKey);
    if (mRenamedSourceKey.empty())
        mRenamedSourceKey = config["SourceKey"].asString();
    GetBool(config, "CopingRawLog", mCopingRawLog);
    return true;
}
bool CommonParserOptions::ShouldAddSourceContent(bool ok) const {
    return (ok && mKeepingSourceWhenParseSucceed) || (!ok && mKeepingSourceWhenParseFail);
}
bool CommonParserOptions::ShouldAddLegacyUnmatchedRawLog(bool ok) const {
    return !ok && mKeepingSourceWhenParseFail && mCopingRawLog;
}
bool CommonParserOptions::ShouldEraseEvent(bool ok, const LogEvent& ev, const GroupMetadata& md) const {
    if (!ok && !mKeepingSourceWhenParseFail) {
        if (ev.Empty())
            return true;
        size_t size = ev.Size();
        auto offsetKey = md.find(EventGroupMetaKey::LOG_FILE_OFFSET_KEY);
        if (size == 1 && offsetKey != md.end() && ev.FirstLive()->first.first == offsetKey->second)
            return true;
        if (size == 2 && ev.HasContent("_time_") && ev.HasContent("_source_"))
            return true;
    }
    return false;
}

CompiledRegex::~CompiledRegex() {
    if (mRe)
        lc_regex_free(mRe);
}
bool CompiledRegex::Compile(const std::string& pattern, std::string& err) {
    if (mRe) {
        lc_regex_free(mRe);
        mRe = nullptr;
    }
    int rc = lc_regex_compile(pattern.data(), pattern.size(), &mRe);
    if (rc != LC_OK) {
        err = lc_last_error();
        if (mRe) {
            lc_regex_free(mRe);
            mRe = nullptr;
        }
        return false;
    }
    return true;
}

static bool EndsWith(const std::string& s, const char* suf) {
    size_t n = strlen(suf);
    return s.size() >= n && !s.compare(s.size() - n, n, suf);
}

bool MultilineOptions::Init(const Json::Value& config, std::string& err) {
    // dotted parameter names resolve to their last segment (ParamExtractor.cpp:23-29)
    struct {
        const char* key;
        std::string* dst;
    } pats[] = {{"StartPattern", &mStartPattern}, {"ContinuePattern", &mContinuePattern}, {"EndPattern", &mEndPattern}};
    bool compiled[3] = {false, false, false};
    int k = 0;
    for (auto& p : pats) {
        std::string pattern;
        if (GetString(config, p.key, pattern)) {
            // validation strips a trailing '$' and trailing ".*"s, yet the ORIGINAL pattern is stored (:205-222)
            std::string probe = pattern;
            if (!probe.empty() && EndsWith(probe, "$"))
                probe.pop_back();
            while (!probe.empty() && EndsWith(probe, ".*"))
                probe.resize(probe.size() - 2);
            bool valid = true;
            if (!probe.empty()) {
                CompiledRegex tmp;
                std::string e;
                lc_regex_t* raw = nullptr;
                int rc = lc_regex_compile(probe.data(), probe.size(), &raw);
                if (raw)
                    lc_regex_free(raw);
                valid = rc != LC_ERR_REGEX_INVALID;
                compiled[k] = valid;
            }
            if (valid)
                *p.dst = pattern;
        }
        ++k;
    }
    if (compiled[0] || compiled[2])
        mIsMultiline = true;
    std::string t;
    if (GetString(config, "UnmatchedContentTreatment", t) && t == "discard")
        mUnmatchedContentTreatment = UnmatchedContentTreatment::DISCARD;
    GetBool(config, "IgnoringUnmatchWarning", mIgnoringUnmatchWarning);
    (void)err;
    return true;
}

// ------------------------------------------------------------------------------------------------ split
const std::string ProcessorSplitLogStringNative::sName = "processor_split_string_native";

bool ProcessorSplitLogStringNative::Init(const Json::Value& config) {
    GetString(config, "SourceKey", mSourceKey);
    if (config.isMember("SplitChar") && config["SplitChar"].isInt())
        mSplitChar = (char)config["SplitChar"].asInt();
    GetBool(config, "EnableRawContent", mEnableRawContent);
    return true;
}

void ProcessorSplitLogStringNative::Process(PipelineEventGroup& group) {
    try {
        ProcessImpl(group);
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // the reference's Process never throws: the group stays as it was
    }
}

void ProcessorSplitLogStringNative::ProcessImpl(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    EventsContainer newEvents;
    std::vector<uint32_t> off, len;
    for (PipelineEventPtr& e : group.MutableEvents()) {
        if (!IsSupportedEvent(e)) {
            newEvents.emplace_back(std::move(e));
            continue;
        }
        LogEvent& src = e.Cast<LogEvent>();
        if (src.Size() != 1 || !src.HasContent(mSourceKey)) {
            newEvents.emplace_back(std::move(e));
            continue;
        }
        StringView val = src.GetContent(mSourceKey);
        StringBuffer sourceKey = group.GetSourceBuffer()->CopyString(mSourceKey);
        if (val.empty())
            continue;
        // a1 on the GPU: one (offset, length) per piece
        uint64_t n = 0;
        uint64_t cap = std::max<uint64_t>(1024, val.size() / 16);
        for (;;) {
            off.resize(cap);
            len.resize(cap);
            int rc = lc_split_lines(Engine(), reinterpret_cast<const uint8_t*>(val.data()), val.size(),
                                    (uint8_t)mSplitChar, off.data(), len.data(), cap, &n);
            if (rc == LC_ERR_CAPACITY) {
                cap = n;
                continue;
            }
            Check(rc, "lc_split_lines");
            break;
        }
        for (uint64_t k = 0; k < n; ++k) {
            StringView content(val.data() + off[k], len[k]);
            bool isLast = (uint64_t)off[k] + len[k] == val.size();
            EmitSplitEvent(group, src, val, sourceKey, content, isLast, mEnableRawContent, newEvents);
        }
    }
    group.SwapEvents(newEvents);
}

// ------------------------------------------------------------------------------------------------ multiline
const std::string ProcessorSplitMultilineLogStringNative::sName = "processor_split_multiline_log_string_native";

bool ProcessorSplitMultilineLogStringNative::Init(const Json::Value& config) {
    GetString(config, "SourceKey", mSourceKey);
    std::string err;
    if (!mMultiline.Init(config, err))
        return Fail(err);
    GetBool(config, "EnableRawContent", mEnableRawContent);
    // the processor compiles the ORIGINAL pattern strings (:70-80); an unsupported pattern fails Init loudly
    if (!mMultiline.mStartPattern.empty() && !mStart.Compile(mMultiline.mStartPattern, err))
        return Fail("Multiline.StartPattern: " + err);
    if (!mMultiline.mContinuePattern.empty() && !mContinue.Compile(mMultiline.mContinuePattern, err))
        return Fail("Multiline.ContinuePattern: " + err);
    if (!mMultiline.mEndPattern.empty() && !mEnd.Compile(mMultiline.mEndPattern, err))
        return Fail("Multiline.EndPattern: " + err);
    return true;
}

std::vector<std::pair<std::string, uint64_t>> ProcessorSplitMultilineLogStringNative::Counters() const {
    return {{"matched_events", mMatchedEventsTotal.GetValue()},
            {"matched_lines", mMatchedLinesTotal.GetValue()},
            {"unmatched_lines", mUnmatchedLinesTotal.GetValue()}};
}

void ProcessorSplitMultilineLogStringNative::Process(PipelineEventGroup& group) {
    try {
        ProcessImpl(group);
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // the reference's Process never throws: the group stays as it was
    }
}

void ProcessorSplitMultilineLogStringNative::ProcessImpl(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    EventsContainer newEvents;
    uint64_t inputLines = 0, unmatchLines = 0;
    std::vector<uint32_t> off, len;
    std::vector<uint8_t> flags;
    for (PipelineEventPtr& e : group.MutableEvents()) {
        if (!IsSupportedEvent(e)) {
            newEvents.emplace_back(std::move(e));
            continue;
        }
        LogEvent& src = e.Cast<LogEvent>();
        if (src.Size() != 1 || !src.HasContent(mSourceKey)) {
            newEvents.emplace_back(std::move(e));
            continue;
        }
        StringView val = src.GetContent(mSourceKey);
        StringBuffer sourceKey = group.GetSourceBuffer()->CopyString(mSourceKey);
        if (val.empty())
            continue;
        uint64_t n = 0, ctr[3] = {0, 0, 0};
        uint64_t cap = std::max<uint64_t>(1024, val.size() / 16);
        for (;;) {
            off.resize(cap);
            len.resize(cap);
            flags.resize(cap);
            uint64_t c[3] = {0, 0, 0};
            int rc = lc_multiline_split(
                Engine(), reinterpret_cast<const uint8_t*>(val.data()), val.size(), mStart.get(), mContinue.get(),
                mEnd.get(), mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD,
                off.data(), len.data(), flags.data(), cap, &n, c);
            if (rc == LC_ERR_CAPACITY) {
                cap = n;
                continue;
            }
            Check(rc, "lc_multiline_split");
            memcpy(ctr, c, sizeof ctr);
            break;
        }
        mMatchedEventsTotal.Add(ctr[0]);
        inputLines += ctr[1];
        unmatchLines += ctr[2];
        for (uint64_t k = 0; k < n; ++k)
            EmitSplitEvent(group, src, val, sourceKey, StringView(val.data() + off[k], len[k]),
                           (flags[k] & LC_ML_IS_LAST) != 0, mEnableRawContent, newEvents);
    }
    mMatchedLinesTotal.Add(inputLines - unmatchLines);
    mUnmatchedLinesTotal.Add(unmatchLines);
    group.SwapEvents(newEvents);
}

// ------------------------------------------------------------------------------------------------ regex parse
const std::string ProcessorParseRegexNative::sName = "processor_parse_regex_native";

static bool GetKeys(const Json::Value& config, std::vector<std::string>& keys) {
    if (!config.isMember("Keys") || !config["Keys"].isArray())
        return false;
    keys.clear();
    for (const auto& k : config["Keys"]) {
        if (!k.isString())
            return false;
        keys.push_back(k.asString());
    }
    return true;
}

bool ProcessorParseRegexNative::Init(const Json::Value& config) {
    if (!GetString(config, "SourceKey", mSourceKey))
        return Fail("mandatory string param SourceKey is missing");
    if (!GetString(config, "Regex", mRegex))
        return Fail("mandatory string param Regex is missing");
    mIsWholeLineMode = mRegex == "(.*)";
    std::string err;
    if (!mIsWholeLineMode && !mReg.Compile(mRegex, err))
        return Fail("mandatory string param Regex is not usable: " + err);
    if (!GetKeys(config, mKeys))
        return Fail("mandatory list param Keys is missing");
    // legacy ["k1,k2"] form (:80-88)
    if (mKeys.size() == 1 && mKeys[0].find(',') != std::string::npos) {
        std::vector<std::string> parts;
        size_t start = 0;
        const std::string joined = mKeys[0];
        for (;;) {
            size_t pos = joined.find(',', start);
            parts.push_back(joined.substr(start, pos == std::string::npos ? std::string::npos : pos - start));
            if (pos == std::string::npos)
                break;
            start = pos + 1;
        }
        mKeys = parts;
    }
    for (const auto& k : mKeys)
        if (k == mSourceKey)
            mSourceKeyOverwritten = true;
    mKeysDistinct = true;
    for (size_t a = 0; a < mKeys.size(); ++a)
        for (size_t b = a + 1; b < mKeys.size(); ++b)
            if (mKeys[a] == mKeys[b])
                mKeysDistinct = false;
    return mCommonParserOptions.Init(config);
}

std::vector<std::pair<std::string, uint64_t>> ProcessorParseRegexNative::Counters() const {
    return {{"discarded", mDiscardedEventsTotal.GetValue()},
            {"out_failed", mOutFailedEventsTotal.GetValue()},
            {"out_key_not_found", mOutKeyNotFoundEventsTotal.GetValue()},
            {"out_successful", mOutSuccessfulEventsTotal.GetValue()},
            {"b200_gather_ns", mGatherNs.GetValue()},
            {"b200_engine_ns", mEngineNs.GetValue()},
            {"b200_epilogue_ns", mEpilogueNs.GetValue()}};
}

void ProcessorParseRegexNative::AddCounters(const LocalCounters& c) {
    if (c.discarded)
        mDiscardedEventsTotal.Add(c.discarded);
    if (c.failed)
        mOutFailedEventsTotal.Add(c.failed);
    if (c.keyNotFound)
        mOutKeyNotFoundEventsTotal.Add(c.keyNotFound);
    if (c.successful)
        mOutSuccessfulEventsTotal.Add(c.successful);
}

// ProcessEvent (:132-168) with the regex verdict already known.  r == nullptr: the event never reached the engine
// (unsupported type, source key absent, or whole-line mode).
bool ProcessorParseRegexNative::FinishEvent(PipelineEventGroup& group, PipelineEventPtr& e,
                                            const LogEvent::Content* src, const EventResult* r,
                                            LocalCounters& c) const {
    if (!IsSupportedEvent(e)) {
        ++c.failed;
        return true;
    }
    LogEvent& ev = e.Cast<LogEvent>();
    if (!src) {
        ++c.keyNotFound;
        return true;
    }
    StringView rawContent = src->first.second;
    bool ok = true;
    if (mIsWholeLineMode) {
        AddLog(ev, mKeys.empty() ? StringView("content") : StringView(mKeys[0]), rawContent);
    } else if (r->status == LC_REGEX_NOMATCH) {
        ++c.failed;
        ok = false;
    } else if (r->status == LC_REGEX_KEYS_MISMATCH) {
        ok = false;
    } else if (mKeysDistinct && !mSourceKeyOverwritten && ev.RawContents().size() == 1) {
        // the event holds nothing but the source key and no key can collide: SetContentNoCopy's look-up per key
        // (LogEvent.cpp:83-95) would find nothing, so the fields are appended directly (same resulting contents)
        for (uint32_t k = 0; k < mKeys.size(); ++k)
            ev.AppendContentNoCopy(mKeys[k], StringView(r->origin + (r->capOff[k] - r->originOff), r->capLen[k]));
    } else {
        for (uint32_t k = 0; k < mKeys.size(); ++k)
            AddLog(ev, mKeys[k], StringView(r->origin + (r->capOff[k] - r->originOff), r->capLen[k]));
    }
    if (!ok || !mSourceKeyOverwritten)
        ev.DelContent(mSourceKey);
    if (mCommonParserOptions.ShouldAddSourceContent(ok))
        AddLog(ev, mCommonParserOptions.mRenamedSourceKey, rawContent, false);
    if (mCommonParserOptions.ShouldAddLegacyUnmatchedRawLog(ok))
        AddLog(ev, CommonParserOptions::legacyUnmatchedRawLogKey, rawContent, false);
    if (mCommonParserOptions.ShouldEraseEvent(ok, ev, group.GetAllMetadata())) {
        ++c.discarded;
        return false;
    }
    ++c.successful;
    return true;
}

// the epilogue of every event of one group; the group's parsed events own rows firstEv, firstEv + 1, ... of the tables
void ProcessorParseRegexNative::EpilogueGroup(PipelineEventGroup& group, uint64_t firstEv, const ThreadScratch& sc,
                                              uint32_t G, LocalCounters& c) const {
    EventsContainer& events = group.MutableEvents();
    size_t wIdx = 0;
    const size_t nev = events.size();
    for (size_t rIdx = 0; rIdx < nev; ++rIdx) {
        // the walk is bound by cache misses on the event objects and their contents arrays (one heap block each, touched
        // once): pull the object 16 events ahead and its contents array 8 events ahead
        if (rIdx + 16 < nev && events[rIdx + 16])
            __builtin_prefetch(events[rIdx + 16].operator->(), 1, 1);
        if (rIdx + 8 < nev && IsSupportedEvent(events[rIdx + 8])) {
            const auto& rc = events[rIdx + 8].Cast<LogEvent>().RawContents();
            if (!rc.empty()) {
                __builtin_prefetch(rc.data(), 1, 1);
                __builtin_prefetch(reinterpret_cast<const char*>(rc.data()) + 256, 1, 1);
            }
        }
        EventResult r{};
        const EventResult* rp = nullptr;
        const LogEvent::Content* src = nullptr;
        const uint64_t i = firstEv + rIdx; // the event's row of the result tables
        if (IsSupportedEvent(events[rIdx])) {
            src = events[rIdx].Cast<LogEvent>().FindContent(mSourceKey);
            if (src && !mIsWholeLineMode) {
                r.status = sc.status.p[i];
                r.capOff = sc.capOff.p + i * G;
                r.capLen = sc.capLen.p + i * G;
                r.origin = src->first.second.data(); // captures map back onto the ORIGINAL bytes, staged or not
                r.originOff = sc.off.p[i];
                rp = &r;
            }
        }
        if (FinishEvent(group, events[rIdx], src, rp, c)) {
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
    }
    events.resize(wIdx);
}

void ProcessorParseRegexNative::Process(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    ProcessBatch(&group, 1);
}

void ProcessorParseRegexNative::Process(std::vector<PipelineEventGroup>& groups) {
    // sub-batches of at most 2048 groups (<= 512 KB each: <= 1 GiB of arena bytes, far below the 4 GiB / 2^30-event
    // limits of one engine call); groups that are larger than the reader's 512 KB make ProcessBatch split further
    const size_t kMaxGroups = 2048;
    for (size_t g0 = 0; g0 < groups.size(); g0 += kMaxGroups)
        ProcessBatch(groups.data() + g0, std::min(kMaxGroups, groups.size() - g0));
}

// One engine call for `ngroups` groups.  Per group the values to parse normally alias ONE arena chunk (all lines of a
// file read): that chunk range is the group's span and goes to the GPU in place; a group whose values are scattered
// over several chunks is packed into pinned staging first.
void ProcessorParseRegexNative::ProcessBatch(PipelineEventGroup* groups, size_t ngroups) {
    struct GroupPlan {
        uint64_t firstEv = 0, nEv = 0; // slice of the flat event table
        const char* lo = nullptr;      // span = [lo, lo + spanLen) in host memory
        uint32_t spanLen = 0, spanDst = 0;
        bool staged = false;
        uint64_t stagedAt = 0;
    };
    std::vector<GroupPlan> plan(ngroups);
    using Clock = std::chrono::steady_clock;
    auto since = [](Clock::time_point t0) {
        return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(Clock::now() - t0).count();
    };
    try {
        uint64_t nb = 0;
        const auto tGather = Clock::now();
        if (!mIsWholeLineMode) {
            // Rows of the flat event table map 1:1 onto the events of the groups (row = firstEv of the group + index of
            // the event): an event that does not reach RegexLogLineParser gets an empty row the engine parses for
            // nothing and the epilogue ignores.  That makes the gather ONE pass over the events.
            for (size_t g = 0; g < ngroups; ++g) {
                plan[g].firstEv = nb;
                plan[g].nEv = groups[g].GetEvents().size();
                nb += plan[g].nEv;
            }
            if (nb) {
                ThreadScratch& sc = Scratch();
                const uint32_t G = mReg.groups();
                uint32_t* off = sc.off.ensure(nb);
                uint32_t* len = sc.len.ensure(nb);
                uint8_t* status = sc.status.ensure(nb);
                uint32_t* capOff = sc.capOff.ensure(nb * G + 1);
                uint32_t* capLen = sc.capLen.ensure(nb * G + 1);
                // ---- pass 1 (parallel over groups): span = the arena chunk that holds the group's values (the reader's
                // <= 512 KB buffer); offsets relative to it for now
                ParallelFor(ngroups, 8, [&](size_t a, size_t b, unsigned) {
                    for (size_t g = a; g < b; ++g) {
                        GroupPlan& p = plan[g];
                        const char* base = nullptr;
                        size_t chunkSize = 0;
                        uint64_t total = 0;
                        uint64_t i = p.firstEv;
                        const EventsContainer& gev = groups[g].GetEvents();
                        for (size_t x = 0; x < gev.size(); ++x) {
                            const PipelineEventPtr& e = gev[x];
                            // (cache misses on the event objects and their contents arrays: pull them in ahead)
                            if (x + 16 < gev.size() && gev[x + 16])
                                __builtin_prefetch(gev[x + 16].operator->(), 0, 1);
                            if (x + 8 < gev.size() && IsSupportedEvent(gev[x + 8])) {
                                const auto& rc = gev[x + 8].Cast<LogEvent>().RawContents();
                                if (!rc.empty())
                                    __builtin_prefetch(rc.data(), 0, 1);
                            }
                            const LogEvent::Content* src =
                                IsSupportedEvent(e) ? e.Cast<LogEvent>().FindContent(mSourceKey) : nullptr;
                            if (!src) {
                                off[i] = 0;
                                len[i] = 0;
                                ++i;
                                continue;
                            }
                            StringView v = src->first.second;
                            if (!base && !p.staged) {
                                base = groups[g].GetSourceBuffer()->ChunkContaining(v.data(), v.size(), &chunkSize);
                                if (!base || chunkSize >= (1ull << 31))
                                    p.staged = true;
                            }
                            if (!p.staged && !(v.data() >= base && v.data() + v.size() <= base + chunkSize))
                                p.staged = true;
                            off[i] = p.staged ? 0u : (uint32_t)(v.data() - base);
                            len[i] = (uint32_t)v.size();
                            total += v.size();
                            ++i;
                        }
                        if (p.staged) {
                            p.spanLen = (uint32_t)total;
                        } else {
                            p.lo = base;
                            p.spanLen = base ? (uint32_t)chunkSize : 0u;
                        }
                    }
                });
                {
                    // (oversized batch: groups far larger than the reader's chunks) split and recurse
                    uint64_t bytes = 0;
                    for (auto& p : plan)
                        bytes += ((uint64_t)p.spanLen + 15) & ~15ull;
                    if (ngroups > 1 && (bytes >= (3ull << 30) || nb >= (1ull << 29))) {
                        ProcessBatch(groups, ngroups / 2);
                        ProcessBatch(groups + ngroups / 2, ngroups - ngroups / 2);
                        return;
                    }
                }
                uint64_t dst = 0, stagedBytes = 0;
                for (auto& p : plan) {
                    p.spanDst = (uint32_t)dst;
                    dst += ((uint64_t)p.spanLen + 15) & ~15ull;
                    if (p.staged) {
                        p.stagedAt = stagedBytes;
                        stagedBytes += ((uint64_t)p.spanLen + 15) & ~15ull;
                    }
                }
                uint8_t* staging = stagedBytes ? sc.staging.ensure(stagedBytes) : nullptr;
                // ---- pass 2 (parallel): packed-arena coordinates; groups whose values are scattered over several
                // chunks are packed into pinned staging here
                ParallelFor(ngroups, 8, [&](size_t a, size_t b, unsigned) {
                    for (size_t g = a; g < b; ++g) {
                        GroupPlan& p = plan[g];
                        uint64_t i = p.firstEv;
                        if (!p.staged) {
                            for (uint64_t k = 0; k < p.nEv; ++k)
                                off[i + k] += p.spanDst;
                            continue;
                        }
                        uint64_t at = 0;
                        p.lo = reinterpret_cast<const char*>(staging + p.stagedAt);
                        for (const auto& e : groups[g].GetEvents()) {
                            const LogEvent::Content* src =
                                IsSupportedEvent(e) ? e.Cast<LogEvent>().FindContent(mSourceKey) : nullptr;
                            if (src) {
                                StringView v = src->first.second;
                                if (v.size())
                                    memcpy(staging + p.stagedAt + at, v.data(), v.size());
                                off[i] = p.spanDst + (uint32_t)at;
                                at += v.size();
                            } else {
                                off[i] = p.spanDst;
                            }
                            ++i;
                        }
                    }
                });
                std::vector<const uint8_t*> spanPtr(ngroups);
                std::vector<uint32_t> spanLen(ngroups), spanDst(ngroups);
                std::vector<uint64_t> spanFirst(ngroups + 1);
                for (size_t g = 0; g < ngroups; ++g) {
                    spanPtr[g] = reinterpret_cast<const uint8_t*>(plan[g].lo);
                    spanLen[g] = plan[g].nEv ? plan[g].spanLen : 0;
                    spanDst[g] = plan[g].spanDst;
                    spanFirst[g] = plan[g].firstEv;
                }
                spanFirst[ngroups] = nb;
                mGatherNs.Add(since(tGather));
                // ---- pass 3: the per-event epilogue of a range of groups (parallel over the groups)
                const uint32_t Gc = mReg.groups();
                std::vector<LocalCounters> local(HostThreads());
                uint64_t epilogueNs = 0;
                auto epilogue = [&](size_t gBegin, size_t gCount) {
                    const auto t0 = Clock::now();
                    ParallelFor(gCount, 4, [&](size_t a, size_t b, unsigned tid) {
                        LocalCounters& c = local[tid];
                        for (size_t g = gBegin + a; g < gBegin + b; ++g)
                            EpilogueGroup(groups[g], plan[g].firstEv, sc, Gc, c);
                    });
                    epilogueNs += since(t0);
                };
                struct Ctx {
                    decltype(epilogue)* fn;
                } cbctx{&epilogue};
                const auto tEngine = Clock::now();
                Check(lc_regex_parse_packed_cb(
                          Engine(), mReg.get(), ngroups, spanPtr.data(), spanLen.data(), spanDst.data(),
                          spanFirst.data(), dst, off, len, nb, (uint32_t)mKeys.size(), status, capOff, capLen,
                          [](void* ctx, uint64_t first, uint64_t count) {
                              (*static_cast<Ctx*>(ctx)->fn)((size_t)first, (size_t)count);
                          },
                          &cbctx),
                      "lc_regex_parse_packed");
                mEngineNs.Add(since(tEngine) - epilogueNs); // the call's own share (the epilogue runs inside it)
                mEpilogueNs.Add(epilogueNs);
                for (const auto& c : local)
                    AddCounters(c);
                return;
            }
        }
        // nothing reached the engine (whole-line mode, or no event carries the source key): epilogue only
        const auto tEpilogue = Clock::now();
        ThreadScratch& sc = Scratch();
        std::vector<LocalCounters> local(HostThreads());
        ParallelFor(ngroups, 8, [&](size_t a, size_t b, unsigned tid) {
            for (size_t g = a; g < b; ++g)
                EpilogueGroup(groups[g], plan[g].firstEv, sc, mReg.groups(), local[tid]);
        });
        for (const auto& c : local)
            AddCounters(c);
        mEpilogueNs.Add(since(tEpilogue));
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // groups not yet rewritten stay untouched (the reference never throws out of Process)
    }
}

// ------------------------------------------------------------------------------------------------ instance wrapper
void ProcessorInstance::Process(std::vector<PipelineEventGroup>& eventGroupList) {
    if (eventGroupList.empty())
        return;
    // the two DataSize() sweeps run on the host threads of the batch when the call carries many groups (the reference
    // spreads them over its ProcessorRunner threads, one group per call)
    auto sweep = [&](Counter& events, Counter& bytes) {
        ParallelFor(eventGroupList.size(), 64, [&](size_t a, size_t b, unsigned) {
            uint64_t ev = 0, by = 0;
            for (size_t g = a; g < b; ++g) {
                ev += eventGroupList[g].GetEvents().size();
                by += eventGroupList[g].DataSize();
            }
            events.Add(ev);
            bytes.Add(by);
        });
    };
    sweep(mInEventsTotal, mInSizeBytes);
    const auto before = std::chrono::steady_clock::now();
    mPlugin->Process(eventGroupList);
    const auto ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - before);
    mTotalProcessTimeNs.Add((uint64_t)ns.count());
    mTotalProcessTimeMs.Add((uint64_t)(ns.count() / 1000000));
    sweep(mOutEventsTotal, mOutSizeBytes);
}

// ------------------------------------------------------------------------------------------------ delimiter
const std::string ProcessorParseDelimiterNative::sName = "processor_parse_delimiter_native";

bool ProcessorParseDelimiterNative::Init(const Json::Value& config) {
    if (!GetString(config, "SourceKey", mSourceKey))
        return Fail("mandatory string param SourceKey is missing");
    if (!GetString(config, "Separator", mSeparator) || mSeparator.empty())
        return Fail("mandatory string param Separator is missing");
    if (mSeparator.size() > 4)
        return Fail("mandatory string param Separator has more than 4 chars");
    if (mSeparator == "\\t")
        mSeparator = "\t";
    std::string quote;
    bool hasQuote = GetString(config, "Quote", quote);
    if (mSeparator.size() == 1) {
        if (hasQuote && quote.size() > 1)
            return Fail("string param Quote is not a single char");
        if (hasQuote && !quote.empty())
            mQuote = quote[0];
    } // multi-char separator: a configured Quote is ignored (warning upstream)
    if (!GetKeys(config, mKeys))
        return Fail("mandatory list param Keys is missing");
    for (const auto& k : mKeys)
        if (k == mSourceKey)
            mSourceKeyOverwritten = true;
    GetBool(config, "AllowingShortenedFields", mAllowingShortenedFields);
    std::string t;
    if (GetString(config, "OverflowedFieldsTreatment", t)) {
        if (t == "keep")
            mOverflowedFieldsTreatment = OverflowedFieldsTreatment::KEEP;
        else if (t == "discard")
            mOverflowedFieldsTreatment = OverflowedFieldsTreatment::DISCARD;
    }
    mExtractingPartialFields = mOverflowedFieldsTreatment == OverflowedFieldsTreatment::DISCARD;
    if (!mCommonParserOptions.Init(config))
        return false;
    // SerializeSls's one-pass device path takes the configurations lc_delim_parse_sls accepts
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    size_t kbytes = mSourceKey.size() + mCommonParserOptions.mRenamedSourceKey.size() + 11;
    for (const auto& k : mKeys) {
        kp.push_back(k.data());
        kl.push_back((uint32_t)k.size());
        kbytes += k.size();
    }
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(mKeys.size() + 4);
    LcDelimSlsCfg c;
    mDeviceSls = lc_delim_sls_setup(reinterpret_cast<const uint8_t*>(mSeparator.data()), (uint32_t)mSeparator.size(),
                                    (uint8_t)mQuote, mOverflowedFieldsTreatment == OverflowedFieldsTreatment::EXTEND,
                                    mExtractingPartialFields, kp.data(), kl.data(), (uint32_t)mKeys.size(),
                                    mSourceKey.data(), (uint32_t)mSourceKey.size(),
                                    mCommonParserOptions.mRenamedSourceKey.data(),
                                    (uint32_t)mCommonParserOptions.mRenamedSourceKey.size(), 0, 0, 0,
                                    (uint32_t)mKeys.size() + 16, &c, kb.data(), at.data()) == nullptr;
    return true;
}

std::vector<std::pair<std::string, uint64_t>> ProcessorParseDelimiterNative::Counters() const {
    return {{"discarded", mDiscardedEventsTotal.GetValue()},
            {"out_failed", mOutFailedEventsTotal.GetValue()},
            {"out_key_not_found", mOutKeyNotFoundEventsTotal.GetValue()},
            {"out_successful", mOutSuccessfulEventsTotal.GetValue()}};
}

void ProcessorParseDelimiterNative::Process(PipelineEventGroup& group) {
    try {
        ProcessImpl(group);
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // the reference's Process never throws: the group stays as it was
    }
}

void ProcessorParseDelimiterNative::ProcessImpl(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    EventsContainer& events = group.MutableEvents();
    FlatBatch batch;
    for (size_t i = 0; i < events.size(); ++i) {
        if (!IsSupportedEvent(events[i]))
            continue;
        const LogEvent& ev = events[i].Cast<LogEvent>();
        if (ev.HasContent(mSourceKey))
            batch.Add(i, ev.GetContent(mSourceKey));
    }
    batch.Finish(*group.GetSourceBuffer());
    const size_t nb = batch.eventIndex.size();
    const bool extend = mOverflowedFieldsTreatment == OverflowedFieldsTreatment::EXTEND;
    const bool useQuote = mSeparator.size() == 1 && mQuote != mSeparator[0];
    // Dense [n][MF] field tables with MF = keys + 16 serve every ordinary line.  A line with more columns than that
    // (log content is untrusted: one 256 KB line of separators must not size a table for the whole group) is parsed
    // again on its own, in small sub-batches whose tables hold exactly its columns -- memory stays O(bytes of those
    // lines), like the reference's per-line vectors (:246-248).
    const uint32_t MF = (uint32_t)mKeys.size() + 16;
    std::vector<uint8_t> status(nb);
    std::vector<uint32_t> nf(nb), fo((size_t)nb * MF), fl((size_t)nb * MF), fd((size_t)nb * MF);
    std::vector<uint32_t> wfo, wfl, wfd;
    std::vector<size_t> wideStart(nb, (size_t)-1);
    if (nb) {
        Check(lc_delim_parse(Engine(), batch.base, batch.baseLen, batch.off.data(), batch.len.data(), nb,
                             reinterpret_cast<const uint8_t*>(mSeparator.data()), (uint32_t)mSeparator.size(),
                             (uint8_t)mQuote, (uint32_t)mKeys.size(), extend, mAllowingShortenedFields, MF,
                             status.data(), nf.data(), fo.data(), fl.data(), fd.data()),
              "lc_delim_parse");
        std::vector<size_t> over;
        for (size_t i = 0; i < nb; ++i)
            if (nf[i] > MF && status[i] != LC_DELIM_PARSE_FAIL && status[i] != LC_DELIM_BLANK)
                over.push_back(i);
        const size_t kMaxEntries = 4u << 20; // 48 MB of tables per sub-batch at most (+ one oversize line alone)
        size_t at = 0;
        while (at < over.size()) {
            size_t cnt = 0;
            uint32_t mx = 0;
            while (at + cnt < over.size()) {
                uint32_t m2 = std::max(mx, nf[over[at + cnt]]);
                if (cnt && (cnt + 1) * (size_t)m2 > kMaxEntries)
                    break;
                mx = m2;
                ++cnt;
            }
            std::vector<uint32_t> so(cnt), sl(cnt), snf(cnt), sfo(cnt * (size_t)mx), sfl(cnt * (size_t)mx),
                sfd(cnt * (size_t)mx);
            std::vector<uint8_t> sst(cnt);
            for (size_t k = 0; k < cnt; ++k) {
                so[k] = batch.off[over[at + k]];
                sl[k] = batch.len[over[at + k]];
            }
            Check(lc_delim_parse(Engine(), batch.base, batch.baseLen, so.data(), sl.data(), cnt,
                                 reinterpret_cast<const uint8_t*>(mSeparator.data()), (uint32_t)mSeparator.size(),
                                 (uint8_t)mQuote, (uint32_t)mKeys.size(), extend, mAllowingShortenedFields, mx,
                                 sst.data(), snf.data(), sfo.data(), sfl.data(), sfd.data()),
                  "lc_delim_parse");
            for (size_t k = 0; k < cnt; ++k) {
                const size_t i = over[at + k];
                wideStart[i] = wfo.size();
                wfo.insert(wfo.end(), sfo.begin() + k * (size_t)mx, sfo.begin() + k * (size_t)mx + nf[i]);
                wfl.insert(wfl.end(), sfl.begin() + k * (size_t)mx, sfl.begin() + k * (size_t)mx + nf[i]);
                wfd.insert(wfd.end(), sfd.begin() + k * (size_t)mx, sfd.begin() + k * (size_t)mx + nf[i]);
            }
            at += cnt;
        }
    }

    size_t wIdx = 0, b = 0;
    std::vector<StringView> cols;
    for (size_t rIdx = 0; rIdx < events.size(); ++rIdx) {
        bool keep = true;
        PipelineEventPtr& e = events[rIdx];
        if (!IsSupportedEvent(e)) {
            mOutFailedEventsTotal.Add(1);
        } else {
            LogEvent& ev = e.Cast<LogEvent>();
            if (!ev.HasContent(mSourceKey)) {
                mOutKeyNotFoundEventsTotal.Add(1);
            } else {
                StringView buffer = ev.GetContent(mSourceKey);
                const uint8_t st = status[b];
                if (st == LC_DELIM_BLANK) {
                    // empty / blank value: out_failed++, event untouched (:220-242)
                    mOutFailedEventsTotal.Add(1);
                } else {
                    bool ok = st == LC_DELIM_OK;
                    if (ok) {
                        cols.clear();
                        SourceBuffer& sb = *group.GetSourceBuffer();
                        const bool wide = wideStart[b] != (size_t)-1;
                        const uint32_t* ro = wide ? wfo.data() + wideStart[b] : fo.data() + (size_t)b * MF;
                        const uint32_t* rl = wide ? wfl.data() + wideStart[b] : fl.data() + (size_t)b * MF;
                        const uint32_t* rd = wide ? wfd.data() + wideStart[b] : fd.data() + (size_t)b * MF;
                        for (uint32_t j = 0; j < nf[b]; ++j) {
                            uint32_t o = ro[j], l = rl[j], dq = rd[j];
                            StringView raw = batch.View(b, o, l);
                            if (useQuote && dq) {
                                // AddFieldWithUnQuote (:83-113): collapse doubled quotes into a fresh arena string
                                StringBuffer f = sb.AllocateStringBuffer(l - dq);
                                size_t w = 0;
                                for (size_t i = 0; i < raw.size(); ++i) {
                                    if (raw[i] == mQuote) {
                                        if (i + 1 < raw.size() && raw[i + 1] == mQuote) {
                                            f.data[w++] = mQuote;
                                            ++i;
                                        }
                                    } else {
                                        f.data[w++] = raw[i];
                                    }
                                }
                                cols.emplace_back(f.data, l - dq);
                            } else {
                                cols.push_back(raw);
                            }
                        }
                        if (useQuote && !extend && cols.size() > mKeys.size()) {
                            // overflow columns re-joined as sep + value each (:258-275)
                            size_t need = 0;
                            for (size_t j = mKeys.size(); j < cols.size(); ++j)
                                need += 1 + cols[j].size();
                            StringBuffer x = sb.AllocateStringBuffer(need);
                            char* p = x.data;
                            for (size_t j = mKeys.size(); j < cols.size(); ++j) {
                                *p++ = mSeparator[0];
                                memcpy(p, cols[j].data(), cols[j].size());
                                p += cols[j].size();
                            }
                            cols.resize(mKeys.size());
                            cols.emplace_back(x.data, need);
                        }
                        for (uint32_t idx = 0; idx < cols.size(); ++idx) {
                            if (idx < mKeys.size()) {
                                if (mExtractingPartialFields && mKeys[idx] == "_")
                                    continue;
                                AddLog(ev, mKeys[idx], cols[idx]);
                            } else {
                                if (mExtractingPartialFields)
                                    continue;
                                std::string key = "__column" + ToString(idx) + "__";
                                StringBuffer kb = sb.CopyString(key);
                                AddLog(ev, StringView(kb.data, kb.size), cols[idx]);
                            }
                        }
                        mOutSuccessfulEventsTotal.Add(1);
                    } else {
                        mOutFailedEventsTotal.Add(1);
                    }
                    if (!ok || !mSourceKeyOverwritten)
                        ev.DelContent(mSourceKey);
                    if (mCommonParserOptions.ShouldAddSourceContent(ok))
                        AddLog(ev, mCommonParserOptions.mRenamedSourceKey, buffer, false);
                    if (mCommonParserOptions.ShouldAddLegacyUnmatchedRawLog(ok))
                        AddLog(ev, CommonParserOptions::legacyUnmatchedRawLogKey, buffer, false);
                    if (mCommonParserOptions.ShouldEraseEvent(ok, ev, group.GetAllMetadata())) {
                        mDiscardedEventsTotal.Add(1);
                        keep = false;
                    }
                }
                ++b;
            }
        }
        if (keep) {
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
    }
    events.resize(wIdx);
}

// ------------------------------------------------------------------------------------------------ filter
const std::string ProcessorFilterNative::sName = "processor_filter_regex_native";

ProcessorFilterNative::~ProcessorFilterNative() {
    for (auto& l : mLeaves)
        delete l.reg;
}

static std::string Lower(std::string s) {
    for (auto& c : s)
        if (c >= 'A' && c <= 'Z')
            c = (char)(c + 32);
    return s;
}

// ParseExpressionFromJSON (:380-425): returns node index or -1
int ProcessorFilterNative::ParseExpression(const Json::Value& v, std::string& err) {
    if (!v.isObject())
        return -1;
    if (v["operator"].isString() && v["operands"].isArray()) {
        std::string op = Lower(v["operator"].asString());
        const Json::Value& ops = v["operands"];
        if (op == "not" && ops.size() == 1) {
            int c = ParseExpression(ops[(size_t)0], err);
            if (c < 0)
                return -1;
            Node n;
            n.op = 1;
            n.left = c;
            mNodes.push_back(n);
            return (int)mNodes.size() - 1;
        }
        if ((op == "and" || op == "or") && ops.size() == 2) {
            int l = ParseExpression(ops[(size_t)0], err);
            int r = ParseExpression(ops[(size_t)1], err);
            if (l < 0 || r < 0)
                return -1;
            Node n;
            n.op = op == "and" ? 2 : 3;
            n.left = l;
            n.right = r;
            mNodes.push_back(n);
            return (int)mNodes.size() - 1;
        }
        return -1;
    }
    if ((v["key"].isString() && v["exp"].isString()) || !v["type"].isString()) {
        if (Lower(v["type"].asString()) != "regex")
            return -1;
        Leaf leaf;
        leaf.key = v["key"].asString();
        leaf.reg = new CompiledRegex;
        if (!leaf.reg->Compile(v["exp"].asString(), err)) {
            delete leaf.reg;
            return -1;
        }
        mLeaves.push_back(leaf);
        Node n;
        n.op = 0;
        n.leaf = (int)mLeaves.size() - 1;
        mNodes.push_back(n);
        return (int)mNodes.size() - 1;
    }
    return -1;
}

bool ProcessorFilterNative::Init(const Json::Value& config) {
    std::string err;
    if (config.isMember("ConditionExp")) {
        if (!config["ConditionExp"].isObject())
            return Fail("object param ConditionExp is not of type object");
        mRoot = ParseExpression(config["ConditionExp"], err);
        if (mRoot < 0)
            return Fail("object param ConditionExp is not valid " + err);
        mFilterMode = Mode::EXPRESSION_MODE;
    }
    auto addRule = [&](const std::string& key, const std::string& pattern) -> bool {
        Leaf leaf;
        leaf.key = key;
        leaf.reg = new CompiledRegex;
        if (!leaf.reg->Compile(pattern, err)) {
            delete leaf.reg;
            return false;
        }
        mLeaves.push_back(leaf);
        return true;
    };
    if (mFilterMode == Mode::BYPASS_MODE && config.isMember("FilterKey") && config.isMember("FilterRegex")) {
        const Json::Value &ks = config["FilterKey"], &rs = config["FilterRegex"];
        if (!ks.isArray() || !rs.isArray() || ks.size() != rs.size())
            return Fail("param FilterKey and FilterRegex does not have the same size");
        for (size_t i = 0; i < ks.size(); ++i)
            if (!addRule(ks[i].asString(), rs[i].asString()))
                return Fail("value in list param FilterRegex is not a usable regex: " + err);
        if (ks.size())
            mFilterMode = Mode::RULE_MODE;
    }
    if (mFilterMode == Mode::BYPASS_MODE && config.isMember("Include") && config["Include"].isObject()) {
        for (const auto& k : config["Include"].getMemberNames())
            if (!addRule(k, config["Include"][k].asString()))
                return Fail("value in map param Include is not a usable regex: " + err);
        if (!mLeaves.empty())
            mFilterMode = Mode::RULE_MODE;
    }
    GetBool(config, "DiscardingNonUTF8", mDiscardingNonUTF8);
    BuildDeviceFilter();
    return true;
}

void ProcessorFilterNative::BuildDeviceFilter() {
    mDevKeys.clear();
    mDevKeyLens.clear();
    mDevRegs.clear();
    mDevProg.clear();
    for (const Leaf& l : mLeaves) {
        mDevKeys.push_back(l.key.data());
        mDevKeyLens.push_back((uint32_t)l.key.size());
        mDevRegs.push_back(l.reg->get());
    }
    uint32_t depth = 0, maxDepth = 0;
    auto push = [&](uint32_t op) {
        mDevProg.push_back(op);
        depth = op < LC_FILTER_NOT ? depth + 1 : op == LC_FILTER_NOT ? depth : depth - 1;
        maxDepth = depth > maxDepth ? depth : maxDepth;
    };
    if (mFilterMode == Mode::RULE_MODE) {
        for (size_t li = 0; li < mLeaves.size(); ++li) {
            push((uint32_t)li);
            if (li)
                push(LC_FILTER_AND);
        }
    } else if (mFilterMode == Mode::EXPRESSION_MODE) {
        auto post = [&](auto&& self, int node) -> void {
            const Node& n = mNodes[node];
            if (n.op == 0) {
                push((uint32_t)n.leaf);
                return;
            }
            self(self, n.left);
            if (n.op != 1)
                self(self, n.right);
            push(n.op == 1 ? LC_FILTER_NOT : n.op == 2 ? LC_FILTER_AND : LC_FILTER_OR);
        };
        post(post, mRoot);
    }
    mDeviceOk = !mDiscardingNonUTF8 && mLeaves.size() <= LC_FILTER_MAX_LEAVES &&
                mDevProg.size() <= LC_FILTER_MAX_PROG && maxDepth <= 32;
}

bool ProcessorFilterNative::DeviceFilter(lc_filter_desc_t* d) const {
    if (!mDeviceOk)
        return false;
    d->nleaves = (uint32_t)mLeaves.size();
    d->keys = mDevKeys.data();
    d->key_lens = mDevKeyLens.data();
    d->regs = mDevRegs.data();
    d->nprog = (uint32_t)mDevProg.size();
    d->prog = mDevProg.data();
    return true;
}

bool ProcessorFilterNative::Eval(int node, const std::vector<std::vector<uint8_t>>& leafResult, size_t ev) const {
    const Node& n = mNodes[node];
    switch (n.op) {
        case 0:
            return leafResult[n.leaf][ev] != 0;
        case 1:
            return !Eval(n.left, leafResult, ev);
        case 2:
            return Eval(n.left, leafResult, ev) && Eval(n.right, leafResult, ev);
        default:
            return Eval(n.left, leafResult, ev) || Eval(n.right, leafResult, ev);
    }
}

// ProcessorFilterNative::noneUtf8 (:297-378): blank every byte that starts an invalid sequence; true if any
static bool BlankNoneUtf8(std::string& s, bool modify) {
    bool bad = false;
    size_t i = 0, n = s.size();
    auto cont = [&](size_t k) { return k < n && ((unsigned char)s[k] & 0xC0) == 0x80; };
    while (i < n) {
        unsigned char c = (unsigned char)s[i];
        size_t step = 1;
        bool inv = false;
        if ((c & 0x80) == 0) {
        } else if ((c & 0xE0) == 0xC0) {
            if (!cont(i + 1)) {
                inv = true;
            } else {
                uint32_t u = ((c & 0x1Fu) << 6) | ((unsigned char)s[i + 1] & 0x3Fu);
                inv = !(u >= 0x80 && u <= 0x7FF);
                step = 2;
            }
        } else if ((c & 0xF0) == 0xE0) {
            if (!cont(i + 1) || !cont(i + 2)) {
                inv = true;
            } else {
                uint32_t u = (((c & 0x0Fu) << 12) | (((unsigned char)s[i + 1] & 0x3Fu) << 6) |
                              ((unsigned char)s[i + 2] & 0x3Fu)) &
                             0xFFFFu;
                inv = !(u >= 0x800);
                step = 3;
            }
        } else if ((c & 0xF8) == 0xF0) {
            if (!cont(i + 1) || !cont(i + 2) || !cont(i + 3)) {
                inv = true;
            } else {
                uint32_t u = ((c & 0x07u) << 18) | (((unsigned char)s[i + 1] & 0x3Fu) << 12) |
                             (((unsigned char)s[i + 2] & 0x3Fu) << 6) | ((unsigned char)s[i + 3] & 0x3Fu);
                inv = !(u >= 0x10000 && u <= 0x10FFFF);
                step = 4;
            }
        } else {
            inv = true;
        }
        if (inv) {
            if (!modify)
                return true;
            s[i] = ' ';
            bad = true;
            i += 1;
        } else {
            i += step;
        }
    }
    return bad;
}

void ProcessorFilterNative::Process(PipelineEventGroup& group) {
    try {
        ProcessImpl(group);
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // the reference's Process never throws: the group stays as it was
    }
}

void ProcessorFilterNative::ProcessImpl(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    EventsContainer& events = group.MutableEvents();
    const size_t ne = events.size();
    // one batched boolean regex_match per leaf over the events that carry its key
    std::vector<std::vector<uint8_t>> leafResult(mLeaves.size(), std::vector<uint8_t>(ne, 0));
    for (size_t li = 0; li < mLeaves.size(); ++li) {
        FlatBatch batch;
        for (size_t i = 0; i < ne; ++i) {
            if (!IsSupportedEvent(events[i]))
                continue;
            const LogEvent& ev = events[i].Cast<LogEvent>();
            if (ev.HasContent(mLeaves[li].key))
                batch.Add(i, ev.GetContent(mLeaves[li].key));
        }
        batch.Finish(*group.GetSourceBuffer());
        const size_t nb = batch.eventIndex.size();
        if (!nb)
            continue;
        std::vector<uint8_t> m(nb);
        Check(lc_regex_match(Engine(), mLeaves[li].reg->get(), batch.base, batch.baseLen, batch.off.data(),
                             batch.len.data(), nb, m.data()),
              "lc_regex_match");
        for (size_t b = 0; b < nb; ++b)
            leafResult[li][batch.eventIndex[b]] = m[b];
    }
    size_t wIdx = 0;
    for (size_t rIdx = 0; rIdx < ne; ++rIdx) {
        bool res = true;
        if (IsSupportedEvent(events[rIdx])) {
            LogEvent& ev = events[rIdx].Cast<LogEvent>();
            if (mFilterMode == Mode::EXPRESSION_MODE) {
                res = !ev.Empty() && Eval(mRoot, leafResult, rIdx);
            } else if (mFilterMode == Mode::RULE_MODE) {
                res = !ev.Empty();
                for (size_t li = 0; res && li < mLeaves.size(); ++li)
                    res = leafResult[li][rIdx] != 0; // a missing key left its slot at 0
            }
            if (res && mDiscardingNonUTF8) {
                std::vector<std::pair<StringView, StringView>> renamed;
                SourceBuffer& sb = *group.GetSourceBuffer();
                // contents are visited in place; keys needing repair are re-added after the walk (:190-211)
                std::vector<LogEvent::Content> snapshot = ev.RawContents();
                for (auto& c : snapshot) {
                    if (!c.second)
                        continue;
                    StringView key = c.first.first, val = c.first.second;
                    std::string v = val.to_string();
                    if (BlankNoneUtf8(v, true)) {
                        StringBuffer vb = sb.CopyString(v);
                        val = StringView(vb.data, vb.size);
                        ev.SetContentNoCopy(key, val);
                    }
                    std::string k = key.to_string();
                    if (BlankNoneUtf8(k, true)) {
                        StringBuffer kb = sb.CopyString(k);
                        renamed.emplace_back(StringView(kb.data, kb.size), val);
                        ev.DelContent(key);
                    }
                }
                for (auto& r : renamed)
                    ev.SetContentNoCopy(r.first, r.second);
            }
        }
        if (res) {
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
    }
    events.resize(wIdx);
}

// ------------------------------------------------------------------------------------------------ merge multiline
const std::string ProcessorMergeMultilineLogNative::sName = "processor_merge_multiline_log_native";
const std::string ProcessorMergeMultilineLogNative::PartLogFlag = "P";

bool ProcessorMergeMultilineLogNative::Init(const Json::Value& config) {
    GetString(config, "SourceKey", mSourceKey);
    std::string mergeType;
    if (!GetString(config, "MergeType", mergeType))
        return Fail("mandatory string param MergeType is missing");
    if (mergeType == "flag") {
        mMergeType = MergeType::BY_FLAG;
        return true;
    }
    if (mergeType != "regex")
        return Fail("string param MergeType is not valid");
    std::string err;
    if (!mMultiline.Init(config, err))
        return Fail(err);
    struct {
        const std::string* pattern;
        CompiledRegex* reg;
        bool* has;
    } regs[] = {{&mMultiline.mStartPattern, &mStartReg, &mHasStart},
                {&mMultiline.mContinuePattern, &mContinueReg, &mHasContinue},
                {&mMultiline.mEndPattern, &mEndReg, &mHasEnd}};
    for (auto& r : regs) {
        std::string p = *r.pattern;
        if (!p.empty() && EndsWith(p, "$"))
            p.pop_back();
        while (!p.empty() && EndsWith(p, ".*"))
            p.resize(p.size() - 2);
        if (p.empty())
            continue;
        if (!r.reg->Compile(p, err))
            return Fail("multiline pattern: " + err); // outside the automaton subset: never approximated
        *r.has = true;
    }
    if (!mHasStart && !mHasEnd && mHasContinue)
        mHasContinue = false;
    else if (mHasStart && mHasContinue && mHasEnd)
        mHasContinue = false;
    return true;
}

std::vector<std::pair<std::string, uint64_t>> ProcessorMergeMultilineLogNative::Counters() const {
    return {{"merged_events_total", mMergedEventsTotal.GetValue()},
            {"unmatched_events_total", mUnmatchedEventsTotal.GetValue()}};
}

void ProcessorMergeMultilineLogNative::Process(PipelineEventGroup& group) {
    try {
        ProcessImpl(group);
    } catch (const std::exception& ex) {
        EngineFailed(ex.what()); // the reference's Process never throws: the group stays as it was
    }
}

void ProcessorMergeMultilineLogNative::ProcessImpl(PipelineEventGroup& group) {
    if (group.GetEvents().empty())
        return;
    if (mMergeType == MergeType::BY_REGEX) {
        MergeLogsByRegex(group);
    } else if (group.HasMetadata(EventGroupMetaKey::HAS_PART_LOG)) {
        MergeLogsByFlag(group);
        group.DelMetadata(EventGroupMetaKey::HAS_PART_LOG);
    }
}

// :320-346.  The reference joins the values IN PLACE (it writes the line break over the byte that follows the target
// value and memmoves the next values down); that is only sound when the values lie in event order inside one
// arena chunk with nothing else in between, which is what the splitters produce.  Same here when that holds (values
// adjacent, at most one separator byte apart), else the joined value is built in a fresh arena allocation -- the
// resulting content is identical.
void ProcessorMergeMultilineLogNative::MergeEvents(PipelineEventGroup& group, std::vector<LogEvent*>& logEvents,
                                                   bool insertLineBreak) {
    if (logEvents.empty())
        return;
    mMergedEventsTotal.Add(logEvents.size());
    if (logEvents.size() == 1) {
        logEvents.clear();
        return;
    }
    LogEvent* target = logEvents[0];
    StringView targetValue = target->GetContent(mSourceKey);
    size_t total = targetValue.size();
    bool inPlace = true;
    const char* end = targetValue.data() + targetValue.size();
    for (size_t i = 1; i < logEvents.size(); ++i) {
        StringView cur = logEvents[i]->GetContent(mSourceKey);
        total += cur.size() + (insertLineBreak ? 1 : 0);
        const char* dst = end + (insertLineBreak ? 1 : 0);
        // adjacent values only (at most the one separator byte the splitter left between them): anything else
        // in the gap -- e.g. another content of the target event -- must not be overwritten
        if (cur.data() < dst || cur.data() > end + 1)
            inPlace = false;
        end = dst + cur.size();
    }
    size_t chunkSize = 0;
    SourceBuffer& sb = *group.GetSourceBuffer();
    if (inPlace && !sb.ChunkContaining(targetValue.data(), total, &chunkSize))
        inPlace = false;
    char* begin;
    if (inPlace) {
        begin = const_cast<char*>(targetValue.data());
    } else {
        StringBuffer b = sb.AllocateStringBuffer(total);
        begin = b.data;
        memcpy(begin, targetValue.data(), targetValue.size());
    }
    char* w = begin + targetValue.size();
    for (size_t i = 1; i < logEvents.size(); ++i) {
        if (insertLineBreak)
            *w++ = '\n';
        StringView cur = logEvents[i]->GetContent(mSourceKey);
        memmove(w, cur.data(), cur.size());
        w += cur.size();
    }
    // the key view must outlive the call: reuse the stored key of the target's content
    StringView key;
    for (auto& c : target->RawContents())
        if (c.second && c.first.first == StringView(mSourceKey))
            key = c.first.first;
    target->SetContentNoCopy(key, StringView(begin, (size_t)(w - begin)));
    logEvents.clear();
}

// :348-385 (alarms / log lines are not produced by this engine)
void ProcessorMergeMultilineLogNative::HandleUnmatchLogs(EventsContainer& logEvents, size_t& newSize, size_t begin,
                                                         size_t end) {
    mUnmatchedEventsTotal.Add(end - begin + 1);
    if (mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD)
        return;
    for (size_t i = begin; i <= end; ++i)
        logEvents[newSize++] = std::move(logEvents[i]);
}

// :116-159.  A record is a run of parts: every part but the last carries the "P" content (the container runtime's
// partial-line marker); a part without it completes the run, and so does the end of the group.  The first part loses
// its marker, the joined value lands in the first part, and the output slot takes the event that FOLLOWS the previous
// record (an empty event there survives in place of the joined one -- the reference's behaviour, kept).
void ProcessorMergeMultilineLogNative::MergeLogsByFlag(PipelineEventGroup& group) {
    EventsContainer& all = group.MutableEvents();
    const size_t n = all.size();
    size_t kept = 0;  // events written back so far
    size_t head = 0;  // index right after the previous record
    bool open = false; // the previous part carried the marker
    std::vector<LogEvent*> parts;
    auto Complete = [&](size_t next) {
        MergeEvents(group, parts, false);
        all[kept++] = std::move(all[head]);
        head = next;
        open = false;
    };
    for (size_t cur = 0; cur < n; ++cur) {
        if (!IsSupportedEvent(all[cur])) {
            // ends the walk: the open run (or, without one, everything from here) is kept as it is
            if (parts.empty())
                head = cur;
            for (size_t i = head; i < n; ++i)
                all[kept++] = std::move(all[i]);
            all.resize(kept);
            return;
        }
        LogEvent* part = &all[cur].Cast<LogEvent>();
        if (part->Empty())
            continue;
        parts.push_back(part);
        const bool marked = part->HasContent(PartLogFlag);
        if (!marked) {
            Complete(cur + 1);
        } else if (!open) {
            part->DelContent(PartLogFlag);
            open = true;
        }
    }
    if (open)
        Complete(n);
    all.resize(kept);
}

// :161-318.  BoostRegexSearch(match_continuous) of every (event, pattern) pair is a pure function of the value, so all
// probes are evaluated up front on the GPU and the walk below only reads flags.
void ProcessorMergeMultilineLogNative::MergeLogsByRegex(PipelineEventGroup& group) {
    EventsContainer& sourceEvents = group.MutableEvents();
    const size_t ne = sourceEvents.size();
    std::vector<uint8_t> mS(ne, 0), mC(ne, 0), mE(ne, 0);
    {
        FlatBatch batch;
        for (size_t i = 0; i < ne; ++i) {
            if (!IsSupportedEvent(sourceEvents[i]))
                break; // the walk stops at the first unsupported event
            const LogEvent& ev = sourceEvents[i].Cast<LogEvent>();
            if (ev.Empty())
                continue;
            if (!ev.HasContent(mSourceKey))
                break;
            batch.Add(i, ev.GetContent(mSourceKey));
        }
        batch.Finish(*group.GetSourceBuffer());
        const size_t nb = batch.eventIndex.size();
        struct {
            bool has;
            CompiledRegex* reg;
            std::vector<uint8_t>* dst;
        } probes[] = {{mHasStart, &mStartReg, &mS}, {mHasContinue, &mContinueReg, &mC}, {mHasEnd, &mEndReg, &mE}};
        std::vector<uint8_t> m(nb);
        for (auto& p : probes) {
            if (!p.has || !nb)
                continue;
            Check(lc_regex_prefix_match(Engine(), p.reg->get(), batch.base, batch.baseLen, batch.off.data(),
                                        batch.len.data(), nb, m.data()),
                  "lc_regex_prefix_match");
            for (size_t b = 0; b < nb; ++b)
                (*p.dst)[batch.eventIndex[b]] = m[b];
        }
    }
    // The walk as a decision table: what a value does depends only on (which patterns exist, whether a record is
    // open, the three probe flags).  Decide() is that pure function; the loop below just executes its verdicts.
    enum class Act {
        OPEN,             // the value starts a record
        ALONE,            // continue + end mode, no record open, the value matches the end pattern: a record by itself
        UNMATCHED,        // no record open and nothing matches
        APPEND,           // joins the open record, which stays open
        APPEND_CLOSE,     // joins the open record and completes it
        APPEND_FAIL,      // joins the open record, which thereby fails as a whole (continue + end, end not matched)
        CLOSE_OPEN,       // the open record is complete WITHOUT this value, which starts the next one
        CLOSE_UNMATCHED,  // the open record is complete without this value, which matches nothing
    };
    const bool S = mHasStart, C = mHasContinue, E = mHasEnd;
    auto Decide = [S, C, E](bool open, bool mS, bool mC, bool mE) -> Act {
        if (!open) {
            if (S ? mS : mC)
                return Act::OPEN;
            return (!S && C && E && mE) ? Act::ALONE : Act::UNMATCHED;
        }
        if (C && mC)
            return Act::APPEND;
        if (E) {
            if (C)
                return mE ? Act::APPEND_CLOSE : Act::APPEND_FAIL;
            return mE ? Act::APPEND_CLOSE : Act::APPEND;
        }
        if (!C)
            return mS ? Act::CLOSE_OPEN : Act::APPEND;
        return mS ? Act::CLOSE_OPEN : Act::CLOSE_UNMATCHED;
    };
    size_t head = 0;  // index of the first event of the open record
    size_t kept = 0;  // events written back so far
    std::vector<LogEvent*> record;
    bool open = !S && !C && E; // with only an end pattern every value belongs to a record
    auto Complete = [&]() {   // the open record becomes one event (the head event carries the joined value)
        MergeEvents(group, record, true);
        sourceEvents[kept++] = std::move(sourceEvents[head]);
    };
    for (size_t cur = 0; cur < ne; ++cur) {
        LogEvent* ev = IsSupportedEvent(sourceEvents[cur]) ? &sourceEvents[cur].Cast<LogEvent>() : nullptr;
        if (ev && ev->Empty())
            continue;
        if (!ev || !ev->HasContent(mSourceKey)) {
            // an unsupported event or one without the source key ends the walk: everything from the head of the
            // open record (or from here) is kept as it is
            if (record.empty())
                head = cur;
            for (size_t i = head; i < ne; ++i)
                sourceEvents[kept++] = std::move(sourceEvents[i]);
            sourceEvents.resize(kept);
            return;
        }
        switch (Decide(open, mS[cur] != 0, mC[cur] != 0, mE[cur] != 0)) {
            case Act::OPEN:
                record.push_back(ev);
                head = cur;
                open = true;
                break;
            case Act::ALONE:
                mMergedEventsTotal.Add(1);
                sourceEvents[kept++] = std::move(sourceEvents[cur]);
                break;
            case Act::UNMATCHED:
                HandleUnmatchLogs(sourceEvents, kept, cur, cur);
                break;
            case Act::APPEND:
                record.push_back(ev);
                break;
            case Act::APPEND_CLOSE:
                record.push_back(ev);
                Complete();
                if (S || C)
                    open = false;
                else
                    head = cur + 1; // only an end pattern: the next record starts right away
                break;
            case Act::APPEND_FAIL:
                record.clear();
                HandleUnmatchLogs(sourceEvents, kept, head, cur);
                open = false;
                break;
            case Act::CLOSE_OPEN:
                Complete();
                head = cur;
                record.push_back(ev);
                break;
            case Act::CLOSE_UNMATCHED:
                Complete();
                HandleUnmatchLogs(sourceEvents, kept, cur, cur);
                open = false;
                break;
        }
    }
    // a record still open at the end of the group: complete when there is no end pattern to wait for, else unmatched
    if (open && head < ne) {
        if (!E)
            Complete();
        else
            HandleUnmatchLogs(sourceEvents, kept, head, ne - 1);
    }
    sourceEvents.resize(kept);
}

// ------------------------------------------------------------------------------------------------ SLS serialise
namespace {
void PutVarint(std::string& out, uint32_t v) {
    while (v >= 0x80u) {
        out.push_back((char)(v | 0x80u));
        v >>= 7;
    }
    out.push_back((char)v);
}
void PutString(std::string& out, StringView s) {
    PutVarint(out, (uint32_t)s.size());
    out.append(s.data(), s.size());
}

// group-level fields in tag (map) order, SLSSerializer.cpp:203-213,239-249
std::string SlsGroupTail(PipelineEventGroup& group) {
    std::string tail;
    for (auto& tag : group.GetTags()) {
        if (tag.first == StringView("__topic__")) {
            tail.push_back(0x1A);
            PutString(tail, tag.second);
        } else if (tag.first == StringView("__source__")) {
            tail.push_back(0x22);
            PutString(tail, tag.second);
        } else if (tag.first == StringView("__machine_uuid__")) {
            tail.push_back(0x2A);
            PutString(tail, tag.second);
        } else {
            std::string inner;
            inner.push_back(0x0A);
            PutString(inner, tag.first);
            inner.push_back(0x12);
            PutString(inner, tag.second);
            tail.push_back(0x32);
            PutVarint(tail, (uint32_t)inner.size());
            tail += inner;
        }
    }
    return tail;
}

std::string SizeLimitError(uint64_t size, int32_t limit) {
    return "log group exceeds size limit\tgroup size: " + ToString(size) + "\tsize limit: " + ToString((uint64_t)limit);
}

// ---- shared by the SerializeSls methods
// Whether every event is flat: a LogEvent whose only content is sourceKey -> line
bool IsFlatGroup(PipelineEventGroup& group, const std::string& sourceKey) {
    for (const PipelineEventPtr& e : group.GetEvents()) {
        if (!e.Is<LogEvent>())
            return false;
        const LogEvent& ev = e.Cast<LogEvent>();
        const LogEvent::Content* c = ev.FirstLive();
        if (!(ev.Size() == 1 && c && c->first.first == StringView(sourceKey)))
            return false;
    }
    return true;
}

// Whether the parse processors' one-pass device path applies: every event is flat and the group carries no
// log.file.offset metadata (ShouldEraseEvent keys off it, CommonParserOptions.cpp:99-117).
bool IsFlatSlsGroup(PipelineEventGroup& group, const std::string& sourceKey) {
    return !group.HasMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY) && IsFlatGroup(group, sourceKey);
}

// the lines of a flat group (batch, finished) and the times the serialiser writes
void GatherFlatSls(PipelineEventGroup& group, bool enableNs, FlatBatch& batch, std::vector<uint32_t>& evTime,
                   std::vector<uint32_t>& evNs) {
    const EventsContainer& events = group.GetEvents();
    const size_t n = events.size();
    evTime.assign(n, 0);
    evNs.assign(n, LC_SLS_NO_NS);
    for (size_t i = 0; i < n; ++i) {
        const LogEvent& ev = events[i].Cast<LogEvent>();
        batch.Add(i, ev.FirstLive()->first.second);
        evTime[i] = (uint32_t)ev.GetTimestamp();
        if (enableNs && ev.GetTimestampNanosecond())
            evNs[i] = ev.GetTimestampNanosecond().value();
    }
    batch.Finish(*group.GetSourceBuffer());
}

// The device pass of SerializeSls: call(out, cap, &need) parses and serialises the group into res, sized by
// `estimate` first and by the exact size when that was short (unless the group is over the size limit anyway).
template <class Call>
void RunSlsDevicePass(Call call, size_t estimate, size_t tailSize, int32_t limit, std::string& res, uint64_t& need,
                      const char* what) {
    res.assign(estimate, '\0');
    int rc = call(reinterpret_cast<uint8_t*>(&res[0]), (uint64_t)res.size(), &need);
    if (rc == LC_ERR_CAPACITY && (int64_t)(need + tailSize) <= (int64_t)limit) {
        res.resize(need);
        rc = call(reinterpret_cast<uint8_t*>(&res[0]), (uint64_t)res.size(), &need);
    }
    if (rc != LC_ERR_CAPACITY)
        Check(rc, what);
}

// SLSEventGroupSerializer::Serialize's checks, in its order, on the result of the device pass (n events in,
// `discarded` of them erased, need wire bytes of Logs records)
bool FinishSls(const SLSEventGroupSerializer& ser, uint64_t n, uint64_t discarded, uint64_t need, std::string& res,
               const std::string& tail, std::string& out, std::string& err) {
    if (n == discarded) {
        err = "empty event group";
        return false;
    }
    if (need == 0) {
        err = "all empty logs";
        return false;
    }
    if ((int64_t)(need + tail.size()) > (int64_t)ser.mMaxSendLogGroupSize) {
        err = SizeLimitError(need + tail.size(), ser.mMaxSendLogGroupSize);
        return false;
    }
    res.resize(need);
    out = res + tail;
    return true;
}

// SerializeSls's bytes as one LZ4 block (the path for groups the one-pass device call does not take)
bool CompressSls(bool ok, std::string& raw, std::string& block, uint64_t& rawSize, std::string& err) {
    if (!ok)
        return false;
    rawSize = raw.size();
    LZ4Compressor c;
    return c.Compress(raw, block, err);
}

// The fused device pass: call(out, cap, &blockLen, &raw) parses, serialises and compresses records ‖ tail, sized by
// `estimate` first and by the exact block size when that was short (unless the group is over the size limit anyway).
// Then SLSEventGroupSerializer::Serialize's checks, in its order, on the raw size.
template <class Call>
bool RunSlsLz4DevicePass(Call call, size_t estimate, const SLSEventGroupSerializer& ser, const uint64_t& n,
                         const uint64_t& discarded, size_t tailSize, std::string& block, uint64_t& rawSize,
                         std::string& err, const char* what) {
    uint64_t blen = 0, raw = 0;
    block.assign(estimate + estimate / 255 + 16, '\0');
    int rc = call(reinterpret_cast<uint8_t*>(&block[0]), (uint64_t)block.size(), &blen, &raw);
    if (rc == LC_ERR_CAPACITY && (int64_t)raw <= (int64_t)ser.mMaxSendLogGroupSize) {
        block.resize(blen);
        rc = call(reinterpret_cast<uint8_t*>(&block[0]), (uint64_t)block.size(), &blen, &raw);
    }
    if (rc != LC_ERR_CAPACITY)
        Check(rc, what);
    if (n == discarded) {
        err = "empty event group";
        return false;
    }
    if (raw == tailSize) {
        err = "all empty logs";
        return false;
    }
    if ((int64_t)raw > (int64_t)ser.mMaxSendLogGroupSize) {
        err = SizeLimitError(raw, ser.mMaxSendLogGroupSize);
        return false;
    }
    block.resize(blen);
    rawSize = raw;
    return true;
}

// The device path of the splitters' SerializeSls on a flat group: every source event's value is split and serialised
// by `call(val, key, okey, pos, time, ns, out, cap, &need, &nevents, ctr)` (lc_split_sls / lc_multiline_split_sls) and
// the records are concatenated in event order; counters[3] += the ctr of each source event's last call.  The records
// are what CreateNewEvent builds (ProcessorSplitLogStringNative.cpp:131-161): RAW events serialise as "content" ->
// piece; LOG events as SourceKey -> piece plus, with log.file.offset metadata, that key -> the piece's file offset.
// An empty value emits nothing.  counters[3..N) are a chained stage's as SplitRegexChainSls lays them out: counters[5]
// + counters[6] are the events it erased or a filter behind it removed.
template <size_t N, class Call>
bool SplitSerializeSls(PipelineEventGroup& group, bool enableNs, const std::string& sourceKey, bool raw, Call call,
                       const char* what, std::string& out, std::string& err, uint64_t (&counters)[N]) {
    SLSEventGroupSerializer ser;
    ser.mEnableTimestampNanosecond = enableNs;
    static const std::string kRawKey = "content"; // DEFAULT_CONTENT_KEY (SLSSerializer.cpp:366-374)
    const std::string& key = raw ? kRawKey : sourceKey;
    const bool hasOffset = !raw && group.HasMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY);
    StringView okey = hasOffset ? group.GetMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY) : StringView();
    if (hasOffset && !okey.data())
        okey = StringView(""); // an empty key is still a key: the C-ABI reads NULL as "no offset key"
    const std::string tail = SlsGroupTail(group);
    const int64_t limit = ser.mMaxSendLogGroupSize;
    std::string res, part;
    uint64_t total = 0, nEvents = 0;
    for (const PipelineEventPtr& e : group.GetEvents()) {
        const LogEvent& src = e.Cast<LogEvent>();
        const StringView val = src.FirstLive()->first.second;
        if (val.empty())
            continue;
        const uint32_t ns =
            enableNs && src.GetTimestampNanosecond() ? src.GetTimestampNanosecond().value() : LC_SLS_NO_NS;
        uint64_t need = 0, nev = 0, ctr[N];
        RunSlsDevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len) {
                memset(ctr, 0, sizeof ctr); // (a second, exactly sized call must not count the lines twice)
                return call(val, key, hasOffset ? &okey : nullptr, src.GetPosition().first,
                            (uint32_t)src.GetTimestamp(), ns, o, cap, len, &nev, ctr);
            },
            2 * val.size() + 4096, tail.size() + total, ser.mMaxSendLogGroupSize, part, need, what);
        if ((int64_t)(total + need + tail.size()) <= limit)
            res.append(part.data(), need);
        // (else the group is over the size limit: the sizes still add up for the error message)
        total += need;
        nEvents += nev;
        for (size_t k = 0; k < N; ++k)
            counters[k] += ctr[k];
    }
    return FinishSls(ser, nEvents, counters[5] + counters[6], total, res, tail, out, err);
}
} // namespace

// The regex stage of the split -> regex chain: a ProcessorParseRegexNative's configuration as the chain calls take it
// (SPLIT_REGEX_STAGE_ARGS), the host check of lc_split_regex_sls_setup, and the counters Process would move.
struct SplitRegexStage {
    ProcessorParseRegexNative& r;
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    const lc_regex_t* re;
    bool wholeLine;
    explicit SplitRegexStage(ProcessorParseRegexNative& next)
        : r(next), re(next.mIsWholeLineMode ? nullptr : next.mReg.get()), wholeLine(next.mIsWholeLineMode) {
        for (const auto& k : r.mKeys) {
            kp.push_back(k.data());
            kl.push_back((uint32_t)k.size());
        }
    }
    const std::string& Renamed() const { return r.mCommonParserOptions.mRenamedSourceKey; }
    const CommonParserOptions& Opt() const { return r.mCommonParserOptions; }
    // whether the chain's device calls take this stage behind a splitter reading sourceKey
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        if (r.mSourceKey != sourceKey)
            return false;
        std::vector<uint32_t> plan(3 * r.mKeys.size() + 24);
        LcSplitRegexSlsCfg c;
        return !lc_split_regex_sls_setup(kp.data(), kl.data(), (uint32_t)r.mKeys.size(), r.mSourceKey.data(),
                                         (uint32_t)r.mSourceKey.size(), Renamed().data(), (uint32_t)Renamed().size(),
                                         okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u,
                                         Opt().mKeepingSourceWhenParseFail, Opt().mKeepingSourceWhenParseSucceed,
                                         Opt().mCopingRawLog, wholeLine, 0, 0, 0, LC_SLS_NO_NS, &c, plan.data());
    }
    void Add(const uint64_t ctr[3]) const {
        r.mOutSuccessfulEventsTotal.Add(ctr[0]);
        r.mOutFailedEventsTotal.Add(ctr[1]);
        r.mDiscardedEventsTotal.Add(ctr[2]);
    }
    void Process(PipelineEventGroup& group) const { r.Process(group); }
};
#define SPLIT_REGEX_STAGE_ARGS(x)                                                                                      \
    (x).kp.data(), (x).kl.data(), (uint32_t)(x).kp.size(), (x).r.mSourceKey.data(), (uint32_t)(x).r.mSourceKey.size(), \
        (x).Renamed().data(), (uint32_t)(x).Renamed().size(), (x).Opt().mKeepingSourceWhenParseFail,                    \
        (x).Opt().mKeepingSourceWhenParseSucceed, (x).Opt().mCopingRawLog, (x).wholeLine

// The delimiter stage of the split -> delimiter chain: a ProcessorParseDelimiterNative's configuration as the chain
// calls take it (SPLIT_DELIM_STAGE_ARGS), the host checks of lc_delim_sls_setup + lc_split_delim_sls_link, and the
// counters Process would move.
struct SplitDelimStage {
    ProcessorParseDelimiterNative& d;
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    explicit SplitDelimStage(ProcessorParseDelimiterNative& next) : d(next) {
        for (const auto& k : d.mKeys) {
            kp.push_back(k.data());
            kl.push_back((uint32_t)k.size());
        }
    }
    const std::string& Renamed() const { return d.mCommonParserOptions.mRenamedSourceKey; }
    const CommonParserOptions& Opt() const { return d.mCommonParserOptions; }
    const uint8_t* Sep() const { return reinterpret_cast<const uint8_t*>(d.mSeparator.data()); }
    bool Extend() const {
        return d.mOverflowedFieldsTreatment == ProcessorParseDelimiterNative::OverflowedFieldsTreatment::EXTEND;
    }
    uint32_t MaxFields() const { return (uint32_t)d.mKeys.size() + 16; }
    // whether the chain's device calls take this stage behind a splitter reading sourceKey
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        if (!d.mDeviceSls || d.mSourceKey != sourceKey)
            return false;
        size_t keyBytes = d.mSourceKey.size() + Renamed().size() + 12;
        for (const auto& k : d.mKeys)
            keyBytes += k.size();
        std::vector<uint8_t> kb(keyBytes);
        std::vector<uint32_t> at(d.mKeys.size() + 4);
        LcDelimSlsCfg dc;
        LcSplitDelimSlsCfg c;
        return !lc_delim_sls_setup(Sep(), (uint32_t)d.mSeparator.size(), (uint8_t)d.mQuote, Extend(),
                                   d.mExtractingPartialFields, kp.data(), kl.data(), (uint32_t)kp.size(),
                                   d.mSourceKey.data(), (uint32_t)d.mSourceKey.size(), Renamed().data(),
                                   (uint32_t)Renamed().size(), Opt().mKeepingSourceWhenParseFail,
                                   Opt().mKeepingSourceWhenParseSucceed, Opt().mCopingRawLog, MaxFields(), &dc,
                                   kb.data(), at.data()) &&
               !lc_split_delim_sls_link(dc, kp.data(), kl.data(), d.mSourceKey.data(), (uint32_t)d.mSourceKey.size(),
                                        Renamed().data(), (uint32_t)Renamed().size(), okey ? okey->data() : nullptr,
                                        okey ? (uint32_t)okey->size() : 0u, 0, 0, LC_SLS_NO_NS, &c);
    }
    // the device calls' counters[4] (successful, failed, discarded, blank) as the chain driver takes a stage's:
    // successful, out_failed (a blank value counts as failed, :220-242), discarded, removed by a filter (none)
    static void Fold(const uint64_t c4[4], uint64_t rctr[4]) {
        rctr[0] = c4[0];
        rctr[1] = c4[1] + c4[3];
        rctr[2] = c4[2];
        rctr[3] = 0;
    }
    void Add(const uint64_t ctr[3]) const {
        d.mOutSuccessfulEventsTotal.Add(ctr[0]);
        d.mOutFailedEventsTotal.Add(ctr[1]);
        d.mDiscardedEventsTotal.Add(ctr[2]);
    }
    void Process(PipelineEventGroup& group) const { d.Process(group); }
};
#define SPLIT_DELIM_STAGE_ARGS(x)                                                                                      \
    (x).Sep(), (uint32_t)(x).d.mSeparator.size(), (uint8_t)(x).d.mQuote, (x).Extend(),                                 \
        (x).d.mExtractingPartialFields, (x).d.mAllowingShortenedFields, (x).MaxFields(), (x).kp.data(),             \
        (x).kl.data(), (uint32_t)(x).kp.size(), (x).d.mSourceKey.data(), (uint32_t)(x).d.mSourceKey.size(),           \
        (x).Renamed().data(), (uint32_t)(x).Renamed().size(), (x).Opt().mKeepingSourceWhenParseFail,                    \
        (x).Opt().mKeepingSourceWhenParseSucceed, (x).Opt().mCopingRawLog

// The delimiter and regex stages of the split -> delimiter -> regex chain: the delimiter stage as SplitDelimStage has
// it, the regex stage's configuration as the chain calls take it (SPLIT_DELIM_REGEX_STAGE_ARGS), the host checks of
// lc_delim_sls_setup + lc_regex_sls_setup + lc_split_delim_regex_sls_link, and the counters both Process calls would
// move.
struct SplitDelimRegexStage {
    SplitDelimStage d;
    ProcessorParseRegexNative& r;
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    const lc_regex_t* re;
    bool wholeLine;
    SplitDelimRegexStage(ProcessorParseDelimiterNative& delim, ProcessorParseRegexNative& regex)
        : d(delim), r(regex), re(regex.mIsWholeLineMode ? nullptr : regex.mReg.get()),
          wholeLine(regex.mIsWholeLineMode) {
        for (const auto& k : r.mKeys) {
            kp.push_back(k.data());
            kl.push_back((uint32_t)k.size());
        }
    }
    const std::string& Renamed() const { return r.mCommonParserOptions.mRenamedSourceKey; }
    const CommonParserOptions& Opt() const { return r.mCommonParserOptions; }
    // whether the chain's device calls take both stages behind a splitter reading sourceKey
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        const ProcessorParseDelimiterNative& p = d.d;
        if (!p.mDeviceSls || p.mSourceKey != sourceKey)
            return false;
        size_t keyBytes = p.mSourceKey.size() + d.Renamed().size() + 12;
        for (const auto& k : p.mKeys)
            keyBytes += k.size();
        std::vector<uint8_t> kb(keyBytes);
        std::vector<uint32_t> at(p.mKeys.size() + 4), plan(3 * r.mKeys.size() + 12);
        LcSplitDelimRegexSlsCfg c;
        memset(&c, 0, sizeof c);
        return !lc_delim_sls_setup(d.Sep(), (uint32_t)p.mSeparator.size(), (uint8_t)p.mQuote, d.Extend(),
                                   p.mExtractingPartialFields, d.kp.data(), d.kl.data(), (uint32_t)d.kp.size(),
                                   p.mSourceKey.data(), (uint32_t)p.mSourceKey.size(), d.Renamed().data(),
                                   (uint32_t)d.Renamed().size(), d.Opt().mKeepingSourceWhenParseFail,
                                   d.Opt().mKeepingSourceWhenParseSucceed, d.Opt().mCopingRawLog, d.MaxFields(),
                                   &c.r.d, kb.data(), at.data()) &&
               !lc_regex_sls_setup(kp.data(), kl.data(), (uint32_t)kp.size(), r.mSourceKey.data(),
                                   (uint32_t)r.mSourceKey.size(), Renamed().data(), (uint32_t)Renamed().size(),
                                   Opt().mKeepingSourceWhenParseFail, Opt().mKeepingSourceWhenParseSucceed,
                                   Opt().mCopingRawLog, wholeLine, 0, &c.r.x, plan.data()) &&
               !lc_split_delim_regex_sls_link(
                   d.kp.data(), d.kl.data(), p.mSourceKey.data(), (uint32_t)p.mSourceKey.size(), d.Renamed().data(),
                   (uint32_t)d.Renamed().size(), kp.data(), kl.data(), (uint32_t)kp.size(), r.mSourceKey.data(),
                   (uint32_t)r.mSourceKey.size(), Renamed().data(), (uint32_t)Renamed().size(),
                   Opt().mKeepingSourceWhenParseFail, Opt().mKeepingSourceWhenParseSucceed, Opt().mCopingRawLog,
                   wholeLine, okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, 0, 0, LC_SLS_NO_NS,
                   &c);
    }
    // the device calls' counters[8] as the chain driver takes a stage's: the delimiter's successful, out_failed (a
    // blank value counts as failed, :220-242) and discarded, the regex stage's discarded (so that [2] + [3] are the
    // events the chain erased), successful, out_failed and out_key_not_found
    static void Fold(const uint64_t c8[8], uint64_t rctr[8]) {
        const uint64_t f[8] = {c8[0], c8[1] + c8[3], c8[2], c8[7], c8[4], c8[5], c8[6], 0};
        memcpy(rctr, f, sizeof f);
    }
    void Add(const uint64_t ctr[7]) const {
        d.Add(ctr);
        r.mDiscardedEventsTotal.Add(ctr[3]);
        r.mOutSuccessfulEventsTotal.Add(ctr[4]);
        r.mOutFailedEventsTotal.Add(ctr[5]);
        r.mOutKeyNotFoundEventsTotal.Add(ctr[6]);
    }
    void Process(PipelineEventGroup& group) const {
        d.Process(group);
        r.Process(group);
    }
};
// the chain calls' arguments after the source value and the splitter's: allow_short, max_fields, then both stages'
#define SPLIT_DELIM_REGEX_STAGE_ARGS(x)                                                                                \
    (x).d.d.mAllowingShortenedFields, (x).d.MaxFields(), (x).d.Sep(), (uint32_t)(x).d.d.mSeparator.size(),             \
        (uint8_t)(x).d.d.mQuote, (x).d.Extend(), (x).d.d.mExtractingPartialFields, (x).d.kp.data(), (x).d.kl.data(),   \
        (uint32_t)(x).d.kp.size(), (x).d.d.mSourceKey.data(), (uint32_t)(x).d.d.mSourceKey.size(),                     \
        (x).d.Renamed().data(), (uint32_t)(x).d.Renamed().size(), (x).d.Opt().mKeepingSourceWhenParseFail,              \
        (x).d.Opt().mKeepingSourceWhenParseSucceed, (x).d.Opt().mCopingRawLog, (x).kp.data(), (x).kl.data(),          \
        (uint32_t)(x).kp.size(), (x).r.mSourceKey.data(), (uint32_t)(x).r.mSourceKey.size(), (x).Renamed().data(),     \
        (uint32_t)(x).Renamed().size(), (x).Opt().mKeepingSourceWhenParseFail,                                          \
        (x).Opt().mKeepingSourceWhenParseSucceed, (x).Opt().mCopingRawLog, (x).wholeLine

// The regex and timestamp stages of the split -> regex -> timestamp chain: the regex stage as SplitRegexStage has it,
// the timestamp stage's SourceKey, program, "now" and history discard as the chain calls take them
// (SPLIT_REGEX_TS_ARGS), and the counters both Process calls would move.  The device calls take a group of exactly
// one source event: the second-level cache would otherwise have to carry across calls.
struct SplitRegexTsStage {
    SplitRegexStage s;
    ProcessorParseTimestampNative& t;
    const PipelineEventGroup& group;
    int64_t now;
    SplitRegexTsStage(ProcessorParseRegexNative& regex, ProcessorParseTimestampNative& ts, const PipelineEventGroup& g)
        : s(regex), t(ts), group(g), now((int64_t)time(nullptr)) {}
    int32_t DiscardInterval() const { return t.mDiscardOldData ? t.mDiscardInterval : -1; }
    const lc_timestamp_t* Program() const { return t.mProgram; }
    // whether the chain's device calls take both stages behind a splitter reading sourceKey: lc_split_regex_sls_setup
    // and lc_split_regex_ts_setup over the key table the C-ABI builds
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        const ProcessorParseRegexNative& r = s.r;
        if (group.GetEvents().size() != 1 || !t.mProgram || r.mSourceKey != sourceKey)
            return false;
        std::vector<uint32_t> plan(3 * r.mKeys.size() + 24);
        LcSplitRegexSlsCfg c;
        const char* ok = okey ? okey->data() : nullptr;
        const uint32_t okl = okey ? (uint32_t)okey->size() : 0u;
        if (lc_split_regex_sls_setup(s.kp.data(), s.kl.data(), (uint32_t)r.mKeys.size(), r.mSourceKey.data(),
                                     (uint32_t)r.mSourceKey.size(), s.Renamed().data(), (uint32_t)s.Renamed().size(),
                                     ok, okl, s.Opt().mKeepingSourceWhenParseFail,
                                     s.Opt().mKeepingSourceWhenParseSucceed, s.Opt().mCopingRawLog, s.wholeLine, 0, 0,
                                     0, LC_SLS_NO_NS, &c, plan.data()))
            return false;
        std::vector<const char*> strings(s.kp.size() + LC_SPLIT_REGEX_SLS_NSTR);
        std::vector<uint32_t> lens(s.kp.size() + LC_SPLIT_REGEX_SLS_NSTR);
        lc_split_regex_sls_strings(s.kp.data(), s.kl.data(), (uint32_t)s.kp.size(), r.mSourceKey.data(),
                                   (uint32_t)r.mSourceKey.size(), s.Renamed().data(), (uint32_t)s.Renamed().size(), ok,
                                   okl, strings.data(), lens.data());
        LcSplitRegexTsCfg tc;
        return !lc_split_regex_ts_setup(c, plan.data(), strings.data(), lens.data(), t.mSourceKey.data(),
                                        (uint32_t)t.mSourceKey.size(), 0, &tc);
    }
    // the device calls' counters[8] (the regex stage's three, then the timestamp stage's key_not_found, out_failed,
    // history_failure, discarded, out_successful) as the chain driver takes a stage's: [2] + [3] = the events the
    // chain erased or discarded
    static void Fold(const uint64_t c8[8], uint64_t rctr[8]) {
        const uint64_t f[8] = {c8[0], c8[1], c8[2], c8[6], c8[3], c8[4], c8[5], c8[7]};
        memcpy(rctr, f, sizeof f);
    }
    void Add(const uint64_t ctr[8]) const {
        s.Add(ctr);
        t.mDiscardedEventsTotal.Add(ctr[3]);
        t.mOutKeyNotFoundEventsTotal.Add(ctr[4]);
        t.mOutFailedEventsTotal.Add(ctr[5]);
        t.mHistoryFailureTotal.Add(ctr[6]);
        t.mOutSuccessfulEventsTotal.Add(ctr[7]);
    }
    void Process(PipelineEventGroup& g) const {
        s.Process(g);
        t.Process(g);
    }
};
// the timestamp calls' arguments behind time_ns
#define SPLIT_REGEX_TS_ARGS(x)                                                                                         \
    (x).t.mSourceKey.data(), (uint32_t)(x).t.mSourceKey.size(), (x).Program(), (x).now, (x).DiscardInterval()

// The delimiter and timestamp stages of the split -> delimiter -> timestamp chain: the delimiter stage as
// SplitDelimStage has it, the timestamp stage's SourceKey, program, "now" and history discard as the chain calls take
// them (SPLIT_REGEX_TS_ARGS), and the counters both Process calls would move.  The device calls take a group of exactly
// one source event: the second-level cache would otherwise have to carry across calls.
struct SplitDelimTsStage {
    SplitDelimStage s;
    ProcessorParseTimestampNative& t;
    const PipelineEventGroup& group;
    int64_t now;
    SplitDelimTsStage(ProcessorParseDelimiterNative& delim, ProcessorParseTimestampNative& ts,
                      const PipelineEventGroup& g)
        : s(delim), t(ts), group(g), now((int64_t)time(nullptr)) {}
    int32_t DiscardInterval() const { return t.mDiscardOldData ? t.mDiscardInterval : -1; }
    const lc_timestamp_t* Program() const { return t.mProgram; }
    // whether the chain's device calls take both stages behind a splitter reading sourceKey: SplitDelimStage's checks
    // and lc_split_delim_ts_setup (which reads the key count and the overflow mode of the delimiter stage)
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        const ProcessorParseDelimiterNative& d = s.d;
        if (group.GetEvents().size() != 1 || !t.mProgram || !s.Accepts(sourceKey, okey))
            return false;
        LcSplitDelimSlsCfg c;
        memset(&c, 0, sizeof c);
        c.d.nkeys = (uint32_t)d.mKeys.size();
        c.d.mode = d.mExtractingPartialFields ? LC_DELIM_SLS_DISCARD
                                              : (s.Extend() ? LC_DELIM_SLS_EXTEND : LC_DELIM_SLS_KEEP);
        LcSplitDelimTsCfg tc;
        return !lc_split_delim_ts_setup(c, s.kp.data(), s.kl.data(), d.mSourceKey.data(),
                                        (uint32_t)d.mSourceKey.size(), s.Renamed().data(),
                                        (uint32_t)s.Renamed().size(), okey ? okey->data() : nullptr,
                                        okey ? (uint32_t)okey->size() : 0u, t.mSourceKey.data(),
                                        (uint32_t)t.mSourceKey.size(), 0, &tc);
    }
    // the device calls' counters[9] (the delimiter stage's successful, failed, discarded, blank, then the timestamp
    // stage's key_not_found, out_failed, history_failure, discarded, out_successful) as the chain driver takes a
    // stage's: successful, out_failed (a blank value counts as failed, :220-242), discarded, then the timestamp stage's
    // discarded (so that [2] + [3] are the events the chain erased or discarded), key_not_found, out_failed,
    // history_failure, out_successful
    static void Fold(const uint64_t c9[9], uint64_t rctr[8]) {
        const uint64_t f[8] = {c9[0], c9[1] + c9[3], c9[2], c9[7], c9[4], c9[5], c9[6], c9[8]};
        memcpy(rctr, f, sizeof f);
    }
    void Add(const uint64_t ctr[8]) const {
        s.Add(ctr);
        t.mDiscardedEventsTotal.Add(ctr[3]);
        t.mOutKeyNotFoundEventsTotal.Add(ctr[4]);
        t.mOutFailedEventsTotal.Add(ctr[5]);
        t.mHistoryFailureTotal.Add(ctr[6]);
        t.mOutSuccessfulEventsTotal.Add(ctr[7]);
    }
    void Process(PipelineEventGroup& g) const {
        s.Process(g);
        t.Process(g);
    }
};

namespace {
// The split -> parse chain of either splitter, with the parse stage x (SplitRegexStage, SplitDelimStage,
// SplitDelimRegexStage): `process(group)` is the splitter's Process; the device calls are sls(val, okey, pos, time, ns,
// out, cap, &len, &nev, rctr, sctr) and lz4(val, okey, pos, time, ns, tail, tailLen, out, cap, &len, &raw, &nev, rctr,
// sctr) (rctr[8] = the stage's counters as x.Add takes them, rctr[2] + rctr[3] = the events it erased or a filter
// behind it removed; sctr[3] = the splitter's).  filter (or
// nullptr): the filter behind the regex stage, whose rule the device calls take when filterOk.  sctr_total[3] += the
// splitter's counters of every device call.  rawSize null: out = the wire bytes; else out = their LZ4 block and
// *rawSize their size.
template <class Stage, class ProcessFn, class Sls, class Lz4>
bool SplitRegexChainSls(PipelineEventGroup& group, const Stage& x, ProcessorFilterNative* filter,
                        bool filterOk, const std::string& sourceKey, bool rawContent, bool enableNs, std::string& out,
                        uint64_t* rawSize, std::string& err, ProcessFn process, Sls sls, Lz4 lz4, const char* what,
                        const char* lzwhat, uint64_t sctrTotal[3]) {
    SLSEventGroupSerializer ser;
    ser.mEnableTimestampNanosecond = enableNs;
    const bool hasOffset = group.HasMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY);
    StringView okey = hasOffset ? group.GetMetadata(EventGroupMetaKey::LOG_FILE_OFFSET_KEY) : StringView();
    if (hasOffset && !okey.data())
        okey = StringView(""); // an empty key is still a key: the C-ABI reads NULL as "no offset key"
    const StringView* okp = hasOffset ? &okey : nullptr;
    if (rawContent || !IsFlatGroup(group, sourceKey) || !x.Accepts(sourceKey, okp) || (filter && !filterOk)) {
        process(group);
        x.Process(group);
        if (filter)
            filter->Process(group);
        if (!rawSize)
            return ser.Serialize(group, out, err);
        std::string raw;
        const bool ok = ser.Serialize(group, raw, err);
        return CompressSls(ok, raw, out, *rawSize, err);
    }
    const EventsContainer& events = group.GetEvents();
    if (rawSize && events.size() == 1 && !events[0].Cast<LogEvent>().FirstLive()->first.second.empty()) {
        // the reader's case: one chunk, split, parsed, serialised and compressed on the device
        const LogEvent& src = events[0].Cast<LogEvent>();
        const StringView val = src.FirstLive()->first.second;
        const uint32_t ns =
            enableNs && src.GetTimestampNanosecond() ? src.GetTimestampNanosecond().value() : LC_SLS_NO_NS;
        const std::string tail = SlsGroupTail(group);
        uint64_t nev = 0, gone = 0, rctr[8] = {0, 0, 0, 0, 0, 0, 0, 0}, sctr[3] = {0, 0, 0};
        const bool ok = RunSlsLz4DevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw) {
                memset(rctr, 0, sizeof rctr);
                memset(sctr, 0, sizeof sctr);
                const int rc = lz4(val, okp, src.GetPosition().first, (uint32_t)src.GetTimestamp(), ns,
                                   reinterpret_cast<const uint8_t*>(tail.data()), (uint64_t)tail.size(), o, cap, len,
                                   raw, &nev, rctr, sctr);
                gone = rctr[2] + rctr[3]; // erased by the stage or removed by the filter
                return rc;
            },
            2 * val.size() + 4096 + tail.size(), ser, nev, gone, tail.size(), out, *rawSize, err, lzwhat);
        x.Add(rctr);
        for (int k = 0; k < 3; ++k)
            sctrTotal[k] += sctr[k];
        return ok;
    }
    auto call = [&](StringView val, const std::string&, const StringView* ok, uint64_t pos, uint32_t time, uint32_t ns,
                    uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* ctr) {
        return sls(val, ok, pos, time, ns, o, cap, len, nev, ctr + 3, ctr);
    };
    uint64_t ctr[11] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    std::string raw;
    const bool ok = SplitSerializeSls(group, enableNs, sourceKey, false, call, what, rawSize ? raw : out, err, ctr);
    x.Add(ctr + 3);
    for (int k = 0; k < 3; ++k)
        sctrTotal[k] += ctr[k];
    return rawSize ? CompressSls(ok, raw, out, *rawSize, err) : ok;
}
} // namespace

bool SLSEventGroupSerializer::Serialize(PipelineEventGroup& group, std::string& res, std::string& errorMsg) const {
    const EventsContainer& events = group.GetEvents();
    if (events.empty()) {
        errorMsg = "empty event group";
        return false;
    }
    // the group's type is its first event's (SLSSerializer.cpp:254-269); metric / span groups are not built, and a
    // group mixing types is refused rather than read as the first event's type
    const bool raw = events[0].Is<RawEvent>();
    for (const PipelineEventPtr& e : events)
        if (!(raw ? e.Is<RawEvent>() : e.Is<LogEvent>())) {
            errorMsg = "unsupported event type in event group";
            return false;
        }
    // flatten the contents of every event into entry tables over the arena; a RAW event is the one content
    // "content" -> its content (SLSSerializer.cpp:366-374,515-528) and is never skipped as empty
    static const StringView kRawKey("content");
    const size_t n = events.size();
    std::vector<uint32_t> evTime(n), evNs(n, LC_SLS_NO_NS);
    std::vector<uint64_t> entBegin(n + 1, 0);
    std::vector<const char*> kPtr, vPtr;
    std::vector<uint32_t> kLen, vLen;
    for (size_t i = 0; i < n; ++i) {
        if (raw) {
            const RawEvent& e = events[i].Cast<RawEvent>();
            evTime[i] = (uint32_t)e.GetTimestamp();
            if (mEnableTimestampNanosecond && e.GetTimestampNanosecond())
                evNs[i] = e.GetTimestampNanosecond().value();
            kPtr.push_back(kRawKey.data());
            kLen.push_back((uint32_t)kRawKey.size());
            vPtr.push_back(e.GetContent().data());
            vLen.push_back((uint32_t)e.GetContent().size());
            entBegin[i + 1] = kPtr.size();
            continue;
        }
        const LogEvent& e = events[i].Cast<LogEvent>();
        evTime[i] = (uint32_t)e.GetTimestamp();
        if (mEnableTimestampNanosecond && e.GetTimestampNanosecond())
            evNs[i] = e.GetTimestampNanosecond().value();
        for (auto& c : e.RawContents()) {
            if (!c.second)
                continue;
            kPtr.push_back(c.first.first.data());
            kLen.push_back((uint32_t)c.first.first.size());
            vPtr.push_back(c.first.second.data());
            vLen.push_back((uint32_t)c.first.second.size());
        }
        entBegin[i + 1] = kPtr.size();
    }
    const size_t m = kPtr.size();
    if (m == 0) {
        errorMsg = "all empty logs";
        return false;
    }
    // one span of the arena if all keys and values live in the same chunk, else a packed copy
    const char* lo = kPtr[0];
    const char* hi = kPtr[0] + kLen[0];
    for (size_t k = 0; k < m; ++k) {
        lo = std::min(lo, std::min(kPtr[k], vPtr[k]));
        hi = std::max(hi, std::max(kPtr[k] + kLen[k], vPtr[k] + vLen[k]));
    }
    std::vector<uint32_t> kOff(m), vOff(m);
    std::vector<uint8_t> packed;
    const uint8_t* base;
    uint64_t baseLen;
    size_t chunkSize = 0;
    if ((uint64_t)(hi - lo) < 0xFFFFFFF0ull && group.GetSourceBuffer()->ChunkContaining(lo, (size_t)(hi - lo), &chunkSize)) {
        base = reinterpret_cast<const uint8_t*>(lo);
        baseLen = (uint64_t)(hi - lo);
        for (size_t k = 0; k < m; ++k) {
            kOff[k] = (uint32_t)(kPtr[k] - lo);
            vOff[k] = (uint32_t)(vPtr[k] - lo);
        }
    } else {
        size_t total = 0;
        for (size_t k = 0; k < m; ++k)
            total += (size_t)kLen[k] + vLen[k];
        packed.resize(total + 1);
        size_t at = 0;
        for (size_t k = 0; k < m; ++k) {
            kOff[k] = (uint32_t)at;
            memcpy(packed.data() + at, kPtr[k], kLen[k]);
            at += kLen[k];
            vOff[k] = (uint32_t)at;
            memcpy(packed.data() + at, vPtr[k], vLen[k]);
            at += vLen[k];
        }
        base = packed.data();
        baseLen = total;
    }
    const std::string tail = SlsGroupTail(group);
    uint64_t need = 0;
    int rc = lc_sls_serialize_logs(Engine(), base, baseLen, n, evTime.data(), evNs.data(), entBegin.data(), kOff.data(),
                                   kLen.data(), vOff.data(), vLen.data(), nullptr, 0, &need);
    if (rc != LC_OK && rc != LC_ERR_CAPACITY)
        Check(rc, "lc_sls_serialize_logs");
    if ((int64_t)(need + tail.size()) > (int64_t)mMaxSendLogGroupSize) {
        errorMsg = SizeLimitError(need + tail.size(), mMaxSendLogGroupSize);
        return false;
    }
    res.resize(need);
    Check(lc_sls_serialize_logs(Engine(), base, baseLen, n, evTime.data(), evNs.data(), entBegin.data(), kOff.data(),
                                kLen.data(), vOff.data(), vLen.data(), reinterpret_cast<uint8_t*>(&res[0]), need, &need),
          "lc_sls_serialize_logs");
    res += tail;
    return true;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out,
                                                 std::string& err) {
    if (!IsFlatGroup(group, mSourceKey)) {
        Process(group);
        SLSEventGroupSerializer ser;
        ser.mEnableTimestampNanosecond = enableNs;
        return ser.Serialize(group, out, err);
    }
    auto call = [&](StringView val, const std::string& key, const StringView* okey, uint64_t pos, uint32_t time,
                    uint32_t ns, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t*) {
        return lc_split_sls(Engine(), reinterpret_cast<const uint8_t*>(val.data()), val.size(), (uint8_t)mSplitChar,
                            key.data(), (uint32_t)key.size(), okey ? okey->data() : nullptr,
                            okey ? (uint32_t)okey->size() : 0u, pos, time, ns, o, cap, len, nev);
    };
    uint64_t unused[7] = {0, 0, 0, 0, 0, 0, 0};
    return SplitSerializeSls(group, enableNs, mSourceKey, mEnableRawContent, call, "lc_split_sls", out, err, unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out,
                                                          std::string& err) {
    if (!IsFlatGroup(group, mSourceKey)) {
        Process(group);
        SLSEventGroupSerializer ser;
        ser.mEnableTimestampNanosecond = enableNs;
        return ser.Serialize(group, out, err);
    }
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto call = [&](StringView val, const std::string& key, const StringView* okey, uint64_t pos, uint32_t time,
                    uint32_t ns, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* ctr) {
        return lc_multiline_split_sls(Engine(), reinterpret_cast<const uint8_t*>(val.data()), val.size(), mStart.get(),
                                      mContinue.get(), mEnd.get(), discard, key.data(), (uint32_t)key.size(),
                                      okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns,
                                      o, cap, len, nev, ctr);
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[7] = {0, 0, 0, 0, 0, 0, 0};
    const bool ok = SplitSerializeSls(group, enableNs, mSourceKey, mEnableRawContent, call, "lc_multiline_split_sls",
                                      out, err, ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                 bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, nullptr, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                    bool enableNs, std::string& block, uint64_t& rawSize,
                                                    std::string& err) {
    return ChainSerializeSls(group, next, nullptr, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                 ProcessorFilterNative& filter, bool enableNs, std::string& out,
                                                 std::string& err) {
    return ChainSerializeSls(group, next, &filter, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                    ProcessorFilterNative& filter, bool enableNs, std::string& block,
                                                    uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, &filter, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                      ProcessorFilterNative* filter, bool enableNs, std::string& out,
                                                      uint64_t* rawSize, std::string& err) {
    const SplitRegexStage x(next);
    lc_filter_desc_t fd{};
    const bool filterOk = filter && filter->DeviceFilter(&fd);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        const char* ok = okey ? okey->data() : nullptr;
        const uint32_t okl = okey ? (uint32_t)okey->size() : 0u;
        return filter ? lc_split_regex_filter_parse_sls(Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar,
                                                        SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, &fd, o, cap,
                                                        len, nev, rctr)
                      : lc_split_regex_parse_sls(Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar,
                                                 SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, o, cap, len, nev,
                                                 rctr);
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        const char* ok = okey ? okey->data() : nullptr;
        const uint32_t okl = okey ? (uint32_t)okey->size() : 0u;
        return filter ? lc_split_regex_filter_parse_sls_lz4(Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar,
                                                            SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, &fd,
                                                            tail, tailLen, o, cap, len, raw, nev, rctr)
                      : lc_split_regex_parse_sls_lz4(Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar,
                                                     SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, tail, tailLen,
                                                     o, cap, len, raw, nev, rctr);
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, filter, filterOk, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4,
        filter ? "lc_split_regex_filter_parse_sls" : "lc_split_regex_parse_sls",
        filter ? "lc_split_regex_filter_parse_sls_lz4" : "lc_split_regex_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                          bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, nullptr, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseRegexNative& next, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, nullptr, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                          ProcessorFilterNative& filter, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, &filter, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseRegexNative& next,
                                                             ProcessorFilterNative& filter, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, &filter, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseRegexNative& next,
                                                               ProcessorFilterNative* filter, bool enableNs,
                                                               std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitRegexStage x(next);
    lc_filter_desc_t fd{};
    const bool filterOk = filter && filter->DeviceFilter(&fd);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        const char* ok = okey ? okey->data() : nullptr;
        const uint32_t okl = okey ? (uint32_t)okey->size() : 0u;
        return filter ? lc_multiline_split_regex_filter_parse_sls(
                            Engine(), x.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
                            SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, &fd, o, cap, len, nev, rctr, sctr)
                      : lc_multiline_split_regex_parse_sls(Engine(), x.re, src(val), val.size(), mStart.get(),
                                                           mContinue.get(), mEnd.get(), discard,
                                                           SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, o, cap,
                                                           len, nev, rctr, sctr);
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        const char* ok = okey ? okey->data() : nullptr;
        const uint32_t okl = okey ? (uint32_t)okey->size() : 0u;
        return filter ? lc_multiline_split_regex_filter_parse_sls_lz4(
                            Engine(), x.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
                            SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, &fd, tail, tailLen, o, cap, len, raw,
                            nev, rctr, sctr)
                      : lc_multiline_split_regex_parse_sls_lz4(
                            Engine(), x.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
                            SPLIT_REGEX_STAGE_ARGS(x), ok, okl, pos, time, ns, tail, tailLen, o, cap, len, raw, nev,
                            rctr, sctr);
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, filter, filterOk, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4,
        filter ? "lc_multiline_split_regex_filter_parse_sls" : "lc_multiline_split_regex_parse_sls",
        filter ? "lc_multiline_split_regex_filter_parse_sls_lz4" : "lc_multiline_split_regex_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                 ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                 std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                    ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                    std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                      ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                      std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitRegexTsStage x(next, timestamp, group);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8];
        const int rc = lc_split_regex_timestamp_parse_sls(
            Engine(), x.s.re, src(val), val.size(), (uint8_t)mSplitChar, SPLIT_REGEX_STAGE_ARGS(x.s),
            okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns, SPLIT_REGEX_TS_ARGS(x),
            enableNs, o, cap, len, nev, c8);
        SplitRegexTsStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8];
        const int rc = lc_split_regex_timestamp_parse_sls_lz4(
            Engine(), x.s.re, src(val), val.size(), (uint8_t)mSplitChar, SPLIT_REGEX_STAGE_ARGS(x.s),
            okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns, SPLIT_REGEX_TS_ARGS(x),
            enableNs, tail, tailLen, o, cap, len, raw, nev, c8);
        SplitRegexTsStage::Fold(c8, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_regex_timestamp_parse_sls",
        "lc_split_regex_timestamp_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                          ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseRegexNative& next,
                                                             ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseRegexNative& next,
                                                               ProcessorParseTimestampNative& timestamp,
                                                               bool enableNs, std::string& out, uint64_t* rawSize,
                                                               std::string& err) {
    const SplitRegexTsStage x(next, timestamp, group);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8];
        const int rc = lc_multiline_split_regex_timestamp_parse_sls(
            Engine(), x.s.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_REGEX_STAGE_ARGS(x.s), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, SPLIT_REGEX_TS_ARGS(x), enableNs, o, cap, len, nev, c8, sctr);
        SplitRegexTsStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8];
        const int rc = lc_multiline_split_regex_timestamp_parse_sls_lz4(
            Engine(), x.s.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_REGEX_STAGE_ARGS(x.s), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, SPLIT_REGEX_TS_ARGS(x), enableNs, tail, tailLen, o, cap, len, raw, nev, c8, sctr);
        SplitRegexTsStage::Fold(c8, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_regex_timestamp_parse_sls",
        "lc_multiline_split_regex_timestamp_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                 bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                    bool enableNs, std::string& block, uint64_t& rawSize,
                                                    std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                      bool enableNs, std::string& out, uint64_t* rawSize,
                                                      std::string& err) {
    const SplitDelimStage x(next);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c4[4] = {0, 0, 0, 0};
        const int rc = lc_split_delim_parse_sls(Engine(), src(val), val.size(), (uint8_t)mSplitChar,
                                                SPLIT_DELIM_STAGE_ARGS(x), okey ? okey->data() : nullptr,
                                                okey ? (uint32_t)okey->size() : 0u, pos, time, ns, o, cap, len, nev,
                                                c4);
        SplitDelimStage::Fold(c4, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c4[4] = {0, 0, 0, 0};
        const int rc = lc_split_delim_parse_sls_lz4(Engine(), src(val), val.size(), (uint8_t)mSplitChar,
                                                    SPLIT_DELIM_STAGE_ARGS(x), okey ? okey->data() : nullptr,
                                                    okey ? (uint32_t)okey->size() : 0u, pos, time, ns, tail, tailLen,
                                                    o, cap, len, raw, nev, c4);
        SplitDelimStage::Fold(c4, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_delim_parse_sls",
        "lc_split_delim_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group,
                                                          ProcessorParseDelimiterNative& next, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseDelimiterNative& next, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseDelimiterNative& next, bool enableNs,
                                                               std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitDelimStage x(next);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c4[4] = {0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_parse_sls(
            Engine(), src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_STAGE_ARGS(x), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, o, cap, len, nev, c4, sctr);
        SplitDelimStage::Fold(c4, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c4[4] = {0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_parse_sls_lz4(
            Engine(), src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_STAGE_ARGS(x), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, tail, tailLen, o, cap, len, raw, nev, c4, sctr);
        SplitDelimStage::Fold(c4, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_delim_parse_sls",
        "lc_multiline_split_delim_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                 ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                 std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                    ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                    std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                      ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                      std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitDelimTsStage x(next, timestamp, group);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_delim_timestamp_parse_sls(
            Engine(), src(val), val.size(), (uint8_t)mSplitChar, SPLIT_DELIM_STAGE_ARGS(x.s),
            okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns, SPLIT_REGEX_TS_ARGS(x),
            enableNs, o, cap, len, nev, c9);
        SplitDelimTsStage::Fold(c9, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_delim_timestamp_parse_sls_lz4(
            Engine(), src(val), val.size(), (uint8_t)mSplitChar, SPLIT_DELIM_STAGE_ARGS(x.s),
            okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns, SPLIT_REGEX_TS_ARGS(x),
            enableNs, tail, tailLen, o, cap, len, raw, nev, c9);
        SplitDelimTsStage::Fold(c9, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_delim_timestamp_parse_sls",
        "lc_split_delim_timestamp_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group,
                                                          ProcessorParseDelimiterNative& next,
                                                          ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseDelimiterNative& next,
                                                             ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseDelimiterNative& next,
                                                               ProcessorParseTimestampNative& timestamp,
                                                               bool enableNs, std::string& out, uint64_t* rawSize,
                                                               std::string& err) {
    const SplitDelimTsStage x(next, timestamp, group);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_timestamp_parse_sls(
            Engine(), src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_STAGE_ARGS(x.s), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, SPLIT_REGEX_TS_ARGS(x), enableNs, o, cap, len, nev, c9, sctr);
        SplitDelimTsStage::Fold(c9, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c9[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_timestamp_parse_sls_lz4(
            Engine(), src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_STAGE_ARGS(x.s), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time,
            ns, SPLIT_REGEX_TS_ARGS(x), enableNs, tail, tailLen, o, cap, len, raw, nev, c9, sctr);
        SplitDelimTsStage::Fold(c9, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_delim_timestamp_parse_sls",
        "lc_multiline_split_delim_timestamp_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                 ProcessorParseRegexNative& regex, bool enableNs, std::string& out,
                                                 std::string& err) {
    return ChainSerializeSls(group, next, regex, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                    ProcessorParseRegexNative& regex, bool enableNs,
                                                    std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, regex, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseDelimiterNative& next,
                                                      ProcessorParseRegexNative& regex, bool enableNs,
                                                      std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitDelimRegexStage x(next, regex);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_delim_regex_parse_sls(Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar,
                                                      SPLIT_DELIM_REGEX_STAGE_ARGS(x), okey ? okey->data() : nullptr,
                                                      okey ? (uint32_t)okey->size() : 0u, pos, time, ns, o, cap, len,
                                                      nev, c8);
        SplitDelimRegexStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_delim_regex_parse_sls_lz4(
            Engine(), x.re, src(val), val.size(), (uint8_t)mSplitChar, SPLIT_DELIM_REGEX_STAGE_ARGS(x),
            okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos, time, ns, tail, tailLen, o, cap,
            len, raw, nev, c8);
        SplitDelimRegexStage::Fold(c8, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_delim_regex_parse_sls",
        "lc_split_delim_regex_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group,
                                                          ProcessorParseDelimiterNative& next,
                                                          ProcessorParseRegexNative& regex, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, regex, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseDelimiterNative& next,
                                                             ProcessorParseRegexNative& regex, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, regex, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseDelimiterNative& next,
                                                               ProcessorParseRegexNative& regex, bool enableNs,
                                                               std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitDelimRegexStage x(next, regex);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_regex_parse_sls(
            Engine(), x.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_REGEX_STAGE_ARGS(x), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos,
            time, ns, o, cap, len, nev, c8, sctr);
        SplitDelimRegexStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_delim_regex_parse_sls_lz4(
            Engine(), x.re, src(val), val.size(), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_DELIM_REGEX_STAGE_ARGS(x), okey ? okey->data() : nullptr, okey ? (uint32_t)okey->size() : 0u, pos,
            time, ns, tail, tailLen, o, cap, len, raw, nev, c8, sctr);
        SplitDelimRegexStage::Fold(c8, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_delim_regex_parse_sls",
        "lc_multiline_split_delim_regex_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

bool ProcessorParseDelimiterNative::SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out,
                                                 std::string& err) {
    return SerializeSlsImpl(group, enableNs, out, nullptr, err);
}

bool ProcessorParseDelimiterNative::SerializeSlsLz4(PipelineEventGroup& group, bool enableNs, std::string& block,
                                                    uint64_t& rawSize, std::string& err) {
    return SerializeSlsImpl(group, enableNs, block, &rawSize, err);
}

// out = the wire bytes (rawSize null) or their LZ4 block (rawSize = their size)
bool ProcessorParseDelimiterNative::SerializeSlsImpl(PipelineEventGroup& group, bool enableNs, std::string& out,
                                                     uint64_t* rawSize, std::string& err) {
    SLSEventGroupSerializer ser;
    ser.mEnableTimestampNanosecond = enableNs;
    if (!mDeviceSls || !IsFlatSlsGroup(group, mSourceKey)) {
        Process(group);
        if (!rawSize)
            return ser.Serialize(group, out, err);
        std::string raw;
        const bool ok = ser.Serialize(group, raw, err);
        return CompressSls(ok, raw, out, *rawSize, err);
    }
    // every event is SourceKey -> line: parse and serialise in one device pass, only the wire bytes come back
    const size_t n = group.GetEvents().size();
    FlatBatch batch;
    std::vector<uint32_t> evTime, evNs;
    GatherFlatSls(group, enableNs, batch, evTime, evNs);
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    size_t keyBytes = 0;
    for (const auto& k : mKeys) {
        kp.push_back(k.data());
        kl.push_back((uint32_t)k.size());
        keyBytes += k.size();
    }
    const std::string& renamed = mCommonParserOptions.mRenamedSourceKey;
    std::string res;
    uint64_t need = 0, ctr[4] = {0, 0, 0, 0};
    const std::string tail = SlsGroupTail(group);
    const size_t estimate = (size_t)(2 * batch.baseLen + n * (64 + keyBytes + renamed.size()) + 64);
    // the arguments both device calls share, up to copy_raw
    auto args = [&](auto fn, auto... rest) {
        return fn(Engine(), batch.base, batch.baseLen, batch.off.data(), batch.len.data(), n, evTime.data(),
                  evNs.data(), reinterpret_cast<const uint8_t*>(mSeparator.data()), (uint32_t)mSeparator.size(),
                  (uint8_t)mQuote, mOverflowedFieldsTreatment == OverflowedFieldsTreatment::EXTEND,
                  mExtractingPartialFields, mAllowingShortenedFields, (uint32_t)mKeys.size() + 16, kp.data(), kl.data(),
                  (uint32_t)mKeys.size(), mSourceKey.data(), (uint32_t)mSourceKey.size(), renamed.data(),
                  (uint32_t)renamed.size(), mCommonParserOptions.mKeepingSourceWhenParseFail,
                  mCommonParserOptions.mKeepingSourceWhenParseSucceed, mCommonParserOptions.mCopingRawLog, rest...);
    };
    bool ok;
    if (rawSize) {
        ok = RunSlsLz4DevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw) {
                return args(lc_delim_parse_sls_lz4, reinterpret_cast<const uint8_t*>(tail.data()),
                            (uint64_t)tail.size(), o, cap, len, raw, ctr);
            },
            estimate + tail.size(), ser, n, ctr[2], tail.size(), out, *rawSize, err, "lc_delim_parse_sls_lz4");
    } else {
        RunSlsDevicePass([&](uint8_t* o, uint64_t cap, uint64_t* len) { return args(lc_delim_parse_sls, o, cap, len, ctr); },
                         estimate, tail.size(), ser.mMaxSendLogGroupSize, res, need, "lc_delim_parse_sls");
    }
    // the counters Process would have moved (a blank value counts as out_failed, :220-242)
    mOutSuccessfulEventsTotal.Add(ctr[0]);
    mOutFailedEventsTotal.Add(ctr[1] + ctr[3]);
    mDiscardedEventsTotal.Add(ctr[2]);
    return rawSize ? ok : FinishSls(ser, n, ctr[2], need, res, tail, out, err);
}

bool ProcessorParseDelimiterNative::SerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                 bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorParseDelimiterNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                    bool enableNs, std::string& block, uint64_t& rawSize,
                                                    std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

// out = the wire bytes (rawSize null) or their LZ4 block (rawSize = their size)
bool ProcessorParseDelimiterNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseRegexNative& next,
                                                      bool enableNs, std::string& out, uint64_t* rawSize,
                                                      std::string& err) {
    SLSEventGroupSerializer ser;
    ser.mEnableTimestampNanosecond = enableNs;
    std::vector<const char*> kp, rkp;
    std::vector<uint32_t> kl, rkl;
    size_t keyBytes = 0;
    for (const auto& k : mKeys) {
        kp.push_back(k.data());
        kl.push_back((uint32_t)k.size());
        keyBytes += k.size();
    }
    for (const auto& k : next.mKeys) {
        rkp.push_back(k.data());
        rkl.push_back((uint32_t)k.size());
        keyBytes += k.size();
    }
    const std::string& renamed = mCommonParserOptions.mRenamedSourceKey;
    const std::string& rrenamed = next.mCommonParserOptions.mRenamedSourceKey;
    const CommonParserOptions& ro = next.mCommonParserOptions;
    // the chain's own checks (lc_delim_regex_sls_link), on top of this processor's (mDeviceSls)
    bool accepted = false;
    if (mDeviceSls) {
        std::vector<uint8_t> kb(keyBytes + mSourceKey.size() + renamed.size() + 12);
        std::vector<uint32_t> at(mKeys.size() + 4), plan(3 * next.mKeys.size() + 12);
        LcDelimRegexSlsCfg c;
        accepted =
            !lc_delim_sls_setup(reinterpret_cast<const uint8_t*>(mSeparator.data()), (uint32_t)mSeparator.size(),
                                (uint8_t)mQuote, mOverflowedFieldsTreatment == OverflowedFieldsTreatment::EXTEND,
                                mExtractingPartialFields, kp.data(), kl.data(), (uint32_t)mKeys.size(),
                                mSourceKey.data(), (uint32_t)mSourceKey.size(), renamed.data(),
                                (uint32_t)renamed.size(), mCommonParserOptions.mKeepingSourceWhenParseFail,
                                mCommonParserOptions.mKeepingSourceWhenParseSucceed,
                                mCommonParserOptions.mCopingRawLog, (uint32_t)mKeys.size() + 16, &c.d, kb.data(),
                                at.data()) &&
            !lc_regex_sls_setup(rkp.data(), rkl.data(), (uint32_t)next.mKeys.size(), next.mSourceKey.data(),
                                (uint32_t)next.mSourceKey.size(), rrenamed.data(), (uint32_t)rrenamed.size(),
                                ro.mKeepingSourceWhenParseFail, ro.mKeepingSourceWhenParseSucceed, ro.mCopingRawLog,
                                next.mIsWholeLineMode, 0, &c.x, plan.data()) &&
            !lc_delim_regex_sls_link(c.d, kp.data(), kl.data(), mSourceKey.data(), (uint32_t)mSourceKey.size(),
                                     renamed.data(), (uint32_t)renamed.size(), rkp.data(), rkl.data(),
                                     (uint32_t)next.mKeys.size(), next.mSourceKey.data(),
                                     (uint32_t)next.mSourceKey.size(), rrenamed.data(), (uint32_t)rrenamed.size(),
                                     ro.mKeepingSourceWhenParseFail, ro.mKeepingSourceWhenParseSucceed,
                                     ro.mCopingRawLog, next.mIsWholeLineMode, &c);
    }
    if (!accepted || !IsFlatSlsGroup(group, mSourceKey)) {
        Process(group);
        next.Process(group);
        if (!rawSize)
            return ser.Serialize(group, out, err);
        std::string raw;
        const bool ok = ser.Serialize(group, raw, err);
        return CompressSls(ok, raw, out, *rawSize, err);
    }
    // every event is SourceKey -> line: both stages and the serialiser in one device pass
    const size_t n = group.GetEvents().size();
    FlatBatch batch;
    std::vector<uint32_t> evTime, evNs;
    GatherFlatSls(group, enableNs, batch, evTime, evNs);
    std::string res;
    uint64_t need = 0, ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const std::string tail = SlsGroupTail(group);
    const size_t estimate =
        (size_t)(2 * batch.baseLen + n * (64 + keyBytes + renamed.size() + rrenamed.size()) + 64);
    // the arguments both device calls share, up to whole_line
    auto args = [&](auto fn, auto... rest) {
        return fn(Engine(), next.mIsWholeLineMode ? nullptr : next.mReg.get(), batch.base, batch.baseLen,
                  batch.off.data(), batch.len.data(), n, evTime.data(), evNs.data(), mAllowingShortenedFields,
                  (uint32_t)mKeys.size() + 16, reinterpret_cast<const uint8_t*>(mSeparator.data()),
                  (uint32_t)mSeparator.size(), (uint8_t)mQuote,
                  mOverflowedFieldsTreatment == OverflowedFieldsTreatment::EXTEND, mExtractingPartialFields,
                  kp.data(), kl.data(), (uint32_t)mKeys.size(), mSourceKey.data(), (uint32_t)mSourceKey.size(),
                  renamed.data(), (uint32_t)renamed.size(), mCommonParserOptions.mKeepingSourceWhenParseFail,
                  mCommonParserOptions.mKeepingSourceWhenParseSucceed, mCommonParserOptions.mCopingRawLog,
                  rkp.data(), rkl.data(), (uint32_t)next.mKeys.size(), next.mSourceKey.data(),
                  (uint32_t)next.mSourceKey.size(), rrenamed.data(), (uint32_t)rrenamed.size(),
                  ro.mKeepingSourceWhenParseFail, ro.mKeepingSourceWhenParseSucceed, ro.mCopingRawLog,
                  next.mIsWholeLineMode, rest...);
    };
    uint64_t erased = 0; // events either stage erased
    bool ok;
    if (rawSize) {
        ok = RunSlsLz4DevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw) {
                const int rc = args(lc_delim_regex_parse_sls_lz4, reinterpret_cast<const uint8_t*>(tail.data()),
                                    (uint64_t)tail.size(), o, cap, len, raw, ctr);
                erased = ctr[2] + ctr[7];
                return rc;
            },
            estimate + tail.size(), ser, n, erased, tail.size(), out, *rawSize, err, "lc_delim_regex_parse_sls_lz4");
    } else {
        RunSlsDevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len) { return args(lc_delim_regex_parse_sls, o, cap, len, ctr); },
            estimate, tail.size(), ser.mMaxSendLogGroupSize, res, need, "lc_delim_regex_parse_sls");
        erased = ctr[2] + ctr[7];
    }
    // the counters both Process calls would have moved (a blank value counts as out_failed, :220-242)
    mOutSuccessfulEventsTotal.Add(ctr[0]);
    mOutFailedEventsTotal.Add(ctr[1] + ctr[3]);
    mDiscardedEventsTotal.Add(ctr[2]);
    next.mOutSuccessfulEventsTotal.Add(ctr[4]);
    next.mOutFailedEventsTotal.Add(ctr[5]);
    next.mOutKeyNotFoundEventsTotal.Add(ctr[6]);
    next.mDiscardedEventsTotal.Add(ctr[7]);
    return rawSize ? ok : FinishSls(ser, n, erased, need, res, tail, out, err);
}

bool ProcessorParseRegexNative::SerializeSls(PipelineEventGroup& group, bool enableNs, std::string& out,
                                             std::string& err) {
    return SerializeSlsImpl(group, enableNs, out, nullptr, err);
}

bool ProcessorParseRegexNative::SerializeSlsLz4(PipelineEventGroup& group, bool enableNs, std::string& block,
                                                uint64_t& rawSize, std::string& err) {
    return SerializeSlsImpl(group, enableNs, block, &rawSize, err);
}

// out = the wire bytes (rawSize null) or their LZ4 block (rawSize = their size)
bool ProcessorParseRegexNative::SerializeSlsImpl(PipelineEventGroup& group, bool enableNs, std::string& out,
                                                 uint64_t* rawSize, std::string& err) {
    SLSEventGroupSerializer ser;
    ser.mEnableTimestampNanosecond = enableNs;
    if (!IsFlatSlsGroup(group, mSourceKey)) {
        Process(group);
        if (!rawSize)
            return ser.Serialize(group, out, err);
        std::string raw;
        const bool ok = ser.Serialize(group, raw, err);
        return CompressSls(ok, raw, out, *rawSize, err);
    }
    // every event is SourceKey -> line: parse and serialise in one device pass, only the wire bytes come back
    const size_t n = group.GetEvents().size();
    FlatBatch batch;
    std::vector<uint32_t> evTime, evNs;
    GatherFlatSls(group, enableNs, batch, evTime, evNs);
    std::vector<const char*> kp;
    std::vector<uint32_t> kl;
    size_t keyBytes = 0;
    for (const auto& k : mKeys) {
        kp.push_back(k.data());
        kl.push_back((uint32_t)k.size());
        keyBytes += k.size();
    }
    const std::string& renamed = mCommonParserOptions.mRenamedSourceKey;
    std::string res;
    uint64_t need = 0, ctr[3] = {0, 0, 0};
    const std::string tail = SlsGroupTail(group);
    const size_t estimate = (size_t)(2 * batch.baseLen + n * (64 + keyBytes + renamed.size()) + 64);
    // the arguments both device calls share, up to whole_line
    auto args = [&](auto fn, auto... rest) {
        return fn(Engine(), mIsWholeLineMode ? nullptr : mReg.get(), batch.base, batch.baseLen, batch.off.data(),
                  batch.len.data(), n, evTime.data(), evNs.data(), kp.data(), kl.data(), (uint32_t)mKeys.size(),
                  mSourceKey.data(), (uint32_t)mSourceKey.size(), renamed.data(), (uint32_t)renamed.size(),
                  mCommonParserOptions.mKeepingSourceWhenParseFail,
                  mCommonParserOptions.mKeepingSourceWhenParseSucceed, mCommonParserOptions.mCopingRawLog,
                  mIsWholeLineMode, rest...);
    };
    bool ok;
    if (rawSize) {
        ok = RunSlsLz4DevicePass(
            [&](uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw) {
                return args(lc_regex_parse_sls_lz4, reinterpret_cast<const uint8_t*>(tail.data()),
                            (uint64_t)tail.size(), o, cap, len, raw, ctr);
            },
            estimate + tail.size(), ser, n, ctr[2], tail.size(), out, *rawSize, err, "lc_regex_parse_sls_lz4");
    } else {
        RunSlsDevicePass([&](uint8_t* o, uint64_t cap, uint64_t* len) { return args(lc_regex_parse_sls, o, cap, len, ctr); },
                         estimate, tail.size(), ser.mMaxSendLogGroupSize, res, need, "lc_regex_parse_sls");
    }
    // the counters Process would have moved (LC_REGEX_KEYS_MISMATCH is not out_failed, :227-244)
    mOutSuccessfulEventsTotal.Add(ctr[0]);
    mOutFailedEventsTotal.Add(ctr[1]);
    mDiscardedEventsTotal.Add(ctr[2]);
    return rawSize ? ok : FinishSls(ser, n, ctr[2], need, res, tail, out, err);
}

bool LZ4Compressor::Compress(const std::string& input, std::string& output, std::string& errorMsg) {
    std::vector<std::string> out;
    if (!Compress(std::vector<std::string>{input}, out, errorMsg))
        return false;
    output.swap(out[0]);
    return true;
}

bool LZ4Compressor::Compress(const std::vector<std::string>& inputs, std::vector<std::string>& outputs,
                             std::string& errorMsg) {
    std::vector<const uint8_t*> ptr;
    std::vector<uint32_t> len;
    uint64_t cap = 0;
    for (const std::string& in : inputs) {
        // LZ4_compressBound(n) is 0 for n > LZ4_MAX_INPUT_SIZE (lz4.h)
        if (in.size() > LC_LZ4_MAX_INPUT) {
            errorMsg = "input size is incorrect";
            return false;
        }
        ptr.push_back(reinterpret_cast<const uint8_t*>(in.data()));
        len.push_back((uint32_t)in.size());
        cap += lc_lz4_bound((uint32_t)in.size());
    }
    outputs.clear();
    if (inputs.empty())
        return true;
    std::string all(cap, '\0');
    std::vector<uint64_t> boff(inputs.size());
    std::vector<uint32_t> blen(inputs.size());
    uint64_t total = 0;
    Check(lc_lz4_compress(Engine(), inputs.size(), ptr.data(), len.data(), reinterpret_cast<uint8_t*>(&all[0]), cap,
                          boff.data(), blen.data(), &total),
          "lc_lz4_compress");
    outputs.reserve(inputs.size());
    for (size_t k = 0; k < inputs.size(); ++k)
        outputs.emplace_back(all, boff[k], blen[k]);
    return true;
}

bool ZstdCompressor::Compress(const std::string& input, std::string& output, std::string& errorMsg) {
    std::vector<std::string> out;
    if (!Compress(std::vector<std::string>{input}, out, errorMsg))
        return false;
    output.swap(out[0]);
    return true;
}

bool ZstdCompressor::Compress(const std::vector<std::string>& inputs, std::vector<std::string>& outputs,
                              std::string& errorMsg) {
    (void)mCompressionLevel;
    std::vector<const uint8_t*> ptr;
    std::vector<uint32_t> len;
    uint64_t cap = 0;
    for (const std::string& in : inputs) {
        // the device parse pass takes at most LZ4_MAX_INPUT_SIZE bytes per input; ZSTD_compress's message for an
        // input it cannot take
        if (in.size() > LC_LZ4_MAX_INPUT) {
            errorMsg = "Src size is incorrect";
            return false;
        }
        ptr.push_back(reinterpret_cast<const uint8_t*>(in.data()));
        len.push_back((uint32_t)in.size());
        cap += lc_zstd_bound(in.size());
    }
    outputs.clear();
    if (inputs.empty())
        return true;
    std::string all(cap, '\0');
    std::vector<uint64_t> foff(inputs.size());
    std::vector<uint32_t> flen(inputs.size());
    uint64_t total = 0;
    Check(lc_zstd_compress(Engine(), inputs.size(), ptr.data(), len.data(), reinterpret_cast<uint8_t*>(&all[0]), cap,
                           foff.data(), flen.data(), &total),
          "lc_zstd_compress");
    outputs.reserve(inputs.size());
    for (size_t k = 0; k < inputs.size(); ++k)
        outputs.emplace_back(all, foff[k], flen[k]);
    return true;
}

// ------------------------------------------------------------------------------------ ProcessorParseTimestampNative
const std::string ProcessorParseTimestampNative::sName = "processor_parse_timestamp_native";

namespace {

// ParseTimeZoneOffsetSecond (TimeUtil.cpp:372-391): "GMT+08:00" -> seconds east
bool ParseGmtOffset(const std::string& tz, int& sec) {
    if (tz.size() != 9 || tz[6] != ':' || (tz[3] != '+' && tz[3] != '-') || tz.compare(0, 3, "GMT") != 0)
        return false;
    auto num = [](const std::string& s, int& v) {
        if (s.empty() || !isdigit((unsigned char)s[0]))
            return false;
        v = 0;
        for (char c : s) {
            if (!isdigit((unsigned char)c))
                return false;
            v = v * 10 + (c - '0');
        }
        return true;
    };
    int h, m;
    if (!num(tz.substr(4, 2), h) || !num(tz.substr(7, 2), m))
        return false;
    sec = h * 3600 + m * 60;
    if (tz[3] == '-')
        sec = -sec;
    return true;
}

int LocalGmtOffset() { // GetLocalTimeZoneOffsetSecond (TimeUtil.cpp:72-79)
    time_t now = time(nullptr);
    struct tm t;
    memset(&t, 0, sizeof t);
    localtime_r(&now, &t);
    return (int)t.tm_gmtoff;
}

} // namespace

bool ProcessorParseTimestampNative::Init(const Json::Value& config) {
    mWarnings.clear();
    if (!GetString(config, "SourceKey", mSourceKey) || mSourceKey.empty())
        return Fail("mandatory string param SourceKey is missing");
    if (!GetString(config, "SourceFormat", mSourceFormat) || mSourceFormat.empty())
        return Fail("mandatory string param SourceFormat is missing");
    mLogTimeZoneOffsetSecond = 0;
    if (config.isMember("SourceTimezone") && !config["SourceTimezone"].isString()) {
        mWarnings.push_back("optional string param SourceTimezone is not of type string");
    } else if (GetString(config, "SourceTimezone", mSourceTimezone) && !mSourceTimezone.empty()) {
        int tz = 0;
        if (ParseGmtOffset(mSourceTimezone, tz))
            mLogTimeZoneOffsetSecond = tz - LocalGmtOffset();
        else
            mWarnings.push_back("string param SourceTimezone is not valid");
    }
    if (config.isMember("SourceYear")) {
        if (config["SourceYear"].isInt())
            mSourceYear = config["SourceYear"].asInt();
        else
            mWarnings.push_back("optional int param SourceYear is not of type int");
    }
    lc_timestamp_free(mProgram);
    mProgram = nullptr;
    if (lc_timestamp_compile(mSourceFormat.data(), mSourceFormat.size(), mSourceYear, mLogTimeZoneOffsetSecond,
                             &mProgram) != LC_OK)
        return Fail(std::string("string param SourceFormat is not supported: ") + lc_last_error());
    return true;
}

void ProcessorParseTimestampNative::Process(PipelineEventGroup& group) {
    std::vector<PipelineEventGroup> one;
    one.emplace_back(std::move(group));
    Process(one);
    group = std::move(one[0]);
}

void ProcessorParseTimestampNative::Process(std::vector<PipelineEventGroup>& groups) {
    if (!mProgram)
        return;
    // values of every group back to back, one event table, group starts
    std::string bytes;
    std::vector<uint32_t> off, len, grp{0};
    for (auto& g : groups) {
        for (PipelineEventPtr& e : g.MutableEvents()) {
            const LogEvent* ev = IsSupportedEvent(e) ? &e.Cast<LogEvent>() : nullptr;
            if (ev && ev->HasContent(mSourceKey)) {
                const StringView v = ev->GetContent(mSourceKey);
                off.push_back((uint32_t)bytes.size());
                len.push_back((uint32_t)v.size());
                bytes.append(v.data(), v.size());
            } else {
                off.push_back(0);
                len.push_back(LC_TS_NO_KEY);
            }
        }
        grp.push_back((uint32_t)off.size());
    }
    const uint64_t n = off.size();
    if (n == 0)
        return;
    std::vector<int64_t> sec(n);
    std::vector<uint32_t> nsec(n);
    std::vector<uint8_t> status(n);
    uint64_t cnt[5];
    try {
        Check(lc_timestamp_parse(Engine(), mProgram, reinterpret_cast<const uint8_t*>(bytes.data()), bytes.size(),
                                 off.data(), len.data(), n, grp.data(), groups.size(), (int64_t)time(nullptr),
                                 mDiscardOldData ? mDiscardInterval : -1, sec.data(), nsec.data(), status.data(), cnt),
              "lc_timestamp_parse");
    } catch (const std::exception& ex) {
        EngineFailed(ex.what());
        return;
    }
    uint64_t i = 0;
    uint64_t unsupported = 0;
    for (auto& g : groups) {
        EventsContainer& events = g.MutableEvents();
        size_t wIdx = 0;
        for (size_t rIdx = 0; rIdx < events.size(); ++rIdx, ++i) {
            if (!IsSupportedEvent(events[rIdx])) {
                unsupported++; // counted as key_not_found by the device: ProcessEvent counts it out_failed
            } else if (status[i] == LC_TS_DISCARDED) {
                continue;
            } else if (status[i] == LC_TS_OK) {
                events[rIdx].Cast<LogEvent>().SetTimestamp(sec[i], nsec[i]);
            }
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
        events.resize(wIdx);
    }
    mOutKeyNotFoundEventsTotal.Add(cnt[0] - unsupported);
    mOutFailedEventsTotal.Add(cnt[1] + unsupported);
    mHistoryFailureTotal.Add(cnt[2]);
    mDiscardedEventsTotal.Add(cnt[3]);
    mOutSuccessfulEventsTotal.Add(cnt[4]);
}

std::vector<std::pair<std::string, uint64_t>> ProcessorParseTimestampNative::Counters() const {
    return {{"discarded", mDiscardedEventsTotal.GetValue()},
            {"out_failed", mOutFailedEventsTotal.GetValue()},
            {"out_key_not_found", mOutKeyNotFoundEventsTotal.GetValue()},
            {"out_successful", mOutSuccessfulEventsTotal.GetValue()},
            {"history_failure", mHistoryFailureTotal.GetValue()}};
}

// ------------------------------------------------------------------------------------- ProcessorParseApsaraNative
const std::string ProcessorParseApsaraNative::sName = "processor_parse_apsara_native";

bool ProcessorParseApsaraNative::Init(const Json::Value& config) {
    mWarnings.clear();
    if (!GetString(config, "SourceKey", mSourceKey))
        return Fail("mandatory string param SourceKey is missing");
    mLogTimeZoneOffsetSecond = 0;
    mTimezone.clear();
    if (config.isMember("Timezone") && !config["Timezone"].isString()) {
        mWarnings.push_back("optional string param Timezone is not of type string");
    } else if (GetString(config, "Timezone", mTimezone) && !mTimezone.empty()) {
        int tz = 0;
        if (ParseGmtOffset(mTimezone, tz))
            mLogTimeZoneOffsetSecond = tz - LocalGmtOffset();
        else
            mWarnings.push_back("string param Timezone is not valid");
    }
    if (!mCommonParserOptions.Init(config))
        return false;
    lc_apsara_free(mProgram);
    mProgram = nullptr;
    if (lc_apsara_compile(mSourceKey.data(), mSourceKey.size(), mLogTimeZoneOffsetSecond, &mProgram) != LC_OK)
        return Fail(std::string("lc_apsara_compile: ") + lc_last_error());
    return true;
}

void ProcessorParseApsaraNative::Process(PipelineEventGroup& group) {
    std::vector<PipelineEventGroup> one;
    one.emplace_back(std::move(group));
    Process(one);
    group = std::move(one[0]);
}

void ProcessorParseApsaraNative::Process(std::vector<PipelineEventGroup>& groups) {
    static const std::string kKeys[4] = {"__LEVEL__", "__THREAD__", "__FILE__", "__LINE__"};
    static const std::string kMicro = "microtime";
    if (!mProgram)
        return;
    // values of every group back to back, one event table, group starts
    std::string bytes;
    std::vector<uint32_t> off, len, grp{0};
    for (auto& g : groups) {
        for (PipelineEventPtr& e : g.MutableEvents()) {
            const LogEvent* ev = IsSupportedEvent(e) ? &e.Cast<LogEvent>() : nullptr;
            if (ev && ev->HasContent(mSourceKey)) {
                const StringView v = ev->GetContent(mSourceKey);
                off.push_back((uint32_t)bytes.size());
                len.push_back((uint32_t)v.size());
                bytes.append(v.data(), v.size());
            } else {
                off.push_back(0);
                len.push_back(LC_TS_NO_KEY);
            }
        }
        grp.push_back((uint32_t)off.size());
    }
    const uint64_t n = off.size();
    if (n == 0)
        return;
    std::vector<int64_t> sec(n), micro(n);
    std::vector<uint32_t> nsec(n);
    std::vector<uint8_t> status(n);
    std::vector<uint64_t> first(n + 1);
    std::vector<lc_apsara_entry_t> ent(n * 8);
    uint64_t cnt[5], nent = 0;
    try {
        for (;;) {
            const int rc = lc_apsara_parse(Engine(), mProgram, reinterpret_cast<const uint8_t*>(bytes.data()),
                                           bytes.size(), off.data(), len.data(), n, grp.data(), groups.size(),
                                           (int64_t)time(nullptr), mDiscardOldData ? mDiscardInterval : -1,
                                           status.data(), sec.data(), nsec.data(), micro.data(), first.data(),
                                           ent.data(), ent.size(), &nent, cnt);
            if (rc != LC_ERR_CAPACITY) {
                Check(rc, "lc_apsara_parse");
                break;
            }
            ent.resize(nent);
        }
    } catch (const std::exception& ex) {
        EngineFailed(ex.what());
        return;
    }
    uint64_t i = 0, unsupported = 0, erased = 0;
    for (auto& g : groups) {
        EventsContainer& events = g.MutableEvents();
        SourceBuffer& sb = *g.GetSourceBuffer();
        const StringBuffer renamed = sb.CopyString(mCommonParserOptions.mRenamedSourceKey);
        const StringView rkey(renamed.data, renamed.size);
        auto addIfAbsent = [](LogEvent& ev, StringView k, StringView v) {
            if (!ev.HasContent(k))
                ev.AppendContentNoCopy(k, v);
        };
        size_t wIdx = 0;
        for (size_t rIdx = 0; rIdx < events.size(); ++rIdx, ++i) {
            const uint32_t st = status[i] & 7u;
            if (!IsSupportedEvent(events[rIdx])) {
                unsupported++; // counted as key_not_found by the device: ProcessEvent counts it out_failed
            } else if (st == LC_APSARA_DISCARDED) {
                continue;
            } else if (st == LC_APSARA_FAILED || st == LC_APSARA_OK) {
                LogEvent& ev = events[rIdx].Cast<LogEvent>();
                const StringView v = ev.GetContent(mSourceKey);
                const bool ok = st == LC_APSARA_OK;
                if (ok) {
                    ev.SetTimestamp(sec[i], nsec[i]);
                    for (uint64_t k = first[i]; k < first[i + 1]; ++k) {
                        const lc_apsara_entry_t& x = ent[k];
                        const StringView val(v.data() + (x.val_off - off[i]), x.val_len);
                        if (x.key_off >= LC_APSARA_KEY_LEVEL)
                            ev.AppendContentNoCopy(kKeys[x.key_off - LC_APSARA_KEY_LEVEL], val);
                        else
                            ev.AppendContentNoCopy(StringView(v.data() + (x.key_off - off[i]), x.key_len), val);
                    }
                    const StringBuffer us = sb.CopyString(std::to_string(micro[i]));
                    ev.AppendContentNoCopy(kMicro, StringView(us.data, us.size));
                    if (!(status[i] & LC_APSARA_OVERWRITTEN))
                        ev.DelContent(mSourceKey);
                    if (mCommonParserOptions.ShouldAddSourceContent(true))
                        addIfAbsent(ev, rkey, v);
                } else {
                    ev.DelContent(mSourceKey);
                    if (mCommonParserOptions.ShouldAddSourceContent(false))
                        addIfAbsent(ev, rkey, v);
                    if (mCommonParserOptions.ShouldAddLegacyUnmatchedRawLog(false))
                        addIfAbsent(ev, CommonParserOptions::legacyUnmatchedRawLogKey, v);
                    if (mCommonParserOptions.ShouldEraseEvent(false, ev, g.GetAllMetadata())) {
                        erased++;
                        continue;
                    }
                }
            }
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
        events.resize(wIdx);
    }
    mOutKeyNotFoundEventsTotal.Add(cnt[0] - unsupported);
    mOutFailedEventsTotal.Add(cnt[1] + unsupported);
    mHistoryFailureTotal.Add(cnt[2]);
    mDiscardedEventsTotal.Add(cnt[3] + erased);
    mOutSuccessfulEventsTotal.Add(cnt[4]);
}

std::vector<std::pair<std::string, uint64_t>> ProcessorParseApsaraNative::Counters() const {
    return {{"discarded", mDiscardedEventsTotal.GetValue()},
            {"out_failed", mOutFailedEventsTotal.GetValue()},
            {"out_key_not_found", mOutKeyNotFoundEventsTotal.GetValue()},
            {"out_successful", mOutSuccessfulEventsTotal.GetValue()},
            {"history_failure", mHistoryFailureTotal.GetValue()}};
}

// ------------------------------------------------------------------------------------- ProcessorParseJsonNative
const std::string ProcessorParseJsonNative::sName = "processor_parse_json_native";

bool ProcessorParseJsonNative::Init(const Json::Value& config) {
    if (!GetString(config, "SourceKey", mSourceKey))
        return Fail("mandatory string param SourceKey is missing");
    if (!mCommonParserOptions.Init(config))
        return false;
    lc_json_free(mProgram);
    mProgram = nullptr;
    if (lc_json_compile(mSourceKey.data(), mSourceKey.size(), &mProgram) != LC_OK)
        return Fail(std::string("lc_json_compile: ") + lc_last_error());
    return true;
}

void ProcessorParseJsonNative::Process(PipelineEventGroup& group) {
    std::vector<PipelineEventGroup> one;
    one.emplace_back(std::move(group));
    Process(one);
    group = std::move(one[0]);
}

void ProcessorParseJsonNative::Process(std::vector<PipelineEventGroup>& groups) {
    if (!mProgram)
        return;
    // one device call for all groups, cut only where the values would reach the call's 2 GiB limit (ProcessBatch
    // cuts again where the arena would)
    size_t g0 = 0;
    uint64_t bytes = 0;
    for (size_t g = 0; g < groups.size(); ++g) {
        uint64_t b = 0;
        for (PipelineEventPtr& e : groups[g].MutableEvents())
            if (IsSupportedEvent(e) && e.Cast<LogEvent>().HasContent(mSourceKey))
                b += e.Cast<LogEvent>().GetContent(mSourceKey).size();
        if (g > g0 && bytes + b >= LC_JSON_ARENA) {
            ProcessBatch(groups, g0, g);
            g0 = g;
            bytes = 0;
        }
        bytes += b;
    }
    if (g0 < groups.size())
        ProcessBatch(groups, g0, groups.size());
}

void ProcessorParseJsonNative::ProcessBatch(std::vector<PipelineEventGroup>& groups, size_t g0, size_t g1) {
    std::string bytes;
    std::vector<uint32_t> off, len;
    for (size_t g = g0; g < g1; ++g) {
        for (PipelineEventPtr& e : groups[g].MutableEvents()) {
            const LogEvent* ev = IsSupportedEvent(e) ? &e.Cast<LogEvent>() : nullptr;
            if (ev && ev->HasContent(mSourceKey)) {
                const StringView v = ev->GetContent(mSourceKey);
                off.push_back((uint32_t)bytes.size());
                len.push_back((uint32_t)v.size());
                bytes.append(v.data(), v.size());
            } else {
                off.push_back(0);
                len.push_back(LC_TS_NO_KEY);
            }
        }
    }
    const uint64_t n = off.size();
    if (n == 0)
        return;
    std::vector<uint8_t> status(n);
    std::vector<uint64_t> first(n + 1);
    std::vector<lc_json_entry_t> ent(n * 8);
    std::string arena(bytes.size() + 64, '\0');
    uint64_t cnt[3], nent = 0, narena = 0;
    try {
        for (;;) {
            const int rc = lc_json_parse(Engine(), mProgram, reinterpret_cast<const uint8_t*>(bytes.data()),
                                         bytes.size(), off.data(), len.data(), n, status.data(), first.data(),
                                         ent.data(), ent.size(), &nent, reinterpret_cast<uint8_t*>(&arena[0]),
                                         arena.size(), &narena, cnt);
            if (rc == LC_ERR_TOO_LARGE && g1 - g0 > 1) {
                // the renderings would reach the arena's 2 GiB (a "%f" can be 60 times its source): cut the batch
                const size_t mid = g0 + (g1 - g0) / 2;
                ProcessBatch(groups, g0, mid);
                ProcessBatch(groups, mid, g1);
                return;
            }
            if (rc != LC_ERR_CAPACITY) {
                Check(rc, "lc_json_parse");
                break;
            }
            ent.resize(nent > ent.size() ? nent : ent.size());
            arena.resize(narena > arena.size() ? narena : arena.size());
        }
    } catch (const std::exception& ex) {
        EngineFailed(ex.what());
        return;
    }
    uint64_t i = 0, unsupported = 0, erased = 0, kept = 0;
    for (size_t g = g0; g < g1; ++g) {
        EventsContainer& events = groups[g].MutableEvents();
        SourceBuffer& sb = *groups[g].GetSourceBuffer();
        const StringBuffer renamed = sb.CopyString(mCommonParserOptions.mRenamedSourceKey);
        const StringView rkey(renamed.data, renamed.size);
        auto addIfAbsent = [](LogEvent& ev, StringView k, StringView v) {
            if (!ev.HasContent(k))
                ev.AppendContentNoCopy(k, v);
        };
        size_t wIdx = 0;
        for (size_t rIdx = 0; rIdx < events.size(); ++rIdx, ++i) {
            const uint32_t st = status[i] & 0x7Fu;
            if (!IsSupportedEvent(events[rIdx])) {
                unsupported++; // counted as key_not_found by the device: ProcessEvent counts it out_failed
            } else if (st != LC_JSON_NOT_FOUND) {
                LogEvent& ev = events[rIdx].Cast<LogEvent>();
                const StringView v = ev.GetContent(mSourceKey);
                const bool ok = st == LC_JSON_OK;
                if (ok) {
                    auto view = [&](uint32_t o, uint32_t l) {
                        if (o & LC_JSON_ARENA) {
                            const StringBuffer b = sb.CopyString(arena.data() + (o & ~LC_JSON_ARENA), l);
                            return StringView(b.data, b.size);
                        }
                        return StringView(v.data() + (o - off[i]), l);
                    };
                    for (uint64_t k = first[i]; k < first[i + 1]; ++k) {
                        const lc_json_entry_t& x = ent[k];
                        ev.SetContentNoCopy(view(x.key_off, x.key_len), view(x.val_off, x.val_len));
                    }
                }
                if (!ok || !(status[i] & LC_JSON_OVERWRITTEN))
                    ev.DelContent(mSourceKey);
                if (mCommonParserOptions.ShouldAddSourceContent(ok))
                    addIfAbsent(ev, rkey, v);
                if (mCommonParserOptions.ShouldAddLegacyUnmatchedRawLog(ok))
                    addIfAbsent(ev, CommonParserOptions::legacyUnmatchedRawLogKey, v);
                if (mCommonParserOptions.ShouldEraseEvent(ok, ev, groups[g].GetAllMetadata())) {
                    erased++;
                    continue;
                }
                kept++;
            }
            if (wIdx != rIdx)
                events[wIdx] = std::move(events[rIdx]);
            ++wIdx;
        }
        events.resize(wIdx);
    }
    mOutKeyNotFoundEventsTotal.Add(cnt[0] - unsupported);
    mOutFailedEventsTotal.Add(cnt[1] + unsupported);
    mDiscardedEventsTotal.Add(erased);
    mOutSuccessfulEventsTotal.Add(kept);
}

std::vector<std::pair<std::string, uint64_t>> ProcessorParseJsonNative::Counters() const {
    return {{"discarded", mDiscardedEventsTotal.GetValue()},
            {"out_failed", mOutFailedEventsTotal.GetValue()},
            {"out_key_not_found", mOutKeyNotFoundEventsTotal.GetValue()},
            {"out_successful", mOutSuccessfulEventsTotal.GetValue()}};
}

Processor* CreateProcessor(const std::string& type) {
    if (type == ProcessorParseJsonNative::sName)
        return new ProcessorParseJsonNative;
    if (type == ProcessorParseApsaraNative::sName)
        return new ProcessorParseApsaraNative;
    if (type == ProcessorParseTimestampNative::sName)
        return new ProcessorParseTimestampNative;
    if (type == ProcessorMergeMultilineLogNative::sName)
        return new ProcessorMergeMultilineLogNative;
    if (type == ProcessorFilterNative::sName)
        return new ProcessorFilterNative;
    if (type == ProcessorSplitLogStringNative::sName)
        return new ProcessorSplitLogStringNative;
    if (type == ProcessorSplitMultilineLogStringNative::sName)
        return new ProcessorSplitMultilineLogStringNative;
    if (type == ProcessorParseRegexNative::sName)
        return new ProcessorParseRegexNative;
    if (type == ProcessorParseDelimiterNative::sName)
        return new ProcessorParseDelimiterNative;
    return nullptr;
}

// ------------------------------------------------------------------------------------------------ split -> JSON
// The JSON stage of the split -> JSON chain: a ProcessorParseJsonNative's configuration as the chain calls take it,
// the host check of lc_split_json_sls_setup, and the counters Process would move.
struct SplitJsonStage {
    ProcessorParseJsonNative& j;
    const std::string& Renamed() const { return j.mCommonParserOptions.mRenamedSourceKey; }
    const CommonParserOptions& Opt() const { return j.mCommonParserOptions; }
    const lc_json_t* Program() const { return j.mProgram; }
    // whether the chain's device calls take this stage behind a splitter reading sourceKey
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        LcSplitJsonSlsCfg c;
        return j.mProgram && j.mSourceKey == sourceKey &&
               !lc_split_json_sls_setup(j.mSourceKey.data(), (uint32_t)j.mSourceKey.size(), Renamed().data(),
                                        (uint32_t)Renamed().size(), okey ? okey->data() : nullptr,
                                        okey ? (uint32_t)okey->size() : 0u, Opt().mKeepingSourceWhenParseFail,
                                        Opt().mKeepingSourceWhenParseSucceed, Opt().mCopingRawLog, 0, 0, LC_SLS_NO_NS,
                                        &c);
    }
    // the device calls' counters[3] (successful, failed, discarded) as the chain driver takes a stage's, with none
    // removed by a filter
    static void Fold(const uint64_t c3[3], uint64_t rctr[4]) {
        rctr[0] = c3[0];
        rctr[1] = c3[1];
        rctr[2] = c3[2];
        rctr[3] = 0;
    }
    void Add(const uint64_t ctr[3]) const {
        j.mOutSuccessfulEventsTotal.Add(ctr[0]);
        j.mOutFailedEventsTotal.Add(ctr[1]);
        j.mDiscardedEventsTotal.Add(ctr[2]);
    }
    void Process(PipelineEventGroup& group) const { j.Process(group); }
};
#define SPLIT_JSON_STAGE_ARGS(x)                                                                                       \
    (x).Program(), src(val), val.size()
#define SPLIT_JSON_STAGE_OPTS(x)                                                                                       \
    (x).Renamed().data(), (uint32_t)(x).Renamed().size(), (x).Opt().mKeepingSourceWhenParseFail,                      \
        (x).Opt().mKeepingSourceWhenParseSucceed, (x).Opt().mCopingRawLog, okey ? okey->data() : nullptr,            \
        okey ? (uint32_t)okey->size() : 0u, pos, time, ns

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                 bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                    bool enableNs, std::string& block, uint64_t& rawSize,
                                                    std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                      bool enableNs, std::string& out, uint64_t* rawSize,
                                                      std::string& err) {
    const SplitJsonStage x{next};
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c3[3] = {0, 0, 0};
        const int rc = lc_split_json_parse_sls(Engine(), SPLIT_JSON_STAGE_ARGS(x), (uint8_t)mSplitChar,
                                               SPLIT_JSON_STAGE_OPTS(x), o, cap, len, nev, c3);
        SplitJsonStage::Fold(c3, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c3[3] = {0, 0, 0};
        const int rc = lc_split_json_parse_sls_lz4(Engine(), SPLIT_JSON_STAGE_ARGS(x), (uint8_t)mSplitChar,
                                                   SPLIT_JSON_STAGE_OPTS(x), tail, tailLen, o, cap, len, raw, nev,
                                                   c3);
        SplitJsonStage::Fold(c3, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_json_parse_sls", "lc_split_json_parse_sls_lz4",
        unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                          bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                             bool enableNs, std::string& block, uint64_t& rawSize,
                                                             std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseJsonNative& next, bool enableNs,
                                                               std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitJsonStage x{next};
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c3[3] = {0, 0, 0};
        const int rc = lc_multiline_split_json_parse_sls(Engine(), SPLIT_JSON_STAGE_ARGS(x), mStart.get(),
                                                         mContinue.get(), mEnd.get(), discard,
                                                         SPLIT_JSON_STAGE_OPTS(x), o, cap, len, nev, c3, sctr);
        SplitJsonStage::Fold(c3, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c3[3] = {0, 0, 0};
        const int rc = lc_multiline_split_json_parse_sls_lz4(Engine(), SPLIT_JSON_STAGE_ARGS(x), mStart.get(),
                                                             mContinue.get(), mEnd.get(), discard,
                                                             SPLIT_JSON_STAGE_OPTS(x), tail, tailLen, o, cap, len, raw,
                                                             nev, c3, sctr);
        SplitJsonStage::Fold(c3, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_json_parse_sls",
        "lc_multiline_split_json_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}

// The JSON and timestamp stages of the split -> JSON -> timestamp chain: the JSON stage as SplitJsonStage has it, the
// timestamp stage's SourceKey, program, "now" and history discard as the chain calls take them (SPLIT_JSON_TS_ARGS),
// and the counters both Process calls would move.  The device calls take a group of exactly one source event: the
// second-level cache would otherwise have to carry across calls.
struct SplitJsonTsStage {
    SplitJsonStage s;
    ProcessorParseTimestampNative& t;
    const PipelineEventGroup& group;
    int64_t now;
    SplitJsonTsStage(ProcessorParseJsonNative& json, ProcessorParseTimestampNative& ts, const PipelineEventGroup& g)
        : s{json}, t(ts), group(g), now((int64_t)time(nullptr)) {}
    int32_t DiscardInterval() const { return t.mDiscardOldData ? t.mDiscardInterval : -1; }
    const lc_timestamp_t* Program() const { return t.mProgram; }
    // whether the chain's device calls take both stages behind a splitter reading sourceKey: lc_split_json_sls_setup
    // and lc_split_json_ts_setup
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        const ProcessorParseJsonNative& j = s.j;
        if (group.GetEvents().size() != 1 || !t.mProgram || !s.Accepts(sourceKey, okey))
            return false;
        LcSplitJsonSlsCfg c;
        lc_split_json_sls_setup(j.mSourceKey.data(), (uint32_t)j.mSourceKey.size(), s.Renamed().data(),
                                (uint32_t)s.Renamed().size(), okey ? okey->data() : nullptr,
                                okey ? (uint32_t)okey->size() : 0u, s.Opt().mKeepingSourceWhenParseFail,
                                s.Opt().mKeepingSourceWhenParseSucceed, s.Opt().mCopingRawLog, 0, 0, LC_SLS_NO_NS, &c);
        LcSplitJsonTsCfg tc;
        return !lc_split_json_ts_setup(c, t.mSourceKey.data(), (uint32_t)t.mSourceKey.size(), 0, &tc);
    }
    // the device calls' counters[8] (the JSON stage's three, then the timestamp stage's key_not_found, out_failed,
    // history_failure, discarded, out_successful) as the chain driver takes a stage's: [2] + [3] = the events the
    // chain erased or discarded
    static void Fold(const uint64_t c8[8], uint64_t rctr[8]) {
        const uint64_t f[8] = {c8[0], c8[1], c8[2], c8[6], c8[3], c8[4], c8[5], c8[7]};
        memcpy(rctr, f, sizeof f);
    }
    void Add(const uint64_t ctr[8]) const {
        s.Add(ctr);
        t.mDiscardedEventsTotal.Add(ctr[3]);
        t.mOutKeyNotFoundEventsTotal.Add(ctr[4]);
        t.mOutFailedEventsTotal.Add(ctr[5]);
        t.mHistoryFailureTotal.Add(ctr[6]);
        t.mOutSuccessfulEventsTotal.Add(ctr[7]);
    }
    void Process(PipelineEventGroup& g) const {
        s.Process(g);
        t.Process(g);
    }
};
// the timestamp calls' arguments behind time_ns
#define SPLIT_JSON_TS_ARGS(x)                                                                                          \
    (x).t.mSourceKey.data(), (uint32_t)(x).t.mSourceKey.size(), (x).Program(), (x).now, (x).DiscardInterval()

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                 ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                 std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                    ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                    std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                      ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                      std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitJsonTsStage x(next, timestamp, group);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_json_timestamp_parse_sls(Engine(), SPLIT_JSON_STAGE_ARGS(x.s), (uint8_t)mSplitChar,
                                                         SPLIT_JSON_STAGE_OPTS(x.s), SPLIT_JSON_TS_ARGS(x), enableNs,
                                                         o, cap, len, nev, c8);
        SplitJsonTsStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_split_json_timestamp_parse_sls_lz4(
            Engine(), SPLIT_JSON_STAGE_ARGS(x.s), (uint8_t)mSplitChar, SPLIT_JSON_STAGE_OPTS(x.s),
            SPLIT_JSON_TS_ARGS(x), enableNs, tail, tailLen, o, cap, len, raw, nev, c8);
        SplitJsonTsStage::Fold(c8, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_json_timestamp_parse_sls",
        "lc_split_json_timestamp_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                          ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                          std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseJsonNative& next,
                                                             ProcessorParseTimestampNative& timestamp, bool enableNs,
                                                             std::string& block, uint64_t& rawSize, std::string& err) {
    return ChainSerializeSls(group, next, timestamp, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseJsonNative& next,
                                                               ProcessorParseTimestampNative& timestamp,
                                                               bool enableNs, std::string& out, uint64_t* rawSize,
                                                               std::string& err) {
    const SplitJsonTsStage x(next, timestamp, group);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_json_timestamp_parse_sls(
            Engine(), SPLIT_JSON_STAGE_ARGS(x.s), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_JSON_STAGE_OPTS(x.s), SPLIT_JSON_TS_ARGS(x), enableNs, o, cap, len, nev, c8, sctr);
        SplitJsonTsStage::Fold(c8, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_json_timestamp_parse_sls_lz4(
            Engine(), SPLIT_JSON_STAGE_ARGS(x.s), mStart.get(), mContinue.get(), mEnd.get(), discard,
            SPLIT_JSON_STAGE_OPTS(x.s), SPLIT_JSON_TS_ARGS(x), enableNs, tail, tailLen, o, cap, len, raw, nev, c8,
            sctr);
        SplitJsonTsStage::Fold(c8, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_json_timestamp_parse_sls",
        "lc_multiline_split_json_timestamp_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}
#undef SPLIT_JSON_TS_ARGS
#undef SPLIT_JSON_STAGE_ARGS
#undef SPLIT_JSON_STAGE_OPTS

// ------------------------------------------------------------------------------------------------ split -> Apsara
// The Apsara stage of the split -> Apsara chain: a ProcessorParseApsaraNative's configuration, "now" and history
// discard as the chain calls take them, the host check of lc_split_apsara_sls_setup, and the counters Process would
// move.  The device calls take a group of exactly one source event: the time cache runs over the whole group in event
// order and would otherwise have to carry across calls.
struct SplitApsaraStage {
    ProcessorParseApsaraNative& a;
    const PipelineEventGroup& group;
    int64_t now;
    SplitApsaraStage(ProcessorParseApsaraNative& ap, const PipelineEventGroup& g)
        : a(ap), group(g), now((int64_t)time(nullptr)) {}
    const std::string& Renamed() const { return a.mCommonParserOptions.mRenamedSourceKey; }
    const CommonParserOptions& Opt() const { return a.mCommonParserOptions; }
    const lc_apsara_t* Program() const { return a.mProgram; }
    int32_t DiscardInterval() const { return a.mDiscardOldData ? a.mDiscardInterval : -1; }
    // whether the chain's device calls take this stage behind a splitter reading sourceKey
    bool Accepts(const std::string& sourceKey, const StringView* okey) const {
        LcSplitApsaraSlsCfg c;
        return group.GetEvents().size() == 1 && a.mProgram && a.mSourceKey == sourceKey &&
               !lc_split_apsara_sls_setup(a.mSourceKey.data(), (uint32_t)a.mSourceKey.size(), Renamed().data(),
                                          (uint32_t)Renamed().size(), okey ? okey->data() : nullptr,
                                          okey ? (uint32_t)okey->size() : 0u, Opt().mKeepingSourceWhenParseFail,
                                          Opt().mKeepingSourceWhenParseSucceed, Opt().mCopingRawLog, 0, 0,
                                          LC_SLS_NO_NS, 0, &c);
    }
    // the device calls' counters[5] (key_not_found, out_failed, history_failure, discarded, out_successful) as the
    // chain driver takes a stage's: successful, out_failed, discarded (every piece the stage erased), none removed by a
    // filter, then key_not_found and history_failure
    static void Fold(const uint64_t c5[5], uint64_t rctr[8]) {
        const uint64_t f[8] = {c5[4], c5[1], c5[3], 0, c5[0], c5[2], 0, 0};
        memcpy(rctr, f, sizeof f);
    }
    void Add(const uint64_t ctr[6]) const {
        a.mOutSuccessfulEventsTotal.Add(ctr[0]);
        a.mOutFailedEventsTotal.Add(ctr[1]);
        a.mDiscardedEventsTotal.Add(ctr[2]);
        a.mOutKeyNotFoundEventsTotal.Add(ctr[4]);
        a.mHistoryFailureTotal.Add(ctr[5]);
    }
    void Process(PipelineEventGroup& g) const { a.Process(g); }
};
#define SPLIT_APSARA_STAGE_ARGS(x)                                                                                     \
    (x).Program(), src(val), val.size()
#define SPLIT_APSARA_STAGE_OPTS(x)                                                                                     \
    (x).Renamed().data(), (uint32_t)(x).Renamed().size(), (x).Opt().mKeepingSourceWhenParseFail,                      \
        (x).Opt().mKeepingSourceWhenParseSucceed, (x).Opt().mCopingRawLog, okey ? okey->data() : nullptr,            \
        okey ? (uint32_t)okey->size() : 0u, pos, time, ns, enableNs, (x).now, (x).DiscardInterval()

bool ProcessorSplitLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next,
                                                 bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitLogStringNative::SerializeSlsLz4(PipelineEventGroup& group, ProcessorParseApsaraNative& next,
                                                    bool enableNs, std::string& block, uint64_t& rawSize,
                                                    std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitLogStringNative::ChainSerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next,
                                                      bool enableNs, std::string& out, uint64_t* rawSize,
                                                      std::string& err) {
    const SplitApsaraStage x(next, group);
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c5[5] = {0, 0, 0, 0, 0};
        const int rc = lc_split_apsara_parse_sls(Engine(), SPLIT_APSARA_STAGE_ARGS(x), (uint8_t)mSplitChar,
                                                 SPLIT_APSARA_STAGE_OPTS(x), o, cap, len, nev, c5);
        SplitApsaraStage::Fold(c5, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t*) {
        uint64_t c5[5] = {0, 0, 0, 0, 0};
        const int rc = lc_split_apsara_parse_sls_lz4(Engine(), SPLIT_APSARA_STAGE_ARGS(x), (uint8_t)mSplitChar,
                                                     SPLIT_APSARA_STAGE_OPTS(x), tail, tailLen, o, cap, len, raw, nev,
                                                     c5);
        SplitApsaraStage::Fold(c5, rctr);
        return rc;
    };
    uint64_t unused[3] = {0, 0, 0};
    return SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_split_apsara_parse_sls",
        "lc_split_apsara_parse_sls_lz4", unused);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSls(PipelineEventGroup& group, ProcessorParseApsaraNative& next,
                                                          bool enableNs, std::string& out, std::string& err) {
    return ChainSerializeSls(group, next, enableNs, out, nullptr, err);
}

bool ProcessorSplitMultilineLogStringNative::SerializeSlsLz4(PipelineEventGroup& group,
                                                             ProcessorParseApsaraNative& next, bool enableNs,
                                                             std::string& block, uint64_t& rawSize,
                                                             std::string& err) {
    return ChainSerializeSls(group, next, enableNs, block, &rawSize, err);
}

bool ProcessorSplitMultilineLogStringNative::ChainSerializeSls(PipelineEventGroup& group,
                                                               ProcessorParseApsaraNative& next, bool enableNs,
                                                               std::string& out, uint64_t* rawSize, std::string& err) {
    const SplitApsaraStage x(next, group);
    const bool discard = mMultiline.mUnmatchedContentTreatment == MultilineOptions::UnmatchedContentTreatment::DISCARD;
    auto src = [](StringView v) { return reinterpret_cast<const uint8_t*>(v.data()); };
    auto sls = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns, uint8_t* o,
                   uint64_t cap, uint64_t* len, uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c5[5] = {0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_apsara_parse_sls(Engine(), SPLIT_APSARA_STAGE_ARGS(x), mStart.get(),
                                                           mContinue.get(), mEnd.get(), discard,
                                                           SPLIT_APSARA_STAGE_OPTS(x), o, cap, len, nev, c5, sctr);
        SplitApsaraStage::Fold(c5, rctr);
        return rc;
    };
    auto lz4 = [&](StringView val, const StringView* okey, uint64_t pos, uint32_t time, uint32_t ns,
                   const uint8_t* tail, uint64_t tailLen, uint8_t* o, uint64_t cap, uint64_t* len, uint64_t* raw,
                   uint64_t* nev, uint64_t* rctr, uint64_t* sctr) {
        uint64_t c5[5] = {0, 0, 0, 0, 0};
        const int rc = lc_multiline_split_apsara_parse_sls_lz4(Engine(), SPLIT_APSARA_STAGE_ARGS(x), mStart.get(),
                                                               mContinue.get(), mEnd.get(), discard,
                                                               SPLIT_APSARA_STAGE_OPTS(x), tail, tailLen, o, cap, len,
                                                               raw, nev, c5, sctr);
        SplitApsaraStage::Fold(c5, rctr);
        return rc;
    };
    // matched_events, input lines, unmatched lines: moved as Process moves them (:82-84,106-107)
    uint64_t ctr[3] = {0, 0, 0};
    const bool ok = SplitRegexChainSls(
        group, x, nullptr, false, mSourceKey, mEnableRawContent, enableNs, out, rawSize, err,
        [&](PipelineEventGroup& g) { Process(g); }, sls, lz4, "lc_multiline_split_apsara_parse_sls",
        "lc_multiline_split_apsara_parse_sls_lz4", ctr);
    mMatchedEventsTotal.Add(ctr[0]);
    mMatchedLinesTotal.Add(ctr[1] - ctr[2]);
    mUnmatchedLinesTotal.Add(ctr[2]);
    return ok;
}
#undef SPLIT_APSARA_STAGE_ARGS
#undef SPLIT_APSARA_STAGE_OPTS

} // namespace logtail
