// host_capi.cpp -- JSON-driven C entry points over the host Processor classes (include/lc_b200_host.h).
#include <dlfcn.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/lc_b200_host.h"
#include "PluginBench.h"
#include "Processors.h"

using namespace logtail;

struct lc_host_processor {
    std::unique_ptr<Processor> proc;
};

static char* dup(const std::string& s) {
    char* p = (char*)malloc(s.size() + 1);
    memcpy(p, s.c_str(), s.size() + 1);
    return p;
}

extern "C" {

lc_host_processor_t* lc_host_processor_create(const char* type, const char* config_json, char** err_out) {
    if (err_out)
        *err_out = nullptr;
    std::unique_ptr<Processor> p(CreateProcessor(type ? type : ""));
    if (!p) {
        if (err_out)
            *err_out = dup(std::string("unknown processor type: ") + (type ? type : "(null)"));
        return nullptr;
    }
    Json::Value cfg(Json::objectValue);
    std::string err;
    const char* cj = config_json ? config_json : "{}";
    if (!Json::Value::parse(cj, cj + strlen(cj), cfg, err)) {
        if (err_out)
            *err_out = dup("config is not valid JSON: " + err);
        return nullptr;
    }
    try {
        if (!p->Init(cfg)) {
            if (err_out)
                *err_out = dup("Init failed: " + p->LastError());
            return nullptr;
        }
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(std::string("Init threw: ") + e.what());
        return nullptr;
    }
    auto* h = new lc_host_processor;
    h->proc = std::move(p);
    return h;
}

void lc_host_processor_destroy(lc_host_processor_t* p) { delete p; }

char* lc_host_processor_process(lc_host_processor_t* p, const char* group_json, int enable_event_meta, char** err_out) {
    if (err_out)
        *err_out = nullptr;
    try {
        auto sb = std::make_shared<SourceBuffer>();
        PipelineEventGroup group(sb);
        if (!group.FromJsonString(group_json ? group_json : "null"))
            throw std::runtime_error("group JSON does not parse");
        const uint64_t errs = p->proc->EngineErrors();
        p->proc->Process(group);
        if (p->proc->EngineErrors() != errs) // Process itself never throws (reference contract); the harness reports it
            throw std::runtime_error("engine error inside Process: " + p->proc->LastError());
        return dup(group.ToJsonString(enable_event_meta != 0));
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(e.what());
        return nullptr;
    }
}

char* lc_host_processor_process_groups(lc_host_processor_t* p, const char* groups_json, int enable_event_meta,
                                       char** err_out) {
    if (err_out)
        *err_out = nullptr;
    try {
        Json::Value arr;
        std::string err;
        const char* gj = groups_json ? groups_json : "[]";
        if (!Json::Value::parse(gj, gj + strlen(gj), arr, err) || !arr.isArray())
            throw std::runtime_error("groups JSON is not an array");
        std::vector<PipelineEventGroup> groups;
        for (size_t k = 0; k < arr.size(); ++k) {
            groups.emplace_back(std::make_shared<SourceBuffer>());
            if (!groups.back().FromJson(arr[k]))
                throw std::runtime_error("group JSON does not parse");
        }
        const uint64_t errs = p->proc->EngineErrors();
        p->proc->Process(groups);
        if (p->proc->EngineErrors() != errs)
            throw std::runtime_error("engine error inside Process: " + p->proc->LastError());
        Json::Value out(Json::arrayValue);
        for (auto& g : groups)
            out.append(g.ToJson(enable_event_meta != 0));
        return dup(out.toString());
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(e.what());
        return nullptr;
    }
}

char* lc_host_processor_counters(const lc_host_processor_t* p) {
    Json::Value v(Json::objectValue);
    for (auto& kv : p->proc->Counters())
        v[kv.first] = Json::Value((uint64_t)kv.second);
    return dup(v.toString());
}

int lc_host_processor_set_discard_old_data(lc_host_processor_t* p, int enabled, int32_t interval) {
    if (auto* t = dynamic_cast<ProcessorParseTimestampNative*>(p->proc.get())) {
        t->mDiscardOldData = enabled != 0;
        t->mDiscardInterval = interval;
        return 0;
    }
    if (auto* a = dynamic_cast<ProcessorParseApsaraNative*>(p->proc.get())) {
        a->mDiscardOldData = enabled != 0;
        a->mDiscardInterval = interval;
        return 0;
    }
    return -1;
}

void lc_host_string_free(char* s) { free(s); }

char* lc_host_sls_serialize(const char* group_json, int enable_ns, unsigned long long* len_out, char** err_out) {
    if (err_out)
        *err_out = nullptr;
    if (len_out)
        *len_out = 0;
    try {
        PipelineEventGroup group(std::make_shared<SourceBuffer>());
        if (group_json && strcmp(group_json, "null") != 0 && !group.FromJsonString(group_json)) {
            if (err_out)
                *err_out = dup("group is not valid JSON");
            return nullptr;
        }
        SLSEventGroupSerializer ser;
        ser.mEnableTimestampNanosecond = enable_ns != 0;
        std::string res, err;
        if (!ser.Serialize(group, res, err)) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        char* p = (char*)malloc(res.size() + 1);
        memcpy(p, res.data(), res.size());
        p[res.size()] = 0;
        if (len_out)
            *len_out = res.size();
        return p;
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(std::string("Serialize threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_processor_serialize_sls(lc_host_processor_t* p, const char* group_json, int enable_ns,
                                      int process_then_serialize, unsigned long long* len_out, char** err_out,
                                      char** fail_out) {
    if (err_out)
        *err_out = nullptr;
    if (fail_out)
        *fail_out = nullptr;
    if (len_out)
        *len_out = 0;
    try {
        // the processors with a device path to the wire format: the same calls on any of them
        auto* d = dynamic_cast<ProcessorParseDelimiterNative*>(p->proc.get());
        auto* r = dynamic_cast<ProcessorParseRegexNative*>(p->proc.get());
        auto* s = dynamic_cast<ProcessorSplitLogStringNative*>(p->proc.get());
        auto* m = dynamic_cast<ProcessorSplitMultilineLogStringNative*>(p->proc.get());
        if (!d && !r && !s && !m)
            throw std::runtime_error("not a processor_parse_delimiter_native, processor_parse_regex_native, "
                                     "processor_split_string_native or processor_split_multiline_log_string_native");
        Processor* proc = p->proc.get();
        PipelineEventGroup group(std::make_shared<SourceBuffer>());
        if (!group.FromJsonString(group_json ? group_json : "null"))
            throw std::runtime_error("group JSON does not parse");
        const uint64_t errs = proc->EngineErrors();
        std::string res, err;
        bool ok;
        if (process_then_serialize) {
            proc->Process(group);
            SLSEventGroupSerializer ser;
            ser.mEnableTimestampNanosecond = enable_ns != 0;
            ok = ser.Serialize(group, res, err);
        } else {
            const bool ns = enable_ns != 0;
            ok = d   ? d->SerializeSls(group, ns, res, err)
                 : r ? r->SerializeSls(group, ns, res, err)
                 : s ? s->SerializeSls(group, ns, res, err)
                     : m->SerializeSls(group, ns, res, err);
        }
        if (proc->EngineErrors() != errs)
            throw std::runtime_error("engine error inside Process: " + proc->LastError());
        if (!ok) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        char* out = (char*)malloc(res.size() + 1);
        memcpy(out, res.data(), res.size());
        out[res.size()] = 0;
        if (len_out)
            *len_out = res.size();
        return out;
    } catch (const std::exception& e) {
        if (fail_out)
            *fail_out = dup(std::string("SerializeSls threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_processor_serialize_sls_lz4(lc_host_processor_t* p, const char* group_json, int enable_ns,
                                          unsigned long long* len_out, unsigned long long* raw_len_out, char** err_out,
                                          char** fail_out) {
    if (err_out)
        *err_out = nullptr;
    if (fail_out)
        *fail_out = nullptr;
    if (len_out)
        *len_out = 0;
    if (raw_len_out)
        *raw_len_out = 0;
    try {
        auto* d = dynamic_cast<ProcessorParseDelimiterNative*>(p->proc.get());
        auto* r = dynamic_cast<ProcessorParseRegexNative*>(p->proc.get());
        if (!d && !r)
            throw std::runtime_error("not a processor_parse_delimiter_native or processor_parse_regex_native");
        Processor* proc = p->proc.get();
        PipelineEventGroup group(std::make_shared<SourceBuffer>());
        if (!group.FromJsonString(group_json ? group_json : "null"))
            throw std::runtime_error("group JSON does not parse");
        const uint64_t errs = proc->EngineErrors();
        std::string block, err;
        uint64_t raw = 0;
        const bool ok = d ? d->SerializeSlsLz4(group, enable_ns != 0, block, raw, err)
                          : r->SerializeSlsLz4(group, enable_ns != 0, block, raw, err);
        if (proc->EngineErrors() != errs)
            throw std::runtime_error("engine error inside Process: " + proc->LastError());
        if (!ok) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        char* out = (char*)malloc(block.size() + 1);
        memcpy(out, block.data(), block.size());
        if (len_out)
            *len_out = block.size();
        if (raw_len_out)
            *raw_len_out = raw;
        return out;
    } catch (const std::exception& e) {
        if (fail_out)
            *fail_out = dup(std::string("SerializeSlsLz4 threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_chain_serialize_sls(lc_host_processor_t* delim, lc_host_processor_t* regex, const char* group_json,
                                  int enable_ns, int mode, unsigned long long* len_out, unsigned long long* raw_len_out,
                                  char** err_out, char** fail_out) {
    if (err_out)
        *err_out = nullptr;
    if (fail_out)
        *fail_out = nullptr;
    if (len_out)
        *len_out = 0;
    if (raw_len_out)
        *raw_len_out = 0;
    try {
        Processor* d = delim->proc.get();
        Processor* second = regex->proc.get();
        auto* r = dynamic_cast<ProcessorParseRegexNative*>(second);
        auto* pd = dynamic_cast<ProcessorParseDelimiterNative*>(d);
        auto* ps = dynamic_cast<ProcessorSplitLogStringNative*>(d);
        auto* pm = dynamic_cast<ProcessorSplitMultilineLogStringNative*>(d);
        auto* sd = (ps || pm) ? dynamic_cast<ProcessorParseDelimiterNative*>(second) : nullptr;
        auto* sj = (ps || pm) ? dynamic_cast<ProcessorParseJsonNative*>(second) : nullptr;
        auto* sa = (ps || pm) ? dynamic_cast<ProcessorParseApsaraNative*>(second) : nullptr;
        if (!((pd || ps || pm) && r) && !sd && !sj && !sa)
            throw std::runtime_error("not a processor_parse_delimiter_native or a splitter, and a "
                                     "processor_parse_regex_native; nor a splitter and a "
                                     "processor_parse_delimiter_native, processor_parse_json_native or "
                                     "processor_parse_apsara_native");
        // the chain's SerializeSls / SerializeSlsLz4 on whichever processor comes first, with the second as next
        auto chain = [&](auto* p, auto& next, PipelineEventGroup& g, std::string& res, uint64_t& raw,
                         std::string& err) {
            return mode == 2 ? p->SerializeSlsLz4(g, next, enable_ns != 0, res, raw, err)
                             : p->SerializeSls(g, next, enable_ns != 0, res, err);
        };
        auto first = [&](auto& next, PipelineEventGroup& g, std::string& res, uint64_t& raw, std::string& err) {
            if constexpr (std::is_same_v<std::decay_t<decltype(next)>, ProcessorParseRegexNative>) {
                if (pd)
                    return chain(pd, next, g, res, raw, err);
            }
            return ps ? chain(ps, next, g, res, raw, err) : chain(pm, next, g, res, raw, err);
        };
        PipelineEventGroup group(std::make_shared<SourceBuffer>());
        if (!group.FromJsonString(group_json ? group_json : "null"))
            throw std::runtime_error("group JSON does not parse");
        const uint64_t errs = d->EngineErrors() + second->EngineErrors();
        std::string res, err;
        uint64_t raw = 0;
        bool ok;
        if (mode == 1) {
            d->Process(group);
            second->Process(group);
            SLSEventGroupSerializer ser;
            ser.mEnableTimestampNanosecond = enable_ns != 0;
            ok = ser.Serialize(group, res, err);
        } else {
            ok = r    ? first(*r, group, res, raw, err)
                 : sd ? first(*sd, group, res, raw, err)
                 : sj ? first(*sj, group, res, raw, err)
                      : first(*sa, group, res, raw, err);
        }
        if (d->EngineErrors() + second->EngineErrors() != errs)
            throw std::runtime_error("engine error inside Process: " + d->LastError() + second->LastError());
        if (!ok) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        char* out = (char*)malloc(res.size() + 1);
        memcpy(out, res.data(), res.size());
        out[res.size()] = 0;
        if (len_out)
            *len_out = res.size();
        if (raw_len_out)
            *raw_len_out = raw;
        return out;
    } catch (const std::exception& e) {
        if (fail_out)
            *fail_out = dup(std::string("chain SerializeSls threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_chain3_serialize_sls(lc_host_processor_t* split, lc_host_processor_t* regex, lc_host_processor_t* filter,
                                   const char* group_json, int enable_ns, int mode, unsigned long long* len_out,
                                   unsigned long long* raw_len_out, char** err_out, char** fail_out) {
    if (err_out)
        *err_out = nullptr;
    if (fail_out)
        *fail_out = nullptr;
    if (len_out)
        *len_out = 0;
    if (raw_len_out)
        *raw_len_out = 0;
    try {
        // (splitter, regex, filter), (splitter, regex, timestamp), (splitter, JSON, timestamp), (splitter, delimiter,
        // regex) or (splitter, delimiter, timestamp)
        Processor* d = split->proc.get();
        Processor* b = regex->proc.get();
        Processor* c = filter->proc.get();
        auto* r = dynamic_cast<ProcessorParseRegexNative*>(b);
        auto* js = dynamic_cast<ProcessorParseJsonNative*>(b);
        auto* f = dynamic_cast<ProcessorFilterNative*>(c);
        auto* ts = dynamic_cast<ProcessorParseTimestampNative*>(c);
        auto* dl = dynamic_cast<ProcessorParseDelimiterNative*>(b);
        auto* dr = dynamic_cast<ProcessorParseRegexNative*>(c);
        auto* ps = dynamic_cast<ProcessorSplitLogStringNative*>(d);
        auto* pm = dynamic_cast<ProcessorSplitMultilineLogStringNative*>(d);
        if (!(ps || pm) || !((r && f) || (r && ts) || (js && ts) || (dl && dr) || (dl && ts)))
            throw std::runtime_error("not a splitter followed by a processor_parse_regex_native and a "
                                     "processor_filter_regex_native or a processor_parse_timestamp_native, by a "
                                     "processor_parse_json_native and a processor_parse_timestamp_native, or by a "
                                     "processor_parse_delimiter_native and a processor_parse_regex_native or a "
                                     "processor_parse_timestamp_native");
        auto chain = [&](auto* p, PipelineEventGroup& g, std::string& res, uint64_t& raw, std::string& err) {
            if (js)
                return mode == 2 ? p->SerializeSlsLz4(g, *js, *ts, enable_ns != 0, res, raw, err)
                                 : p->SerializeSls(g, *js, *ts, enable_ns != 0, res, err);
            if (dl && ts)
                return mode == 2 ? p->SerializeSlsLz4(g, *dl, *ts, enable_ns != 0, res, raw, err)
                                 : p->SerializeSls(g, *dl, *ts, enable_ns != 0, res, err);
            if (dl)
                return mode == 2 ? p->SerializeSlsLz4(g, *dl, *dr, enable_ns != 0, res, raw, err)
                                 : p->SerializeSls(g, *dl, *dr, enable_ns != 0, res, err);
            if (ts)
                return mode == 2 ? p->SerializeSlsLz4(g, *r, *ts, enable_ns != 0, res, raw, err)
                                 : p->SerializeSls(g, *r, *ts, enable_ns != 0, res, err);
            return mode == 2 ? p->SerializeSlsLz4(g, *r, *f, enable_ns != 0, res, raw, err)
                             : p->SerializeSls(g, *r, *f, enable_ns != 0, res, err);
        };
        PipelineEventGroup group(std::make_shared<SourceBuffer>());
        if (!group.FromJsonString(group_json ? group_json : "null"))
            throw std::runtime_error("group JSON does not parse");
        const uint64_t errs = d->EngineErrors() + b->EngineErrors() + c->EngineErrors();
        std::string res, err;
        uint64_t raw = 0;
        bool ok;
        if (mode == 1) {
            d->Process(group);
            b->Process(group);
            c->Process(group);
            SLSEventGroupSerializer ser;
            ser.mEnableTimestampNanosecond = enable_ns != 0;
            ok = ser.Serialize(group, res, err);
        } else {
            ok = ps ? chain(ps, group, res, raw, err) : chain(pm, group, res, raw, err);
        }
        if (d->EngineErrors() + b->EngineErrors() + c->EngineErrors() != errs)
            throw std::runtime_error("engine error inside Process: " + d->LastError() + b->LastError() +
                                     c->LastError());
        if (!ok) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        char* out = (char*)malloc(res.size() + 1);
        memcpy(out, res.data(), res.size());
        out[res.size()] = 0;
        if (len_out)
            *len_out = res.size();
        if (raw_len_out)
            *raw_len_out = raw;
        return out;
    } catch (const std::exception& e) {
        if (fail_out)
            *fail_out = dup(std::string("chain3 SerializeSls threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_lz4_compress(const char* const* data, const unsigned long long* len, unsigned long long n,
                           unsigned long long* len_out, unsigned long long* blk_len, char** err_out) {
    if (err_out)
        *err_out = nullptr;
    if (len_out)
        *len_out = 0;
    try {
        std::vector<std::string> in, out;
        for (unsigned long long k = 0; k < n; ++k)
            in.emplace_back(data[k], len[k]);
        std::string err;
        LZ4Compressor c;
        if (!c.Compress(in, out, err)) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        std::string all;
        for (unsigned long long k = 0; k < n; ++k) {
            blk_len[k] = out[k].size();
            all += out[k];
        }
        char* res = (char*)malloc(all.size() + 1);
        memcpy(res, all.data(), all.size());
        if (len_out)
            *len_out = all.size();
        return res;
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(std::string("LZ4Compressor::Compress threw: ") + e.what());
        return nullptr;
    }
}

char* lc_host_zstd_compress(const char* const* data, const unsigned long long* len, unsigned long long n,
                            unsigned long long* len_out, unsigned long long* frm_len, char** err_out) {
    if (err_out)
        *err_out = nullptr;
    if (len_out)
        *len_out = 0;
    try {
        std::vector<std::string> in, out;
        for (unsigned long long k = 0; k < n; ++k)
            in.emplace_back(data[k], len[k]);
        std::string err;
        ZstdCompressor c(CompressType::ZSTD);
        if (!c.Compress(in, out, err)) {
            if (err_out)
                *err_out = dup(err);
            return nullptr;
        }
        std::string all;
        for (unsigned long long k = 0; k < n; ++k) {
            frm_len[k] = out[k].size();
            all += out[k];
        }
        char* res = (char*)malloc(all.size() + 1);
        memcpy(res, all.data(), all.size());
        if (len_out)
            *len_out = all.size();
        return res;
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(std::string("ZstdCompressor::Compress threw: ") + e.what());
        return nullptr;
    }
}

// What PluginRegistry::LoadProcessorPlugin + DynamicCProcessorProxy do with a dynamic plugin
// (PluginRegistry.cpp:218-275, DynamicCProcessorProxy.cpp:21-36), step by step, on the plugin at so_path.
char* lc_host_dynamic_plugin_roundtrip(const char* so_path, const char* config_json, const char* group_json,
                                       int enable_event_meta, int* version_out, char** name_out, char** err_out) {
    struct Iface { // CProcessor.h:23-45
        int version;
        const char* name;
        const char* language;
        int (*init)(void* ins, void* config, void* context);
        void (*finalize)(void* state);
        void (*process)(void* state, void* group);
    };
    struct Instance {
        const Iface* plugin;
        void* plugin_state;
    };
    if (err_out)
        *err_out = nullptr;
    void* h = dlopen(so_path, RTLD_NOW | RTLD_LOCAL);
    if (!h) {
        if (err_out)
            *err_out = dup(std::string("dlopen: ") + dlerror());
        return nullptr;
    }
    char* result = nullptr;
    try {
        const Iface* plugin = static_cast<const Iface*>(dlsym(h, "processor_interface"));
        if (!plugin)
            throw std::runtime_error("symbol processor_interface not found");
        if (version_out)
            *version_out = plugin->version;
        if (name_out)
            *name_out = dup(plugin->name ? plugin->name : "");
        if (plugin->version != 100)
            throw std::runtime_error("plugin interface version mismatch");
        Json::Value cfg(Json::objectValue);
        std::string err;
        const char* cj = config_json ? config_json : "{}";
        if (!Json::Value::parse(cj, cj + strlen(cj), cfg, err))
            throw std::runtime_error("config is not valid JSON: " + err);
        Instance ins{plugin, reinterpret_cast<void*>(0xdeadbeef)}; // the proxy leaves plugin_state uninitialised
        int ctx = 0;
        if (plugin->init(&ins, &cfg, &ctx) != 0) {
            if (ins.plugin_state != nullptr)
                throw std::runtime_error("init failed and left plugin_state dangling");
            throw std::runtime_error("init returned non-zero");
        }
        if (group_json) {
            PipelineEventGroup group(std::make_shared<SourceBuffer>());
            if (!group.FromJsonString(group_json))
                throw std::runtime_error("group JSON does not parse");
            plugin->process(ins.plugin_state, &group);
            result = dup(group.ToJsonString(enable_event_meta != 0));
        } else {
            result = dup("null");
        }
        plugin->finalize(ins.plugin_state);
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(e.what());
        result = nullptr;
    }
    dlclose(h);
    return result;
}

void lc_host_use_pinned_arenas(int on) {
    if (on)
        SourceBuffer::SetChunkAllocator(&lc_host_alloc, &lc_host_free);
    else
        SourceBuffer::SetChunkAllocator(nullptr, nullptr);
}

int lc_host_bench_plugin(const char* type, const char* config_json, const uint8_t* data, const uint32_t* line_off,
                         const uint32_t* line_len, uint64_t n_lines, uint32_t group_bytes, int mode, int reps,
                         double* seconds_out, uint64_t stats_out[16], char** err_out) {
    if (err_out)
        *err_out = nullptr;
    try {
        std::unique_ptr<Processor> p(CreateProcessor(type ? type : ""));
        if (!p)
            throw std::runtime_error(std::string("unknown processor type: ") + (type ? type : "(null)"));
        Json::Value cfg(Json::objectValue);
        std::string err;
        const char* cj = config_json ? config_json : "{}";
        if (!Json::Value::parse(cj, cj + strlen(cj), cfg, err))
            throw std::runtime_error("config is not valid JSON: " + err);
        ProcessorInstance inst(p.release());
        if (!inst.Init(cfg))
            throw std::runtime_error("Init failed: " + inst.GetPlugin()->LastError());
        PluginBench bench(data, line_off, line_len, n_lines, group_bytes, 16);
        PluginBenchResult r = bench.Run(reps, [&](std::vector<PipelineEventGroup>& groups) {
            if (mode == 1) {
                inst.Process(groups); // ProcessorInstance::Process(vector<PipelineEventGroup>&), the pipeline's call
            } else {
                // one call per group, as a ProcessorRunner thread does with the groups it pops
                // (ProcessorRunner.cpp:128-143): the vector holds ONE group each time
                std::vector<PipelineEventGroup> one;
                for (auto& g : groups) {
                    one.clear();
                    one.emplace_back(std::move(g));
                    inst.Process(one);
                    g = std::move(one[0]);
                }
            }
        });
        if (inst.GetPlugin()->EngineErrors())
            throw std::runtime_error("engine error inside Process: " + inst.GetPlugin()->LastError());
        for (int k = 0; k < reps && seconds_out; ++k)
            seconds_out[k] = r.seconds[k];
        if (stats_out) {
            stats_out[0] = r.groups;
            stats_out[1] = r.inEvents;
            stats_out[2] = r.outEvents;
            stats_out[3] = r.liveContents;
            stats_out[4] = r.checksum;
            stats_out[5] = r.arenaBytes;
            stats_out[6] = inst.mInEventsTotal.GetValue();
            stats_out[7] = inst.mOutEventsTotal.GetValue();
            stats_out[8] = inst.mInSizeBytes.GetValue();
            stats_out[9] = inst.mOutSizeBytes.GetValue();
            stats_out[10] = inst.mTotalProcessTimeNs.GetValue();
            stats_out[11] = inst.mTotalProcessTimeMs.GetValue();
            stats_out[12] = stats_out[13] = stats_out[14] = stats_out[15] = 0;
            for (auto& kv : inst.GetPlugin()->Counters()) { // phase breakdown of the batched path, when the plugin has one
                if (kv.first == "b200_gather_ns")
                    stats_out[12] = kv.second;
                else if (kv.first == "b200_engine_ns")
                    stats_out[13] = kv.second;
                else if (kv.first == "b200_epilogue_ns")
                    stats_out[14] = kv.second;
            }
        }
        return 0;
    } catch (const std::exception& e) {
        if (err_out)
            *err_out = dup(e.what());
        return 1;
    }
}

}
