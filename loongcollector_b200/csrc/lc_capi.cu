// lc_capi.cu -- implementation of the C-ABI declared in include/lc_b200.h: engine (stream, grow-only
// HBM workspace, look-back descriptors), host<->device staging, and the per-processor pipelines.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/lc_b200.h"
#include "lc_exec.cuh"
#include "lc_kernels.cuh"
#include "lc_tables.h"
#include "regex_compiler.h"

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

#define CU_TRY(expr)                                                                                                  \
    do {                                                                                                               \
        cudaError_t _e = (expr);                                                                                       \
        if (_e != cudaSuccess)                                                                                         \
            return fail(LC_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                               \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap)
            return cudaSuccess;
        if (p)
            cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256; // grow-only with slack
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess)
            cap = want;
        return e;
    }
    void release() {
        if (p)
            cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <class T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

std::atomic<uint64_t> g_regex_ids{1};

// engines alive in this process: lc_regex_free() tells each of them to drop its device copies of the tables
std::mutex g_engines_mu;
std::vector<lc_engine*> g_engines;

} // namespace

struct lc_regex {
    uint64_t id;
    lcb200::CompileResult res;
    std::string pattern;
};

struct lc_engine {
    int device = 0;
    cudaStream_t stream = nullptr;     // the stream every call of this engine is queued on
    cudaStream_t own_stream = nullptr; // created with the engine; `stream` unless lc_engine_set_stream replaced it
    uint64_t launches = 0;
    int num_sms = 148;
    int smem_per_block_optin = 0;
    int smem_per_sm = 0;
    bool force_basic_regex = false;   // env LC_B200_REGEX_KERNEL=basic   (tables in global memory)
    int regex_variant = 0; // env LC_B200_REGEX_KERNEL: 0 auto, 1 "fast" (stride-1), 2 "fast2" (stride-2), 3 "generic",
                           // 4 "tdfa" (single pass); "basic" sets force_basic_regex, anything else means auto
    uint64_t scratch_hint = 0;
    int length_order = -1; // env LC_B200_LENGTH_ORDER: 1 = always order ragged batches by length, 0 = never, unset = auto
    uint32_t max_warps = 32;   // env LC_B200_MAX_WARPS (tuning knob: resident warps per block of the regex kernels)
    bool multi_split = false;  // env LC_B200_MULTI_SPLIT=1: lc_regex_parse_multi launches one pattern at a time (test knob)
    // staging / workspace (grow-only)
    DevBuf in, ev_off, ev_len, out_a, out_b, out_c, out_d, out_e;
    DevBuf lines_off, lines_len, flags, state, cnt, pos, lab_sizes, lab_off, lab, order;
    DevBuf desc;   // look-back descriptors of exclusive sums
    DevBuf split_scratch; // masks + per-tile counts of the three-pass split (lck::split_scratch_bytes)
    DevBuf sls_plan; // content plans + key strings of the regex-fed SLS serialiser (`order` is the regex stage's)
    // LZ4 compressor: sequences, chunk summaries, chunk sizes / anchors, chunk and block offsets, host-call tables and
    // output; no parse or SLS stage uses them
    DevBuf z_seq, z_info, z_size, z_first, z_choff, z_tab, z_out;
    // zstd compressor (behind the LZ4 parse pass): per-segment first block, per-block body sizes and frame bytes,
    // block offsets, one LC_ZSTD_BLOCK slot per block for its compressed body
    DevBuf zs_first, zs_size, zs_off, zs_slot;
    // delimiter -> regex -> SLS chain: the delimiter's key strings, the value table, the regex tables over it, side-copy
    // sizes and slots, the per-chunk scan descriptors of the tap; no stage of the chain uses them for anything else
    DevBuf dr_keys, dr_val_off, dr_val_len, dr_status, dr_cap_off, dr_cap_len, dr_copy, dr_slot, dr_desc;
    // split -> regex -> filter chain: one leaf's value tables, the match bytes of every leaf, the offset-digit scratch,
    // the removed-piece counter and the keep bytes; the chain's piece and regex tables live elsewhere (in, out_a,
    // out_b, out_c, dr_*), and so does the scratch of the boolean match (out_d, out_e, lab*, order, desc)
    DevBuf fl_tab, fl_match, fl_dig, fl_keep;
    // split -> delimiter -> regex chain: the delimiter tables over the pieces (status, column counts, f_off, f_len,
    // f_dq) and the offset key; its value, regex and tap tables are the dr_* of the delimiter -> regex chain
    DevBuf sdr_status, sdr_nf, sdr_f_off, sdr_f_len, sdr_f_dq, sdr_okey;
    // timestamp parse: the LcTsConf of the program ts_conf_id (uploaded on its first call here), the full-parse
    // results, the host call's counters
    DevBuf ts_conf, ts_full, ts_cnt;
    uint64_t ts_conf_id = 0;
    // split -> regex -> timestamp chain: the tap's value table and group starts, the timestamp tables over the pieces;
    // the chain's piece and regex tables are the split -> regex chain's (in, out_a, out_b, dr_*)
    DevBuf st_val, st_sec, st_nsec, st_status;
    // Apsara parse: the handle ap_conf_id's zone table and SourceKey, the scan results, the entry counts, the
    // counters and the out-of-range flag; the host call's copies of its outputs
    DevBuf ap_conf, ap_ev, ap_nent, ap_small;
    uint64_t ap_conf_id = 0;
    DevBuf ap_status, ap_sec, ap_nsec, ap_micro, ap_first, ap_ent;
    // JSON parse: SourceKey (js_conf_id's), the counts, the slow flags and list, the arena starts, the flags; the host
    // call's copies of its outputs
    DevBuf js_conf, js_nent, js_narena, js_slow, js_list, js_afirst, js_small, js_pow5;
    uint64_t js_conf_id = 0;
    DevBuf js_status, js_first, js_ent, js_arena, js_cnt;
    // split -> JSON -> SLS chain: the resolve's per-entry winners, per-piece records, list of pieces to sort (behind
    // its count) and sort scratch; the chain's piece and JSON tables are in, out_a, out_b and the js_* buffers
    DevBuf sj_win, sj_ev, sj_list, sj_sort;
    // split -> JSON -> timestamp chain: the value buffer the tap copies each piece's value into (chunk bytes, then arena
    // bytes); its value and timestamp tables are the split -> regex -> timestamp chain's st_* buffers.  The split ->
    // delimiter -> timestamp chain uses the same three (its values are chunk bytes only).
    DevBuf sjt_val;
    // split -> Apsara -> SLS chain: its one-group table; the piece and Apsara tables are in, out_a, out_b and the ap_*
    // buffers
    DevBuf sa_grp;
    DevBuf small;  // tickets + counters: [0..3] u32 tickets, +16: u32 n_out, +32: u64 total, +64: u64 counters[2]
    void* h_small = nullptr; // pinned mirror of `small`
    std::unordered_map<uint64_t, void*> blobs; // regex id * 4 + layout -> device blob
    std::mutex freed_mu;
    std::vector<uint64_t> freed_ids; // regexes freed since the last call (their blobs are released lazily)
    // copy pipeline of the host-pointer entry points
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    std::vector<cudaEvent_t> ev_h2d, ev_comp, ev_d2h;
};

namespace {

cudaError_t engine_blob(lc_engine* e, const lc_regex* r, const void** out, int layout = 0) {
    *out = nullptr;
    if (!r)
        return cudaSuccess;
    const std::vector<uint8_t>& src = layout == 3   ? r->res.tdfa_blob
                                      : layout == 2 ? r->res.fast2_blob
                                                    : (layout == 1 ? r->res.fast_blob : r->res.blob);
    const uint64_t key = r->id * 4 + (uint64_t)layout;
    {
        // device tables of regexes freed since the last call (lc_regex_free): released here, on the engine's own
        // thread, after the stream has drained
        std::vector<uint64_t> dead;
        {
            std::lock_guard<std::mutex> lk(e->freed_mu);
            dead.swap(e->freed_ids);
        }
        if (!dead.empty()) {
            cudaStreamSynchronize(e->stream);
            for (uint64_t id : dead)
                for (uint64_t l = 0; l < 4; ++l) {
                    auto f = e->blobs.find(id * 4 + l);
                    if (f != e->blobs.end()) {
                        cudaFree(f->second);
                        e->blobs.erase(f);
                    }
                }
        }
    }
    auto it = e->blobs.find(key);
    if (it != e->blobs.end()) {
        *out = it->second;
        return cudaSuccess;
    }
    void* d = nullptr;
    cudaError_t er = cudaMalloc(&d, src.size());
    if (er != cudaSuccess)
        return er;
    er = cudaMemcpyAsync(d, src.data(), src.size(), cudaMemcpyHostToDevice, e->stream);
    if (er != cudaSuccess) {
        cudaFree(d);
        return er;
    }
    e->blobs[key] = d;
    *out = d;
    return cudaSuccess;
}

struct Small {
    uint32_t tickets[4];
    uint32_t n_out;
    uint32_t overflow;
    uint32_t pad0[2];
    uint64_t total;
    unsigned long long bump;
    unsigned long long next_batch;
    unsigned long long total_chars; // un-truncated split-char count of the last split
    unsigned long long counters[2];
};

int bind(lc_engine* e) {
    CU_TRY(cudaSetDevice(e->device));
    return LC_OK;
}

// zeroed look-back descriptors for an exclusive sum over `ntiles` tiles (lck::scan_tiles); zeroes Small too
int prep_desc(lc_engine* e, size_t ntiles, uint64_t** desc) {
    CU_TRY(e->desc.ensure((ntiles + 1) * 8));
    CU_TRY(cudaMemsetAsync(e->desc.p, 0, (ntiles + 1) * 8, e->stream));
    CU_TRY(cudaMemsetAsync(e->small.p, 0, sizeof(Small), e->stream));
    *desc = e->desc.as<uint64_t>();
    return LC_OK;
}

int ensure_copy_streams(lc_engine* e, int nchunks) {
    if (!e->s_h2d)
        CU_TRY(cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking));
    if (!e->s_d2h)
        CU_TRY(cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking));
    while ((int)e->ev_h2d.size() < nchunks) {
        cudaEvent_t a, b, c;
        CU_TRY(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
        CU_TRY(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
        CU_TRY(cudaEventCreateWithFlags(&c, cudaEventDisableTiming));
        e->ev_h2d.push_back(a);
        e->ev_comp.push_back(b);
        e->ev_d2h.push_back(c);
    }
    return LC_OK;
}

// host-pointer entry points: every event must lie inside [0, base_len) -- a bad table would make the kernels read
// (or, for the serialiser, write) outside the staged arena
int check_events(const uint32_t* off, const uint32_t* len, uint64_t n, uint64_t base_len, const char* what) {
    uint64_t hi = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t en = (uint64_t)off[i] + len[i];
        hi = en > hi ? en : hi;
    }
    if (hi > base_len)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event beyond base_len");
    return LC_OK;
}

// first-byte filter + empty-line verdict of pattern slot p for the fused split + probe pass (prefix DFA of the blob)
void fill_probe_slot(lck::MlConfig& cfg, int p, const lc_regex* r) {
    memset(cfg.first[p], 0, sizeof cfg.first[p]);
    if (!r)
        return;
    const uint8_t* b = r->res.blob.data();
    const LcRegexHeader* h = reinterpret_cast<const LcRegexHeader*>(b);
    const uint8_t* cls = b + h->off_byte_class;
    const uint16_t* pre_next = reinterpret_cast<const uint16_t*>(b + h->off_pre_next);
    const uint8_t* pre_acc = b + h->off_pre_acc;
    for (uint32_t c = 0; c < 256; ++c)
        if (pre_next[h->pre_start * h->nclasses + cls[c]] != LC_PREFIX_DEAD)
            cfg.first[p][c >> 5] |= 1u << (c & 31);
    if (pre_acc[h->pre_start])
        cfg.empty_flags |= 1u << p;
}

int check_regex_usable(const lc_regex* r, const char* what) {
    if (!r->res.supported)
        return fail(r->res.valid ? LC_ERR_REGEX_UNSUPPORTED : LC_ERR_REGEX_INVALID,
                    std::string(what) + ": " + r->res.error);
    return LC_OK;
}

} // namespace

extern "C" {

const char* lc_version(void) { return "loongcollector_b200 0.1.0 (sm_90a)"; }
const char* lc_last_error(void) { return g_err.c_str(); }

int lc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int lc_engine_create(int device, lc_engine_t** out) {
    if (!out)
        return fail(LC_ERR_INVALID_ARG, "lc_engine_create: out is NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t er = cudaGetDeviceCount(&n);
    if (er != cudaSuccess || n == 0)
        return fail(LC_ERR_CUDA, std::string("lc_engine_create: no usable CUDA device (") +
                                     (er != cudaSuccess ? cudaGetErrorString(er) : "device count 0") +
                                     "); this engine has no CPU fallback");
    if (device < 0 || device >= n)
        return fail(LC_ERR_INVALID_ARG, "lc_engine_create: bad device index");
    lc_engine* e = new (std::nothrow) lc_engine;
    if (!e)
        return fail(LC_ERR_CUDA, "out of host memory");
    e->device = device;
    CU_TRY(cudaSetDevice(device));
    // a blocking stream: device buffers a caller filled on the legacy default stream (PyTorch's default stream) are
    // ready before a *_dev call's kernels read them, and that stream's later work waits for the engine's writes
    CU_TRY(cudaStreamCreateWithFlags(&e->own_stream, cudaStreamDefault));
    e->stream = e->own_stream;
    CU_TRY(cudaDeviceGetAttribute(&e->num_sms, cudaDevAttrMultiProcessorCount, device));
    CU_TRY(cudaDeviceGetAttribute(&e->smem_per_block_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    CU_TRY(cudaDeviceGetAttribute(&e->smem_per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device));
    {
        const char* k = getenv("LC_B200_REGEX_KERNEL");
        e->force_basic_regex = k && !strcmp(k, "basic");
        const char* mw = getenv("LC_B200_MAX_WARPS");
        if (mw && atoi(mw) >= 4 && atoi(mw) <= 32)
            e->max_warps = (uint32_t)atoi(mw);
        const char* msp = getenv("LC_B200_MULTI_SPLIT");
        e->multi_split = msp && !strcmp(msp, "1");
        const char* lo = getenv("LC_B200_LENGTH_ORDER");
        e->length_order = !lo ? -1 : (!strcmp(lo, "1") ? 1 : 0);
        e->regex_variant = !k ? 0 : (!strcmp(k, "fast") ? 1 : (!strcmp(k, "fast2") ? 2 : (!strcmp(k, "generic") ? 3 : (!strcmp(k, "tdfa") ? 4 : 0))));
    }
    CU_TRY(e->small.ensure(sizeof(Small)));
    CU_TRY(cudaMallocHost(&e->h_small, sizeof(Small)));
    {
        std::lock_guard<std::mutex> lk(g_engines_mu);
        g_engines.push_back(e);
    }
    *out = e;
    return LC_OK;
}

void lc_engine_destroy(lc_engine_t* e) {
    if (!e)
        return;
    {
        std::lock_guard<std::mutex> lk(g_engines_mu);
        g_engines.erase(std::remove(g_engines.begin(), g_engines.end(), e), g_engines.end());
    }
    cudaSetDevice(e->device);
    if (e->stream)
        cudaStreamSynchronize(e->stream);
    DevBuf* bufs[] = {&e->in, &e->ev_off, &e->ev_len, &e->out_a, &e->out_b, &e->out_c, &e->out_d, &e->out_e,
                      &e->lines_off, &e->lines_len, &e->flags, &e->state, &e->cnt, &e->pos, &e->lab_sizes,
                      &e->lab_off, &e->lab, &e->order, &e->desc, &e->small, &e->split_scratch, &e->sls_plan,
                      &e->z_seq, &e->z_info, &e->z_size, &e->z_first, &e->z_choff, &e->z_tab, &e->z_out,
                      &e->zs_first, &e->zs_size, &e->zs_off, &e->zs_slot,
                      &e->dr_keys, &e->dr_val_off, &e->dr_val_len, &e->dr_status, &e->dr_cap_off, &e->dr_cap_len,
                      &e->dr_copy, &e->dr_slot, &e->dr_desc, &e->fl_tab, &e->fl_match, &e->fl_dig, &e->fl_keep,
                      &e->sdr_status, &e->sdr_nf, &e->sdr_f_off, &e->sdr_f_len, &e->sdr_f_dq, &e->sdr_okey,
                      &e->ts_conf, &e->ts_full, &e->ts_cnt, &e->st_val, &e->st_sec, &e->st_nsec, &e->st_status,
                      &e->ap_conf, &e->ap_ev, &e->ap_nent, &e->ap_small, &e->ap_status, &e->ap_sec, &e->ap_nsec,
                      &e->ap_micro, &e->ap_first, &e->ap_ent, &e->js_conf, &e->js_nent, &e->js_narena,
                      &e->js_slow, &e->js_list, &e->js_afirst, &e->js_small, &e->js_status, &e->js_first, &e->js_ent,
                      &e->js_arena, &e->js_cnt, &e->js_pow5, &e->sj_win, &e->sj_ev, &e->sj_list, &e->sj_sort,
                      &e->sa_grp, &e->sjt_val};
    for (DevBuf* b : bufs)
        b->release();
    for (auto& kv : e->blobs)
        cudaFree(kv.second);
    if (e->h_small)
        cudaFreeHost(e->h_small);
    for (cudaEvent_t ev : e->ev_h2d)
        cudaEventDestroy(ev);
    for (cudaEvent_t ev : e->ev_comp)
        cudaEventDestroy(ev);
    for (cudaEvent_t ev : e->ev_d2h)
        cudaEventDestroy(ev);
    if (e->s_h2d)
        cudaStreamDestroy(e->s_h2d);
    if (e->s_d2h)
        cudaStreamDestroy(e->s_d2h);
    if (e->own_stream)
        cudaStreamDestroy(e->own_stream);
    delete e;
}

int lc_engine_sync(lc_engine_t* e) {
    if (!e)
        return fail(LC_ERR_INVALID_ARG, "engine is NULL");
    CU_TRY(cudaSetDevice(e->device));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

void* lc_engine_stream(lc_engine_t* e) { return e ? (void*)e->stream : nullptr; }

int lc_engine_set_stream(lc_engine_t* e, void* stream) {
    if (!e)
        return fail(LC_ERR_INVALID_ARG, "engine is NULL");
    CU_TRY(cudaSetDevice(e->device));
    CU_TRY(cudaStreamSynchronize(e->stream)); // workspace reuse is ordered by the stream: drain the old one first
    e->stream = stream ? (cudaStream_t)stream : e->own_stream;
    return LC_OK;
}
uint64_t lc_engine_launch_count(const lc_engine_t* e) { return e ? e->launches : 0; }

void* lc_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) {
        g_err = "lc_host_alloc: cudaMallocHost failed";
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void lc_host_free(void* p) {
    if (p)
        cudaFreeHost(p);
}

// ------------------------------------------------------------------------------------------------ regex
int lc_regex_compile(const char* pattern, size_t len, lc_regex_t** out) {
    if (!out || (!pattern && len))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_compile: bad arguments");
    lc_regex* r = new (std::nothrow) lc_regex;
    if (!r)
        return fail(LC_ERR_CUDA, "out of host memory");
    r->id = g_regex_ids.fetch_add(1);
    r->pattern.assign(pattern ? pattern : "", len);
    r->res = lcb200::compile_regex(r->pattern.data(), r->pattern.size());
    *out = r;
    if (!r->res.valid)
        return fail(LC_ERR_REGEX_INVALID, r->res.error);
    if (!r->res.supported)
        return fail(LC_ERR_REGEX_UNSUPPORTED, r->res.error);
    return LC_OK;
}

void lc_regex_free(lc_regex_t* r) {
    if (!r)
        return;
    {
        std::lock_guard<std::mutex> lk(g_engines_mu);
        for (lc_engine* e : g_engines) {
            std::lock_guard<std::mutex> lk2(e->freed_mu);
            e->freed_ids.push_back(r->id);
        }
    }
    delete r;
}
const char* lc_regex_error(const lc_regex_t* r) { return r ? r->res.error.c_str() : ""; }
uint32_t lc_regex_ngroups(const lc_regex_t* r) { return r ? r->res.ngroups : 0; }

void lc_regex_info(const lc_regex_t* r, uint32_t info[8]) {
    memset(info, 0, 8 * sizeof(uint32_t));
    if (!r || !r->res.supported)
        return;
    const LcRegexHeader* h = reinterpret_cast<const LcRegexHeader*>(r->res.blob.data());
    info[0] = h->mode;
    info[1] = h->nclasses;
    info[2] = h->nw;
    info[3] = h->npc;
    info[4] = h->rev_nstates;
    info[5] = h->pre_nstates;
    info[6] = h->total_bytes;
    info[7] = r->res.n_insts;
}

// ------------------------------------------------------------------------------------------------ split
int lc_split_lines_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, uint8_t split_char, uint32_t* d_out_off,
                       uint32_t* d_out_len, uint64_t cap, uint64_t* n_out) {
    if (!e || !n_out || (len && !d_buf))
        return fail(LC_ERR_INVALID_ARG, "lc_split_lines_dev: bad arguments");
    *n_out = 0;
    if (len == 0)
        return LC_OK;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(cudaMemsetAsync(e->small.p, 0, sizeof(Small), e->stream)); // n_out, total_chars
    Small* ds = e->small.as<Small>();
    uint32_t cap32 = cap > 0x3FFFFFFFull ? 0x3FFFFFFFu : (uint32_t)cap;
    CU_TRY(e->split_scratch.ensure(lck::split_scratch_bytes(len, false)));
    e->launches += lck::launch_split(d_buf, (uint32_t)len, split_char, d_out_off, d_out_len, cap32, &ds->n_out,
                                     &ds->total_chars, e->split_scratch.as<uint64_t>(), e->stream);
    CU_TRY(cudaGetLastError());
    Small* hs = (Small*)e->h_small;
    CU_TRY(cudaMemcpyAsync(hs, ds, sizeof(Small), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (hs->total_chars >= (1ull << 30) - 1)
        return fail(LC_ERR_TOO_LARGE, "more than 2^30 pieces in one call");
    *n_out = hs->n_out;
    if (*n_out > cap)
        return fail(LC_ERR_CAPACITY, "lc_split_lines: output capacity too small");
    return LC_OK;
}

int lc_split_lines(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, uint32_t* out_off,
                   uint32_t* out_len, uint64_t cap, uint64_t* n_out) {
    if (!e || !n_out || (len && !buf))
        return fail(LC_ERR_INVALID_ARG, "lc_split_lines: bad arguments");
    *n_out = 0;
    if (len == 0)
        return LC_OK;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    int rc = bind(e);
    if (rc)
        return rc;
    uint64_t dcap = cap < len ? cap : len;
    CU_TRY(e->in.ensure(len + 16));
    CU_TRY(e->out_a.ensure((dcap + 1) * 4));
    CU_TRY(e->out_b.ensure((dcap + 1) * 4));
    CU_TRY(cudaMemcpyAsync(e->in.p, buf, len, cudaMemcpyHostToDevice, e->stream));
    rc = lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                            e->out_b.as<uint32_t>(), dcap, n_out);
    if (rc)
        return rc;
    if (*n_out) {
        CU_TRY(cudaMemcpyAsync(out_off, e->out_a.p, *n_out * 4, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaMemcpyAsync(out_len, e->out_b.p, *n_out * 4, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    return LC_OK;
}

// ------------------------------------------------------------------------------------------------ regex parse
// span_bytes: bytes of the arena this batch's events cover (== base_len for a whole-arena call; the chunked host path
// passes the chunk's own span so that per-batch heuristics see the batch, not the arena).  ev_stride: distance in
// elements between consecutive entries of d_ev_off / d_ev_len (1 = dense tables).
static int regex_parse_dev_impl(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                                uint64_t span_bytes, const uint32_t* d_ev_off, const uint32_t* d_ev_len,
                                uint32_t ev_stride, uint64_t n, uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off,
                                uint32_t* d_cap_len, bool bool_only);

int lc_regex_parse_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint32_t nkeys,
                       uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len) {
    return regex_parse_dev_impl(e, re, d_base, base_len, base_len, d_ev_off, d_ev_len, 1, n, nkeys, d_status, d_cap_off,
                                d_cap_len, false);
}

int lc_regex_parse_strided_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                               const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint32_t ev_stride, uint64_t n,
                               uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off, uint32_t* d_cap_len) {
    if (ev_stride == 0)
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_strided_dev: ev_stride must be >= 1");
    return regex_parse_dev_impl(e, re, d_base, base_len, base_len, d_ev_off, d_ev_len, ev_stride, n, nkeys, d_status,
                                d_cap_off, d_cap_len, false);
}

int lc_regex_match_dev(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                       const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint8_t* d_out_match) {
    return regex_parse_dev_impl(e, re, d_base, base_len, base_len, d_ev_off, d_ev_len, 1, n, 0, d_out_match, nullptr,
                                nullptr, true);
}

int lc_regex_match(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                   const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint8_t* out_match) {
    if (!e || !re || (n && (!ev_off || !ev_len || !out_match)) || (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_match: bad arguments");
    int rc = check_regex_usable(re, "lc_regex_match");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    rc = check_events(ev_off, ev_len, n, base_len, "lc_regex_match");
    if (rc)
        return rc;
    rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    rc = lc_regex_match_dev(e, re, e->in.as<uint8_t>(), base_len, e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                            e->out_a.as<uint8_t>());
    if (rc)
        return rc;
    CU_TRY(cudaMemcpyAsync(out_match, e->out_a.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// gathers a strided event table into the engine's dense scratch tables (the two-pass fall-back kernels take dense
// tables only)
static int densify_events(lc_engine_t* e, const uint32_t*& d_ev_off, const uint32_t*& d_ev_len, uint32_t ev_stride,
                          uint64_t n) {
    CU_TRY(e->lines_off.ensure(n * 4));
    CU_TRY(e->lines_len.ensure(n * 4));
    CU_TRY(cudaMemcpy2DAsync(e->lines_off.p, 4, d_ev_off, (size_t)ev_stride * 4, 4, n, cudaMemcpyDeviceToDevice,
                             e->stream));
    CU_TRY(cudaMemcpy2DAsync(e->lines_len.p, 4, d_ev_len, (size_t)ev_stride * 4, 4, n, cudaMemcpyDeviceToDevice,
                             e->stream));
    d_ev_off = e->lines_off.as<uint32_t>();
    d_ev_len = e->lines_len.as<uint32_t>();
    return LC_OK;
}

static int regex_parse_dev_impl(lc_engine_t* e, const lc_regex_t* re, const uint8_t* d_base, uint64_t base_len,
                                uint64_t span_bytes, const uint32_t* d_ev_off, const uint32_t* d_ev_len,
                                uint32_t ev_stride, uint64_t n, uint32_t nkeys, uint8_t* d_status, uint32_t* d_cap_off,
                                uint32_t* d_cap_len, bool bool_only) {
    if (!e || !re)
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_dev: bad arguments");
    int rc = check_regex_usable(re, "lc_regex_parse");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB and < 2^30 events per call");
    rc = bind(e);
    if (rc)
        return rc;
    const void* d_blob;
    CU_TRY(engine_blob(e, re, &d_blob));
    const LcRegexHeader* h = reinterpret_cast<const LcRegexHeader*>(re->res.blob.data());
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    const bool force_basic = e->force_basic_regex;
    const size_t smem_max = (size_t)e->smem_per_block_optin;
    // ---- single-pass tagged DFA: the preferred kernel whenever the pattern's TDFA fits shared memory.  Nothing on
    // this path waits for the device: ragged-batch ordering is decided by a device-side flag and events too long for
    // the 16-bit capture registers are redone by a follow-up kernel that exits at once when there was none.
    if (!force_basic && (e->regex_variant == 0 || e->regex_variant == 4) && !re->res.tdfa_blob.empty()) {
        const LcTdfaHeader* th = reinterpret_cast<const LcTdfaHeader*>(re->res.tdfa_blob.data());
        const uint32_t tb = (uint32_t)re->res.tdfa_blob.size();
        auto smem_need = [&](uint32_t warps) { return lck::tdfa_staged_smem_bytes(tb, th->nregs, warps * 32); };
        uint32_t warps = e->max_warps;
        while (warps > 4 && smem_need(warps) > smem_max)
            warps -= 2;
        if (smem_need(warps) <= smem_max) {
            const void* d_tblob;
            CU_TRY(engine_blob(e, re, &d_tblob, 3));
            const uint32_t threads = warps * 32;
            const uint64_t need_blocks = (n + threads - 1) / threads;
            const uint32_t grid = (uint32_t)std::min<uint64_t>(need_blocks, (uint64_t)e->num_sms);
            // Ragged batches of long lines: a warp costs its longest line, so visit the events by descending length
            // bucket.  Only built when the mean length makes the three small pre-pass kernels negligible; the scan
            // kernel leaves a flag saying whether the lengths really are ragged, which the regex kernel reads.
            // LC_B200_LENGTH_ORDER=1 forces the pre-pass, =0 disables it.
            const uint32_t* d_order = nullptr;
            const uint32_t* d_order_flag = nullptr;
            if (ev_stride == 1 && n >= 4096 && e->length_order != 0 &&
                (e->length_order == 1 || span_bytes / n >= 1024)) {
                CU_TRY(e->order.ensure(n * 4 + 512));
                uint32_t* hist = e->order.as<uint32_t>() + n;
                lck::launch_length_order(d_ev_len, n, hist, e->order.as<uint32_t>(), e->stream);
                e->launches += 3;
                d_order = e->order.as<uint32_t>();
                d_order_flag = e->length_order == 1 ? nullptr : hist + 64;
            }
            CU_TRY(cudaMemsetAsync(&ds->overflow, 0, offsetof(Small, total_chars) - offsetof(Small, overflow),
                                   e->stream));
            int er = lck::launch_regex_tdfa_staged(d_tblob, tb, th->has_slow != 0, th->nregs, d_base, d_ev_off,
                                                   d_ev_len, ev_stride, n, nkeys, d_status,
                                                   bool_only ? nullptr : d_cap_off, bool_only ? nullptr : d_cap_len,
                                                   threads, grid, &ds->next_batch, &ds->overflow, d_order,
                                                   d_order_flag, e->stream);
            e->launches++;
            if (er)
                return fail(LC_ERR_CUDA, std::string("regex kernel launch: ") + cudaGetErrorString((cudaError_t)er));
            if (base_len >= 65535) {
                lck::TdfaMultiArgs ma;
                memset(&ma, 0, sizeof ma);
                ma.blob[0] = d_tblob;
                ma.blob_bytes[0] = tb;
                ma.nkeys[0] = nkeys;
                ma.npat = 1;
                lck::launch_regex_tdfa_long(ma, d_base, d_ev_off, d_ev_len, ev_stride, n, nullptr, nullptr, d_status,
                                            d_cap_off, d_cap_len, th->ngroups, &ds->overflow, bool_only, e->stream);
                e->launches++;
                CU_TRY(cudaGetLastError());
            }
            return LC_OK;
        }
    }
    if (ev_stride != 1) {
        rc = densify_events(e, d_ev_off, d_ev_len, ev_stride, n);
        if (rc)
            return rc;
    }
    if (!force_basic) {
        // ---- pick the kernel variant: stride-2 layout > stride-1 fast layout > generic shared-memory interpreter
        uint64_t mx = 0, avg = span_bytes / n + 1;
        if (h->mode == LC_MODE_TWOPASS) {
            // size the per-thread label area from the actual length distribution: cover the longest event when
            // the batch is near-uniform, else ~1.25x the mean (longer events spill to the global slab)
            CU_TRY(cudaMemsetAsync(ds->counters, 0, sizeof ds->counters, e->stream));
            lck::launch_len_stats(d_ev_len, n, ds->counters, e->stream);
            e->launches++;
            CU_TRY(cudaMemcpyAsync(hs->counters, ds->counters, sizeof ds->counters, cudaMemcpyDeviceToHost,
                                   e->stream));
            CU_TRY(cudaStreamSynchronize(e->stream));
            mx = hs->counters[0];
            avg = hs->counters[1] / n + 1;
        }
        const uint64_t cover = (mx <= avg + avg / 2 + 64) ? mx : (avg + avg / 4);
        enum { V_FAST2, V_FAST, V_GENERIC } variant = V_GENERIC;
        if (e->regex_variant == 0 || e->regex_variant == 2)
            if (!re->res.fast2_blob.empty() && mx < 65535 && re->res.fast2_blob.size() + 32768 <= smem_max)
                variant = V_FAST2;
        if (variant == V_GENERIC && (e->regex_variant == 0 || e->regex_variant == 1) && !re->res.fast_blob.empty() &&
            re->res.fast_blob.size() + 32768 <= smem_max)
            variant = V_FAST;
        const std::vector<uint8_t>& vb =
            variant == V_FAST2 ? re->res.fast2_blob : (variant == V_FAST ? re->res.fast_blob : re->res.blob);
        bool convert_status = false;
        if (bool_only && variant != V_FAST2) { // these kernels always write captures: give them scratch tables
            CU_TRY(e->out_d.ensure(n * h->ngroups * 4 + 4));
            CU_TRY(e->out_e.ensure(n * h->ngroups * 4 + 4));
            d_cap_off = e->out_d.as<uint32_t>();
            d_cap_len = e->out_e.as<uint32_t>();
            convert_status = true;
        }
        const uint32_t blob_bytes = (uint32_t)vb.size();
        if (blob_bytes + 4096 <= smem_max) {
            const void* d_vblob = d_blob;
            if (variant != V_GENERIC)
                CU_TRY(engine_blob(e, re, &d_vblob, variant == V_FAST2 ? 2 : 1));
            // labels per 32-bit word: stride-2 -> 8 bytes of input, stride-1 u8 -> 4, u16 -> 2
            const uint32_t per = variant == V_FAST2 ? 8u
                                                    : ((h->mode == LC_MODE_TWOPASS && h->rev_label_bytes == 2 &&
                                                        variant == V_GENERIC)
                                                           ? 2u
                                                           : 4u);
            uint32_t lab_words = 0, threads = 512, blocks_per_sm = 2;
            size_t slot_bytes = 0; // per warp
            if (h->mode == LC_MODE_TWOPASS) {
                lab_words = (uint32_t)((cover + 15) / per + 2); // + 15: labels are shifted by the 16 B misalignment
                if (lab_words < 8)
                    lab_words = 8;
                if (variant == V_FAST2)
                    slot_bytes = (size_t)32 * lck::fast2_slot_pitch(h->ngroups) * 2;
                else if (variant == V_FAST)
                    slot_bytes = (size_t)32 * lck::fast_slot_pitch(h->ngroups) * 4;
                size_t budget = smem_max - blob_bytes - 1024;
                uint32_t warps = (uint32_t)(budget / ((size_t)lab_words * 128 + slot_bytes));
                // Long lines: labels in shared memory would leave a handful of resident warps (many times
                // slower).  Keep >= kMinWarps warps resident and let events that do not fit keep their labels in
                // the global slab instead (L2-resident while in flight; +1 B of traffic per input byte worst case).
                // The stride-2 kernel evaluates oversized events in checkpointed blocks (labels of one block only),
                // so it can afford the full 32 warps; the others keep whole-event labels in the global slab.
                const uint32_t kMinWarps = variant == V_FAST2 ? 32 : 20;
                if (warps < kMinWarps) {
                    warps = kMinWarps;
                    size_t per_warp = budget / kMinWarps;
                    lab_words = per_warp > slot_bytes + 8 * 128 ? (uint32_t)((per_warp - slot_bytes) / 128) : 8;
                    while (warps > 4 && (size_t)warps * ((size_t)lab_words * 128 + slot_bytes) > budget)
                        --warps;
                }
                if (warps > e->max_warps)
                    warps = e->max_warps;
                threads = warps * 32;
                blocks_per_sm = 1;
                if (warps <= 16 && 2 * (blob_bytes + (size_t)warps * (lab_words * 128 + slot_bytes) + 1024) <=
                                       (size_t)e->smem_per_sm)
                    blocks_per_sm = 2;
            }
            uint64_t need_blocks = (n + threads - 1) / threads;
            uint32_t grid = (uint32_t)std::min<uint64_t>(need_blocks, (uint64_t)e->num_sms * blocks_per_sm);
            // global label slab for events longer than the shared-memory budget: start small, remember what worked
            uint64_t full = span_bytes / per + 2 * n + 1024;
            uint64_t scratch_words = std::max<uint64_t>(e->scratch_hint, std::min<uint64_t>(full, 16ull << 20));
            if (h->mode == LC_MODE_TWOPASS && (mx + 15) / per + 2 > lab_words) {
                // some events spill: provision the upper bound of what ALL events could need (no retry runs)
                uint64_t bound = (hs->counters[1] + 16 * n) / per + 2 * n + 1024;
                if (variant == V_FAST2) // checkpointed blocks: 2 B per (lab_words * 8)-byte block of a long event
                    bound = 4 * n + hs->counters[1] / 32 + 1024;
                scratch_words = std::max(scratch_words, bound);
            }
            // ragged batch: visit events in descending length-bucket order (a warp costs its longest line)
            const uint32_t* d_order = nullptr;
            // (slower on C5, Zipf 64 B-8 KB: the scattered visiting order costs more L2 locality than the
            //  balanced warps win -- kept opt-in: LC_B200_LENGTH_ORDER=1)
            if (e->length_order == 1 && h->mode == LC_MODE_TWOPASS && mx > 2 * avg + 64 && n >= 4096) {
                CU_TRY(e->order.ensure(n * 4 + 512));
                uint32_t* hist = e->order.as<uint32_t>() + n;
                lck::launch_length_order(d_ev_len, n, hist, e->order.as<uint32_t>(), e->stream);
                e->launches += 3;
                d_order = e->order.as<uint32_t>();
            }
            for (int attempt = 0; attempt < 8; ++attempt) {
                if (h->mode == LC_MODE_TWOPASS)
                    CU_TRY(e->lab.ensure(scratch_words * 4));
                CU_TRY(cudaMemsetAsync(&ds->overflow, 0, offsetof(Small, total_chars) - offsetof(Small, overflow), e->stream));
                int er;
                if (variant == V_FAST2) {
                    const LcFast2Header* f2h = reinterpret_cast<const LcFast2Header*>(vb.data());
                    const bool multi = f2h->has_multi != 0;
                    er = lck::launch_regex_fast2(d_vblob, blob_bytes, multi, f2h->pair_shift == 2, h->ngroups, d_base,
                                                 d_ev_off, d_ev_len, n,
                                                 nkeys, d_status, d_cap_off, d_cap_len, lab_words, threads, grid,
                                                 e->lab.as<uint32_t>(), scratch_words, &ds->bump, &ds->overflow,
                                                 &ds->next_batch, d_order, e->stream);
                } else if (variant == V_FAST) {
                    const bool multi = reinterpret_cast<const LcFastHeader*>(vb.data())->reserved[0] != 0;
                    er = lck::launch_regex_twopass_fast(d_vblob, blob_bytes, multi, h->ngroups, d_base, d_ev_off,
                                                        d_ev_len, n, nkeys, d_status, d_cap_off, d_cap_len, lab_words,
                                                        threads, grid, e->lab.as<uint32_t>(), scratch_words, &ds->bump,
                                                        &ds->overflow, &ds->next_batch, d_order, e->stream);
                } else {
                    er = lck::launch_regex_parse_fast(d_vblob, blob_bytes, h->rev_label_bytes, h->ngroups, d_base,
                                                      d_ev_off, d_ev_len, n, nkeys, d_status, d_cap_off, d_cap_len,
                                                      lab_words, threads, grid, e->lab.as<uint32_t>(), scratch_words,
                                                      &ds->bump, &ds->overflow, &ds->next_batch, d_order, e->stream);
                }
                e->launches++;
                if (er)
                    return fail(LC_ERR_CUDA,
                                std::string("regex kernel launch: ") + cudaGetErrorString((cudaError_t)er));
                if (h->mode != LC_MODE_TWOPASS) {
                    if (convert_status) {
                        lck::launch_status_to_bool(d_status, n, e->stream);
                        e->launches++;
                    }
                    return LC_OK;
                }
                CU_TRY(cudaMemcpyAsync(&hs->overflow, &ds->overflow, 4, cudaMemcpyDeviceToHost, e->stream));
                CU_TRY(cudaStreamSynchronize(e->stream));
                if (!hs->overflow) {
                    e->scratch_hint = scratch_words;
                    if (convert_status) {
                        lck::launch_status_to_bool(d_status, n, e->stream);
                        e->launches++;
                    }
                    return LC_OK;
                }
                scratch_words = scratch_words < full ? std::min<uint64_t>(full, scratch_words * 4) : scratch_words * 2;
            }
            return fail(LC_ERR_CUDA, "label scratch exhausted after retries");
        }
    }
    // ---- baseline kernel (tables in global memory); kept for A/B checks and for automata beyond shared memory
    const uint64_t* d_lab_off = nullptr;
    uint16_t* d_lab = nullptr;
    if (h->mode == LC_MODE_TWOPASS) {
        uint64_t* desc;
        rc = prep_desc(e, lck::scan_tiles(n), &desc);
        if (rc)
            return rc;
        CU_TRY(e->lab_sizes.ensure(n * 4));
        CU_TRY(e->lab_off.ensure(n * 8));
        lck::launch_label_sizes(d_ev_len, n, e->lab_sizes.as<uint32_t>(), e->stream);
        lck::launch_exclusive_sum(e->lab_sizes.as<uint32_t>(), n, e->lab_off.as<uint64_t>(), &ds->total, desc,
                                  &ds->tickets[2], e->stream);
        e->launches += 2;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        CU_TRY(e->lab.ensure(hs->total * 2 + 16));
        d_lab_off = e->lab_off.as<uint64_t>();
        d_lab = e->lab.as<uint16_t>();
    }
    if (bool_only) {
        CU_TRY(e->out_d.ensure(n * h->ngroups * 4 + 4));
        CU_TRY(e->out_e.ensure(n * h->ngroups * 4 + 4));
        d_cap_off = e->out_d.as<uint32_t>();
        d_cap_len = e->out_e.as<uint32_t>();
    }
    lck::launch_regex_parse_basic(d_blob, h->mode, h->ngroups, d_base, d_ev_off, d_ev_len, n, nkeys, d_status,
                                  d_cap_off, d_cap_len, d_lab_off, d_lab, e->stream);
    e->launches++;
    if (bool_only) {
        lck::launch_status_to_bool(d_status, n, e->stream);
        e->launches++;
    }
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

} // extern "C"

// Pipelined host-pointer batch: the arena is cut into chunks of whole events; chunk c's bytes and event table go up on a
// copy stream, its kernels run on the engine stream as soon as they have landed, and its result tables travel back on
// a third stream while later chunks are still being uploaded (PCIe is full duplex).  `run(c, i0, cnt, span)` queues
// the chunk's kernels; `down(c, i0, cnt)` queues its D2H copies on s_d2h.  Event ranges are validated chunk by chunk
// right before their upload is queued, so the check overlaps the copies of the previous chunks.
template <class Run, class Down>
static int pipelined_events(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                            const uint32_t* ev_len, uint64_t n, uint64_t nchunks, const char* what, Run run, Down down) {
    int rc = ensure_copy_streams(e, (int)nchunks);
    if (rc)
        return rc;
    uint8_t* d_in = e->in.as<uint8_t>();
    uint32_t* d_off = e->ev_off.as<uint32_t>();
    uint32_t* d_len = e->ev_len.as<uint32_t>();
    // every exit path drains the copy streams: they read and write caller buffers
    auto drain = [&](int code) {
        cudaStreamSynchronize(e->s_h2d);
        cudaStreamSynchronize(e->stream);
        cudaStreamSynchronize(e->s_d2h);
        return code;
    };
    // the engine stream may still be reading the workspace on behalf of an earlier asynchronous call
    cudaEvent_t ev0 = e->ev_comp[0];
    if (cudaEventRecord(ev0, e->stream) != cudaSuccess || cudaStreamWaitEvent(e->s_h2d, ev0, 0) != cudaSuccess)
        return fail(LC_ERR_CUDA, "stream ordering failed");
    for (uint64_t c = 0; c < nchunks; ++c) {
        const uint64_t i0 = n * c / nchunks, i1 = n * (c + 1) / nchunks, cnt = i1 - i0;
        uint64_t lo = ~0ull, hi = 0;
        for (uint64_t i = i0; i < i1; ++i) {
            const uint64_t o = ev_off[i], en = o + ev_len[i];
            lo = o < lo ? o : lo;
            hi = en > hi ? en : hi;
        }
        if (hi > base_len)
            return drain(fail(LC_ERR_INVALID_ARG, std::string(what) + ": event beyond base_len"));
        lo = lo == ~0ull ? 0 : (lo & ~15ull);
#define LC_PIPE_TRY(expr)                                                                                              \
    do {                                                                                                               \
        cudaError_t _e = (expr);                                                                                       \
        if (_e != cudaSuccess)                                                                                         \
            return drain(fail(LC_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)));                        \
    } while (0)
        if (hi > lo)
            LC_PIPE_TRY(cudaMemcpyAsync(d_in + lo, base + lo, hi - lo, cudaMemcpyHostToDevice, e->s_h2d));
        LC_PIPE_TRY(cudaMemcpyAsync(d_off + i0, ev_off + i0, cnt * 4, cudaMemcpyHostToDevice, e->s_h2d));
        LC_PIPE_TRY(cudaMemcpyAsync(d_len + i0, ev_len + i0, cnt * 4, cudaMemcpyHostToDevice, e->s_h2d));
        LC_PIPE_TRY(cudaEventRecord(e->ev_h2d[c], e->s_h2d));
        LC_PIPE_TRY(cudaStreamWaitEvent(e->stream, e->ev_h2d[c], 0));
        rc = run(c, i0, cnt, hi > lo ? hi - lo : 0);
        if (rc)
            return drain(rc);
        LC_PIPE_TRY(cudaEventRecord(e->ev_comp[c], e->stream));
        LC_PIPE_TRY(cudaStreamWaitEvent(e->s_d2h, e->ev_comp[c], 0));
        rc = down(c, i0, cnt);
        if (rc)
            return drain(rc);
#undef LC_PIPE_TRY
    }
    CU_TRY(cudaStreamSynchronize(e->s_d2h));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

static uint64_t pipeline_chunks(uint64_t base_len, uint64_t n) {
    const uint64_t kChunkBytes = 48ull << 20;
    uint64_t nchunks = (base_len + kChunkBytes - 1) / kChunkBytes;
    if (nchunks > 64)
        nchunks = 64;
    if (nchunks < 2 || n < nchunks * 1024)
        return 1;
    return nchunks;
}

extern "C" {

int lc_regex_parse(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                   const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint32_t nkeys, uint8_t* status,
                   uint32_t* cap_off, uint32_t* cap_len) {
    if (!e || !re || (n && (!ev_off || !ev_len || !status)) || (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse: bad arguments");
    int rc = check_regex_usable(re, "lc_regex_parse");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    const uint32_t G = re->res.ngroups;
    if (G && (!cap_off || !cap_len))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse: bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB and < 2^30 events per call");
    rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * G * 4 + 4));
    CU_TRY(e->out_c.ensure(n * G * 4 + 4));
    const uint64_t nchunks = pipeline_chunks(base_len, n);
    if (nchunks == 1) {
        rc = check_events(ev_off, ev_len, n, base_len, "lc_regex_parse");
        if (rc)
            return rc;
        CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
        rc = lc_regex_parse_dev(e, re, e->in.as<uint8_t>(), base_len, e->ev_off.as<uint32_t>(),
                                e->ev_len.as<uint32_t>(), n, nkeys, e->out_a.as<uint8_t>(), e->out_b.as<uint32_t>(),
                                e->out_c.as<uint32_t>());
        if (rc) {
            cudaStreamSynchronize(e->stream);
            return rc;
        }
        CU_TRY(cudaMemcpyAsync(status, e->out_a.p, n, cudaMemcpyDeviceToHost, e->stream));
        if (G) {
            CU_TRY(cudaMemcpyAsync(cap_off, e->out_b.p, n * G * 4, cudaMemcpyDeviceToHost, e->stream));
            CU_TRY(cudaMemcpyAsync(cap_len, e->out_c.p, n * G * 4, cudaMemcpyDeviceToHost, e->stream));
        }
        CU_TRY(cudaStreamSynchronize(e->stream));
        return LC_OK;
    }
    uint8_t* d_in = e->in.as<uint8_t>();
    auto run = [&](uint64_t, uint64_t i0, uint64_t cnt, uint64_t span) {
        return regex_parse_dev_impl(e, re, d_in, base_len, span, e->ev_off.as<uint32_t>() + i0,
                                    e->ev_len.as<uint32_t>() + i0, 1, cnt, nkeys, e->out_a.as<uint8_t>() + i0,
                                    e->out_b.as<uint32_t>() + i0 * G, e->out_c.as<uint32_t>() + i0 * G, false);
    };
    auto down = [&](uint64_t, uint64_t i0, uint64_t cnt) {
        CU_TRY(cudaMemcpyAsync(status + i0, e->out_a.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, e->s_d2h));
        if (G) {
            CU_TRY(cudaMemcpyAsync(cap_off + i0 * G, e->out_b.as<uint32_t>() + i0 * G, cnt * G * 4,
                                   cudaMemcpyDeviceToHost, e->s_d2h));
            CU_TRY(cudaMemcpyAsync(cap_len + i0 * G, e->out_c.as<uint32_t>() + i0 * G, cnt * G * 4,
                                   cudaMemcpyDeviceToHost, e->s_d2h));
        }
        return (int)LC_OK;
    };
    return pipelined_events(e, base, base_len, ev_off, ev_len, n, nchunks, "lc_regex_parse", run, down);
}

// Batched event groups: span k (one group's arena bytes, ideally pinned: lc_host_alloc) is uploaded to
// [span_dst[k], + span_len[k]) of ONE packed device arena; the event table addresses the packed arena.  Chunks of
// ~32 MB of whole spans flow through the same three-stream pipeline as lc_regex_parse.
int lc_regex_parse_packed(lc_engine_t* e, const lc_regex_t* re, uint64_t nspans, const uint8_t* const* span_ptr,
                          const uint32_t* span_len, const uint32_t* span_dst, const uint64_t* span_first_ev,
                          uint64_t packed_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                          uint32_t nkeys, uint8_t* status, uint32_t* cap_off, uint32_t* cap_len) {
    return lc_regex_parse_packed_cb(e, re, nspans, span_ptr, span_len, span_dst, span_first_ev, packed_len, ev_off, ev_len,
                                    n, nkeys, status, cap_off, cap_len, nullptr, nullptr);
}

int lc_regex_parse_packed_cb(lc_engine_t* e, const lc_regex_t* re, uint64_t nspans, const uint8_t* const* span_ptr,
                             const uint32_t* span_len, const uint32_t* span_dst, const uint64_t* span_first_ev,
                             uint64_t packed_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                             uint32_t nkeys, uint8_t* status, uint32_t* cap_off, uint32_t* cap_len,
                             lc_spans_done_fn on_done, void* ctx) {
    if (!e || !re || (nspans && (!span_ptr || !span_len || !span_dst || !span_first_ev)) ||
        (n && (!ev_off || !ev_len || !status)))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_packed: bad arguments");
    int rc = check_regex_usable(re, "lc_regex_parse_packed");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    const uint32_t G = re->res.ngroups;
    if (G && (!cap_off || !cap_len))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_packed: bad arguments");
    if (packed_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "packed arena must be < 4 GiB and < 2^30 events per call");
    if (nspans == 0 || span_first_ev[0] != 0 || span_first_ev[nspans] != n)
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_packed: span_first_ev must cover [0, n]");
    rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(packed_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * G * 4 + 4));
    CU_TRY(e->out_c.ensure(n * G * 4 + 4));
    // chunk boundaries (in spans): ~32 MB of arena bytes each, at most 64 chunks
    std::vector<uint64_t> cut{0};
    {
        const uint64_t target = std::max<uint64_t>(32ull << 20, packed_len / 64 + 1);
        uint64_t acc = 0;
        for (uint64_t k = 0; k < nspans; ++k) {
            acc += span_len[k];
            if (acc >= target && k + 1 < nspans) {
                cut.push_back(k + 1);
                acc = 0;
            }
        }
        cut.push_back(nspans);
    }
    const uint64_t nchunks = cut.size() - 1;
    rc = ensure_copy_streams(e, (int)nchunks);
    if (rc)
        return rc;
    uint8_t* d_in = e->in.as<uint8_t>();
    uint32_t* d_off = e->ev_off.as<uint32_t>();
    uint32_t* d_len = e->ev_len.as<uint32_t>();
    auto drain = [&](int code) {
        cudaStreamSynchronize(e->s_h2d);
        cudaStreamSynchronize(e->stream);
        cudaStreamSynchronize(e->s_d2h);
        return code;
    };
#define LC_PIPE_TRY(expr)                                                                                              \
    do {                                                                                                               \
        cudaError_t _e = (expr);                                                                                       \
        if (_e != cudaSuccess)                                                                                         \
            return drain(fail(LC_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)));                        \
    } while (0)
    LC_PIPE_TRY(cudaEventRecord(e->ev_comp[0], e->stream));
    LC_PIPE_TRY(cudaStreamWaitEvent(e->s_h2d, e->ev_comp[0], 0));
    for (uint64_t c = 0; c < nchunks; ++c) {
        const uint64_t k0 = cut[c], k1 = cut[c + 1];
        const uint64_t i0 = span_first_ev[k0], i1 = span_first_ev[k1], cnt = i1 - i0;
        uint64_t span_bytes = 0;
        for (uint64_t k = k0; k < k1; ++k) {
            const uint64_t lo = span_dst[k], hi = lo + span_len[k];
            if ((lo & 15u) || hi > packed_len || span_first_ev[k] > span_first_ev[k + 1] ||
                (k + 1 < nspans && hi > span_dst[k + 1]))
                return drain(fail(LC_ERR_INVALID_ARG, "lc_regex_parse_packed: spans must be 16-byte aligned, ordered "
                                                      "and inside the packed arena"));
            for (uint64_t i = span_first_ev[k]; i < span_first_ev[k + 1]; ++i)
                if (ev_off[i] < lo || (uint64_t)ev_off[i] + ev_len[i] > hi)
                    return drain(fail(LC_ERR_INVALID_ARG, "lc_regex_parse_packed: event outside its span"));
            if (span_len[k])
                LC_PIPE_TRY(cudaMemcpyAsync(d_in + lo, span_ptr[k], span_len[k], cudaMemcpyHostToDevice, e->s_h2d));
            span_bytes += span_len[k];
        }
        if (cnt) {
            LC_PIPE_TRY(cudaMemcpyAsync(d_off + i0, ev_off + i0, cnt * 4, cudaMemcpyHostToDevice, e->s_h2d));
            LC_PIPE_TRY(cudaMemcpyAsync(d_len + i0, ev_len + i0, cnt * 4, cudaMemcpyHostToDevice, e->s_h2d));
        }
        LC_PIPE_TRY(cudaEventRecord(e->ev_h2d[c], e->s_h2d));
        if (!cnt) {
            LC_PIPE_TRY(cudaEventRecord(e->ev_d2h[c], e->s_d2h));
            continue;
        }
        LC_PIPE_TRY(cudaStreamWaitEvent(e->stream, e->ev_h2d[c], 0));
        rc = regex_parse_dev_impl(e, re, d_in, packed_len, span_bytes, d_off + i0, d_len + i0, 1, cnt, nkeys,
                                  e->out_a.as<uint8_t>() + i0, e->out_b.as<uint32_t>() + i0 * G,
                                  e->out_c.as<uint32_t>() + i0 * G, false);
        if (rc)
            return drain(rc);
        LC_PIPE_TRY(cudaEventRecord(e->ev_comp[c], e->stream));
        LC_PIPE_TRY(cudaStreamWaitEvent(e->s_d2h, e->ev_comp[c], 0));
        LC_PIPE_TRY(cudaMemcpyAsync(status + i0, e->out_a.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, e->s_d2h));
        if (G) {
            LC_PIPE_TRY(cudaMemcpyAsync(cap_off + i0 * G, e->out_b.as<uint32_t>() + i0 * G, cnt * G * 4,
                                        cudaMemcpyDeviceToHost, e->s_d2h));
            LC_PIPE_TRY(cudaMemcpyAsync(cap_len + i0 * G, e->out_c.as<uint32_t>() + i0 * G, cnt * G * 4,
                                        cudaMemcpyDeviceToHost, e->s_d2h));
        }
        LC_PIPE_TRY(cudaEventRecord(e->ev_d2h[c], e->s_d2h));
    }
    if (on_done) {
        // hand the chunks back in order as their result tables land, while later chunks are still on the GPU
        for (uint64_t c = 0; c < nchunks; ++c) {
            LC_PIPE_TRY(cudaEventSynchronize(e->ev_d2h[c]));
            on_done(ctx, cut[c], cut[c + 1] - cut[c]);
        }
    }
#undef LC_PIPE_TRY
    return drain(LC_OK);
}

// ------------------------------------------------------------------------------------------------ multi-pattern
int lc_regex_parse_multi_dev(lc_engine_t* e, const lc_regex_t* const* res, uint32_t npat, const uint32_t* nkeys,
                             const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                             const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_sel, uint8_t* d_which,
                             uint8_t* d_status, uint32_t row_pitch, uint32_t* d_cap_off, uint32_t* d_cap_len) {
    if (!e || !res || !nkeys || npat == 0 || npat > lck::LC_MULTI_MAX)
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_multi_dev: bad arguments (1..8 patterns)");
    int rc;
    uint32_t gmax = 0, max_nregs = 0;
    bool slow = false;
    for (uint32_t p = 0; p < npat; ++p) {
        if (!res[p])
            return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_multi_dev: NULL pattern");
        if ((rc = check_regex_usable(res[p], "lc_regex_parse_multi")))
            return rc;
        if (res[p]->res.tdfa_blob.empty())
            return fail(LC_ERR_REGEX_UNSUPPORTED,
                        "lc_regex_parse_multi: pattern " + std::to_string(p) +
                            " has no single-pass tables (too many states / registers); parse it with lc_regex_parse");
        const LcTdfaHeader* th = reinterpret_cast<const LcTdfaHeader*>(res[p]->res.tdfa_blob.data());
        gmax = std::max(gmax, th->ngroups);
        max_nregs = std::max(max_nregs, th->nregs);
        slow = slow || th->has_slow != 0;
    }
    if (row_pitch < gmax)
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_multi_dev: row_pitch smaller than the largest group count");
    if (n == 0)
        return LC_OK;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB and < 2^30 events per call");
    rc = bind(e);
    if (rc)
        return rc;
    Small* ds = e->small.as<Small>();
    const size_t smem_max = (size_t)e->smem_per_block_optin;
    lck::TdfaMultiArgs all;
    memset(&all, 0, sizeof all);
    all.npat = npat;
    for (uint32_t p = 0; p < npat; ++p) {
        CU_TRY(engine_blob(e, res[p], &all.blob[p], 3));
        all.blob_bytes[p] = (uint32_t)res[p]->res.tdfa_blob.size();
        all.nkeys[p] = nkeys[p];
    }
    // ragged batches: same device-side decision as the single-pattern path
    const uint32_t* d_order = nullptr;
    const uint32_t* d_order_flag = nullptr;
    if (n >= 4096 && e->length_order != 0 && (e->length_order == 1 || base_len / n >= 1024)) {
        CU_TRY(e->order.ensure(n * 4 + 512));
        uint32_t* hist = e->order.as<uint32_t>() + n;
        lck::launch_length_order(d_ev_len, n, hist, e->order.as<uint32_t>(), e->stream);
        e->launches += 3;
        d_order = e->order.as<uint32_t>();
        d_order_flag = e->length_order == 1 ? nullptr : hist + 64;
    }
    // Group consecutive patterns whose tables fit shared memory together (and below shared address 64 Ki: the pair
    // tables are addressed with 16 bits).  One group = one launch; normally everything is one group.
    uint32_t p0 = 0;
    bool first = true;
    while (p0 < npat) {
        lck::TdfaMultiArgs ga;
        memset(&ga, 0, sizeof ga);
        uint32_t warps = 0;
        uint32_t p1 = p0;
        while (p1 < npat) {
            lck::TdfaMultiArgs tryg = ga;
            tryg.blob[tryg.npat] = all.blob[p1];
            tryg.blob_bytes[tryg.npat] = all.blob_bytes[p1];
            tryg.nkeys[tryg.npat] = all.nkeys[p1];
            tryg.npat++;
            // last pair table must end below 64 Ki (LC_TDFA_REBASE_ROOM covers the window base and static shared memory)
            const bool addressable = LC_TDFA_REBASE_ROOM + lck::tdfa_multi_table_bytes(tryg) <= 65535u;
            uint32_t w = e->max_warps;
            while (w > 4 && lck::tdfa_multi_smem_bytes(tryg, max_nregs, w * 32) > smem_max)
                w -= 2;
            const bool fits = lck::tdfa_multi_smem_bytes(tryg, max_nregs, w * 32) <= smem_max && w >= 16;
            if (tryg.npat > 1 && (!(addressable && fits) || e->multi_split))
                break;
            if (tryg.npat == 1 && lck::tdfa_multi_smem_bytes(tryg, max_nregs, w * 32) > smem_max)
                return fail(LC_ERR_REGEX_UNSUPPORTED, "lc_regex_parse_multi: tables do not fit shared memory");
            ga = tryg;
            warps = w;
            ++p1;
        }
        const uint32_t threads = warps * 32;
        const uint32_t grid = (uint32_t)std::min<uint64_t>((n + threads - 1) / threads, (uint64_t)e->num_sms);
        CU_TRY(cudaMemsetAsync(&ds->next_batch, 0, sizeof ds->next_batch, e->stream));
        if (first)
            CU_TRY(cudaMemsetAsync(&ds->overflow, 0, sizeof ds->overflow, e->stream));
        int er = lck::launch_regex_tdfa_multi(ga, p0, !first, slow, max_nregs, d_base, d_ev_off, d_ev_len, n, d_sel,
                                              d_which, d_status, d_cap_off, d_cap_len, row_pitch, threads, grid,
                                              &ds->next_batch, &ds->overflow, d_order, d_order_flag, e->stream);
        e->launches++;
        if (er)
            return fail(LC_ERR_CUDA, std::string("regex kernel launch: ") + cudaGetErrorString((cudaError_t)er));
        first = false;
        p0 = p1;
    }
    if (base_len >= 65535) {
        lck::launch_regex_tdfa_long(all, d_base, d_ev_off, d_ev_len, 1, n, d_sel, d_which, d_status, d_cap_off,
                                    d_cap_len, row_pitch, &ds->overflow, false, e->stream);
        e->launches++;
        CU_TRY(cudaGetLastError());
    }
    return LC_OK;
}

int lc_regex_parse_multi(lc_engine_t* e, const lc_regex_t* const* res, uint32_t npat, const uint32_t* nkeys,
                         const uint8_t* base, uint64_t base_len, const uint32_t* ev_off, const uint32_t* ev_len,
                         uint64_t n, const uint8_t* sel, uint8_t* which, uint8_t* status, uint32_t row_pitch,
                         uint32_t* cap_off, uint32_t* cap_len) {
    if (!e || !res || !nkeys || (n && (!ev_off || !ev_len || !status || !which)) || (base_len && !base) ||
        (n && row_pitch && (!cap_off || !cap_len)))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_multi: bad arguments");
    if (n == 0)
        return LC_OK;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB and < 2^30 events per call");
    int rc = bind(e);
    if (rc)
        return rc;
    const uint64_t G = row_pitch;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * G * 4 + 4));
    CU_TRY(e->out_c.ensure(n * G * 4 + 4));
    CU_TRY(e->out_d.ensure(n));
    CU_TRY(e->flags.ensure(n));
    if (sel) {
        for (uint64_t i = 0; i < n; ++i)
            if (sel[i] != 0xFFu && sel[i] >= npat)
                return fail(LC_ERR_INVALID_ARG, "lc_regex_parse_multi: selector names a pattern that does not exist");
        CU_TRY(cudaMemcpyAsync(e->flags.p, sel, n, cudaMemcpyHostToDevice, e->stream));
    }
    const uint8_t* d_sel = sel ? e->flags.as<uint8_t>() : nullptr;
    uint8_t* d_in = e->in.as<uint8_t>();
    const uint64_t nchunks = pipeline_chunks(base_len, n);
    auto run = [&](uint64_t, uint64_t i0, uint64_t cnt, uint64_t) {
        return lc_regex_parse_multi_dev(e, res, npat, nkeys, d_in, base_len, e->ev_off.as<uint32_t>() + i0,
                                        e->ev_len.as<uint32_t>() + i0, cnt, d_sel ? d_sel + i0 : nullptr,
                                        e->out_d.as<uint8_t>() + i0, e->out_a.as<uint8_t>() + i0, row_pitch,
                                        e->out_b.as<uint32_t>() + i0 * G, e->out_c.as<uint32_t>() + i0 * G);
    };
    auto down_on = [&](cudaStream_t st, uint64_t i0, uint64_t cnt) {
        CU_TRY(cudaMemcpyAsync(status + i0, e->out_a.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaMemcpyAsync(which + i0, e->out_d.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, st));
        if (G) {
            CU_TRY(cudaMemcpyAsync(cap_off + i0 * G, e->out_b.as<uint32_t>() + i0 * G, cnt * G * 4,
                                   cudaMemcpyDeviceToHost, st));
            CU_TRY(cudaMemcpyAsync(cap_len + i0 * G, e->out_c.as<uint32_t>() + i0 * G, cnt * G * 4,
                                   cudaMemcpyDeviceToHost, st));
        }
        return (int)LC_OK;
    };
    if (nchunks == 1) {
        rc = check_events(ev_off, ev_len, n, base_len, "lc_regex_parse_multi");
        if (rc)
            return rc;
        CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
        rc = run(0, 0, n, base_len);
        if (!rc)
            rc = down_on(e->stream, 0, n);
        cudaError_t er = cudaStreamSynchronize(e->stream);
        if (!rc && er != cudaSuccess)
            return fail(LC_ERR_CUDA, cudaGetErrorString(er));
        return rc;
    }
    auto down = [&](uint64_t, uint64_t i0, uint64_t cnt) { return down_on(e->s_d2h, i0, cnt); };
    return pipelined_events(e, base, base_len, ev_off, ev_len, n, nchunks, "lc_regex_parse_multi", run, down);
}

int lc_regex_prefix_match(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                          const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, uint8_t* out_match) {
    if (!e || !re || (n && (!ev_off || !ev_len || !out_match)) || (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_regex_prefix_match: bad arguments");
    int rc = check_regex_usable(re, "lc_regex_prefix_match");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    rc = check_events(ev_off, ev_len, n, base_len, "lc_regex_prefix_match");
    if (rc)
        return rc;
    rc = bind(e);
    if (rc)
        return rc;
    const void* d_blob;
    CU_TRY(engine_blob(e, re, &d_blob));
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    lck::launch_prefix_match(d_blob, e->in.as<uint8_t>(), e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                             e->out_a.as<uint8_t>(), e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out_match, e->out_a.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// ------------------------------------------------------------------------------------------------ multiline
int lc_multiline_split_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, const lc_regex_t* start,
                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, uint32_t* d_out_off,
                           uint32_t* d_out_len, uint8_t* d_out_flags, uint64_t cap, uint64_t* n_out,
                           uint64_t counters[3]) {
    if (!e || !n_out || (len && !d_buf))
        return fail(LC_ERR_INVALID_ARG, "lc_multiline_split_dev: bad arguments");
    *n_out = 0;
    int rc;
    for (const lc_regex_t* r : {start, cont, end})
        if (r && (rc = check_regex_usable(r, "lc_multiline_split")))
            return rc;
    if (len == 0)
        return LC_OK;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    rc = bind(e);
    if (rc)
        return rc;
    lck::MlConfig cfg;
    memset(&cfg, 0, sizeof cfg);
    CU_TRY(engine_blob(e, start, &cfg.blob_start));
    CU_TRY(engine_blob(e, cont, &cfg.blob_cont));
    CU_TRY(engine_blob(e, end, &cfg.blob_end));
    cfg.discard = discard_unmatched;
    fill_probe_slot(cfg, 0, start);
    fill_probe_slot(cfg, 1, cont);
    fill_probe_slot(cfg, 2, end);

    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    // Two steps, no host round trip in between: (1) split + per-line probes, (2) the multiline passes (state scan,
    // counts, slots, emission), which read the line count from device memory.  The line table is sized from an
    // estimate and the call repeats with the exact size in the rare case it was too small.
    uint64_t lcap = len / 24 + 4096;
    for (;;) {
        if (lcap > len)
            lcap = len;
        if (lcap > 0x3FFFFFF0ull)
            lcap = 0x3FFFFFF0ull;
        CU_TRY(e->lines_off.ensure((lcap + 1) * 4));
        CU_TRY(e->lines_len.ensure((lcap + 1) * 4));
        CU_TRY(e->flags.ensure(lcap + 1));
        CU_TRY(cudaMemsetAsync(e->small.p, 0, sizeof(Small), e->stream)); // n_out, total_chars, total, counters
        CU_TRY(e->split_scratch.ensure(lck::split_scratch_bytes(len, true)));
        e->launches += lck::launch_split_probe(cfg, d_buf, (uint32_t)len, e->lines_off.as<uint32_t>(),
                                               e->lines_len.as<uint32_t>(), e->flags.as<uint8_t>(), (uint32_t)lcap,
                                               &ds->n_out, &ds->total_chars, e->split_scratch.as<uint64_t>(),
                                               e->stream) - 1;
        CU_TRY(e->state.ensure((size_t)lck::ml_pass_scratch_bytes(lcap)));
        e->launches += 1 + lck::launch_ml_passes(cfg, e->flags.as<uint8_t>(), e->lines_off.as<uint32_t>(),
                                                 e->lines_len.as<uint32_t>(), &ds->n_out, (uint32_t)lcap,
                                                 (uint32_t)len, d_out_off, d_out_len, d_out_flags, cap,
                                                 e->state.as<uint64_t>(), ds->counters, &ds->total, e->stream);
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(hs, ds, sizeof(Small), cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        if (hs->total_chars >= (1ull << 30) - 2)
            return fail(LC_ERR_TOO_LARGE, "more than 2^30 lines in one call");
        if (hs->n_out <= lcap)
            break;
        lcap = hs->n_out;
    }
    *n_out = hs->total;
    if (counters) {
        counters[0] += hs->counters[0];
        counters[1] += hs->n_out;
        counters[2] += hs->counters[1];
    }
    if (*n_out > cap)
        return fail(LC_ERR_CAPACITY, "lc_multiline_split: output capacity too small");
    return LC_OK;
}

int lc_multiline_split(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                       const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, uint32_t* out_off,
                       uint32_t* out_len, uint8_t* out_flags, uint64_t cap, uint64_t* n_out, uint64_t counters[3]) {
    if (!e || !n_out || (len && !buf))
        return fail(LC_ERR_INVALID_ARG, "lc_multiline_split: bad arguments");
    *n_out = 0;
    if (len == 0)
        return LC_OK;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    int rc = bind(e);
    if (rc)
        return rc;
    uint64_t dcap = cap < len ? cap : len; // an output event covers at least one input byte or one line
    CU_TRY(e->in.ensure(len + 16));
    CU_TRY(e->out_a.ensure((dcap + 1) * 4));
    CU_TRY(e->out_b.ensure((dcap + 1) * 4));
    CU_TRY(e->out_c.ensure(dcap + 1));
    CU_TRY(cudaMemcpyAsync(e->in.p, buf, len, cudaMemcpyHostToDevice, e->stream));
    rc = lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,
                                e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), dcap, n_out,
                                counters);
    if (rc)
        return rc;
    if (*n_out) {
        CU_TRY(cudaMemcpyAsync(out_off, e->out_a.p, *n_out * 4, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaMemcpyAsync(out_len, e->out_b.p, *n_out * 4, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaMemcpyAsync(out_flags, e->out_c.p, *n_out, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    return LC_OK;
}

// ------------------------------------------------------------------------------------------------ last incomplete log
int lc_remove_last_incomplete_log_dev(lc_engine_t* e, const uint8_t* d_buf, uint64_t len, const lc_regex_t* start,
                                      const lc_regex_t* end, int allow_rollback, uint64_t* keep_bytes,
                                      int32_t* rollback_line_feeds) {
    if (!e || !keep_bytes || !rollback_line_feeds || (len && !d_buf))
        return fail(LC_ERR_INVALID_ARG, "lc_remove_last_incomplete_log_dev: bad arguments");
    int rc;
    for (const lc_regex_t* r : {start, end})
        if (r && (rc = check_regex_usable(r, "lc_remove_last_incomplete_log")))
            return rc;
    *keep_bytes = len;
    if (!allow_rollback || len == 0) // :1999-2001: nothing to do, the caller's count stays as it is
        return LC_OK;
    if (len >= 0x7FFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "chunk must be < 2 GiB (the reference's sizes are int32_t)");
    rc = bind(e);
    if (rc)
        return rc;
    lck::MlConfig cfg;
    memset(&cfg, 0, sizeof cfg);
    CU_TRY(engine_blob(e, start, &cfg.blob_start));
    cfg.blob_cont = nullptr;
    CU_TRY(engine_blob(e, end, &cfg.blob_end));
    cfg.discard = 0;
    fill_probe_slot(cfg, 0, start);
    fill_probe_slot(cfg, 2, end);
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    uint64_t lcap = len / 24 + 4096;
    for (;;) {
        if (lcap > len)
            lcap = len;
        CU_TRY(e->lines_off.ensure((lcap + 1) * 4));
        CU_TRY(e->lines_len.ensure((lcap + 1) * 4));
        CU_TRY(e->flags.ensure(lcap + 1));
        CU_TRY(cudaMemsetAsync(e->small.p, 0, sizeof(Small), e->stream)); // n_out, total_chars, counters
        CU_TRY(e->split_scratch.ensure(lck::split_scratch_bytes(len, true)));
        e->launches += lck::launch_split_probe(cfg, d_buf, (uint32_t)len, e->lines_off.as<uint32_t>(),
                                               e->lines_len.as<uint32_t>(), e->flags.as<uint8_t>(), (uint32_t)lcap,
                                               &ds->n_out, &ds->total_chars, e->split_scratch.as<uint64_t>(),
                                               e->stream) - 1;
        lck::launch_last_record(e->flags.as<uint8_t>(), e->lines_off.as<uint32_t>(), e->lines_len.as<uint32_t>(),
                                &ds->n_out, (uint32_t)lcap, (uint32_t)len, start != nullptr, end != nullptr,
                                ds->counters, e->stream);
        e->launches += 2;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(hs, ds, sizeof(Small), cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        if (hs->n_out <= lcap)
            break;
        lcap = hs->n_out;
    }
    *keep_bytes = hs->counters[0];
    *rollback_line_feeds = (int32_t)hs->counters[1];
    return LC_OK;
}

int lc_remove_last_incomplete_log(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                  const lc_regex_t* end, int allow_rollback, uint64_t* keep_bytes,
                                  int32_t* rollback_line_feeds) {
    if (!e || !keep_bytes || !rollback_line_feeds || (len && !buf))
        return fail(LC_ERR_INVALID_ARG, "lc_remove_last_incomplete_log: bad arguments");
    *keep_bytes = len;
    if (!allow_rollback || len == 0)
        return LC_OK;
    if (len >= 0x7FFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "chunk must be < 2 GiB (the reference's sizes are int32_t)");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(len + 16));
    CU_TRY(cudaMemcpyAsync(e->in.p, buf, len, cudaMemcpyHostToDevice, e->stream));
    return lc_remove_last_incomplete_log_dev(e, e->in.as<uint8_t>(), len, start, end, allow_rollback, keep_bytes,
                                             rollback_line_feeds);
}

// ------------------------------------------------------------------------------------------------ delimiter
int lc_delim_parse_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                       const uint32_t* d_ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                       uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* d_status,
                       uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len, uint32_t* d_f_dq) {
    return lc_delim_parse_tap_dev(e, d_base, base_len, d_ev_off, d_ev_len, n, sep, sep_len, quote, nkeys, extend,
                                  allow_short, max_fields, d_status, d_nfields, d_f_off, d_f_len, d_f_dq, 0xFFFFFFFFu,
                                  nullptr, nullptr);
}

int lc_delim_parse_tap_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                           const uint32_t* d_ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                           uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* d_status,
                           uint32_t* d_nfields, uint32_t* d_f_off, uint32_t* d_f_len, uint32_t* d_f_dq,
                           uint32_t tap_col, uint32_t* d_tap_off, uint32_t* d_tap_len) {
    if (!e || !sep || sep_len < 1 || sep_len > 4 || max_fields == 0 || ((d_tap_off == nullptr) != (d_tap_len == nullptr)) ||
        (d_tap_off && tap_col >= max_fields))
        return fail(LC_ERR_INVALID_ARG, "lc_delim_parse_dev: bad arguments (separator must be 1..4 bytes)");
    if (n == 0)
        return LC_OK;
    if (base_len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    int rc = bind(e);
    if (rc)
        return rc;
    lck::DelimConfig cfg;
    memset(&cfg, 0, sizeof cfg);
    memcpy(cfg.sep, sep, sep_len);
    cfg.sep_len = sep_len;
    cfg.quote = quote;
    cfg.nkeys = nkeys;
    cfg.extend = extend;
    cfg.allow_short = allow_short;
    cfg.max_fields = max_fields;
    cfg.tap_col = tap_col;
    cfg.tap_off = d_tap_off;
    cfg.tap_len = d_tap_len;
    Small* ds = e->small.as<Small>();
    CU_TRY(cudaMemsetAsync(&ds->next_batch, 0, sizeof ds->next_batch, e->stream));
    lck::launch_delim(cfg, d_base, d_ev_off, d_ev_len, n, d_status, d_nfields, d_f_off, d_f_len, d_f_dq,
                      &ds->next_batch, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int lc_delim_regex_chain(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                         const uint32_t* ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                         uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* status,
                         uint32_t* nfields, uint32_t* f_off, uint32_t* f_len, uint32_t* f_dq, uint32_t column,
                         const lc_regex_t* re, uint32_t regex_nkeys, uint8_t* re_status, uint32_t* cap_off,
                         uint32_t* cap_len) {
    if (!e || !re || !sep || sep_len < 1 || sep_len > 4 || max_fields == 0 || column >= max_fields ||
        (n && (!ev_off || !ev_len || !status || !nfields || !f_off || !f_len || !f_dq || !re_status)) ||
        (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_delim_regex_chain: bad arguments");
    int rc = check_regex_usable(re, "lc_delim_regex_chain");
    if (rc)
        return rc;
    if (n == 0)
        return LC_OK;
    const uint32_t G = re->res.ngroups;
    if (G && (!cap_off || !cap_len))
        return fail(LC_ERR_INVALID_ARG, "lc_delim_regex_chain: bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 columns per call");
    rc = bind(e);
    if (rc)
        return rc;
    const uint64_t MF = max_fields, fbytes = n * MF * 4;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * 4));
    CU_TRY(e->out_c.ensure(fbytes));
    CU_TRY(e->out_d.ensure(fbytes));
    CU_TRY(e->out_e.ensure(fbytes));
    CU_TRY(e->lines_off.ensure(n * 4)); // the tapped column = the regex stage's event table
    CU_TRY(e->lines_len.ensure(n * 4));
    CU_TRY(e->flags.ensure(n));
    CU_TRY(e->cnt.ensure(n * G * 4 + 4));
    CU_TRY(e->pos.ensure(n * G * 4 + 4));
    uint8_t* d_in = e->in.as<uint8_t>();
    auto run = [&](uint64_t, uint64_t i0, uint64_t cnt, uint64_t span) {
        int r = lc_delim_parse_tap_dev(e, d_in, base_len, e->ev_off.as<uint32_t>() + i0, e->ev_len.as<uint32_t>() + i0,
                                       cnt, sep, sep_len, quote, nkeys, extend, allow_short, max_fields,
                                       e->out_a.as<uint8_t>() + i0, e->out_b.as<uint32_t>() + i0,
                                       e->out_c.as<uint32_t>() + i0 * MF, e->out_d.as<uint32_t>() + i0 * MF,
                                       e->out_e.as<uint32_t>() + i0 * MF, column, e->lines_off.as<uint32_t>() + i0,
                                       e->lines_len.as<uint32_t>() + i0);
        if (r)
            return r;
        return regex_parse_dev_impl(e, re, d_in, base_len, span, e->lines_off.as<uint32_t>() + i0,
                                    e->lines_len.as<uint32_t>() + i0, 1, cnt, regex_nkeys, e->flags.as<uint8_t>() + i0,
                                    e->cnt.as<uint32_t>() + i0 * G, e->pos.as<uint32_t>() + i0 * G, false);
    };
    auto down = [&](uint64_t, uint64_t i0, uint64_t cnt) {
        CU_TRY(cudaMemcpyAsync(status + i0, e->out_a.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, e->s_d2h));
        CU_TRY(cudaMemcpyAsync(nfields + i0, e->out_b.as<uint32_t>() + i0, cnt * 4, cudaMemcpyDeviceToHost, e->s_d2h));
        CU_TRY(cudaMemcpyAsync(f_off + i0 * MF, e->out_c.as<uint32_t>() + i0 * MF, cnt * MF * 4, cudaMemcpyDeviceToHost,
                               e->s_d2h));
        CU_TRY(cudaMemcpyAsync(f_len + i0 * MF, e->out_d.as<uint32_t>() + i0 * MF, cnt * MF * 4, cudaMemcpyDeviceToHost,
                               e->s_d2h));
        CU_TRY(cudaMemcpyAsync(f_dq + i0 * MF, e->out_e.as<uint32_t>() + i0 * MF, cnt * MF * 4, cudaMemcpyDeviceToHost,
                               e->s_d2h));
        CU_TRY(cudaMemcpyAsync(re_status + i0, e->flags.as<uint8_t>() + i0, cnt, cudaMemcpyDeviceToHost, e->s_d2h));
        if (G) {
            CU_TRY(cudaMemcpyAsync(cap_off + i0 * G, e->cnt.as<uint32_t>() + i0 * G, cnt * G * 4, cudaMemcpyDeviceToHost,
                                   e->s_d2h));
            CU_TRY(cudaMemcpyAsync(cap_len + i0 * G, e->pos.as<uint32_t>() + i0 * G, cnt * G * 4, cudaMemcpyDeviceToHost,
                                   e->s_d2h));
        }
        return (int)LC_OK;
    };
    uint64_t nchunks = pipeline_chunks(base_len, n);
    if (nchunks > 1 && nchunks < 8 && n >= 8 * 1024)
        nchunks = 8; // the tables going back are as large as the arena going up: shorter chunks, earlier overlap
    return pipelined_events(e, base, base_len, ev_off, ev_len, n, nchunks, "lc_delim_regex_chain", run, down);
}

int lc_delim_parse(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                   const uint32_t* ev_len, uint64_t n, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                   uint32_t nkeys, int extend, int allow_short, uint32_t max_fields, uint8_t* status,
                   uint32_t* nfields, uint32_t* f_off, uint32_t* f_len, uint32_t* f_dq) {
    if (!e || (n && (!ev_off || !ev_len || !status || !nfields || !f_off || !f_len || !f_dq)) || (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_delim_parse: bad arguments");
    if (n == 0)
        return LC_OK;
    int rc = check_events(ev_off, ev_len, n, base_len, "lc_delim_parse");
    if (rc)
        return rc;
    rc = bind(e);
    if (rc)
        return rc;
    size_t fbytes = (size_t)n * max_fields * 4;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * 4));
    CU_TRY(e->out_c.ensure(fbytes));
    CU_TRY(e->out_d.ensure(fbytes));
    CU_TRY(e->out_e.ensure(fbytes));
    CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    rc = lc_delim_parse_dev(e, e->in.as<uint8_t>(), base_len, e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                            sep, sep_len, quote, nkeys, extend, allow_short, max_fields, e->out_a.as<uint8_t>(),
                            e->out_b.as<uint32_t>(), e->out_c.as<uint32_t>(), e->out_d.as<uint32_t>(),
                            e->out_e.as<uint32_t>());
    if (rc)
        return rc;
    CU_TRY(cudaMemcpyAsync(status, e->out_a.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(nfields, e->out_b.p, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(f_off, e->out_c.p, fbytes, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(f_len, e->out_d.p, fbytes, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(f_dq, e->out_e.p, fbytes, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

int lc_sls_serialize_logs(lc_engine_t* e, const uint8_t* base, uint64_t base_len, uint64_t n, const uint32_t* ev_time,
                          const uint32_t* ev_time_ns, const uint64_t* ent_begin, const uint32_t* ent_koff,
                          const uint32_t* ent_klen, const uint32_t* ent_voff, const uint32_t* ent_vlen, uint8_t* out,
                          uint64_t out_cap, uint64_t* out_len) {
    if (!e || !out_len || (n && (!ev_time || !ent_begin)) || (base_len && !base))
        return fail(LC_ERR_INVALID_ARG, "lc_sls_serialize_logs: bad arguments");
    *out_len = 0;
    if (n == 0)
        return LC_OK;
    const uint64_t m = ent_begin[n];
    if (m && (!ent_koff || !ent_klen || !ent_voff || !ent_vlen))
        return fail(LC_ERR_INVALID_ARG, "lc_sls_serialize_logs: bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || m >= (1ull << 31))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^31 contents per call");
    for (uint64_t i = 0; i < n; ++i)
        if (ent_begin[i] > ent_begin[i + 1])
            return fail(LC_ERR_INVALID_ARG, "lc_sls_serialize_logs: ent_begin must be non-decreasing");
    if (ent_begin[0] != 0)
        return fail(LC_ERR_INVALID_ARG, "lc_sls_serialize_logs: ent_begin[0] must be 0");
    int rc = check_events(ent_koff, ent_klen, m, base_len, "lc_sls_serialize_logs (keys)");
    if (!rc)
        rc = check_events(ent_voff, ent_vlen, m, base_len, "lc_sls_serialize_logs (values)");
    if (rc)
        return rc;
    rc = bind(e);
    if (rc)
        return rc;
    // workspace: in = arena, ev_off/ev_len = key spans, out_b/out_c = value spans, lines_off/lines_len = time / ns,
    // pos = ent_begin, lab_sizes / cnt = record / body sizes, lab_off = record offsets, out_d = the wire bytes
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(m * 4 + 4));
    CU_TRY(e->ev_len.ensure(m * 4 + 4));
    CU_TRY(e->out_b.ensure(m * 4 + 4));
    CU_TRY(e->out_c.ensure(m * 4 + 4));
    CU_TRY(e->lines_off.ensure(n * 4));
    CU_TRY(e->lines_len.ensure(n * 4));
    CU_TRY(e->pos.ensure((n + 1) * 8));
    CU_TRY(e->lab_sizes.ensure(n * 4));
    CU_TRY(e->cnt.ensure(n * 4));
    CU_TRY(e->lab_off.ensure(n * 8));
    uint64_t* desc;
    rc = prep_desc(e, lck::scan_tiles(n), &desc);
    if (rc)
        return rc;
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    if (m) {
        CU_TRY(cudaMemcpyAsync(e->ev_off.p, ent_koff, m * 4, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->ev_len.p, ent_klen, m * 4, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->out_b.p, ent_voff, m * 4, cudaMemcpyHostToDevice, e->stream));
        CU_TRY(cudaMemcpyAsync(e->out_c.p, ent_vlen, m * 4, cudaMemcpyHostToDevice, e->stream));
    }
    CU_TRY(cudaMemcpyAsync(e->lines_off.p, ev_time, n * 4, cudaMemcpyHostToDevice, e->stream));
    if (ev_time_ns)
        CU_TRY(cudaMemcpyAsync(e->lines_len.p, ev_time_ns, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->pos.p, ent_begin, (n + 1) * 8, cudaMemcpyHostToDevice, e->stream));
    const uint32_t* d_ns = ev_time_ns ? e->lines_len.as<uint32_t>() : nullptr;
    lck::launch_sls_sizes(e->pos.as<uint64_t>(), e->ev_len.as<uint32_t>(), e->out_c.as<uint32_t>(), d_ns, n,
                          e->lab_sizes.as<uint32_t>(), e->cnt.as<uint32_t>(), e->stream);
    lck::launch_exclusive_sum(e->lab_sizes.as<uint32_t>(), n, e->lab_off.as<uint64_t>(), &ds->total, desc,
                              &ds->tickets[2], e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    *out_len = hs->total;
    if (hs->total > out_cap)
        return fail(LC_ERR_CAPACITY, "lc_sls_serialize_logs: output capacity too small");
    if (hs->total == 0)
        return LC_OK;
    if (!out)
        return fail(LC_ERR_INVALID_ARG, "lc_sls_serialize_logs: bad arguments");
    CU_TRY(e->out_d.ensure(hs->total));
    lck::launch_sls_emit(e->in.as<uint8_t>(), e->lines_off.as<uint32_t>(), d_ns, e->pos.as<uint64_t>(),
                         e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), e->out_b.as<uint32_t>(),
                         e->out_c.as<uint32_t>(), n, e->lab_off.as<uint64_t>(), e->cnt.as<uint32_t>(),
                         e->out_d.as<uint8_t>(), e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, e->out_d.p, hs->total, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

} // extern "C"

// ------------------------------------------------------------------------------------------------ processor -> SLS
namespace {

// The fused LZ4 calls (lc_regex_parse_sls_lz4, lc_delim_parse_sls_lz4): the group-level fields that follow the
// records, and where the records' size plus theirs goes
struct Lz4Tail {
    const uint8_t* tail;
    uint64_t len;
    uint64_t* raw_len;
};
int lz4_one_block(lc_engine_t* e, const char* what, const uint8_t* d_src, uint64_t raw, uint8_t* out, uint64_t out_cap,
                  uint64_t* out_len);

// Where serialize_sls_dev's records go besides d_out, and a counter that refuses the call
struct SlsTo {
    uint8_t* host = nullptr;    // d_out == nullptr: the records are staged in `lab` and copied back here
    const Lz4Tail* z = nullptr; // records ‖ z->tail become one LZ4 block, copied back to `host`
    int too_large = -1;         // counter k > 0: a record would reach 4 GiB, LC_ERR_TOO_LARGE
};

// Serialise from device tables (lc_sls_serialize_delim_dev / _regex_dev / _parsed_dev / _split_regex_dev and the
// split -> regex host calls): `sizes(rec_size, body_size, d_counters)` queues the size pass, an exclusive sum gives the
// record offsets, `emit(rec_off, body_size, d_out)` queues the emit pass.  counters (host, or nullptr) receive the
// ncounters device counters of the size pass.  `to` (host copy, LZ4 block, refusing counter) as SlsTo says; with z,
// out_cap and *out_len are the block's.
template <class Sizes, class Emit>
int serialize_sls_dev(lc_engine_t* e, const char* what, uint64_t n, uint32_t ncounters, Sizes sizes, Emit emit,
                      uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t* counters, const SlsTo& to = {}) {
    CU_TRY(e->lab_sizes.ensure(n * 4));
    CU_TRY(e->cnt.ensure(n * 4));
    CU_TRY(e->lab_off.ensure(n * 8));
    unsigned long long* d_ctr = nullptr;
    if (counters && ncounters) {
        CU_TRY(e->state.ensure(ncounters * sizeof(unsigned long long)));
        d_ctr = e->state.as<unsigned long long>();
        CU_TRY(cudaMemsetAsync(d_ctr, 0, ncounters * sizeof(unsigned long long), e->stream));
    }
    uint64_t* desc;
    int rc = prep_desc(e, lck::scan_tiles(n), &desc);
    if (rc)
        return rc;
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    sizes(e->lab_sizes.as<uint32_t>(), e->cnt.as<uint32_t>(), d_ctr);
    lck::launch_exclusive_sum(e->lab_sizes.as<uint32_t>(), n, e->lab_off.as<uint64_t>(), &ds->total, desc,
                              &ds->tickets[2], e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
    unsigned long long ctr[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (d_ctr)
        CU_TRY(cudaMemcpyAsync(ctr, d_ctr, ncounters * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    for (uint32_t k = 0; d_ctr && k < ncounters; ++k)
        counters[k] = ctr[k];
    if (to.too_large >= 0 && ctr[to.too_large])
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": a record would reach 4 GiB");
    const uint64_t total = hs->total;
    if (to.z) {
        const uint64_t raw = total + to.z->len;
        *to.z->raw_len = raw;
        if (raw > LC_LZ4_MAX_INPUT)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": records and tail are larger than LZ4_MAX_INPUT_SIZE");
        CU_TRY(e->lab.ensure(raw + 16));
        if (total) {
            emit(e->lab_off.as<uint64_t>(), e->cnt.as<uint32_t>(), e->lab.as<uint8_t>());
            e->launches++;
            CU_TRY(cudaGetLastError());
        }
        if (to.z->len)
            CU_TRY(cudaMemcpyAsync(e->lab.as<uint8_t>() + total, to.z->tail, to.z->len, cudaMemcpyHostToDevice,
                                   e->stream));
        return lz4_one_block(e, what, e->lab.as<uint8_t>(), raw, to.host, out_cap, out_len);
    }
    *out_len = total;
    if (total > out_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": output capacity too small");
    if (total == 0)
        return LC_OK;
    if (!d_out && !to.host)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (!d_out)
        CU_TRY(e->lab.ensure(total));
    emit(e->lab_off.as<uint64_t>(), e->cnt.as<uint32_t>(), d_out ? d_out : e->lab.as<uint8_t>());
    e->launches++;
    CU_TRY(cudaGetLastError());
    if (!d_out)
        CU_TRY(cudaMemcpyAsync(to.host, e->lab.p, total, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// a fused call without events: the block of the tail alone
int lz4_tail_only(lc_engine_t* e, const char* what, const Lz4Tail& z, uint8_t* out, uint64_t out_cap,
                  uint64_t* out_len) {
    *z.raw_len = z.len;
    if (z.len > LC_LZ4_MAX_INPUT)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": tail larger than LZ4_MAX_INPUT_SIZE");
    CU_TRY(e->lab.ensure(z.len + 16));
    if (z.len)
        CU_TRY(cudaMemcpyAsync(e->lab.p, z.tail, z.len, cudaMemcpyHostToDevice, e->stream));
    return lz4_one_block(e, what, e->lab.as<uint8_t>(), z.len, out, out_cap, out_len);
}

// Parse and serialise host buffers in one call (lc_delim_parse_sls, lc_regex_parse_sls).  The arena goes up once, in
// chunks of whole events on a copy stream (pipelined_events); per chunk the event times go up, `parse(i0, cnt, span)`
// queues the processor's kernels and `sizes(i0, cnt, d_ns, rec_size, body_size, d_counters)` the size pass.  No table
// comes back.  Then one exclusive sum, `emit(d_time, d_ns, rec_off, body_size, d_wire)` over all n events, and one
// copy of the wire bytes.  Workspace besides the arena, the event table and the processor's own tables: lines_off /
// lines_len = times / ns, flags / cnt = record / body sizes, pos = record offsets, state = the counters, lab = the
// wire bytes.  The regex and delimiter stages touch none of them while the chunks are parsed.  With z (the fused LZ4
// calls) the tail lands after the records in `lab`, records ‖ tail become one LZ4 block and only the block comes back:
// out_cap and *out_len are then the block's.
template <class Parse, class Sizes, class Emit>
int parse_sls_host(lc_engine_t* e, const char* what, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                   const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time, const uint32_t* ev_time_ns,
                   uint32_t ncounters, Parse parse, Sizes sizes, Emit emit, uint8_t* out, uint64_t out_cap,
                   uint64_t* out_len, uint64_t* counters, const Lz4Tail* z = nullptr) {
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->lines_off.ensure(n * 4));
    CU_TRY(e->lines_len.ensure(n * 4));
    CU_TRY(e->flags.ensure(n * 4));
    CU_TRY(e->cnt.ensure(n * 4));
    CU_TRY(e->pos.ensure(n * 8));
    CU_TRY(e->state.ensure(ncounters * sizeof(unsigned long long)));
    unsigned long long* d_ctr = e->state.as<unsigned long long>();
    CU_TRY(cudaMemsetAsync(d_ctr, 0, ncounters * sizeof(unsigned long long), e->stream));
    uint32_t* d_time = e->lines_off.as<uint32_t>();
    uint32_t* d_ns = ev_time_ns ? e->lines_len.as<uint32_t>() : nullptr;
    uint32_t* d_rec = e->flags.as<uint32_t>();
    uint32_t* d_body = e->cnt.as<uint32_t>();
    auto run = [&](uint64_t, uint64_t i0, uint64_t cnt, uint64_t span) {
        CU_TRY(cudaMemcpyAsync(d_time + i0, ev_time + i0, cnt * 4, cudaMemcpyHostToDevice, e->stream));
        if (d_ns)
            CU_TRY(cudaMemcpyAsync(d_ns + i0, ev_time_ns + i0, cnt * 4, cudaMemcpyHostToDevice, e->stream));
        int r = parse(i0, cnt, span);
        if (r)
            return r;
        sizes(i0, cnt, d_ns ? d_ns + i0 : nullptr, d_rec + i0, d_body + i0, d_ctr);
        e->launches++;
        CU_TRY(cudaGetLastError());
        return (int)LC_OK;
    };
    auto down = [&](uint64_t, uint64_t, uint64_t) { return (int)LC_OK; };
    int rc = pipelined_events(e, base, base_len, ev_off, ev_len, n, pipeline_chunks(base_len, n), what, run, down);
    if (rc)
        return rc;
    uint64_t* desc;
    rc = prep_desc(e, lck::scan_tiles(n), &desc); // (after the parse: the regex stage's fall-back kernels use desc)
    if (rc)
        return rc;
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    lck::launch_exclusive_sum(d_rec, n, e->pos.as<uint64_t>(), &ds->total, desc, &ds->tickets[2], e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
    unsigned long long ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    CU_TRY(cudaMemcpyAsync(ctr, d_ctr, ncounters * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    for (uint32_t k = 0; k < ncounters; ++k)
        counters[k] = ctr[k];
    if (z) {
        const uint64_t total = hs->total, raw = total + z->len;
        *z->raw_len = raw;
        if (raw > LC_LZ4_MAX_INPUT)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": records and tail are larger than LZ4_MAX_INPUT_SIZE");
        CU_TRY(e->lab.ensure(raw + 16));
        if (total) {
            emit(d_time, d_ns, e->pos.as<uint64_t>(), d_body, e->lab.as<uint8_t>());
            e->launches++;
            CU_TRY(cudaGetLastError());
        }
        if (z->len)
            CU_TRY(cudaMemcpyAsync(e->lab.as<uint8_t>() + total, z->tail, z->len, cudaMemcpyHostToDevice, e->stream));
        return lz4_one_block(e, what, e->lab.as<uint8_t>(), raw, out, out_cap, out_len);
    }
    *out_len = hs->total;
    if (hs->total > out_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": output capacity too small");
    if (hs->total == 0)
        return LC_OK;
    if (!out)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    CU_TRY(e->lab.ensure(hs->total));
    emit(d_time, d_ns, e->pos.as<uint64_t>(), d_body, e->lab.as<uint8_t>());
    e->launches++;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(out, e->lab.p, hs->total, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// the configuration of the delimiter-fed serialiser, its key strings staged on the device (`dst`, by default the engine
// `order` buffer)
int delim_sls_config(lc_engine_t* e, const char* what, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                     uint8_t quote, int extend, int discard, const char* const* keys, const uint32_t* key_lens,
                     uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, LcDelimSlsCfg* c,
                     DevBuf* dst = nullptr) {
    if (!sep || (nkeys && (!keys || !key_lens)) || (source_key_len && !source_key) ||
        (renamed_key_len && !renamed_key))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    for (uint32_t k = 0; k < nkeys; ++k)
        if (key_lens[k] && !keys[k])
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    uint64_t kbytes = (uint64_t)source_key_len + renamed_key_len + 11;
    for (uint32_t k = 0; k < nkeys; ++k)
        kbytes += key_lens[k];
    if (kbytes >= (1ull << 31))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": keys too long");
    std::vector<uint8_t> kb(kbytes + 1);
    std::vector<uint32_t> at(nkeys + 4);
    const char* why = lc_delim_sls_setup(sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                                         source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw,
                                         max_fields, c, kb.data(), at.data());
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    const size_t at_bytes = at.size() * 4;
    DevBuf& d = dst ? *dst : e->order;
    CU_TRY(d.ensure(at_bytes + kb.size() + 16));
    CU_TRY(cudaMemcpyAsync(d.p, at.data(), at_bytes, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(d.as<uint8_t>() + at_bytes, kb.data(), kb.size(), cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream)); // (pageable sources: their bytes must be on the device before they die)
    c->key_at = d.as<uint32_t>();
    c->keys = d.as<uint8_t>() + at_bytes;
    return LC_OK;
}

// the content plans (2 * (n_ok + n_fail) words) and key table of a regex-fed serialiser, staged on the device (engine
// `sls_plan` buffer; the regex stage may reuse `order` for its length ordering while a host-buffer call runs)
int stage_regex_sls(lc_engine_t* e, const char* what, const uint32_t* plan, const char* const* strings,
                    const uint32_t* lens, uint32_t nstrings, LcRegexSlsCfg* c) {
    uint64_t kbytes = 0;
    for (uint32_t k = 0; k < nstrings; ++k)
        kbytes += lens[k];
    if (kbytes >= (1ull << 31))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": keys too long");
    const size_t pb = (size_t)2 * (c->n_ok + c->n_fail) * 4, ab = ((size_t)nstrings + 1) * 4;
    std::vector<uint8_t> blob(pb + ab + kbytes + 1);
    if (pb)
        memcpy(blob.data(), plan, pb);
    lc_sls_key_table(strings, lens, nstrings, blob.data() + pb + ab, reinterpret_cast<uint32_t*>(blob.data() + pb));
    CU_TRY(e->sls_plan.ensure(blob.size() + 16));
    CU_TRY(cudaMemcpyAsync(e->sls_plan.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream)); // (pageable source: its bytes must be on the device before it dies)
    uint8_t* d = e->sls_plan.as<uint8_t>();
    c->plan = reinterpret_cast<const uint32_t*>(d);
    c->key_at = reinterpret_cast<const uint32_t*>(d + pb);
    c->keys = d + pb + ab;
    return LC_OK;
}

// the configuration of the regex-fed serialiser: lc_regex_sls_setup's plans over the key table keys..., SourceKey,
// RenamedSourceKey, "__raw_log__", "content", staged on the device
int regex_sls_config(lc_engine_t* e, const char* what, const char* const* keys, const uint32_t* key_lens,
                     uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                     uint32_t pitch, LcRegexSlsCfg* c) {
    std::vector<uint32_t> plan(3 * (size_t)nkeys + 12);
    const char* why = lc_regex_sls_setup(keys, key_lens, nkeys, source_key, source_key_len, renamed_key,
                                         renamed_key_len, keep_fail, keep_succeed, copy_raw, whole_line, pitch, c,
                                         plan.data());
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    std::vector<const char*> strings(keys, keys + nkeys);
    std::vector<uint32_t> lens(key_lens, key_lens + nkeys);
    strings.insert(strings.end(), {source_key, renamed_key, "__raw_log__", "content"});
    lens.insert(lens.end(), {source_key_len, renamed_key_len, 11u, 7u});
    return stage_regex_sls(e, what, plan.data(), strings.data(), lens.data(), nkeys + 4, c);
}

// The configuration of the delimiter -> regex chain (both stages' arguments, CHAIN_ARGS below): the delimiter's
// configuration and keys (engine `dr_keys` buffer), the regex plans over its key k (`sls_plan`) and the chain's own
// checks (lc_delim_regex_sls_link).  pitch = the regex tables' row pitch.
#define CHAIN_PARAMS                                                                                                   \
    const uint8_t *sep, uint32_t sep_len, uint8_t quote, int extend, int discard, const char *const *keys,             \
        const uint32_t *key_lens, uint32_t nkeys, const char *source_key, uint32_t source_key_len,                     \
        const char *renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,              \
        const char *const *rkeys, const uint32_t *rkey_lens, uint32_t rnkeys, const char *rsource_key,                 \
        uint32_t rsource_key_len, const char *rrenamed_key, uint32_t rrenamed_key_len, int rkeep_fail,                 \
        int rkeep_succeed, int rcopy_raw, int whole_line
#define CHAIN_ARGS                                                                                                     \
    sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key, source_key_len, renamed_key,              \
        renamed_key_len, keep_fail, keep_succeed, copy_raw, rkeys, rkey_lens, rnkeys, rsource_key, rsource_key_len,    \
        rrenamed_key, rrenamed_key_len, rkeep_fail, rkeep_succeed, rcopy_raw, whole_line
int chain_config(lc_engine_t* e, const char* what, uint32_t max_fields, CHAIN_PARAMS, uint32_t pitch,
                 LcDelimRegexSlsCfg* c) {
    memset(c, 0, sizeof *c);
    int rc = delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys,
                              source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed,
                              copy_raw, &c->d, &e->dr_keys);
    if (rc)
        return rc;
    rc = regex_sls_config(e, what, rkeys, rkey_lens, rnkeys, rsource_key, rsource_key_len, rrenamed_key,
                          rrenamed_key_len, rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, pitch, &c->x);
    if (rc)
        return rc;
    const char* why = lc_delim_regex_sls_link(c->d, keys, key_lens, source_key, source_key_len, renamed_key,
                                              renamed_key_len, rkeys, rkey_lens, rnkeys, rsource_key, rsource_key_len,
                                              rrenamed_key, rrenamed_key_len, rkeep_fail, rkeep_succeed, rcopy_raw,
                                              whole_line, c);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    return LC_OK;
}

// Queues the value tap of n rows: copy sizes into d_copy, their exclusive sum into d_slot (look-back descriptors
// `desc`, zeroed, scan_tiles(n) + 3 words: the total and the ticket follow them), then the value table and the side
// copies at d_base[side_at + slot).
void queue_tap(lc_engine_t* e, const LcDelimRegexSlsCfg& c, const lck::DelimSlsTables& t, uint64_t n,
               uint64_t side_at, uint8_t* d_base, uint32_t* d_copy, uint64_t* d_slot, uint64_t* desc,
               uint32_t* d_val_off, uint32_t* d_val_len) {
    const uint32_t tiles = lck::scan_tiles(n);
    lck::launch_delim_regex_tap_sizes(c, t, n, d_copy, e->stream);
    lck::launch_exclusive_sum(d_copy, n, d_slot, desc + tiles + 1, desc, reinterpret_cast<uint32_t*>(desc + tiles + 2),
                              e->stream);
    lck::launch_delim_regex_tap(c, t, n, d_slot, side_at, d_base, d_val_off, d_val_len, e->stream);
    e->launches += 3;
}

// The configuration of the split-fed serialiser over one source value d_src[0, src_len); the keys are staged on the
// device in the engine's `sls_plan` buffer, which neither splitter uses.  A record is its piece plus at most
// key_len + offset_key_len + 96 bytes of framing and digits, so record sizes stay below 2^32.
int span_sls_config(lc_engine_t* e, const char* what, const uint8_t* d_src, uint64_t src_len, const char* key,
                    uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                    uint32_t time, uint32_t time_ns, LcSpanSlsCfg* c) {
    if ((key_len && !key) || (src_len && !d_src))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (src_len + key_len + (uint64_t)offset_key_len + 96 > 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": source value and keys must stay below 4 GiB");
    const bool replace = offset_key && offset_key_len == key_len && !memcmp(offset_key, key, key_len);
    std::vector<uint8_t> kb(key_len + (offset_key ? offset_key_len : 0u) + 1);
    if (key_len)
        memcpy(kb.data(), key, key_len);
    if (offset_key && offset_key_len)
        memcpy(kb.data() + key_len, offset_key, offset_key_len);
    CU_TRY(e->sls_plan.ensure(kb.size() + 16));
    CU_TRY(cudaMemcpyAsync(e->sls_plan.p, kb.data(), kb.size(), cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream)); // (pageable source: its bytes must be on the device before it dies)
    memset(c, 0, sizeof *c);
    c->src = d_src;
    c->src_len = src_len;
    c->key = e->sls_plan.as<uint8_t>();
    c->klen = key_len;
    c->okey = c->key + key_len;
    c->oklen = offset_key ? offset_key_len : 0u;
    c->mode = !offset_key ? LC_SPAN_PIECE : replace ? LC_SPAN_OFFSET : LC_SPAN_PIECE_OFFSET;
    c->time = time < (1u << 28) ? (1u << 28) : time;
    c->has_ns = time_ns != LC_SLS_NO_NS;
    c->ns = c->has_ns ? time_ns : 0u;
    c->src_pos = src_pos;
    return LC_OK;
}

// size pass, exclusive sum and the output-tiled emit over the pieces d_off / d_len (serialize_sls_dev)
int serialize_spans(lc_engine_t* e, const char* what, LcSpanSlsCfg& c, const uint32_t* d_off, const uint32_t* d_len,
                    uint64_t n, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len) {
    c.off = d_off;
    c.len = d_len;
    return serialize_sls_dev(
        e, what, n, 0, [&](uint32_t* rec, uint32_t*, unsigned long long*) { lck::launch_span_sls_sizes(c, n, rec, e->stream); },
        // serialize_sls_dev has set *out_len to the total before it queues the emit
        [&](const uint64_t* rec_off, const uint32_t*, uint8_t* out) {
            lck::launch_span_sls_emit(c, rec_off, n, *out_len, out, e->stream);
        },
        d_out, out_cap, out_len, nullptr);
}

// Host-buffer split + serialise (lc_split_sls, lc_multiline_split_sls): the source goes up once into `in`,
// `split(&n)` cuts it into the piece tables out_a / out_b (and out_c flags), the records are written to `lab` and only
// they come back.  The serialiser's tables (lab_sizes, cnt, lab_off, desc, sls_plan) are none of the splitters'.
template <class Split>
int split_sls_host(lc_engine_t* e, const char* what, const uint8_t* buf, uint64_t len, Split split, const char* key,
                   uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                   uint32_t time, uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                   uint64_t* n_events) {
    if (!e || !out_len || (len && !buf))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (n_events)
        *n_events = 0;
    if (len == 0)
        return LC_OK;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(len + 16));
    CU_TRY(e->out_a.ensure((len + 1) * 4));
    CU_TRY(e->out_b.ensure((len + 1) * 4));
    CU_TRY(e->out_c.ensure(len + 1));
    CU_TRY(cudaMemcpyAsync(e->in.p, buf, len, cudaMemcpyHostToDevice, e->stream));
    uint64_t n = 0;
    rc = split(&n);
    if (rc)
        return rc;
    if (n_events)
        *n_events = n;
    LcSpanSlsCfg c;
    rc = span_sls_config(e, what, e->in.as<uint8_t>(), len, key, key_len, offset_key, offset_key_len, src_pos, time,
                         time_ns, &c);
    if (rc)
        return rc;
    // the wire bytes never exceed the pieces plus a record's framing each
    const uint64_t bound = len + n * ((uint64_t)key_len + offset_key_len + 128);
    const uint64_t cap = out_cap < bound ? out_cap : bound;
    CU_TRY(e->lab.ensure(cap));
    rc = serialize_spans(e, what, c, e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), n, e->lab.as<uint8_t>(), cap,
                         out_len);
    if (rc == LC_OK && *out_len) {
        if (!out)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
        CU_TRY(cudaMemcpyAsync(out, e->lab.p, *out_len, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    return rc;
}

} // namespace

extern "C" {

int lc_sls_serialize_parsed_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                                const uint32_t* d_ev_len, const uint8_t* d_status, const uint32_t* d_cap_off,
                                const uint32_t* d_cap_len, uint32_t row_pitch, uint64_t n, const char* const* keys,
                                const uint32_t* key_lens, uint32_t nkeys, const char* fail_key, uint32_t fail_key_len,
                                const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                                uint64_t out_cap, uint64_t* out_len) {
    static const char* what = "lc_sls_serialize_parsed_dev";
    if (!e || !out_len || (n && (!d_base || !d_ev_off || !d_ev_len || !d_status || !d_ev_time)) ||
        (nkeys && (!keys || !key_lens || !d_cap_off || !d_cap_len)) || nkeys > row_pitch || nkeys > LC_MAX_GROUPS)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (n == 0)
        return LC_OK;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB and < 2^30 events per call");
    for (uint32_t a = 0; a < nkeys; ++a)
        for (uint32_t b = a + 1; b < nkeys; ++b)
            if (key_lens[a] == key_lens[b] && !memcmp(keys[a], keys[b], key_lens[a]))
                return fail(LC_ERR_INVALID_ARG, std::string(what) + ": keys must be distinct (a repeated key "
                                                                    "overwrites its earlier content, LogEvent.cpp:83-95)");
    int rc = bind(e);
    if (rc)
        return rc;
    // the plans of this fixed configuration: keys[k] -> capture k on parsed rows; fail_key -> the line on failed rows
    // when there is one (they are erased otherwise)
    LcRegexSlsCfg c;
    memset(&c, 0, sizeof c);
    std::vector<uint32_t> plan;
    for (uint32_t k = 0; k < nkeys; ++k)
        plan.insert(plan.end(), {k, k});
    if (fail_key)
        plan.insert(plan.end(), {nkeys, LC_REGEX_SLS_LINE});
    c.n_ok = nkeys;
    c.n_fail = fail_key ? 1u : 0u;
    c.pitch = row_pitch;
    c.ok_fits = 1;
    c.keep_fail = fail_key != nullptr;
    std::vector<const char*> strings(keys, keys + nkeys);
    std::vector<uint32_t> lens(key_lens, key_lens + nkeys);
    strings.push_back(fail_key);
    lens.push_back(fail_key ? fail_key_len : 0u);
    rc = stage_regex_sls(e, what, plan.data(), strings.data(), lens.data(), nkeys + 1, &c);
    if (rc)
        return rc;
    const lck::RegexSlsTables t{d_base, d_ev_off, d_ev_len, d_status, d_cap_off, d_cap_len};
    return serialize_sls_dev(
        e, what, n, 0,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* ctr) {
            lck::launch_regex_sls_sizes(c, t, d_ev_time_ns, n, rec, body, ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* out) {
            lck::launch_regex_sls_emit(c, t, d_ev_time, d_ev_time_ns, n, rec_off, body, out, e->stream);
        },
        d_out, out_cap, out_len, nullptr);
}

int lc_sls_serialize_regex_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                               const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status, const uint32_t* d_cap_off,
                               const uint32_t* d_cap_len, uint32_t row_pitch, const char* const* keys,
                               const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                               uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                               int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                               const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                               uint64_t out_cap, uint64_t* out_len, uint64_t counters[3]) {
    static const char* what = "lc_sls_serialize_regex_dev";
    const bool caps = !whole_line && nkeys && nkeys <= row_pitch; // the parsed plan reads the capture tables
    if (!e || !out_len || (n && (!d_base || !d_ev_off || !d_ev_len || !d_ev_time)) ||
        (n && !whole_line && !d_status) || (n && caps && (!d_cap_off || !d_cap_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, 3 * sizeof(uint64_t));
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)row_pitch >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 captures per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcRegexSlsCfg c;
    rc = regex_sls_config(e, what, keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len,
                          keep_fail, keep_succeed, copy_raw, whole_line, row_pitch, &c);
    if (rc || n == 0)
        return rc;
    const lck::RegexSlsTables t{d_base, d_ev_off, d_ev_len, whole_line ? nullptr : d_status,
                                caps ? d_cap_off : nullptr, caps ? d_cap_len : nullptr};
    return serialize_sls_dev(
        e, what, n, 3,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* ctr) {
            lck::launch_regex_sls_sizes(c, t, d_ev_time_ns, n, rec, body, ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* out) {
            lck::launch_regex_sls_emit(c, t, d_ev_time, d_ev_time_ns, n, rec_off, body, out, e->stream);
        },
        d_out, out_cap, out_len, counters);
}

} // extern "C"

static int regex_parse_sls_impl(lc_engine_t* e, const char* what, const lc_regex_t* re, const uint8_t* base,
                                uint64_t base_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                                const uint32_t* ev_time, const uint32_t* ev_time_ns, const char* const* keys,
                                const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                int keep_fail, int keep_succeed, int copy_raw, int whole_line, uint8_t* out,
                                uint64_t out_cap, uint64_t* out_len, uint64_t counters[3], const Lz4Tail* z) {
    if (!e || (!re && !whole_line) || !out_len || !counters || (n && (!ev_off || !ev_len || !ev_time)) ||
        (base_len && !base) || (z && (!z->raw_len || (z->len && !z->tail))))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (z)
        *z->raw_len = 0;
    memset(counters, 0, 3 * sizeof(uint64_t));
    int rc = whole_line ? (int)LC_OK : check_regex_usable(re, what);
    if (rc)
        return rc;
    const uint32_t G = whole_line ? 0u : re->res.ngroups;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)G >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 captures per call");
    rc = bind(e);
    if (rc)
        return rc;
    LcRegexSlsCfg c;
    rc = regex_sls_config(e, what, keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len,
                          keep_fail, keep_succeed, copy_raw, whole_line, G, &c);
    if (rc || n == 0)
        return rc || !z ? rc : lz4_tail_only(e, what, *z, out, out_cap, out_len);
    // the regex tables (out_a = status, out_b / out_c = captures) stay on the device; whole-line mode runs no regex
    if (!whole_line) {
        CU_TRY(e->out_a.ensure(n));
        CU_TRY(e->out_b.ensure(n * G * 4 + 4));
        CU_TRY(e->out_c.ensure(n * G * 4 + 4));
    }
    auto tables = [&](uint64_t i0) {
        return lck::RegexSlsTables{e->in.as<uint8_t>(), e->ev_off.as<uint32_t>() + i0, e->ev_len.as<uint32_t>() + i0,
                                   whole_line ? nullptr : e->out_a.as<uint8_t>() + i0,
                                   whole_line ? nullptr : e->out_b.as<uint32_t>() + i0 * G,
                                   whole_line ? nullptr : e->out_c.as<uint32_t>() + i0 * G};
    };
    // per chunk: the launch sequence of lc_regex_parse_dev (incl. the follow-up kernel for events >= 64 KB)
    auto parse = [&](uint64_t i0, uint64_t cnt, uint64_t span) {
        if (whole_line)
            return (int)LC_OK;
        return regex_parse_dev_impl(e, re, e->in.as<uint8_t>(), base_len, span, e->ev_off.as<uint32_t>() + i0,
                                    e->ev_len.as<uint32_t>() + i0, 1, cnt, nkeys, e->out_a.as<uint8_t>() + i0,
                                    e->out_b.as<uint32_t>() + i0 * G, e->out_c.as<uint32_t>() + i0 * G, false);
    };
    auto sizes = [&](uint64_t i0, uint64_t cnt, const uint32_t* d_ns, uint32_t* rec, uint32_t* body,
                     unsigned long long* ctr) {
        lck::launch_regex_sls_sizes(c, tables(i0), d_ns, cnt, rec, body, ctr, e->stream);
    };
    auto emit = [&](const uint32_t* d_time, const uint32_t* d_ns, const uint64_t* rec_off, const uint32_t* body,
                    uint8_t* d_wire) {
        lck::launch_regex_sls_emit(c, tables(0), d_time, d_ns, n, rec_off, body, d_wire, e->stream);
    };
    return parse_sls_host(e, what, base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns, 3, parse, sizes, emit, out,
                          out_cap, out_len, counters, z);
}

extern "C" {

int lc_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                       const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                       const uint32_t* ev_time_ns, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                       const char* source_key, uint32_t source_key_len, const char* renamed_key,
                       uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[3]) {
    return regex_parse_sls_impl(e, "lc_regex_parse_sls", re, base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns,
                                keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len,
                                keep_fail, keep_succeed, copy_raw, whole_line, out, out_cap, out_len, counters,
                                nullptr);
}

int lc_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                           const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                           const uint32_t* ev_time_ns, const char* const* keys, const uint32_t* key_lens,
                           uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                           uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, int whole_line,
                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* raw_len, uint64_t counters[3]) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return regex_parse_sls_impl(e, "lc_regex_parse_sls_lz4", re, base, base_len, ev_off, ev_len, n, ev_time,
                                ev_time_ns, keys, key_lens, nkeys, source_key, source_key_len, renamed_key,
                                renamed_key_len, keep_fail, keep_succeed, copy_raw, whole_line, out, out_cap, out_len,
                                counters, &z);
}

int lc_sls_serialize_delim_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len, const uint32_t* d_ev_off,
                               const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status, const uint32_t* d_nfields,
                               const uint32_t* d_f_off, const uint32_t* d_f_len, const uint32_t* d_f_dq,
                               uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
                               int discard, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                               const char* source_key, uint32_t source_key_len, const char* renamed_key,
                               uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                               const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns, uint8_t* d_out,
                               uint64_t out_cap, uint64_t* out_len) {
    static const char* what = "lc_sls_serialize_delim_dev";
    if (!e || !out_len || (n && (!d_base || !d_ev_off || !d_ev_len || !d_status || !d_nfields || !d_f_off || !d_f_len ||
                                 !d_f_dq || !d_ev_time)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcDelimSlsCfg c;
    rc = delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                          source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw, &c);
    if (rc || n == 0)
        return rc;
    const lck::DelimSlsTables t{d_base, d_ev_off, d_ev_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq};
    return serialize_sls_dev(
        e, what, n, 0,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* ctr) {
            lck::launch_delim_sls_sizes(c, t, d_ev_time_ns, n, rec, body, ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* out) {
            lck::launch_delim_sls_emit(c, t, d_ev_time, d_ev_time_ns, n, rec_off, body, out, e->stream);
        },
        d_out, out_cap, out_len, nullptr);
}

} // extern "C"

static int delim_parse_sls_impl(lc_engine_t* e, const char* what, const uint8_t* base, uint64_t base_len,
                                const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                                const uint32_t* ev_time_ns, const uint8_t* sep, uint32_t sep_len, uint8_t quote,
                                int extend, int discard, int allow_short, uint32_t max_fields, const char* const* keys,
                                const uint32_t* key_lens, uint32_t nkeys, const char* source_key,
                                uint32_t source_key_len, const char* renamed_key, uint32_t renamed_key_len,
                                int keep_fail, int keep_succeed, int copy_raw, uint8_t* out, uint64_t out_cap,
                                uint64_t* out_len, uint64_t counters[4], const Lz4Tail* z) {
    if (!e || !out_len || !counters || (n && (!ev_off || !ev_len || !ev_time)) || (base_len && !base) ||
        (z && (!z->raw_len || (z->len && !z->tail))))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (z)
        *z->raw_len = 0;
    memset(counters, 0, 4 * sizeof(uint64_t));
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcDelimSlsCfg c;
    rc = delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys, source_key,
                          source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw, &c);
    if (rc || n == 0)
        return rc || !z ? rc : lz4_tail_only(e, what, *z, out, out_cap, out_len);
    // the delimiter tables (out_a = status, out_b = column counts, out_c..out_e = [n][max_fields]) stay on the device
    const uint64_t MF = max_fields, fbytes = n * MF * 4;
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * 4));
    CU_TRY(e->out_c.ensure(fbytes));
    CU_TRY(e->out_d.ensure(fbytes));
    CU_TRY(e->out_e.ensure(fbytes));
    auto tables = [&](uint64_t i0) {
        return lck::DelimSlsTables{e->in.as<uint8_t>(),          e->ev_off.as<uint32_t>() + i0,
                                   e->ev_len.as<uint32_t>() + i0, e->out_a.as<uint8_t>() + i0,
                                   e->out_b.as<uint32_t>() + i0,  e->out_c.as<uint32_t>() + i0 * MF,
                                   e->out_d.as<uint32_t>() + i0 * MF, e->out_e.as<uint32_t>() + i0 * MF};
    };
    auto parse = [&](uint64_t i0, uint64_t cnt, uint64_t) {
        const lck::DelimSlsTables t = tables(i0);
        return lc_delim_parse_dev(e, t.base, base_len, t.ev_off, t.ev_len, cnt, sep, sep_len, quote, nkeys, extend,
                                  allow_short, max_fields, e->out_a.as<uint8_t>() + i0, e->out_b.as<uint32_t>() + i0,
                                  e->out_c.as<uint32_t>() + i0 * MF, e->out_d.as<uint32_t>() + i0 * MF,
                                  e->out_e.as<uint32_t>() + i0 * MF);
    };
    auto sizes = [&](uint64_t i0, uint64_t cnt, const uint32_t* d_ns, uint32_t* rec, uint32_t* body,
                     unsigned long long* ctr) {
        lck::launch_delim_sls_sizes(c, tables(i0), d_ns, cnt, rec, body, ctr, e->stream);
    };
    auto emit = [&](const uint32_t* d_time, const uint32_t* d_ns, const uint64_t* rec_off, const uint32_t* body,
                    uint8_t* d_wire) {
        lck::launch_delim_sls_emit(c, tables(0), d_time, d_ns, n, rec_off, body, d_wire, e->stream);
    };
    return parse_sls_host(e, what, base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns, 4, parse, sizes, emit, out,
                          out_cap, out_len, counters, z);
}

extern "C" {

int lc_delim_parse_sls(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                       const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time, const uint32_t* ev_time_ns,
                       const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard, int allow_short,
                       uint32_t max_fields, const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                       const char* source_key, uint32_t source_key_len, const char* renamed_key,
                       uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw, uint8_t* out,
                       uint64_t out_cap, uint64_t* out_len, uint64_t counters[4]) {
    return delim_parse_sls_impl(e, "lc_delim_parse_sls", base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns, sep,
                                sep_len, quote, extend, discard, allow_short, max_fields, keys, key_lens, nkeys,
                                source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed,
                                copy_raw, out, out_cap, out_len, counters, nullptr);
}

int lc_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                           const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time, const uint32_t* ev_time_ns,
                           const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend, int discard,
                           int allow_short, uint32_t max_fields, const char* const* keys, const uint32_t* key_lens,
                           uint32_t nkeys, const char* source_key, uint32_t source_key_len, const char* renamed_key,
                           uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                           const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* raw_len, uint64_t counters[4]) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return delim_parse_sls_impl(e, "lc_delim_parse_sls_lz4", base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns,
                                sep, sep_len, quote, extend, discard, allow_short, max_fields, keys, key_lens, nkeys,
                                source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed,
                                copy_raw, out, out_cap, out_len, counters, &z);
}

int lc_delim_regex_tap_dev(lc_engine_t* e, uint8_t* d_base, uint64_t base_len, uint64_t base_cap,
                           const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status,
                           const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                           const uint32_t* d_f_dq, uint32_t max_fields, CHAIN_PARAMS, uint32_t* d_val_off,
                           uint32_t* d_val_len, uint64_t* side_len) {
    static const char* what = "lc_delim_regex_tap_dev";
    if (!e || !side_len || (n && (!d_base || !d_ev_off || !d_ev_len || !d_status || !d_nfields || !d_f_off ||
                                  !d_f_len || !d_f_dq || !d_val_off || !d_val_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *side_len = 0;
    const uint64_t side_at = (base_len + 15) & ~15ull;
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcDelimRegexSlsCfg c;
    rc = chain_config(e, what, max_fields, CHAIN_ARGS, 0, &c);
    if (rc || n == 0)
        return rc;
    const lck::DelimSlsTables t{d_base, d_ev_off, d_ev_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq};
    const uint32_t tiles = lck::scan_tiles(n);
    CU_TRY(e->dr_copy.ensure(n * 4));
    CU_TRY(e->dr_slot.ensure(n * 8));
    CU_TRY(e->dr_desc.ensure(((uint64_t)tiles + 3) * 8));
    uint64_t* desc = e->dr_desc.as<uint64_t>();
    CU_TRY(cudaMemsetAsync(desc, 0, ((uint64_t)tiles + 3) * 8, e->stream));
    // sizes and slots first: nothing is written before the side region is known to fit
    lck::launch_delim_regex_tap_sizes(c, t, n, e->dr_copy.as<uint32_t>(), e->stream);
    lck::launch_exclusive_sum(e->dr_copy.as<uint32_t>(), n, e->dr_slot.as<uint64_t>(), desc + tiles + 1, desc,
                              reinterpret_cast<uint32_t*>(desc + tiles + 2), e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    uint64_t need = 0;
    CU_TRY(cudaMemcpyAsync(&need, desc + tiles + 1, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    *side_len = need;
    if (side_at + need + 16 >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": line buffer and side copies must stay below 4 GiB");
    if (need && side_at + need > base_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": no room for the side copies behind base_len");
    lck::launch_delim_regex_tap(c, t, n, e->dr_slot.as<uint64_t>(), side_at, d_base, d_val_off, d_val_len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int lc_sls_serialize_delim_regex_dev(lc_engine_t* e, const uint8_t* d_base, uint64_t base_len,
                                     const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
                                     const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off,
                                     const uint32_t* d_f_len, const uint32_t* d_f_dq, uint32_t max_fields,
                                     CHAIN_PARAMS, const uint32_t* d_val_off, const uint32_t* d_val_len,
                                     const uint8_t* d_re_status, const uint32_t* d_cap_off, const uint32_t* d_cap_len,
                                     uint32_t row_pitch, const uint32_t* d_ev_time, const uint32_t* d_ev_time_ns,
                                     uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]) {
    static const char* what = "lc_sls_serialize_delim_regex_dev";
    const bool caps = !whole_line && rnkeys && rnkeys <= row_pitch; // the parsed plan reads the capture tables
    if (!e || !out_len || (n && (!d_base || !d_ev_off || !d_ev_len || !d_status || !d_nfields || !d_f_off || !d_f_len ||
                                 !d_f_dq || !d_val_off || !d_val_len || !d_ev_time)) ||
        (n && !whole_line && !d_re_status) || (n && caps && (!d_cap_off || !d_cap_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, 8 * sizeof(uint64_t));
    if (base_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32) ||
        n * (uint64_t)row_pitch >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 events and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcDelimRegexSlsCfg c;
    rc = chain_config(e, what, max_fields, CHAIN_ARGS, row_pitch, &c);
    if (rc || n == 0)
        return rc;
    const lck::DelimRegexSlsTables t{{d_base, d_ev_off, d_ev_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq},
                                     d_val_off,
                                     d_val_len,
                                     whole_line ? nullptr : d_re_status,
                                     caps ? d_cap_off : nullptr,
                                     caps ? d_cap_len : nullptr};
    return serialize_sls_dev(
        e, what, n, 8,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* ctr) {
            lck::launch_delim_regex_sls_sizes(c, t, d_ev_time_ns, n, rec, body, ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* out) {
            lck::launch_delim_regex_sls_emit(c, t, d_ev_time, d_ev_time_ns, n, rec_off, body, out, e->stream);
        },
        d_out, out_cap, out_len, counters);
}

} // extern "C"

// lc_delim_regex_parse_sls[_lz4]: per upload chunk the delimiter stage, the value tap, the regex stage over the values
// and the size pass; the tables never leave the device.  The side copies of chunk c go behind the arena at a bound the
// host knows without a round trip: a copy is never longer than its line, so chunk c's copies fit in the sum of its
// line lengths, and chunk c starts where the bounds of the chunks before it end.
static int delim_regex_parse_sls_impl(lc_engine_t* e, const char* what, const lc_regex_t* re, const uint8_t* base,
                                      uint64_t base_len, const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n,
                                      const uint32_t* ev_time, const uint32_t* ev_time_ns, int allow_short,
                                      uint32_t max_fields, CHAIN_PARAMS, uint8_t* out, uint64_t out_cap,
                                      uint64_t* out_len, uint64_t counters[8], const Lz4Tail* z) {
    if (!e || (!re && !whole_line) || !out_len || !counters || (n && (!ev_off || !ev_len || !ev_time)) ||
        (base_len && !base) || (z && (!z->raw_len || (z->len && !z->tail))))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (z)
        *z->raw_len = 0;
    memset(counters, 0, 8 * sizeof(uint64_t));
    int rc = whole_line ? (int)LC_OK : check_regex_usable(re, what);
    if (rc)
        return rc;
    const uint32_t G = whole_line ? 0u : re->res.ngroups;
    uint64_t side_cap = 0;
    for (uint64_t i = 0; i < n; ++i)
        side_cap += ev_len[i];
    const uint64_t side_at = (base_len + 15) & ~15ull, arena = side_at + side_cap;
    if (arena + 16 >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32) ||
        n * (uint64_t)G >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "lines plus their total length must be < 4 GiB, < 2^30 events, < 2^32 columns "
                                      "and < 2^32 captures per call");
    rc = bind(e);
    if (rc)
        return rc;
    LcDelimRegexSlsCfg c;
    rc = chain_config(e, what, max_fields, CHAIN_ARGS, G, &c);
    if (rc || n == 0)
        return rc || !z ? rc : lz4_tail_only(e, what, *z, out, out_cap, out_len);
    // delimiter tables out_a .. out_e, value table, regex tables, tap scratch: all stay on the device
    const uint64_t MF = max_fields, fbytes = n * MF * 4, nchunks = pipeline_chunks(base_len, n);
    const uint64_t dwords = lck::scan_tiles(n) + 4 * nchunks + 8;
    CU_TRY(e->in.ensure(arena + 16));
    CU_TRY(e->out_a.ensure(n));
    CU_TRY(e->out_b.ensure(n * 4));
    CU_TRY(e->out_c.ensure(fbytes));
    CU_TRY(e->out_d.ensure(fbytes));
    CU_TRY(e->out_e.ensure(fbytes));
    CU_TRY(e->dr_val_off.ensure(n * 4));
    CU_TRY(e->dr_val_len.ensure(n * 4));
    CU_TRY(e->dr_status.ensure(n));
    CU_TRY(e->dr_cap_off.ensure(n * G * 4 + 4));
    CU_TRY(e->dr_cap_len.ensure(n * G * 4 + 4));
    CU_TRY(e->dr_copy.ensure(n * 4));
    CU_TRY(e->dr_slot.ensure(n * 8));
    CU_TRY(e->dr_desc.ensure(dwords * 8));
    CU_TRY(cudaMemsetAsync(e->dr_desc.p, 0, dwords * 8, e->stream));
    const bool caps = !whole_line && rnkeys && rnkeys <= G;
    auto dtables = [&](uint64_t i0) {
        return lck::DelimSlsTables{e->in.as<uint8_t>(),          e->ev_off.as<uint32_t>() + i0,
                                   e->ev_len.as<uint32_t>() + i0, e->out_a.as<uint8_t>() + i0,
                                   e->out_b.as<uint32_t>() + i0,  e->out_c.as<uint32_t>() + i0 * MF,
                                   e->out_d.as<uint32_t>() + i0 * MF, e->out_e.as<uint32_t>() + i0 * MF};
    };
    auto tables = [&](uint64_t i0) {
        return lck::DelimRegexSlsTables{dtables(i0),
                                        e->dr_val_off.as<uint32_t>() + i0,
                                        e->dr_val_len.as<uint32_t>() + i0,
                                        whole_line ? nullptr : e->dr_status.as<uint8_t>() + i0,
                                        caps ? e->dr_cap_off.as<uint32_t>() + i0 * G : nullptr,
                                        caps ? e->dr_cap_len.as<uint32_t>() + i0 * G : nullptr};
    };
    uint64_t side_used = 0, dpos = 0; // the side bound and the scan descriptors of the chunks queued so far
    auto parse = [&](uint64_t i0, uint64_t cnt, uint64_t span) {
        const lck::DelimSlsTables t = dtables(i0);
        int r = lc_delim_parse_dev(e, t.base, base_len, t.ev_off, t.ev_len, cnt, sep, sep_len, quote, nkeys, extend,
                                   allow_short, max_fields, e->out_a.as<uint8_t>() + i0, e->out_b.as<uint32_t>() + i0,
                                   e->out_c.as<uint32_t>() + i0 * MF, e->out_d.as<uint32_t>() + i0 * MF,
                                   e->out_e.as<uint32_t>() + i0 * MF);
        if (r)
            return r;
        uint64_t bound = 0;
        for (uint64_t i = i0; i < i0 + cnt; ++i)
            bound += ev_len[i];
        queue_tap(e, c, t, cnt, side_at + side_used, e->in.as<uint8_t>(), e->dr_copy.as<uint32_t>() + i0,
                  e->dr_slot.as<uint64_t>() + i0, e->dr_desc.as<uint64_t>() + dpos, e->dr_val_off.as<uint32_t>() + i0,
                  e->dr_val_len.as<uint32_t>() + i0);
        CU_TRY(cudaGetLastError());
        side_used += bound;
        dpos += lck::scan_tiles(cnt) + 3;
        if (whole_line)
            return (int)LC_OK;
        return regex_parse_dev_impl(e, re, e->in.as<uint8_t>(), arena, span + bound, e->dr_val_off.as<uint32_t>() + i0,
                                    e->dr_val_len.as<uint32_t>() + i0, 1, cnt, rnkeys, e->dr_status.as<uint8_t>() + i0,
                                    e->dr_cap_off.as<uint32_t>() + i0 * G, e->dr_cap_len.as<uint32_t>() + i0 * G,
                                    false);
    };
    auto sizes = [&](uint64_t i0, uint64_t cnt, const uint32_t* d_ns, uint32_t* rec, uint32_t* body,
                     unsigned long long* ctr) {
        lck::launch_delim_regex_sls_sizes(c, tables(i0), d_ns, cnt, rec, body, ctr, e->stream);
    };
    auto emit = [&](const uint32_t* d_time, const uint32_t* d_ns, const uint64_t* rec_off, const uint32_t* body,
                    uint8_t* d_wire) {
        lck::launch_delim_regex_sls_emit(c, tables(0), d_time, d_ns, n, rec_off, body, d_wire, e->stream);
    };
    return parse_sls_host(e, what, base, base_len, ev_off, ev_len, n, ev_time, ev_time_ns, 8, parse, sizes, emit, out,
                          out_cap, out_len, counters, z);
}

extern "C" {

int lc_delim_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                             const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                             const uint32_t* ev_time_ns, int allow_short, uint32_t max_fields, CHAIN_PARAMS,
                             uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]) {
    return delim_regex_parse_sls_impl(e, "lc_delim_regex_parse_sls", re, base, base_len, ev_off, ev_len, n, ev_time,
                                      ev_time_ns, allow_short, max_fields, CHAIN_ARGS, out, out_cap, out_len, counters,
                                      nullptr);
}

int lc_delim_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* base, uint64_t base_len,
                                 const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* ev_time,
                                 const uint32_t* ev_time_ns, int allow_short, uint32_t max_fields, CHAIN_PARAMS,
                                 const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                 uint64_t* out_len, uint64_t* raw_len, uint64_t counters[8]) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return delim_regex_parse_sls_impl(e, "lc_delim_regex_parse_sls_lz4", re, base, base_len, ev_off, ev_len, n,
                                      ev_time, ev_time_ns, allow_short, max_fields, CHAIN_ARGS, out, out_cap, out_len,
                                      counters, &z);
}

int lc_sls_serialize_spans_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                               const uint32_t* d_len, uint64_t n, const char* key, uint32_t key_len,
                               const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                               uint32_t time_ns, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len) {
    static const char* what = "lc_sls_serialize_spans_dev";
    if (!e || !out_len || (n && (!d_off || !d_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (n == 0)
        return LC_OK;
    if (n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, "< 2^30 pieces per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSpanSlsCfg c;
    rc = span_sls_config(e, what, d_src, src_len, key, key_len, offset_key, offset_key_len, src_pos, time, time_ns, &c);
    if (rc)
        return rc;
    return serialize_spans(e, what, c, d_off, d_len, n, d_out, out_cap, out_len);
}

int lc_split_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char, const char* key,
                 uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time,
                 uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_sls_host(e, "lc_split_sls", buf, len, split, key, key_len, offset_key, offset_key_len, src_pos, time,
                          time_ns, out, out_cap, out_len, n_events);
}

int lc_multiline_split_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, const char* key,
                           uint32_t key_len, const char* offset_key, uint32_t offset_key_len, uint64_t src_pos,
                           uint32_t time, uint32_t time_ns, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                           uint64_t* n_events, uint64_t counters[3]) {
    for (const lc_regex_t* r : {start, cont, end}) {
        int rc;
        if (r && (rc = check_regex_usable(r, "lc_multiline_split_sls")))
            return rc;
    }
    auto split = [&](uint64_t* n) {
        return lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,
                                      e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), len, n,
                                      counters);
    };
    return split_sls_host(e, "lc_multiline_split_sls", buf, len, split, key, key_len, offset_key, offset_key_len,
                          src_pos, time, time_ns, out, out_cap, out_len, n_events);
}

} // extern "C"

// ------------------------------------------------------------------------------------------------ split -> regex -> SLS
static_assert(LC_FILTER_MAX_LEAVES == LC_FILTER_SLS_LEAVES && LC_FILTER_MAX_PROG == LC_FILTER_SLS_PROG &&
                  LC_FILTER_NOT == LC_FILTER_SLS_NOT && LC_FILTER_AND == LC_FILTER_SLS_AND &&
                  LC_FILTER_OR == LC_FILTER_SLS_OR,
              "lc_b200.h and lc_exec.cuh disagree on the filter program");
// The regex stage's configuration and the offset content of the split events (CHAIN_PARAMS's regex half, plus
// offset_key -- NULL = no log.file.offset metadata -- and the source event's position, time and ns)
#define SPLIT_REGEX_PARAMS                                                                                             \
    const char *const *keys, const uint32_t *key_lens, uint32_t nkeys, const char *source_key,                         \
        uint32_t source_key_len, const char *renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,   \
        int copy_raw, int whole_line, const char *offset_key, uint32_t offset_key_len, uint64_t src_pos,              \
        uint32_t time, uint32_t time_ns
#define SPLIT_REGEX_ARGS                                                                                               \
    keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed,          \
        copy_raw, whole_line, offset_key, offset_key_len, src_pos, time, time_ns

namespace {

// The timestamp stage of the split -> regex -> timestamp calls: its SourceKey, the compiled SourceFormat, the call's
// time(NULL), the history discard (-1 = none) and mEnableTimestampNanosecond
struct TsArgs {
    const char* tkey;
    uint32_t tkey_len;
    const lc_timestamp_t* ts;
    int64_t now;
    int32_t discard_interval;
    int enable_ns;
};

int ts_run(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, const LcTsSpans& sp, uint64_t n,
           const uint32_t* d_grp, uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec,
           uint32_t* d_nsec, uint8_t* d_status, uint64_t* d_counters);

// lc_split_regex_sls_setup's plans over the key table keys..., SourceKey, RenamedSourceKey, "__raw_log__", "content",
// offset_key, staged on the device (`sls_plan`, which neither splitter nor the regex stage uses).  Every single
// content then stays below 4 GiB; a record that would not is caught by the size pass.  With fd, the filter behind the
// chain is checked and resolved against those plans into *f (lc_filter_sls_setup); with tkey (the timestamp calls),
// the timestamp stage's SourceKey into *tc (lc_split_regex_ts_setup).
int split_regex_sls_config(lc_engine_t* e, const char* what, uint64_t src_len, SPLIT_REGEX_PARAMS, uint32_t pitch,
                           LcSplitRegexSlsCfg* c, const lc_filter_desc_t* fd = nullptr, LcFilterSlsCfg* f = nullptr,
                           const TsArgs* ta = nullptr, LcSplitRegexTsCfg* tc = nullptr) {
    if ((nkeys && (!keys || !key_lens)) || (source_key_len && !source_key) || (renamed_key_len && !renamed_key))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    uint64_t kbytes = (uint64_t)source_key_len + renamed_key_len + (offset_key ? offset_key_len : 0u) + 18;
    for (uint32_t k = 0; k < nkeys; ++k) {
        if (key_lens[k] && !keys[k])
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
        kbytes += key_lens[k];
    }
    if (src_len + kbytes + 96 > 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": source value and keys must stay below 4 GiB");
    std::vector<uint32_t> plan(3 * (size_t)nkeys + 24);
    const char* why = lc_split_regex_sls_setup(keys, key_lens, nkeys, source_key, source_key_len, renamed_key,
                                               renamed_key_len, offset_key, offset_key_len, keep_fail, keep_succeed,
                                               copy_raw, whole_line, pitch, src_pos, time, time_ns, c, plan.data());
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    std::vector<const char*> strings(nkeys + LC_SPLIT_REGEX_SLS_NSTR);
    std::vector<uint32_t> lens(nkeys + LC_SPLIT_REGEX_SLS_NSTR);
    lc_split_regex_sls_strings(keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len,
                               offset_key, offset_key_len, strings.data(), lens.data());
    if (fd) {
        why = lc_filter_sls_setup(plan.data(), c->x.n_ok, c->x.n_fail, strings.data(), lens.data(), fd->nleaves,
                                  fd->keys, fd->key_lens, fd->nprog, fd->prog, f);
        if (why)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
        for (uint32_t l = 0; fd->nprog && l < fd->nleaves; ++l) {
            if (!fd->regs || !fd->regs[l])
                return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
            const int rc = check_regex_usable(fd->regs[l], what);
            if (rc)
                return rc;
        }
    }
    if (ta) {
        why = lc_split_regex_ts_setup(*c, plan.data(), strings.data(), lens.data(), ta->tkey, ta->tkey_len,
                                      ta->enable_ns, tc);
        if (why)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    }
    return stage_regex_sls(e, what, plan.data(), strings.data(), lens.data(), nkeys + LC_SPLIT_REGEX_SLS_NSTR, &c->x);
}

// The split -> regex -> timestamp chain's tap and timestamp passes over the n pieces of t: the value table into
// st_val, then lc_timestamp_parse_dev's two passes with the whole source value as one group into *ts (st_status,
// st_sec, st_nsec).  The stage's counters are the size pass's, so the passes' own go to ts_cnt unread.
int split_regex_ts_run(lc_engine_t* e, const LcSplitRegexSlsCfg& c, const LcSplitRegexTsCfg& tc, const TsArgs& ta,
                       const lck::RegexSlsTables& t, uint64_t n, lck::TsRowTables* ts) {
    CU_TRY(e->st_val.ensure(n * 8 + 8));
    CU_TRY(e->st_sec.ensure(n * 8));
    CU_TRY(e->st_nsec.ensure(n * 4));
    CU_TRY(e->st_status.ensure(n));
    CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
    uint32_t* off = e->st_val.as<uint32_t>();
    uint32_t *len = off + n, *grp = off + 2 * n;
    const uint32_t g[2] = {0u, (uint32_t)n};
    CU_TRY(cudaMemcpyAsync(grp, g, sizeof g, cudaMemcpyHostToDevice, e->stream));
    lck::launch_split_regex_ts_tap(c, tc, t, n, off, len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    const int rc = ts_run(e, ta.ts, t.base, LcTsSpans{off, len, nullptr, 1}, n, grp, 1, ta.now, ta.discard_interval,
                          e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>(), e->st_status.as<uint8_t>(),
                          e->ts_cnt.as<uint64_t>());
    *ts = lck::TsRowTables{e->st_status.as<uint8_t>(), e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>()};
    return rc;
}

// The filter over the n pieces of t: leaf by leaf, the tap and the boolean match over the source value (and over the
// digit scratch when the leaf reads the offset digits), then the keep bytes and the removed count.  *keep = the keep
// bytes (nullptr in BYPASS mode); *d_removed = the device counter of removed pieces (read after the size pass).
int filter_sls_run(lc_engine_t* e, const char* what, const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f,
                   const lc_filter_desc_t* fd, const lck::RegexSlsTables& t, uint64_t n, uint64_t src_len,
                   const uint8_t** keep, const uint64_t** d_removed) {
    *keep = nullptr;
    *d_removed = nullptr;
    if (f.nprog == 0 || n == 0)
        return LC_OK;
    const uint64_t nl = f.nleaves, dig_bytes = f.any_digits ? n * LC_FILTER_SLS_DIGIT_PITCH : 0;
    if (dig_bytes + 16 >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the offset digits of the pieces must stay below 4 GiB");
    CU_TRY(e->fl_tab.ensure(n * 16));
    CU_TRY(e->fl_match.ensure(nl * n * (f.any_digits ? 2 : 1) + 1));
    CU_TRY(e->fl_keep.ensure(n + 16));
    if (f.any_digits)
        CU_TRY(e->fl_dig.ensure(dig_bytes + 16));
    uint32_t* off = e->fl_tab.as<uint32_t>();
    uint32_t *len = off + n, *doff = off + 2 * n, *dlen = off + 3 * n;
    uint8_t* m = e->fl_match.as<uint8_t>();
    uint64_t* removed = e->fl_keep.as<uint64_t>();
    CU_TRY(cudaMemsetAsync(removed, 0, 8, e->stream));
    for (uint32_t l = 0; l < f.nleaves; ++l) {
        bool src = false, dig = false;
        for (int v = 0; v < 2; ++v) {
            dig = dig || f.src[l][v] == LC_REGEX_SLS_DIGITS;
            src = src || (f.src[l][v] != LC_REGEX_SLS_DIGITS && f.src[l][v] != LC_FILTER_SLS_ABSENT);
        }
        if (!src && !dig)
            continue; // absent everywhere: the leaf never holds
        lck::launch_filter_tap(c, f, l, t, n, off, len, dig ? doff : nullptr, dlen, e->fl_dig.as<uint8_t>(),
                               e->stream);
        e->launches++;
        CU_TRY(cudaGetLastError());
        int rc = src ? lc_regex_match_dev(e, fd->regs[l], t.base, src_len, off, len, n, m + l * n) : (int)LC_OK;
        if (!rc && dig)
            rc = lc_regex_match_dev(e, fd->regs[l], e->fl_dig.as<uint8_t>(), dig_bytes, doff, dlen, n,
                                    m + (nl + l) * n);
        if (rc)
            return rc;
    }
    uint8_t* k = e->fl_keep.as<uint8_t>() + 16;
    lck::launch_filter_eval(c, f, t.status, n, m, k, reinterpret_cast<unsigned long long*>(removed), e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    *keep = k;
    *d_removed = removed;
    return LC_OK;
}

// The size pass and the emit of the chain over n pieces (serialize_sls_dev): into d_out (the device-fed call), or
// back to the host buffer out, or -- with z -- records ‖ tail as one LZ4 block.  counters[3] = successful, failed,
// discarded; set whenever the size pass ran.  With tc (the timestamp calls), each record's time comes from the
// timestamp tables ts and counters has LC_SRTS_COUNTERS entries.
int split_regex_sls_run(lc_engine_t* e, const char* what, const LcSplitRegexSlsCfg& c, const lck::RegexSlsTables& t,
                        uint64_t n, uint8_t* d_out, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                        uint64_t* counters, const Lz4Tail* z, const uint8_t* keep = nullptr,
                        const LcSplitRegexTsCfg* tc = nullptr, const lck::TsRowTables* ts = nullptr) {
    const uint32_t nstage = tc ? LC_SRTS_COUNTERS : 3u;
    uint64_t ctr[LC_SRTS_COUNTERS + 1] = {0}; // + pieces whose record would reach 4 GiB
    SlsTo to;
    to.host = out;
    to.z = z;
    to.too_large = (int)nstage;
    const int rc = serialize_sls_dev(
        e, what, n, nstage + 1,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* d_ctr) {
            if (tc)
                lck::launch_split_regex_ts_sls_sizes(c, *tc, t, *ts, n, rec, body, d_ctr, e->stream);
            else
                lck::launch_split_regex_sls_sizes(c, t, n, keep, rec, body, d_ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* dst) {
            if (tc)
                lck::launch_split_regex_ts_sls_emit(c, *tc, t, *ts, n, rec_off, body, dst, e->stream);
            else
                lck::launch_split_regex_sls_emit(c, t, n, rec_off, body, dst, e->stream);
        },
        d_out, out_cap, out_len, ctr, to);
    memcpy(counters, ctr, nstage * sizeof(uint64_t));
    return rc;
}

// Host-buffer split + parse + serialise (the split -> regex and split -> delimiter calls): the source goes up once into
// `in`, `split(&n)` cuts it into the piece tables out_a / out_b (and out_c flags), then the parse stage and the
// serialiser run over them and only the wire bytes (or, with z, records ‖ tail as one LZ4 block) come back.  The
// stage's part: stage_args = its own arguments are usable; begin() = its checks before the engine is bound (it zeroes
// its counters); config() = its configuration, staged on the device before the split; run(n) = parse, size pass and
// emit over the n > 0 pieces.
template <class Split, class Begin, class Config, class Run>
int split_chain_sls_host(lc_engine_t* e, const char* what, const uint8_t* buf, uint64_t len, Split split,
                         bool stage_args, Begin begin, Config config, Run run, uint8_t* out, uint64_t out_cap,
                         uint64_t* out_len, uint64_t* n_events, const Lz4Tail* z) {
    if (!e || !stage_args || !out_len || (len && !buf) || (z && (!z->raw_len || (z->len && !z->tail))))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (n_events)
        *n_events = 0;
    if (z)
        *z->raw_len = 0;
    int rc = begin();
    if (rc)
        return rc;
    if (len >= 0xFFFFFFF0ull)
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB per call");
    rc = bind(e);
    if (rc)
        return rc;
    rc = config();
    if (rc)
        return rc;
    uint64_t n = 0;
    if (len) {
        CU_TRY(e->in.ensure(len + 16));
        CU_TRY(e->out_a.ensure((len + 1) * 4));
        CU_TRY(e->out_b.ensure((len + 1) * 4));
        CU_TRY(e->out_c.ensure(len + 1));
        CU_TRY(cudaMemcpyAsync(e->in.p, buf, len, cudaMemcpyHostToDevice, e->stream));
        rc = split(&n);
        if (rc)
            return rc;
    }
    if (n_events)
        *n_events = n;
    if (n == 0)
        return z ? lz4_tail_only(e, what, *z, out, out_cap, out_len) : (int)LC_OK;
    return run(n);
}

// The regex stage of the split -> regex calls (split_regex_sls_host) over the n pieces: the regex tables go to
// dr_status / dr_cap_off / dr_cap_len; with fd (the _filter_ calls), the filter runs between the regex stage and the
// size pass and counters has a 4th entry; with ta (the _timestamp_ calls), the tap and the timestamp passes run there
// and counters has LC_SRTS_COUNTERS entries.
int split_regex_sls_stage(lc_engine_t* e, const char* what, const lc_regex_t* re, uint64_t len, uint64_t n, uint32_t G,
                          uint32_t nkeys, int whole_line, const LcSplitRegexSlsCfg& c, const LcFilterSlsCfg& f,
                          const lc_filter_desc_t* fd, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                          size_t nctr, uint64_t* counters, const Lz4Tail* z, const TsArgs* ta = nullptr,
                          const LcSplitRegexTsCfg* tc = nullptr) {
    uint64_t ctr[LC_SRTS_COUNTERS] = {0};
    int rc;
    if (n * (uint64_t)G >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^32 captures per call");
    const bool caps = !whole_line && nkeys && nkeys <= G;
    if (!whole_line) {
        CU_TRY(e->dr_status.ensure(n));
        CU_TRY(e->dr_cap_off.ensure(n * G * 4 + 4));
        CU_TRY(e->dr_cap_len.ensure(n * G * 4 + 4));
        rc = regex_parse_dev_impl(e, re, e->in.as<uint8_t>(), len, len, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), 1, n, nkeys, e->dr_status.as<uint8_t>(),
                                  e->dr_cap_off.as<uint32_t>(), e->dr_cap_len.as<uint32_t>(), false);
        if (rc)
            return rc;
    }
    const lck::RegexSlsTables t{e->in.as<uint8_t>(), e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(),
                                whole_line ? nullptr : e->dr_status.as<uint8_t>(),
                                caps ? e->dr_cap_off.as<uint32_t>() : nullptr,
                                caps ? e->dr_cap_len.as<uint32_t>() : nullptr};
    const uint8_t* keep = nullptr;
    const uint64_t* d_removed = nullptr;
    if (fd) {
        rc = filter_sls_run(e, what, c, f, fd, t, n, len, &keep, &d_removed);
        if (rc)
            return rc;
    }
    lck::TsRowTables ts{};
    if (ta) {
        rc = split_regex_ts_run(e, c, *tc, *ta, t, n, &ts);
        if (rc)
            return rc;
    }
    rc = split_regex_sls_run(e, what, c, t, n, nullptr, out, out_cap, out_len, ctr, z, keep, ta ? tc : nullptr, &ts);
    if (d_removed && (rc == LC_OK || rc == LC_ERR_CAPACITY)) {
        CU_TRY(cudaMemcpyAsync(&ctr[3], d_removed, 8, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    if (counters)
        memcpy(counters, ctr, nctr * sizeof(uint64_t));
    return rc;
}

// Host-buffer split + regex + serialise (lc_split_regex_parse_sls and the multiline / LZ4 siblings)
template <class Split>
int split_regex_sls_host(lc_engine_t* e, const char* what, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                         Split split, SPLIT_REGEX_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                         uint64_t* n_events, uint64_t* counters, const Lz4Tail* z,
                         const lc_filter_desc_t* fd = nullptr, const TsArgs* ta = nullptr) {
    const size_t nctr = fd ? 4 : ta ? LC_SRTS_COUNTERS : 3;
    uint32_t G = 0;
    LcSplitRegexSlsCfg c;
    LcFilterSlsCfg f;
    LcSplitRegexTsCfg tc;
    auto begin = [&]() {
        if (counters)
            memset(counters, 0, nctr * sizeof(uint64_t));
        return whole_line ? (int)LC_OK : check_regex_usable(re, what);
    };
    auto config = [&]() {
        G = whole_line ? 0u : re->res.ngroups;
        return split_regex_sls_config(e, what, len, SPLIT_REGEX_ARGS, G, &c, fd, &f, ta, &tc);
    };
    auto run = [&](uint64_t n) {
        return split_regex_sls_stage(e, what, re, len, n, G, nkeys, whole_line, c, f, fd, out, out_cap, out_len, nctr,
                                     counters, z, ta, &tc);
    };
    return split_chain_sls_host(e, what, buf, len, split, (re || whole_line) && (!ta || ta->ts), begin, config, run,
                                out, out_cap, out_len, n_events, z);
}

template <class Split>
int split_regex_lz4_host(lc_engine_t* e, const char* what, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                         Split split, SPLIT_REGEX_PARAMS, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                         uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                         uint64_t* counters, const lc_filter_desc_t* fd = nullptr, const TsArgs* ta = nullptr) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_regex_sls_host(e, what, re, buf, len, split, SPLIT_REGEX_ARGS, out, out_cap, out_len, n_events,
                                counters, &z, fd, ta);
}

// lc_sls_serialize_split_regex_dev and its _filter_ sibling (fd; counters then has a 4th entry) and _timestamp_
// sibling (tc, ts: the timestamp tables; counters then has LC_SRTS_COUNTERS entries)
int split_regex_sls_dev(lc_engine_t* e, const char* what, const uint8_t* d_src, uint64_t src_len,
                        const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                        const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch, SPLIT_REGEX_PARAMS,
                        const lc_filter_desc_t* fd, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
                        uint64_t* counters, const LcSplitRegexTsCfg* tc = nullptr,
                        const lck::TsRowTables* ts = nullptr) {
    const bool caps = !whole_line && nkeys && nkeys <= row_pitch; // the parsed plan reads the capture tables
    if (!e || !out_len || (n && (!d_src || !d_off || !d_len)) || (n && !whole_line && !d_status) ||
        (n && caps && (!d_cap_off || !d_cap_len)) || (n && tc && (!ts->status || !ts->sec || !ts->nsec)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    const size_t nctr = fd ? 4 : tc ? LC_SRTS_COUNTERS : 3;
    if (counters)
        memset(counters, 0, nctr * sizeof(uint64_t));
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)row_pitch >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces and < 2^32 captures per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitRegexSlsCfg c;
    LcFilterSlsCfg f;
    rc = split_regex_sls_config(e, what, src_len, SPLIT_REGEX_ARGS, row_pitch, &c, fd, &f);
    if (rc)
        return rc;
    const char* why = tc ? lc_split_regex_ts_ns_check(c, (int)tc->enable_ns) : nullptr;
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    if (n == 0)
        return LC_OK;
    const lck::RegexSlsTables t{d_src, d_off, d_len, whole_line ? nullptr : d_status, caps ? d_cap_off : nullptr,
                                caps ? d_cap_len : nullptr};
    const uint8_t* keep = nullptr;
    const uint64_t* d_removed = nullptr;
    if (fd) {
        rc = filter_sls_run(e, what, c, f, fd, t, n, src_len, &keep, &d_removed);
        if (rc)
            return rc;
    }
    uint64_t ctr[LC_SRTS_COUNTERS] = {0};
    rc = split_regex_sls_run(e, what, c, t, n, d_out, nullptr, out_cap, out_len, ctr, nullptr, keep, tc, ts);
    if (d_removed && (rc == LC_OK || rc == LC_ERR_CAPACITY)) {
        CU_TRY(cudaMemcpyAsync(&ctr[3], d_removed, 8, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    if (counters)
        memcpy(counters, ctr, nctr * sizeof(uint64_t));
    return rc;
}

} // namespace

extern "C" {

int lc_sls_serialize_split_regex_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
                                     SPLIT_REGEX_PARAMS, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
                                     uint64_t counters[3]) {
    return split_regex_sls_dev(e, "lc_sls_serialize_split_regex_dev", d_src, src_len, d_off, d_len, n, d_status,
                               d_cap_off, d_cap_len, row_pitch, SPLIT_REGEX_ARGS, nullptr, d_out, out_cap, out_len,
                               counters);
}

int lc_sls_serialize_split_regex_filter_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len,
                                            const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                            const uint8_t* d_status, const uint32_t* d_cap_off,
                                            const uint32_t* d_cap_len, uint32_t row_pitch, SPLIT_REGEX_PARAMS,
                                            const lc_filter_desc_t* filter, uint8_t* d_out, uint64_t out_cap,
                                            uint64_t* out_len, uint64_t counters[4]) {
    static const char* what = "lc_sls_serialize_split_regex_filter_dev";
    if (!filter)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    return split_regex_sls_dev(e, what, d_src, src_len, d_off, d_len, n, d_status, d_cap_off, d_cap_len, row_pitch,
                               SPLIT_REGEX_ARGS, filter, d_out, out_cap, out_len, counters);
}

int lc_split_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                             uint8_t split_char, SPLIT_REGEX_PARAMS, uint8_t* out, uint64_t out_cap,
                             uint64_t* out_len, uint64_t* n_events, uint64_t counters[3]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_sls_host(e, "lc_split_regex_parse_sls", re, buf, len, split, SPLIT_REGEX_ARGS, out, out_cap,
                                out_len, n_events, counters, nullptr);
}

int lc_split_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                 uint8_t split_char, SPLIT_REGEX_PARAMS, const uint8_t* tail, uint64_t tail_len,
                                 uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                 uint64_t* n_events, uint64_t counters[3]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_lz4_host(e, "lc_split_regex_parse_sls_lz4", re, buf, len, split, SPLIT_REGEX_ARGS, tail,
                                tail_len, out, out_cap, out_len, raw_len, n_events, counters);
}

// (the multiline splitter's own counters[3] are added to ml_counters as lc_multiline_split_dev adds them)
#define ML_SPLIT                                                                                                       \
    [&](uint64_t* n) {                                                                                                 \
        return lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,               \
                                      e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), len,  \
                                      n, ml_counters);                                                                 \
    }

int lc_multiline_split_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                       const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                       int discard_unmatched, SPLIT_REGEX_PARAMS, uint8_t* out, uint64_t out_cap,
                                       uint64_t* out_len, uint64_t* n_events, uint64_t counters[3],
                                       uint64_t ml_counters[3]) {
    return split_regex_sls_host(e, "lc_multiline_split_regex_parse_sls", re, buf, len, ML_SPLIT, SPLIT_REGEX_ARGS,
                                out, out_cap, out_len, n_events, counters, nullptr);
}

int lc_multiline_split_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                           const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                           int discard_unmatched, SPLIT_REGEX_PARAMS, const uint8_t* tail,
                                           uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                           uint64_t* raw_len, uint64_t* n_events, uint64_t counters[3],
                                           uint64_t ml_counters[3]) {
    return split_regex_lz4_host(e, "lc_multiline_split_regex_parse_sls_lz4", re, buf, len, ML_SPLIT,
                                SPLIT_REGEX_ARGS, tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters);
}

#define FILTER_CHECK(name)                                                                                             \
    if (!filter)                                                                                                       \
        return fail(LC_ERR_INVALID_ARG, std::string(name) + ": bad arguments");

int lc_split_regex_filter_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                    uint8_t split_char, SPLIT_REGEX_PARAMS, const lc_filter_desc_t* filter,
                                    uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                    uint64_t counters[4]) {
    FILTER_CHECK("lc_split_regex_filter_parse_sls")
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_sls_host(e, "lc_split_regex_filter_parse_sls", re, buf, len, split, SPLIT_REGEX_ARGS, out,
                                out_cap, out_len, n_events, counters, nullptr, filter);
}

int lc_split_regex_filter_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                        uint8_t split_char, SPLIT_REGEX_PARAMS, const lc_filter_desc_t* filter,
                                        const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                        uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                        uint64_t counters[4]) {
    FILTER_CHECK("lc_split_regex_filter_parse_sls_lz4")
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_lz4_host(e, "lc_split_regex_filter_parse_sls_lz4", re, buf, len, split, SPLIT_REGEX_ARGS, tail,
                                tail_len, out, out_cap, out_len, raw_len, n_events, counters, filter);
}

int lc_multiline_split_regex_filter_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                              const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                              int discard_unmatched, SPLIT_REGEX_PARAMS,
                                              const lc_filter_desc_t* filter, uint8_t* out, uint64_t out_cap,
                                              uint64_t* out_len, uint64_t* n_events, uint64_t counters[4],
                                              uint64_t ml_counters[3]) {
    FILTER_CHECK("lc_multiline_split_regex_filter_parse_sls")
    return split_regex_sls_host(e, "lc_multiline_split_regex_filter_parse_sls", re, buf, len, ML_SPLIT,
                                SPLIT_REGEX_ARGS, out, out_cap, out_len, n_events, counters, nullptr, filter);
}

int lc_multiline_split_regex_filter_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf,
                                                  uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
                                                  const lc_regex_t* end, int discard_unmatched, SPLIT_REGEX_PARAMS,
                                                  const lc_filter_desc_t* filter, const uint8_t* tail,
                                                  uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                                  uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                                  uint64_t counters[4], uint64_t ml_counters[3]) {
    FILTER_CHECK("lc_multiline_split_regex_filter_parse_sls_lz4")
    return split_regex_lz4_host(e, "lc_multiline_split_regex_filter_parse_sls_lz4", re, buf, len, ML_SPLIT,
                                SPLIT_REGEX_ARGS, tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters,
                                filter);
}
#undef FILTER_CHECK

int lc_split_regex_timestamp_tap_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
                                     const char* const* keys, const uint32_t* key_lens, uint32_t nkeys,
                                     const char* source_key, uint32_t source_key_len, const char* renamed_key,
                                     uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,
                                     int whole_line, const char* offset_key, uint32_t offset_key_len,
                                     const char* tkey, uint32_t tkey_len, uint32_t* d_val_off, uint32_t* d_val_len) {
    static const char* what = "lc_split_regex_timestamp_tap_dev";
    const bool caps = !whole_line && nkeys && nkeys <= row_pitch;
    if (!e || (n && (!d_src || !d_off || !d_len || !d_val_off || !d_val_len)) || (n && !whole_line && !d_status) ||
        (n && caps && (!d_cap_off || !d_cap_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)row_pitch >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces and < 2^32 captures per call");
    int rc = bind(e);
    if (rc)
        return rc;
    const uint64_t src_pos = 0;
    const uint32_t time = 0, time_ns = LC_SLS_NO_NS;
    const TsArgs ta{tkey, tkey_len, nullptr, 0, -1, 0};
    LcSplitRegexSlsCfg c;
    LcSplitRegexTsCfg tc;
    rc = split_regex_sls_config(e, what, src_len, SPLIT_REGEX_ARGS, row_pitch, &c, nullptr, nullptr, &ta, &tc);
    if (rc || n == 0)
        return rc;
    const lck::RegexSlsTables t{d_src, d_off, d_len, whole_line ? nullptr : d_status, caps ? d_cap_off : nullptr,
                                caps ? d_cap_len : nullptr};
    lck::launch_split_regex_ts_tap(c, tc, t, n, d_val_off, d_val_len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int lc_sls_serialize_split_regex_timestamp_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len,
                                               const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                               const uint8_t* d_status, const uint32_t* d_cap_off,
                                               const uint32_t* d_cap_len, uint32_t row_pitch, SPLIT_REGEX_PARAMS,
                                               const uint8_t* d_ts_status, const int64_t* d_ts_sec,
                                               const uint32_t* d_ts_nsec, int enable_ns, uint8_t* d_out,
                                               uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]) {
    const LcSplitRegexTsCfg tc{{LC_FILTER_SLS_ABSENT, LC_FILTER_SLS_ABSENT}, enable_ns != 0 ? 1u : 0u};
    const lck::TsRowTables ts{d_ts_status, d_ts_sec, d_ts_nsec};
    return split_regex_sls_dev(e, "lc_sls_serialize_split_regex_timestamp_dev", d_src, src_len, d_off, d_len, n,
                               d_status, d_cap_off, d_cap_len, row_pitch, SPLIT_REGEX_ARGS, nullptr, d_out, out_cap,
                               out_len, counters, &tc, &ts);
}

#define TS_ARGS_OF_CALL const TsArgs ta{tkey, tkey_len, ts, now, discard_interval, enable_ns};

int lc_split_regex_timestamp_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                       uint8_t split_char, SPLIT_REGEX_PARAMS, const char* tkey, uint32_t tkey_len,
                                       const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns,
                                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                       uint64_t counters[8]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_sls_host(e, "lc_split_regex_timestamp_parse_sls", re, buf, len, split, SPLIT_REGEX_ARGS, out,
                                out_cap, out_len, n_events, counters, nullptr, nullptr, &ta);
}

int lc_split_regex_timestamp_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                           uint8_t split_char, SPLIT_REGEX_PARAMS, const char* tkey,
                                           uint32_t tkey_len, const lc_timestamp_t* ts, int64_t now,
                                           int32_t discard_interval, int enable_ns, const uint8_t* tail,
                                           uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                           uint64_t* raw_len, uint64_t* n_events, uint64_t counters[8]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_regex_lz4_host(e, "lc_split_regex_timestamp_parse_sls_lz4", re, buf, len, split, SPLIT_REGEX_ARGS,
                                tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters, nullptr, &ta);
}

int lc_multiline_split_regex_timestamp_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf,
                                                 uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
                                                 const lc_regex_t* end, int discard_unmatched, SPLIT_REGEX_PARAMS,
                                                 const char* tkey, uint32_t tkey_len, const lc_timestamp_t* ts,
                                                 int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out,
                                                 uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                                 uint64_t counters[8], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    return split_regex_sls_host(e, "lc_multiline_split_regex_timestamp_parse_sls", re, buf, len, ML_SPLIT,
                                SPLIT_REGEX_ARGS, out, out_cap, out_len, n_events, counters, nullptr, nullptr, &ta);
}

int lc_multiline_split_regex_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, SPLIT_REGEX_PARAMS, const char* tkey,
    uint32_t tkey_len, const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns,
    const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
    uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    return split_regex_lz4_host(e, "lc_multiline_split_regex_timestamp_parse_sls_lz4", re, buf, len, ML_SPLIT,
                                SPLIT_REGEX_ARGS, tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters,
                                nullptr, &ta);
}
#undef TS_ARGS_OF_CALL

} // extern "C"

// ------------------------------------------------------------------------------------ split -> delimiter -> SLS
// The delimiter stage's key configuration (lc_sls_serialize_delim_dev's keys .. copy_raw) and the offset content of the
// split events (offset_key -- NULL = no log.file.offset metadata -- and the source event's position, time and ns)
#define DELIM_KEY_PARAMS                                                                                               \
    const char *const *keys, const uint32_t *key_lens, uint32_t nkeys, const char *source_key,                         \
        uint32_t source_key_len, const char *renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed,   \
        int copy_raw
#define DELIM_KEY_ARGS                                                                                                 \
    keys, key_lens, nkeys, source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw
#define OFFSET_PARAMS const char *offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns
#define OFFSET_ARGS offset_key, offset_key_len, src_pos, time, time_ns
// the host-buffer calls' delimiter arguments (lc_delim_parse_sls's sep .. copy_raw) and the offset content
#define SPLIT_DELIM_PARAMS                                                                                             \
    const uint8_t *sep, uint32_t sep_len, uint8_t quote, int extend, int discard, int allow_short,                     \
        uint32_t max_fields, DELIM_KEY_PARAMS, OFFSET_PARAMS
#define SPLIT_DELIM_ARGS sep, sep_len, quote, extend, discard, allow_short, max_fields, DELIM_KEY_ARGS, OFFSET_ARGS

namespace {

// lc_delim_sls_setup + lc_split_delim_sls_link: the delimiter's key strings are staged in `dr_keys`, the offset key in
// `sls_plan`; neither splitter, nor lc_delim_parse_dev, nor the serialiser uses them.  With ta (the timestamp calls),
// the timestamp stage's SourceKey is checked and resolved into *tc (lc_split_delim_ts_setup).
int split_delim_sls_config(lc_engine_t* e, const char* what, uint32_t max_fields, const uint8_t* sep,
                           uint32_t sep_len, uint8_t quote, int extend, int discard, DELIM_KEY_PARAMS, OFFSET_PARAMS,
                           LcSplitDelimSlsCfg* c, const TsArgs* ta = nullptr, LcSplitDelimTsCfg* tc = nullptr) {
    LcDelimSlsCfg d;
    int rc = delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, DELIM_KEY_ARGS, &d,
                              &e->dr_keys);
    if (rc)
        return rc;
    const char* why = lc_split_delim_sls_link(d, keys, key_lens, source_key, source_key_len, renamed_key,
                                              renamed_key_len, offset_key, offset_key_len, src_pos, time, time_ns, c);
    if (!why && ta)
        why = lc_split_delim_ts_setup(*c, keys, key_lens, source_key, source_key_len, renamed_key, renamed_key_len,
                                      offset_key, offset_key_len, ta->tkey, ta->tkey_len, ta->enable_ns, tc);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    if (offset_key) {
        CU_TRY(e->sls_plan.ensure(offset_key_len + 16));
        if (offset_key_len) {
            CU_TRY(cudaMemcpyAsync(e->sls_plan.p, offset_key, offset_key_len, cudaMemcpyHostToDevice, e->stream));
            // (pageable source: its bytes must be on the device before it dies)
            CU_TRY(cudaStreamSynchronize(e->stream));
        }
        c->okey = e->sls_plan.as<uint8_t>();
    }
    return LC_OK;
}

// The size pass and the emit of the chain over the n pieces of t (serialize_sls_dev): into d_out (the device-fed
// call), or back to the host buffer out, or -- with z -- records ‖ tail as one LZ4 block.  counters[4] (or nullptr) =
// successful, failed, discarded, blank; set whenever the size pass ran.  With tc (the timestamp calls), each record's
// time comes from the timestamp tables ts and counters has LC_SDTS_COUNTERS entries.
int split_delim_sls_run(lc_engine_t* e, const char* what, const LcSplitDelimSlsCfg& c, const lck::DelimSlsTables& t,
                        uint64_t n, uint8_t* d_out, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                        uint64_t* counters, const Lz4Tail* z, const LcSplitDelimTsCfg* tc = nullptr,
                        const lck::TsRowTables* ts = nullptr) {
    const uint32_t nstage = tc ? LC_SDTS_COUNTERS : 4u;
    uint64_t ctr[LC_SDTS_COUNTERS + 1] = {0}; // + pieces whose record would reach 4 GiB
    SlsTo to;
    to.host = out;
    to.z = z;
    to.too_large = (int)nstage;
    const int rc = serialize_sls_dev(
        e, what, n, nstage + 1,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* d_ctr) {
            if (tc)
                lck::launch_split_delim_ts_sls_sizes(c, *tc, t, *ts, n, rec, body, d_ctr, e->stream);
            else
                lck::launch_split_delim_sls_sizes(c, t, n, rec, body, d_ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* dst) {
            if (tc)
                lck::launch_split_delim_ts_sls_emit(c, *tc, t, *ts, n, rec_off, body, dst, e->stream);
            else
                lck::launch_split_delim_sls_emit(c, t, n, rec_off, body, dst, e->stream);
        },
        d_out, out_cap, out_len, ctr, to);
    if (counters)
        memcpy(counters, ctr, nstage * sizeof(uint64_t));
    return rc;
}

// The split -> delimiter -> timestamp chain's tap and timestamp passes over the n pieces of t: the value buffer
// `sjt_val` (as long as the source value) and the value table into st_val, then lc_timestamp_parse_dev's two passes
// with the whole source value as one group into *ts (st_status, st_sec, st_nsec).  The stage's counters are the size
// pass's, so the passes' own go to ts_cnt unread.
int split_delim_ts_run(lc_engine_t* e, const LcSplitDelimSlsCfg& c, const LcSplitDelimTsCfg& tc, const TsArgs& ta,
                       const lck::DelimSlsTables& t, uint64_t n, uint64_t src_len, lck::TsRowTables* ts) {
    CU_TRY(e->st_val.ensure(n * 8 + 8));
    CU_TRY(e->st_sec.ensure(n * 8));
    CU_TRY(e->st_nsec.ensure(n * 4));
    CU_TRY(e->st_status.ensure(n));
    CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
    CU_TRY(e->sjt_val.ensure(src_len + 16));
    uint32_t* off = e->st_val.as<uint32_t>();
    uint32_t *len = off + n, *grp = off + 2 * n;
    const uint32_t g[2] = {0u, (uint32_t)n};
    CU_TRY(cudaMemcpyAsync(grp, g, sizeof g, cudaMemcpyHostToDevice, e->stream));
    lck::launch_split_delim_ts_tap(c, tc, t, n, e->sjt_val.as<uint8_t>(), off, len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    const int rc = ts_run(e, ta.ts, e->sjt_val.as<uint8_t>(), LcTsSpans{off, len, nullptr, 1}, n, grp, 1, ta.now,
                          ta.discard_interval, e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>(),
                          e->st_status.as<uint8_t>(), e->ts_cnt.as<uint64_t>());
    *ts = lck::TsRowTables{e->st_status.as<uint8_t>(), e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>()};
    return rc;
}

// Host-buffer split + delimiter + serialise (lc_split_delim_parse_sls and the multiline / LZ4 siblings, through
// split_chain_sls_host).  Workspace: the source in `in`, the piece tables in out_a / out_b (out_c: the multiline
// flags), the delimiter tables in dr_status (status), dr_val_off (column counts), out_d / out_e / dr_cap_off (f_off /
// f_len / f_dq, [n][max_fields]), the key strings in dr_keys and sls_plan.  The splitters, lc_delim_parse_dev (its
// tiled kernel stages in shared memory) and the serialiser (lab_sizes, cnt, lab_off, state, desc, lab, z_*) use none
// of the others'.  With ta (the _timestamp_ calls), the tap and the timestamp passes (sjt_val, st_*, ts_*) run between
// the delimiter stage and the size pass and counters has LC_SDTS_COUNTERS entries.
template <class Split>
int split_delim_sls_host(lc_engine_t* e, const char* what, const uint8_t* buf, uint64_t len, Split split,
                         SPLIT_DELIM_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                         uint64_t* counters, const Lz4Tail* z, const TsArgs* ta = nullptr) {
    LcSplitDelimSlsCfg c;
    LcSplitDelimTsCfg tc;
    auto begin = [&]() {
        if (counters)
            memset(counters, 0, (ta ? LC_SDTS_COUNTERS : 4) * sizeof(uint64_t));
        return (int)LC_OK;
    };
    auto config = [&]() {
        return split_delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, DELIM_KEY_ARGS,
                                      OFFSET_ARGS, &c, ta, &tc);
    };
    auto run = [&](uint64_t n) {
        if (n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^30 pieces and < 2^32 columns per call");
        const uint64_t fbytes = n * max_fields * 4;
        CU_TRY(e->dr_status.ensure(n));
        CU_TRY(e->dr_val_off.ensure(n * 4));
        CU_TRY(e->out_d.ensure(fbytes));
        CU_TRY(e->out_e.ensure(fbytes));
        CU_TRY(e->dr_cap_off.ensure(fbytes));
        const lck::DelimSlsTables t{e->in.as<uint8_t>(),         e->out_a.as<uint32_t>(),
                                    e->out_b.as<uint32_t>(),     e->dr_status.as<uint8_t>(),
                                    e->dr_val_off.as<uint32_t>(), e->out_d.as<uint32_t>(),
                                    e->out_e.as<uint32_t>(),     e->dr_cap_off.as<uint32_t>()};
        int rc = lc_delim_parse_dev(e, t.base, len, t.ev_off, t.ev_len, n, sep, sep_len, quote, nkeys, extend,
                                    allow_short, max_fields, e->dr_status.as<uint8_t>(),
                                    e->dr_val_off.as<uint32_t>(), e->out_d.as<uint32_t>(), e->out_e.as<uint32_t>(),
                                    e->dr_cap_off.as<uint32_t>());
        if (rc)
            return rc;
        lck::TsRowTables ts{};
        if (ta) {
            rc = split_delim_ts_run(e, c, tc, *ta, t, n, len, &ts);
            if (rc)
                return rc;
        }
        return split_delim_sls_run(e, what, c, t, n, nullptr, out, out_cap, out_len, counters, z, ta ? &tc : nullptr,
                                   &ts);
    };
    return split_chain_sls_host(e, what, buf, len, split, sep != nullptr && (!ta || ta->ts), begin, config, run, out,
                                out_cap, out_len, n_events, z);
}

} // namespace

extern "C" {

int lc_sls_serialize_split_delim_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                                     const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                                     uint8_t quote, int extend, int discard, DELIM_KEY_PARAMS, OFFSET_PARAMS,
                                     uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t counters[4]) {
    static const char* what = "lc_sls_serialize_split_delim_dev";
    if (!e || !out_len || (n && (!d_src || !d_off || !d_len || !d_status || !d_nfields || !d_f_off || !d_f_len ||
                                 !d_f_dq)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, 4 * sizeof(uint64_t));
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitDelimSlsCfg c;
    rc = split_delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, DELIM_KEY_ARGS, OFFSET_ARGS,
                                &c);
    if (rc || n == 0)
        return rc;
    const lck::DelimSlsTables t{d_src, d_off, d_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq};
    return split_delim_sls_run(e, what, c, t, n, d_out, nullptr, out_cap, out_len, counters, nullptr);
}

int lc_split_delim_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char,
                             SPLIT_DELIM_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                             uint64_t* n_events, uint64_t counters[4]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_delim_sls_host(e, "lc_split_delim_parse_sls", buf, len, split, SPLIT_DELIM_ARGS, out, out_cap,
                                out_len, n_events, counters, nullptr);
}

int lc_split_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char,
                                 SPLIT_DELIM_PARAMS, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                                 uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                 uint64_t counters[4]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_sls_host(e, "lc_split_delim_parse_sls_lz4", buf, len, split, SPLIT_DELIM_ARGS, out, out_cap,
                                out_len, n_events, counters, &z);
}

int lc_multiline_split_delim_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                       const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched,
                                       SPLIT_DELIM_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                       uint64_t* n_events, uint64_t counters[4], uint64_t ml_counters[3]) {
    return split_delim_sls_host(e, "lc_multiline_split_delim_parse_sls", buf, len, ML_SPLIT, SPLIT_DELIM_ARGS, out,
                                out_cap, out_len, n_events, counters, nullptr);
}

int lc_multiline_split_delim_parse_sls_lz4(lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
                                           const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched,
                                           SPLIT_DELIM_PARAMS, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                                           uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                           uint64_t* n_events, uint64_t counters[4], uint64_t ml_counters[3]) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_sls_host(e, "lc_multiline_split_delim_parse_sls_lz4", buf, len, ML_SPLIT, SPLIT_DELIM_ARGS,
                                out, out_cap, out_len, n_events, counters, &z);
}
} // extern "C"

// ------------------------------------------------------------------------------ split -> delimiter -> regex -> SLS
namespace {

// lc_delim_sls_setup + lc_regex_sls_setup + lc_split_delim_regex_sls_link: the delimiter's key strings are staged in
// `dr_keys`, the regex plans in `sls_plan` and the offset key in `sdr_okey`.  pitch = the regex tables' row pitch.
int split_delim_regex_config(lc_engine_t* e, const char* what, uint32_t max_fields, CHAIN_PARAMS, OFFSET_PARAMS,
                             uint32_t pitch, LcSplitDelimRegexSlsCfg* c) {
    memset(c, 0, sizeof *c);
    int rc = delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, keys, key_lens, nkeys,
                              source_key, source_key_len, renamed_key, renamed_key_len, keep_fail, keep_succeed,
                              copy_raw, &c->r.d, &e->dr_keys);
    if (rc)
        return rc;
    rc = regex_sls_config(e, what, rkeys, rkey_lens, rnkeys, rsource_key, rsource_key_len, rrenamed_key,
                          rrenamed_key_len, rkeep_fail, rkeep_succeed, rcopy_raw, whole_line, pitch, &c->r.x);
    if (rc)
        return rc;
    const char* why = lc_split_delim_regex_sls_link(keys, key_lens, source_key, source_key_len, renamed_key,
                                                    renamed_key_len, rkeys, rkey_lens, rnkeys, rsource_key,
                                                    rsource_key_len, rrenamed_key, rrenamed_key_len, rkeep_fail,
                                                    rkeep_succeed, rcopy_raw, whole_line, OFFSET_ARGS, c);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    if (offset_key) {
        CU_TRY(e->sdr_okey.ensure(offset_key_len + 16));
        if (offset_key_len) {
            CU_TRY(cudaMemcpyAsync(e->sdr_okey.p, offset_key, offset_key_len, cudaMemcpyHostToDevice, e->stream));
            // (pageable source: its bytes must be on the device before it dies)
            CU_TRY(cudaStreamSynchronize(e->stream));
        }
        c->s.okey = e->sdr_okey.as<uint8_t>();
    }
    return LC_OK;
}

// The size pass and the emit of the chain over the n pieces of t (serialize_sls_dev): into d_out (the device-fed
// call), or back to the host buffer out, or -- with z -- records ‖ tail as one LZ4 block.  counters[8] (or nullptr) as
// lc_delim_regex_verdict orders them; set whenever the size pass ran.
int split_delim_regex_sls_run(lc_engine_t* e, const char* what, const LcSplitDelimRegexSlsCfg& c,
                              const lck::DelimRegexSlsTables& t, uint64_t n, uint8_t* d_out, uint8_t* out,
                              uint64_t out_cap, uint64_t* out_len, uint64_t* counters, const Lz4Tail* z) {
    uint64_t ctr[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; // + pieces whose record would reach 4 GiB
    SlsTo to;
    to.host = out;
    to.z = z;
    to.too_large = 8;
    const int rc = serialize_sls_dev(
        e, what, n, 9,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* d_ctr) {
            lck::launch_split_delim_regex_sls_sizes(c, t, n, rec, body, d_ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* dst) {
            lck::launch_split_delim_regex_sls_emit(c, t, n, rec_off, body, dst, e->stream);
        },
        d_out, out_cap, out_len, ctr, to);
    if (counters)
        memcpy(counters, ctr, 8 * sizeof(uint64_t));
    return rc;
}

// Host-buffer split + delimiter + tap + regex + serialise (lc_split_delim_regex_parse_sls and the multiline / LZ4
// siblings, through split_chain_sls_host).  Workspace:
//   in                      the source [0, len), then the tap's side copies from align16(len): a copy is never longer
//                           than its piece and the pieces do not overlap, so len bytes hold them all
//   out_a / out_b (out_c)   the piece tables (the multiline flags)
//   sdr_status, sdr_nf,     the delimiter tables over the pieces (status, column counts, [n][max_fields] f_off /
//   sdr_f_off / _len / _dq  f_len / f_dq); the split -> delimiter chain's dr_status / dr_val_off / out_d / out_e /
//                           dr_cap_off are the value and regex tables or the regex stage's scratch here
//   dr_val_off / dr_val_len the value table (the tap), dr_copy / dr_slot / dr_desc its sizes, slots and scan
//   dr_status, dr_cap_off / dr_cap_len   the regex tables over the values
//   dr_keys, sls_plan, sdr_okey          the delimiter's key strings, the regex plans, the offset key
// The splitters, lc_delim_parse_dev (its tiled kernel stages in shared memory), the regex stage (order, lab*, desc,
// small; out_d / out_e only for a match without captures) and the serialiser (lab_sizes, cnt, lab_off, state, desc,
// lab, z_*) use none of the others'.
template <class Split>
int split_delim_regex_sls_host(lc_engine_t* e, const char* what, const lc_regex_t* re, const uint8_t* buf,
                               uint64_t len, Split split, int allow_short, uint32_t max_fields, CHAIN_PARAMS,
                               OFFSET_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                               uint64_t counters[8], const Lz4Tail* z) {
    const uint64_t side_at = (len + 15) & ~15ull, arena = side_at + len;
    uint32_t G = 0;
    LcSplitDelimRegexSlsCfg c;
    auto begin = [&]() {
        if (counters)
            memset(counters, 0, 8 * sizeof(uint64_t));
        if (arena + 16 >= 0xFFFFFFF0ull)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the source and its side copies must stay below 4 GiB");
        return whole_line ? (int)LC_OK : check_regex_usable(re, what);
    };
    auto config = [&]() {
        G = whole_line ? 0u : re->res.ngroups;
        const int rc = split_delim_regex_config(e, what, max_fields, CHAIN_ARGS, OFFSET_ARGS, G, &c);
        if (rc)
            return rc;
        CU_TRY(e->in.ensure(arena + 16)); // before the upload: `in` does not keep its bytes when it grows
        return (int)LC_OK;
    };
    auto run = [&](uint64_t n) {
        if (n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32) || n * (uint64_t)G >= (1ull << 32))
            return fail(LC_ERR_TOO_LARGE,
                        std::string(what) + ": < 2^30 pieces, < 2^32 columns and < 2^32 captures per call");
        const uint64_t fbytes = n * max_fields * 4, dwords = lck::scan_tiles(n) + 3;
        CU_TRY(e->sdr_status.ensure(n));
        CU_TRY(e->sdr_nf.ensure(n * 4));
        CU_TRY(e->sdr_f_off.ensure(fbytes));
        CU_TRY(e->sdr_f_len.ensure(fbytes));
        CU_TRY(e->sdr_f_dq.ensure(fbytes));
        CU_TRY(e->dr_val_off.ensure(n * 4));
        CU_TRY(e->dr_val_len.ensure(n * 4));
        CU_TRY(e->dr_copy.ensure(n * 4));
        CU_TRY(e->dr_slot.ensure(n * 8));
        CU_TRY(e->dr_desc.ensure(dwords * 8));
        CU_TRY(cudaMemsetAsync(e->dr_desc.p, 0, dwords * 8, e->stream));
        uint8_t* base = e->in.as<uint8_t>();
        const lck::DelimSlsTables dt{base,
                                     e->out_a.as<uint32_t>(),
                                     e->out_b.as<uint32_t>(),
                                     e->sdr_status.as<uint8_t>(),
                                     e->sdr_nf.as<uint32_t>(),
                                     e->sdr_f_off.as<uint32_t>(),
                                     e->sdr_f_len.as<uint32_t>(),
                                     e->sdr_f_dq.as<uint32_t>()};
        int rc = lc_delim_parse_dev(e, base, len, dt.ev_off, dt.ev_len, n, sep, sep_len, quote, nkeys, extend,
                                    allow_short, max_fields, e->sdr_status.as<uint8_t>(), e->sdr_nf.as<uint32_t>(),
                                    e->sdr_f_off.as<uint32_t>(), e->sdr_f_len.as<uint32_t>(),
                                    e->sdr_f_dq.as<uint32_t>());
        if (rc)
            return rc;
        queue_tap(e, c.r, dt, n, side_at, base, e->dr_copy.as<uint32_t>(), e->dr_slot.as<uint64_t>(),
                  e->dr_desc.as<uint64_t>(), e->dr_val_off.as<uint32_t>(), e->dr_val_len.as<uint32_t>());
        CU_TRY(cudaGetLastError());
        const bool caps = !whole_line && rnkeys && rnkeys <= G;
        if (!whole_line) {
            CU_TRY(e->dr_status.ensure(n));
            CU_TRY(e->dr_cap_off.ensure(n * G * 4 + 4));
            CU_TRY(e->dr_cap_len.ensure(n * G * 4 + 4));
            // (the values lie in the pieces or their side copies: len bytes at most)
            rc = regex_parse_dev_impl(e, re, base, arena, len, e->dr_val_off.as<uint32_t>(),
                                      e->dr_val_len.as<uint32_t>(), 1, n, rnkeys, e->dr_status.as<uint8_t>(),
                                      e->dr_cap_off.as<uint32_t>(), e->dr_cap_len.as<uint32_t>(), false);
            if (rc)
                return rc;
        }
        const lck::DelimRegexSlsTables t{dt,
                                         e->dr_val_off.as<uint32_t>(),
                                         e->dr_val_len.as<uint32_t>(),
                                         whole_line ? nullptr : e->dr_status.as<uint8_t>(),
                                         caps ? e->dr_cap_off.as<uint32_t>() : nullptr,
                                         caps ? e->dr_cap_len.as<uint32_t>() : nullptr};
        return split_delim_regex_sls_run(e, what, c, t, n, nullptr, out, out_cap, out_len, counters, z);
    };
    return split_chain_sls_host(e, what, buf, len, split, (re || whole_line) && sep != nullptr, begin, config, run,
                                out, out_cap, out_len, n_events, z);
}

} // namespace

// the host-buffer calls' stage arguments: the delimiter's allow_short / max_fields and both stages' (CHAIN_PARAMS),
// then the offset content
#define SPLIT_DELIM_REGEX_PARAMS int allow_short, uint32_t max_fields, CHAIN_PARAMS, OFFSET_PARAMS
#define SPLIT_DELIM_REGEX_ARGS allow_short, max_fields, CHAIN_ARGS, OFFSET_ARGS

extern "C" {

int lc_sls_serialize_split_delim_regex_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len,
                                           const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                           const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off,
                                           const uint32_t* d_f_len, const uint32_t* d_f_dq, uint32_t max_fields,
                                           CHAIN_PARAMS, OFFSET_PARAMS, const uint32_t* d_val_off,
                                           const uint32_t* d_val_len, const uint8_t* d_re_status,
                                           const uint32_t* d_cap_off, const uint32_t* d_cap_len, uint32_t row_pitch,
                                           uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
                                           uint64_t counters[8]) {
    static const char* what = "lc_sls_serialize_split_delim_regex_dev";
    const bool caps = !whole_line && rnkeys && rnkeys <= row_pitch; // the parsed plan reads the capture tables
    if (!e || !out_len || (n && (!d_src || !d_off || !d_len || !d_status || !d_nfields || !d_f_off || !d_f_len ||
                                 !d_f_dq || !d_val_off || !d_val_len)) ||
        (n && !whole_line && !d_re_status) || (n && caps && (!d_cap_off || !d_cap_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, 8 * sizeof(uint64_t));
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32) ||
        n * (uint64_t)row_pitch >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces, < 2^32 columns and < 2^32 captures "
                                      "per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitDelimRegexSlsCfg c;
    rc = split_delim_regex_config(e, what, max_fields, CHAIN_ARGS, OFFSET_ARGS, row_pitch, &c);
    if (rc || n == 0)
        return rc;
    const lck::DelimRegexSlsTables t{{d_src, d_off, d_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq},
                                     d_val_off,
                                     d_val_len,
                                     whole_line ? nullptr : d_re_status,
                                     caps ? d_cap_off : nullptr,
                                     caps ? d_cap_len : nullptr};
    return split_delim_regex_sls_run(e, what, c, t, n, d_out, nullptr, out_cap, out_len, counters, nullptr);
}

int lc_split_delim_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                   uint8_t split_char, SPLIT_DELIM_REGEX_PARAMS, uint8_t* out, uint64_t out_cap,
                                   uint64_t* out_len, uint64_t* n_events, uint64_t counters[8]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_delim_regex_sls_host(e, "lc_split_delim_regex_parse_sls", re, buf, len, split,
                                      SPLIT_DELIM_REGEX_ARGS, out, out_cap, out_len, n_events, counters, nullptr);
}

int lc_split_delim_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                       uint8_t split_char, SPLIT_DELIM_REGEX_PARAMS, const uint8_t* tail,
                                       uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                       uint64_t* raw_len, uint64_t* n_events, uint64_t counters[8]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_regex_sls_host(e, "lc_split_delim_regex_parse_sls_lz4", re, buf, len, split,
                                      SPLIT_DELIM_REGEX_ARGS, out, out_cap, out_len, n_events, counters, &z);
}

int lc_multiline_split_delim_regex_parse_sls(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf, uint64_t len,
                                             const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                             int discard_unmatched, SPLIT_DELIM_REGEX_PARAMS, uint8_t* out,
                                             uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                             uint64_t counters[8], uint64_t ml_counters[3]) {
    return split_delim_regex_sls_host(e, "lc_multiline_split_delim_regex_parse_sls", re, buf, len, ML_SPLIT,
                                      SPLIT_DELIM_REGEX_ARGS, out, out_cap, out_len, n_events, counters, nullptr);
}

int lc_multiline_split_delim_regex_parse_sls_lz4(lc_engine_t* e, const lc_regex_t* re, const uint8_t* buf,
                                                 uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
                                                 const lc_regex_t* end, int discard_unmatched,
                                                 SPLIT_DELIM_REGEX_PARAMS, const uint8_t* tail, uint64_t tail_len,
                                                 uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                                 uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_regex_sls_host(e, "lc_multiline_split_delim_regex_parse_sls_lz4", re, buf, len, ML_SPLIT,
                                      SPLIT_DELIM_REGEX_ARGS, out, out_cap, out_len, n_events, counters, &z);
}
#undef ML_SPLIT
#undef SPLIT_DELIM_REGEX_PARAMS
#undef SPLIT_DELIM_REGEX_ARGS

} // extern "C"

// ------------------------------------------------------------------------- split -> delimiter -> timestamp -> SLS
// (the multiline splitter's own counters[3] are added to ml_counters as lc_multiline_split_dev adds them)
#define ML_SPLIT                                                                                                       \
    [&](uint64_t* n) {                                                                                                 \
        return lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,               \
                                      e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), len,  \
                                      n, ml_counters);                                                                 \
    }
#define TS_ARGS_OF_CALL const TsArgs ta{tkey, tkey_len, ts, now, discard_interval, enable_ns};

extern "C" {

int lc_split_delim_timestamp_tap_dev(lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off,
                                     const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                     const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
                                     const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len,
                                     uint8_t quote, int extend, int discard, DELIM_KEY_PARAMS, const char* offset_key,
                                     uint32_t offset_key_len, const char* tkey, uint32_t tkey_len, uint8_t* d_val,
                                     uint64_t val_cap, uint32_t* d_val_off, uint32_t* d_val_len) {
    static const char* what = "lc_split_delim_timestamp_tap_dev";
    if (!e || (tkey_len && !tkey) ||
        (n && (!d_src || !d_off || !d_len || !d_status || !d_nfields || !d_f_off || !d_f_len || !d_f_dq || !d_val ||
               !d_val_off || !d_val_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces and < 2^32 columns per call");
    if (n && val_cap < src_len)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": the value buffer must hold src_len bytes");
    int rc = bind(e);
    if (rc)
        return rc;
    const uint64_t src_pos = 0;
    const uint32_t time = 0, time_ns = LC_SLS_NO_NS;
    const TsArgs ta{tkey, tkey_len, nullptr, 0, -1, 0};
    LcSplitDelimSlsCfg c;
    LcSplitDelimTsCfg tc;
    rc = split_delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, DELIM_KEY_ARGS, OFFSET_ARGS,
                                &c, &ta, &tc);
    if (rc || n == 0)
        return rc;
    const lck::DelimSlsTables t{d_src, d_off, d_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq};
    lck::launch_split_delim_ts_tap(c, tc, t, n, d_val, d_val_off, d_val_len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int lc_sls_serialize_split_delim_timestamp_dev(
    lc_engine_t* e, const uint8_t* d_src, uint64_t src_len, const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
    const uint8_t* d_status, const uint32_t* d_nfields, const uint32_t* d_f_off, const uint32_t* d_f_len,
    const uint32_t* d_f_dq, uint32_t max_fields, const uint8_t* sep, uint32_t sep_len, uint8_t quote, int extend,
    int discard, DELIM_KEY_PARAMS, OFFSET_PARAMS, const uint8_t* d_ts_status, const int64_t* d_ts_sec,
    const uint32_t* d_ts_nsec, int enable_ns, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
    uint64_t counters[9]) {
    static const char* what = "lc_sls_serialize_split_delim_timestamp_dev";
    if (!e || !out_len ||
        (n && (!d_src || !d_off || !d_len || !d_status || !d_nfields || !d_f_off || !d_f_len || !d_f_dq ||
               !d_ts_status || !d_ts_sec || !d_ts_nsec)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, LC_SDTS_COUNTERS * sizeof(uint64_t));
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30) || n * (uint64_t)max_fields >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, "buffer must be < 4 GiB, < 2^30 pieces and < 2^32 columns per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitDelimSlsCfg c;
    rc = split_delim_sls_config(e, what, max_fields, sep, sep_len, quote, extend, discard, DELIM_KEY_ARGS, OFFSET_ARGS,
                                &c);
    if (rc)
        return rc;
    const char* why = lc_split_regex_ts_ns_check(c, enable_ns);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    if (n == 0)
        return LC_OK;
    LcSplitDelimTsCfg tc;
    memset(&tc, 0, sizeof tc);
    tc.enable_ns = enable_ns != 0;
    const lck::DelimSlsTables t{d_src, d_off, d_len, d_status, d_nfields, d_f_off, d_f_len, d_f_dq};
    const lck::TsRowTables ts{d_ts_status, d_ts_sec, d_ts_nsec};
    return split_delim_sls_run(e, what, c, t, n, d_out, nullptr, out_cap, out_len, counters, nullptr, &tc, &ts);
}

int lc_split_delim_timestamp_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char,
                                       SPLIT_DELIM_PARAMS, const char* tkey, uint32_t tkey_len,
                                       const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns,
                                       uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                       uint64_t counters[9]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_delim_sls_host(e, "lc_split_delim_timestamp_parse_sls", buf, len, split, SPLIT_DELIM_ARGS, out,
                                out_cap, out_len, n_events, counters, nullptr, &ta);
}

int lc_split_delim_timestamp_parse_sls_lz4(lc_engine_t* e, const uint8_t* buf, uint64_t len, uint8_t split_char,
                                           SPLIT_DELIM_PARAMS, const char* tkey, uint32_t tkey_len,
                                           const lc_timestamp_t* ts, int64_t now, int32_t discard_interval,
                                           int enable_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                                           uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                           uint64_t counters[9]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_sls_host(e, "lc_split_delim_timestamp_parse_sls_lz4", buf, len, split, SPLIT_DELIM_ARGS, out,
                                out_cap, out_len, n_events, counters, &z, &ta);
}

int lc_multiline_split_delim_timestamp_parse_sls(lc_engine_t* e, const uint8_t* buf, uint64_t len,
                                                 const lc_regex_t* start, const lc_regex_t* cont,
                                                 const lc_regex_t* end, int discard_unmatched, SPLIT_DELIM_PARAMS,
                                                 const char* tkey, uint32_t tkey_len, const lc_timestamp_t* ts,
                                                 int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out,
                                                 uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                                 uint64_t counters[9], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    return split_delim_sls_host(e, "lc_multiline_split_delim_timestamp_parse_sls", buf, len, ML_SPLIT,
                                SPLIT_DELIM_ARGS, out, out_cap, out_len, n_events, counters, nullptr, &ta);
}

int lc_multiline_split_delim_timestamp_parse_sls_lz4(
    lc_engine_t* e, const uint8_t* buf, uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
    const lc_regex_t* end, int discard_unmatched, SPLIT_DELIM_PARAMS, const char* tkey, uint32_t tkey_len,
    const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns, const uint8_t* tail,
    uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
    uint64_t counters[9], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_delim_sls_host(e, "lc_multiline_split_delim_timestamp_parse_sls_lz4", buf, len, ML_SPLIT,
                                SPLIT_DELIM_ARGS, out, out_cap, out_len, n_events, counters, &z, &ta);
}

} // extern "C"
#undef TS_ARGS_OF_CALL
#undef ML_SPLIT

// ------------------------------------------------------------------------------------------------ LZ4
namespace {

// chunk tables of the segments in g (g.in, g.seg_off, g.seg_len, g.nseg set): g.first / g.nchunks, and room for the
// parse.  first_host (or nullptr): the chunk table already built on the host, uploaded instead of counted.
int lz4_chunk_tables(lc_engine_t* e, const char* what, lck::Lz4Segs& g, const uint64_t* first_host,
                     uint64_t nchunks_host) {
    CU_TRY(e->z_first.ensure(g.nseg * 8 + 8));
    uint64_t* d_first = e->z_first.as<uint64_t>();
    if (first_host) {
        CU_TRY(cudaMemcpyAsync(d_first, first_host, g.nseg * 8, cudaMemcpyHostToDevice, e->stream));
        g.nchunks = nchunks_host;
    } else {
        CU_TRY(e->z_size.ensure(g.nseg * 4 + 4));
        uint64_t* desc;
        int rc = prep_desc(e, lck::scan_tiles(g.nseg), &desc);
        if (rc)
            return rc;
        Small* ds = e->small.as<Small>();
        Small* hs = (Small*)e->h_small;
        lck::launch_lz4_chunks(g.seg_len, g.nseg, e->z_size.as<uint32_t>(), &ds->overflow, e->stream);
        lck::launch_exclusive_sum(e->z_size.as<uint32_t>(), g.nseg, d_first, &ds->total, desc, &ds->tickets[2],
                                  e->stream);
        e->launches += 2;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(hs, ds, sizeof(Small), cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        if (hs->overflow)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": a segment is larger than LZ4_MAX_INPUT_SIZE");
        g.nchunks = hs->total;
    }
    g.first = d_first;
    CU_TRY(e->z_seq.ensure(g.nchunks * LC_LZ4_SEQ_CAP * sizeof(LcLz4Seq)));
    CU_TRY(e->z_info.ensure(g.nchunks * sizeof(LcLz4Chunk)));
    CU_TRY(e->z_size.ensure(g.nchunks * 8));
    CU_TRY(e->z_choff.ensure(g.nchunks * 8 + 8));
    return LC_OK;
}

// After the parse of every chunk: sizes, block offsets, and (when the total fits out_cap) the blocks at d_out and the
// per-segment table.  *out_len = the total on LC_OK and on LC_ERR_CAPACITY.  d_out == nullptr: the engine's z_out.
int lz4_finish(lc_engine_t* e, const char* what, const lck::Lz4Segs& g, uint8_t* d_out, uint64_t out_cap,
               uint64_t* d_blk_off, uint32_t* d_blk_len, uint64_t* out_len) {
    LcLz4Chunk* d_info = e->z_info.as<LcLz4Chunk>();
    uint32_t* d_csize = e->z_size.as<uint32_t>();
    uint32_t* d_anchor = d_csize + g.nchunks;
    lck::launch_lz4_sizes(g, d_info, d_csize, d_anchor, e->stream);
    uint64_t* desc;
    int rc = prep_desc(e, lck::scan_tiles(g.nchunks), &desc);
    if (rc)
        return rc;
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    lck::launch_exclusive_sum(d_csize, g.nchunks, e->z_choff.as<uint64_t>(), &ds->total, desc, &ds->tickets[2],
                              e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    *out_len = hs->total;
    if (hs->total > out_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": output capacity too small");
    if (!d_out) {
        CU_TRY(e->z_out.ensure(hs->total));
        d_out = e->z_out.as<uint8_t>();
    }
    lck::launch_lz4_emit(g, e->z_seq.as<LcLz4Seq>(), d_info, d_anchor, e->z_choff.as<uint64_t>(), &ds->total, d_out,
                         d_blk_off, d_blk_len, e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

// One block of d_src[0, raw) (the fused calls' records ‖ tail) in z_out; only the block comes back to out.
int lz4_one_block(lc_engine_t* e, const char* what, const uint8_t* d_src, uint64_t raw, uint8_t* out, uint64_t out_cap,
                  uint64_t* out_len) {
    CU_TRY(e->z_tab.ensure(24));
    uint64_t* d_soff = e->z_tab.as<uint64_t>();
    uint64_t* d_boff = d_soff + 1;
    uint32_t* d_slen = reinterpret_cast<uint32_t*>(d_boff + 1);
    uint32_t* d_blen = d_slen + 1;
    const uint64_t zero = 0;
    const uint32_t len32 = (uint32_t)raw;
    CU_TRY(cudaMemcpyAsync(d_soff, &zero, 8, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(d_slen, &len32, 4, cudaMemcpyHostToDevice, e->stream));
    lck::Lz4Segs g{d_src, d_soff, d_slen, nullptr, 1, 0};
    int rc = lz4_chunk_tables(e, what, g, &zero, lc_lz4_nchunks(len32));
    if (rc)
        return rc;
    lck::launch_lz4_parse(g, 0, g.nchunks, e->z_seq.as<LcLz4Seq>(), e->z_info.as<LcLz4Chunk>(), e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    rc = lz4_finish(e, what, g, nullptr, out_cap, d_boff, d_blen, out_len);
    if (rc)
        return rc;
    if (!out)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    CU_TRY(cudaMemcpyAsync(out, e->z_out.p, *out_len, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// The parse pass over device segments (lc_lz4_compress_dev, lc_zstd_compress_dev; g.in, g.seg_off, g.seg_len and
// g.nseg >= 1 set): the chunk tables, then every chunk's matches.
int parse_dev(lc_engine_t* e, const char* what, lck::Lz4Segs& g) {
    if (g.nseg >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^32 segments per call");
    int rc = bind(e);
    if (rc)
        return rc;
    rc = lz4_chunk_tables(e, what, g, nullptr, 0);
    if (rc)
        return rc;
    lck::launch_lz4_parse(g, 0, g.nchunks, e->z_seq.as<LcLz4Seq>(), e->z_info.as<LcLz4Chunk>(), e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int drain_copies(lc_engine_t* e, int code) {
    cudaStreamSynchronize(e->s_h2d);
    cudaStreamSynchronize(e->stream);
    return code;
}

// The parse pass over nseg >= 1 HOST segments (lc_lz4_compress, lc_zstd_compress): they are packed at 16-byte aligned
// offsets of the engine's input buffer (g), going up in groups of whole segments on the copy stream while each landed
// group's chunks are parsed.  *d_off / *d_len: room for the per-segment output table.  A failure after the first
// upload returns through drain_copies().
int parse_host(lc_engine_t* e, const char* what, uint64_t nseg, const uint8_t* const* seg_ptr, const uint32_t* seg_len,
               lck::Lz4Segs& g, uint64_t** d_off, uint32_t** d_len) {
    if (nseg >= (1ull << 32))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^32 segments per call");
    // the chunk table is built here
    std::vector<uint64_t> soff(nseg), first(nseg);
    uint64_t total_in = 0, nchunks = 0;
    for (uint64_t k = 0; k < nseg; ++k) {
        if (seg_len[k] && !seg_ptr[k])
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
        if (seg_len[k] > LC_LZ4_MAX_INPUT)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": a segment is larger than LZ4_MAX_INPUT_SIZE");
        soff[k] = total_in;
        total_in += (seg_len[k] + 15ull) & ~15ull;
        first[k] = nchunks;
        nchunks += lc_lz4_nchunks(seg_len[k]);
    }
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(total_in + 16));
    CU_TRY(e->z_tab.ensure(nseg * 24));
    uint64_t* d_soff = e->z_tab.as<uint64_t>();
    *d_off = d_soff + nseg;
    uint32_t* d_slen = reinterpret_cast<uint32_t*>(*d_off + nseg);
    *d_len = d_slen + nseg;
    CU_TRY(cudaMemcpyAsync(d_soff, soff.data(), nseg * 8, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(d_slen, seg_len, nseg * 4, cudaMemcpyHostToDevice, e->stream));
    g = lck::Lz4Segs{e->in.as<uint8_t>(), d_soff, d_slen, nullptr, nseg, 0};
    rc = lz4_chunk_tables(e, what, g, first.data(), nchunks);
    if (rc)
        return rc;
    const uint64_t kGroupBytes = 32ull << 20;
    uint64_t ngroups = (total_in + kGroupBytes - 1) / kGroupBytes;
    ngroups = ngroups < 1 ? 1 : ngroups > 64 ? 64 : ngroups;
    if (ngroups > nseg)
        ngroups = nseg;
    rc = ensure_copy_streams(e, (int)ngroups);
    if (rc)
        return rc;
    if (cudaEventRecord(e->ev_comp[0], e->stream) != cudaSuccess ||
        cudaStreamWaitEvent(e->s_h2d, e->ev_comp[0], 0) != cudaSuccess)
        return drain_copies(e, fail(LC_ERR_CUDA, "stream ordering failed"));
    uint8_t* d_in = e->in.as<uint8_t>();
    uint64_t s0 = 0;
    for (uint64_t c = 0; c < ngroups; ++c) {
        uint64_t s1 = s0;
        const uint64_t goal = total_in * (c + 1) / ngroups;
        while (s1 < nseg && (s1 == s0 || soff[s1] < goal || c + 1 == ngroups))
            ++s1;
        for (uint64_t k = s0; k < s1; ++k)
            if (seg_len[k] && cudaMemcpyAsync(d_in + soff[k], seg_ptr[k], seg_len[k], cudaMemcpyHostToDevice,
                                              e->s_h2d) != cudaSuccess)
                return drain_copies(e, fail(LC_ERR_CUDA, std::string(what) + ": upload failed"));
        if (cudaEventRecord(e->ev_h2d[c], e->s_h2d) != cudaSuccess ||
            cudaStreamWaitEvent(e->stream, e->ev_h2d[c], 0) != cudaSuccess)
            return drain_copies(e, fail(LC_ERR_CUDA, "stream ordering failed"));
        const uint64_t k1 = s1 < nseg ? first[s1] : nchunks;
        lck::launch_lz4_parse(g, s0 < nseg ? first[s0] : nchunks, k1, e->z_seq.as<LcLz4Seq>(),
                              e->z_info.as<LcLz4Chunk>(), e->stream);
        e->launches++;
        s0 = s1;
    }
    if (cudaGetLastError() != cudaSuccess)
        return drain_copies(e, fail(LC_ERR_CUDA, std::string(what) + ": parse launch failed"));
    return LC_OK;
}

// The host calls' ending: the output (in z_out) and the per-segment table back to the host.
int copy_back(lc_engine_t* e, const char* what, uint64_t nseg, uint8_t* out, uint64_t* off, uint32_t* len,
              const uint64_t* d_off, const uint32_t* d_len, uint64_t out_len) {
    if (out_len && !out)
        return drain_copies(e, fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments"));
    CU_TRY(cudaMemcpyAsync(out, e->z_out.p, out_len, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(off, d_off, nseg * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(len, d_len, nseg * 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// After the parse pass: the zstd block table (bfirst_host / nblocks from the host, or counted here), every block's
// body in its slot, the frame offsets, and (when the total fits out_cap) the frames at d_out and the per-segment
// table.  *out_len = the total on LC_OK and on LC_ERR_CAPACITY.  d_out == nullptr: the engine's z_out.
int zstd_finish(lc_engine_t* e, const char* what, const lck::Lz4Segs& g, const uint64_t* bfirst_host, uint64_t nblocks,
                uint8_t* d_out, uint64_t out_cap, uint64_t* d_frm_off, uint32_t* d_frm_len, uint64_t* out_len) {
    Small* ds = e->small.as<Small>();
    Small* hs = (Small*)e->h_small;
    CU_TRY(e->zs_first.ensure(g.nseg * 8 + 8));
    uint64_t* d_bfirst = e->zs_first.as<uint64_t>();
    uint64_t* desc;
    int rc;
    if (bfirst_host) {
        CU_TRY(cudaMemcpyAsync(d_bfirst, bfirst_host, g.nseg * 8, cudaMemcpyHostToDevice, e->stream));
    } else {
        CU_TRY(e->zs_size.ensure(g.nseg * 4 + 4));
        rc = prep_desc(e, lck::scan_tiles(g.nseg), &desc);
        if (rc)
            return rc;
        lck::launch_zstd_nblocks(g.seg_len, g.nseg, e->zs_size.as<uint32_t>(), e->stream);
        lck::launch_exclusive_sum(e->zs_size.as<uint32_t>(), g.nseg, d_bfirst, &ds->total, desc, &ds->tickets[2],
                                  e->stream);
        e->launches += 2;
        CU_TRY(cudaGetLastError());
        CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        nblocks = hs->total;
    }
    CU_TRY(e->zs_size.ensure(nblocks * 8));
    CU_TRY(e->zs_off.ensure(nblocks * 8 + 8));
    CU_TRY(e->zs_slot.ensure(nblocks * LC_ZSTD_BLOCK));
    uint32_t* d_body = e->zs_size.as<uint32_t>();
    uint32_t* d_esz = d_body + nblocks;
    lck::launch_zstd_blocks(g, d_bfirst, nblocks, e->z_seq.as<LcLz4Seq>(), e->z_info.as<LcLz4Chunk>(),
                            e->zs_slot.as<uint8_t>(), d_body, d_esz, e->stream);
    rc = prep_desc(e, lck::scan_tiles(nblocks), &desc);
    if (rc)
        return rc;
    lck::launch_exclusive_sum(d_esz, nblocks, e->zs_off.as<uint64_t>(), &ds->total, desc, &ds->tickets[2], e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(&hs->total, &ds->total, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    *out_len = hs->total;
    if (hs->total > out_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": output capacity too small");
    if (!d_out) {
        CU_TRY(e->z_out.ensure(hs->total));
        d_out = e->z_out.as<uint8_t>();
    }
    lck::launch_zstd_emit(g, d_bfirst, nblocks, e->zs_slot.as<uint8_t>(), d_body, e->zs_off.as<uint64_t>(), &ds->total,
                          d_out, d_frm_off, d_frm_len, e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

} // namespace

extern "C" {

int lc_lz4_compress_dev(lc_engine_t* e, const uint8_t* d_in, uint64_t nseg, const uint64_t* d_seg_off,
                        const uint32_t* d_seg_len, uint8_t* d_out, uint64_t out_cap, uint64_t* d_blk_off,
                        uint32_t* d_blk_len, uint64_t* out_len) {
    static const char* what = "lc_lz4_compress_dev";
    if (!e || !out_len || (nseg && (!d_in || !d_seg_off || !d_seg_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (nseg == 0)
        return LC_OK;
    lck::Lz4Segs g{d_in, d_seg_off, d_seg_len, nullptr, nseg, 0};
    int rc = parse_dev(e, what, g);
    if (rc)
        return rc;
    // without an output (a sizing query) every total is over capacity: blocks are at least one byte
    rc = lz4_finish(e, what, g, d_out, d_out && d_blk_off && d_blk_len ? out_cap : 0, d_blk_off, d_blk_len, out_len);
    if (rc)
        return rc;
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

int lc_lz4_compress(lc_engine_t* e, uint64_t nseg, const uint8_t* const* seg_ptr, const uint32_t* seg_len,
                    uint8_t* out, uint64_t out_cap, uint64_t* blk_off, uint32_t* blk_len, uint64_t* out_len) {
    static const char* what = "lc_lz4_compress";
    if (!e || !out_len || (nseg && (!seg_ptr || !seg_len || !blk_off || !blk_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (nseg == 0)
        return LC_OK;
    lck::Lz4Segs g;
    uint64_t* d_boff;
    uint32_t* d_blen;
    int rc = parse_host(e, what, nseg, seg_ptr, seg_len, g, &d_boff, &d_blen);
    if (rc)
        return rc;
    rc = lz4_finish(e, what, g, nullptr, out_cap, d_boff, d_blen, out_len);
    return rc ? drain_copies(e, rc) : copy_back(e, what, nseg, out, blk_off, blk_len, d_boff, d_blen, *out_len);
}

int lc_zstd_compress_dev(lc_engine_t* e, const uint8_t* d_in, uint64_t nseg, const uint64_t* d_seg_off,
                         const uint32_t* d_seg_len, uint8_t* d_out, uint64_t out_cap, uint64_t* d_frm_off,
                         uint32_t* d_frm_len, uint64_t* out_len) {
    static const char* what = "lc_zstd_compress_dev";
    if (!e || !out_len || (nseg && (!d_in || !d_seg_off || !d_seg_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (nseg == 0)
        return LC_OK;
    lck::Lz4Segs g{d_in, d_seg_off, d_seg_len, nullptr, nseg, 0};
    int rc = parse_dev(e, what, g);
    if (rc)
        return rc;
    // without an output (a sizing query) every total is over capacity: frames are at least 9 bytes
    rc = zstd_finish(e, what, g, nullptr, 0, d_out, d_out && d_frm_off && d_frm_len ? out_cap : 0, d_frm_off,
                     d_frm_len, out_len);
    if (rc)
        return rc;
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

int lc_zstd_compress(lc_engine_t* e, uint64_t nseg, const uint8_t* const* seg_ptr, const uint32_t* seg_len,
                     uint8_t* out, uint64_t out_cap, uint64_t* frm_off, uint32_t* frm_len, uint64_t* out_len) {
    static const char* what = "lc_zstd_compress";
    if (!e || !out_len || (nseg && (!seg_ptr || !seg_len || !frm_off || !frm_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (nseg == 0)
        return LC_OK;
    lck::Lz4Segs g;
    uint64_t* d_foff;
    uint32_t* d_flen;
    int rc = parse_host(e, what, nseg, seg_ptr, seg_len, g, &d_foff, &d_flen);
    if (rc)
        return rc;
    std::vector<uint64_t> bfirst(nseg);
    uint64_t nblocks = 0;
    for (uint64_t k = 0; k < nseg; ++k) {
        bfirst[k] = nblocks;
        nblocks += lc_zstd_nblocks(seg_len[k]);
    }
    rc = zstd_finish(e, what, g, bfirst.data(), nblocks, nullptr, out_cap, d_foff, d_flen, out_len);
    return rc ? drain_copies(e, rc) : copy_back(e, what, nseg, out, frm_off, frm_len, d_foff, d_flen, *out_len);
}

} // extern "C"

// ------------------------------------------------------------------------------------------------ timestamp parse
struct lc_timestamp {
    uint64_t id;
    LcTsConf conf;
};

int lc_timestamp_compile(const char* format, size_t len, int32_t source_year, int32_t tz_adjust,
                         lc_timestamp_t** out) {
    if (!out || (!format && len))
        return fail(LC_ERR_INVALID_ARG, "lc_timestamp_compile: bad arguments");
    *out = nullptr;
    lc_timestamp* t = new (std::nothrow) lc_timestamp;
    if (!t)
        return fail(LC_ERR_INVALID_ARG, "out of host memory");
    memset(&t->conf, 0, sizeof t->conf);
    const char* err = nullptr;
    if (lc_ts_compile(format ? format : "", len, t->conf, &err) != 0) {
        delete t;
        return fail(LC_ERR_INVALID_ARG, std::string("lc_timestamp_compile: ") + err);
    }
    t->conf.source_year = source_year;
    t->conf.adjust = tz_adjust;
    lc_ts_probe_zone(t->conf);
    t->id = g_regex_ids.fetch_add(1);
    *out = t;
    return LC_OK;
}

void lc_timestamp_free(lc_timestamp_t* t) { delete t; }

namespace {

// both passes over the value table `sp`; d_counters (u64[5], device) are written
int ts_run(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, const LcTsSpans& sp, uint64_t n,
           const uint32_t* d_grp, uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec,
           uint32_t* d_nsec, uint8_t* d_status, uint64_t* d_counters) {
    int rc = bind(e);
    if (rc)
        return rc;
    LcTsNow t;
    t.now = now;
    const time_t tn = (time_t)now;
    struct tm lt;
    memset(&lt, 0, sizeof lt);
    localtime_r(&tn, &lt);
    t.year = lt.tm_year;
    t.mon = lt.tm_mon;
    t.mday = lt.tm_mday;
    t.discard_interval = discard_interval;
    if (e->ts_conf_id != ts->id) {
        CU_TRY(e->ts_conf.ensure(sizeof(LcTsConf)));
        CU_TRY(cudaMemcpyAsync(e->ts_conf.p, &ts->conf, sizeof(LcTsConf), cudaMemcpyHostToDevice, e->stream));
        e->ts_conf_id = ts->id;
    }
    CU_TRY(cudaMemsetAsync(d_counters, 0, 5 * sizeof(uint64_t), e->stream));
    if (n) {
        CU_TRY(e->ts_full.ensure(n * sizeof(LcTsFull)));
        lck::launch_ts_full(e->ts_conf.as<LcTsConf>(), t, d_base, sp, n, e->ts_full.as<LcTsFull>(), e->stream);
        lck::launch_ts_resolve(e->ts_conf.as<LcTsConf>(), t, d_base, sp, e->ts_full.as<LcTsFull>(), d_grp, ngroups, d_sec,
                               d_nsec, d_status, reinterpret_cast<unsigned long long*>(d_counters), e->stream);
        e->launches += 2;
    }
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

} // namespace

int lc_timestamp_parse_dev(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, uint64_t base_len,
                           const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint32_t* d_grp,
                           uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec, uint32_t* d_nsec,
                           uint8_t* d_status, uint64_t* d_counters) {
    if (!e || !ts || !d_counters || (n && (!d_base || !d_ev_off || !d_ev_len || !d_grp || !ngroups || !d_sec ||
                                           !d_nsec || !d_status)))
        return fail(LC_ERR_INVALID_ARG, "lc_timestamp_parse_dev: bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, "lc_timestamp_parse_dev: buffer must be < 4 GiB and < 2^32 events per call");
    return ts_run(e, ts, d_base, LcTsSpans{d_ev_off, d_ev_len, nullptr, 1}, n, d_grp, ngroups, now,
                  discard_interval, d_sec, d_nsec, d_status, d_counters);
}

int lc_timestamp_parse_capture_dev(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* d_base, uint64_t base_len,
                                   const uint8_t* d_rx_status, const uint32_t* d_cap_off, const uint32_t* d_cap_len,
                                   uint32_t row_pitch, uint32_t k, uint64_t n, const uint32_t* d_grp,
                                   uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* d_sec,
                                   uint32_t* d_nsec, uint8_t* d_status, uint64_t* d_counters) {
    if (!e || !ts || !d_counters || k >= row_pitch ||
        (n && (!d_base || !d_rx_status || !d_cap_off || !d_cap_len || !d_grp || !ngroups || !d_sec || !d_nsec ||
               !d_status)))
        return fail(LC_ERR_INVALID_ARG, "lc_timestamp_parse_capture_dev: bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE,
                    "lc_timestamp_parse_capture_dev: buffer must be < 4 GiB and < 2^32 events per call");
    return ts_run(e, ts, d_base, LcTsSpans{d_cap_off + k, d_cap_len + k, d_rx_status, row_pitch}, n, d_grp, ngroups,
                  now, discard_interval, d_sec, d_nsec, d_status, d_counters);
}

int lc_timestamp_parse(lc_engine_t* e, const lc_timestamp_t* ts, const uint8_t* base, uint64_t base_len,
                       const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* grp,
                       uint64_t ngroups, int64_t now, int32_t discard_interval, int64_t* sec, uint32_t* nsec,
                       uint8_t* status, uint64_t* counters) {
    static const char* what = "lc_timestamp_parse";
    if (!e || !ts || !counters || (n && (!base || !ev_off || !ev_len || !grp || !ngroups || !sec || !nsec || !status)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= 0xFFFFFFFFull || ngroups >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": buffer must be < 4 GiB and < 2^32 events per call");
    memset(counters, 0, 5 * sizeof(uint64_t));
    if (n == 0)
        return LC_OK;
    if (grp[0] != 0 || grp[ngroups] != n)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": groups must cover the events");
    for (uint64_t g = 0; g < ngroups; ++g)
        if (grp[g + 1] < grp[g])
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": group starts must not decrease");
    for (uint64_t i = 0; i < n; ++i)
        if (ev_len[i] != LC_TS_NO_KEY && (uint64_t)ev_off[i] + ev_len[i] > base_len)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event outside the buffer");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->lines_off.ensure((ngroups + 1) * 4));
    CU_TRY(e->out_a.ensure(n * 8));
    CU_TRY(e->out_b.ensure(n * 4));
    CU_TRY(e->out_c.ensure(n));
    CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
    CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->lines_off.p, grp, (ngroups + 1) * 4, cudaMemcpyHostToDevice, e->stream));
    rc = ts_run(e, ts, e->in.as<uint8_t>(), LcTsSpans{e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), nullptr, 1},
                n, e->lines_off.as<uint32_t>(), ngroups, now, discard_interval, e->out_a.as<int64_t>(),
                e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), e->ts_cnt.as<uint64_t>());
    if (rc)
        return rc;
    CU_TRY(cudaMemcpyAsync(sec, e->out_a.p, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(nsec, e->out_b.p, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(status, e->out_c.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(counters, e->ts_cnt.p, 5 * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return LC_OK;
}

// ------------------------------------------------------------------------------------------------ Apsara parse
struct lc_apsara {
    uint64_t id;
    LcTsConf conf; // adjust and the zone table; the format program is not used
    std::string skey;
};

int lc_apsara_compile(const char* source_key, size_t key_len, int32_t tz_adjust, lc_apsara_t** out) {
    if (!out || (!source_key && key_len) || key_len >= 0xFFFFFFFFull)
        return fail(LC_ERR_INVALID_ARG, "lc_apsara_compile: bad arguments");
    *out = nullptr;
    lc_apsara* a = new (std::nothrow) lc_apsara;
    if (!a)
        return fail(LC_ERR_INVALID_ARG, "out of host memory");
    memset(&a->conf, 0, sizeof a->conf);
    a->conf.adjust = tz_adjust;
    lc_ts_probe_zone(a->conf);
    a->skey.assign(source_key ? source_key : "", key_len);
    a->id = g_regex_ids.fetch_add(1);
    *out = a;
    return LC_OK;
}

void lc_apsara_free(lc_apsara_t* a) { delete a; }

static_assert(sizeof(lc_apsara_entry_t) == sizeof(LcApEntry), "entry layout");

namespace {

// The scan, resolve and count passes (on the caller's device tables) up to the entry total, which *n_entries receives
// after a wait for the device.  An event past base_len gives LC_ERR_INVALID_ARG.
int ap_count(lc_engine_t* e, const lc_apsara_t* ap, const char* what, const uint8_t* d_base, uint64_t base_len,
             const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint32_t* d_grp, uint64_t ngroups,
             int64_t now, int32_t discard_interval, uint8_t* d_status, int64_t* d_sec, uint32_t* d_nsec,
             int64_t* d_micro, uint64_t* d_first, uint64_t* n_entries, uint64_t* d_counters) {
    int rc = bind(e);
    if (rc)
        return rc;
    *n_entries = 0;
    CU_TRY(cudaMemsetAsync(d_counters, 0, 5 * sizeof(uint64_t), e->stream));
    if (n == 0) {
        CU_TRY(cudaMemsetAsync(d_first, 0, 8, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        return LC_OK;
    }
    LcTsNow t;
    memset(&t, 0, sizeof t);
    t.now = now;
    t.discard_interval = discard_interval;
    if (e->ap_conf_id != ap->id) {
        CU_TRY(e->ap_conf.ensure(sizeof(LcTsConf) + ap->skey.size() + 1));
        CU_TRY(cudaMemcpyAsync(e->ap_conf.p, &ap->conf, sizeof(LcTsConf), cudaMemcpyHostToDevice, e->stream));
        if (!ap->skey.empty())
            CU_TRY(cudaMemcpyAsync(e->ap_conf.as<uint8_t>() + sizeof(LcTsConf), ap->skey.data(), ap->skey.size(),
                                   cudaMemcpyHostToDevice, e->stream));
        e->ap_conf_id = ap->id;
    }
    CU_TRY(e->ap_ev.ensure(n * sizeof(LcApEv)));
    CU_TRY(e->ap_nent.ensure(n * 4));
    CU_TRY(e->ap_small.ensure(16));
    CU_TRY(cudaMemsetAsync(e->ap_small.p, 0, 16, e->stream));
    uint32_t* d_bad = e->ap_small.as<uint32_t>();
    const LcTsConf* d_conf = e->ap_conf.as<LcTsConf>();
    lck::launch_ap_scan(d_conf, d_base, base_len, d_ev_off, d_ev_len, n, e->ap_conf.as<uint8_t>() + sizeof(LcTsConf),
                        (uint32_t)ap->skey.size(), e->ap_ev.as<LcApEv>(), d_bad, e->stream);
    lck::launch_ap_resolve(t, e->ap_ev.as<LcApEv>(), d_grp, ngroups, d_status, d_sec, d_nsec, d_micro,
                           e->ap_nent.as<uint32_t>(), reinterpret_cast<unsigned long long*>(d_counters), e->stream);
    uint64_t* desc;
    rc = prep_desc(e, lck::scan_tiles(n), &desc);
    if (rc)
        return rc;
    lck::launch_exclusive_sum(e->ap_nent.as<uint32_t>(), n, d_first, d_first + n, desc, &e->small.as<Small>()->tickets[2],
                              e->stream);
    e->launches += 3;
    CU_TRY(cudaGetLastError());
    uint32_t bad = 0;
    CU_TRY(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(n_entries, d_first + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (bad) {
        *n_entries = 0;
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event outside the buffer");
    }
    return LC_OK;
}

// The emit pass of ap_count's events into d_entries (room for the total); queued, not waited for.
int ap_emit(lc_engine_t* e, const uint8_t* d_base, const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n,
            const uint8_t* d_status, const uint64_t* d_first, lc_apsara_entry_t* d_entries) {
    lck::launch_ap_emit(d_base, d_ev_off, d_ev_len, d_status, n, d_first, reinterpret_cast<LcApEntry*>(d_entries),
                        e->stream);
    e->launches += 1;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

} // namespace

int lc_apsara_parse_dev(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* d_base, uint64_t base_len,
                        const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, const uint32_t* d_grp,
                        uint64_t ngroups, int64_t now, int32_t discard_interval, uint8_t* d_status, int64_t* d_sec,
                        uint32_t* d_nsec, int64_t* d_micro, uint64_t* d_first, lc_apsara_entry_t* d_entries,
                        uint64_t entry_cap, uint64_t* n_entries, uint64_t* d_counters) {
    static const char* what = "lc_apsara_parse_dev";
    if (!e || !ap || !d_counters || !n_entries || !d_first || (entry_cap && !d_entries) ||
        (n && (!d_base || !d_ev_off || !d_ev_len || !d_grp || !ngroups || !d_status || !d_sec || !d_nsec ||
               !d_micro)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= 0xFFFFFFFFull || ngroups >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": buffer must be < 4 GiB and < 2^32 events per call");
    int rc = ap_count(e, ap, what, d_base, base_len, d_ev_off, d_ev_len, n, d_grp, ngroups, now, discard_interval,
                      d_status, d_sec, d_nsec, d_micro, d_first, n_entries, d_counters);
    if (rc)
        return rc;
    if (*n_entries > entry_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": entry capacity too small");
    if (*n_entries) {
        rc = ap_emit(e, d_base, d_ev_off, d_ev_len, n, d_status, d_first, d_entries);
        if (rc)
            return rc;
        CU_TRY(cudaStreamSynchronize(e->stream));
    }
    return LC_OK;
}

int lc_apsara_parse(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* base, uint64_t base_len,
                    const uint32_t* ev_off, const uint32_t* ev_len, uint64_t n, const uint32_t* grp, uint64_t ngroups,
                    int64_t now, int32_t discard_interval, uint8_t* status, int64_t* sec, uint32_t* nsec,
                    int64_t* micro, uint64_t* first, lc_apsara_entry_t* entries, uint64_t entry_cap,
                    uint64_t* n_entries, uint64_t* counters) {
    static const char* what = "lc_apsara_parse";
    if (!e || !ap || !counters || !n_entries || !first || (entry_cap && !entries) ||
        (n && (!base || !ev_off || !ev_len || !grp || !ngroups || !status || !sec || !nsec || !micro)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (base_len >= 0xFFFFFFF0ull || n >= 0xFFFFFFFFull || ngroups >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": buffer must be < 4 GiB and < 2^32 events per call");
    memset(counters, 0, 5 * sizeof(uint64_t));
    *n_entries = 0;
    first[0] = 0;
    if (n == 0)
        return LC_OK;
    if (grp[0] != 0 || grp[ngroups] != n)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": groups must cover the events");
    for (uint64_t g = 0; g < ngroups; ++g)
        if (grp[g + 1] < grp[g])
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": group starts must not decrease");
    for (uint64_t i = 0; i < n; ++i)
        if (ev_len[i] != LC_AP_NO_KEY && (uint64_t)ev_off[i] + ev_len[i] > base_len)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event outside the buffer");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->lines_off.ensure((ngroups + 1) * 4));
    CU_TRY(e->ap_status.ensure(n));
    CU_TRY(e->ap_sec.ensure(n * 8));
    CU_TRY(e->ap_nsec.ensure(n * 4));
    CU_TRY(e->ap_micro.ensure(n * 8));
    CU_TRY(e->ap_first.ensure((n + 1) * 8));
    CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
    if (base_len)
        CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->lines_off.p, grp, (ngroups + 1) * 4, cudaMemcpyHostToDevice, e->stream));
    rc = ap_count(e, ap, what, e->in.as<uint8_t>(), base_len, e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                  e->lines_off.as<uint32_t>(), ngroups, now, discard_interval, e->ap_status.as<uint8_t>(),
                  e->ap_sec.as<int64_t>(), e->ap_nsec.as<uint32_t>(), e->ap_micro.as<int64_t>(),
                  e->ap_first.as<uint64_t>(), n_entries, e->ts_cnt.as<uint64_t>());
    if (rc)
        return rc;
    const uint64_t m = *n_entries;
    if (m > entry_cap) {
        rc = fail(LC_ERR_CAPACITY, std::string(what) + ": entry capacity too small");
    } else if (m) {
        // the device entries are sized from the count, not from entry_cap
        CU_TRY(e->ap_ent.ensure(m * sizeof(LcApEntry)));
        rc = ap_emit(e, e->in.as<uint8_t>(), e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                     e->ap_status.as<uint8_t>(), e->ap_first.as<uint64_t>(), e->ap_ent.as<lc_apsara_entry_t>());
        if (rc)
            return rc;
        CU_TRY(cudaMemcpyAsync(entries, e->ap_ent.p, m * sizeof(LcApEntry), cudaMemcpyDeviceToHost, e->stream));
    }
    CU_TRY(cudaMemcpyAsync(status, e->ap_status.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(sec, e->ap_sec.p, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(nsec, e->ap_nsec.p, n * 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(micro, e->ap_micro.p, n * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(first, e->ap_first.p, (n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(counters, e->ts_cnt.p, 5 * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return rc;
}

// ------------------------------------------------------------------------------------------------ JSON parse
struct lc_json {
    uint64_t id;
    std::string skey;
};

int lc_json_compile(const char* source_key, size_t key_len, lc_json_t** out) {
    if (!out || (!source_key && key_len) || key_len >= 0xFFFFFFFFull)
        return fail(LC_ERR_INVALID_ARG, "lc_json_compile: bad arguments");
    *out = nullptr;
    lc_json* j = new (std::nothrow) lc_json;
    if (!j)
        return fail(LC_ERR_INVALID_ARG, "out of host memory");
    j->skey.assign(source_key ? source_key : "", key_len);
    j->id = g_regex_ids.fetch_add(1);
    *out = j;
    return LC_OK;
}

void lc_json_free(lc_json_t* j) { delete j; }

static_assert(sizeof(lc_json_entry_t) == sizeof(LcJsonEntry), "entry layout");

namespace {

// The count passes (fast, then slow over the events the fast walk gave up on) and both exclusive sums, on the caller's
// device tables, up to the totals, which the host receives after a wait for the device.
int js_count(lc_engine_t* e, const lc_json_t* js, const char* what, const uint8_t* d_base, uint64_t base_len,
             const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint8_t* d_status, uint64_t* d_first,
             uint64_t* n_entries, uint64_t* arena_bytes, uint64_t* d_counters) {
    int rc = bind(e);
    if (rc)
        return rc;
    *n_entries = *arena_bytes = 0;
    CU_TRY(cudaMemsetAsync(d_counters, 0, 3 * sizeof(uint64_t), e->stream));
    if (n == 0) {
        CU_TRY(cudaMemsetAsync(d_first, 0, 8, e->stream));
        CU_TRY(cudaStreamSynchronize(e->stream));
        return LC_OK;
    }
    if (!e->js_pow5.p) { // the Eisel-Lemire table, uploaded once per engine
        CU_TRY(e->js_pow5.ensure(sizeof lc_json_pow5));
        CU_TRY(cudaMemcpyAsync(e->js_pow5.p, lc_json_pow5, sizeof lc_json_pow5, cudaMemcpyHostToDevice, e->stream));
    }
    if (e->js_conf_id != js->id) {
        CU_TRY(e->js_conf.ensure(js->skey.size() + 1));
        if (!js->skey.empty())
            CU_TRY(cudaMemcpyAsync(e->js_conf.p, js->skey.data(), js->skey.size(), cudaMemcpyHostToDevice, e->stream));
        e->js_conf_id = js->id;
    }
    CU_TRY(e->js_nent.ensure(n * 4));
    CU_TRY(e->js_narena.ensure(n * 4));
    CU_TRY(e->js_slow.ensure(n));
    CU_TRY(e->js_list.ensure(n * 4));
    CU_TRY(e->js_afirst.ensure((n + 1) * 8));
    CU_TRY(e->js_small.ensure(16));
    CU_TRY(cudaMemsetAsync(e->js_small.p, 0, 16, e->stream));
    uint32_t* d_bad = e->js_small.as<uint32_t>();
    uint32_t* d_nslow = d_bad + 1;
    const uint8_t* d_skey = e->js_conf.as<uint8_t>();
    const uint32_t sklen = (uint32_t)js->skey.size();
    auto* cnt = reinterpret_cast<unsigned long long*>(d_counters);
    const uint64_t* d_pow5 = e->js_pow5.as<uint64_t>();
    lck::launch_json_count(d_base, base_len, d_ev_off, d_ev_len, n, d_skey, sklen, d_pow5, d_status, e->js_nent.as<uint32_t>(),
                           e->js_narena.as<uint32_t>(), e->js_slow.as<uint8_t>(), e->js_list.as<uint32_t>(), d_nslow,
                           d_bad, cnt, e->stream);
    lck::launch_json_count_slow(d_base, d_ev_off, d_ev_len, d_skey, sklen, d_pow5, e->js_list.as<uint32_t>(), d_nslow,
                                d_status, e->js_nent.as<uint32_t>(), e->js_narena.as<uint32_t>(), cnt, e->stream);
    const size_t tiles = lck::scan_tiles(n);
    uint64_t* desc;
    rc = prep_desc(e, 2 * tiles + 1, &desc);
    if (rc)
        return rc;
    lck::launch_exclusive_sum(e->js_nent.as<uint32_t>(), n, d_first, d_first + n, desc, &e->small.as<Small>()->tickets[2],
                              e->stream);
    lck::launch_exclusive_sum(e->js_narena.as<uint32_t>(), n, e->js_afirst.as<uint64_t>(),
                              e->js_afirst.as<uint64_t>() + n, desc + tiles + 1, &e->small.as<Small>()->tickets[3],
                              e->stream);
    e->launches += 4;
    CU_TRY(cudaGetLastError());
    uint32_t bad = 0;
    CU_TRY(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(n_entries, d_first + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(arena_bytes, e->js_afirst.as<uint64_t>() + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (bad) {
        *n_entries = *arena_bytes = 0;
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event outside the buffer");
    }
    if (*arena_bytes >= LC_JSON_ARENA)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the arena would reach 2 GiB");
    return LC_OK;
}

// The emit passes of js_count's events into d_entries / d_arena (room for both totals), waited for; LC_ERR_INTERNAL
// when an event would have left its ranges.
int js_emit(lc_engine_t* e, const lc_json_t* js, const char* what, const uint8_t* d_base, const uint32_t* d_ev_off,
            const uint32_t* d_ev_len, uint64_t n, const uint8_t* d_status, const uint64_t* d_first,
            lc_json_entry_t* d_entries, uint8_t* d_arena) {
    uint32_t* d_bad = e->js_small.as<uint32_t>();
    const uint8_t* d_skey = e->js_conf.as<uint8_t>();
    const uint32_t sklen = (uint32_t)js->skey.size();
    auto* ent = reinterpret_cast<LcJsonEntry*>(d_entries);
    const uint64_t* d_pow5 = e->js_pow5.as<uint64_t>();
    lck::launch_json_emit(d_base, d_ev_off, d_ev_len, n, d_skey, sklen, d_pow5, d_status, e->js_slow.as<uint8_t>(), d_first,
                          e->js_afirst.as<uint64_t>(), ent, d_arena, d_bad, e->stream);
    lck::launch_json_emit_slow(d_base, d_ev_off, d_ev_len, d_skey, sklen, d_pow5, d_status, e->js_list.as<uint32_t>(),
                               d_bad + 1, d_first, e->js_afirst.as<uint64_t>(), ent, d_arena, d_bad, e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    uint32_t bad = 0;
    CU_TRY(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (bad)
        return fail(LC_ERR_INTERNAL, std::string(what) + ": an emit pass would have left its event's output range");
    return LC_OK;
}

} // namespace

int lc_json_parse_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_base, uint64_t base_len,
                      const uint32_t* d_ev_off, const uint32_t* d_ev_len, uint64_t n, uint8_t* d_status,
                      uint64_t* d_first, lc_json_entry_t* d_entries, uint64_t entry_cap, uint64_t* n_entries,
                      uint8_t* d_arena, uint64_t arena_cap, uint64_t* arena_bytes, uint64_t* d_counters) {
    static const char* what = "lc_json_parse_dev";
    if (!e || !js || !d_counters || !n_entries || !arena_bytes || !d_first || (entry_cap && !d_entries) ||
        (arena_cap && !d_arena) || (n && (!d_base || !d_ev_off || !d_ev_len || !d_status)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (base_len >= LC_JSON_ARENA || n >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": buffer must be < 2 GiB and < 2^32 events per call");
    int rc = js_count(e, js, what, d_base, base_len, d_ev_off, d_ev_len, n, d_status, d_first, n_entries, arena_bytes,
                      d_counters);
    if (rc)
        return rc;
    if (*n_entries > entry_cap || *arena_bytes > arena_cap)
        return fail(LC_ERR_CAPACITY, std::string(what) + ": entry or arena capacity too small");
    if (*n_entries)
        return js_emit(e, js, what, d_base, d_ev_off, d_ev_len, n, d_status, d_first, d_entries, d_arena);
    return LC_OK;
}

int lc_json_parse(lc_engine_t* e, const lc_json_t* js, const uint8_t* base, uint64_t base_len, const uint32_t* ev_off,
                  const uint32_t* ev_len, uint64_t n, uint8_t* status, uint64_t* first, lc_json_entry_t* entries,
                  uint64_t entry_cap, uint64_t* n_entries, uint8_t* arena, uint64_t arena_cap, uint64_t* arena_bytes,
                  uint64_t* counters) {
    static const char* what = "lc_json_parse";
    if (!e || !js || !counters || !n_entries || !arena_bytes || !first || (entry_cap && !entries) ||
        (arena_cap && !arena) || (n && (!base || !ev_off || !ev_len || !status)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (base_len >= LC_JSON_ARENA || n >= 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": buffer must be < 2 GiB and < 2^32 events per call");
    memset(counters, 0, 3 * sizeof(uint64_t));
    *n_entries = *arena_bytes = 0;
    first[0] = 0;
    if (n == 0)
        return LC_OK;
    for (uint64_t i = 0; i < n; ++i)
        if (ev_len[i] != LC_JSON_NO_KEY && (uint64_t)ev_off[i] + ev_len[i] > base_len)
            return fail(LC_ERR_INVALID_ARG, std::string(what) + ": event outside the buffer");
    int rc = bind(e);
    if (rc)
        return rc;
    CU_TRY(e->in.ensure(base_len + 16));
    CU_TRY(e->ev_off.ensure(n * 4));
    CU_TRY(e->ev_len.ensure(n * 4));
    CU_TRY(e->js_status.ensure(n));
    CU_TRY(e->js_first.ensure((n + 1) * 8));
    CU_TRY(e->js_cnt.ensure(3 * sizeof(uint64_t)));
    if (base_len)
        CU_TRY(cudaMemcpyAsync(e->in.p, base, base_len, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_off.p, ev_off, n * 4, cudaMemcpyHostToDevice, e->stream));
    CU_TRY(cudaMemcpyAsync(e->ev_len.p, ev_len, n * 4, cudaMemcpyHostToDevice, e->stream));
    const uint8_t* d_base = e->in.as<uint8_t>();
    rc = js_count(e, js, what, d_base, base_len, e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                  e->js_status.as<uint8_t>(), e->js_first.as<uint64_t>(), n_entries, arena_bytes,
                  e->js_cnt.as<uint64_t>());
    if (rc)
        return rc;
    const uint64_t m = *n_entries, a = *arena_bytes;
    if (m > entry_cap || a > arena_cap) {
        rc = fail(LC_ERR_CAPACITY, std::string(what) + ": entry or arena capacity too small");
    } else if (m) {
        // the device copies are sized from the totals, not from the caps
        CU_TRY(e->js_ent.ensure(m * sizeof(LcJsonEntry)));
        CU_TRY(e->js_arena.ensure(a + 1));
        rc = js_emit(e, js, what, d_base, e->ev_off.as<uint32_t>(), e->ev_len.as<uint32_t>(), n,
                     e->js_status.as<uint8_t>(), e->js_first.as<uint64_t>(), e->js_ent.as<lc_json_entry_t>(),
                     e->js_arena.as<uint8_t>());
        if (rc)
            return rc;
        CU_TRY(cudaMemcpyAsync(entries, e->js_ent.p, m * sizeof(LcJsonEntry), cudaMemcpyDeviceToHost, e->stream));
        if (a)
            CU_TRY(cudaMemcpyAsync(arena, e->js_arena.p, a, cudaMemcpyDeviceToHost, e->stream));
    }
    CU_TRY(cudaMemcpyAsync(status, e->js_status.p, n, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(first, e->js_first.p, (n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaMemcpyAsync(counters, e->js_cnt.p, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    return rc;
}

// ------------------------------------------------------------------------------------------------ split -> JSON -> SLS
// The JSON stage's CommonParserOptions and the offset content of the split events (offset_key NULL = no
// log.file.offset metadata), with the source event's position, time and ns
#define SPLIT_JSON_PARAMS                                                                                              \
    const char *renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,                 \
        const char *offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns
#define SPLIT_JSON_ARGS                                                                                                \
    renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw, offset_key, offset_key_len, src_pos, time, time_ns

namespace {

// lc_split_json_sls_setup over js's SourceKey, with SourceKey, RenamedSourceKey, the offset key and "__raw_log__"
// staged on the device (`sls_plan`, which neither splitter nor the JSON stage uses) and *c pointing at them.  With ta
// (the timestamp calls), the timestamp stage's SourceKey is checked into *tc (lc_split_json_ts_setup) and staged
// behind them.
int split_json_sls_config(lc_engine_t* e, const char* what, const lc_json_t* js, SPLIT_JSON_PARAMS,
                          LcSplitJsonSlsCfg* c, const TsArgs* ta = nullptr, LcSplitJsonTsCfg* tc = nullptr) {
    if (!js || (renamed_key_len && !renamed_key) || (offset_key_len && !offset_key))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    const uint32_t oklen = offset_key ? offset_key_len : 0u, tklen = ta ? ta->tkey_len : 0u;
    if ((uint64_t)js->skey.size() + renamed_key_len + oklen + tklen + 16 > 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": keys must stay below 4 GiB");
    const char* why = lc_split_json_sls_setup(js->skey.data(), (uint32_t)js->skey.size(), renamed_key,
                                              renamed_key_len, offset_key, oklen, keep_fail, keep_succeed, copy_raw,
                                              src_pos, time, time_ns, c);
    if (!why && ta)
        why = lc_split_json_ts_setup(*c, ta->tkey, tklen, ta->enable_ns, tc);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    std::string keys = js->skey;
    keys.append(renamed_key ? renamed_key : "", renamed_key_len);
    keys.append(offset_key ? offset_key : "", oklen);
    keys.append("__raw_log__", 11);
    if (ta)
        keys.append(ta->tkey ? ta->tkey : "", tklen);
    CU_TRY(e->sls_plan.ensure(keys.size() + 1));
    if (!keys.empty())
        CU_TRY(cudaMemcpyAsync(e->sls_plan.p, keys.data(), keys.size(), cudaMemcpyHostToDevice, e->stream));
    const uint8_t* d = e->sls_plan.as<uint8_t>();
    c->skey = d;
    c->rkey = d + c->sklen;
    c->okey = d + c->sklen + c->rklen;
    c->raw = c->okey + c->oklen;
    if (ta)
        tc->tkey = c->raw + 11;
    return LC_OK;
}

// The split -> JSON -> timestamp chain's tap and timestamp passes over the n pieces of t (a: the arena's bytes): the
// value buffer `sjt_val` and the value table into st_val, then lc_timestamp_parse_dev's two passes with the whole
// source value as one group into *ts (st_status, st_sec, st_nsec).  The stage's counters are the size pass's, so the
// passes' own go to ts_cnt unread.
int split_json_ts_run(lc_engine_t* e, const LcSplitJsonSlsCfg& c, LcSplitJsonTsCfg tc, const TsArgs& ta,
                      const lck::SplitJsonSlsTables& t, uint64_t n, uint64_t src_len, uint64_t a,
                      lck::TsRowTables* ts) {
    CU_TRY(e->st_val.ensure(n * 8 + 8));
    CU_TRY(e->st_sec.ensure(n * 8));
    CU_TRY(e->st_nsec.ensure(n * 4));
    CU_TRY(e->st_status.ensure(n));
    CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
    CU_TRY(e->sjt_val.ensure(src_len + a + 16));
    tc.arena_at = src_len;
    tc.val_cap = src_len + a;
    uint32_t* off = e->st_val.as<uint32_t>();
    uint32_t *len = off + n, *grp = off + 2 * n;
    const uint32_t g[2] = {0u, (uint32_t)n};
    CU_TRY(cudaMemcpyAsync(grp, g, sizeof g, cudaMemcpyHostToDevice, e->stream));
    lck::launch_split_json_ts_tap(c, tc, t, n, e->sjt_val.as<uint8_t>(), off, len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    const int rc = ts_run(e, ta.ts, e->sjt_val.as<uint8_t>(), LcTsSpans{off, len, nullptr, 1}, n, grp, 1, ta.now,
                          ta.discard_interval, e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>(),
                          e->st_status.as<uint8_t>(), e->ts_cnt.as<uint64_t>());
    *ts = lck::TsRowTables{e->st_status.as<uint8_t>(), e->st_sec.as<int64_t>(), e->st_nsec.as<uint32_t>()};
    return rc;
}

// The resolve pass, the size pass and the emit of the chain over the n pieces of t (m entries in all; t.win and t.ev
// are set here): into d_out (the device-fed call), or back to the host buffer out, or -- with z -- records ‖ tail as
// one LZ4 block.  counters[3] = successful, failed, discarded; set whenever the size pass ran.  With tc (the timestamp
// calls), each record's time comes from the timestamp tables ts and counters has LC_SRTS_COUNTERS entries.
int split_json_sls_run(lc_engine_t* e, const char* what, const LcSplitJsonSlsCfg& c, lck::SplitJsonSlsTables t,
                       uint64_t n, uint64_t m, uint8_t* d_out, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                       uint64_t* counters, const Lz4Tail* z, const LcSplitJsonTsCfg* tc = nullptr,
                       const lck::TsRowTables* ts = nullptr) {
    CU_TRY(e->sj_win.ensure(m * 4 + 4));
    CU_TRY(e->sj_ev.ensure(n * sizeof(LcJsonSlsEv)));
    CU_TRY(e->sj_list.ensure(n * 4 + 4));
    CU_TRY(e->sj_sort.ensure(3 * m * 4 + 4));
    uint32_t* nlist = e->sj_list.as<uint32_t>();
    CU_TRY(cudaMemsetAsync(nlist, 0, 4, e->stream));
    t.win = e->sj_win.as<uint32_t>();
    t.ev = e->sj_ev.as<LcJsonSlsEv>();
    lck::launch_json_resolve(c, t, n, m, nlist + 1, nlist, e->sj_sort.as<uint32_t>(), e->stream);
    e->launches += 2;
    CU_TRY(cudaGetLastError());
    const uint32_t nstage = tc ? LC_SRTS_COUNTERS : 3u;
    uint64_t ctr[LC_SRTS_COUNTERS + 1] = {0}; // + pieces whose record would reach 4 GiB
    SlsTo to;
    to.host = out;
    to.z = z;
    to.too_large = (int)nstage;
    const int rc = serialize_sls_dev(
        e, what, n, nstage + 1,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* d_ctr) {
            if (tc)
                lck::launch_split_json_ts_sls_sizes(c, *tc, t, *ts, n, rec, body, d_ctr, e->stream);
            else
                lck::launch_split_json_sls_sizes(c, t, n, rec, body, d_ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* dst) {
            if (tc)
                lck::launch_split_json_ts_sls_emit(c, *tc, t, *ts, n, rec_off, body, dst, e->stream);
            else
                lck::launch_split_json_sls_emit(c, t, n, rec_off, body, dst, e->stream);
        },
        d_out, out_cap, out_len, ctr, to);
    if (counters)
        memcpy(counters, ctr, nstage * sizeof(uint64_t));
    return rc;
}

// Host-buffer split + JSON + serialise (lc_split_json_parse_sls and the multiline / LZ4 siblings): the JSON stage
// runs js_count / js_emit over the pieces into the js_* buffers of lc_json_parse, then split_json_sls_run.  With ta
// (the _timestamp_ calls), the tap and the timestamp passes run between them and counters has LC_SRTS_COUNTERS
// entries.
template <class Split>
int split_json_sls_host(lc_engine_t* e, const char* what, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                        Split split, SPLIT_JSON_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                        uint64_t* n_events, uint64_t* counters, const Lz4Tail* z, const TsArgs* ta = nullptr) {
    LcSplitJsonSlsCfg c;
    LcSplitJsonTsCfg tc;
    auto begin = [&]() {
        if (counters)
            memset(counters, 0, (ta ? LC_SRTS_COUNTERS : 3) * sizeof(uint64_t));
        if (len >= LC_JSON_ARENA)
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the source value must be < 2 GiB");
        return (int)LC_OK;
    };
    auto config = [&]() { return split_json_sls_config(e, what, js, SPLIT_JSON_ARGS, &c, ta, &tc); };
    auto run = [&](uint64_t n) {
        if (n >= (1ull << 30))
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^30 pieces per call");
        CU_TRY(e->js_status.ensure(n));
        CU_TRY(e->js_first.ensure((n + 1) * 8));
        CU_TRY(e->js_cnt.ensure(3 * sizeof(uint64_t)));
        const uint8_t* d_src = e->in.as<uint8_t>();
        const uint32_t *off = e->out_a.as<uint32_t>(), *ln = e->out_b.as<uint32_t>();
        uint64_t m = 0, a = 0;
        int rc = js_count(e, js, what, d_src, len, off, ln, n, e->js_status.as<uint8_t>(), e->js_first.as<uint64_t>(),
                          &m, &a, e->js_cnt.as<uint64_t>());
        if (rc)
            return rc;
        CU_TRY(e->js_ent.ensure(m * sizeof(LcJsonEntry) + 16));
        CU_TRY(e->js_arena.ensure(a + 16));
        if (m) {
            rc = js_emit(e, js, what, d_src, off, ln, n, e->js_status.as<uint8_t>(), e->js_first.as<uint64_t>(),
                         e->js_ent.as<lc_json_entry_t>(), e->js_arena.as<uint8_t>());
            if (rc)
                return rc;
        }
        const lck::SplitJsonSlsTables t{d_src, off, ln, e->js_status.as<uint8_t>(), e->js_first.as<uint64_t>(),
                                        e->js_ent.as<LcJsonEntry>(), e->js_arena.as<uint8_t>(), nullptr, nullptr};
        lck::TsRowTables ts{};
        if (ta) {
            rc = split_json_ts_run(e, c, tc, *ta, t, n, len, a, &ts);
            if (rc)
                return rc;
        }
        return split_json_sls_run(e, what, c, t, n, m, nullptr, out, out_cap, out_len, counters, z,
                                  ta ? &tc : nullptr, &ts);
    };
    return split_chain_sls_host(e, what, buf, len, split, js != nullptr && (!ta || ta->ts), begin, config, run, out,
                                out_cap, out_len, n_events, z);
}

template <class Split>
int split_json_lz4_host(lc_engine_t* e, const char* what, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                        Split split, SPLIT_JSON_PARAMS, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                        uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                        uint64_t* counters, const TsArgs* ta = nullptr) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_json_sls_host(e, what, js, buf, len, split, SPLIT_JSON_ARGS, out, out_cap, out_len, n_events,
                               counters, &z, ta);
}

// lc_sls_serialize_split_json_dev and its _timestamp_ sibling (tc, ts: the timestamp tables; counters then has
// LC_SRTS_COUNTERS entries)
int split_json_sls_dev(lc_engine_t* e, const char* what, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len,
                       const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                       const uint64_t* d_first, const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                       SPLIT_JSON_PARAMS, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len, uint64_t* counters,
                       const LcSplitJsonTsCfg* tc = nullptr, const lck::TsRowTables* ts = nullptr) {
    if (!e || !js || !out_len || (n && (!d_src || !d_off || !d_len || !d_status || !d_first)) ||
        (n && tc && (!ts->status || !ts->sec || !ts->nsec)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, (tc ? LC_SRTS_COUNTERS : 3) * sizeof(uint64_t));
    if (src_len >= LC_JSON_ARENA || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the source value must be < 2 GiB, < 2^30 pieces per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitJsonSlsCfg c;
    rc = split_json_sls_config(e, what, js, SPLIT_JSON_ARGS, &c);
    if (rc)
        return rc;
    const char* why = tc ? lc_split_regex_ts_ns_check(c, (int)tc->enable_ns) : nullptr;
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    if (n == 0)
        return LC_OK;
    uint64_t m = 0;
    CU_TRY(cudaMemcpyAsync(&m, d_first + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (m && (!d_entries || !d_arena))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    const lck::SplitJsonSlsTables t{d_src, d_off, d_len, d_status, d_first,
                                    reinterpret_cast<const LcJsonEntry*>(d_entries), d_arena, nullptr, nullptr};
    return split_json_sls_run(e, what, c, t, n, m, d_out, nullptr, out_cap, out_len, counters, nullptr, tc, ts);
}

} // namespace

// (the multiline splitter's own counters[3] are added to ml_counters as lc_multiline_split_dev adds them)
#define ML_SPLIT                                                                                                       \
    [&](uint64_t* n) {                                                                                                 \
        return lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,               \
                                      e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), len,  \
                                      n, ml_counters);                                                                 \
    }

extern "C" {

int lc_sls_serialize_split_json_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len,
                                    const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                    const uint64_t* d_first, const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                                    SPLIT_JSON_PARAMS, uint8_t* d_out, uint64_t out_cap, uint64_t* out_len,
                                    uint64_t counters[3]) {
    return split_json_sls_dev(e, "lc_sls_serialize_split_json_dev", js, d_src, src_len, d_off, d_len, n, d_status,
                              d_first, d_entries, d_arena, SPLIT_JSON_ARGS, d_out, out_cap, out_len, counters);
}

int lc_split_json_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, uint8_t split_char,
                            SPLIT_JSON_PARAMS, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                            uint64_t counters[3]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_json_sls_host(e, "lc_split_json_parse_sls", js, buf, len, split, SPLIT_JSON_ARGS, out, out_cap,
                               out_len, n_events, counters, nullptr);
}

int lc_split_json_parse_sls_lz4(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                uint8_t split_char, SPLIT_JSON_PARAMS, const uint8_t* tail, uint64_t tail_len,
                                uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                uint64_t* n_events, uint64_t counters[3]) {
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_json_lz4_host(e, "lc_split_json_parse_sls_lz4", js, buf, len, split, SPLIT_JSON_ARGS, tail,
                               tail_len, out, out_cap, out_len, raw_len, n_events, counters);
}

int lc_multiline_split_json_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                      const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                      int discard_unmatched, SPLIT_JSON_PARAMS, uint8_t* out, uint64_t out_cap,
                                      uint64_t* out_len, uint64_t* n_events, uint64_t counters[3],
                                      uint64_t ml_counters[3]) {
    return split_json_sls_host(e, "lc_multiline_split_json_parse_sls", js, buf, len, ML_SPLIT, SPLIT_JSON_ARGS, out,
                               out_cap, out_len, n_events, counters, nullptr);
}

int lc_multiline_split_json_parse_sls_lz4(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                          const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                          int discard_unmatched, SPLIT_JSON_PARAMS, const uint8_t* tail,
                                          uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                          uint64_t* raw_len, uint64_t* n_events, uint64_t counters[3],
                                          uint64_t ml_counters[3]) {
    return split_json_lz4_host(e, "lc_multiline_split_json_parse_sls_lz4", js, buf, len, ML_SPLIT, SPLIT_JSON_ARGS,
                               tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters);
}

int lc_split_json_timestamp_tap_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src, uint64_t src_len,
                                    const uint32_t* d_off, const uint32_t* d_len, uint64_t n, const uint8_t* d_status,
                                    const uint64_t* d_first, const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                                    const char* renamed_key, uint32_t renamed_key_len, int keep_fail,
                                    int keep_succeed, int copy_raw, const char* offset_key, uint32_t offset_key_len,
                                    const char* tkey, uint32_t tkey_len, uint8_t* d_val, uint64_t val_cap,
                                    uint32_t* d_val_off, uint32_t* d_val_len) {
    static const char* what = "lc_split_json_timestamp_tap_dev";
    if (!e || !js || (n && (!d_src || !d_off || !d_len || !d_status || !d_first || !d_val || !d_val_off ||
                            !d_val_len)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    if (src_len >= LC_JSON_ARENA || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the source value must be < 2 GiB, < 2^30 pieces per call");
    if (n && val_cap < src_len)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": the value buffer must hold src_len + arena bytes");
    int rc = bind(e);
    if (rc)
        return rc;
    const uint64_t src_pos = 0;
    const uint32_t time = 0, time_ns = LC_SLS_NO_NS;
    const TsArgs ta{tkey, tkey_len, nullptr, 0, -1, 0};
    LcSplitJsonSlsCfg c;
    LcSplitJsonTsCfg tc;
    rc = split_json_sls_config(e, what, js, SPLIT_JSON_ARGS, &c, &ta, &tc);
    if (rc || n == 0)
        return rc;
    tc.arena_at = src_len;
    tc.val_cap = val_cap;
    const lck::SplitJsonSlsTables t{d_src, d_off, d_len, d_status, d_first,
                                    reinterpret_cast<const LcJsonEntry*>(d_entries), d_arena, nullptr, nullptr};
    lck::launch_split_json_ts_tap(c, tc, t, n, d_val, d_val_off, d_val_len, e->stream);
    e->launches++;
    CU_TRY(cudaGetLastError());
    return LC_OK;
}

int lc_sls_serialize_split_json_timestamp_dev(lc_engine_t* e, const lc_json_t* js, const uint8_t* d_src,
                                              uint64_t src_len, const uint32_t* d_off, const uint32_t* d_len,
                                              uint64_t n, const uint8_t* d_status, const uint64_t* d_first,
                                              const lc_json_entry_t* d_entries, const uint8_t* d_arena,
                                              SPLIT_JSON_PARAMS, const uint8_t* d_ts_status, const int64_t* d_ts_sec,
                                              const uint32_t* d_ts_nsec, int enable_ns, uint8_t* d_out,
                                              uint64_t out_cap, uint64_t* out_len, uint64_t counters[8]) {
    LcSplitJsonTsCfg tc;
    memset(&tc, 0, sizeof tc);
    tc.enable_ns = enable_ns != 0;
    const lck::TsRowTables ts{d_ts_status, d_ts_sec, d_ts_nsec};
    return split_json_sls_dev(e, "lc_sls_serialize_split_json_timestamp_dev", js, d_src, src_len, d_off, d_len, n,
                              d_status, d_first, d_entries, d_arena, SPLIT_JSON_ARGS, d_out, out_cap, out_len,
                              counters, &tc, &ts);
}

#define TS_ARGS_OF_CALL const TsArgs ta{tkey, tkey_len, ts, now, discard_interval, enable_ns};

int lc_split_json_timestamp_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                      uint8_t split_char, SPLIT_JSON_PARAMS, const char* tkey, uint32_t tkey_len,
                                      const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns,
                                      uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                      uint64_t counters[8]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_json_sls_host(e, "lc_split_json_timestamp_parse_sls", js, buf, len, split, SPLIT_JSON_ARGS, out,
                               out_cap, out_len, n_events, counters, nullptr, &ta);
}

int lc_split_json_timestamp_parse_sls_lz4(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len,
                                          uint8_t split_char, SPLIT_JSON_PARAMS, const char* tkey, uint32_t tkey_len,
                                          const lc_timestamp_t* ts, int64_t now, int32_t discard_interval,
                                          int enable_ns, const uint8_t* tail, uint64_t tail_len, uint8_t* out,
                                          uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events,
                                          uint64_t counters[8]) {
    TS_ARGS_OF_CALL
    auto split = [&](uint64_t* n) {
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),
                                  e->out_b.as<uint32_t>(), len, n);
    };
    return split_json_lz4_host(e, "lc_split_json_timestamp_parse_sls_lz4", js, buf, len, split, SPLIT_JSON_ARGS, tail,
                               tail_len, out, out_cap, out_len, raw_len, n_events, counters, &ta);
}

int lc_multiline_split_json_timestamp_parse_sls(lc_engine_t* e, const lc_json_t* js, const uint8_t* buf,
                                                uint64_t len, const lc_regex_t* start, const lc_regex_t* cont,
                                                const lc_regex_t* end, int discard_unmatched, SPLIT_JSON_PARAMS,
                                                const char* tkey, uint32_t tkey_len, const lc_timestamp_t* ts,
                                                int64_t now, int32_t discard_interval, int enable_ns, uint8_t* out,
                                                uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                                                uint64_t counters[8], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    return split_json_sls_host(e, "lc_multiline_split_json_timestamp_parse_sls", js, buf, len, ML_SPLIT,
                               SPLIT_JSON_ARGS, out, out_cap, out_len, n_events, counters, nullptr, &ta);
}

int lc_multiline_split_json_timestamp_parse_sls_lz4(
    lc_engine_t* e, const lc_json_t* js, const uint8_t* buf, uint64_t len, const lc_regex_t* start,
    const lc_regex_t* cont, const lc_regex_t* end, int discard_unmatched, SPLIT_JSON_PARAMS, const char* tkey,
    uint32_t tkey_len, const lc_timestamp_t* ts, int64_t now, int32_t discard_interval, int enable_ns,
    const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
    uint64_t* n_events, uint64_t counters[8], uint64_t ml_counters[3]) {
    TS_ARGS_OF_CALL
    return split_json_lz4_host(e, "lc_multiline_split_json_timestamp_parse_sls_lz4", js, buf, len, ML_SPLIT,
                               SPLIT_JSON_ARGS, tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters,
                               &ta);
}
#undef TS_ARGS_OF_CALL

} // extern "C"
#undef ML_SPLIT
#undef SPLIT_JSON_PARAMS
#undef SPLIT_JSON_ARGS

// ---------------------------------------------------------------------------------------------- split -> Apsara -> SLS
// The Apsara stage's CommonParserOptions, the offset content of the split events (offset_key NULL = no
// log.file.offset metadata) with the source event's position, time and ns, and mEnableTimestampNanosecond
#define SPLIT_APSARA_PARAMS                                                                                            \
    const char *renamed_key, uint32_t renamed_key_len, int keep_fail, int keep_succeed, int copy_raw,                 \
        const char *offset_key, uint32_t offset_key_len, uint64_t src_pos, uint32_t time, uint32_t time_ns,           \
        int enable_ns
#define SPLIT_APSARA_ARGS                                                                                              \
    renamed_key, renamed_key_len, keep_fail, keep_succeed, copy_raw, offset_key, offset_key_len, src_pos, time,       \
        time_ns, enable_ns

namespace {

// lc_split_apsara_sls_setup over ap's SourceKey, with SourceKey, RenamedSourceKey, the offset key and the fixed names
// staged on the device (`sls_plan`, which neither splitter nor the Apsara stage uses) and *c pointing at them
int split_apsara_sls_config(lc_engine_t* e, const char* what, const lc_apsara_t* ap, SPLIT_APSARA_PARAMS,
                            LcSplitApsaraSlsCfg* c) {
    if (!ap || (renamed_key_len && !renamed_key) || (offset_key_len && !offset_key))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    const uint32_t oklen = offset_key ? offset_key_len : 0u;
    if ((uint64_t)ap->skey.size() + renamed_key_len + oklen + LC_AP_SLS_NAMES_LEN + 16 > 0xFFFFFFFFull)
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": keys must stay below 4 GiB");
    const char* why = lc_split_apsara_sls_setup(ap->skey.data(), (uint32_t)ap->skey.size(), renamed_key,
                                                renamed_key_len, offset_key, oklen, keep_fail, keep_succeed, copy_raw,
                                                src_pos, time, time_ns, enable_ns, c);
    if (why)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": " + why);
    std::string keys = ap->skey;
    keys.append(renamed_key ? renamed_key : "", renamed_key_len);
    keys.append(offset_key ? offset_key : "", oklen);
    keys.append(LC_AP_SLS_NAMES, LC_AP_SLS_NAMES_LEN);
    CU_TRY(e->sls_plan.ensure(keys.size() + 1));
    CU_TRY(cudaMemcpyAsync(e->sls_plan.p, keys.data(), keys.size(), cudaMemcpyHostToDevice, e->stream));
    const uint8_t* d = e->sls_plan.as<uint8_t>();
    c->skey = d;
    c->rkey = d + c->sklen;
    c->okey = d + c->sklen + c->rklen;
    c->names = c->okey + c->oklen;
    return LC_OK;
}

// The size pass and the emit of the chain over the n pieces of t: into d_out (the device-fed call), or back to the
// host buffer out, or -- with z -- records ‖ tail as one LZ4 block.  counters[5] in lc_apsara_parse's order; set
// whenever the size pass ran.
int split_apsara_sls_run(lc_engine_t* e, const char* what, const LcSplitApsaraSlsCfg& c,
                         const lck::SplitApsaraSlsTables& t, uint64_t n, uint8_t* d_out, uint8_t* out,
                         uint64_t out_cap, uint64_t* out_len, uint64_t* counters, const Lz4Tail* z) {
    uint64_t ctr[LC_AP_SLS_COUNTERS + 1] = {0}; // + pieces whose record would reach 4 GiB
    SlsTo to;
    to.host = out;
    to.z = z;
    to.too_large = LC_AP_SLS_COUNTERS;
    const int rc = serialize_sls_dev(
        e, what, n, LC_AP_SLS_COUNTERS + 1,
        [&](uint32_t* rec, uint32_t* body, unsigned long long* d_ctr) {
            lck::launch_split_apsara_sls_sizes(c, t, n, rec, body, d_ctr, e->stream);
        },
        [&](const uint64_t* rec_off, const uint32_t* body, uint8_t* dst) {
            lck::launch_split_apsara_sls_emit(c, t, n, rec_off, body, dst, e->stream);
        },
        d_out, out_cap, out_len, ctr, to);
    if (counters)
        memcpy(counters, ctr, LC_AP_SLS_COUNTERS * sizeof(uint64_t));
    return rc;
}

// Host-buffer split + Apsara + serialise (lc_split_apsara_parse_sls and the multiline / LZ4 siblings): the Apsara
// stage runs ap_count / ap_emit over the pieces, the chunk as their base and one group, into the ap_* buffers of
// lc_apsara_parse, then split_apsara_sls_run.  The stage's counters are the size pass's, so ap_count's own go to
// ts_cnt unread.
template <class Split>
int split_apsara_sls_host(lc_engine_t* e, const char* what, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                          Split split, SPLIT_APSARA_PARAMS, int64_t now, int32_t discard_interval, uint8_t* out,
                          uint64_t out_cap, uint64_t* out_len, uint64_t* n_events, uint64_t* counters,
                          const Lz4Tail* z) {
    LcSplitApsaraSlsCfg c;
    auto begin = [&]() {
        if (counters)
            memset(counters, 0, LC_AP_SLS_COUNTERS * sizeof(uint64_t));
        return (int)LC_OK;
    };
    auto config = [&]() { return split_apsara_sls_config(e, what, ap, SPLIT_APSARA_ARGS, &c); };
    auto run = [&](uint64_t n) {
        if (n >= (1ull << 30))
            return fail(LC_ERR_TOO_LARGE, std::string(what) + ": < 2^30 pieces per call");
        CU_TRY(e->ap_status.ensure(n));
        CU_TRY(e->ap_sec.ensure(n * 8));
        CU_TRY(e->ap_nsec.ensure(n * 4));
        CU_TRY(e->ap_micro.ensure(n * 8));
        CU_TRY(e->ap_first.ensure((n + 1) * 8));
        CU_TRY(e->ts_cnt.ensure(5 * sizeof(uint64_t)));
        CU_TRY(e->sa_grp.ensure(8));
        const uint32_t g[2] = {0u, (uint32_t)n};
        CU_TRY(cudaMemcpyAsync(e->sa_grp.p, g, sizeof g, cudaMemcpyHostToDevice, e->stream));
        const uint8_t* d_src = e->in.as<uint8_t>();
        const uint32_t *off = e->out_a.as<uint32_t>(), *ln = e->out_b.as<uint32_t>();
        uint64_t m = 0;
        int rc = ap_count(e, ap, what, d_src, len, off, ln, n, e->sa_grp.as<uint32_t>(), 1, now, discard_interval,
                          e->ap_status.as<uint8_t>(), e->ap_sec.as<int64_t>(), e->ap_nsec.as<uint32_t>(),
                          e->ap_micro.as<int64_t>(), e->ap_first.as<uint64_t>(), &m, e->ts_cnt.as<uint64_t>());
        if (rc)
            return rc;
        CU_TRY(e->ap_ent.ensure(m * sizeof(LcApEntry) + 16));
        if (m) {
            rc = ap_emit(e, d_src, off, ln, n, e->ap_status.as<uint8_t>(), e->ap_first.as<uint64_t>(),
                         e->ap_ent.as<lc_apsara_entry_t>());
            if (rc)
                return rc;
        }
        const lck::SplitApsaraSlsTables t{d_src,
                                          off,
                                          ln,
                                          e->ap_status.as<uint8_t>(),
                                          e->ap_sec.as<int64_t>(),
                                          e->ap_nsec.as<uint32_t>(),
                                          e->ap_micro.as<int64_t>(),
                                          e->ap_first.as<uint64_t>(),
                                          e->ap_ent.as<LcApEntry>()};
        return split_apsara_sls_run(e, what, c, t, n, nullptr, out, out_cap, out_len, counters, z);
    };
    return split_chain_sls_host(e, what, buf, len, split, ap != nullptr, begin, config, run, out, out_cap, out_len,
                                n_events, z);
}

template <class Split>
int split_apsara_lz4_host(lc_engine_t* e, const char* what, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                          Split split, SPLIT_APSARA_PARAMS, int64_t now, int32_t discard_interval,
                          const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                          uint64_t* raw_len, uint64_t* n_events, uint64_t* counters) {
    const Lz4Tail z{tail, tail_len, raw_len};
    return split_apsara_sls_host(e, what, ap, buf, len, split, SPLIT_APSARA_ARGS, now, discard_interval, out, out_cap,
                                 out_len, n_events, counters, &z);
}

} // namespace

// (the multiline splitter's own counters[3] are added to ml_counters as lc_multiline_split_dev adds them)
#define ML_SPLIT                                                                                                       \
    [&](uint64_t* n) {                                                                                                 \
        return lc_multiline_split_dev(e, e->in.as<uint8_t>(), len, start, cont, end, discard_unmatched,               \
                                      e->out_a.as<uint32_t>(), e->out_b.as<uint32_t>(), e->out_c.as<uint8_t>(), len,  \
                                      n, ml_counters);                                                                 \
    }
#define LINE_SPLIT                                                                                                     \
    [&](uint64_t* n) {                                                                                                 \
        return lc_split_lines_dev(e, e->in.as<uint8_t>(), len, split_char, e->out_a.as<uint32_t>(),                   \
                                  e->out_b.as<uint32_t>(), len, n);                                                    \
    }

extern "C" {

int lc_sls_serialize_split_apsara_dev(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* d_src, uint64_t src_len,
                                      const uint32_t* d_off, const uint32_t* d_len, uint64_t n,
                                      const uint8_t* d_status, const int64_t* d_sec, const uint32_t* d_nsec,
                                      const int64_t* d_micro, const uint64_t* d_first,
                                      const lc_apsara_entry_t* d_entries, SPLIT_APSARA_PARAMS, uint8_t* d_out,
                                      uint64_t out_cap, uint64_t* out_len, uint64_t counters[5]) {
    static const char* what = "lc_sls_serialize_split_apsara_dev";
    if (!e || !ap || !out_len ||
        (n && (!d_src || !d_off || !d_len || !d_status || !d_sec || !d_nsec || !d_micro || !d_first)))
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    *out_len = 0;
    if (counters)
        memset(counters, 0, LC_AP_SLS_COUNTERS * sizeof(uint64_t));
    if (src_len >= 0xFFFFFFF0ull || n >= (1ull << 30))
        return fail(LC_ERR_TOO_LARGE, std::string(what) + ": the source value must be < 4 GiB, < 2^30 pieces per call");
    int rc = bind(e);
    if (rc)
        return rc;
    LcSplitApsaraSlsCfg c;
    rc = split_apsara_sls_config(e, what, ap, SPLIT_APSARA_ARGS, &c);
    if (rc || n == 0)
        return rc;
    uint64_t m = 0;
    CU_TRY(cudaMemcpyAsync(&m, d_first + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CU_TRY(cudaStreamSynchronize(e->stream));
    if (m && !d_entries)
        return fail(LC_ERR_INVALID_ARG, std::string(what) + ": bad arguments");
    const lck::SplitApsaraSlsTables t{d_src,   d_off,   d_len,
                                      d_status, d_sec,  d_nsec,
                                      d_micro, d_first, reinterpret_cast<const LcApEntry*>(d_entries)};
    return split_apsara_sls_run(e, what, c, t, n, d_out, nullptr, out_cap, out_len, counters, nullptr);
}

int lc_split_apsara_parse_sls(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                              uint8_t split_char, SPLIT_APSARA_PARAMS, int64_t now, int32_t discard_interval,
                              uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* n_events,
                              uint64_t counters[5]) {
    return split_apsara_sls_host(e, "lc_split_apsara_parse_sls", ap, buf, len, LINE_SPLIT, SPLIT_APSARA_ARGS, now,
                                 discard_interval, out, out_cap, out_len, n_events, counters, nullptr);
}

int lc_split_apsara_parse_sls_lz4(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                  uint8_t split_char, SPLIT_APSARA_PARAMS, int64_t now, int32_t discard_interval,
                                  const uint8_t* tail, uint64_t tail_len, uint8_t* out, uint64_t out_cap,
                                  uint64_t* out_len, uint64_t* raw_len, uint64_t* n_events, uint64_t counters[5]) {
    return split_apsara_lz4_host(e, "lc_split_apsara_parse_sls_lz4", ap, buf, len, LINE_SPLIT, SPLIT_APSARA_ARGS, now,
                                 discard_interval, tail, tail_len, out, out_cap, out_len, raw_len, n_events, counters);
}

int lc_multiline_split_apsara_parse_sls(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                        const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                        int discard_unmatched, SPLIT_APSARA_PARAMS, int64_t now,
                                        int32_t discard_interval, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                                        uint64_t* n_events, uint64_t counters[5], uint64_t ml_counters[3]) {
    return split_apsara_sls_host(e, "lc_multiline_split_apsara_parse_sls", ap, buf, len, ML_SPLIT, SPLIT_APSARA_ARGS,
                                 now, discard_interval, out, out_cap, out_len, n_events, counters, nullptr);
}

int lc_multiline_split_apsara_parse_sls_lz4(lc_engine_t* e, const lc_apsara_t* ap, const uint8_t* buf, uint64_t len,
                                            const lc_regex_t* start, const lc_regex_t* cont, const lc_regex_t* end,
                                            int discard_unmatched, SPLIT_APSARA_PARAMS, int64_t now,
                                            int32_t discard_interval, const uint8_t* tail, uint64_t tail_len,
                                            uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* raw_len,
                                            uint64_t* n_events, uint64_t counters[5], uint64_t ml_counters[3]) {
    return split_apsara_lz4_host(e, "lc_multiline_split_apsara_parse_sls_lz4", ap, buf, len, ML_SPLIT,
                                 SPLIT_APSARA_ARGS, now, discard_interval, tail, tail_len, out, out_cap, out_len,
                                 raw_len, n_events, counters);
}

} // extern "C"
#undef ML_SPLIT
#undef LINE_SPLIT
#undef SPLIT_APSARA_PARAMS
#undef SPLIT_APSARA_ARGS
