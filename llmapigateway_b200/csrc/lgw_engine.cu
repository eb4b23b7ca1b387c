// llmgw_b200 engine: C ABI (include/llmgw_b200.h) over the sm_90a (H100) kernels.
// No CPU fallback anywhere in this file: every entry point either runs on the device or fails.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <array>
#include <string>
#include <vector>

#include "../../include/llmgw_b200.h"
#include "stream_machine.cuh"
#include "sse_kernels.cuh"
#include "rollup.cuh"
#include "listing.cuh"
#include "retain.cuh"
#include "append.cuh"
#include "load.cuh"
#include "save.cuh"
#include "body_kernels.cuh"
#include "doc_kernels.cuh"
#include "transcript.cuh"

using namespace lgw;

static_assert(sizeof(Val) == sizeof(lgw_val), "lgw_val layout");
static_assert(sizeof(UsageRec) == sizeof(lgw_usage_rec), "lgw_usage_rec layout");
static_assert(sizeof(StreamState) == sizeof(lgw_stream_state), "lgw_stream_state layout");
static_assert(sizeof(RowEvent) == sizeof(lgw_row_event), "lgw_row_event layout");
static_assert(sizeof(SegResult) == sizeof(lgw_seg_result), "lgw_seg_result layout");
static_assert(sizeof(RollupRow) == sizeof(lgw_rollup_row), "lgw_rollup_row layout");
static_assert(sizeof(DocUsage) == sizeof(lgw_doc_usage), "lgw_doc_usage layout");
static_assert(sizeof(TextMark) == sizeof(lgw_text_mark), "lgw_text_mark layout");
static_assert(sizeof(SaveText) == sizeof(lgw_save_text), "lgw_save_text layout");

static thread_local std::string g_create_error;

// Grow-only device staging.  reserve() keeps the buffer while it is large enough; otherwise it frees it and allocates
// need + slack bytes (cudaFree synchronises the device, so callers whose sizes creep upward pass a slack).  The contents do
// not survive a growth.  Freed with the engine that holds it.
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    cudaError_t reserve(size_t need, size_t slack = 0) {
        if (need <= cap) return cudaSuccess;
        release();
        const cudaError_t r = cudaMalloc(&p, need + slack);
        if (r == cudaSuccess) cap = need + slack;
        return r;
    }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

// The same for page-locked host staging (cudaHostAlloc).
struct HostBuf {
    void* p = nullptr; size_t cap = 0;
    HostBuf() = default;
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { if (p) cudaFreeHost(p); }
    cudaError_t reserve(size_t need, size_t slack = 0) {
        if (need <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        const cudaError_t r = cudaHostAlloc(&p, need + slack, cudaHostAllocDefault);
        if (r == cudaSuccess) cap = need + slack;
        return r;
    }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

// The arrays of one step as the kernels see them (device memory, or page-locked host memory in the direct modes).
struct StepArrays {
    const uint8_t* bytes; uint64_t n_bytes;
    const uint32_t* chunk_off; uint32_t n_chunks;
    const uint32_t *seg_chunk, *seg_slot; uint32_t n_segs;
    uint8_t* out; SegResult* seg_out;
};

// One launch set's share of a step: segments [s0, s1), chunks [c0, c1), bytes [b0, b1).  All are absolute, so the slices of a
// pipelined step share the device arrays.
struct StepSlice {
    uint32_t s0, s1, c0, c1, b0; uint64_t b1;
    static StepSlice whole(uint32_t n_segs, uint32_t n_chunks, uint64_t n_bytes) { return {0, n_segs, 0, n_chunks, 0, n_bytes}; }
};

struct lgw_engine {
    int device = 0;
    lgw_limits lim{};
    int sm_count = 132;
    int mode = 0;                   // 0: fast path + general fix-up, 1: general path only
    cudaStream_t own_stream = nullptr, stream = nullptr;
    cudaStream_t s_in = nullptr, s_out = nullptr;       // copy streams of the pipelined host entry point
    uint64_t launches = 0;
    std::string err;
    // What the engine owns on the device and how it goes away: fixed-size allocations (dev_alloc) and events (new_events)
    // are recorded here and released by the destructor; grow-only staging is DevBuf members, which release themselves.
    std::vector<void*> allocs;
    std::vector<cudaEvent_t> events;
    DeviceTables t{};               // persistent per-slot state
    uint32_t* d_rowq_count = nullptr; RowEvent* d_rowq = nullptr;
    StepScratch scratch{};          // per-step scratch (sized by max_step_chunks / max_streams)
    uint32_t* d_slots = nullptr; int32_t* d_status = nullptr; StreamState* d_state_stage = nullptr;   // slot lists of open / state / close
    struct Open {                   // lgw_streams_open is stream-ordered: the caller's lists are copied here first, so they are free on return
        HostBuf h;                  // page-locked: slots[max_streams] ++ status[max_streams]
        cudaEvent_t done = nullptr; bool pending = false;   // recorded after the uploads; waited for before the staging is written again
    } open;
    DevBuf details;                 // staging of lgw_streams_details
    struct Step {
        uint8_t *d_in = nullptr, *d_out = nullptr;      // staging for the host-pointer entry point
        uint32_t *d_chunk_off = nullptr, *d_seg_chunk = nullptr, *d_seg_slot = nullptr; SegResult* d_seg_out = nullptr;
        cudaEvent_t ev_in[16]{}, ev_k[16]{};    // upload done / kernels done, per slice; [14] and [15] join the three streams at the step's ends
        cudaEvent_t ev[7]{};            // [0..4] bracket prime / relay / commit / usage extract; [5],[6] the host-buffer step
        cudaEvent_t tr[3][16]{};        // LGW_TRACE: upload / kernels / download done, per slice; created by the first traced step
        float ms[5]{0, 0, 0, 0, 0};     // prime, relay, commit, usage extract, whole host-buffer step
        bool timed = false, kernel_times_valid = false;
        bool per_kernel_timing = false; // true: events between the step's kernels (lgw_last_step_kernel_ms); false: programmatic dependent launches
        bool last_direct = false;       // the last host-buffer step ran in direct mode (kernel-driven PCIe traffic)
        StepArrays last{};              // the arrays of the last step: what lgw_step_transcript_run works on
    } step;
    struct Rollup {
        DevBuf rows, partial, tiles; unsigned long long* d_nrows = nullptr;
        bool attr_set = false, force_global = false;
        cudaEvent_t ev[4]{}; float ms[2]{0, 0};
    } rollup;
    struct Listing {                // record listing (listing.cuh): one scratch buffer, events created on first use
        DevBuf buf; bool attr_set = false;
        cudaEvent_t ev[2]{}; float ms = 0;
    } listing;
    struct Retain {                 // deleting old records (retain.cuh): tile counts / offsets and the total, events created on first use
        DevBuf tiles;
        cudaEvent_t ev[2]{}; float ms = 0;
    } retain;
    struct Append {                 // inserted records (append.cuh): the new rows and the rank map, staged page-locked, then on the device
        HostBuf host; DevBuf dev;
        cudaEvent_t ev[2]{}; float ms = 0;
    } append;
    struct Load {                   // loading the usage table from a tokens_usage file (load.cuh); stage 1: decoded, 2: marked
        DevBuf file, walk, recs, dict, maps, out;
        DbGeom g{}; LoadRecs r{}; LoadDict d[2]{};
        uint32_t n = 0, tiles = 0, n_names[2]{}; uint64_t n_keep = 0; int stage = 0;
        std::vector<uint8_t> refused[2];        // the maps' refusals at mark time
        cudaEvent_t ev[8]{}; float ms[4]{0, 0, 0, 0};
    } load;
    struct Save {                   // saving the usage table as a tokens_usage file (save.cuh); stage 1: planned
        DevBuf in, recs, sort, pack, pool, img;
        SaveCtx c{}; uint32_t n = 0, kept = 0, n_pool = 0, n_ovfl = 0, pages = 0; int64_t* refused = nullptr; int stage = 0;
        cudaEvent_t ev[8]{}; float ms[6]{0, 0, 0, 0, 0, 0};
    } save;
    struct Bodies {                 // request-body rewrite (rows a1-a4) and the document kernels, which share its input staging
        DevBuf plans, ops, blob; uint32_t n_plans = 0, n_ops = 0;       // the rule tables of lgw_rules_load
        DevBuf in, off, out_off, plan_idx, results, scans;      // per call: the packed bodies and five arrays indexed by body
        DevBuf slots, out, models, redo;
        DevBuf doc_out, doc_text;   // results of lgw_documents_usage / lgw_documents_error_detail
        int mode = 0;               // 0: data-parallel path + exact machine for the rest, 1: exact machine only (tests)
        cudaEvent_t ev[4]{}; float ms[3]{0, 0, 0};
    } bodies;
    struct DocsText {               // lgw_documents_text (doc_kernels.cuh): input in the body staging, events created on first use
        DevBuf sparse, len, flags, off, text;
        cudaEvent_t ev[2]{}; float ms = 0;
    } docs_text;
    struct Text {                   // transcript tap (transcript.cuh; off until lgw_transcripts_enable)
        bool on = false, pending = false, ready = false;
        TextTap* tap = nullptr; uint8_t *carry = nullptr, *sparse = nullptr, *text = nullptr;
        uint32_t *piece_len = nullptr, *seg_len = nullptr, *seg_flags = nullptr, *markq_count = nullptr;
        unsigned long long* seg_off = nullptr; TextMark* markq = nullptr;
        uint64_t total = 0; uint32_t marks = 0;
        cudaEvent_t ev[2]{}; float ms = 0;
    } text;

    ~lgw_engine() {                 // (the caller has made `device` current)
        for (void* p : allocs) cudaFree(p);
        for (cudaEvent_t ev : events) cudaEventDestroy(ev);
        if (s_in) cudaStreamDestroy(s_in);
        if (s_out) cudaStreamDestroy(s_out);
        if (own_stream) cudaStreamDestroy(own_stream);
    }
};

#define CK(e, call) do { cudaError_t _r = (call); if (_r != cudaSuccess) { \
    (e)->err = std::string(#call) + ": " + cudaGetErrorString(_r); return LGW_ERR_CUDA; } } while (0)
// the same for a call that returns an LGW_* code (and has set e->err)
#define TRY(call) do { const int _rc = (call); if (_rc != LGW_OK) return _rc; } while (0)

// A fixed-size device allocation that lives as long as the engine.
template <class T> static cudaError_t dev_alloc(lgw_engine* e, T*& p, size_t bytes) {
    const cudaError_t r = cudaMalloc((void**)&p, bytes);
    if (r == cudaSuccess) e->allocs.push_back(p);
    return r;
}

// n events that live as long as the engine.
static cudaError_t new_events(lgw_engine* e, cudaEvent_t* ev, int n, unsigned flags = cudaEventDefault) {
    for (int i = 0; i < n; ++i) {
        const cudaError_t r = cudaEventCreateWithFlags(&ev[i], flags);
        if (r != cudaSuccess) return r;
        e->events.push_back(ev[i]);
    }
    return cudaSuccess;
}

// ms = the time between two recorded events; kept as it was when they cannot be read (not recorded yet, or not complete).
static void read_ms(cudaEvent_t from, cudaEvent_t to, float& ms) {
    float t = 0;
    if (cudaEventElapsedTime(&t, from, to) == cudaSuccess) ms = t;
}

// Blocks for n_items at per_block items a block, at most blocks_per_sm for each SM (the kernels stride over the rest).
static unsigned grid_for(const lgw_engine* e, uint64_t n_items, uint32_t per_block, uint32_t blocks_per_sm) {
    const uint64_t want = (n_items + per_block - 1) / per_block, most = (uint64_t)e->sm_count * blocks_per_sm;
    return (unsigned)(want < most ? want : most);
}

static int check_slots(lgw_engine* e, const uint32_t* slots, uint32_t n) {
    for (uint32_t i = 0; i < n; ++i) if (slots[i] >= e->lim.max_streams) { e->err = "slot out of range"; return LGW_ERR_ARG; }
    return LGW_OK;
}

// A checked slot list into d_slots (which holds max_streams of them), on the engine stream.
static int stage_slots(lgw_engine* e, const uint32_t* slots, uint32_t n) {
    if (n > e->lim.max_streams) { e->err = "more slots than max_streams"; return LGW_ERR_CAPACITY; }
    TRY(check_slots(e, slots, n));
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaMemcpyAsync(e->d_slots, slots, n * 4, cudaMemcpyHostToDevice, e->stream));
    return LGW_OK;
}

extern "C" int lgw_abi_version(void) { return LGW_ABI_VERSION; }

extern "C" const char* lgw_last_error(const lgw_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

extern "C" int lgw_engine_create(int device, const lgw_limits* limits, lgw_engine** out) {
    if (!out || !limits) { g_create_error = "null argument"; return LGW_ERR_ARG; }
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) {
        g_create_error = "no usable CUDA device (this engine has no CPU path)";
        return LGW_ERR_NO_DEVICE;
    }
    lgw_engine* e = new lgw_engine();
    e->device = device; e->lim = *limits;
    if (e->lim.max_streams == 0 || e->lim.carry_cap < 64 || e->lim.detail_cap < 64 || e->lim.max_step_chunks == 0 || e->lim.max_step_bytes == 0) {
        g_create_error = "limits out of range"; delete e; return LGW_ERR_ARG;
    }
    auto fail = [&](const char* what, cudaError_t r) { g_create_error = std::string(what) + ": " + cudaGetErrorString(r); lgw_engine_destroy(e); return LGW_ERR_CUDA; };
    cudaError_t r;
    if ((r = cudaSetDevice(device)) != cudaSuccess) return fail("cudaSetDevice", r);
    cudaDeviceProp prop;
    if ((r = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail("cudaGetDeviceProperties", r);
    e->sm_count = prop.multiProcessorCount;
    if ((r = cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", r);
    e->stream = e->own_stream;
    if ((r = cudaStreamCreateWithFlags(&e->s_in, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", r);
    if ((r = cudaStreamCreateWithFlags(&e->s_out, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", r);
    if ((r = new_events(e, e->step.ev_in, 16, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", r);
    if ((r = new_events(e, e->step.ev_k, 16, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", r);
    if ((r = new_events(e, e->step.ev, 7)) != cudaSuccess) return fail("cudaEventCreate", r);
    if ((r = new_events(e, e->rollup.ev, 4)) != cudaSuccess) return fail("cudaEventCreate", r);
    if ((r = new_events(e, e->bodies.ev, 4)) != cudaSuccess) return fail("cudaEventCreate", r);
    const size_t S = e->lim.max_streams, C = e->lim.max_step_chunks, B = e->lim.max_step_bytes;
#define ALLOC(ptr, bytes) if ((r = dev_alloc(e, ptr, (bytes))) != cudaSuccess) return fail("cudaMalloc " #ptr, r)
    ALLOC(e->t.state, S * sizeof(StreamState));
    ALLOC(e->t.carry_a, S * (size_t)e->lim.carry_cap);
    ALLOC(e->t.carry_b, S * (size_t)e->lim.carry_cap);
    ALLOC(e->t.detail, S * (size_t)e->lim.detail_cap);
    ALLOC(e->t.pending, S * (size_t)LGW_PENDING_STRIDE);
    e->t.carry_cap = e->lim.carry_cap; e->t.detail_cap = e->lim.detail_cap; e->t.max_streams = e->lim.max_streams;
    ALLOC(e->d_rowq, (size_t)(e->lim.rowq_cap + 1) * sizeof(RowEvent));
    ALLOC(e->d_rowq_count, 16);
    ALLOC(e->step.d_in, B + 64); ALLOC(e->step.d_out, B + 64);
    ALLOC(e->step.d_chunk_off, (C + 1) * 4); ALLOC(e->step.d_seg_chunk, (S + 1) * 4); ALLOC(e->step.d_seg_slot, S * 4);
    ALLOC(e->step.d_seg_out, S * sizeof(SegResult));
    ALLOC(e->d_slots, S * 4); ALLOC(e->d_status, S * 4); ALLOC(e->d_state_stage, S * sizeof(StreamState));
#undef ALLOC
    if ((r = e->open.h.reserve(S * 8)) != cudaSuccess) return fail("cudaHostAlloc", r);
    if ((r = new_events(e, &e->open.done, 1, cudaEventDisableTiming)) != cudaSuccess) return fail("cudaEventCreate", r);
    if ((r = scratch_alloc(e->scratch, S, [e](auto*& p, size_t bytes) { return dev_alloc(e, p, bytes); })) != cudaSuccess) return fail("scratch_alloc", r);
    if ((r = cudaMemset(e->t.state, 0, S * sizeof(StreamState))) != cudaSuccess) return fail("cudaMemset", r);
    if ((r = cudaMemset(e->d_rowq_count, 0, 16)) != cudaSuccess) return fail("cudaMemset", r);
    const char* m = getenv("LGW_FORCE_GENERAL");
    e->mode = (m && m[0] == '1') ? 1 : 0;
    *out = e;
    return LGW_OK;
}

extern "C" int lgw_engine_destroy(lgw_engine* e) {
    if (!e) return LGW_OK;
    cudaSetDevice(e->device);
    delete e;
    return LGW_OK;
}

extern "C" int lgw_engine_set_stream(lgw_engine* e, void* s) {
    if (!e) return LGW_ERR_ARG;
    e->stream = s ? (cudaStream_t)s : e->own_stream;
    return LGW_OK;
}

extern "C" int lgw_engine_set_kernel_timing(lgw_engine* e, int on) {   // 1: CUDA events between the kernels of a step (they then run back to back, not overlapped)
    if (!e) return LGW_ERR_ARG;
    e->step.per_kernel_timing = on != 0;
    return LGW_OK;
}

extern "C" int lgw_engine_set_mode(lgw_engine* e, int mode) {     // 0 fast+fix-up, 1 general only (tests)
    if (!e) return LGW_ERR_ARG;
    e->mode = mode; e->bodies.mode = mode;
    return LGW_OK;
}

// Stream-ordered: returns once the work is enqueued, without waiting for the GPU (a serving loop enqueues the next step behind
// it while earlier work still runs).  The caller's arrays are copied into the engine's page-locked staging first, so the caller
// may reuse or free them on return, pinned or not; the staging itself is written again only after its last upload is done.
extern "C" int lgw_streams_open(lgw_engine* e, const uint32_t* slots, const int32_t* http_status, uint32_t n) {
    if (!e || !slots || !http_status) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    if (n > e->lim.max_streams) { e->err = "more slots than max_streams"; return LGW_ERR_CAPACITY; }
    TRY(check_slots(e, slots, n));
    CK(e, cudaSetDevice(e->device));
    if (e->open.pending) { CK(e, cudaEventSynchronize(e->open.done)); e->open.pending = false; }
    uint32_t* h_slots = e->open.h.as<uint32_t>();
    int32_t* h_status = reinterpret_cast<int32_t*>(h_slots + e->lim.max_streams);
    memcpy(h_slots, slots, (size_t)n * 4); memcpy(h_status, http_status, (size_t)n * 4);
    CK(e, cudaMemcpyAsync(e->d_slots, h_slots, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaMemcpyAsync(e->d_status, h_status, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaEventRecord(e->open.done, e->stream));
    e->open.pending = true;
    k_streams_open<<<(n + 127) / 128, 128, 0, e->stream>>>(e->t, e->d_slots, e->d_status, n);
    ++e->launches;
    if (e->text.on) { k_text_open<<<(n + 127) / 128, 128, 0, e->stream>>>(e->text.tap, e->d_slots, n); ++e->launches; }
    CK(e, cudaGetLastError());
    return LGW_OK;
}

static int gather_states(lgw_engine* e, const uint32_t* slots, uint32_t n, lgw_stream_state* out, int free_after) {
    if (!e || !slots || !out) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    TRY(stage_slots(e, slots, n));
    k_streams_gather<<<(n + 127) / 128, 128, 0, e->stream>>>(e->t, e->d_slots, n, e->d_state_stage, free_after);
    ++e->launches;
    CK(e, cudaGetLastError());
    CK(e, cudaMemcpyAsync(out, e->d_state_stage, n * sizeof(StreamState), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

extern "C" int lgw_streams_state(lgw_engine* e, const uint32_t* slots, uint32_t n, lgw_stream_state* out) { return gather_states(e, slots, n, out, 0); }
extern "C" int lgw_streams_close(lgw_engine* e, const uint32_t* slots, uint32_t n, lgw_stream_state* out) { return gather_states(e, slots, n, out, 1); }

extern "C" int lgw_stream_detail(lgw_engine* e, uint32_t slot, uint8_t* buf, uint32_t cap, uint32_t* len) {
    if (!e || !buf || !len || slot >= e->lim.max_streams) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    StreamState st;
    CK(e, cudaMemcpyAsync(&st, e->t.state + slot, sizeof(st), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    uint32_t n = st.h.detail_len < cap ? st.h.detail_len : cap;
    if (n) CK(e, cudaMemcpyAsync(buf, e->t.detail + (size_t)slot * e->lim.detail_cap, n, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    *len = n;
    return LGW_OK;
}

// error details of many failed attempts in one round trip: a gather kernel packs min(detail_len, stride) bytes per slot
namespace lgw {
__global__ void k_details_gather(DeviceTables t, const uint32_t* slots, uint32_t n, uint8_t* out, uint32_t stride, uint32_t* lens) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= n) return;
    const uint32_t slot = slots[w];
    uint32_t len = t.state[slot].h.detail_len;
    if (len > t.detail_cap) len = t.detail_cap;
    if (len > stride) len = stride;
    const uint8_t* src = t.detail + (size_t)slot * t.detail_cap;
    uint8_t* dst = out + (size_t)w * stride;
    for (uint32_t i = lane; i < len; i += 32) dst[i] = src[i];
    if (lane == 0) lens[w] = len;
}
}  // namespace lgw

extern "C" int lgw_streams_details(lgw_engine* e, const uint32_t* slots, uint32_t n, uint8_t* buf, uint32_t stride, uint32_t* lens) {
    if (!e || (n && (!slots || !buf || !lens)) || stride == 0) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    TRY(check_slots(e, slots, n));
    CK(e, cudaSetDevice(e->device));
    // staging owned by the engine (a stream-ordered allocation per call gave memory back to the OS at every synchronisation)
    const size_t need = (size_t)n * 8 + (size_t)n * stride;
    CK(e, e->details.reserve(need, need / 2));
    uint32_t* d_slots = e->details.as<uint32_t>(); uint32_t* d_lens = d_slots + n; uint8_t* d_out = e->details.as<uint8_t>() + (size_t)n * 8;
    CK(e, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, e->stream));
    lgw::k_details_gather<<<(n * 32 + 255) / 256, 256, 0, e->stream>>>(e->t, d_slots, n, d_out, stride, d_lens);
    ++e->launches;
    CK(e, cudaMemcpyAsync(lens, d_lens, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(buf, d_out, (size_t)n * stride, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

// ---- the step ------------------------------------------------------------------------------------
static int check_step_limits(lgw_engine* e, uint32_t n_segs, uint32_t n_chunks, uint64_t n_bytes) {
    if (n_segs > e->lim.max_streams || n_chunks > e->lim.max_step_chunks || n_bytes > e->lim.max_step_bytes) {
        e->err = "step exceeds the limits given to lgw_engine_create"; return LGW_ERR_CAPACITY;
    }
    if (n_bytes >= 0xFFFF0000ull) { e->err = "step larger than 4 GiB - 64 KiB"; return LGW_ERR_CAPACITY; }
    return LGW_OK;
}

// The step the transcript pass will tap, once.
static void remember_step(lgw_engine* e, const StepArrays& s) {
    e->step.last = s;
    e->text.pending = e->text.on; e->text.ready = false;
}

// One launch set over a slice of a step whose limits have been checked.
static int step_device(lgw_engine* e, const StepArrays& s, const StepSlice& sl, bool reset_rows) {
    StepArgs a{};
    a.t = e->t; a.data = s.bytes; a.n_bytes = (uint32_t)sl.b1; a.chunk_off = s.chunk_off; a.n_chunks = s.n_chunks;
    a.tile_base = sl.b0; a.chunk_lo = sl.c0; a.chunk_hi = sl.c1;
    a.seg_chunk = s.seg_chunk + sl.s0; a.seg_slot = s.seg_slot + sl.s0; a.n_segs = sl.s1 - sl.s0; a.out = s.out; a.seg_out = s.seg_out + sl.s0;
    a.rowq = e->d_rowq; a.rowq_count = e->d_rowq_count; a.rowq_cap = e->lim.rowq_cap; a.s = e->scratch;
    // the bulk path's first kernel empties the row queue; one call fewer on the host between the caller's enqueue and the kernels
    a.reset_rows = reset_rows && e->mode == 0 && a.n_segs ? 1u : 0u;
    if (reset_rows && !a.reset_rows) CK(e, cudaMemsetAsync(e->d_rowq_count, 0, 4, e->stream));
    int launched = 0;
    const bool pk = e->step.per_kernel_timing || e->mode == 1;
    cudaError_t r = launch_step(a, e->mode, e->sm_count, e->stream, e->step.ev, &launched, pk);
    e->step.kernel_times_valid = pk;
    e->launches += (uint64_t)launched;
    if (r != cudaSuccess) { e->err = std::string("step launch: ") + cudaGetErrorString(r); return LGW_ERR_CUDA; }
    e->step.timed = true;
    return LGW_OK;
}

extern "C" int lgw_sse_step_device(lgw_engine* e, const uint8_t* d_bytes, uint64_t n_bytes, const uint32_t* d_chunk_off, uint32_t n_chunks,
                                   const uint32_t* d_seg_chunk, const uint32_t* d_seg_slot, uint32_t n_segs,
                                   uint8_t* d_out, lgw_seg_result* d_seg_out) {
    if (!e || (!d_bytes && n_bytes) || !d_chunk_off || !d_seg_chunk || !d_seg_slot || (!d_out && n_bytes) || !d_seg_out) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    const StepArrays s{d_bytes, n_bytes, d_chunk_off, n_chunks, d_seg_chunk, d_seg_slot, n_segs, d_out, (SegResult*)d_seg_out};
    remember_step(e, s);
    TRY(check_step_limits(e, n_segs, n_chunks, n_bytes));
    return step_device(e, s, StepSlice::whole(n_segs, n_chunks, n_bytes), true);
}

extern "C" int lgw_fetch_rows(lgw_engine* e, lgw_row_event* rows_out, uint32_t rows_cap, uint32_t* n_rows) {
    if (!e || !n_rows || (!rows_out && rows_cap)) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    uint32_t cnt = 0;
    CK(e, cudaMemcpyAsync(&cnt, e->d_rowq_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    if (cnt > e->lim.rowq_cap) cnt = e->lim.rowq_cap;
    if (cnt > rows_cap) cnt = rows_cap;
    if (cnt) CK(e, cudaMemcpyAsync(rows_out, e->d_rowq, (size_t)cnt * sizeof(RowEvent), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    *n_rows = cnt;
    return LGW_OK;
}

extern "C" int lgw_sync(lgw_engine* e) {
    if (!e) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

// cheap host-side validation of a host step's layout (offsets sorted, segments cover chunks in order)
static int check_step_layout(lgw_engine* e, uint64_t n_bytes, const uint32_t* chunk_off, uint32_t n_chunks,
                             const uint32_t* seg_chunk, const uint32_t* seg_slot, uint32_t n_segs) {
    if (chunk_off[0] != 0 || chunk_off[n_chunks] != n_bytes) { e->err = "chunk_off must start at 0 and end at n_bytes"; return LGW_ERR_ARG; }
    if (n_segs && (seg_chunk[0] != 0 || seg_chunk[n_segs] != n_chunks)) { e->err = "seg_chunk must cover all chunks"; return LGW_ERR_ARG; }
    for (uint32_t s = 0; s < n_segs; ++s) if (seg_chunk[s] > seg_chunk[s + 1] || seg_slot[s] >= e->lim.max_streams) { e->err = "bad segment table"; return LGW_ERR_ARG; }
    return LGW_OK;
}

// Host buffers that are page-locked (lgw_alloc_pinned, cudaHostAlloc, torch pin_memory) need no staging copy: the bulk kernel's
// TMA loads can read the packed chunks straight from the host buffer ("direct in") and its TMA stores can write the re-emitted
// bytes straight into the host output buffer ("direct out"); the parse of a tile then overlaps its own PCIe transfer.
//   LGW_DIRECT = 0 (default) | in | out | both
// The direct modes are correct and save the device staging buffers, but SM-issued PCIe traffic competes with the copy-engine
// stream of the other direction, so the staged, sliced pipeline is the default.
// Sets each pointer to the buffer's device address when that direction may run direct, else to null.
static void probe_direct(const lgw_engine* e, const uint8_t* bytes, uint8_t* out_bytes, uint64_t n_bytes, const uint8_t** direct_in, uint8_t** direct_out) {
    static const int allow = [] { const char* v = getenv("LGW_DIRECT"); if (!v || v[0] == '0') return 0; if (v[0] == 'b') return 3; if (v[0] == 'o') return 2; return 1; }();
    cudaPointerAttributes pa{};
    const bool big = e->mode == 0 && n_bytes >= (1u << 20);
    *direct_in = nullptr; *direct_out = nullptr;
    if (big && (allow & 1) && ((uintptr_t)bytes & 15) == 0 && cudaPointerGetAttributes(&pa, bytes) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer)
        *direct_in = (const uint8_t*)pa.devicePointer;
    if (big && out_bytes && (allow & 2) && ((uintptr_t)out_bytes & 15) == 0 && cudaPointerGetAttributes(&pa, out_bytes) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer)
        *direct_out = (uint8_t*)pa.devicePointer;
    cudaGetLastError();                 // (cudaPointerGetAttributes on an unregistered pointer may leave an error behind)
}

// The step is cut at segment boundaries into slices so that whatever goes through the copy engines overlaps with the kernels:
// upload of slice k+1 | kernels of slice k | download of slice k-1 (PCIe is full duplex).   LGW_SLICES = 1..14
static uint32_t choose_slices(const lgw_engine* e, uint64_t n_bytes, uint32_t n_segs, bool all_direct) {
    uint32_t n_slices = n_bytes >= (8u << 20) && n_segs >= 16 ? 8u : 1u;
    if (all_direct) n_slices = 1;
    if (const char* sl = getenv("LGW_SLICES")) { int v = atoi(sl); if (v >= 1 && v <= 14) n_slices = (uint32_t)v; }
    if (e->mode == 1) n_slices = 1;
    return n_slices;
}

// LGW_TRACE = 1: the slice timeline of the step that just ran.  A slice without segments ran nothing and prints -1.
static void print_trace(lgw_engine* e, bool direct_in, bool direct_out, const uint32_t* cut, uint32_t n_slices) {
    cudaDeviceSynchronize();
    fprintf(stderr, "[lgw trace] direct_in=%d direct_out=%d slices=%u total=%.3f ms; per slice (ms after step start): upload done | kernels done | download done\n", direct_in, direct_out, n_slices, e->step.ms[4]);
    for (uint32_t j = 0; j < n_slices; ++j) {
        float ms[3] = {-1, -1, -1};
        if (cut[j + 1] > cut[j] || n_slices == 1) for (int k = 0; k < 3; ++k) read_ms(e->step.ev[5], e->step.tr[k][j], ms[k]);
        fprintf(stderr, "[lgw trace]   %2u  %.3f | %.3f | %.3f\n", j, ms[0], ms[1], ms[2]);
    }
    cudaGetLastError();
}

extern "C" int lgw_sse_step(lgw_engine* e, const uint8_t* bytes, uint64_t n_bytes, const uint32_t* chunk_off, uint32_t n_chunks,
                            const uint32_t* seg_chunk, const uint32_t* seg_slot, uint32_t n_segs,
                            uint8_t* out_bytes, lgw_seg_result* seg_out, lgw_row_event* rows_out, uint32_t rows_cap, uint32_t* n_rows) {
    if (!e || (!bytes && n_bytes) || !chunk_off || !seg_chunk || !seg_slot || !seg_out || !n_rows) return LGW_ERR_ARG;
    // out_bytes == NULL: the caller relays its own copy of the chunk bytes (the relayed bytes ARE the original bytes, request_handler.py:141-142);
    // the kernels run unchanged (the re-emit lands in the device staging buffer), only the download of the bytes is left out
    TRY(check_step_limits(e, n_segs, n_chunks, n_bytes));
    TRY(check_step_layout(e, n_bytes, chunk_off, n_chunks, seg_chunk, seg_slot, n_segs));
    lgw_engine::Step& st = e->step;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaEventRecord(st.ev[5], e->stream));
    static const bool trace = [] { const char* v = getenv("LGW_TRACE"); return v && v[0] == '1'; }();
    const uint8_t* direct_in; uint8_t* direct_out;
    probe_direct(e, bytes, out_bytes, n_bytes, &direct_in, &direct_out);
    st.last_direct = direct_in || direct_out;
    const StepArrays dev{direct_in ? direct_in : st.d_in, n_bytes, st.d_chunk_off, n_chunks, st.d_seg_chunk, st.d_seg_slot, n_segs,
                         direct_out ? direct_out : st.d_out, st.d_seg_out};
    remember_step(e, dev);
    uint32_t cut[18];
    const uint32_t n_slices = step_slice_cuts(n_bytes, chunk_off, seg_chunk, n_segs, choose_slices(e, n_bytes, n_segs, direct_in && direct_out), cut);
    CK(e, cudaMemsetAsync(e->d_rowq_count, 0, 4, e->stream));
    const bool piped = n_slices > 1;
    cudaStream_t sin = piped ? e->s_in : e->stream, sout = piped ? e->s_out : e->stream;
    if (piped) { CK(e, cudaEventRecord(st.ev_k[15], e->stream)); CK(e, cudaStreamWaitEvent(sin, st.ev_k[15], 0)); }   // the copy stream starts after ev[5]
    // offsets and segment tables: slice 0's part first (its kernels can start), everything else in one batch right behind it
    CK(e, cudaMemcpyAsync(st.d_chunk_off, chunk_off, (size_t)(seg_chunk[cut[1]] + 1) * 4, cudaMemcpyHostToDevice, sin));
    CK(e, cudaMemcpyAsync(st.d_seg_chunk, seg_chunk, (size_t)(n_segs + 1) * 4, cudaMemcpyHostToDevice, sin));
    if (n_segs) CK(e, cudaMemcpyAsync(st.d_seg_slot, seg_slot, (size_t)n_segs * 4, cudaMemcpyHostToDevice, sin));
    if (trace && !st.tr[0][0]) CK(e, new_events(e, &st.tr[0][0], 3 * 16));
    for (uint32_t j = 0; j < n_slices; ++j) {
        const uint32_t s0 = cut[j], s1 = cut[j + 1];
        if (s1 <= s0 && piped) continue;
        const uint32_t c0 = seg_chunk[s0], c1 = seg_chunk[s1];
        const uint32_t b0 = chunk_off[c0]; const uint64_t b1 = chunk_off[c1];
        if (!direct_in && b1 > b0) CK(e, cudaMemcpyAsync(st.d_in + b0, bytes + b0, b1 - b0, cudaMemcpyHostToDevice, sin));
        if (piped && (j == 0 || !direct_in)) { CK(e, cudaEventRecord(st.ev_in[j], sin)); CK(e, cudaStreamWaitEvent(e->stream, st.ev_in[j], 0)); }
        if (trace) cudaEventRecord(st.tr[0][j], sin);
        if (j == 0 && n_slices > 1 && n_chunks > seg_chunk[cut[1]]) {      // the rest of the chunk offsets, while slice 0 is at work
            const uint32_t cc = seg_chunk[cut[1]];
            CK(e, cudaMemcpyAsync(st.d_chunk_off + cc + 1, chunk_off + cc + 1, (size_t)(n_chunks - cc) * 4, cudaMemcpyHostToDevice, sin));
            if (direct_in) { CK(e, cudaEventRecord(st.ev_in[1], sin)); CK(e, cudaStreamWaitEvent(e->stream, st.ev_in[1], 0)); }
        }
        TRY(step_device(e, dev, StepSlice{s0, s1, c0, c1, b0, b1}, false));
        if (trace) cudaEventRecord(st.tr[1][j], e->stream);
        if (!direct_out) {
            if (piped) { CK(e, cudaEventRecord(st.ev_k[j], e->stream)); CK(e, cudaStreamWaitEvent(sout, st.ev_k[j], 0)); }
            if (b1 > b0 && out_bytes) CK(e, cudaMemcpyAsync(out_bytes + b0, st.d_out + b0, b1 - b0, cudaMemcpyDeviceToHost, sout));
        }
        if (trace) cudaEventRecord(st.tr[2][j], sout);
    }
    // per-segment results: one copy at the end (a copy into pageable host memory blocks the host thread,
    // which would serialise the pipeline if it were issued per slice)
    if (n_segs) CK(e, cudaMemcpyAsync(seg_out, st.d_seg_out, (size_t)n_segs * sizeof(SegResult), cudaMemcpyDeviceToHost, e->stream));
    if (piped) {                            // ev[6] closes the step on the engine stream: it has to see the downloads too
        CK(e, cudaEventRecord(st.ev_k[14], sout)); CK(e, cudaStreamWaitEvent(e->stream, st.ev_k[14], 0));
        CK(e, cudaEventRecord(st.ev_in[15], sin)); CK(e, cudaStreamWaitEvent(e->stream, st.ev_in[15], 0));
    }
    CK(e, cudaEventRecord(st.ev[6], e->stream));
    TRY(lgw_fetch_rows(e, rows_out, rows_cap, n_rows));
    if (piped) { CK(e, cudaStreamSynchronize(e->s_out)); CK(e, cudaStreamSynchronize(e->s_in)); }
    read_ms(st.ev[5], st.ev[6], st.ms[4]);
    if (trace) print_trace(e, direct_in != nullptr, direct_out != nullptr, cut, n_slices);
    return LGW_OK;
}

static int read_step_ms(lgw_engine* e) {
    lgw_engine::Step& st = e->step;
    if (st.timed) {
        CK(e, cudaSetDevice(e->device));
        CK(e, cudaEventSynchronize(st.ev[4]));
        if (st.kernel_times_valid) {
            for (int i = 0; i < 4; ++i) read_ms(st.ev[i], st.ev[i + 1], st.ms[i]);
        } else {                            // kernels overlap (programmatic dependent launch): only their total is meaningful
            st.ms[0] = st.ms[2] = st.ms[3] = 0;
            read_ms(st.ev[0], st.ev[4], st.ms[1]);
        }
    }
    return LGW_OK;
}
extern "C" int lgw_last_step_ms(lgw_engine* e, float ms[4]) {
    if (!e || !ms) return LGW_ERR_ARG;
    TRY(read_step_ms(e));
    ms[0] = e->step.ms[0]; ms[1] = e->step.ms[1]; ms[2] = e->step.ms[2] + e->step.ms[3]; ms[3] = e->step.ms[4];
    return LGW_OK;
}
extern "C" int lgw_last_step_kernel_ms(lgw_engine* e, float ms[4]) {
    if (!e || !ms) return LGW_ERR_ARG;
    TRY(read_step_ms(e));
    for (int i = 0; i < 4; ++i) ms[i] = e->step.ms[i];
    return LGW_OK;
}

extern "C" int lgw_last_step_direct(lgw_engine* e) { return e && e->step.last_direct ? 1 : 0; }

extern "C" int lgw_launch_count(lgw_engine* e, uint64_t* out) {
    if (!e || !out) return LGW_ERR_ARG;
    *out = e->launches;
    return LGW_OK;
}

// Page-locked host memory is the caller's until lgw_free_pinned: the engine keeps no record of it.
extern "C" int lgw_alloc_pinned(lgw_engine* e, uint64_t bytes, void** out) {
    if (!e || !out) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    return LGW_OK;
}
extern "C" int lgw_free_pinned(lgw_engine* e, void* p) {
    if (!e) return LGW_ERR_ARG;
    CK(e, cudaFreeHost(p));
    return LGW_OK;
}

// ---- usage-stats rollup ----------------------------------------------------------------------------
extern "C" int64_t lgw_rollup_bucket_of(int64_t ts_us, int period) { return bucket_of(ts_us, period); }
extern "C" int lgw_rollup_buckets_of(const int64_t* ts_us, uint64_t n, int period, int64_t* out) {
    if ((n && (!ts_us || !out)) || period < 0 || period > 3) return LGW_ERR_ARG;
    for (uint64_t i = 0; i < n; ++i) out[i] = bucket_of(ts_us[i], period);
    return LGW_OK;
}

extern "C" int lgw_usage_rollup_accum(lgw_engine* e, const int64_t* d_ts_us, const int32_t* d_model_rank,
                                      const int32_t* d_prompt, const int32_t* d_completion, const int32_t* d_total,
                                      const int32_t* d_reasoning, const int32_t* d_cached, const double* d_cost, uint64_t n,
                                      int period, int has_start, int64_t start_us, int has_end, int64_t end_us,
                                      int64_t bucket0, uint32_t n_buckets, uint32_t n_models,
                                      uint64_t* d_table, uint32_t* d_inexact, uint32_t* d_oob) {
    if (!e || !d_table || !d_inexact || !d_oob || period < 0 || period > 3 || n_buckets == 0 || n_models == 0) return LGW_ERR_ARG;
    if (n && (!d_ts_us || !d_model_rank || !d_prompt || !d_completion || !d_total || !d_reasoning || !d_cached || !d_cost)) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    lgw_engine::Rollup& ru = e->rollup;
    RollupArgs a{};
    a.ts_us = d_ts_us; a.model_rank = d_model_rank; a.tok[0] = d_prompt; a.tok[1] = d_completion; a.tok[2] = d_total;
    a.tok[3] = d_reasoning; a.tok[4] = d_cached; a.cost = d_cost; a.n = n; a.period = period;
    a.start_us = start_us; a.end_us = end_us; a.has_start = has_start; a.has_end = has_end;
    a.bucket0 = bucket0; a.n_buckets = n_buckets; a.n_models = n_models;
    a.table = (unsigned long long*)d_table; a.inexact = d_inexact; a.oob = d_oob;
    const uint64_t groups = (uint64_t)n_buckets * n_models;
    const bool privatised = groups <= LGW_ROLLUP_SMEM_GROUPS && n >= 65536 && n < 0xFFFFFFFFull && !ru.force_global;
    if (privatised) {                     // scratch for the per-block partial tables (allocated outside the timed region)
        CK(e, ru.partial.reserve((size_t)e->sm_count * groups * (LGW_ROLLUP_CELLS * 8 + 4)));
        if (!ru.attr_set) {
            CK(e, cudaFuncSetAttribute(k_rollup_accum_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rollup_smem_bytes(LGW_ROLLUP_SMEM_GROUPS)));
            ru.attr_set = true;
        }
    }
    CK(e, cudaEventRecord(ru.ev[0], e->stream));
    if (n && privatised) {
        const unsigned grid = (unsigned)e->sm_count;
        unsigned long long* partial = ru.partial.as<unsigned long long>();
        uint32_t* pflag = (uint32_t*)(ru.partial.as<uint8_t>() + (size_t)grid * groups * LGW_ROLLUP_CELLS * 8);
        k_rollup_accum_smem<<<grid, 1024, rollup_smem_bytes((uint32_t)groups), e->stream>>>(a, partial, pflag);
        k_rollup_merge<<<dim3((unsigned)((groups * LGW_ROLLUP_CELLS + 255) / 256), LGW_ROLLUP_MERGE_SLICES), 256, 0, e->stream>>>(partial, pflag, grid, (uint32_t)groups, a.table, a.inexact);
        e->launches += 2;
    } else if (n) {
        k_rollup_accum<<<grid_for(e, n, 256, 16), 256, 0, e->stream>>>(a);
        ++e->launches;
    }
    CK(e, cudaEventRecord(ru.ev[1], e->stream));
    CK(e, cudaGetLastError());
    return LGW_OK;
}

extern "C" int lgw_usage_rollup_emit(lgw_engine* e, const uint64_t* d_table, const uint32_t* d_inexact,
                                     int64_t bucket0, uint32_t n_buckets, uint32_t n_models,
                                     lgw_rollup_row* rows_out, uint64_t rows_cap, uint64_t* n_rows) {
    if (!e || !d_table || !d_inexact || !n_rows || (!rows_out && rows_cap) || n_buckets == 0 || n_models == 0) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    lgw_engine::Rollup& ru = e->rollup;
    const uint64_t groups = (uint64_t)n_buckets * n_models;
    const uint64_t cap = rows_cap < groups ? rows_cap : groups;
    CK(e, ru.rows.reserve(cap * sizeof(RollupRow)));
    if (!ru.d_nrows) CK(e, dev_alloc(e, ru.d_nrows, 8));
    const uint32_t n_tiles = (uint32_t)((groups + 1023) / 1024);
    CK(e, ru.tiles.reserve((size_t)n_tiles * 4));
    CK(e, cudaEventRecord(ru.ev[2], e->stream));
    k_rollup_count<<<n_tiles, 1024, 0, e->stream>>>((const unsigned long long*)d_table, n_buckets, n_models, ru.tiles.as<uint32_t>());
    k_rollup_scan<<<1, 1024, 0, e->stream>>>(ru.tiles.as<uint32_t>(), n_tiles, ru.d_nrows);
    k_rollup_write<<<n_tiles, 1024, 0, e->stream>>>((const unsigned long long*)d_table, d_inexact, n_buckets, n_models, bucket0, ru.tiles.as<uint32_t>(), ru.rows.as<RollupRow>(), cap);
    e->launches += 3;
    CK(e, cudaEventRecord(ru.ev[3], e->stream));
    CK(e, cudaGetLastError());
    unsigned long long cnt = 0;
    CK(e, cudaMemcpyAsync(&cnt, ru.d_nrows, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    *n_rows = cnt;
    const uint64_t take = cnt < cap ? cnt : cap;
    if (take) CK(e, cudaMemcpyAsync(rows_out, ru.rows.p, take * sizeof(RollupRow), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

extern "C" int lgw_rollup_set_path(lgw_engine* e, int force_global) {   // 0 (default): privatised when the table fits; 1: global reductions only
    if (!e) return LGW_ERR_ARG;
    e->rollup.force_global = force_global != 0;
    return LGW_OK;
}

extern "C" int lgw_rollup_last_ms(lgw_engine* e, float ms[2]) {
    if (!e || !ms) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    lgw_engine::Rollup& ru = e->rollup;
    cudaEventSynchronize(ru.ev[1]); cudaEventSynchronize(ru.ev[3]);
    read_ms(ru.ev[0], ru.ev[1], ru.ms[0]);
    read_ms(ru.ev[2], ru.ev[3], ru.ms[1]);
    ms[0] = ru.ms[0]; ms[1] = ru.ms[1];
    return LGW_OK;
}

// ---- record listing (SURVEY.md 8(f) rank 2; tokens_usage_db.py:69-117) --------------------------------------------------------
extern "C" int lgw_usage_latest(lgw_engine* e, const int64_t* d_ts_us, uint64_t n, uint64_t first, uint64_t count, uint64_t* idx_out) {
    if (!e || n >= (1ull << 32) || count > n || first > n - count) return LGW_ERR_ARG;
    if (count && (!d_ts_us || !idx_out || ((uintptr_t)d_ts_us & 15))) return LGW_ERR_ARG;
    lgw_engine::Listing& li = e->listing;
    li.ms = 0;
    if (!count) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    const uint32_t N = (uint32_t)n, M = (uint32_t)count, cap = N / LGW_LIST_CAND_DIV;
    const uint32_t ctiles = (N + LGW_LIST_CTILE - 1) / LGW_LIST_CTILE, stiles = (M + LGW_LIST_STILE - 1) / LGW_LIST_STILE;
    const size_t scan_n = ctiles > 256ull * stiles ? ctiles : 256ull * stiles;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t o_cand = al(sizeof(ListSel)), o_keys = o_cand + al((size_t)(cap ? cap : 1) * sizeof(ListPair));
    const size_t o_idx = o_keys + al((size_t)M * 16), o_out = o_idx + al((size_t)M * 8), o_scan = o_out + al((size_t)M * 8);
    CK(e, li.buf.reserve(o_scan + al((scan_n + 257) * 4)));
    if (!li.ev[0]) CK(e, new_events(e, li.ev, 2));
    if (!li.attr_set) {
        CK(e, cudaFuncSetAttribute(k_list_sort_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(LGW_LIST_SMEM_SORT * 12)));
        li.attr_set = true;
    }
    uint8_t* l_buf = li.buf.as<uint8_t>();
    ListSel* sel = (ListSel*)l_buf;
    ListPair* cand = (ListPair*)(l_buf + o_cand);
    uint64_t* keys[2] = {(uint64_t*)(l_buf + o_keys), (uint64_t*)(l_buf + o_keys) + M};
    uint32_t* idx[2] = {(uint32_t*)(l_buf + o_idx), (uint32_t*)(l_buf + o_idx) + M};
    uint64_t* out = (uint64_t*)(l_buf + o_out);
    uint32_t* scan = (uint32_t*)(l_buf + o_scan);
    uint32_t* totals = scan + scan_n;                   // [256] column totals of the LSD scans
    uint32_t* selected = totals + 256;                  // records between the two boundaries (== count)
    const unsigned grid = grid_for(e, ((uint64_t)N + 1) / 2, 256, 8);
    CK(e, cudaEventRecord(li.ev[0], e->stream));
    k_list_init<<<1, 256, 0, e->stream>>>(sel, first, first + count - 1);
    for (int d = 0; d < LGW_LIST_DIGITS; ++d) {
        k_list_hist<<<grid, 256, 0, e->stream>>>(d_ts_us, N, cand, sel, d);
        k_list_pick<<<1, 256, 0, e->stream>>>(sel, d, cap);
        if (d + 1 < LGW_LIST_DIGITS) k_list_cand<<<grid, 256, 0, e->stream>>>(d_ts_us, N, cand, sel, d + 1);
    }
    k_list_tile_count<<<ctiles, 1024, 0, e->stream>>>(d_ts_us, N, sel, scan);
    k_list_scan<<<1, 1024, 0, e->stream>>>(scan, ctiles, selected);
    k_list_tile_write<<<ctiles, 1024, 0, e->stream>>>(d_ts_us, N, sel, scan, M, keys[0], idx[0]);
    e->launches += 1 + 3 * LGW_LIST_DIGITS - 1 + 3;
    if (M <= LGW_LIST_SMEM_SORT) {
        uint32_t p = 1;
        while (p < M) p <<= 1;
        k_list_sort_small<<<1, 1024, (size_t)p * 12, e->stream>>>(keys[0], idx[0], M, out);
        ++e->launches;
    } else {
        int cur = 0;
        for (int shift = 0; shift < 64; shift += 8, cur ^= 1) {
            k_lsd_hist<<<stiles, 256, 0, e->stream>>>(keys[cur], M, shift, scan, stiles);
            k_list_scan<<<256, 1024, 0, e->stream>>>(scan, stiles, totals);
            k_lsd_scatter<<<stiles, 256, 0, e->stream>>>(keys[cur], idx[cur], M, shift, scan, totals, stiles, keys[cur ^ 1], idx[cur ^ 1]);
        }
        k_list_widen<<<grid_for(e, M, 256, 8), 256, 0, e->stream>>>(idx[cur], M, out);
        e->launches += 8 * 3 + 1;
    }
    CK(e, cudaEventRecord(li.ev[1], e->stream));
    CK(e, cudaGetLastError());
    uint32_t got = 0;
    CK(e, cudaMemcpyAsync(idx_out, out, (size_t)M * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(&got, selected, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(li.ev[0], li.ev[1], li.ms);
    if (got != M) { e->err = "usage listing: " + std::to_string(got) + " records between the boundary keys, expected " + std::to_string(M); return LGW_ERR_CUDA; }
    return LGW_OK;
}

extern "C" int lgw_usage_latest_last_ms(lgw_engine* e, float* ms) {
    if (!e || !ms) return LGW_ERR_ARG;
    *ms = e->listing.ms;
    return LGW_OK;
}

// ---- deleting old records (tokens_usage_db.py:164-198) ---------------------------------------------------------------------------
extern "C" int lgw_usage_retain(lgw_engine* e, void* const d_in[8], void* const d_out[8], uint64_t n, int64_t cutoff_us, uint64_t n_keep) {
    if (!e || n >= (1ull << 32) || n_keep > n) return LGW_ERR_ARG;
    if (n && (!d_in || !d_out)) return LGW_ERR_ARG;
    for (int c = 0; n && c < 8; ++c) if (!d_in[c] || (n_keep && !d_out[c])) return LGW_ERR_ARG;
    if (n && ((uintptr_t)d_in[0] & 15)) return LGW_ERR_ARG;
    lgw_engine::Retain& rt = e->retain;
    rt.ms = 0;
    if (!n) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    const uint32_t N = (uint32_t)n, tiles = (N + LGW_LIST_CTILE - 1) / LGW_LIST_CTILE;
    CK(e, rt.tiles.reserve(((size_t)tiles + 1) * 4));
    if (!rt.ev[0]) CK(e, new_events(e, rt.ev, 2));
    uint32_t* off = rt.tiles.as<uint32_t>();
    uint32_t* total = off + tiles;
    RetainCols in{(int64_t*)d_in[0], {}, (double*)d_in[7]}, out{(int64_t*)d_out[0], {}, (double*)d_out[7]};
    for (int c = 0; c < 6; ++c) { in.i32[c] = (int32_t*)d_in[1 + c]; out.i32[c] = (int32_t*)d_out[1 + c]; }
    CK(e, cudaEventRecord(rt.ev[0], e->stream));
    k_retain_count<<<tiles, 1024, 0, e->stream>>>(in.ts, N, cutoff_us, off);
    k_list_scan<<<1, 1024, 0, e->stream>>>(off, tiles, total);
    k_retain_write<<<tiles, 1024, 0, e->stream>>>(in, N, cutoff_us, off, (uint32_t)n_keep, out);
    e->launches += 3;
    CK(e, cudaEventRecord(rt.ev[1], e->stream));
    CK(e, cudaGetLastError());
    uint32_t got = 0;
    CK(e, cudaMemcpyAsync(&got, total, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(rt.ev[0], rt.ev[1], rt.ms);
    if (got != n_keep) { e->err = "usage retain: " + std::to_string(got) + " records at or after the cutoff, expected " + std::to_string(n_keep); return LGW_ERR_CUDA; }
    return LGW_OK;
}

extern "C" int lgw_usage_retain_last_ms(lgw_engine* e, float* ms) {
    if (!e || !ms) return LGW_ERR_ARG;
    *ms = e->retain.ms;
    return LGW_OK;
}

// ---- inserted records (tokens_usage_db.py:119-162) -------------------------------------------------------------------------------
extern "C" int lgw_usage_append(lgw_engine* e, void* const d_cols[8], void* const d_grow[8], uint64_t n,
                                const void* const h_new[8], uint64_t m, const int32_t* rank_map, uint32_t n_map) {
    if (!e || n >= (1ull << 32) || m >= (1ull << 32) || n + m >= (1ull << 32) || (rank_map && n_map == 0)) return LGW_ERR_ARG;
    const bool grow = d_grow != nullptr, remap = rank_map != nullptr;
    const uint64_t old = (grow || remap) ? n : 0;
    const bool need_cols = old > 0 || (!grow && m > 0);            // d_cols is read, or written in place
    if (need_cols) {
        if (!d_cols) return LGW_ERR_ARG;
        for (int c = 0; c < 8; ++c) if (!d_cols[c]) return LGW_ERR_ARG;
        if ((uintptr_t)d_cols[0] & 15) return LGW_ERR_ARG;
    }
    if (grow && old + m > 0) {
        for (int c = 0; c < 8; ++c) if (!d_grow[c]) return LGW_ERR_ARG;
        if ((uintptr_t)d_grow[0] & 15) return LGW_ERR_ARG;
    }
    if (m && !h_new) return LGW_ERR_ARG;
    for (int c = 0; m && c < 8; ++c) if (!h_new[c]) return LGW_ERR_ARG;
    lgw_engine::Append& ap = e->append;
    ap.ms = 0;
    if (old + m == 0) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    // staging: m timestamps, m costs, the six int32 columns, the map, the bad-rank counter (zero, copied up with the rest)
    const size_t o_cost = 8 * m, o_i32 = 16 * m, o_map = 40 * m, o_bad = o_map + (remap ? 4ull * n_map : 0), bytes = o_bad + 4;
    CK(e, ap.host.reserve(bytes, bytes / 4 + 4096));
    CK(e, ap.dev.reserve(bytes, bytes / 4 + 4096));
    if (!ap.ev[0]) CK(e, new_events(e, ap.ev, 2));
    uint8_t* st = ap.host.as<uint8_t>();
    if (m) {
        memcpy(st, h_new[0], 8 * m);
        memcpy(st + o_cost, h_new[7], 8 * m);
        for (int c = 0; c < 6; ++c) memcpy(st + o_i32 + 4 * m * c, h_new[1 + c], 4 * m);
    }
    if (remap) memcpy(st + o_map, rank_map, 4ull * n_map);
    memset(st + o_bad, 0, 4);
    uint8_t* dv = ap.dev.as<uint8_t>();
    void* const* dst = grow ? d_grow : d_cols;
    AppendArgs a{};
    if (need_cols) {
        a.src.ts = (int64_t*)d_cols[0]; a.src.cost = (double*)d_cols[7];
        for (int c = 0; c < 6; ++c) a.src.i32[c] = (int32_t*)d_cols[1 + c];
    }
    a.dst.ts = (int64_t*)dst[0]; a.dst.cost = (double*)dst[7];
    for (int c = 0; c < 6; ++c) a.dst.i32[c] = (int32_t*)dst[1 + c];
    if (!grow) a.src = a.dst;
    a.new_ts = (const int64_t*)dv; a.new_cost = (const double*)(dv + o_cost); a.new_i32 = (const int32_t*)(dv + o_i32);
    a.map = remap ? (const int32_t*)(dv + o_map) : nullptr;
    a.n_map = remap ? n_map : 0; a.n = (uint32_t)n; a.m = (uint32_t)m; a.old = (uint32_t)old;
    a.bad = (uint32_t*)(dv + o_bad);
    CK(e, cudaEventRecord(ap.ev[0], e->stream));
    CK(e, cudaMemcpyAsync(dv, st, bytes, cudaMemcpyHostToDevice, e->stream));
    k_usage_append<<<grid_for(e, old + m, 256, 8), 256, 0, e->stream>>>(a);
    ++e->launches;
    CK(e, cudaEventRecord(ap.ev[1], e->stream));
    CK(e, cudaGetLastError());
    uint32_t bad = 0;
    CK(e, cudaMemcpyAsync(&bad, a.bad, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(ap.ev[0], ap.ev[1], ap.ms);
    if (bad) { e->err = "usage append: " + std::to_string(bad) + " resident model ranks at or past the map's " + std::to_string(n_map) + " entries"; return LGW_ERR_CUDA; }
    return LGW_OK;
}

extern "C" int lgw_usage_append_last_ms(lgw_engine* e, float* ms) {
    if (!e || !ms) return LGW_ERR_ARG;
    *ms = e->append.ms;
    return LGW_OK;
}

// ---- loading the usage table from a tokens_usage file (tokens_usage_db.py:37-50) -----------------------------------------------
// Consecutive 256-byte aligned pieces of one buffer: take(bytes) hands out the next one (base null: only counts).
struct Carve {
    uint8_t* base; size_t used = 0;
    template <class T> T* take(size_t bytes) { T* p = (T*)(base ? base + used : nullptr); used += (bytes + 255) & ~(size_t)255; return p; }
};

// lgw_usage_load_finish's part of `out`: {ids, provider codes, refused ids, end}, after the tile offsets of k_load_mark; each
// sized for all n records, so that mark reserves it once and finish never moves the offsets
static std::array<size_t, 4> load_out_layout(uint32_t tiles, size_t n) {
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    const size_t o_ids = al(4ull * tiles + 16), o_prov = o_ids + al(8 * n), o_ref = o_prov + al(4 * n);
    return {o_ids, o_prov, o_ref, o_ref + 8 * n + 8};
}

static void carve_recs(Carve& c, LoadRecs& r, size_t n) {
    r.id = c.take<int64_t>(8 * n); r.ts = c.take<int64_t>(8 * n); r.cost = c.take<double>(8 * n);
    for (int k = 0; k < 5; ++k) r.tok[k] = c.take<int32_t>(4 * n);
    r.status = c.take<uint32_t>(4 * n); r.cell = c.take<CellRef>(sizeof(CellRef) * n);
    for (int f = 0; f < 2; ++f) { r.text[f] = c.take<TextRef>(sizeof(TextRef) * n); r.slot[f] = c.take<uint32_t>(4 * n); }
}

extern "C" int lgw_usage_load_decode(lgw_engine* e, const uint8_t* h_file, uint64_t n_bytes, uint32_t page_size, uint32_t n_pages, uint32_t root, uint64_t out[6]) {
    if (!e || !h_file || !out || page_size < 512 || page_size > 65536 || (page_size & (page_size - 1)) || n_pages == 0 ||
        (uint64_t)n_pages * page_size > n_bytes || n_bytes >= (1ull << 33)) return LGW_ERR_ARG;
    lgw_engine::Load& ld = e->load;
    ld.stage = 0;
    for (float& m : ld.ms) m = 0;
    CK(e, cudaSetDevice(e->device));
    const uint64_t bytes = (uint64_t)n_pages * page_size;
    CK(e, ld.file.reserve(bytes));
    if (!ld.ev[0]) CK(e, new_events(e, ld.ev, 8));
    // walk scratch: two levels and their counts (n_pages + 1 each), the visited bitmap, then kinds / error / total / codes / bytes
    const size_t lv = (size_t)n_pages + 1, words = n_pages / 32 + 1;
    Carve wc{nullptr};
    wc.take<uint32_t>(4 * lv); wc.take<uint32_t>(4 * lv); wc.take<uint32_t>(4 * lv); wc.take<uint32_t>(4 * words); wc.take<uint32_t>(64);
    CK(e, ld.walk.reserve(wc.used));
    Carve w{ld.walk.as<uint8_t>()};
    uint32_t* level[2] = {w.take<uint32_t>(4 * lv), w.take<uint32_t>(4 * lv)};
    uint32_t* cnt = w.take<uint32_t>(4 * lv);
    uint32_t* visited = w.take<uint32_t>(4 * words);
    uint32_t* ctr = w.take<uint32_t>(64);           // [0] kinds [1] error [2] total [3..4] codes, [6..9] name bytes (two u64)
    CK(e, cudaEventRecord(ld.ev[0], e->stream));
    CK(e, cudaMemcpyAsync(ld.file.p, h_file, bytes, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaEventRecord(ld.ev[1], e->stream));
    CK(e, cudaMemsetAsync(visited, 0, 4 * words, e->stream));
    CK(e, cudaMemsetAsync(ctr, 0, 64, e->stream));
    CK(e, cudaMemcpyAsync(level[0], &root, 4, cudaMemcpyHostToDevice, e->stream));
    const DbGeom g{ld.file.as<uint8_t>(), page_size, n_pages};
    ld.g = g;
    uint32_t m = 1, cur = 0, err = 0, seen = 1, host_ctr[3] = {0, 0, 0};
    for (uint32_t depth = 0;; ++depth) {           // one level a round; the host learns its kind and the next level's size
        if (depth == LGW_LOAD_MAX_DEPTH) { err = LOAD_BAD_TREE; break; }
        CK(e, cudaMemsetAsync(ctr, 0, 4, e->stream));
        k_load_count<<<grid_for(e, m, 256, 8), 256, 0, e->stream>>>(g, level[cur], m, cnt, visited, ctr, ctr + 1);
        k_list_scan<<<1, 1024, 0, e->stream>>>(cnt, m, ctr + 2);
        e->launches += 2;
        CK(e, cudaGetLastError());
        CK(e, cudaMemcpyAsync(host_ctr, ctr, 12, cudaMemcpyDeviceToHost, e->stream));
        CK(e, cudaStreamSynchronize(e->stream));
        err = host_ctr[1];
        if (err) break;
        if (host_ctr[0] == 3) { err = LOAD_BAD_TREE; break; }
        if (host_ctr[0] == 2) break;                 // the leaf level: cnt holds each leaf's first record
        seen += host_ctr[2];
        if (seen > n_pages) { err = LOAD_BAD_TREE; break; }
        k_load_children<<<grid_for(e, m, 1, 64), 128, 0, e->stream>>>(g, level[cur], m, cnt, level[cur ^ 1], ctr + 1);
        ++e->launches;
        m = host_ctr[2];
        cur ^= 1;
    }
    const uint32_t n = err ? 0 : host_ctr[2];
    // records and dictionaries: a table of at least 2n slots a field
    uint32_t cap = 64;
    while (cap < 2ull * n) cap <<= 1;
    Carve rc{nullptr};
    LoadRecs r{};
    carve_recs(rc, r, n);
    CK(e, ld.recs.reserve(rc.used));
    rc = Carve{ld.recs.as<uint8_t>()};
    carve_recs(rc, r, n);
    Carve dc{nullptr};
    for (int f = 0; f < 2; ++f) { dc.take<uint64_t>(8ull * cap); dc.take<uint32_t>(4ull * cap); dc.take<NameRef>(sizeof(NameRef) * (size_t)(n ? n : 1)); }
    CK(e, ld.dict.reserve(dc.used));
    dc = Carve{ld.dict.as<uint8_t>()};
    LoadDict d[2];
    for (int f = 0; f < 2; ++f) {
        d[f].table = dc.take<uint64_t>(8ull * cap); d[f].slot_code = dc.take<uint32_t>(4ull * cap);
        d[f].names = dc.take<NameRef>(sizeof(NameRef) * (size_t)(n ? n : 1)); d[f].cap = cap;
        d[f].n_codes = ctr + 3 + f; d[f].n_bytes = (unsigned long long*)(ctr + 6) + f;
        CK(e, cudaMemsetAsync(d[f].table, 0, 8ull * cap, e->stream));
    }
    if (n) {
        k_load_decode<<<grid_for(e, m, 1, 64), 128, 0, e->stream>>>(g, level[cur], m, cnt, r, ctr + 1);
        ++e->launches;
    }
    CK(e, cudaEventRecord(ld.ev[2], e->stream));
    if (n) {
        k_load_dict<<<grid_for(e, n, 256, 8), 256, 0, e->stream>>>(g, r, n, d[0], d[1], ctr + 1);
        ++e->launches;
    }
    CK(e, cudaEventRecord(ld.ev[3], e->stream));
    CK(e, cudaGetLastError());
    uint32_t res[10] = {};
    CK(e, cudaMemcpyAsync(res, ctr, 40, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(ld.ev[0], ld.ev[1], ld.ms[0]);
    read_ms(ld.ev[1], ld.ev[2], ld.ms[1]);
    read_ms(ld.ev[2], ld.ev[3], ld.ms[2]);
    if (!err) err = res[1];
    uint64_t nb[2];
    memcpy(nb, res + 6, 16);
    out[0] = err; out[1] = n; out[2] = res[3]; out[3] = res[4]; out[4] = nb[0]; out[5] = nb[1];
    ld.r = r; ld.d[0] = d[0]; ld.d[1] = d[1];
    ld.n = n; ld.n_names[0] = res[3]; ld.n_names[1] = res[4];
    if (err) return lgw_usage_load_release(e);
    ld.stage = 1;
    return LGW_OK;
}

extern "C" int lgw_usage_load_names(lgw_engine* e, const uint8_t* h_file, int field, uint8_t* buf, uint64_t* offs) {
    if (!e || !h_file || !offs || field < 0 || field > 1) return LGW_ERR_ARG;
    lgw_engine::Load& ld = e->load;
    if (ld.stage < 1) { e->err = "usage load: names before a decode"; return LGW_ERR_ARG; }
    const uint32_t k = ld.n_names[field];
    std::vector<NameRef> refs(k);
    CK(e, cudaSetDevice(e->device));
    if (k) CK(e, cudaMemcpyAsync(refs.data(), ld.d[field].names, k * sizeof(NameRef), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    const DbGeom hg{h_file, ld.g.ps, ld.g.n_pages};
    uint64_t at = 0;
    for (uint32_t c = 0; c < k; ++c) {
        offs[c] = at;
        text_copy(hg, refs[c].cell, refs[c].t, buf + at);
        at += refs[c].t.len;
    }
    offs[k] = at;
    return LGW_OK;
}

// the two maps into the device staging; refusals recorded (mark) or checked against mark's (finish)
static int load_maps(lgw_engine* e, const int32_t* model_map, const int32_t* prov_map, bool check, int32_t*& dm, int32_t*& dp) {
    lgw_engine::Load& ld = e->load;
    const int32_t* maps[2] = {model_map, prov_map};
    for (int f = 0; f < 2; ++f) {
        if (ld.n_names[f] && !maps[f]) return LGW_ERR_ARG;
        std::vector<uint8_t> ref(ld.n_names[f]);
        for (uint32_t c = 0; c < ld.n_names[f]; ++c) ref[c] = maps[f][c] < 0;
        if (check && ref != ld.refused[f]) { e->err = "usage load: the maps refuse other texts than at mark"; return LGW_ERR_ARG; }
        ld.refused[f] = std::move(ref);
    }
    const size_t n0 = ld.n_names[0], n1 = ld.n_names[1];
    CK(e, ld.maps.reserve(4 * (n0 + n1) + n0 + 16));
    dm = ld.maps.as<int32_t>();
    dp = dm + n0;
    if (n0) CK(e, cudaMemcpyAsync(dm, model_map, 4 * n0, cudaMemcpyHostToDevice, e->stream));
    if (n1) CK(e, cudaMemcpyAsync(dp, prov_map, 4 * n1, cudaMemcpyHostToDevice, e->stream));
    return LGW_OK;
}

extern "C" int lgw_usage_load_mark(lgw_engine* e, const int32_t* model_map, const int32_t* prov_map, uint8_t* model_used, uint64_t* n_keep) {
    if (!e || !n_keep || (e->load.n_names[0] && !model_used)) return LGW_ERR_ARG;
    lgw_engine::Load& ld = e->load;
    if (ld.stage < 1) { e->err = "usage load: mark before a decode"; return LGW_ERR_ARG; }
    CK(e, cudaSetDevice(e->device));
    int32_t *dm, *dp;
    TRY(load_maps(e, model_map, prov_map, false, dm, dp));
    const uint32_t n = ld.n, tiles = (n + LGW_LOAD_TILE - 1) / LGW_LOAD_TILE;
    uint8_t* used = (uint8_t*)(dp + ld.n_names[1]);
    CK(e, ld.out.reserve(load_out_layout(tiles, n)[3]));
    uint32_t* tile = ld.out.as<uint32_t>();
    CK(e, cudaMemsetAsync(used, 0, ld.n_names[0] + 1, e->stream));
    CK(e, cudaMemsetAsync(tile + tiles, 0, 4, e->stream));
    CK(e, cudaEventRecord(ld.ev[4], e->stream));
    if (tiles) {
        k_load_mark<<<tiles, 1024, 0, e->stream>>>(ld.r, n, ld.d[0].slot_code, ld.d[1].slot_code, dm, dp, used, tile);
        k_list_scan<<<1, 1024, 0, e->stream>>>(tile, tiles, tile + tiles);
        e->launches += 2;
    }
    CK(e, cudaEventRecord(ld.ev[5], e->stream));
    CK(e, cudaGetLastError());
    uint32_t kept = 0;
    CK(e, cudaMemcpyAsync(&kept, tile + tiles, 4, cudaMemcpyDeviceToHost, e->stream));
    if (ld.n_names[0]) CK(e, cudaMemcpyAsync(model_used, used, ld.n_names[0], cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    ld.n_keep = *n_keep = kept;
    ld.tiles = tiles;
    ld.stage = 2;
    return LGW_OK;
}

extern "C" int lgw_usage_load_finish(lgw_engine* e, const int32_t* model_map, const int32_t* prov_map, void* const d_cols[8], void* const h_cols[8],
                                     int64_t* h_ids, int32_t* h_prov, int64_t* h_refused) {
    if (!e) return LGW_ERR_ARG;
    lgw_engine::Load& ld = e->load;
    if (ld.stage != 2) { e->err = "usage load: finish before a mark"; return LGW_ERR_ARG; }
    const uint64_t n = ld.n, k = ld.n_keep;
    if (k && (!d_cols || !h_cols || !h_ids || !h_prov)) return LGW_ERR_ARG;
    for (int c = 0; k && c < 8; ++c) if (!d_cols[c] || !h_cols[c]) return LGW_ERR_ARG;
    if (n > k && !h_refused) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    int32_t *dm, *dp;
    TRY(load_maps(e, model_map, prov_map, true, dm, dp));
    const std::array<size_t, 4> lay = load_out_layout(ld.tiles, ld.n);          // (mark sized `out` for all of it)
    const size_t o_ids = lay[0], o_prov = lay[1], o_ref = lay[2];
    uint8_t* ob = ld.out.as<uint8_t>();
    LoadOut o{(int64_t*)(k ? d_cols[0] : nullptr), {}, (double*)(k ? d_cols[7] : nullptr), (int64_t*)(ob + o_ids), (int32_t*)(ob + o_prov), (int64_t*)(ob + o_ref)};
    for (int c = 0; c < 6; ++c) o.i32[c] = (int32_t*)(k ? d_cols[1 + c] : nullptr);
    CK(e, cudaEventRecord(ld.ev[6], e->stream));
    if (ld.tiles) {
        k_load_finish<<<ld.tiles, 1024, 0, e->stream>>>(ld.r, (uint32_t)n, ld.d[0].slot_code, ld.d[1].slot_code, dm, dp, ld.out.as<uint32_t>(), (uint32_t)k, o);
        ++e->launches;
    }
    CK(e, cudaEventRecord(ld.ev[7], e->stream));
    CK(e, cudaGetLastError());
    static const size_t width[8] = {8, 4, 4, 4, 4, 4, 4, 8};
    for (int c = 0; k && c < 8; ++c) CK(e, cudaMemcpyAsync(h_cols[c], d_cols[c], width[c] * k, cudaMemcpyDeviceToHost, e->stream));
    if (k) CK(e, cudaMemcpyAsync(h_ids, o.id, 8 * k, cudaMemcpyDeviceToHost, e->stream));
    if (k) CK(e, cudaMemcpyAsync(h_prov, o.prov, 4 * k, cudaMemcpyDeviceToHost, e->stream));
    if (n > k) CK(e, cudaMemcpyAsync(h_refused, o.refused, 8 * (n - k), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    float a = 0, b = 0;
    read_ms(ld.ev[4], ld.ev[5], a);
    read_ms(ld.ev[6], ld.ev[7], b);
    ld.ms[3] = a + b;
    return lgw_usage_load_release(e);
}

extern "C" int lgw_usage_load_release(lgw_engine* e) {
    if (!e) return LGW_ERR_ARG;
    lgw_engine::Load& ld = e->load;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    for (DevBuf* b : {&ld.file, &ld.walk, &ld.recs, &ld.dict, &ld.maps, &ld.out}) b->release();
    ld.stage = 0;
    ld.n = ld.n_names[0] = ld.n_names[1] = 0;
    ld.refused[0].clear(); ld.refused[1].clear();
    return LGW_OK;
}

extern "C" int lgw_usage_load_last_ms(lgw_engine* e, float ms[4]) {
    if (!e || !ms) return LGW_ERR_ARG;
    for (int k = 0; k < 4; ++k) ms[k] = e->load.ms[k];
    return LGW_OK;
}

// ---- saving the usage table as a tokens_usage file (save.cuh) ---------------------------------------------------------------
extern "C" int lgw_usage_save_plan(lgw_engine* e, void* const d_cols[8], uint64_t n, const int64_t* h_ids, const int32_t* h_prov,
                                   const lgw_save_text* models, const lgw_save_text* providers, uint32_t page_size, uint64_t out[5]) {
    if (!e || !out || !models || !providers || n >= (1ull << 32) || page_size < 1024 || page_size > 65536 || (page_size & (page_size - 1))) return LGW_ERR_ARG;
    if (n && (!d_cols || !h_ids || !h_prov)) return LGW_ERR_ARG;
    for (int c = 0; n && c < 8; ++c) if (!d_cols[c]) return LGW_ERR_ARG;
    if (n && ((uintptr_t)d_cols[0] & 15)) return LGW_ERR_ARG;
    const lgw_save_text* tx[2] = {models, providers};
    uint64_t blob[2];
    for (int f = 0; f < 2; ++f) {
        if (!tx[f]->n || !tx[f]->off || !tx[f]->len) return LGW_ERR_ARG;
        blob[f] = tx[f]->off[tx[f]->n];
        if (blob[f] && !tx[f]->blob) return LGW_ERR_ARG;
    }
    TRY(lgw_usage_save_release(e));
    lgw_engine::Save& sv = e->save;
    for (float& m : sv.ms) m = 0;
    if (!sv.ev[0]) CK(e, new_events(e, sv.ev, 8));
    const uint32_t N = (uint32_t)n, U = page_size, M = N ? N : 1;
    const uint32_t ktiles = (N + LGW_LOAD_TILE - 1) / LGW_LOAD_TILE;
    // inputs: ids, provider codes, the two text tables
    auto carve_in = [&](Carve& c, int64_t*& ids, int32_t*& prov, SaveText* t) {
        ids = c.take<int64_t>(8ull * N); prov = c.take<int32_t>(4ull * N);
        for (int f = 0; f < 2; ++f) {
            t[f].off = c.take<uint64_t>(8ull * (tx[f]->n + 1)); t[f].len = c.take<uint32_t>(4ull * tx[f]->n);
            t[f].blob = c.take<uint8_t>(blob[f]); t[f].n = tx[f]->n; t[f].pad = 0;
        }
    };
    int64_t* ids; int32_t* prov; SaveText t[2];
    Carve ic{nullptr};
    carve_in(ic, ids, prov, t);
    CK(e, sv.in.reserve(ic.used));
    ic = Carve{sv.in.as<uint8_t>()};
    carve_in(ic, ids, prov, t);
    // per record: kept record, table cell size, overflow pages, two sort keys and indices, refused ids; keep tiles; counters
    auto carve_recs = [&](Carve& c, uint32_t*& kidx, uint32_t*& lsz, uint32_t*& lov, uint64_t** key, uint32_t** idx, int64_t*& ref,
                          uint32_t*& tiles, unsigned long long*& ctr) {
        kidx = c.take<uint32_t>(4ull * M); lsz = c.take<uint32_t>(4ull * M); lov = c.take<uint32_t>(4ull * M);
        key[0] = c.take<uint64_t>(8ull * M); key[1] = c.take<uint64_t>(8ull * M);
        idx[0] = c.take<uint32_t>(4ull * M); idx[1] = c.take<uint32_t>(4ull * M);
        ref = c.take<int64_t>(8ull * M); tiles = c.take<uint32_t>(4ull * (ktiles + 1)); ctr = c.take<unsigned long long>(32);
    };
    uint32_t *kidx, *lsz, *lov, *idx[2], *tcount; uint64_t* key[2]; int64_t* refused; unsigned long long* ctr;
    Carve rc{nullptr};
    carve_recs(rc, kidx, lsz, lov, key, idx, refused, tcount, ctr);
    CK(e, sv.recs.reserve(rc.used));
    rc = Carve{sv.recs.as<uint8_t>()};
    carve_recs(rc, kidx, lsz, lov, key, idx, refused, tcount, ctr);
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaEventRecord(sv.ev[0], e->stream));
    if (N) CK(e, cudaMemcpyAsync(ids, h_ids, 8ull * N, cudaMemcpyHostToDevice, e->stream));
    if (N) CK(e, cudaMemcpyAsync(prov, h_prov, 4ull * N, cudaMemcpyHostToDevice, e->stream));
    for (int f = 0; f < 2; ++f) {
        CK(e, cudaMemcpyAsync((void*)t[f].off, tx[f]->off, 8ull * (tx[f]->n + 1), cudaMemcpyHostToDevice, e->stream));
        CK(e, cudaMemcpyAsync((void*)t[f].len, tx[f]->len, 4ull * tx[f]->n, cudaMemcpyHostToDevice, e->stream));
        if (blob[f]) CK(e, cudaMemcpyAsync((void*)t[f].blob, tx[f]->blob, blob[f], cudaMemcpyHostToDevice, e->stream));
    }
    CK(e, cudaEventRecord(sv.ev[1], e->stream));
    // 1. keep
    SaveIn in{};
    if (N) {
        in.ts = (const int64_t*)d_cols[0]; in.cost = (const double*)d_cols[7];
        for (int c = 0; c < 6; ++c) in.i32[c] = (const int32_t*)d_cols[1 + c];
    }
    in.id = ids; in.prov = prov; in.text[0] = t[0]; in.text[1] = t[1];
    CK(e, cudaMemsetAsync(ctr, 0xFF, 8, e->stream));
    CK(e, cudaMemsetAsync(ctr + 1, 0, 24, e->stream));
    CK(e, cudaMemsetAsync(tcount + ktiles, 0, 4, e->stream));
    if (ktiles) {
        k_save_count<<<ktiles, 1024, 0, e->stream>>>(in, N, tcount, ctr, ctr + 1, (uint32_t*)(ctr + 2));
        k_list_scan<<<1, 1024, 0, e->stream>>>(tcount, ktiles, tcount + ktiles);
        e->launches += 2;
    }
    CK(e, cudaGetLastError());
    unsigned long long res[3];
    uint32_t K = 0;
    CK(e, cudaMemcpyAsync(res, ctr, 24, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(&K, tcount + ktiles, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    if (res[2] & 2) { e->err = "usage save: a model rank or provider code outside its text table"; lgw_usage_save_release(e); return LGW_ERR_ARG; }
    if (res[2] & 1) { e->err = "usage save: ids not ascending in record order"; lgw_usage_save_release(e); return LGW_ERR_ARG; }
    if (ktiles) {
        k_save_keep<<<ktiles, 1024, 0, e->stream>>>(in, N, U, tcount, ctr, kidx, lsz, lov, key[0], idx[0], refused);
        ++e->launches;
    }
    CK(e, cudaEventRecord(sv.ev[2], e->stream));
    // 2. sort: the stable LSD passes over the digits the key range needs
    const uint64_t range = K ? res[1] - res[0] : 0;
    int bits = 0;
    while (bits < 64 && (range >> bits)) ++bits;
    const int passes = (bits + 7) / 8;
    const uint32_t stiles = (K + LGW_LIST_STILE - 1) / LGW_LIST_STILE;
    uint32_t cur = 0;
    if (passes && K > 1) {
        CK(e, sv.sort.reserve((256ull * stiles + 256) * 4));
        uint32_t* hist = sv.sort.as<uint32_t>();
        uint32_t* totals = hist + 256ull * stiles;
        for (int p = 0; p < passes; ++p) {
            k_lsd_hist<<<stiles, 256, 0, e->stream>>>(key[cur], K, 8 * p, hist, stiles);
            k_list_scan<<<256, 1024, 0, e->stream>>>(hist, stiles, totals);
            k_lsd_scatter<<<stiles, 256, 0, e->stream>>>(key[cur], idx[cur], K, 8 * p, hist, totals, stiles, key[cur ^ 1], idx[cur ^ 1]);
            e->launches += 3;
            cur ^= 1;
        }
    }
    CK(e, cudaEventRecord(sv.ev[3], e->stream));
    // 3. pack, level by level; the pool holds at most twice each tree's leaves (every interior page has two children or more)
    const uint32_t tile = save_tile(U), ptiles = pack_tiles(K, tile), pool_cap = 4 * M + 4 * LGW_SAVE_MAX_LEVELS;
    Carve pc{nullptr};
    for (int k = 0; k < 4; ++k) pc.take<uint32_t>(4ull * M);
    pc.take<uint32_t>(4ull * (ptiles + 1)); pc.take<uint32_t>(4ull * (ptiles + 1));
    CK(e, sv.pack.reserve(pc.used));
    pc = Carve{sv.pack.as<uint8_t>()};
    uint32_t *pstart = pc.take<uint32_t>(4ull * M), *pcnt = pc.take<uint32_t>(4ull * M), *isz_a = pc.take<uint32_t>(4ull * M), *isz_b = pc.take<uint32_t>(4ull * M);
    uint32_t *tpages = pc.take<uint32_t>(4ull * (ptiles + 1)), *tovfl = pc.take<uint32_t>(4ull * (ptiles + 1));
    CK(e, sv.pool.reserve((size_t)pool_cap * sizeof(PageDesc)));
    SaveCtx c{};
    c.in = in; c.U = U; c.kidx = kidx; c.sidx = idx[cur]; c.lsz = lsz; c.lov = lov; c.pool = sv.pool.as<PageDesc>(); c.lock = (1u << 30) / U + 1;
    uint32_t used = 0, n_ovfl = 0;
    for (uint32_t tree = 0; tree < 2; ++tree) {
        const uint32_t* isz = lsz;
        uint32_t* next = isz_a;
        if (tree == 1) {
            if (K) k_save_entry_sizes<<<grid_for(e, K, 256, 8), 256, 0, e->stream>>>(in, kidx, c.sidx, K, isz_a);
            isz = isz_a; next = isz_b;
        }
        uint32_t m = K, kind = tree ? SAVE_INDEX_LEAF : SAVE_TABLE_LEAF;
        for (uint32_t level = 0;; ++level) {
            if (level == LGW_SAVE_MAX_LEVELS) { e->err = "usage save: b-tree deeper than LGW_SAVE_MAX_LEVELS"; lgw_usage_save_release(e); return LGW_ERR_CAPACITY; }
            const uint32_t tiles = pack_tiles(m, tile);
            const bool ovfl = tree == 0 && level == 0;
            k_save_pack<<<(tiles + 127) / 128, 128, 0, e->stream>>>(isz, m, tiles, kind, U, pstart, pcnt, tpages, ovfl ? lov : nullptr, tovfl);
            k_list_scan<<<1, 1024, 0, e->stream>>>(tpages, tiles, tpages + tiles);
            if (ovfl) k_list_scan<<<1, 1024, 0, e->stream>>>(tovfl, tiles, tovfl + tiles);
            e->launches += 2 + ovfl;
            CK(e, cudaGetLastError());
            uint32_t P = 0;
            CK(e, cudaMemcpyAsync(&P, tpages + tiles, 4, cudaMemcpyDeviceToHost, e->stream));
            if (ovfl) CK(e, cudaMemcpyAsync(&n_ovfl, tovfl + tiles, 4, cudaMemcpyDeviceToHost, e->stream));
            CK(e, cudaStreamSynchronize(e->stream));
            if ((uint64_t)used + P > pool_cap) { e->err = "usage save: page pool overflow"; lgw_usage_save_release(e); return LGW_ERR_CUDA; }
            c.base[tree][level] = used;
            k_save_gather<<<grid_for(e, tiles, 1, 64), 128, 0, e->stream>>>(c, tree, level, m, tiles, tpages, pstart, pcnt, sv.pool.as<PageDesc>(), used, next);
            ++e->launches;
            used += P;
            if (P == 1) { c.levels[tree] = level + 1; c.base[tree][level + 1] = used; break; }
            m = tree ? P - 1 : P;
            kind = tree ? SAVE_INDEX_INTERIOR : SAVE_TABLE_INTERIOR;
            isz = next;
            next = next == isz_a ? isz_b : isz_a;
        }
    }
    const uint64_t laid = 2ull + used + n_ovfl, pages = laid + (laid >= c.lock);      // (the lock-byte page, unused)
    if (pages > 0xFFFFFFFEull) { e->err = "usage save: more pages than a SQLite file holds"; lgw_usage_save_release(e); return LGW_ERR_ARG; }
    if (K) k_save_ovfl_abs<<<grid_for(e, K, 256, 8), 256, 0, e->stream>>>(lov, K, ptiles, tile, tovfl, LGW_SAVE_POOL0 + used);
    CK(e, cudaEventRecord(sv.ev[4], e->stream));
    CK(e, cudaGetLastError());
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(sv.ev[0], sv.ev[1], sv.ms[0]);
    read_ms(sv.ev[1], sv.ev[2], sv.ms[1]);
    read_ms(sv.ev[2], sv.ev[3], sv.ms[2]);
    read_ms(sv.ev[3], sv.ev[4], sv.ms[3]);
    sv.c = c; sv.n = N; sv.kept = K; sv.n_pool = used; sv.n_ovfl = n_ovfl; sv.pages = (uint32_t)pages; sv.refused = refused; sv.stage = 1;
    out[0] = pages; out[1] = save_page(c, LGW_SAVE_POOL0 + c.base[0][c.levels[0] - 1]); out[2] = save_page(c, LGW_SAVE_POOL0 + c.base[1][c.levels[1] - 1]);
    out[3] = K; out[4] = N - K;
    return LGW_OK;
}

extern "C" int lgw_usage_save_write(lgw_engine* e, uint8_t* h_file, int64_t* h_refused) {
    if (!e) return LGW_ERR_ARG;
    lgw_engine::Save& sv = e->save;
    if (sv.stage != 1) { e->err = "usage save: write before a plan"; return LGW_ERR_ARG; }
    if (!h_file || (sv.n > sv.kept && !h_refused)) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    const uint32_t U = sv.c.U;
    const uint64_t bytes = (uint64_t)(sv.pages - 2) * U;
    CK(e, sv.img.reserve(bytes));
    if (sv.pages > sv.c.lock) CK(e, cudaMemsetAsync(sv.img.as<uint8_t>() + (uint64_t)(sv.c.lock - LGW_SAVE_POOL0) * U, 0, U, e->stream));
    CK(e, cudaFuncSetAttribute(k_save_pages, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)U));
    CK(e, cudaEventRecord(sv.ev[5], e->stream));
    k_save_pages<<<grid_for(e, sv.n_pool, 1, 16), 128, U, e->stream>>>(sv.c, sv.n_pool, sv.img.as<uint8_t>());
    ++e->launches;
    if (sv.n_ovfl) { k_save_chains<<<grid_for(e, sv.kept, 256, 8), 256, 0, e->stream>>>(sv.c, sv.kept, sv.img.as<uint8_t>()); ++e->launches; }
    CK(e, cudaEventRecord(sv.ev[6], e->stream));
    CK(e, cudaGetLastError());
    CK(e, cudaMemcpyAsync(h_file + 2ull * U, sv.img.p, bytes, cudaMemcpyDeviceToHost, e->stream));
    if (sv.n > sv.kept) CK(e, cudaMemcpyAsync(h_refused, sv.refused, 8ull * (sv.n - sv.kept), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaEventRecord(sv.ev[7], e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(sv.ev[5], sv.ev[6], sv.ms[4]);
    read_ms(sv.ev[6], sv.ev[7], sv.ms[5]);
    return lgw_usage_save_release(e);
}

extern "C" int lgw_usage_save_release(lgw_engine* e) {
    if (!e) return LGW_ERR_ARG;
    lgw_engine::Save& sv = e->save;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    for (DevBuf* b : {&sv.in, &sv.recs, &sv.sort, &sv.pack, &sv.pool, &sv.img}) b->release();
    sv.stage = 0;
    sv.n = sv.kept = sv.n_pool = sv.n_ovfl = sv.pages = 0;
    sv.refused = nullptr;
    return LGW_OK;
}

extern "C" int lgw_usage_save_last_ms(lgw_engine* e, float ms[6]) {
    if (!e || !ms) return LGW_ERR_ARG;
    for (int k = 0; k < 6; ++k) ms[k] = e->save.ms[k];
    return LGW_OK;
}

// ---- transcript tap (SURVEY.md 8(f) rank 3; chat_logging.py:108-139) ---------------------------------------------------------
extern "C" int lgw_transcripts_enable(lgw_engine* e) {
    if (!e) return LGW_ERR_ARG;
    lgw_engine::Text& tx = e->text;
    if (tx.on) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    const size_t S = e->lim.max_streams, C = e->lim.max_step_chunks, B = e->lim.max_step_bytes, cc = e->lim.carry_cap;
    CK(e, dev_alloc(e, tx.tap, S * sizeof(TextTap)));
    CK(e, cudaMemset(tx.tap, 0, S * sizeof(TextTap)));
    CK(e, dev_alloc(e, tx.carry, S * cc));
    CK(e, dev_alloc(e, tx.sparse, 2 * (B + S * cc) + 64));  // per segment: twice its carry and its bytes (content pieces + "error" event texts)
    CK(e, dev_alloc(e, tx.text, 2 * (B + S * cc) + 64));
    CK(e, dev_alloc(e, tx.piece_len, (C + 1) * 4));
    CK(e, dev_alloc(e, tx.seg_len, (S + 1) * 4));
    CK(e, dev_alloc(e, tx.seg_flags, (S + 1) * 4));
    CK(e, dev_alloc(e, tx.seg_off, (S + 2) * 8));
    CK(e, dev_alloc(e, tx.markq, (size_t)(e->lim.rowq_cap + 1) * sizeof(TextMark)));
    CK(e, dev_alloc(e, tx.markq_count, 16));
    CK(e, new_events(e, tx.ev, 2));
    tx.on = true;
    return LGW_OK;
}

extern "C" int lgw_step_transcript_run(lgw_engine* e, uint64_t* text_bytes, uint32_t* n_marks) {
    if (!e || !text_bytes || !n_marks) return LGW_ERR_ARG;
    lgw_engine::Text& tx = e->text;
    if (!tx.on) { e->err = "transcripts are not enabled (lgw_transcripts_enable)"; return LGW_ERR_ARG; }
    if (!tx.pending) { e->err = "no step to tap (the transcript pass runs once after each lgw_sse_step / lgw_sse_step_device)"; return LGW_ERR_ARG; }
    CK(e, cudaSetDevice(e->device));
    tx.pending = false;
    const StepArrays& s = e->step.last;
    TextArgs a{};
    a.data = s.bytes; a.chunk_off = s.chunk_off; a.seg_chunk = s.seg_chunk; a.seg_slot = s.seg_slot; a.n_segs = s.n_segs;
    a.seg_res = s.seg_out; a.tap = tx.tap; a.carry = tx.carry; a.carry_cap = e->lim.carry_cap; a.sparse = tx.sparse;
    a.piece_len = tx.piece_len; a.seg_len = tx.seg_len; a.seg_flags = tx.seg_flags; a.seg_off = tx.seg_off; a.text = tx.text;
    a.markq = tx.markq; a.markq_count = tx.markq_count; a.markq_cap = e->lim.rowq_cap;
    CK(e, cudaMemsetAsync(tx.markq_count, 0, 4, e->stream));
    CK(e, cudaEventRecord(tx.ev[0], e->stream));
    const uint32_t n = a.n_segs;
    if (n) {
        k_text_extract<<<(n + TX_WARPS - 1) / TX_WARPS, TX_WARPS * 32, 0, e->stream>>>(a);
        k_text_scan<<<1, 1024, 0, e->stream>>>(a.seg_len, n, a.seg_off);
        k_text_pack<<<(n + TX_WARPS - 1) / TX_WARPS, TX_WARPS * 32, 0, e->stream>>>(a);
        e->launches += 3;
    } else CK(e, cudaMemsetAsync(tx.seg_off, 0, 8, e->stream));
    CK(e, cudaEventRecord(tx.ev[1], e->stream));
    CK(e, cudaGetLastError());
    unsigned long long total = 0; uint32_t marks = 0;
    CK(e, cudaMemcpyAsync(&total, tx.seg_off + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(&marks, tx.markq_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    if (marks > e->lim.rowq_cap) marks = e->lim.rowq_cap;
    tx.total = total; tx.marks = marks; tx.ready = true;
    read_ms(tx.ev[0], tx.ev[1], tx.ms);
    *text_bytes = total; *n_marks = marks;
    return LGW_OK;
}

extern "C" int lgw_step_transcript_fetch(lgw_engine* e, uint8_t* text_out, uint64_t* seg_text_off, uint32_t* seg_flags, lgw_text_mark* marks_out) {
    if (!e || !seg_text_off || !seg_flags || (!text_out && e->text.total) || (!marks_out && e->text.marks)) return LGW_ERR_ARG;
    lgw_engine::Text& tx = e->text;
    if (!tx.ready) { e->err = "lgw_step_transcript_run has not run for the last step"; return LGW_ERR_ARG; }
    CK(e, cudaSetDevice(e->device));
    const uint32_t n = e->step.last.n_segs;
    if (tx.total) CK(e, cudaMemcpyAsync(text_out, tx.text, tx.total, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(seg_text_off, tx.seg_off, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    if (n) CK(e, cudaMemcpyAsync(seg_flags, tx.seg_flags, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    if (tx.marks) CK(e, cudaMemcpyAsync(marks_out, tx.markq, (size_t)tx.marks * sizeof(TextMark), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

extern "C" int lgw_transcript_last_ms(lgw_engine* e, float* ms) {
    if (!e || !ms) return LGW_ERR_ARG;
    *ms = e->text.ms;
    return LGW_OK;
}

// Device memory handed out by lgw_device_alloc is the caller's until lgw_device_free, like the pinned buffers.
extern "C" int lgw_device_alloc(lgw_engine* e, uint64_t bytes, void** out) {
    if (!e || !out) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaMalloc(out, bytes ? bytes : 1));
    return LGW_OK;
}
extern "C" int lgw_device_free(lgw_engine* e, void* p) { if (!e) return LGW_ERR_ARG; CK(e, cudaSetDevice(e->device)); CK(e, cudaFree(p)); return LGW_OK; }
extern "C" int lgw_device_upload(lgw_engine* e, void* d, const void* h, uint64_t bytes) {
    if (!e || (bytes && (!d || !h))) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, e->stream)); CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}
extern "C" int lgw_device_download(lgw_engine* e, void* h, const void* d, uint64_t bytes) {
    if (!e || (bytes && (!d || !h))) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, e->stream)); CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}
extern "C" int lgw_device_zero(lgw_engine* e, void* d, uint64_t bytes) {
    if (!e || (bytes && !d)) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaMemsetAsync(d, 0, bytes, e->stream));
    return LGW_OK;
}

#ifdef LGW_DEBUG_TIMING
extern "C" int lgw_debug_read(unsigned long long* out) { return cudaMemcpyFromSymbol(out, lgw::g_dbg, sizeof(unsigned long long) * 16) == cudaSuccess ? 0 : -2; }
#endif


// ---- request-body rewrite (rows a1, a3, a4) -------------------------------------------------------
static_assert(sizeof(BodyOp) == sizeof(lgw_body_op), "lgw_body_op");
static_assert(sizeof(BodyPlan) == sizeof(lgw_body_plan), "lgw_body_plan");
static_assert(sizeof(BodyResult) == sizeof(lgw_body_result), "lgw_body_result");
static_assert(sizeof(BodyScan) == sizeof(lgw_body_scan), "lgw_body_scan");

// Room for n elements in a staging buffer of the body calls.  Batch sizes vary from call to call, so these grow by a quarter
// and 64 elements beyond the request that outgrew them.
static cudaError_t reserve_body(DevBuf& b, uint64_t n, size_t elem_size = 1) { return b.reserve(n * elem_size, (n / 4 + 64) * elem_size); }

extern "C" int lgw_rules_load(lgw_engine* e, const lgw_body_plan* plans, uint32_t n_plans,
                              const lgw_body_op* ops, uint32_t n_ops, const uint8_t* blob, uint32_t blob_len) {
    if (!e || (n_plans && !plans) || (n_ops && !ops) || (blob_len && !blob)) return LGW_ERR_ARG;
    for (uint32_t i = 0; i < n_plans; ++i) {
        if (plans[i].op_begin > plans[i].op_end || plans[i].op_end > n_ops || plans[i].op_end - plans[i].op_begin > 32 || (plans[i].mode & 0xffu) > 2 || (plans[i].mode & ~0x1ffu)) {
            e->err = "lgw_rules_load: malformed plan"; return LGW_ERR_ARG; }
    }
    for (uint32_t i = 0; i < n_ops; ++i) {
        const lgw_body_op& o = ops[i];
        if ((uint64_t)o.key_off + o.key_len > blob_len || (uint64_t)o.rkey_off + o.rkey_len > blob_len || (uint64_t)o.rval_off + o.rval_len > blob_len) {
            e->err = "lgw_rules_load: op outside the blob"; return LGW_ERR_ARG; }
    }
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, bo.plans.reserve((n_plans + 1) * sizeof(BodyPlan)));
    CK(e, bo.ops.reserve((n_ops + 1) * sizeof(BodyOp)));
    CK(e, bo.blob.reserve((size_t)blob_len + 16));
    if (n_plans) CK(e, cudaMemcpyAsync(bo.plans.p, plans, n_plans * sizeof(BodyPlan), cudaMemcpyHostToDevice, e->stream));
    if (n_ops) CK(e, cudaMemcpyAsync(bo.ops.p, ops, n_ops * sizeof(BodyOp), cudaMemcpyHostToDevice, e->stream));
    if (blob_len) CK(e, cudaMemcpyAsync(bo.blob.p, blob, blob_len, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    bo.n_plans = n_plans; bo.n_ops = n_ops;
    return LGW_OK;
}

static int bodies_stage_in(lgw_engine* e, const uint8_t* bodies, const uint64_t* body_off, uint32_t n) {
    const uint64_t n_bytes = body_off[n];
    for (uint32_t i = 0; i < n; ++i) if (body_off[i + 1] < body_off[i] || body_off[i + 1] - body_off[i] > 0xFFFFFFF0ull) { e->err = "body offsets not monotonic"; return LGW_ERR_ARG; }
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, reserve_body(bo.in, n_bytes + 64));
    CK(e, reserve_body(bo.off, n + 1, sizeof(uint64_t)));
    CK(e, reserve_body(bo.out_off, n + 1, sizeof(uint64_t)));
    CK(e, reserve_body(bo.plan_idx, n + 1, sizeof(uint32_t)));
    CK(e, reserve_body(bo.results, n + 1, sizeof(BodyResult)));
    CK(e, reserve_body(bo.scans, n + 1, sizeof(BodyScan)));
    if (n_bytes) CK(e, cudaMemcpyAsync(bo.in.p, bodies, n_bytes, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaMemcpyAsync(bo.off.p, body_off, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
    return LGW_OK;
}

extern "C" int lgw_bodies_scan(lgw_engine* e, const uint8_t* bodies, const uint64_t* body_off, uint32_t n,
                               uint32_t model_cap, lgw_body_scan* scans_out, uint8_t* models_out) {
    if (!e || !body_off || (!bodies && n && body_off[n]) || !scans_out || (model_cap && !models_out)) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    TRY(bodies_stage_in(e, bodies, body_off, n));
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, reserve_body(bo.models, (uint64_t)n * model_cap + 16));
    k_body_scan<<<(n + LGW_BODY_WARPS - 1) / LGW_BODY_WARPS, 32 * LGW_BODY_WARPS, 0, e->stream>>>(bo.in.as<uint8_t>(), bo.off.as<uint64_t>(), n, model_cap, bo.scans.as<BodyScan>(), bo.models.as<uint8_t>());
    ++e->launches;
    CK(e, cudaGetLastError());
    CK(e, cudaMemcpyAsync(scans_out, bo.scans.p, n * sizeof(BodyScan), cudaMemcpyDeviceToHost, e->stream));
    if (model_cap) CK(e, cudaMemcpyAsync(models_out, bo.models.p, (uint64_t)n * model_cap, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

static int bodies_launch(lgw_engine* e, const uint8_t* d_bodies, const uint64_t* d_body_off, uint32_t n, const uint32_t* d_plan_idx,
                         uint32_t slot_cap, uint8_t* d_out, uint64_t out_cap, uint64_t* d_out_off, BodyResult* d_results) {
    lgw_engine::Bodies& bo = e->bodies;
    if (!bo.plans.p) { e->err = "lgw_bodies_rewrite before lgw_rules_load"; return LGW_ERR_ARG; }
    CK(e, reserve_body(bo.slots, (uint64_t)n * slot_cap + 64));
    CK(e, reserve_body(bo.redo, (uint64_t)n + 4, sizeof(uint32_t)));
    const BodyPlan* d_plans = bo.plans.as<BodyPlan>(); const BodyOp* d_ops = bo.ops.as<BodyOp>(); const uint8_t* d_blob = bo.blob.as<uint8_t>();
    uint8_t* d_slots = bo.slots.as<uint8_t>();
    uint32_t* redo = bo.redo.as<uint32_t>(); uint32_t* redo_count = redo + n;            // list first, counter behind it
    const unsigned seq_grid = grid_for(e, n, LGW_BODY_WARPS, 4);
    CK(e, cudaEventRecord(bo.ev[0], e->stream));
    if (bo.mode == 0) {
        CK(e, cudaMemsetAsync(redo_count, 0, 4, e->stream));
        k_body_fast<<<n, LGW_FAST_THREADS, 0, e->stream>>>(d_bodies, d_body_off, n, d_plan_idx, d_plans, bo.n_plans, d_ops, d_blob,
                                                             d_slots, slot_cap, d_results, redo_count, redo);
        k_body_rewrite<<<seq_grid, 32 * LGW_BODY_WARPS, 0, e->stream>>>(d_bodies, d_body_off, n, d_plan_idx, d_plans, bo.n_plans, d_ops, d_blob,
                                                                        d_slots, slot_cap, d_results, redo_count, redo);
        ++e->launches;
    } else {
        k_body_rewrite<<<seq_grid, 32 * LGW_BODY_WARPS, 0, e->stream>>>(d_bodies, d_body_off, n, d_plan_idx, d_plans, bo.n_plans, d_ops, d_blob,
                                                                        d_slots, slot_cap, d_results, nullptr, nullptr);
    }
    CK(e, cudaEventRecord(bo.ev[1], e->stream));
    k_body_offsets<<<1, 1024, 0, e->stream>>>(d_results, n, out_cap, d_out_off);
    CK(e, cudaEventRecord(bo.ev[2], e->stream));
    k_body_pack<<<grid_for(e, n, 1, 8), 256, 0, e->stream>>>(d_slots, slot_cap, d_results, n, d_out_off, d_out, out_cap);
    CK(e, cudaEventRecord(bo.ev[3], e->stream));
    e->launches += 3;
    CK(e, cudaGetLastError());
    return LGW_OK;
}

extern "C" int lgw_bodies_rewrite_device(lgw_engine* e, const uint8_t* d_bodies, const uint64_t* d_body_off, uint32_t n, uint64_t n_bytes,
                                         const uint32_t* d_plan_idx, uint32_t slot_cap, uint8_t* d_out, uint64_t out_cap,
                                         uint64_t* d_out_off, lgw_body_result* d_results) {
    (void)n_bytes;
    if (!e || !d_bodies || !d_body_off || !d_plan_idx || !d_out || !d_out_off || !d_results || slot_cap == 0) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    return bodies_launch(e, d_bodies, d_body_off, n, d_plan_idx, slot_cap, d_out, out_cap, d_out_off, (BodyResult*)d_results);
}

extern "C" int lgw_bodies_rewrite(lgw_engine* e, const uint8_t* bodies, const uint64_t* body_off, uint32_t n,
                                  const uint32_t* plan_idx, uint32_t slot_cap,
                                  uint8_t* out, uint64_t out_cap, uint64_t* out_off, lgw_body_result* results) {
    if (!e || !body_off || (!bodies && n && body_off[n]) || !plan_idx || (!out && out_cap) || !out_off || !results || slot_cap == 0) return LGW_ERR_ARG;
    if (n == 0) { out_off[0] = 0; return LGW_OK; }
    CK(e, cudaSetDevice(e->device));
    TRY(bodies_stage_in(e, bodies, body_off, n));
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, cudaMemcpyAsync(bo.plan_idx.p, plan_idx, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    CK(e, reserve_body(bo.out, out_cap + 64));
    TRY(bodies_launch(e, bo.in.as<uint8_t>(), bo.off.as<uint64_t>(), n, bo.plan_idx.as<uint32_t>(), slot_cap, bo.out.as<uint8_t>(), out_cap,
                      bo.out_off.as<uint64_t>(), bo.results.as<BodyResult>()));
    // the packed size is only known on the device: offsets first, then exactly that many bytes
    CK(e, cudaMemcpyAsync(out_off, bo.out_off.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(results, bo.results.p, n * sizeof(BodyResult), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    const uint64_t total = out_off[n] < out_cap ? out_off[n] : out_cap;
    if (total) CK(e, cudaMemcpyAsync(out, bo.out.p, total, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

// ---- response tap of non-streaming responses (row a8, non-stream mode) ---------------------------------
extern "C" int lgw_documents_usage(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, lgw_doc_usage* out) {
    if (!e || !doc_off || (!docs && n && doc_off[n]) || (!out && n)) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    TRY(bodies_stage_in(e, docs, doc_off, n));           // (the request-body staging buffers: same layout)
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, bo.doc_out.reserve((size_t)n * sizeof(DocUsage)));
    k_docs_usage<<<grid_for(e, n, LGW_DOC_WARPS, 8), LGW_DOC_WARPS * 32, 0, e->stream>>>(bo.in.as<uint8_t>(), bo.off.as<uint64_t>(), n, bo.doc_out.as<DocUsage>());
    ++e->launches;
    CK(e, cudaGetLastError());
    CK(e, cudaMemcpyAsync(out, bo.doc_out.p, (size_t)n * sizeof(DocUsage), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

// ---- error detail of failing non-streaming responses (row a12, request_handler.py:167-169) ---------------
extern "C" int lgw_documents_error_detail(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, lgw_doc_error* out, uint8_t* text, uint32_t text_stride) {
    if (!e || !doc_off || (!docs && n && doc_off[n]) || (n && (!out || !text)) || text_stride == 0) return LGW_ERR_ARG;
    if (n == 0) return LGW_OK;
    CK(e, cudaSetDevice(e->device));
    TRY(bodies_stage_in(e, docs, doc_off, n));
    lgw_engine::Bodies& bo = e->bodies;
    CK(e, bo.doc_out.reserve((size_t)n * sizeof(DocError)));
    CK(e, bo.doc_text.reserve((size_t)n * text_stride));
    k_docs_error_detail<<<grid_for(e, n, LGW_DOC_WARPS, 8), LGW_DOC_WARPS * 32, 0, e->stream>>>(bo.in.as<uint8_t>(), bo.off.as<uint64_t>(), n, bo.doc_out.as<DocError>(), bo.doc_text.as<uint8_t>(), text_stride);
    ++e->launches;
    CK(e, cudaGetLastError());
    CK(e, cudaMemcpyAsync(out, bo.doc_out.p, (size_t)n * sizeof(DocError), cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(text, bo.doc_text.p, (size_t)n * text_stride, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

// ---- text of the non-streaming tap (row a8, chat_logging.py:124-139): walk, scan of the lengths, pack -----------------------
extern "C" int lgw_documents_text(lgw_engine* e, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                                  uint8_t* text_out, uint64_t text_cap, uint64_t* text_off, uint32_t* flags) {
    if (!e || !doc_off || (!docs && n && doc_off[n]) || !text_off || (!flags && n) || (!text_out && text_cap)) return LGW_ERR_ARG;
    if (n == 0) { text_off[0] = 0; return LGW_OK; }
    for (uint32_t i = 0; i < n; ++i)
        if (doc_off[i + 1] >= doc_off[i] && doc_off[i + 1] - doc_off[i] > 0x7FFFFFFFull) { e->err = "document longer than 2^31 bytes"; return LGW_ERR_ARG; }
    CK(e, cudaSetDevice(e->device));
    TRY(bodies_stage_in(e, docs, doc_off, n));           // (the request-body staging buffers: same layout)
    lgw_engine::DocsText& dt = e->docs_text;
    if (!dt.ev[0]) CK(e, new_events(e, dt.ev, 2));
    const uint64_t room = 2 * (doc_off[n] - doc_off[0]);  // a document's text is at most twice its length (transcript.cuh text_part)
    CK(e, reserve_body(dt.sparse, room + 64));
    CK(e, reserve_body(dt.text, room + 64));
    CK(e, reserve_body(dt.len, n + 1, sizeof(uint32_t)));
    CK(e, reserve_body(dt.flags, n + 1, sizeof(uint32_t)));
    CK(e, reserve_body(dt.off, n + 1, sizeof(unsigned long long)));
    const uint64_t* d_off = e->bodies.off.as<uint64_t>();
    const unsigned grid = grid_for(e, n, LGW_DOC_WARPS, 8);
    CK(e, cudaEventRecord(dt.ev[0], e->stream));
    k_docs_text<<<grid, LGW_DOC_WARPS * 32, 0, e->stream>>>(e->bodies.in.as<uint8_t>(), d_off, n, dt.sparse.as<uint8_t>(), dt.len.as<uint32_t>(), dt.flags.as<uint32_t>());
    k_text_scan<<<1, 1024, 0, e->stream>>>(dt.len.as<uint32_t>(), n, dt.off.as<unsigned long long>());
    k_docs_text_pack<<<grid, LGW_DOC_WARPS * 32, 0, e->stream>>>(d_off, n, dt.sparse.as<uint8_t>(), dt.len.as<uint32_t>(), dt.off.as<unsigned long long>(), dt.text.as<uint8_t>());
    CK(e, cudaEventRecord(dt.ev[1], e->stream));
    e->launches += 3;
    CK(e, cudaGetLastError());
    unsigned long long total = 0;
    CK(e, cudaMemcpyAsync(&total, dt.off.as<unsigned long long>() + n, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    read_ms(dt.ev[0], dt.ev[1], dt.ms);
    if (total > text_cap) { e->err = "lgw_documents_text: text_cap is smaller than the text (" + std::to_string(total) + " bytes)"; return LGW_ERR_CAPACITY; }
    if (total) CK(e, cudaMemcpyAsync(text_out, dt.text.p, total, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(text_off, dt.off.p, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaMemcpyAsync(flags, dt.flags.p, (size_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    return LGW_OK;
}

extern "C" int lgw_documents_text_last_ms(lgw_engine* e, float* ms) {
    if (!e || !ms) return LGW_ERR_ARG;
    *ms = e->docs_text.ms;
    return LGW_OK;
}

extern "C" int lgw_bodies_last_ms(lgw_engine* e, float ms[3]) {
    if (!e || !ms) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    lgw_engine::Bodies& bo = e->bodies;
    cudaEventSynchronize(bo.ev[3]);
    for (int i = 0; i < 3; ++i) { read_ms(bo.ev[i], bo.ev[i + 1], bo.ms[i]); ms[i] = bo.ms[i]; }
    return LGW_OK;
}

// diagnostics (not part of the public header): how the segments of all steps so far were settled
// out[0] redone sequentially, [1] folded from the bulk kernel, [2] usage records read from template spans, [3] usage events stashed
extern "C" int lgw_debug_counters(lgw_engine* e, uint32_t out[4]) {
    if (!e || !out) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    CK(e, cudaMemcpy(out, e->scratch.counters, 16, cudaMemcpyDeviceToHost));
    return LGW_OK;
}

// diagnostics (not part of the public header, like lgw_engine_set_mode): the engine-wide event-template cache
// out[0..15] = state[4], len[4], flags[4], hits[4]; text = first `cap` bytes of each slot's template (4 x cap bytes)
extern "C" int lgw_debug_template_cache(lgw_engine* e, uint32_t out[16], uint8_t* text, uint32_t cap) {
    if (!e || !out) return LGW_ERR_ARG;
    CK(e, cudaSetDevice(e->device));
    CK(e, cudaStreamSynchronize(e->stream));
    std::vector<uint8_t> buf(sizeof(TemplateCache2));
    CK(e, cudaMemcpy(buf.data(), e->scratch.tpl_cache2, sizeof(TemplateCache2), cudaMemcpyDeviceToHost));
    const TemplateCache2* h = reinterpret_cast<const TemplateCache2*>(buf.data());
    for (int i = 0; i < 4; ++i) { out[i] = h->state[i]; out[4 + i] = h->tpl[i].m.len; out[8 + i] = h->tpl[i].m.flags | (h->tpl[i].m.usage_ok << 31); out[12 + i] = h->hits[i]; }
    if (cap > R2_TEXT) cap = R2_TEXT;
    if (text) for (int i = 0; i < 4; ++i) memcpy(text + (size_t)i * cap, h->tpl[i].text, cap);
    return LGW_OK;
}
