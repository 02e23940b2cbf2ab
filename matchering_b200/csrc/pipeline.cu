// Batch entry point: several tracks in flight, host buffers in and out.
//
// mgb_process_host masters one track and returns when its result is back in host memory, so its
// PCIe copies (190 MB for a 3-minute track) and its kernels run one after the other.  Tracks are
// independent (SURVEY.md 8e), so a pipeline of `depth` slots overlaps them: track k+1's
// host->device copy (copy engine 1) runs while track k computes and track k-1's result returns
// (copy engine 2).  Three streams, three events per slot; nothing blocks the host except
// mgb_pipeline_wait and the reuse of a slot whose previous result has not been collected.
#include <string.h>

#include <algorithm>
#include <vector>

#include "kernels.cuh"

namespace mgb {

struct Slot {
    float* d_target = nullptr;
    float* d_reference = nullptr;
    float* d_result = nullptr;
    float* d_out = nullptr;
    void* d_workspace = nullptr;
    void* d_pcm_in = nullptr;   // raw PCM of target then reference (submit_pcm)
    void* d_pcm_out = nullptr;  // quantised result
    mgb_track_state* d_state = nullptr;
    mgb_track_state* h_state = nullptr;  // pinned
    void* d_meter_ws = nullptr;          // metering only (mgb_pipeline_enable_loudness)
    mgb_loudness_result* d_meter = nullptr;
    mgb_loudness_result* h_meter = nullptr;  // pinned
    void* d_search_ws = nullptr;         // loudness target only (mgb_pipeline_enable_loudness_target)
    mgb_loudness_target_report* d_report = nullptr;
    mgb_loudness_target_report* h_report = nullptr;  // pinned
    mgb_track_layout layout;
    bool busy = false;
#ifndef MGB_EMULATE
    cudaEvent_t h2d_done = nullptr, compute_done = nullptr, d2h_done = nullptr;
    cudaStream_t compute = nullptr;  // one compute stream per slot: the small latency-bound kernels of
                                     // one track (FIR design: 2 CTAs) overlap another track's streaming ones
#endif
};

}  // namespace mgb

struct mgb_pipeline {
    mgb_plan plan;
    int64_t max_target = 0, max_reference = 0;
    int64_t workspace_bytes = 0;
    std::vector<mgb::Slot> slots;
    int next = 0;
    bool submitted = false;
    bool meter = false;  // mgb_pipeline_enable_loudness
    mgb_loudness_params meter_params;
    int64_t meter_ws_bytes = 0;
    bool target = false;  // mgb_pipeline_enable_loudness_target
    mgb_loudness_target target_params;
    int64_t search_ws_bytes = 0;
    bool dither = false;  // mgb_pipeline_enable_dither
    mgb_dither_params dither_params;
#ifndef MGB_EMULATE
    cudaStream_t s_h2d = nullptr, s_compute = nullptr, s_d2h = nullptr;
#endif
};

using namespace mgb;

namespace {
// A submit that fails after its copies were enqueued must not leave the slot looking free while the
// device still reads or writes its buffers: drain the streams it used before reporting the error.
struct SubmitGuard {
    mgb_pipeline* p;
    Slot* s;
    bool ok = false;
    ~SubmitGuard() {
        if (ok) return;
#ifndef MGB_EMULATE
        cudaStreamSynchronize(p->s_h2d);
        if (s->compute) cudaStreamSynchronize(s->compute);
        cudaStreamSynchronize(p->s_d2h);
#endif
        s->busy = false;
    }
};
}  // namespace

// With the "poison_alloc" option every new buffer starts as 0xFF bytes (NaN as float or double, -1 as an
// integer), so that a kernel reading slot memory nothing wrote shows up in the results.
#ifdef MGB_EMULATE
#define MGB_CUDA_OK(call) (void)0
static void* dev_alloc(size_t bytes) {
    const size_t padded = (bytes + 255) / 256 * 256;
    void* p = aligned_alloc(256, padded);
    if (p && g_poison_alloc) memset(p, 0xFF, padded);
    return p;
}
static void dev_free(void* p) { free(p); }
#else
#define MGB_CUDA_OK(call)                                                             \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) {                                                      \
            set_error("%s: %s", #call, cudaGetErrorString(e_));                       \
            return MGB_ERR_CUDA;                                                      \
        }                                                                             \
    } while (0)
static void* dev_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
    // (cudaMemset runs on the legacy default stream, which the pipeline's non-blocking streams do not wait for:
    // the fill must be complete before the first submit's copies and kernels touch the buffer)
    if (g_poison_alloc && (cudaMemset(p, 0xFF, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)) {
        cudaFree(p);
        return nullptr;
    }
    return p;
}
static void dev_free(void* p) { cudaFree(p); }
#endif

extern "C" {

// (inside mgb_pipeline_create: a failed CUDA call releases what was created so far)
#ifdef MGB_EMULATE
#define MGB_CUDA_OR_DESTROY(call) (void)0
#else
#define MGB_CUDA_OR_DESTROY(call)                                                     \
    do {                                                                              \
        cudaError_t e_ = (call);                                                      \
        if (e_ != cudaSuccess) {                                                      \
            set_error("%s: %s", #call, cudaGetErrorString(e_));                       \
            mgb_pipeline_destroy(p);                                                  \
            return MGB_ERR_CUDA;                                                      \
        }                                                                             \
    } while (0)
#endif

int mgb_pipeline_create(const mgb_plan* plan, int64_t max_target_frames, int64_t max_reference_frames, int32_t depth,
                        mgb_pipeline** out) {
    MGB_REQUIRE(plan && out, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE(depth >= 1 && depth <= 8, MGB_ERR_INVALID, "pipeline: depth must be 1..8");
    mgb_track_layout biggest;
    MGB_TRY(mgb_track_layout_init(plan, max_target_frames, max_reference_frames, &biggest));
    mgb_pipeline* p = new mgb_pipeline();
    p->plan = *plan;
    p->max_target = max_target_frames;
    p->max_reference = max_reference_frames;
    // the workspace grows with the frame counts and the number of pieces (both largest for the longest
    // track) and with the analysis items = divisions x slots, which do NOT: slots = 3*SMs / divisions
    // rounds down, so a shorter track with fewer pieces can have more items.  Items never exceed
    // max(3*SMs, divisions); size for that.
    {
        mgb_track_layout worst = biggest;
        const int64_t cap = 3LL * num_sms();
        worst.target_slots = (int32_t)((std::max<int64_t>(cap, worst.target_divisions) + worst.target_divisions - 1) / worst.target_divisions);
        worst.reference_slots = (int32_t)((std::max<int64_t>(cap, worst.reference_divisions) + worst.reference_divisions - 1) / worst.reference_divisions);
        p->workspace_bytes = carve_workspace(*plan, worst, nullptr).total_bytes;
        // a profiled job has the same target regions, no reference regions and a copy of the profile, which
        // can be larger than a short reference's regions
        mgb_track_layout profiled = worst;
        profiled.reference_frames = profiled.reference_piece = 0;
        profiled.reference_divisions = profiled.reference_slots = 0;
        p->workspace_bytes = std::max(p->workspace_bytes, carve_workspace(*plan, profiled, nullptr).total_bytes);
    }
    p->slots.resize(depth);
#ifndef MGB_EMULATE
    MGB_CUDA_OR_DESTROY(cudaStreamCreateWithFlags(&p->s_h2d, cudaStreamNonBlocking));
    MGB_CUDA_OR_DESTROY(cudaStreamCreateWithFlags(&p->s_compute, cudaStreamNonBlocking));
    MGB_CUDA_OR_DESTROY(cudaStreamCreateWithFlags(&p->s_d2h, cudaStreamNonBlocking));
#endif
    for (auto& s : p->slots) {
        s.d_target = (float*)dev_alloc((size_t)max_target_frames * 8);
        s.d_reference = (float*)dev_alloc((size_t)max_reference_frames * 8);
        s.d_result = (float*)dev_alloc((size_t)max_target_frames * 8);
        s.d_out = (float*)dev_alloc((size_t)max_target_frames * 8);
        s.d_workspace = dev_alloc((size_t)p->workspace_bytes);
        s.d_pcm_in = dev_alloc((size_t)(max_target_frames + max_reference_frames) * 6 + 512);
        s.d_pcm_out = dev_alloc((size_t)max_target_frames * 6 + 256);
        s.d_state = (mgb_track_state*)dev_alloc(sizeof(mgb_track_state));
        if (!s.d_target || !s.d_reference || !s.d_result || !s.d_out || !s.d_workspace || !s.d_state || !s.d_pcm_in ||
            !s.d_pcm_out) {
            set_error("pipeline: device allocation failed");
            mgb_pipeline_destroy(p);
            return MGB_ERR_CUDA;
        }
#ifdef MGB_EMULATE
        s.h_state = (mgb_track_state*)malloc(sizeof(mgb_track_state));
#else
        MGB_CUDA_OR_DESTROY(cudaMallocHost((void**)&s.h_state, sizeof(mgb_track_state)));
        MGB_CUDA_OR_DESTROY(cudaEventCreateWithFlags(&s.h2d_done, cudaEventDisableTiming));
        MGB_CUDA_OR_DESTROY(cudaEventCreateWithFlags(&s.compute_done, cudaEventDisableTiming));
        MGB_CUDA_OR_DESTROY(cudaEventCreateWithFlags(&s.d2h_done, cudaEventDisableTiming));
        MGB_CUDA_OR_DESTROY(cudaStreamCreateWithFlags(&s.compute, cudaStreamNonBlocking));
#endif
    }
    *out = p;
    return MGB_OK;
}

int mgb_pipeline_destroy(mgb_pipeline* p) {
    if (!p) return MGB_OK;
#ifndef MGB_EMULATE
    cudaDeviceSynchronize();
#endif
    for (auto& s : p->slots) {
        dev_free(s.d_target);
        dev_free(s.d_reference);
        dev_free(s.d_result);
        dev_free(s.d_out);
        dev_free(s.d_workspace);
        dev_free(s.d_pcm_in);
        dev_free(s.d_pcm_out);
        dev_free(s.d_state);
        if (s.d_meter_ws) dev_free(s.d_meter_ws);
        if (s.d_meter) dev_free(s.d_meter);
        if (s.d_search_ws) dev_free(s.d_search_ws);
        if (s.d_report) dev_free(s.d_report);
#ifdef MGB_EMULATE
        free(s.h_state);
        free(s.h_meter);
        free(s.h_report);
#else
        if (s.h_state) cudaFreeHost(s.h_state);
        if (s.h_meter) cudaFreeHost(s.h_meter);
        if (s.h_report) cudaFreeHost(s.h_report);
        if (s.h2d_done) cudaEventDestroy(s.h2d_done);
        if (s.compute_done) cudaEventDestroy(s.compute_done);
        if (s.d2h_done) cudaEventDestroy(s.d2h_done);
        if (s.compute) cudaStreamDestroy(s.compute);
#endif
    }
#ifndef MGB_EMULATE
    if (p->s_h2d) cudaStreamDestroy(p->s_h2d);
    if (p->s_compute) cudaStreamDestroy(p->s_compute);
    if (p->s_d2h) cudaStreamDestroy(p->s_d2h);
#endif
    delete p;
    return MGB_OK;
}

int mgb_pipeline_wait(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out) {
    MGB_REQUIRE(p && slot >= 0 && slot < (int)p->slots.size(), MGB_ERR_INVALID, "pipeline: bad slot");
    Slot& s = p->slots[slot];
    if (s.busy) {
#ifndef MGB_EMULATE
        MGB_CUDA_OK(cudaEventSynchronize(s.d2h_done));
#endif
        s.busy = false;
    }
    if (state_out) *state_out = *s.h_state;
    return MGB_OK;
}

int mgb_pipeline_enable_loudness(mgb_pipeline* p, const mgb_loudness_params* params) {
    MGB_REQUIRE(p && params, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE(!p->submitted && !p->meter, MGB_ERR_INVALID, "pipeline: metering is enabled once, before the first submit");
    MGB_REQUIRE(params->d_tables, MGB_ERR_INVALID, "pipeline: loudness tables missing");
    const int64_t bytes = mgb_loudness_workspace_bytes(params, std::max<int64_t>(p->max_target, 1));
    MGB_REQUIRE(bytes > 0, MGB_ERR_INVALID, "pipeline: bad loudness parameters");
    for (auto& s : p->slots) {
        s.d_meter_ws = dev_alloc((size_t)bytes);
        s.d_meter = (mgb_loudness_result*)dev_alloc(sizeof(mgb_loudness_result));
#ifdef MGB_EMULATE
        s.h_meter = (mgb_loudness_result*)malloc(sizeof(mgb_loudness_result));
#else
        if (cudaMallocHost((void**)&s.h_meter, sizeof(mgb_loudness_result)) != cudaSuccess) s.h_meter = nullptr;
#endif
        if (!s.d_meter_ws || !s.d_meter || !s.h_meter) {
            set_error("pipeline: allocation of the meter buffers failed");
            return MGB_ERR_CUDA;  // (what was allocated is released by mgb_pipeline_destroy)
        }
        memset(s.h_meter, 0, sizeof(mgb_loudness_result));
    }
    p->meter_params = *params;
    p->meter_ws_bytes = bytes;
    p->meter = true;
    return MGB_OK;
}

int mgb_pipeline_wait_loudness(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out, mgb_loudness_result* loudness_out) {
    MGB_REQUIRE(p && p->meter, MGB_ERR_INVALID, "pipeline: metering is not enabled");
    MGB_TRY(mgb_pipeline_wait(p, slot, state_out));
    if (loudness_out) *loudness_out = *p->slots[slot].h_meter;
    return MGB_OK;
}

int mgb_pipeline_enable_loudness_target(mgb_pipeline* p, const mgb_loudness_target* target) {
    MGB_REQUIRE(p != nullptr, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE(p->meter, MGB_ERR_INVALID, "pipeline: a loudness target needs metering (mgb_pipeline_enable_loudness) first");
    MGB_REQUIRE(!p->submitted && !p->target, MGB_ERR_INVALID, "pipeline: a loudness target is set once, before the first submit");
    MGB_TRY(loudness_target_validate(target, &p->meter_params));
    MGB_REQUIRE(p->meter_params.sample_rate == p->plan.sample_rate, MGB_ERR_INVALID,
                "pipeline: the meter's rate %d differs from the plan's %d", p->meter_params.sample_rate, p->plan.sample_rate);
    const int64_t bytes = mgb_loudness_target_workspace_bytes(&p->meter_params, std::max<int64_t>(p->max_target, 1));
    MGB_REQUIRE(bytes > 0, MGB_ERR_INVALID, "pipeline: bad loudness parameters");
    for (auto& s : p->slots) {
        s.d_search_ws = dev_alloc((size_t)bytes);
        s.d_report = (mgb_loudness_target_report*)dev_alloc(sizeof(mgb_loudness_target_report));
#ifdef MGB_EMULATE
        s.h_report = (mgb_loudness_target_report*)malloc(sizeof(mgb_loudness_target_report));
#else
        if (cudaMallocHost((void**)&s.h_report, sizeof(mgb_loudness_target_report)) != cudaSuccess) s.h_report = nullptr;
#endif
        if (!s.d_search_ws || !s.d_report || !s.h_report) {
            set_error("pipeline: allocation of the loudness-target buffers failed");
            return MGB_ERR_CUDA;  // (what was allocated is released by mgb_pipeline_destroy)
        }
        memset(s.h_report, 0, sizeof(mgb_loudness_target_report));
    }
    p->target_params = *target;
    p->search_ws_bytes = bytes;
    p->target = true;
    return MGB_OK;
}

int mgb_pipeline_wait_loudness_target(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out,
                                      mgb_loudness_result* loudness_out, mgb_loudness_target_report* report_out) {
    MGB_REQUIRE(p && p->target, MGB_ERR_INVALID, "pipeline: no loudness target is set");
    MGB_TRY(mgb_pipeline_wait_loudness(p, slot, state_out, loudness_out));
    if (report_out) *report_out = *p->slots[slot].h_report;
    return MGB_OK;
}

int mgb_pipeline_enable_dither(mgb_pipeline* p, const mgb_dither_params* params) {
    MGB_REQUIRE(p != nullptr, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE(!p->submitted && !p->dither, MGB_ERR_INVALID, "pipeline: dither is enabled once, before the first submit");
    MGB_TRY(dither_validate(params));
    p->dither_params = *params;
    p->dither = true;
    return MGB_OK;
}

// Stage 4 of a submission: the limited output into d_out, at the pipeline's loudness target if it has one.
static int submit_finalize(mgb_pipeline* p, Slot& s, void* sc) {
    if (!p->target) return mgb_finalize(&p->plan, &s.layout, s.d_result, s.d_out, nullptr, nullptr, s.d_workspace, s.d_state, sc);
    return mgb_finalize_to_loudness(&p->plan, &s.layout, &p->meter_params, &p->target_params, s.d_result, s.d_out,
                                    s.d_workspace, s.d_search_ws, p->search_ws_bytes, s.d_state, s.d_report, sc);
}

// Metering of a submission's float32 limited output, on the slot's compute stream (nothing without metering).
static int submit_meter(mgb_pipeline* p, Slot& s, int64_t frames, void* sc) {
    if (!p->meter) return MGB_OK;
    return mgb_loudness(&p->meter_params, s.d_out, frames, s.d_meter_ws, p->meter_ws_bytes, s.d_meter, sc);
}

// Stage 1 of a submission: the reference's samples (d_profile == nullptr) or a profile.
static int submit_levels(mgb_pipeline* p, Slot& s, const void* d_profile, void* sc) {
    if (d_profile) return mgb_match_levels_profiled(&p->plan, &s.layout, s.d_target, d_profile, s.d_workspace, s.d_state, sc);
    return mgb_match_levels(&p->plan, &s.layout, s.d_target, s.d_reference, s.d_workspace, s.d_state, sc);
}

static int submit_impl(mgb_pipeline* p, const float* h_target_lr, int64_t target_frames, const float* h_reference_lr,
                       int64_t reference_frames, const void* d_profile, float* h_out_limited, int32_t* slot_out) {
    MGB_REQUIRE(p && h_target_lr && (h_reference_lr || d_profile) && h_out_limited, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE(target_frames <= p->max_target && reference_frames <= p->max_reference, MGB_ERR_INVALID,
                "pipeline: track longer than the pipeline was created for");
    const int idx = p->next;
    p->next = (p->next + 1) % (int)p->slots.size();
    Slot& s = p->slots[idx];
    MGB_TRY(mgb_pipeline_wait(p, idx, nullptr));  // the slot's previous result must have left the device
    SubmitGuard guard{p, &s};
    p->submitted = true;
    if (d_profile)
        MGB_TRY(mgb_track_layout_init_profiled(&p->plan, target_frames, &s.layout));
    else
        MGB_TRY(mgb_track_layout_init(&p->plan, target_frames, reference_frames, &s.layout));
    MGB_REQUIRE(s.layout.workspace_bytes <= p->workspace_bytes, MGB_ERR_WORKSPACE, "pipeline: workspace too small");
    const size_t tb = (size_t)target_frames * 8, rb = (size_t)reference_frames * 8;
#ifdef MGB_EMULATE
    memcpy(s.d_target, h_target_lr, tb);
    if (!d_profile) memcpy(s.d_reference, h_reference_lr, rb);
    void* sc = nullptr;
#else
    MGB_CUDA_OK(cudaMemcpyAsync(s.d_target, h_target_lr, tb, cudaMemcpyHostToDevice, p->s_h2d));
    if (!d_profile) MGB_CUDA_OK(cudaMemcpyAsync(s.d_reference, h_reference_lr, rb, cudaMemcpyHostToDevice, p->s_h2d));
    MGB_CUDA_OK(cudaEventRecord(s.h2d_done, p->s_h2d));
    MGB_CUDA_OK(cudaStreamWaitEvent(s.compute, s.h2d_done, 0));
    void* sc = (void*)s.compute;
#endif
    MGB_TRY(submit_levels(p, s, d_profile, sc));
    MGB_TRY(mgb_match_frequencies(&p->plan, &s.layout, s.d_target, s.d_result, nullptr, s.d_workspace, s.d_state, sc));
    MGB_TRY(mgb_correct_levels(&p->plan, &s.layout, s.d_workspace, s.d_state, sc));
    MGB_TRY(submit_finalize(p, s, sc));
    MGB_TRY(submit_meter(p, s, target_frames, sc));
#ifdef MGB_EMULATE
    memcpy(h_out_limited, s.d_out, tb);
    memcpy(s.h_state, s.d_state, sizeof(mgb_track_state));
    if (p->meter) memcpy(s.h_meter, s.d_meter, sizeof(mgb_loudness_result));
    if (p->target) memcpy(s.h_report, s.d_report, sizeof(mgb_loudness_target_report));
#else
    MGB_CUDA_OK(cudaEventRecord(s.compute_done, s.compute));
    MGB_CUDA_OK(cudaStreamWaitEvent(p->s_d2h, s.compute_done, 0));
    MGB_CUDA_OK(cudaMemcpyAsync(h_out_limited, s.d_out, tb, cudaMemcpyDeviceToHost, p->s_d2h));
    MGB_CUDA_OK(cudaMemcpyAsync(s.h_state, s.d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToHost, p->s_d2h));
    if (p->meter)
        MGB_CUDA_OK(cudaMemcpyAsync(s.h_meter, s.d_meter, sizeof(mgb_loudness_result), cudaMemcpyDeviceToHost, p->s_d2h));
    if (p->target)
        MGB_CUDA_OK(cudaMemcpyAsync(s.h_report, s.d_report, sizeof(mgb_loudness_target_report), cudaMemcpyDeviceToHost,
                                    p->s_d2h));
    MGB_CUDA_OK(cudaEventRecord(s.d2h_done, p->s_d2h));
#endif
    s.busy = true;
    guard.ok = true;
    if (slot_out) *slot_out = idx;
    return MGB_OK;
}

int mgb_pipeline_submit(mgb_pipeline* p, const float* h_target_lr, int64_t target_frames, const float* h_reference_lr,
                        int64_t reference_frames, float* h_out_limited, int32_t* slot_out) {
    MGB_REQUIRE(h_reference_lr, MGB_ERR_INVALID, "pipeline: NULL argument");
    return submit_impl(p, h_target_lr, target_frames, h_reference_lr, reference_frames, nullptr, h_out_limited, slot_out);
}

int mgb_pipeline_submit_profiled(mgb_pipeline* p, const float* h_target_lr, int64_t target_frames, const void* d_profile,
                                 float* h_out_limited, int32_t* slot_out) {
    MGB_REQUIRE(d_profile, MGB_ERR_INVALID, "pipeline: NULL argument");
    return submit_impl(p, h_target_lr, target_frames, nullptr, 0, d_profile, h_out_limited, slot_out);
}

static int submit_pcm_impl(mgb_pipeline* p, const void* h_target_pcm, int32_t target_bits, int64_t target_frames,
                           const void* h_reference_pcm, int32_t reference_bits, int64_t reference_frames, const void* d_profile,
                           void* h_out_pcm, int32_t out_bits, int32_t* slot_out) {
    MGB_REQUIRE(p && h_target_pcm && (h_reference_pcm || d_profile) && h_out_pcm, MGB_ERR_INVALID, "pipeline: NULL argument");
    MGB_REQUIRE((target_bits == 16 || target_bits == 24) && (d_profile || reference_bits == 16 || reference_bits == 24) &&
                    (out_bits == 16 || out_bits == 24),
                MGB_ERR_UNSUPPORTED, "pipeline: PCM widths must be 16 or 24 bits");
    MGB_REQUIRE(target_frames <= p->max_target && reference_frames <= p->max_reference, MGB_ERR_INVALID,
                "pipeline: track longer than the pipeline was created for");
    const int idx = p->next;
    p->next = (p->next + 1) % (int)p->slots.size();
    Slot& s = p->slots[idx];
    MGB_TRY(mgb_pipeline_wait(p, idx, nullptr));
    SubmitGuard guard{p, &s};
    p->submitted = true;
    if (d_profile)
        MGB_TRY(mgb_track_layout_init_profiled(&p->plan, target_frames, &s.layout));
    else
        MGB_TRY(mgb_track_layout_init(&p->plan, target_frames, reference_frames, &s.layout));
    MGB_REQUIRE(s.layout.workspace_bytes <= p->workspace_bytes, MGB_ERR_WORKSPACE, "pipeline: workspace too small");
    const size_t tb = (size_t)target_frames * 2 * (target_bits / 8), rb = (size_t)reference_frames * 2 * (reference_bits / 8);
    const size_t ob = (size_t)target_frames * 2 * (out_bits / 8);
    unsigned char* pcm_t = (unsigned char*)s.d_pcm_in;
    unsigned char* pcm_r = pcm_t + (tb + 255) / 256 * 256;
#ifdef MGB_EMULATE
    memcpy(pcm_t, h_target_pcm, tb);
    if (!d_profile) memcpy(pcm_r, h_reference_pcm, rb);
    void* sc = nullptr;
#else
    MGB_CUDA_OK(cudaMemcpyAsync(pcm_t, h_target_pcm, tb, cudaMemcpyHostToDevice, p->s_h2d));
    if (!d_profile) MGB_CUDA_OK(cudaMemcpyAsync(pcm_r, h_reference_pcm, rb, cudaMemcpyHostToDevice, p->s_h2d));
    MGB_CUDA_OK(cudaEventRecord(s.h2d_done, p->s_h2d));
    MGB_CUDA_OK(cudaStreamWaitEvent(s.compute, s.h2d_done, 0));
    void* sc = (void*)s.compute;
#endif
    MGB_TRY(mgb_pcm_decode(pcm_t, target_bits, s.d_target, target_frames * 2, sc));
    if (!d_profile) MGB_TRY(mgb_pcm_decode(pcm_r, reference_bits, s.d_reference, reference_frames * 2, sc));
    MGB_TRY(submit_levels(p, s, d_profile, sc));
    MGB_TRY(mgb_match_frequencies(&p->plan, &s.layout, s.d_target, s.d_result, nullptr, s.d_workspace, s.d_state, sc));
    MGB_TRY(mgb_correct_levels(&p->plan, &s.layout, s.d_workspace, s.d_state, sc));
    MGB_TRY(submit_finalize(p, s, sc));
    MGB_TRY(submit_meter(p, s, target_frames, sc));  // (the float32 output, before quantisation)
    if (p->dither)
        MGB_TRY(mgb_pcm_encode_dithered(&p->dither_params, s.d_out, target_frames, out_bits, s.d_pcm_out, sc));
    else
        MGB_TRY(mgb_pcm_encode(s.d_out, out_bits, s.d_pcm_out, target_frames * 2, sc));
#ifdef MGB_EMULATE
    memcpy(h_out_pcm, s.d_pcm_out, ob);
    memcpy(s.h_state, s.d_state, sizeof(mgb_track_state));
    if (p->meter) memcpy(s.h_meter, s.d_meter, sizeof(mgb_loudness_result));
    if (p->target) memcpy(s.h_report, s.d_report, sizeof(mgb_loudness_target_report));
#else
    MGB_CUDA_OK(cudaEventRecord(s.compute_done, s.compute));
    MGB_CUDA_OK(cudaStreamWaitEvent(p->s_d2h, s.compute_done, 0));
    MGB_CUDA_OK(cudaMemcpyAsync(h_out_pcm, s.d_pcm_out, ob, cudaMemcpyDeviceToHost, p->s_d2h));
    MGB_CUDA_OK(cudaMemcpyAsync(s.h_state, s.d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToHost, p->s_d2h));
    if (p->meter)
        MGB_CUDA_OK(cudaMemcpyAsync(s.h_meter, s.d_meter, sizeof(mgb_loudness_result), cudaMemcpyDeviceToHost, p->s_d2h));
    if (p->target)
        MGB_CUDA_OK(cudaMemcpyAsync(s.h_report, s.d_report, sizeof(mgb_loudness_target_report), cudaMemcpyDeviceToHost,
                                    p->s_d2h));
    MGB_CUDA_OK(cudaEventRecord(s.d2h_done, p->s_d2h));
#endif
    s.busy = true;
    guard.ok = true;
    if (slot_out) *slot_out = idx;
    return MGB_OK;
}

int mgb_pipeline_submit_pcm(mgb_pipeline* p, const void* h_target_pcm, int32_t target_bits, int64_t target_frames,
                            const void* h_reference_pcm, int32_t reference_bits, int64_t reference_frames,
                            void* h_out_pcm, int32_t out_bits, int32_t* slot_out) {
    MGB_REQUIRE(h_reference_pcm, MGB_ERR_INVALID, "pipeline: NULL argument");
    return submit_pcm_impl(p, h_target_pcm, target_bits, target_frames, h_reference_pcm, reference_bits, reference_frames,
                           nullptr, h_out_pcm, out_bits, slot_out);
}

int mgb_pipeline_submit_pcm_profiled(mgb_pipeline* p, const void* h_target_pcm, int32_t target_bits, int64_t target_frames,
                                     const void* d_profile, void* h_out_pcm, int32_t out_bits, int32_t* slot_out) {
    MGB_REQUIRE(d_profile, MGB_ERR_INVALID, "pipeline: NULL argument");
    return submit_pcm_impl(p, h_target_pcm, target_bits, target_frames, nullptr, 16, 0, d_profile, h_out_pcm, out_bits,
                           slot_out);
}

int mgb_pipeline_streams(mgb_pipeline* p, void** h2d, void** compute, void** d2h) {
    MGB_REQUIRE(p, MGB_ERR_INVALID, "pipeline: NULL");
#ifdef MGB_EMULATE
    if (h2d) *h2d = nullptr;
    if (compute) *compute = nullptr;
    if (d2h) *d2h = nullptr;
#else
    if (h2d) *h2d = (void*)p->s_h2d;
    if (compute) *compute = (void*)p->s_compute;
    if (d2h) *d2h = (void*)p->s_d2h;
#endif
    return MGB_OK;
}

}  // extern "C"
