// K6l -- loudness targets: the search that drives the limiter until its output reads a given integrated loudness
// (include/matchering_b200.h, mgb_finalize_to_loudness / mgb_limit_to_loudness; DESIGN.md section 4).
//
//   y(x) = limit(s * 10^(x/20))   the unchanged limiter (halo or wide-window path, sample-peak or true-peak mode),
//                                 pre-gain gain * 10^(x/20) read from the search header, no post-gain
//   I(.)                          the meter's integrated loudness (loudness.cuh, integrated only)
//
//   loudness_target_init_kernel   one thread: x_1 from I(s), the pre-gain and early-out flag of pass 1
//   loudness_target_step_kernel   one thread, after pass k: record (x_k, I_k), stop or choose x_(k+1)
// The host cannot know how many passes a track needs without a synchronisation, so run_loudness_search launches all
// MGB_LOUDNESS_TARGET_MAX_PASSES of them; every kernel of a pass is a GATED instance that returns at once once the
// search has set its skip flag.  The true-peak detector runs once, before the first pass: d is linear in the input and
// the limiter applies its pre-gain to d.  The search itself is float64 in one thread, deterministic given the measured
// loudness values; tests/loudness_target_oracle.py restates it line for line.
// (included by limiter.cu, after loudness.cuh)
#pragma once
#include <math.h>

namespace mgb {

namespace {

// The search workspace's header (then the meter's workspace, 256-byte aligned).  Cleared before every search;
// every field a kernel reads is written on the stream before it.
struct TargetSearch {
    double pre_gain;     // gain * 10^(x/20) of the pass about to run: the limiter's pre-gain
    int32_t engaged;     // that pass's early-out flag (limiter_engaged_kernel's rule)
    int32_t skip;        // 1 once the search has stopped: every later pass's kernels return at once
    double measured;     // the last meter run's integrated loudness: I(s) before pass 1, then I(y(x_k))
    double peak_s;       // the peak of s the early-out rule scales (sample peak, or max(d) in true-peak mode)
    double gain;         // the correction gain (1 for mgb_limit_to_loudness)
    double x, x_lo, f_lo, x_hi, f_hi;  // the pass's drive; the bracket: largest drive below the target, smallest above
    int32_t has_lo, has_hi;
    int32_t undefined;   // I(s) = -inf: one pass at x = 0, then UNDEFINED
    int32_t pad;
    mgb_loudness_target_report report;
};
constexpr int64_t kTargetHeader = (sizeof(TargetSearch) + 255) / 256 * 256;

__device__ __forceinline__ void target_set_pass(TargetSearch* s, double x, double threshold) {
    const double k = pow(10.0, x / 20.0);
    s->x = x;
    s->pre_gain = s->gain * k;
    // engaged = not all(isclose(rectified, 1.0)) at the loudest frame (limiter_engaged_kernel, hyrax.py:83)
    const double peak = s->peak_s * k;
    const double r = fmax(peak, threshold) / threshold;
    s->engaged = (fabs(r - 1.0) <= 1e-8 + 1e-5 * 1.0) ? 0 : 1;
    s->skip = 0;
}

// peak_d: the peak of s itself (mgb_finalize's result_peak), or else peak_bits * gain (float bits of an absmax or max(d))
__global__ void loudness_target_init_kernel(mgb_loudness_target t, double threshold, const double* __restrict__ gain,
                                            const double* __restrict__ peak_d, const float* __restrict__ peak_bits,
                                            TargetSearch* __restrict__ s) {
    s->gain = gain ? *gain : 1.0;
    s->peak_s = peak_d ? *peak_d : (double)(*peak_bits) * s->gain;
    s->has_lo = s->has_hi = 0;
    s->x_lo = s->f_lo = s->x_hi = s->f_hi = 0.0;
    const double in = s->measured;
    mgb_loudness_target_report* r = &s->report;
    r->input_integrated = in;
    r->passes = 0;
    r->status = 0;
    for (int k = 0; k < MGB_LOUDNESS_TARGET_MAX_PASSES; ++k) r->trace_gain_db[k] = r->trace_integrated[k] = 0.0;
    s->undefined = isfinite(in) ? 0 : 1;
    target_set_pass(s, s->undefined ? 0.0 : fmin(t.target_lufs - in, t.max_gain_db), threshold);
}

__global__ void loudness_target_step_kernel(mgb_loudness_target t, double threshold, int k, TargetSearch* __restrict__ s,
                                            mgb_loudness_target_report* __restrict__ out) {
    if (s->skip) return;
    mgb_loudness_target_report* r = &s->report;
    const double x = s->x, I = s->measured, f = I - t.target_lufs, X = t.max_gain_db;
    r->trace_gain_db[k - 1] = x;
    r->trace_integrated[k - 1] = I;
    r->passes = k;
    r->gain_db = x;
    r->integrated = I;
    int status = 0;
    if (s->undefined || !isfinite(I)) {
        status = MGB_LOUDNESS_UNDEFINED;
    } else if (fabs(f) <= MGB_LOUDNESS_TARGET_TOLERANCE) {
        status = MGB_LOUDNESS_REACHED;
    } else if (f < 0.0 && x >= X) {
        status = MGB_LOUDNESS_UNREACHABLE;
    } else {
        if (f < 0.0 && (!s->has_lo || x > s->x_lo)) {
            s->has_lo = 1;
            s->x_lo = x;
            s->f_lo = f;
        }
        if (f > 0.0 && (!s->has_hi || x < s->x_hi)) {
            s->has_hi = 1;
            s->x_hi = x;
            s->f_hi = f;
        }
        if (s->has_lo && s->has_hi && s->x_hi - s->x_lo < 1e-3) status = MGB_LOUDNESS_BRACKET;
        else if (k >= MGB_LOUDNESS_TARGET_MAX_PASSES) status = MGB_LOUDNESS_PASSES;
    }
    if (status == 0) {
        // the secant through the last two points; slope 1 on the first pass and where the secant's is not positive
        double m = 1.0;
        if (k >= 2) {
            const double dx = x - r->trace_gain_db[k - 2];
            const double ms = dx != 0.0 ? (f - (r->trace_integrated[k - 2] - t.target_lufs)) / dx : 0.0;
            if (ms > 0.0 && isfinite(ms)) m = ms;
        }
        double c = x - f / m;
        // a limiter cannot raise loudness faster than 1 LU per dB: x - f bounds the root from the side already seen
        if (s->has_lo && !s->has_hi) c = fmax(c, s->x_lo - s->f_lo);
        if (s->has_hi && !s->has_lo) c = fmin(c, s->x_hi - s->f_hi);
        if (s->has_lo && s->has_hi && !(c > s->x_lo && c < s->x_hi)) c = 0.5 * (s->x_lo + s->x_hi);
        target_set_pass(s, fmin(c, X), threshold);
    } else {
        r->status = status;
        s->skip = 1;
    }
    *out = *r;
}

int clear_meter_words(const MeterWorkspace& w, cudaStream_t st) {
#ifdef MGB_EMULATE
    (void)st;
    memset(w.words, 0, w.words_bytes);
#else
    if (cudaMemsetAsync(w.words, 0, w.words_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    return MGB_OK;
}

// a pass's meter kernels up to the momentary windows, for one track (its look-back words cleared by the caller)
int launch_pass_windows(const mgb_loudness_params& lp, const float2* x, int64_t frames, const MeterWorkspace& w,
                        const int* skip, cudaStream_t st) {
    // the K-weighting does not depend on the oversampling; OS = 1 keeps the (unused) true peak cheap
    const MeterTables* tabs = (const MeterTables*)lp.d_tables;
    MGB_TRY(launch("loudness_kernel", loudness_kernel<1, true>, dim3((unsigned)w.chunks), dim3(NT), 0, st, lp, x,
                   (long long)frames, w.words, w.part, w.peak, tabs, skip));
    const long long B = lp.block;
    MGB_TRY(launch("loudness_fold_kernel", loudness_fold_kernel<true>, dim3((unsigned)((w.nb + 255) / 256)), dim3(256), 0, st,
                   B, (long long)w.nb, (const double*)w.part, w.energy, skip));
    return launch("loudness_windows_kernel", loudness_windows_kernel<true>, dim3((unsigned)((w.nm + 255) / 256)), dim3(256),
                  0, st, B, (long long)w.nb, (const double*)w.energy, w.mom, w.st, skip);
}

int launch_pass_integrated(const MeterWorkspace& w, const int* skip, double* integrated, cudaStream_t st) {
    return launch("loudness_integrated_kernel", loudness_integrated_kernel, dim3(1), dim3(kMeterFinishThreads), 0, st,
                  (long long)w.nm, (const double*)w.mom, skip, integrated);
}

int launch_pass_meter(const mgb_loudness_params& lp, const float2* x, int64_t frames, const MeterWorkspace& w,
                      const int* skip, double* integrated, cudaStream_t st) {
    MGB_TRY(clear_meter_words(w, st));
    MGB_TRY(launch_pass_windows(lp, x, frames, w, skip, st));
    return launch_pass_integrated(w, skip, integrated, st);
}

// ---- album loudness targets (mgb_album_finalize_to_loudness; DESIGN.md section 4 "Album loudness") ----------------
// One drive x for K limiters: the search above runs unchanged on the album's integrated loudness (the integrated
// kernel over the tracks' pooled momentary windows, carve_album_meter), and album_target_fanout_kernel turns each drive
// into every track's pre-gain and early-out flag.

// What the fan-out reads per track: the correction gain and the peak of s, as loudness_target_init_kernel reads them
struct AlbumTargetTrack {
    const double* gain;
    const double* peak_d;
    const float* peak_bits;
};
struct AlbumTargetTable {
    int count;
    AlbumTargetTrack t[MGB_MAX_ALBUM_TRACKS];
};

// The album search's header: the single-track search state, then the limiters' per-track inputs and what they follow
// from (read once, on the first fan-out: the true-peak maximum sits in the limiter words every pass clears)
struct AlbumTargetSearch {
    TargetSearch s;
    double pre_gain[MGB_MAX_ALBUM_TRACKS];
    int32_t engaged[MGB_MAX_ALBUM_TRACKS];
    double gain[MGB_MAX_ALBUM_TRACKS];
    double peak_s[MGB_MAX_ALBUM_TRACKS];
};
constexpr int64_t kAlbumTargetHeader = (sizeof(AlbumTargetSearch) + 255) / 256 * 256;

// one thread per track: target_set_pass's pre-gain and early-out flag at the drive the search chose, from the track's
// own gain and peak (taken as loudness_target_init_kernel takes them, on the fan-out after it: `first`)
__global__ void album_target_fanout_kernel(const __grid_constant__ AlbumTargetTable tab, double threshold, int first,
                                           AlbumTargetSearch* __restrict__ h) {
    const int t = threadIdx.x;
    if (t >= tab.count || h->s.skip) return;
    if (first) {
        const AlbumTargetTrack e = tab.t[t];
        h->gain[t] = *e.gain;
        h->peak_s[t] = e.peak_d ? *e.peak_d : (double)(*e.peak_bits) * h->gain[t];
    }
    const double k = pow(10.0, h->s.x / 20.0);
    h->pre_gain[t] = h->gain[t] * k;
    const double peak = h->peak_s[t] * k;
    const double r = fmax(peak, threshold) / threshold;
    h->engaged[t] = (fabs(r - 1.0) <= 1e-8 + 1e-5 * 1.0) ? 0 : 1;
}

}  // namespace

int loudness_target_validate(const mgb_loudness_target* t, const mgb_loudness_params* meter) {
    MGB_REQUIRE(t != nullptr, MGB_ERR_INVALID, "loudness target: target is NULL");
    MGB_REQUIRE(isfinite(t->target_lufs) && t->target_lufs < 0.0 && t->target_lufs > -70.0, MGB_ERR_INVALID,
                "loudness target: %g LUFS (finite, below 0 and above the absolute gate at -70)", t->target_lufs);
    MGB_REQUIRE(t->max_gain_db >= 0.0 && t->max_gain_db <= MGB_LOUDNESS_TARGET_MAX_GAIN_DB, MGB_ERR_INVALID,
                "loudness target: max_gain_db %g outside [0, %g]", t->max_gain_db, MGB_LOUDNESS_TARGET_MAX_GAIN_DB);
    MGB_TRY(loudness_validate(meter));
    MGB_REQUIRE(meter->d_tables != nullptr && ((uintptr_t)meter->d_tables & 15) == 0, MGB_ERR_INVALID,
                "loudness target: meter tables NULL or misaligned");
    return MGB_OK;
}

int64_t loudness_target_search_bytes(const mgb_loudness_params& meter, int64_t frames) {
    return kTargetHeader + carve_meter(meter, frames, nullptr).total;
}

// The whole search on `stream`.  in: the limiter's input (s / gain); s_metered: s as samples (the first meter run);
// out: the limited output; zero / zero_bytes: the limiter's look-back words (and ticket), cleared before every pass;
// ticket: a separate ticket word to clear as well (or null).  Arguments checked by the callers.
int run_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& t,
                        const float2* in, const float2* s_metered, float2* out, int64_t frames, const double* gain,
                        const double* peak_d, const float* peak_bits, void* zero, int64_t zero_bytes, int* ticket,
                        void* lookback, void* planes, const void* tables, const float* tp_d, void* search_ws,
                        mgb_loudness_target_report* report, cudaStream_t st) {
    TargetSearch* s = (TargetSearch*)search_ws;
    const MeterWorkspace w = carve_meter(meter, frames, (unsigned char*)search_ws + kTargetHeader);
    auto clear = [&](void* p, int64_t bytes) -> int {
#ifdef MGB_EMULATE
        memset(p, 0, bytes);
#else
        if (cudaMemsetAsync(p, 0, bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
        return MGB_OK;
    };
    MGB_TRY(clear(s, kTargetHeader));  // skip = 0 for the first meter run
    MGB_TRY(launch_pass_meter(meter, s_metered, frames, w, &s->skip, &s->measured, st));
    MGB_TRY(launch("loudness_target_init_kernel", loudness_target_init_kernel, dim3(1), dim3(1), 0, st, t, lp.threshold, gain,
                   peak_d, peak_bits, s));
    for (int k = 1; k <= MGB_LOUDNESS_TARGET_MAX_PASSES; ++k) {
        MGB_TRY(clear(zero, zero_bytes));
        if (ticket) MGB_TRY(clear(ticket, 16));
        MGB_TRY(launch_limiter(lp, in, out, frames, &s->pre_gain, nullptr, &s->engaged, ticket ? ticket : (int*)zero, lookback,
                               planes, tables, st, false, tp_d, &s->skip));
        MGB_TRY(launch_pass_meter(meter, out, frames, w, &s->skip, &s->measured, st));
        MGB_TRY(launch("loudness_target_step_kernel", loudness_target_step_kernel, dim3(1), dim3(1), 0, st, t, lp.threshold, k, s,
                       report));
    }
    return MGB_OK;
}

// Linked versions (mgb_finalize_versions_to_loudness): the main's search, unchanged, with its limiter reading the linked
// detector plane d (set true_peak so the kernels that take the plane serve it; in sample-peak mode d holds max(|L|, |R|),
// which P1 rectifies exactly as the sample path does) and its early-out taking max(d).  The header then holds the drive
// and the early-out flag of the pass the search ended on: one linked pass there writes every entry, the main's samples
// being that pass's own.
int run_versions_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& t,
                                 const VersionPlanes& vp, const float2* s_metered, int64_t frames, const double* gain,
                                 const float* d_max, const float* d, void* zero, int64_t zero_bytes, void* lookback, void* planes,
                                 const void* tables, void* search_ws, mgb_loudness_target_report* report, cudaStream_t st) {
    mgb_limiter_params lpd = lp;
    if (!lpd.true_peak) lpd.true_peak = 1;
    MGB_TRY(run_loudness_search(lpd, meter, t, vp.in[0], s_metered, vp.out[0], frames, gain, nullptr, d_max, zero, zero_bytes,
                                nullptr, lookback, planes, tables, d, search_ws, report, st));
    TargetSearch* s = (TargetSearch*)search_ws;
#ifdef MGB_EMULATE
    memset(zero, 0, zero_bytes);
#else
    if (cudaMemsetAsync(zero, 0, zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_limiter_versions(lp, vp, frames, &s->pre_gain, nullptr, &s->engaged, (int*)zero, lookback, planes, tables, d,
                                   st);
}

int64_t album_loudness_target_search_bytes(const mgb_loudness_params& meter, int tracks, const int64_t* frames) {
    MeterWorkspace w[MGB_MAX_ALBUM_TRACKS];
    return kAlbumTargetHeader + carve_album_meter(meter, tracks, frames, nullptr, w).total;
}

// The album's search on `stream`: run_loudness_search with every pass limiting and metering each track, the meter
// pooled over the album.  Arguments checked by the caller.
int run_album_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& t,
                              const AlbumSearchTrack* tracks, int count, const void* tables, void* search_ws,
                              mgb_loudness_target_report* report, cudaStream_t st) {
    AlbumTargetSearch* h = (AlbumTargetSearch*)search_ws;
    TargetSearch* s = &h->s;
    int64_t frames[MGB_MAX_ALBUM_TRACKS];
    AlbumTargetTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.count = count;
    for (int k = 0; k < count; ++k) {
        frames[k] = tracks[k].frames;
        tab.t[k].gain = tracks[k].gain;
        tab.t[k].peak_d = tracks[k].peak_d;
        tab.t[k].peak_bits = tracks[k].peak_bits;
    }
    MeterWorkspace w[MGB_MAX_ALBUM_TRACKS];
    const AlbumMeter a = carve_album_meter(meter, count, frames, (unsigned char*)search_ws + kAlbumTargetHeader, w);
    auto clear = [&](void* p, int64_t bytes) -> int {
#ifdef MGB_EMULATE
        memset(p, 0, bytes);
#else
        if (cudaMemsetAsync(p, 0, bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
        return MGB_OK;
    };
    auto pass_meter = [&](bool limited) -> int {
        MGB_TRY(clear_meter_words(a.all, st));
        for (int k = 0; k < count; ++k)
            MGB_TRY(launch_pass_windows(meter, limited ? tracks[k].out : tracks[k].s_metered, frames[k], w[k], &s->skip, st));
        return launch_pass_integrated(a.all, &s->skip, &s->measured, st);
    };
    auto fanout = [&](int first) {
        return launch("album_target_fanout_kernel", album_target_fanout_kernel, dim3(1), dim3(count), 0, st, tab,
                      lp.threshold, first, h);
    };
    MGB_TRY(clear(h, kAlbumTargetHeader));  // skip = 0 for the first meter run
    MGB_TRY(pass_meter(false));
    // (the init kernel's own pre-gain and flag are track 0's; the fan-out writes every track's)
    MGB_TRY(launch("loudness_target_init_kernel", loudness_target_init_kernel, dim3(1), dim3(1), 0, st, t, lp.threshold,
                   tracks[0].gain, tracks[0].peak_d, tracks[0].peak_bits, s));
    MGB_TRY(fanout(1));
    for (int pass = 1; pass <= MGB_LOUDNESS_TARGET_MAX_PASSES; ++pass) {
        for (int k = 0; k < count; ++k) {
            const AlbumSearchTrack& e = tracks[k];
            MGB_TRY(clear(e.zero, e.zero_bytes));
            MGB_TRY(launch_limiter(lp, e.in, e.out, e.frames, &h->pre_gain[k], nullptr, &h->engaged[k], (int*)e.zero,
                                   e.lookback, e.planes, tables, st, false, e.tp_d, &s->skip));
        }
        MGB_TRY(pass_meter(true));
        MGB_TRY(launch("loudness_target_step_kernel", loudness_target_step_kernel, dim3(1), dim3(1), 0, st, t, lp.threshold,
                       pass, s, report));
        if (pass < MGB_LOUDNESS_TARGET_MAX_PASSES) MGB_TRY(fanout(0));
    }
    return MGB_OK;
}

}  // namespace mgb

extern "C" {

int64_t mgb_loudness_target_workspace_bytes(const mgb_loudness_params* meter, int64_t frames) {
    if (mgb::loudness_validate(meter) != MGB_OK || frames <= 0) return -1;
    return mgb::loudness_target_search_bytes(*meter, frames);
}

int64_t mgb_album_loudness_target_workspace_bytes(const mgb_loudness_params* meter, int32_t tracks,
                                                  const mgb_track_layout* layouts) {
    if (mgb::loudness_validate(meter) != MGB_OK || tracks < 1 || tracks > MGB_MAX_ALBUM_TRACKS || layouts == nullptr) return -1;
    int64_t frames[MGB_MAX_ALBUM_TRACKS];
    for (int t = 0; t < tracks; ++t) {
        if (layouts[t].target_frames <= 0) return -1;
        frames[t] = layouts[t].target_frames;
    }
    return mgb::album_loudness_target_search_bytes(*meter, tracks, frames);
}

// workspace: mgb_limit's (limit_impl's layout), then the search's
int mgb_limit_to_loudness(const mgb_limiter_params* params, const mgb_loudness_params* meter, const mgb_loudness_target* target,
                          const float* d_in_lr, float* d_out_lr, int64_t frames, void* d_workspace, int64_t workspace_bytes,
                          mgb_loudness_target_report* d_report, void* stream) {
    using namespace mgb;
    MGB_REQUIRE(params != nullptr, MGB_ERR_INVALID, "limit_to_loudness: params is NULL");
    MGB_TRY(limiter_validate(*params));
    MGB_TRY(loudness_target_validate(target, meter));
    auto aligned = [](const void* p) { return p != nullptr && ((uintptr_t)p & 15) == 0; };
    MGB_REQUIRE(aligned(d_in_lr) && aligned(d_out_lr) && aligned(d_workspace) && aligned(d_report), MGB_ERR_INVALID,
                "limit_to_loudness: NULL or misaligned pointer (16 bytes needed)");
    MGB_REQUIRE(frames > 6, MGB_ERR_INVALID, "limit_to_loudness: the input must be longer than filtfilt's padlen (6)");
    MGB_REQUIRE((const void*)d_in_lr != (const void*)d_out_lr, MGB_ERR_INVALID,
                "limit_to_loudness: d_out_lr must not be d_in_lr (every pass reads the input)");
    MGB_REQUIRE(frames <= (int64_t)INT32_MAX * LC, MGB_ERR_INVALID, "limit_to_loudness: too many frames");
    const int64_t lim_bytes = mgb_limiter_workspace_bytes(params, frames);
    const int64_t need = lim_bytes + loudness_target_search_bytes(*meter, frames);
    MGB_REQUIRE(workspace_bytes >= need, MGB_ERR_WORKSPACE, "limit_to_loudness: workspace of %lld bytes, need %lld",
                (long long)workspace_bytes, (long long)need);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = (unsigned char*)d_workspace;
    // mgb_limit's layout: [0,4) peak bits  [16,20) ticket  [32,36) max(d)  [256, header) tables, then look-back words,
    // the wide-window planes and the detector plane
    const int64_t header = lim_bytes - limiter_lookback_bytes(*params, frames) - limiter_plane_bytes(*params, frames) -
                           true_peak_plane_bytes(*params, frames);
    const int64_t lookback_bytes = limiter_lookback_bytes(*params, frames);
#ifdef MGB_EMULATE
    memset(base, 0, 256);
#else
    if (cudaMemsetAsync(base, 0, 256, st) != cudaSuccess) return cuda_status("memset");
#endif
    void* tables = base + 256;
    MGB_TRY(launch_limiter_tables(*params, tables, st));
    const float2* x = (const float2*)d_in_lr;
    float* tp_d = nullptr;
    const float* peak = (const float*)base;
    if (params->true_peak) {
        tp_d = (float*)(base + header + lookback_bytes + limiter_plane_bytes(*params, frames));
        peak = (const float*)(base + 32);
        MGB_TRY(launch_true_peak_detect(params->true_peak, x, frames, tp_d, (float*)(base + 32), st));
    } else {
        MGB_TRY(launch_absmax(x, frames, (float*)base, st));
    }
    return run_loudness_search(*params, *meter, *target, x, x, (float2*)d_out_lr, frames, nullptr, nullptr, peak,
                               base + header, lookback_bytes, (int*)(base + 16), base + header,
                               base + header + lookback_bytes, tables, tp_d, base + lim_bytes, d_report, st);
}

}  // extern "C"
