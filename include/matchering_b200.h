/* matchering_b200 -- C ABI of the CUDA-native (H100, sm_90a) Matchering hot path.
 *
 * The reference (sergree/matchering v2.0.6) is pure Python and has no FFI layer; the seam this
 * library plugs into is the pair of Python call sites
 *     matchering/core.py:77-86      -> stages.main(target, reference, config, need_*...)
 *     matchering/stages.py:202      -> limiter.limit(array, config)
 * Each entry point below cites the reference function(s) it replaces.  The reference-side
 * binding a maintainer would add (a ctypes stub) is shown in INTEGRATION.md.
 *
 * Conventions
 *   - plain C, no exceptions: every call returns MGB_OK (0) or a negative mgb_status;
 *     mgb_last_error_string() describes the last failure on the calling thread.
 *   - audio is interleaved stereo float32: frame n = (L, R) at x[2n], x[2n+1].
 *   - all `d_*` pointers are DEVICE pointers owned by the caller and 16-byte aligned; nothing
 *     here allocates device memory.  Calls are asynchronous on `stream` (a cudaStream_t passed
 *     as void*); scalar results stay in device memory (mgb_track_state), so no call syncs.
 *   - Config-only tables (spline factorisations, LOWESS plan, filter coefficients, FFT twiddles)
 *     live in an mgb_plan that the host builds once per Config (matchering_b200/plan.py) and
 *     uploads; data-dependent arithmetic never runs on the host.
 */
#ifndef MATCHERING_B200_H
#define MATCHERING_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGB_VERSION 200 /* 0.2.0 */

typedef enum mgb_status {
    MGB_OK = 0,
    MGB_ERR_INVALID = -1,     /* bad argument (null / misaligned pointer, size out of range) */
    MGB_ERR_UNSUPPORTED = -2, /* legal reference Config this build has no kernel for */
    MGB_ERR_WORKSPACE = -3,   /* workspace too small */
    MGB_ERR_CUDA = -4         /* CUDA runtime / launch failure */
} mgb_status;

/* Limiter constants derived from Config (matchering/defaults.py:25-58, limiter/hyrax.py:44-72,
 * utils.py:50-55).  The hold and release low-passes are Butterworth sections of order 1 (the reference
 * default) or 2, as scipy.signal.butter returns them (transfer-function form, a[0] = 1), zero-padded above
 * the order.  Orders above 2 are rejected with MGB_ERR_UNSUPPORTED: at the limiter's cut-offs (7 Hz and 0.27 Hz
 * against 44.1 kHz) the transfer-function form the reference runs (scipy lfilter) is itself ill-conditioned
 * there -- measured in the build container, its float64 output differs from an extended-precision run of the
 * same coefficients by 5e-5 (release, order 3) to 2e-4 (hold, order 4), above the 1e-5 parity bound, and the
 * order-4 release filter's rounded coefficients are unstable (output 7e7) -- so there is no reference result
 * to be faithful to. */
#define MGB_MAX_FILTER_ORDER 2
typedef struct mgb_limiter_params {
    double threshold;   /* Config.threshold */
    int32_t reach;      /* make_odd(attack_samples) - 1 : half width of the centred max */
    int32_t hold;       /* hold_samples : length of the trailing max */
    int32_t warmup;     /* samples after which attack_c^n < 1e-8: the halo kernel's warm-up of the attack filter.  Where
                           warm-up, centred max and hold do not fit that kernel's span (8192 samples around a chunk),
                           the library runs its wide-window path, which carries every window and filter state
                           across chunks instead and needs more workspace (mgb_limiter_workspace_bytes) */
    int32_t hold_order;    /* LimiterConfig.hold_filter_order    (defaults.py:48-50) */
    int32_t release_order; /* LimiterConfig.release_filter_order (defaults.py:54-56) */
    int32_t true_peak;  /* 0: the reference's rectifier max(|L|, |R|).  1, 2 or 4: true-peak mode, the detector's oversampling
                           factor L (4 below 96 kHz, 2 below 192 kHz, 1 above): the limiter bounds the interpolated
                           signal, d[n] = max(u[n], u[n-1]) with u the largest |value| of both channels at n + ph/L,
                           ph = 0 .. L-1, through the meter's interpolator (mgb_true_peak_taps).  Other values:
                           MGB_ERR_INVALID */
    double attack_c;    /* exp(attack_filter_coefficient / attack_samples) */
    double hold_b[MGB_MAX_FILTER_ORDER + 1], hold_a[MGB_MAX_FILTER_ORDER + 1];       /* butter(order, hold_filter_coefficient, fs) */
    double release_b[MGB_MAX_FILTER_ORDER + 1], release_a[MGB_MAX_FILTER_ORDER + 1]; /* butter(order, release_filter_coefficient/release, fs) */
} mgb_limiter_params;

/* Config-only device tables (all double unless noted).  n_lin = fft_size/2+1,
 * n_log = (fft_size/2)*lin_log_oversampling+1. */
typedef struct mgb_plan {
    int32_t sample_rate;
    int32_t fft_size;          /* F: 512, 1024, 2048, 4096, 8192 or 16384 */
    int32_t n_lin, n_log;
    int32_t rms_correction_steps;
    int32_t lowess_k;          /* neighbourhood size int(frac*n_log + 1e-10) */
    int32_t lowess_nfit;       /* number of regression points */
    int32_t lowess_nrows;      /* distinct coefficient rows in d_lw_rows */
    int32_t lowess_it;         /* robustness iterations (dsp.py:103-106 `it`; 0 at the reference defaults).  > 0 makes
                                * LOWESS non-linear in the data: no smoothing operator, the direct chain re-weights the
                                * regressions with bisquare weights of the residuals (6 * median scale) */
    int32_t reserved0;
    double max_piece_size;     /* samples, as Config stores it (defaults.py:109) */
    double threshold;
    double min_value;
    mgb_limiter_params limiter;
    /* spline A: knots = linear grid, evaluated on the log grid (match_frequencies.py:60-61) */
    const double* d_sa_hinv;   /* [n_lin-1] 1/h_i */
    const double* d_sa_lu;     /* [3][n_lin-2] Thomas factors: sub/denominator, 1/denominator, super' */
    const double* d_sa_end;    /* [4] not-a-knot closure: M0 = e0*M1 + e1*M2, Mlast = e2*M[n-2] + e3*M[n-3] */
    const int32_t* d_sa_eval_idx; /* [n_log] interval index */
    const double* d_sa_eval_w;    /* [n_log][4] weights of (y_i, y_i+1, M_i, M_i+1) */
    /* spline B: knots = log grid, evaluated on the linear grid (match_frequencies.py:67-70) */
    const double* d_sb_hinv;   /* [n_log-1] */
    const double* d_sb_lu;     /* [3][n_log-2] */
    const double* d_sb_end;    /* [4] */
    const int32_t* d_sb_eval_idx; /* [n_lin] */
    const double* d_sb_eval_w;    /* [n_lin][4] */
    /* LOWESS (dsp.py:103-106, statsmodels semantics, it = 0) as a Config-only linear operator */
    const int32_t* d_lw_fit_idx; /* [lowess_nfit] abscissae with a local regression */
    const int32_t* d_lw_fit_left;/* [lowess_nfit] left edge of each neighbourhood [left, left+k) */
    const int32_t* d_lw_seg;     /* [n_log] position in fit_idx of the last regression point <= j */
    const double* d_lw_alpha;    /* [n_log] weight of the next regression point (delta interpolation) */
    const double* d_lw_rows;     /* [n_rows][lowess_k] regression coefficients: fit = row . y[left..] */
    const int32_t* d_lw_row_idx; /* [lowess_nfit] row of each regression point */
    /* window (scipy.signal.windows.hann(F), match_frequencies.py:99) */
    const double* d_hann;        /* [F] */
    /* FFT twiddles, filled by mgb_plan_fill_twiddles */
    void* d_tw_f32_F;    /* float2  table of the F-point transform  */
    void* d_tw_f32_2F;   /* float2  table of the 2F-point transform */
    void* d_tw_f64_F;    /* double2 table of the F-point transform  */
    void* d_tw_f64_2F;   /* double2 table of the 2F-point transform (then the 4F-point one for fft_size 2048, 4096) */
    void* d_limiter_tables; /* powers of the limiter's three poles (blocked-scan carries) */
    /* optional: the whole smoothing chain (spline, LOWESS, spline, overrides) as one Config-only matrix,
     * s = S m, S [n_lin][n_lin].  mgb_plan_build_operator builds it densely on the device; it is numerically
     * BANDED (LOWESS window 307 of 8193 log-grid points, spline influence decaying 0.27^n), so the plan keeps
     * only each row's band: row r = `count` entries of d_smooth_op from `offset` on, multiplying m[first ..]
     * (offsets even: 16-byte aligned rows; 4.8 MB instead of 33.6 MB at the default Config; what lies outside
     * the bands is below 1e-18 of the largest entry).  NULL = run the chain directly per track (slower:
     * latency-bound CTAs). */
    const double* d_smooth_op;
    const int32_t* d_smooth_op_rows; /* [n_lin][4]: offset, first column, count, 0 */
    /* native-rate plans only (mgb_match_frequencies_native; NULL in every other plan): how the native FIR's curve s'[j],
     * j = 0 .. n_lin-1 at frequencies j * sample_rate / fft_size, samples the analysis plan's smoothed curve s
     * (matchering_b200/plan.py native_tables).  Up to the edge f_e = 0.9 * R/2 of the analysis rate R,
     * s'[j] = s[i] + w (s[i+1] - s[i]) with i = d_native_idx[j], w = d_native_w[j]; above it d_native_idx[j] = -1 and
     * d_native_w[j] = t, the crossfade position (1 from R/2 on).  Entry n_lin is the edge itself, g_e = s(f_e). */
    const int32_t* d_native_idx; /* [n_lin + 1] */
    const double* d_native_w;    /* [n_lin + 1] */
} mgb_plan;

/* Per-track scalars, resident in device memory (one struct per track in flight). */
#define MGB_MAX_CORRECTION_STEPS 16
typedef struct mgb_track_state {
    double reference_peak;        /* max|reference|                         dsp.py:97            */
    double final_amplitude_coef;  /* normalize_reference's coefficient      match_levels.py:29-44 */
    double target_match_rms;      /* match_levels.py:62-71                                        */
    double reference_match_rms;   /* of the NORMALISED reference                                   */
    double rms_coefficient;       /* c0 = ref/max(eps,target)               match_levels.py:106-111 */
    double gain;                  /* product of the RMS-correction coefficients so far             */
    double correction[MGB_MAX_CORRECTION_STEPS]; /* stages.py:161-168, one per step                */
    double result_peak;           /* max|result| after the correction gain                         */
    double normalize_coef;        /* stages.py:186-191 coefficient of the normalised output        */
    float conv_peak_bits;         /* max|L|,|R| of the convolution output before correction        */
    int32_t target_loud_pieces;   /* number of pieces with rms >= average (target)                 */
    int32_t reference_loud_pieces;
    int32_t limiter_engaged;      /* 0 when hyrax.py:83-85 takes its early-out                     */
    int32_t steps_done;
    float fir_peak_mid_bits;      /* max |H_mid[k]| of the designed FIR spectrum (as applied)         */
    float fir_peak_side_bits;     /* max |H_side[k]|                                                  */
    int32_t conv_precise;         /* 1 when the convolution ran with float64 transforms (FIR gain x target peak too
                                     large for float32 frames, convolve.cu), 0 otherwise                       */
} mgb_track_state;

/* Geometry of one mastering job, computed by mgb_track_layout from sizes + plan (host side). */
typedef struct mgb_track_layout {
    int64_t target_frames, reference_frames;
    int64_t target_piece, reference_piece;        /* match_levels.py:47-59 */
    int32_t target_divisions, reference_divisions;
    int32_t target_slots, reference_slots;        /* analysis CTAs per piece */
    int64_t workspace_bytes;                      /* device scratch the stage calls need */
} mgb_track_layout;

int mgb_version(void);
const char* mgb_last_error_string(void);

/* Runtime switches for A/B measurements and tests.  "tma": 1 = cp.async.bulk frame loads (default),
 * 0 = plain coalesced loads.  "twiddle_chain": convolution FFTs build twiddle powers in registers
 * (1, default) or read them all from the table (0).  "conv_fused": the convolution keeps the last
 * forward pass, the spectral product, the first inverse pass and the epilogue in registers (1, default,
 * fft_size 4096 and 8192) or sends every pass through shared memory (0).  "conv_frame": overlap-save
 * frame of the convolution in FIR lengths, 4 (default: a 4F-point transform pair yields 3F outputs; fft_size
 * 2048 and 4096 with pieces of at least 3F samples) or 2 (2F-point pair, F outputs).  "conv_persistent": the 16384-point convolution frames are
 * walked by one CTA per SM with the next frame's bulk copy under the epilogue (1, default) or take one CTA each (0).
 * "analyze_chain": the analysis FFT builds twiddle powers in registers (1, default) or reads them all (0).  "design_direct": mgb_test_design_fir runs the
 * spline/LOWESS chain directly even when the plan has a smoothing operator.  "lookback_inclusive":
 * 0 makes limiter chunks publish aggregates only, so every look-back walks to its cut-off.  "limiter_ticket":
 * 1 hands the limiter's chunks out by an atomic ticket instead of the block index (0, default).  "poison_alloc"
 * (tests): 1 makes mgb_pipeline_create fill every device buffer it allocates with 0xFF bytes (NaN as a float or
 * double, -1 as an integer), so that a read of slot memory no kernel wrote shows up in the results; 0 (default)
 * leaves them as cudaMalloc returns them.
 * Returns MGB_ERR_INVALID for an unknown name. */
int mgb_set_option(const char* name, int value);

/* Measurement hooks (bench.py): number of kernel launches made by this library so far; and, while
 * profiling is enabled, a CUDA-event pair is recorded around every launch on its stream --
 * mgb_profile_collect synchronises the device, writes up to `capacity` durations (ms) in launch
 * order with their kernel names ('\n'-separated) and returns how many it wrote. */
long long mgb_launch_count(void);
int mgb_profile_enable(int on);
int mgb_profile_collect(char* names, int names_capacity, float* ms, int capacity);

/* Bytes of the four twiddle tables for `fft_size` and of d_limiter_tables, in the order of the
 * mgb_plan fields. */
int mgb_plan_twiddle_bytes(int32_t fft_size, int64_t bytes_out[5]);
/* Fill plan->d_tw_* and plan->d_limiter_tables (device buffers of the sizes above) on `stream`. */
int mgb_plan_fill_twiddles(const mgb_plan* plan, void* stream);

/* Build the DENSE smoothing operator of `plan` (plan->d_smooth_op may be NULL in the plan passed here)
 * into d_operator_out [n_lin*n_lin doubles, row-major]; the host keeps each row's band (matchering_b200/plan.py
 * band_operator) and uploads that as plan->d_smooth_op / _ptr / _lo using d_workspace of mgb_plan_operator_workspace_bytes. */
int64_t mgb_plan_operator_workspace_bytes(const mgb_plan* plan);
int mgb_plan_build_operator(const mgb_plan* plan, double* d_operator_out, void* d_workspace, int64_t workspace_bytes,
                            void* stream);

/* match_levels.py:47-59 piece geometry + launch geometry + workspace size. */
int mgb_track_layout_init(const mgb_plan* plan, int64_t target_frames, int64_t reference_frames,
                          mgb_track_layout* out);

/* ---- stage 1: stages.__match_levels (stages.py:38-104) --------------------------------------
 * One pass over each signal: max|x| (dsp.normalize, dsp.py:93-100), mid/side (dsp.lr_to_ms,
 * dsp.py:57-64), per-piece sum(mid^2) (dsp.batch_rms, dsp.py:80-86) and per-piece sums of
 * |rfft(frame)| for mid and side (match_frequencies.__average_fft, match_frequencies.py:30-42),
 * then the loudest-piece masks, match RMS values, c0 and final_amplitude_coefficient
 * (match_levels.py:62-131) into *d_state. */
int mgb_match_levels(const mgb_plan* plan, const mgb_track_layout* layout, const float* d_target_lr,
                     const float* d_reference_lr, void* d_workspace, mgb_track_state* d_state, void* stream);

/* ---- reference profiles: analyse a reference once, master any number of targets against it ----
 * Everything stages 2-4 take from the reference depends on the reference and on five Config fields only
 * (sample_rate, fft_size, max_piece_size, threshold, min_value): its peak and final_amplitude_coefficient
 * (match_levels.py:29-44 normalize_reference), the match RMS of the normalised reference and its number of
 * loud pieces (match_levels.py:47-71 analyze_levels), and the two average spectra of the normalised reference
 * over its loudest pieces (match_frequencies.py:30-42,93-94 __average_fft).  A profile holds exactly those, in
 * one device blob of mgb_reference_profile_bytes(): this header, then double spectra[2][n_lin] (mid, side:
 * mean |rfft(frame)| / fft_size of the normalised reference over its loud pieces).  A job that takes its
 * reference from a profile computes exactly what the job that takes the reference's samples computes: the same
 * level statistics, c0 and FIR bit for bit, and from there on the same kernels on the same data (whose per-piece
 * float64 atomic sums make two device runs of ONE job differ in the last bits; where the order is fixed, as in the
 * CPU emulator, outputs and mgb_track_state are bit-identical too).  Every Config field outside the fingerprint (limiter, LOWESS,
 * lin_log_oversampling, rms_correction_steps) may differ between the profile's Config and the job's. */
#define MGB_REFERENCE_PROFILE_VERSION 1
typedef struct mgb_reference_profile {
    int32_t version;              /* MGB_REFERENCE_PROFILE_VERSION */
    int32_t sample_rate, fft_size, n_lin;
    double max_piece_size, threshold, min_value;    /* the Config fields the reference side depends on */
    int64_t reference_frames, reference_piece;
    int32_t reference_divisions, reference_loud_pieces;
    double reference_peak;        /* max|reference|                                  */
    double final_amplitude_coef;  /* normalize_reference's coefficient               */
    double reference_match_rms;   /* of the NORMALISED reference                      */
    int64_t reserved;             /* 0; the spectra follow at sizeof(mgb_reference_profile) = 96 */
} mgb_reference_profile;

/* bytes of a profile blob for this plan's fft_size (header + spectra) */
int64_t mgb_reference_profile_bytes(const mgb_plan* plan);
/* device scratch mgb_analyze_reference needs for a reference of `reference_frames` frames */
int64_t mgb_reference_workspace_bytes(const mgb_plan* plan, int64_t reference_frames);
/* One analysis pass over the reference (the pass mgb_match_levels makes over it) and its fold into a profile
 * at d_profile (device, mgb_reference_profile_bytes).  Asynchronous on `stream`. */
int mgb_analyze_reference(const mgb_plan* plan, const float* d_reference_lr, int64_t reference_frames, void* d_workspace,
                          int64_t workspace_bytes, void* d_profile, void* stream);
/* Compares a HOST copy of a profile's header with the plan: version, sample_rate, fft_size, n_lin, max_piece_size,
 * threshold and min_value must match exactly (MGB_ERR_INVALID naming the first field that does not).  The device
 * entry points below cannot read the device header without a synchronisation, so they trust the caller to have
 * made this check. */
int mgb_reference_profile_check(const mgb_plan* plan, const mgb_reference_profile* h_header);
/* Layout of a job whose reference comes from a profile: the target's geometry as mgb_track_layout_init gives it;
 * reference_frames, reference_piece, reference_divisions and reference_slots are 0, which marks the layout as
 * profiled.  Its workspace has no reference regions and one region for a copy of the profile. */
int mgb_track_layout_init_profiled(const mgb_plan* plan, int64_t target_frames, mgb_track_layout* out);
/* Stage 1 with the reference from a profile: copies the blob into the workspace on `stream` (the caller may reuse
 * or free d_profile once that copy has run), analyses the target, and the next stage's first kernel combines the
 * target's statistics with the profile's.  MGB_ERR_INVALID with a paired layout, as mgb_match_levels gives with a
 * profiled one.  Stages 2-4 take a profiled layout like a paired one. */
int mgb_match_levels_profiled(const mgb_plan* plan, const mgb_track_layout* layout, const float* d_target_lr,
                              const void* d_profile, void* d_workspace, mgb_track_state* d_state, void* stream);

/* ---- stage 2: stages.__match_frequencies (stages.py:107-135) --------------------------------
 * FIR design for mid and side (match_frequencies.get_fir, :78-101, incl. __smooth_exponentially
 * :45-75 and dsp.smooth_lowess) and convolution of the level-matched target with both FIRs
 * (match_frequencies.convolve :104-119 == scipy fftconvolve 'same'), mid/side -> L/R
 * (dsp.ms_to_lr, dsp.py:67-68).  Writes the un-corrected result (d_result_lr), the first correction
 * step's per-piece sum(clip(mid)^2) and, per piece, the list of mid samples loud enough that a later
 * correction step may clip them (workspace).  The later stages read d_result_lr again: it must stay
 * unchanged until mgb_finalize has run.
 * d_fir_out (optional, may be NULL): [2][F] doubles, the mid and side FIRs, for inspection. */
int mgb_match_frequencies(const mgb_plan* plan, const mgb_track_layout* layout, const float* d_target_lr,
                          float* d_result_lr, double* d_fir_out, void* d_workspace, mgb_track_state* d_state,
                          void* stream);
/* The FIR design of mgb_match_frequencies without its convolution: the level statistics into *d_state, the mid and
 * side FIRs' spectra and the smoothed matching curves into the workspace.  mgb_match_frequencies is this call followed
 * by the convolution. */
int mgb_design_frequencies(const mgb_plan* plan, const mgb_track_layout* layout, double* d_fir_out, void* d_workspace,
                           mgb_track_state* d_state, void* stream);

/* ---- native-rate masters: stages 2-4 at the target's own rate R' (DESIGN.md section 4) -----------------------------
 * The analysis job (plan, layout, d_workspace, d_state at the internal rate R) has run stage 1 and
 * mgb_design_frequencies on the target resampled to R.  This call carries its smoothed curves to the FIR of
 * native_plan (rate R', fft_size F' = F * 2^round(log2(R'/R)), with the d_native_* tables for R, F and R'), folds c0
 * into that FIR's spectra, and convolves the native target (native_layout->target_frames frames at R') into
 * d_native_result.  *d_native_state starts as a copy of *d_state (c0, the reference's match RMS, the final amplitude
 * coefficient); the native FIR's peaks and the native target's peak choose the convolution's precision.  After it,
 * mgb_correct_levels, mgb_finalize and mgb_finalize_to_loudness take native_plan, native_layout, d_native_workspace
 * and d_native_state as they are.  native_layout is a profiled layout (mgb_track_layout_init_profiled) of
 * native_plan.  MGB_ERR_INVALID: equal rates, an F' that does not follow from the rates, missing tables, a paired
 * native layout; MGB_ERR_UNSUPPORTED: F' outside 512 .. 16384.
 * d_fir_out (optional): [2][F'] doubles, the native mid and side FIRs. */
int mgb_match_frequencies_native(const mgb_plan* plan, const mgb_track_layout* layout, const void* d_workspace,
                                 const mgb_track_state* d_state, const mgb_plan* native_plan,
                                 const mgb_track_layout* native_layout, const float* d_native_target, float* d_native_result,
                                 double* d_fir_out, void* d_native_workspace, mgb_track_state* d_native_state, void* stream);

/* ---- album mastering: one level match and one matching FIR for K tracks (DESIGN.md section 4) --------------------
 * Stages 1-3 of K jobs whose reference comes from one profile, with their statistics pooled over the album:
 *   - stage 1: every piece (t, p) of every track counts once in the average, the loud mask and the match RMS
 *     (match_levels.py:62-71 over the union of the tracks' pieces); one c0 = reference match RMS / max(eps, album match);
 *   - stage 2: the target spectra are the mean |rfft| over every boxcar frame of every loud piece of every track, ONE
 *     FIR is designed from them and every track is convolved with it (each track picks its float32 or float64
 *     convolution from its own peak, as a single job does);
 *   - stage 3: each step's coefficient comes from the per-piece sums of all tracks, pooled the same way, and multiplies
 *     every track.
 * Each track keeps its own piece layout.  After the call every track is where mgb_correct_levels leaves a single job:
 * the caller runs mgb_finalize (or mgb_finalize_to_loudness) per track with its layout, workspace and state.  A one-track
 * album computes bit for bit what the profiled job computes.  The tracks' analysis, convolution and finalize kernels are
 * the single job's; the pooled steps are one launch each over all tracks. */
#define MGB_MAX_ALBUM_TRACKS 64
typedef struct mgb_album_track {
    const mgb_track_layout* layout; /* mgb_track_layout_init_profiled of the plan */
    const float* d_target_lr;       /* layout->target_frames stereo frames at the plan's rate */
    float* d_result_lr;             /* the stage-2 result, as mgb_match_frequencies writes it (not d_target_lr) */
    void* d_workspace;              /* layout->workspace_bytes */
    mgb_track_state* d_state;
} mgb_album_track;
/* device scratch of the album's design (the FIR's spectra on both convolution grids); -1 for bad arguments */
int64_t mgb_album_workspace_bytes(const mgb_plan* plan, int32_t tracks, const mgb_track_layout* layouts);
/* MGB_ERR_INVALID: no tracks or more than MGB_MAX_ALBUM_TRACKS, NULL or misaligned pointers, a layout that is not a
 * profiled layout of this plan, a result buffer that is its track's target, a profile whose header does not match the
 * plan (mgb_reference_profile_check; the call reads the header back, which waits for `stream`).  MGB_ERR_WORKSPACE: a
 * short album workspace.  MGB_ERR_UNSUPPORTED: more pieces than the pooled statistics fit in one CTA's shared memory.
 * d_fir_out (optional): [2][F] doubles, the album's mid and side FIRs. */
int mgb_album_match(const mgb_plan* plan, int32_t tracks, const mgb_album_track* t, const void* d_profile, double* d_fir_out,
                    void* d_album_ws, int64_t album_ws_bytes, void* stream);

/* ---- stage 3: stages.__correct_levels (stages.py:138-170) -----------------------------------
 * rms_correction_steps iterations of clip -> per-piece RMS -> loudest mask -> coefficient.  The
 * coefficients accumulate in d_state->gain; the samples are scaled once, by the consumer.  A step
 * reads the loud lists, or the result of mgb_match_frequencies where a list cannot give the exact sum. */
int mgb_correct_levels(const mgb_plan* plan, const mgb_track_layout* layout, void* d_workspace,
                       mgb_track_state* d_state, void* stream);

/* ---- stage 4: stages.__finalize (stages.py:173-207) -----------------------------------------
 * Any of the three outputs may be NULL (the reference's need_* flags, core.py:81-85):
 *   d_out_limited     = limit(result * gain) * final_amplitude_coefficient   (stages.py:201-203)
 *   d_out_no_limiter  = result * gain                                       (stages.py:205)
 *   d_out_normalized  = normalize(result * gain, normalize_clipped=True)    (stages.py:185-191) */
int mgb_finalize(const mgb_plan* plan, const mgb_track_layout* layout, const float* d_result_lr,
                 float* d_out_limited, float* d_out_no_limiter, float* d_out_normalized, void* d_workspace,
                 mgb_track_state* d_state, void* stream);

/* ---- limiter.limit (limiter/hyrax.py:78-99), standalone ---------------------------------------
 * d_out = limit(d_in) for `frames` stereo frames.  d_engaged (int32, device) receives 0 when the
 * reference would return its input untouched (hyrax.py:83-85; d_out is then a copy of d_in).  In true-peak mode
 * (params->true_peak != 0) the early-out and the gain follow the detector d instead of the sample peaks, and the
 * workspace holds d as well (4 B per frame). */
int64_t mgb_limiter_workspace_bytes(const mgb_limiter_params* params, int64_t frames);
int mgb_limit(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
              void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream);
/* The true-peak mode's interpolator (mgb_limiter_params.true_peak): the 12 * oversample + 1 taps
 * sinc((m - 6 L)/L) * kaiser(12 L + 1, beta = 8)[m], computed on the host in long double, into out (host memory).
 * oversample 1, 2 or 4; MGB_ERR_INVALID otherwise.  The same taps as the loudness meter's tp_taps. */
int mgb_true_peak_taps(int32_t oversample, double* out);

/* ---- loudness meter: ITU-R BS.1770-4 / EBU R 128 ---------------------------------------------
 * Integrated loudness (gated), loudness range (EBU Tech 3342), maximum momentary and short-term loudness,
 * sample peak and true peak of `frames` interleaved stereo float32 frames, both channels weighted 1.
 * K-weighting = the shelf section, then the high-pass section, each an order-2 recursive filter started from rest
 * (scipy.signal.lfilter), run in float64.  Sub-blocks of `block` = (sample_rate + 5) / 10 frames; momentary =
 * 4 sub-blocks, short-term = 30, complete windows only.  True peak = max |upfirdn(tp_taps, x_channel, up=oversample)|.
 * matchering_b200/plan.py (loudness_constants) derives every field below from the sample rate. */
#define MGB_LOUDNESS_MAX_TAPS 49 /* 12 * oversample + 1 at oversample 4 */
typedef struct mgb_loudness_params {
    int32_t sample_rate;      /* 8000 .. 384000 */
    int32_t block;            /* sub-block length in frames: (sample_rate + 5) / 10 */
    int32_t oversample;       /* true-peak oversampling: 4 below 96 kHz, 2 below 192 kHz, else 1 */
    int32_t taps;             /* 12 * oversample + 1 */
    double shelf_b[3], shelf_a[3];       /* K-weighting stage 1 (a[0] = 1) */
    double highpass_b[3], highpass_a[3]; /* K-weighting stage 2 (a[0] = 1) */
    double tp_taps[MGB_LOUDNESS_MAX_TAPS]; /* true-peak interpolator, `taps` used */
    const void* d_tables;     /* mgb_loudness_tables_bytes() of device memory filled by mgb_loudness_fill_tables */
} mgb_loudness_params;

/* Written to device memory by mgb_loudness.  Loudness in LUFS, range in LU: -inf where undefined (no complete
 * window, or every window gated out); loudness_range 0 when no short-term window survives its gates.  Peaks are
 * linear (max |x| and max |interpolated x| per channel). */
typedef struct mgb_loudness_result {
    double integrated;
    double loudness_range;
    double momentary_max;
    double short_term_max;
    double sample_peak[2];
    double true_peak[2];
    int64_t momentary_count;   /* complete 400 ms windows: max(0, sub-blocks - 3) */
    int64_t short_term_count;  /* complete 3 s windows: max(0, sub-blocks - 29) */
} mgb_loudness_result;

/* device bytes of the rate's filter tables (powers of the sections' companion matrices) */
int64_t mgb_loudness_tables_bytes(void);
/* builds the tables on the host and copies them to d_tables on `stream` (staged before the call returns) */
int mgb_loudness_fill_tables(const mgb_loudness_params* params, void* d_tables, void* stream);
int64_t mgb_loudness_workspace_bytes(const mgb_loudness_params* params, int64_t frames);
/* Meters d_lr into *d_result (device).  Asynchronous on `stream`; the workspace needs no initialisation.
 * MGB_ERR_INVALID for a rate outside [8000, 384000], fields that do not follow from the rate, no frames, a
 * pointer that is not 16-byte aligned or a workspace smaller than mgb_loudness_workspace_bytes. */
int mgb_loudness(const mgb_loudness_params* params, const float* d_lr, int64_t frames, void* d_workspace,
                 int64_t workspace_bytes, mgb_loudness_result* d_result, void* stream);

/* ---- loudness targets: drive the limiter until the limited output reads a given integrated loudness ----
 * Let s be the signal the limiter would take (mgb_finalize: result * gain, the correction gain; mgb_limit: the input),
 * T the target (LUFS) and X the largest drive (dB).  The output is y(x) = limit(s * 10^(x/20)) at the drive x the search
 * ends on, the unchanged limiter
 * in the plan's (params') peak mode, WITHOUT final_amplitude_coefficient: that coefficient only carries a quiet
 * reference's level, which the target replaces, and keeping it would move the ceiling below the threshold.  x* comes
 * from a search on the device (one thread, float64; I = the meter's integrated loudness, f = I - T):
 *   I_s = I(s).  -inf (silence, or no complete 400 ms window): one pass at x = 0, status UNDEFINED.
 *   x_1 = min(T - I_s, X).  Pass k: limit at x_k, meter, f_k.  Stop on |f_k| <= MGB_LOUDNESS_TARGET_TOLERANCE
 *   (REACHED), f_k < 0 at x_k >= X (UNREACHABLE), a bracket narrower than 1e-3 dB (BRACKET), MAX_PASSES passes
 *   (PASSES), or I(y(x_k)) = -inf (UNDEFINED).  Otherwise the secant through the last two points (slope 1 on the first
 *   pass, and where the secant's slope is not positive), held to at least x_lo - f_lo while only points below the
 *   target are known and to at most x_hi - f_hi while only points above are known (a limiter cannot raise loudness
 *   faster than 1 LU per dB), replaced by the bracket's midpoint where it leaves the open bracket, capped at X.
 * The output holds the last pass's samples, and the report the loudness measured on them.  Every pass is launched
 * (the host cannot know how many a track needs without a synchronisation); the kernels of a pass the search did
 * not need return at once.  Nothing here synchronises. */
#define MGB_LOUDNESS_TARGET_MAX_PASSES 8
#define MGB_LOUDNESS_TARGET_TOLERANCE 0.01 /* LU */
#define MGB_LOUDNESS_TARGET_MAX_GAIN_DB 48.0
enum { MGB_LOUDNESS_REACHED = 1, MGB_LOUDNESS_UNREACHABLE = 2, MGB_LOUDNESS_BRACKET = 3, MGB_LOUDNESS_PASSES = 4,
       MGB_LOUDNESS_UNDEFINED = 5 };
typedef struct mgb_loudness_target {
    double target_lufs;  /* finite, below 0 and above the absolute gate (-70 LUFS) */
    double max_gain_db;  /* X, in [0, MGB_LOUDNESS_TARGET_MAX_GAIN_DB] */
} mgb_loudness_target;
typedef struct mgb_loudness_target_report {
    double gain_db;          /* x*: drive into the limiter, on top of the correction gain */
    double integrated;       /* I(y(x*)), LUFS, measured on the samples written */
    double input_integrated; /* I_s */
    double trace_gain_db[MGB_LOUDNESS_TARGET_MAX_PASSES], trace_integrated[MGB_LOUDNESS_TARGET_MAX_PASSES]; /* passes used */
    int32_t passes, status;  /* MGB_LOUDNESS_REACHED / _UNREACHABLE / _BRACKET / _PASSES / _UNDEFINED */
} mgb_loudness_target_report;
/* The search's own workspace (a header, then the meter's workspace); -1 for bad arguments.  Needs no initialisation. */
int64_t mgb_loudness_target_workspace_bytes(const mgb_loudness_params* meter, int64_t frames);
/* Stage 4's limited output at the target, after mgb_correct_levels, into d_out_limited (which also serves as the
 * search's scratch until the first pass, so it must not be d_result_lr: MGB_ERR_INVALID).  d_workspace is the job's; it keeps its layout.  d_report: device. */
int mgb_finalize_to_loudness(const mgb_plan* plan, const mgb_track_layout* layout, const mgb_loudness_params* meter,
                             const mgb_loudness_target* target, const float* d_result_lr, float* d_out_limited,
                             void* d_workspace, void* d_search_ws, int64_t search_ws_bytes, mgb_track_state* d_state,
                             mgb_loudness_target_report* d_report, void* stream);
/* mgb_limit at the target; one workspace of mgb_limiter_workspace_bytes + mgb_loudness_target_workspace_bytes.  Every
 * pass reads d_in_lr, so d_out_lr must be another buffer (MGB_ERR_INVALID). */
int mgb_limit_to_loudness(const mgb_limiter_params* params, const mgb_loudness_params* meter, const mgb_loudness_target* target,
                          const float* d_in_lr, float* d_out_lr, int64_t frames, void* d_workspace, int64_t workspace_bytes,
                          mgb_loudness_target_report* d_report, void* stream);

/* ---- album loudness: an album metered as one programme, and driven to a target with one drive (DESIGN.md section 4) --
 * The album meter: each of the K tracks is K-weighted from rest and cut into its own sub-blocks and windows, exactly as
 * mgb_loudness does; no window straddles two tracks.  The album's integrated loudness and loudness range are then
 * mgb_loudness's gates and percentiles over the union of all tracks' windows (every window counts once), and its
 * maxima and peaks the maxima over the tracks (libebur128's ebur128_loudness_global_multiple / _range_multiple).  It is
 * not the meter of the tracks concatenated.  A one-track album is mgb_loudness bit for bit. */
int64_t mgb_album_loudness_workspace_bytes(const mgb_loudness_params* params, int32_t tracks, const int64_t* frames);
/* d_lr[t]: frames[t] stereo frames per track (host arrays of device pointers).  *d_album_result: the album's result,
 * its momentary_count / short_term_count the pooled counts.  d_track_results (optional, device, [tracks]): each
 * track's own mgb_loudness result.  MGB_ERR_INVALID: no tracks or more than MGB_MAX_ALBUM_TRACKS, a track without
 * frames, NULL or misaligned pointers; MGB_ERR_WORKSPACE: a short workspace.  The workspace needs no initialisation. */
int mgb_album_loudness(const mgb_loudness_params* params, int32_t tracks, const float* const* d_lr, const int64_t* frames,
                       void* d_workspace, int64_t workspace_bytes, mgb_loudness_result* d_album_result,
                       mgb_loudness_result* d_track_results, void* stream);
/* The album target, after mgb_album_match: s_t = result_t * gain (the album's correction gain, the same in every
 * track), y_t(x) = limit_t(s_t * 10^(x/20)) with each track's own limiter in the plan's peak mode and no
 * final_amplitude_coefficient, and ONE drive x for every track, searched by mgb_finalize_to_loudness's rule with I the
 * album meter's integrated loudness of y_1(x) .. y_K(x).  Where no limiter engages the tracks keep their relative levels
 * exactly.  d_out_limited[t] (host array of device pointers) receives y_t(x*); it also stages s_t, so it must not be the
 * track's d_result_lr.  d_report (device): the album's report.  Each track's workspace and state are its
 * mgb_album_match entry's.  MGB_ERR_INVALID: bad track count, NULL or misaligned pointers, an output that is its track's
 * result, a layout not of this plan, a meter rate that is not the plan's, a target mgb_finalize_to_loudness rejects;
 * MGB_ERR_WORKSPACE: a short search workspace.  A one-track album computes what mgb_finalize_to_loudness computes, bit
 * for bit.  Nothing here synchronises. */
int64_t mgb_album_loudness_target_workspace_bytes(const mgb_loudness_params* meter, int32_t tracks,
                                                  const mgb_track_layout* layouts);
int mgb_album_finalize_to_loudness(const mgb_plan* plan, int32_t tracks, const mgb_album_track* t,
                                   float* const* d_out_limited, const mgb_loudness_params* meter,
                                   const mgb_loudness_target* target, void* d_search_ws, int64_t search_ws_bytes,
                                   mgb_loudness_target_report* d_report, void* stream);

/* ---- linked versions: a mix's instrumental, a cappella, TV mix or clean edit mastered with the main's match and its
 * limiter gain, so that every version nulls against the master (DESIGN.md section 4 "Linked versions") --------------
 * The main x_0 runs stages 1-3 as a single job (paired or profiled).  Each version x_v (the same frame count) is then
 * convolved with the main's FIR spectra (c0 folded in) and scaled by the main's correction gain G; no correction step
 * runs on it.  Stage 4 limits all of them with ONE gain envelope e, computed from D[n] = the maximum over the main and
 * every version of the limiter's detector (max(|L|, |R|), or the true-peak detector d[n]) of s_v = result_v * G:
 *   limited_v    = s_v * e * final_amplitude_coefficient   (the same float64 gain for every entry)
 *   no limiter   = s_v
 *   normalized_v = s_v / max(eps, G * max(D) / threshold)
 * Where no version's detector exceeds the main's, the main's outputs are the single job's bit for bit. */
#define MGB_MAX_VERSIONS 8
typedef struct mgb_version_track {
    const mgb_track_layout* layout; /* mgb_track_layout_init_profiled of the plan, for the main's frame count */
    const float* d_target_lr;       /* the version: layout->target_frames stereo frames at the plan's rate */
    float* d_result_lr;             /* its stage-2 result (neither a target nor another result) */
    void* d_workspace;              /* layout->workspace_bytes, its own */
    mgb_track_state* d_state;       /* its own; starts as a copy of the main's */
} mgb_version_track;
/* Stage 2 of `versions` versions (1 .. MGB_MAX_VERSIONS) with the main's FIR, after the main's mgb_correct_levels
 * (plan, layout, d_workspace and d_state are the main's).  A version takes the float64 convolution where the main does or
 * where the main's rule, applied to the version's own peak, calls for it.  MGB_ERR_INVALID: a bad count, NULL or
 * misaligned pointers, a frame count that is not the main's, a layout that is not this plan's profiled layout of it, a
 * result that is any target or result. */
int mgb_version_match_frequencies(const mgb_plan* plan, const mgb_track_layout* layout, const void* d_workspace,
                                  const mgb_track_state* d_state, int32_t versions, const mgb_version_track* v, void* stream);
/* One entry of stage 4: entry 0 is the main (its d_result_lr from mgb_match_frequencies), then the versions' results.
 * Each output may be NULL, as in mgb_finalize. */
typedef struct mgb_version_entry {
    const float* d_result_lr;
    float* d_out_limited;
    float* d_out_no_limiter;
    float* d_out_normalized;
} mgb_version_entry;
/* device scratch of stage 4 with versions (the linked detector plane, its maximum, a copy of the main's scalars); -1 for
 * bad arguments */
int64_t mgb_versions_workspace_bytes(const mgb_plan* plan, const mgb_track_layout* layout);
/* Stage 4 of the main and its versions: `entries` = 1 + versions (1 .. 1 + MGB_MAX_VERSIONS) entries, the main first;
 * d_workspace and d_state are the main's.  d_state is not changed.  MGB_ERR_INVALID: a bad count, NULL or misaligned
 * pointers, an output that aliases any result or another output; MGB_ERR_WORKSPACE: a short versions workspace. */
int mgb_finalize_versions(const mgb_plan* plan, const mgb_track_layout* layout, int32_t entries, const mgb_version_entry* e,
                          void* d_workspace, const mgb_track_state* d_state, void* d_versions_ws, int64_t versions_ws_bytes,
                          void* stream);
/* The limited outputs at a loudness target (mgb_finalize_to_loudness's search on the main's integrated loudness, its
 * limiter reading D): every entry receives limit at the drive x* the search ends on, no final_amplitude_coefficient.
 * Every entry's d_out_limited is required, and its other two outputs must be NULL (mgb_finalize_versions writes those).
 * d_report (device): the main's report.  Errors as mgb_finalize_versions and mgb_finalize_to_loudness. */
int mgb_finalize_versions_to_loudness(const mgb_plan* plan, const mgb_track_layout* layout, const mgb_loudness_params* meter,
                                      const mgb_loudness_target* target, int32_t entries, const mgb_version_entry* e,
                                      void* d_workspace, const mgb_track_state* d_state, void* d_versions_ws,
                                      int64_t versions_ws_bytes, void* d_search_ws, int64_t search_ws_bytes,
                                      mgb_loudness_target_report* d_report, void* stream);

/* ---- whole job with HOST buffers (the call the end-to-end benchmark times) --------------------
 * h_* are host pointers (pinned for full speed).  Copies target and reference to the device,
 * runs stages 1-4 and copies the requested outputs back; synchronises `stream` before returning.
 * d_target / d_reference / d_result / d_out are caller-provided device staging buffers of
 * target_frames (reference_frames) stereo frames each. */
int mgb_process_host(const mgb_plan* plan, const mgb_track_layout* layout, const float* h_target_lr,
                     const float* h_reference_lr, float* h_out_limited, float* h_out_no_limiter,
                     float* h_out_normalized, float* d_target_lr, float* d_reference_lr, float* d_result_lr,
                     float* d_out_lr, void* d_workspace, mgb_track_state* d_state, mgb_track_state* h_state_out,
                     void* stream);

/* ---- the reference's own seam with the reference's own buffers ---------------------------------
 * matchering/core.py:77-86 calls stages.main(target, reference, ...) with PAGEABLE float64 (frames, 2)
 * numpy arrays and gets float64 arrays back; matchering/stages.py:202 calls limit() the same way.
 * mgb_host_io moves such arrays at link speed without asking the caller to pin anything: a persistent
 * pool of worker threads narrows float64 -> float32 (or copies float32) into a ring of pinned chunks
 * while the calling thread issues one asynchronous copy per finished chunk; results come back either
 * widened on the device and DMA'd straight into pinned memory from mgb_host_alloc (one copy, no host
 * pass), or as float32 chunks through the same ring, widened by the workers (half the bytes over the link).
 * `*_width` = bytes per sample of the host arrays: 4 (float32) or 8 (float64).
 * threads / chunk_samples / ring <= 0 pick defaults (16 workers, fewer under a smaller affinity mask or cgroup
 * CPU quota; six chunks of 1 Mi samples written with streaming stores -- with MGB_HOST_NT=0 sixteen chunks of
 * 64 Ki samples, a 4 MB ring that stays in the cores' caches).  One transfer at a time per mgb_host_io. */
typedef struct mgb_host_io mgb_host_io;
int mgb_host_io_create(int32_t threads, int64_t chunk_samples, int32_t ring, mgb_host_io** out);
int mgb_host_io_destroy(mgb_host_io* io);
int mgb_host_io_threads(const mgb_host_io* io);
/* pinned host memory for results (cudaHostAlloc); NULL on failure */
void* mgb_host_alloc(int64_t bytes);
void mgb_host_free(void* p);
/* host array -> device float32; returns when the last chunk has left the staging ring */
int mgb_host_upload(mgb_host_io* io, const void* h_src, int32_t src_width, float* d_dst, int64_t samples, void* stream);
/* device float32 -> host array.  Pinned float32 destinations (mgb_host_alloc) are written by ONE DMA.  Pinned
 * float64 destinations: up to 64 Mi samples as float32 chunks through the ring, widened by the workers; above
 * that (or with option host_download_ring = 0) widened on the device into d_wide (`samples` doubles; NULL = no
 * such route) and written by ONE DMA.  Anything else is filled by the workers from chunks that come through the
 * ring.  Synchronises `stream`. */
int mgb_host_download(mgb_host_io* io, const float* d_src, void* h_dst, int32_t dst_width, int64_t samples,
                      double* d_wide, void* stream);
/* 1 if a pinned float64 result of `samples` samples crosses the link as float32 (ring route), 0 if as float64 */
int mgb_host_download_through_ring(int64_t samples);

/* device staging of one job, provided by the caller (PyTorch allocations on the Python side) */
typedef struct mgb_host_buffers {
    float* d_target_lr;    /* target_frames stereo frames */
    float* d_reference_lr; /* reference_frames */
    float* d_result_lr;    /* target_frames */
    float* d_out_lr;       /* target_frames */
    double* d_wide;        /* optional: 2 * target_frames doubles (direct float64 download) */
    void* d_workspace;     /* layout->workspace_bytes */
    mgb_track_state* d_state;
} mgb_host_buffers;

/* stages.main (matchering/stages.py:210-272) in ONE call on the caller's host arrays: upload, stages
 * 1-4, download of every requested output (NULL = not needed, like the reference's need_* flags).
 * Returns after the outputs and *h_state_out (optional) are in host memory. */
int mgb_stages_main_host(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* layout, const void* h_target,
                         const void* h_reference, int32_t in_width, void* h_out_limited, void* h_out_no_limiter,
                         void* h_out_normalized, int32_t out_width, const mgb_host_buffers* dev,
                         mgb_track_state* h_state_out, void* stream);
/* The same with the reference from a device profile (mgb_analyze_reference): only the target crosses the link.
 * dev->d_reference_lr is not used and may be NULL; `layout` comes from mgb_track_layout_init_profiled. */
int mgb_stages_main_host_profiled(mgb_host_io* io, const mgb_plan* plan, const mgb_track_layout* layout,
                                  const void* h_target, int32_t in_width, const void* d_profile, void* h_out_limited,
                                  void* h_out_no_limiter, void* h_out_normalized, int32_t out_width,
                                  const mgb_host_buffers* dev, mgb_track_state* h_state_out, void* stream);
/* limiter.limit (matchering/limiter/hyrax.py:78-99) on a host array.  *h_engaged_out = 0 means the
 * reference would return its input object untouched (hyrax.py:83-85): h_out is then NOT written. */
int mgb_limit_host(mgb_host_io* io, const mgb_limiter_params* params, const void* h_in, int32_t in_width, void* h_out,
                   int32_t out_width, int64_t frames, float* d_in_lr, float* d_out_lr, double* d_wide, void* d_workspace,
                   int64_t workspace_bytes, int32_t* d_engaged, int32_t* h_engaged_out, void* stream);

/* ---- batches of tracks with HOST buffers: `depth` tracks in flight ------------------------------
 * mgb_process_host serialises copies and kernels of one track; tracks are independent, so a
 * pipeline overlaps track k+1's host->device copy, track k's kernels and track k-1's device->host
 * copy on three streams.  The pipeline object owns its device staging buffers (the one place in
 * this library that calls cudaMalloc).  Host buffers should be pinned and must stay valid until
 * mgb_pipeline_wait returns for their slot.  submit blocks only when the slot it is about to reuse
 * still holds an uncollected result. */
typedef struct mgb_pipeline mgb_pipeline;
int mgb_pipeline_create(const mgb_plan* plan, int64_t max_target_frames, int64_t max_reference_frames, int32_t depth,
                        mgb_pipeline** out);
int mgb_pipeline_submit(mgb_pipeline* p, const float* h_target_lr, int64_t target_frames, const float* h_reference_lr,
                        int64_t reference_frames, float* h_out_limited, int32_t* slot_out);
/* Same with PCM host buffers (what audio files hold): interleaved int16 or packed int24 in, the
 * limited result out as int16 / int24; a quarter to a half of the PCIe bytes of the float32 entry. */
int mgb_pipeline_submit_pcm(mgb_pipeline* p, const void* h_target_pcm, int32_t target_bits, int64_t target_frames,
                            const void* h_reference_pcm, int32_t reference_bits, int64_t reference_frames,
                            void* h_out_pcm, int32_t out_bits, int32_t* slot_out);
/* Both with the reference from a device profile instead of reference samples: no reference bytes cross the link.
 * d_profile must stay valid until mgb_pipeline_wait returns for the slot.  Paired and profiled submissions may be
 * mixed in one pipeline; its slot workspace covers both. */
int mgb_pipeline_submit_profiled(mgb_pipeline* p, const float* h_target_lr, int64_t target_frames, const void* d_profile,
                                 float* h_out_limited, int32_t* slot_out);
int mgb_pipeline_submit_pcm_profiled(mgb_pipeline* p, const void* h_target_pcm, int32_t target_bits, int64_t target_frames,
                                     const void* d_profile, void* h_out_pcm, int32_t out_bits, int32_t* slot_out);
int mgb_pipeline_wait(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out);
/* Meter every later submission: called before the first submit, it allocates each slot's meter workspace and
 * result.  Every submit then runs mgb_loudness on its float32 limited output (before any PCM quantisation) on
 * the slot's compute stream and copies the result back with the state.  params->d_tables must stay valid until
 * the pipeline is destroyed.  A pipeline that never calls this allocates and launches nothing for metering. */
int mgb_pipeline_enable_loudness(mgb_pipeline* p, const mgb_loudness_params* params);
/* mgb_pipeline_wait, and the slot's meter (MGB_ERR_INVALID when metering is not enabled) */
int mgb_pipeline_wait_loudness(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out,
                               mgb_loudness_result* loudness_out);
/* Master every later submission's limited output at a loudness target (mgb_finalize_to_loudness in place of
 * mgb_finalize, on the slot's compute stream); the slot's meter then meters the searched output and the report is copied
 * back with the state and the meter.  Called after mgb_pipeline_enable_loudness (the search uses its meter) and before
 * the first submit; MGB_ERR_INVALID otherwise, or for a target mgb_finalize_to_loudness would reject.  Allocates each
 * slot's search workspace and report.  A pipeline that never calls this runs exactly what it did before. */
int mgb_pipeline_enable_loudness_target(mgb_pipeline* p, const mgb_loudness_target* target);
/* mgb_pipeline_wait_loudness, and the slot's loudness-target report (MGB_ERR_INVALID when no target is set) */
int mgb_pipeline_wait_loudness_target(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out,
                                      mgb_loudness_result* loudness_out, mgb_loudness_target_report* report_out);
int mgb_pipeline_streams(mgb_pipeline* p, void** h2d, void** compute, void** d2h);
int mgb_pipeline_destroy(mgb_pipeline* p);

/* float64 <-> float32 interleaved conversion on the device (the reference hands float64 arrays
 * to stages.main; core.py:53-62 / soundfile's default read dtype). */
int mgb_convert_f64_to_f32(const double* d_in, float* d_out, int64_t count, void* stream);
int mgb_convert_f32_to_f64(const float* d_in, double* d_out, int64_t count, void* stream);

/* PCM <-> float32 on the device, the conversions libsndfile performs at the reference's file
 * boundary (matchering/loader.py:35 sf.read -> x / 2^(bits-1); matchering/saver.py:32 sf.write ->
 * lrint(x * (2^(bits-1) - 1)), clipped).  bits = 16 (int16) or 24 (packed little-endian triplets);
 * `count` = samples (frames * channels). */
int mgb_pcm_decode(const void* d_pcm, int32_t bits, float* d_out, int64_t count, void* stream);
int mgb_pcm_encode(const float* d_in, int32_t bits, void* d_pcm, int64_t count, void* stream);

/* Dithered PCM encode: TPDF dither, optionally noise-shaped by error feedback, then rounding to 16 or 24 bits, in place
 * of mgb_pcm_encode's plain rounding (DESIGN.md §4 "Dither" states the definition the output follows to the bit).  Per
 * channel of the stereo float32 frames at d_lr, in float64, top = 2^(bits-1) - 1:
 *   d[n, c] = (a - b) / 2^24, a = z >> 40, b = (z >> 16) & 0xFFFFFF, z = splitmix64 finaliser of
 *             seed + (2n + c + 1) * 0x9E3779B97F4A7C15 (mod 2^64)                TPDF in (-1, 1) LSB
 *   fb = sum of h[k-1] * e[n-k] for k = taps .. 1, oldest first, every product and sum rounded (no FMA)
 *   v = x * top - fb, q = rint(v + d) (ties to even), e[n] = q - v, out = clip(q, -top - 1, top)
 *   (a non-finite q: e[n] = 0 and mgb_pcm_encode's sample)
 * Each channel runs in segments of 1024 frames, each from a zero error history 32 frames before its first frame (at
 * frame 0 for the first), so the output depends on neither the grid nor the stream.  |e| < 1.5 LSB for any taps.
 * taps = 0 is flat TPDF.  Zero taps appended to h change no bit.  d_pcm: int16 pairs or packed little-endian 24-bit
 * triplets, `frames` frames.  MGB_ERR_UNSUPPORTED for bits other than 16 / 24; MGB_ERR_INVALID for taps outside
 * [0, MGB_MAX_DITHER_TAPS], a non-finite h[0 .. taps), a nonzero `reserved`, NULL or not 16-byte aligned pointers, or
 * frames < 0.  frames = 0 does nothing.  No workspace. */
#define MGB_MAX_DITHER_TAPS 32
typedef struct mgb_dither_params {
    uint64_t seed;
    int32_t taps;     /* shaping taps h_1 .. h_taps in h[0 .. taps) */
    int32_t reserved; /* 0 */
    double h[MGB_MAX_DITHER_TAPS];
} mgb_dither_params;
int mgb_pcm_encode_dithered(const mgb_dither_params* params, const float* d_lr, int64_t frames, int32_t bits, void* d_pcm,
                            void* stream);
/* The batch pipeline (above): dither every later PCM submission.  Its limited output is then quantised by
 * mgb_pcm_encode_dithered with these parameters instead of mgb_pcm_encode; float32 submissions are unaffected.  Called
 * once, before the first submit; MGB_ERR_INVALID otherwise, or for parameters mgb_pcm_encode_dithered would reject.  A
 * pipeline that never calls this runs exactly what it did before. */
int mgb_pipeline_enable_dither(mgb_pipeline* p, const mgb_dither_params* params);

/* Checker reductions on the device (matchering/checker.py:64-88,140-142; dsp.count_max_peaks
 * dsp.py:49-54).  mgb_check_peaks: d_scratch16 (16 bytes, device) receives {float peak; pad;
 * uint64 count of samples with isclose(|x|, peak)} for `frames` stereo frames.
 * mgb_check_equality: d_scratch8 receives the uint64 number of samples where the two signals are
 * not allclose (0 => the reference would raise ERROR_TARGET_EQUALS_REFERENCE). */
int mgb_check_peaks(const float* d_lr, int64_t frames, void* d_scratch16, void* stream);
int mgb_check_equality(const float* d_a_lr, const float* d_b_lr, int64_t frames, void* d_scratch8, void* stream);

/* Preview creator on the device (matchering/preview_creator.py:30-94; dsp.strided_app_2d,
 * batch_rms_2d, fade: dsp.py:128-152).
 * mgb_window_energy: d_energy[w] = sum of L^2 + R^2 (float64) over the window [w*step, w*step+window)
 * for w < count -- the argmax of the reference's per-window RMS picks the preview.
 * mgb_preview_piece: d_out = clip(d_in, +-clip_to) (clip_to <= 0: no clip; the reference clips the
 * target at the threshold) with linspace(0, 1, fade_frames) fades at both ends (0: no fade). */
int mgb_window_energy(const float* d_lr, int64_t frames, int64_t window, int64_t step, int32_t count, double* d_energy,
                      void* stream);
int mgb_preview_piece(const float* d_in_lr, float* d_out_lr, int64_t frames, double clip_to, int64_t fade_frames,
                      void* stream);

/* Resampling to Config.internal_sample_rate (matchering/checker.py:30-44 = resampy.resample(array, rate_in,
 * rate_out, axis=0), filter "kaiser_best"; resampy/core.py, resampy/interpn.py).  d_win_delta: nwin pairs of
 * doubles (table entry, forward difference to the next entry; the last difference is 0) -- half of the
 * Kaiser-windowed sinc at num_table entries per zero crossing, already scaled by rate_out/rate_in when that is
 * below 1 (built by matchering_b200/resample.py).  frames_out must equal mgb_resample_frames(): resampy's
 * int(frames_in * rate_out / rate_in). */
int64_t mgb_resample_frames(int64_t frames_in, int32_t rate_in, int32_t rate_out);
int mgb_resample(const float* d_in_lr, int64_t frames_in, int32_t rate_in, float* d_out_lr, int64_t frames_out,
                 int32_t rate_out, const double* d_win_delta, int32_t nwin, int32_t num_table, void* stream);

/* ---- building blocks exported for the parity tests (tests/ only) ------------------------------ */
/* forward or inverse (dir = +1 / -1) complex FFT of `batch` frames of n points through the same
 * shared-memory kernel the pipeline uses; is_f64 selects the double variant (n in {F, 2F}). */
int mgb_test_fft(int32_t n, int32_t is_f64, int32_t dir, const void* d_in, void* d_out, int32_t batch,
                 const void* d_twiddles, void* stream);
/* the limiter's two scanned gain envelopes instead of its output: d_gains_out[n] = (attack gain g_att[n]
 * (hyrax.py:48-51, the filtfilt result), release gain max(hold_out, release_out)[n] (hyrax.py:56-75)).  Same
 * arguments as mgb_limit; served on the halo kernel for the 44.1 / 96 kHz default windows, and for every Config that
 * takes the wide-window path (windows wider than the halo kernel's span). */
int mgb_test_limiter_gains(const mgb_limiter_params* params, const float* d_in_lr, float* d_gains_out, int64_t frames,
                           void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream);
/* the true-peak limiter's detector plane alone (the kernel mgb_limit runs in true-peak mode): d_out[n] = d[n] =
 * max(u[n], u[n-1]) for the `frames` stereo frames at d_lr, oversampling 1, 2 or 4 (mgb_limiter_params.true_peak), and
 * *d_max = max(*d_max, max(d)).  *d_max must hold 0 (or a smaller value) before the call.  Every pointer 16-byte
 * aligned. */
int mgb_test_true_peak_detect(int32_t oversample, const float* d_lr, int64_t frames, float* d_out, float* d_max,
                              void* stream);
/* the FIR design alone from given average spectra: d_avg = [4][n_lin] doubles
 * (target mid, target side, reference mid, reference side), already scaled. d_fir_out [2][F]. */
int mgb_test_design_fir(const mgb_plan* plan, const double* d_avg, double* d_fir_out, void* d_workspace,
                        void* stream);
/* where the stages leave their hand-off values in a job's workspace: out[0..12] = byte offsets from d_workspace of
 * spec_part_t, spec_part_r, sumsq_part_t, sumsq_part_r, absmax_part_t, absmax_part_r, mask_t, mask_r, h_mid, h_side,
 * loud_values, piece_sums, loud_count; out[13] = loud_capacity (entries per piece); out[14] = byte offset and out[15] =
 * size of the limiter's tickets and look-back words (cleared by mgb_finalize before every limiter launch). */
int mgb_test_workspace_regions(const mgb_plan* plan, const mgb_track_layout* layout, int64_t out[16]);

#ifdef __cplusplus
}
#endif
#endif /* MATCHERING_B200_H */
