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
    int32_t warmup;     /* samples after which attack_c^n < 1e-10 (halo of the attack filter) */
    int32_t hold_order;    /* LimiterConfig.hold_filter_order    (defaults.py:48-50) */
    int32_t release_order; /* LimiterConfig.release_filter_order (defaults.py:54-56) */
    int32_t reserved;
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
 * 1 hands the limiter's chunks out by an atomic ticket instead of the block index (0, default).
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
 * reference would return its input untouched (hyrax.py:83-85; d_out is then a copy of d_in). */
int64_t mgb_limiter_workspace_bytes(const mgb_limiter_params* params, int64_t frames);
int mgb_limit(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
              void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream);

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
int mgb_pipeline_wait(mgb_pipeline* p, int32_t slot, mgb_track_state* state_out);
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
 * arguments as mgb_limit; kernels exist for the 44.1 / 96 kHz default windows. */
int mgb_test_limiter_gains(const mgb_limiter_params* params, const float* d_in_lr, float* d_gains_out, int64_t frames,
                           void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream);
/* the FIR design alone from given average spectra: d_avg = [4][n_lin] doubles
 * (target mid, target side, reference mid, reference side), already scaled. d_fir_out [2][F]. */
int mgb_test_design_fir(const mgb_plan* plan, const double* d_avg, double* d_fir_out, void* d_workspace,
                        void* stream);
/* where the stages leave their hand-off values in a job's workspace: out[0..12] = byte offsets from d_workspace of
 * spec_part_t, spec_part_r, sumsq_part_t, sumsq_part_r, absmax_part_t, absmax_part_r, mask_t, mask_r, h_mid, h_side,
 * loud_values, piece_sums, loud_count; out[13] = loud_capacity (entries per piece); out[14..15] = 0. */
int mgb_test_workspace_regions(const mgb_plan* plan, const mgb_track_layout* layout, int64_t out[16]);

#ifdef __cplusplus
}
#endif
#endif /* MATCHERING_B200_H */
