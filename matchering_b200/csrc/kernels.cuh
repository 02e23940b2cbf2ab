// Internal interfaces between the translation units of libmatchering_b200.
#pragma once
#include "common.cuh"

namespace mgb {

// Device scratch of one track, carved out of the caller's workspace (all 256-byte aligned).
struct Workspace {
    float* spec_part_t;     // [Dt][St][2][n_lin]   per-(piece, slot) sums of |rfft| : mid, side
    float* spec_part_r;     // [Dr][Sr][2][n_lin]
    double* sumsq_part_t;   // [Dt][St]             per-(piece, slot) sums of mid^2
    double* sumsq_part_r;   // [Dr][Sr]
    float* absmax_part_t;   // [Dt*St + 1]
    float* absmax_part_r;   // [Dr*Sr + 1]
    unsigned char* mask_t;  // [Dt] loudest-piece mask of the target
    unsigned char* mask_r;  // [Dr]
    double* design;         // [2 channels][4 CTAs][design_stride] float64 vectors of the FIR design
    float2* h_mid;          // [2F+1] spectrum of the mid FIR on the convolution's N = 2F or 4F grid (bins 0..N/2), c0/N folded in
    float2* h_side;         // [2F+1]
    float* loud_values;     // [Dt][loud_capacity] counted mid samples of the convolution result with |mid| >= kLoudMid, per piece
    const float2** result_slot;  // device address of the convolution's result, recorded by the convolution kernel
    float* target_peak;     // max|target|, written by spectrum_mean_kernel: the convolution's choice of precision needs it
    float2* conv_scratch;   // fft_size 16384 only: one padded 2F-point frame per CTA of convolve_global_kernel
    // ---- zeroed at the start of every job (one memset) ----
    unsigned char* zero_begin;
    double* piece_sums;     // [MGB_MAX_CORRECTION_STEPS][Dt] sums of clip(mid*gain)^2
    unsigned* loud_count;   // [Dt] appends to each piece's loud list (may exceed loud_capacity: the list overflowed)
    unsigned char* zero_end;
    int64_t loud_capacity;  // entries per piece
    // ---- zeroed before every limiter launch (limiter_zero_bytes from `tickets` on) ----
    int* tickets;           // [64] zeroed counters: 0 = limiter chunk ticket
    unsigned char* lookback;// [nchunks] LookbackSlot
    float* tp_peak;         // true-peak mode: max(d), float bits (the last word of the zeroed range; else null)
    int64_t limiter_zero_bytes;
    unsigned char* limiter_planes;
    float* tp_plane;        // true-peak mode: the detector plane d (true_peak_plane_bytes; else null)  // the wide-window limiter's planes (limiter_plane_bytes; none for the halo kernel)
    const mgb_reference_profile* profile;  // profiled layouts only: the job's copy of the reference profile (else null)
    int64_t design_stride;  // doubles per channel in `design`
    int64_t total_bytes;
};

// Piece geometry of one signal (match_levels.py:47-59) and its analysis work items.
struct ReferenceGeometry {
    int64_t frames, piece;
    int32_t divisions, slots;
};
// mgb_analyze_reference's workspace: the analysis partials of the reference and its loudest-piece mask
struct ReferenceRegions {
    float* spec_part;     // [D][S][2][n_lin]
    double* sumsq_part;   // [D][S]
    float* absmax_part;   // [D*S + 1]
    unsigned char* mask;  // [D]
    int64_t total_bytes;
};
inline int64_t reference_profile_bytes(const mgb_plan& plan) {
    return (int64_t)sizeof(mgb_reference_profile) + 2LL * plan.n_lin * 8;
}

// One chunk's published scan state: value and status travel in ONE aligned 16-byte word, so a
// reader gets a consistent pair from a single load (no flag-then-fence-then-value round trips).
struct alignas(16) LookbackWord {
    double value;         // status 1: the chunk's zero-carry aggregate; status 2: its inclusive end state
    long long status;     // 0 = nothing yet
};
// (a chunk's words: the hold section's `order capacity` state components, then the release section's)

// powers of a pole for a blocked scan with `ept` elements per thread (limiter.cu)
struct ScanPow {
    double pe[27];  // p^k, k = 0..kLimiterSpanEptMax + 1 (an odd count keeps sizeof a multiple of 16: SectionTab follows it in the table)
    double ql[33];  // q^k, q = p^ept
    double qw[17];  // Q^k, Q = q^32
    double pc[33];  // P^k, P = p^kLimiterCore: weight of a chunk k chunks back (look-back)
};

constexpr int kLookbackJumps = 64;  // look-back windows with tabulated weights: 2048 chunks = 9.4 M samples back

// Powers of the companion matrix C of an order-N recursive section (hold / release low-pass) for the same blocked
// scan over its state (y[n-1], ..., y[n-N]); N = 1 is a scalar pole.
template <int N>
struct SectionTab {
    double pe[9][N];      // row 0 of C^(e+1): what the state before the thread's first element adds to element e
    double ql[33][N][N];  // C^(ept*k)
    double qw[17][N][N];  // C^(ept*32*k)
    double pc[33][N][N];  // C^(kLimiterCore*k): a chunk k chunks back (look-back)
    double pj[kLookbackJumps][N][N];  // C^(kLimiterCore*32*j): the look-back's j-th window of 32 chunks, tabulated
                                      // directly (a running product of pc[32] loses a digit per step for a pole pair)
};

constexpr int kLimiterThreads = 512;
constexpr int kLimiterCoreEpt = 9;                                   // core samples per thread
constexpr int kLimiterCore = kLimiterThreads * kLimiterCoreEpt;      // 4608 samples per chunk
constexpr int kLimiterSpanEptMax = 25;                               // span samples per thread (odd): up to 8192 samples of halo (215 KB of shared memory)

// RMS-correction steps 2..n from loud lists.  The convolution's epilogue appends every counted mid sample m with
// |m| >= kLoudMid to its piece's loud list; all other samples ("quiet") enter the later steps only through
// S_quiet = (step-0 sum) - sum over the list of clip(m)^2.  A later step at accumulated gain g takes
// g^2 S_quiet + sum over the list of clip(m*g)^2, which is exact as long as no quiet sample can clip:
// g * kLoudMid <= 1 - kLoudMargin (the margin covers the float32 rounding of the gain and the product).
// Otherwise, or when a piece's list overflowed, the step re-reads that piece of the result instead.
// 0.5 keeps the list exact up to 6 dB of correction (the benchmark tracks need at most 0.2 dB); 12-13 % of
// the samples of the c2 benchmark tracks are that loud, 5 % of c3's (11 % in its loudest piece), so a
// capacity of a quarter of the piece leaves room for twice that.
constexpr float kLoudMid = 0.5f;
constexpr double kLoudMargin = 1e-6;
inline int64_t loud_capacity(int64_t piece) { return ((piece + 3) / 4 + 3) / 4 * 4; }  // a multiple of 4: float4 rows

struct LoudList {
    float* values;
    unsigned* count;
    long long capacity;
    const float2** result_slot;
};

Workspace carve_workspace(const mgb_plan& plan, const mgb_track_layout& layout, void* base);
int64_t limiter_lookback_bytes(const mgb_limiter_params& lp, int64_t frames);
int64_t limiter_tables_bytes();

// analyze.cu ------------------------------------------------------------------------------------
int launch_analyze(const mgb_plan& plan, const float2* x, int64_t frames, int64_t piece, int divisions, int slots,
                   float* spec_part, double* sumsq_part, float* absmax_part, cudaStream_t stream);

// design.cu -------------------------------------------------------------------------------------
int launch_design(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws,
                  const double* avg_override, double* fir_out, mgb_track_state* state, cudaStream_t stream);
int64_t design_doubles_per_channel(const mgb_plan& plan);
// native-rate jobs: the curve launch_design left in `ws` (plan's job) -> the FIR of nplan's length and its spectra in `nws`
int launch_design_native(const mgb_plan& plan, const Workspace& ws, const mgb_plan& nplan, const mgb_track_layout& nlayout,
                         const Workspace& nws, double* fir_out, mgb_track_state* nstate, cudaStream_t stream);
// the reference's analysis partials (ReferenceRegions) -> a profile blob at `out` (header + spectra)
int launch_reference_profile(const mgb_plan& plan, const ReferenceGeometry& g, const ReferenceRegions& r,
                             mgb_reference_profile* out, cudaStream_t stream);
int64_t operator_workspace_bytes(const mgb_plan& plan);
int build_operator(const mgb_plan& plan, double* op_out, void* workspace, cudaStream_t stream);
extern int g_design_direct;  // tests: force the direct (non-operator) smoothing in mgb_test_design_fir

// album mastering (mgb_album_match): one entry per track, in album order
struct AlbumTrack {
    mgb_track_layout layout;
    Workspace ws;
    mgb_track_state* state;
};
// design.cu: the pooled level statistics and target spectra of the album into every track's state, mask and target peak,
// and the matching curve into `design` (a job's design blocks); then launch_design_fir
size_t album_mean_smem(const AlbumTrack* tracks, int count);
int launch_album_mean(const mgb_plan& plan, const AlbumTrack* tracks, int count, const mgb_reference_profile* profile,
                      double* design, int64_t design_stride, cudaStream_t stream);
// the smoothing and design_kernel over a matching curve already in `design`: FIR spectra on the ovs*F grid into
// h_mid / h_side, their peaks into *state
int launch_design_fir(const mgb_plan& plan, double* design, int64_t design_stride, int ovs, float2* h_mid, float2* h_side,
                      double* fir_out, mgb_track_state* state, cudaStream_t stream);
// correct.cu: RMS-correction step `step` (1 .. steps-1) and the closing kernel, pooled over the album, one launch each
int launch_album_loud_sumsq(const mgb_plan& plan, const AlbumTrack* tracks, int count, int step, cudaStream_t stream);
int launch_album_correction_final(const mgb_plan& plan, const AlbumTrack* tracks, int count, cudaStream_t stream);

// convolve.cu -----------------------------------------------------------------------------------
int conv_frame_ovs(int fft_size, long long target_piece);  // 2 or 4: transform length of the convolution in FIR lengths
int launch_convolve(const mgb_plan& plan, const mgb_track_layout& layout, const float2* target, float2* result,
                    const Workspace& ws, mgb_track_state* state, cudaStream_t stream);

// correct.cu ------------------------------------------------------------------------------------
int launch_correction_final(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws,
                            mgb_track_state* state, cudaStream_t stream);
int launch_loud_sumsq(const mgb_plan& plan, const mgb_track_layout& layout, const Workspace& ws, int step,
                      mgb_track_state* state, cudaStream_t stream);
int launch_scale(const float2* in, float2* out, int64_t frames, const double* gain, const double* divisor,
                 cudaStream_t stream);
int launch_absmax(const float2* in, int64_t frames, float* out_bits, cudaStream_t stream);
int launch_peak_count(const float* x, int64_t count, float* peak_bits, unsigned long long* n_close, cudaStream_t stream);
int launch_count_different(const float* a, const float* b, int64_t count, unsigned long long* n_diff, cudaStream_t stream);
int launch_window_energy(const float2* x, int64_t window, int64_t step, int count, double* energy, cudaStream_t stream);
int launch_preview_piece(const float2* in, float2* out, int64_t frames, float clip_to, int64_t fade, cudaStream_t stream);
int launch_pcm_decode(const void* in, int bits, float* out, int64_t count, cudaStream_t stream);
int launch_pcm_encode(const float* in, int bits, void* out, int64_t count, cudaStream_t stream);
int dither_validate(const mgb_dither_params* p);  // MGB_ERR_INVALID for parameters the dithered encoder rejects
int launch_pcm_encode_dithered(const mgb_dither_params& p, const float* in, int64_t frames, int bits, void* out,
                               cudaStream_t stream);
int launch_convert_f64_f32(const double* in, float* out, int64_t count, cudaStream_t stream);
int launch_convert_f32_f64(const float* in, double* out, int64_t count, cudaStream_t stream);

// linked versions (mgb_finalize_versions): the limiter's and the detector's entries, the main first
struct VersionPlanes {
    int count;  // 1 + versions
    const float2* in[1 + MGB_MAX_VERSIONS];
    float2* out[1 + MGB_MAX_VERSIONS];
};

// limiter.cu ------------------------------------------------------------------------------------
// (the halo kernel where its span fits, the wide-window path otherwise; wide_planes: limiter_plane_bytes of workspace)
int launch_limiter(const mgb_limiter_params& lp, const float2* in, float2* out, int64_t frames, const double* pre_gain,
                   const double* post_gain, const int* engaged, int* ticket, void* lookback, void* wide_planes,
                   const void* tables, cudaStream_t stream, bool gains_only = false, const float* tp_d = nullptr,
                   const int* skip = nullptr);  // skip: gated kernels that return at once while *skip != 0
int limiter_validate(const mgb_limiter_params& lp);
bool limiter_span_too_wide(const mgb_limiter_params& lp);  // the wide-window path serves these parameters
int64_t limiter_plane_bytes(const mgb_limiter_params& lp, int64_t frames);  // its workspace planes; 0 for the halo kernel

// limiter_wide.cuh --------------------------------------------------------------------------------
int64_t limiter_wide_lookback_bytes(const mgb_limiter_params& lp, int64_t frames, int order_capacity);
int64_t limiter_wide_plane_bytes(const mgb_limiter_params& lp, int64_t frames);
int launch_limiter_wide(const mgb_limiter_params& lp, int order_capacity, int publish_inclusive, const float2* in, float2* out,
                        int64_t frames, const double* pre_gain, const double* post_gain, const int* engaged, void* lookback,
                        void* planes, const void* tables, cudaStream_t stream, bool gains_only, const float* tp_d,
                        const int* skip, const VersionPlanes* vp = nullptr);  // vp: the linked limiter's entries
int launch_limiter_tables(const mgb_limiter_params& lp, void* tables, cudaStream_t stream);
// the linked limiter: the gain envelope of the detector plane d (D: max over the entries' detectors), applied to every
// entry of vp with the same float64 gain; the halo kernel's or the wide-window path's
int launch_limiter_versions(const mgb_limiter_params& lp, const VersionPlanes& vp, int64_t frames, const double* pre_gain,
                            const double* post_gain, const int* engaged, int* ticket, void* lookback, void* wide_planes,
                            const void* tables, const float* d, cudaStream_t stream);
int launch_limiter_engaged(const float* peak_bits, const double* pre_gain, double threshold, int* engaged,
                           cudaStream_t stream);

// true_peak.cuh -----------------------------------------------------------------------------------
void true_peak_filter(int oversample, double* h);  // the 12 L + 1 interpolator taps
int64_t true_peak_plane_bytes(const mgb_limiter_params& lp, int64_t frames);  // the detector plane; 0 without true_peak
int launch_true_peak_detect(int oversample, const float2* x, int64_t frames, float* d, float* d_max, cudaStream_t stream);
// d[n] = max(d[n], the detector of x at n) and *d_max = max(*d_max, that): a version's detector added to the main's
int launch_true_peak_accumulate(int oversample, const float2* x, int64_t frames, float* d, float* d_max, cudaStream_t stream);
// sample-peak mode's linked detector: d[n] = max over the entries of max(|L|, |R|) at n, and its maximum into *d_max
int launch_versions_detect(const VersionPlanes& vp, int64_t frames, float* d, float* d_max, cudaStream_t stream);
int launch_true_peak_final(const float* d_max, double eps, double threshold, mgb_track_state* state, cudaStream_t stream);

// loudness_target.cuh -------------------------------------------------------------------------------
int loudness_target_validate(const mgb_loudness_target* target, const mgb_loudness_params* meter);
int64_t loudness_target_search_bytes(const mgb_loudness_params& meter, int64_t frames);
int run_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& target,
                        const float2* in, const float2* s_metered, float2* out, int64_t frames, const double* gain,
                        const double* peak_d, const float* peak_bits, void* zero, int64_t zero_bytes, int* ticket,
                        void* lookback, void* planes, const void* tables, const float* tp_d, void* search_ws,
                        mgb_loudness_target_report* report, cudaStream_t stream);
// album loudness targets: one entry per track, in album order (run_loudness_search's per-track arguments)
struct AlbumSearchTrack {
    const float2* in;         // the limiter's input (s / gain)
    const float2* s_metered;  // s as samples, for the first meter run (the track's output buffer)
    float2* out;
    int64_t frames;
    const double* gain;
    const double* peak_d;
    const float* peak_bits;
    void* zero;  // the limiter's look-back words and ticket, cleared before every pass
    int64_t zero_bytes;
    void* lookback;
    void* planes;
    const float* tp_d;
};
// mgb_finalize_versions_to_loudness: run_loudness_search on entry 0 (the main) with the limiter reading the linked detector
// plane d (d_max its maximum), then one linked pass at the drive the search ended on, which writes every entry of vp
int run_versions_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& target,
                                 const VersionPlanes& vp, const float2* s_metered, int64_t frames, const double* gain,
                                 const float* d_max, const float* d, void* zero, int64_t zero_bytes, void* lookback, void* planes,
                                 const void* tables, void* search_ws, mgb_loudness_target_report* report, cudaStream_t stream);
int64_t album_loudness_target_search_bytes(const mgb_loudness_params& meter, int tracks, const int64_t* frames);
int run_album_loudness_search(const mgb_limiter_params& lp, const mgb_loudness_params& meter, const mgb_loudness_target& target,
                              const AlbumSearchTrack* tracks, int count, const void* tables, void* search_ws,
                              mgb_loudness_target_report* report, cudaStream_t stream);

// fft test entry (api.cu) uses these -------------------------------------------------------------
int launch_test_fft(int n, int is_f64, int dir, const void* in, void* out, int batch, const void* tw,
                    cudaStream_t stream);
int fill_twiddles(int n, int is_f64, void* table, cudaStream_t stream);
int twiddle_count(int n);
int inverse_twiddle_count(int n);

int conv_global_ctas(int fft_size, long long target_frames);  // convolve.cu: CTAs / scratch of the fft_size 16384 convolution
int64_t conv_global_scratch_bytes(int fft_size, long long target_frames);
extern int g_use_tma;
bool host_set_option(const char* name, int value);  // hostio.cu: the host transport's tuning switches
extern int g_limiter_ticket;      // limiter chunks by atomic ticket (1) or by block index (0, default)
extern int g_lookback_inclusive;  // limiter chunks publish their inclusive state (1, default) or aggregates only (0, tests)
extern int g_conv_ovs;       // convolution: FIR lengths per overlap-save frame where the long-frame kernel exists (4, default) or 2
extern int g_conv_fused;     // convolution: ends of both transforms in registers where the schedule allows (1)
extern int g_conv_persistent;  // convolution (16384-point frames): one CTA per SM walks its frames, next frame's bulk copy under the epilogue
extern int g_analyze_chain;  // analysis FFT: twiddle powers built in registers (1) or all read from the table (0)
extern int g_twiddle_chain;  // convolution FFTs: build twiddle powers in registers (1) or read them all (0)
extern int g_poison_alloc;   // tests: mgb_pipeline_create fills its device buffers with 0xFF bytes (1) or leaves them as allocated (0)

}  // namespace mgb
