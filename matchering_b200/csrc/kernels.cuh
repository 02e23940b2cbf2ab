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
    int64_t limiter_zero_bytes;
    int64_t design_stride;  // doubles per channel in `design`
    int64_t total_bytes;
};

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
int64_t operator_workspace_bytes(const mgb_plan& plan);
int build_operator(const mgb_plan& plan, double* op_out, void* workspace, cudaStream_t stream);
extern int g_design_direct;  // tests: force the direct (non-operator) smoothing in mgb_test_design_fir

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
int launch_convert_f64_f32(const double* in, float* out, int64_t count, cudaStream_t stream);
int launch_convert_f32_f64(const float* in, double* out, int64_t count, cudaStream_t stream);

// limiter.cu ------------------------------------------------------------------------------------
int launch_limiter(const mgb_limiter_params& lp, const float2* in, float2* out, int64_t frames, const double* pre_gain,
                   const double* post_gain, const int* engaged, int* ticket, void* lookback, const void* tables,
                   cudaStream_t stream, bool gains_only = false);
int launch_limiter_tables(const mgb_limiter_params& lp, void* tables, cudaStream_t stream);
int launch_limiter_engaged(const float* peak_bits, const double* pre_gain, double threshold, int* engaged,
                           cudaStream_t stream);

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

}  // namespace mgb
