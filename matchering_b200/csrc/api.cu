// C ABI of libmatchering_b200 (include/matchering_b200.h): argument checking, workspace carving,
// stage sequencing.  No kernel lives here except the FFT test harness.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "fft.cuh"
#include "kernels.cuh"

namespace mgb {

int g_use_tma = 1;
int g_twiddle_chain = 1;
int g_analyze_chain = 1;
int g_conv_persistent = 1;
int g_conv_fused = 1;
int g_conv_ovs = 4;
int g_lookback_inclusive = 1;
int g_limiter_ticket = 0;

#ifndef MGB_EMULATE
long long g_launch_count = 0;
int g_profile = 0;
namespace {
struct ProfileRecord {
    const char* what;
    cudaEvent_t start, stop;
};
std::vector<ProfileRecord> g_records;
}  // namespace
void profile_mark(const char* what, cudaStream_t stream, bool begin) {
    if (begin) {
        ProfileRecord r;
        r.what = what;
        cudaEventCreate(&r.start);
        cudaEventCreate(&r.stop);
        cudaEventRecord(r.start, stream);
        g_records.push_back(r);
    } else if (!g_records.empty()) {
        cudaEventRecord(g_records.back().stop, stream);
    }
}
#endif

static thread_local char g_error[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

#ifdef MGB_EMULATE
int cuda_status(const char*) { return MGB_OK; }
int num_sms() { return 8; }
#else
int cuda_status(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return MGB_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return MGB_ERR_CUDA;
}
int num_sms() {
    static int cached = 0;
    if (!cached) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;  // the H100 SXM's SM count
    }
    return cached;
}
#endif

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

// With base_ptr == nullptr every pointer of the result holds its region's byte offset (mgb_test_workspace_regions).
Workspace carve_workspace(const mgb_plan& plan, const mgb_track_layout& L, void* base_ptr) {
    Workspace w;
    const uintptr_t base = reinterpret_cast<uintptr_t>(base_ptr);
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        unsigned char* p = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
        off += align256(bytes);
        return p;
    };
    const int64_t HB = plan.n_lin, F = plan.fft_size;
    const int64_t items_t = (int64_t)L.target_divisions * L.target_slots;
    const int64_t items_r = (int64_t)L.reference_divisions * L.reference_slots;
    w.spec_part_t = (float*)take(items_t * 2 * HB * 4);
    w.spec_part_r = (float*)take(items_r * 2 * HB * 4);
    w.sumsq_part_t = (double*)take(items_t * 8);
    w.sumsq_part_r = (double*)take(items_r * 8);
    w.absmax_part_t = (float*)take((items_t + 1) * 4);
    w.absmax_part_r = (float*)take((items_r + 1) * 4);
    w.mask_t = take(L.target_divisions);
    w.mask_r = take(L.reference_divisions);
    w.design_stride = (design_doubles_per_channel(plan) + 31) / 32 * 32;
    w.design = (double*)take(8 * w.design_stride * 8);  // 2 channels x up to 4 design CTAs
    w.h_mid = (float2*)take((2 * F + 1) * 8);           // FIR spectrum bins 0..N/2 of the N = 2F or 4F grid
    w.h_side = (float2*)take((2 * F + 1) * 8);
    w.loud_capacity = loud_capacity(L.target_piece);
    w.loud_values = (float*)take(w.loud_capacity * L.target_divisions * 4);
    w.result_slot = (const float2**)take(8);
    w.target_peak = (float*)take(4);
    w.conv_scratch = (float2*)take(conv_global_scratch_bytes(plan.fft_size, L.target_frames));
    w.zero_begin = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
    w.piece_sums = (double*)take((int64_t)MGB_MAX_CORRECTION_STEPS * L.target_divisions * 8);
    w.loud_count = (unsigned*)take((int64_t)L.target_divisions * 4);
    w.zero_end = reinterpret_cast<unsigned char*>(base + (uintptr_t)off);
    // zeroed by mgb_finalize right before every limiter launch (a second finalize on the same track
    // must not find the first one's tickets and published carries)
    const int64_t limiter_zero_from = off;
    w.tickets = (int*)take(256);
    w.lookback = take(limiter_lookback_bytes(plan.limiter, L.target_frames));
    w.limiter_zero_bytes = off - limiter_zero_from;
    w.total_bytes = off;
    return w;
}

static int check_plan(const mgb_plan* plan) {
    MGB_REQUIRE(plan != nullptr, MGB_ERR_INVALID, "plan is NULL");
    const int F = plan->fft_size;
    MGB_REQUIRE(F == 512 || F == 1024 || F == 2048 || F == 4096 || F == 8192 || F == 16384, MGB_ERR_UNSUPPORTED,
                "fft_size %d: kernels exist for 512, 1024, 2048, 4096, 8192, 16384", F);
    MGB_REQUIRE(plan->n_lin == F / 2 + 1 && plan->n_log >= 4, MGB_ERR_INVALID, "plan grid sizes inconsistent");
    MGB_REQUIRE(plan->rms_correction_steps >= 0 && plan->rms_correction_steps <= MGB_MAX_CORRECTION_STEPS,
                MGB_ERR_UNSUPPORTED, "rms_correction_steps %d > %d", plan->rms_correction_steps, MGB_MAX_CORRECTION_STEPS);
    MGB_REQUIRE(plan->lowess_k >= 2 && plan->lowess_k <= plan->n_log && plan->lowess_nfit >= 2, MGB_ERR_INVALID,
                "plan LOWESS sizes inconsistent");
    return MGB_OK;
}

static int check_aligned(const void* p, const char* name) {
    MGB_REQUIRE(p != nullptr, MGB_ERR_INVALID, "%s is NULL", name);
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, MGB_ERR_INVALID, "%s is not 16-byte aligned", name);
    return MGB_OK;
}

// ------------------------------------------------------------------------------------------------
// FFT test harness: one frame per CTA through fft_run, global -> shared -> global
// ------------------------------------------------------------------------------------------------
template <typename T> struct TestPlanes { using type = SplitPlanes<T>; };
template <> struct TestPlanes<float> { using type = PackedPlanes; };  // what the float32 kernels use

template <int N, int DIR, typename T, int THREADS>
__global__ void __launch_bounds__(THREADS) test_fft_kernel(const cpx<T>* __restrict__ in, cpx<T>* __restrict__ out,
                                                           const cpx<T>* __restrict__ tw) {
    MGB_DYN_SMEM(smem);
    using P = typename TestPlanes<T>::type;
    P planes;
    if constexpr (sizeof(T) == 4) {
        planes.z = reinterpret_cast<float2*>(smem);
    } else {
        planes.re = reinterpret_cast<T*>(smem);
        planes.im = planes.re + P::elems(N);
    }
    const cpx<T>* src = in + (long long)blockIdx.x * N;
    cpx<T>* dst = out + (long long)blockIdx.x * N;
    auto first = [&](int i) { return src[i]; };
    auto last = [&](int i, cpx<T> v) { dst[i] = v; };
    fft_run<N, DIR, THREADS, T, sizeof(T) == 4>(planes, tw, first, last, false, false);
}

template <int N, typename T, int THREADS>
static int launch_test_fft_t(int dir, const void* in, void* out, int batch, const void* tw, cudaStream_t stream) {
    const size_t smem = TestPlanes<T>::type::bytes(N);
    if (dir > 0)
        return launch("test_fft_kernel", test_fft_kernel<N, +1, T, THREADS>, dim3(batch), dim3(THREADS), smem, stream,
                      (const cpx<T>*)in, (cpx<T>*)out, (const cpx<T>*)tw);
    return launch("test_fft_kernel", test_fft_kernel<N, -1, T, THREADS>, dim3(batch), dim3(THREADS), smem, stream,
                  (const cpx<T>*)in, (cpx<T>*)out, (const cpx<T>*)tw);
}

int launch_test_fft(int n, int is_f64, int dir, const void* in, void* out, int batch, const void* tw,
                    cudaStream_t stream) {
#define MGB_FFT_CASE(NN)                                                                                      \
    case NN:                                                                                                  \
        return is_f64 ? launch_test_fft_t<NN, double, 512>(dir, in, out, batch, tw, stream)                   \
                      : launch_test_fft_t<NN, float, NN / 16>(dir, in, out, batch, tw, stream);
    switch (n) {
        MGB_FFT_CASE(512)
        MGB_FFT_CASE(1024)
        MGB_FFT_CASE(2048)
        MGB_FFT_CASE(4096)
        MGB_FFT_CASE(8192)
        case 16384:
            if (!is_f64) return launch_test_fft_t<16384, float, 1024>(dir, in, out, batch, tw, stream);
            break;
        default: break;
    }
#undef MGB_FFT_CASE
    set_error("fft: size %d (%s) has no kernel", n, is_f64 ? "f64" : "f32");
    return MGB_ERR_UNSUPPORTED;
}

template <int N>
static void radices_of(int* npass, int r[4]) {
    *npass = Radices<N>::n;
    for (int i = 0; i < 4; ++i) r[i] = Radices<N>::r[i];
}
static bool radix_schedule(int n, int* npass, int r[4]) {
    switch (n) {
        case 512: radices_of<512>(npass, r); return true;
        case 1024: radices_of<1024>(npass, r); return true;
        case 2048: radices_of<2048>(npass, r); return true;
        case 4096: radices_of<4096>(npass, r); return true;
        case 8192: radices_of<8192>(npass, r); return true;
        case 16384: radices_of<16384>(npass, r); return true;
        case 32768: radices_of<32768>(npass, r); return true;
        default: return false;
    }
}
template <int N>
static bool inverse_radices_of(int* npass, int r[4]) {
    if constexpr (InverseRadices<N>::fused) {
        *npass = InverseRadices<N>::n;
        for (int i = 0; i < 4; ++i) r[i] = InverseRadices<N>::r[i];
        return true;
    } else {
        return false;
    }
}
// the second schedule the fused convolution keeps behind the forward one in the 2F float table
static bool inverse_schedule(int n, int* npass, int r[4]) {
    switch (n) {
        case 8192: return inverse_radices_of<8192>(npass, r);
        case 16384: return inverse_radices_of<16384>(npass, r);
        default: return false;
    }
}
static int schedule_count(int npass, const int r[4]) {
    int total = 0, ns = r[0];
    for (int p = 1; p < npass; ++p) {
        total += (r[p] - 1) * ns;
        ns *= r[p];
    }
    return total;
}
int twiddle_count(int n) {
    int npass, r[4];
    if (!radix_schedule(n, &npass, r)) return -1;
    return schedule_count(npass, r);
}
int inverse_twiddle_count(int n) {
    int npass, r[4];
    if (!inverse_schedule(n, &npass, r)) return 0;
    return schedule_count(npass, r);
}
// the 4F-point transform pair of the long-frame convolution (conv_frame_ovs == 4), kept behind the 2F tables
int long_frame_twiddle_count(int fft_size) {
    const int n4 = 4 * fft_size;
    int npass, r[4];
    if (!inverse_schedule(n4, &npass, r)) return 0;
    return twiddle_count(n4) + inverse_twiddle_count(n4);
}
int fill_twiddles(int n, int is_f64, void* table, cudaStream_t stream) {
    int npass, r[4];
    MGB_REQUIRE(radix_schedule(n, &npass, r), MGB_ERR_UNSUPPORTED, "fft: size %d has no radix schedule", n);
    if (is_f64)
        return launch("fft_twiddle_kernel", fft_twiddle_kernel<double>, dim3(16), dim3(256), 0, stream, (cpx<double>*)table,
                      npass, r[0], r[1], r[2], r[3]);
    return launch("fft_twiddle_kernel", fft_twiddle_kernel<float>, dim3(16), dim3(256), 0, stream, (cpx<float>*)table,
                  npass, r[0], r[1], r[2], r[3]);
}
int fill_inverse_twiddles(int n, cpx<float>* table, cudaStream_t stream) {
    int npass, r[4];
    if (!inverse_schedule(n, &npass, r)) return MGB_OK;
    return launch("fft_twiddle_kernel", fft_twiddle_kernel<float>, dim3(16), dim3(256), 0, stream, table + twiddle_count(n),
                  npass, r[0], r[1], r[2], r[3]);
}

}  // namespace mgb

using namespace mgb;

// ================================================================================================
extern "C" {

int mgb_version(void) { return MGB_VERSION; }
const char* mgb_last_error_string(void) { return g_error; }

int mgb_set_option(const char* name, int value) {
    MGB_REQUIRE(name != nullptr, MGB_ERR_INVALID, "option name is NULL");
    if (strcmp(name, "tma") == 0) {
        g_use_tma = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "conv_frame") == 0) {
        MGB_REQUIRE(value == 2 || value == 4, MGB_ERR_INVALID, "conv_frame must be 2 or 4 (FIR lengths per overlap-save frame)");
        g_conv_ovs = value;
        return MGB_OK;
    }
    if (strcmp(name, "conv_fused") == 0) {
        g_conv_fused = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "twiddle_chain") == 0) {
        g_twiddle_chain = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "conv_persistent") == 0) {
        g_conv_persistent = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "analyze_chain") == 0) {
        g_analyze_chain = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "lookback_inclusive") == 0) {
        g_lookback_inclusive = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "limiter_ticket") == 0) {
        g_limiter_ticket = value ? 1 : 0;
        return MGB_OK;
    }
    if (strcmp(name, "design_direct") == 0) {
        g_design_direct = value ? 1 : 0;
        return MGB_OK;
    }
    if (host_set_option(name, value)) return MGB_OK;
    set_error("unknown option '%s'", name);
    return MGB_ERR_INVALID;
}

long long mgb_launch_count(void) {
#ifdef MGB_EMULATE
    return 0;
#else
    return g_launch_count;
#endif
}

int mgb_profile_enable(int on) {
#ifndef MGB_EMULATE
    g_profile = on ? 1 : 0;
#else
    (void)on;
#endif
    return MGB_OK;
}

int mgb_profile_collect(char* names, int names_capacity, float* ms, int capacity) {
#ifdef MGB_EMULATE
    (void)names; (void)names_capacity; (void)ms; (void)capacity;
    return 0;
#else
    cudaDeviceSynchronize();
    int n = 0;
    int used = 0;
    if (names && names_capacity > 0) names[0] = 0;
    for (auto& r : g_records) {
        float t = 0.0f;
        cudaEventElapsedTime(&t, r.start, r.stop);
        if (n < capacity && ms) {
            ms[n] = t;
            if (names) {
                const int len = (int)strlen(r.what);
                if (used + len + 2 <= names_capacity) {
                    memcpy(names + used, r.what, len);
                    used += len;
                    names[used++] = '\n';
                    names[used] = 0;
                }
            }
            ++n;
        }
        cudaEventDestroy(r.start);
        cudaEventDestroy(r.stop);
    }
    g_records.clear();
    return n;
#endif
}

int mgb_plan_twiddle_bytes(int32_t fft_size, int64_t bytes_out[5]) {
    MGB_REQUIRE(bytes_out != nullptr, MGB_ERR_INVALID, "bytes_out is NULL");
    const int cf = twiddle_count(fft_size), c2 = twiddle_count(2 * fft_size);
    MGB_REQUIRE(cf > 0 && c2 > 0, MGB_ERR_UNSUPPORTED, "fft_size %d has no kernel", fft_size);
    bytes_out[0] = (int64_t)cf * 8;
    bytes_out[1] = (int64_t)(c2 + inverse_twiddle_count(2 * fft_size) + long_frame_twiddle_count(fft_size)) * 8;
    bytes_out[2] = (int64_t)cf * 16;
    // the convolution's float64 tables (convolve_precise_kernel): 2F points, and 4F behind them where 4F frames exist
    bytes_out[3] = (int64_t)(c2 + (long_frame_twiddle_count(fft_size) ? twiddle_count(4 * fft_size) : 0)) * 16;
    bytes_out[4] = limiter_tables_bytes();
    return MGB_OK;
}

int mgb_plan_fill_twiddles(const mgb_plan* plan, void* stream) {
    MGB_TRY(check_plan(plan));
    cudaStream_t st = (cudaStream_t)stream;
    MGB_TRY(check_aligned(plan->d_tw_f32_F, "d_tw_f32_F"));
    MGB_TRY(check_aligned(plan->d_tw_f32_2F, "d_tw_f32_2F"));
    MGB_TRY(check_aligned(plan->d_tw_f64_F, "d_tw_f64_F"));
    MGB_TRY(fill_twiddles(plan->fft_size, 0, plan->d_tw_f32_F, st));
    MGB_TRY(fill_twiddles(2 * plan->fft_size, 0, plan->d_tw_f32_2F, st));
    MGB_TRY(fill_inverse_twiddles(2 * plan->fft_size, (cpx<float>*)plan->d_tw_f32_2F, st));
    if (long_frame_twiddle_count(plan->fft_size)) {
        cpx<float>* tw4 = (cpx<float>*)plan->d_tw_f32_2F + twiddle_count(2 * plan->fft_size) + inverse_twiddle_count(2 * plan->fft_size);
        MGB_TRY(fill_twiddles(4 * plan->fft_size, 0, tw4, st));
        MGB_TRY(fill_inverse_twiddles(4 * plan->fft_size, tw4, st));
    }
    MGB_TRY(fill_twiddles(plan->fft_size, 1, plan->d_tw_f64_F, st));
    if (plan->d_tw_f64_2F) {
        MGB_TRY(fill_twiddles(2 * plan->fft_size, 1, plan->d_tw_f64_2F, st));
        if (long_frame_twiddle_count(plan->fft_size))
            MGB_TRY(fill_twiddles(4 * plan->fft_size, 1, (cpx<double>*)plan->d_tw_f64_2F + twiddle_count(2 * plan->fft_size), st));
    }
    if (!plan->d_limiter_tables) return MGB_OK;  // FFT-only plans (tests); mgb_finalize insists on the tables
    MGB_TRY(check_aligned(plan->d_limiter_tables, "d_limiter_tables"));
    return launch_limiter_tables(plan->limiter, plan->d_limiter_tables, st);
}

int64_t mgb_plan_operator_workspace_bytes(const mgb_plan* plan) {
    if (check_plan(plan) != MGB_OK) return -1;
    return operator_workspace_bytes(*plan);
}

int mgb_plan_build_operator(const mgb_plan* plan, double* d_operator_out, void* d_workspace, int64_t workspace_bytes,
                            void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_TRY(check_aligned(d_operator_out, "d_operator_out"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_REQUIRE(workspace_bytes >= operator_workspace_bytes(*plan), MGB_ERR_WORKSPACE, "operator workspace too small");
    return build_operator(*plan, d_operator_out, d_workspace, (cudaStream_t)stream);
}

int mgb_track_layout_init(const mgb_plan* plan, int64_t target_frames, int64_t reference_frames,
                          mgb_track_layout* out) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(out != nullptr, MGB_ERR_INVALID, "layout is NULL");
    // core.py:69-74 guarantees both signals are longer than fft_size
    MGB_REQUIRE(target_frames > plan->fft_size && reference_frames > plan->fft_size, MGB_ERR_INVALID,
                "target (%lld) and reference (%lld) must be longer than fft_size (%d)", (long long)target_frames,
                (long long)reference_frames, plan->fft_size);
    MGB_REQUIRE(plan->max_piece_size > 0, MGB_ERR_INVALID, "max_piece_size must be positive");
    memset(out, 0, sizeof(*out));
    out->target_frames = target_frames;
    out->reference_frames = reference_frames;
    const int sms = num_sms();
    for (int sig = 0; sig < 2; ++sig) {
        const int64_t n = sig == 0 ? target_frames : reference_frames;
        // match_levels.py:47-59: float division, then int() truncation
        const double q = (double)n / plan->max_piece_size;
        MGB_REQUIRE(q < 8000.0, MGB_ERR_UNSUPPORTED, "more than 8000 pieces (their statistics live in one CTA's shared memory)");
        const int32_t divisions = (int32_t)q + 1;
        const int64_t piece = (int64_t)((double)n / (double)divisions);
        MGB_REQUIRE(piece >= plan->fft_size, MGB_ERR_UNSUPPORTED,
                    "piece of %lld samples is shorter than fft_size %d (the reference's STFT degenerates there)",
                    (long long)piece, plan->fft_size);
        const int64_t frames_per_piece = piece / plan->fft_size;
        // analysis work items: one wave of three resident CTAs per SM (register/shared-memory limit of
        // analyze_kernel), never more items than that so that no tail wave forms
        int64_t slots = (3LL * sms) / divisions;
        if (slots > frames_per_piece) slots = frames_per_piece;
        if (slots < 1) slots = 1;
        if (sig == 0) {
            out->target_divisions = divisions;
            out->target_piece = piece;
            out->target_slots = (int32_t)slots;
        } else {
            out->reference_divisions = divisions;
            out->reference_piece = piece;
            out->reference_slots = (int32_t)slots;
        }
    }
    out->workspace_bytes = carve_workspace(*plan, *out, nullptr).total_bytes;
    return MGB_OK;
}

int mgb_match_levels(const mgb_plan* plan, const mgb_track_layout* L, const float* d_target_lr,
                     const float* d_reference_lr, void* d_workspace, mgb_track_state* d_state, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_target_lr, "d_target_lr"));
    MGB_TRY(check_aligned(d_reference_lr, "d_reference_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
#ifdef MGB_EMULATE
    memset(ws.zero_begin, 0, ws.zero_end - ws.zero_begin);
#else
    if (cudaMemsetAsync(ws.zero_begin, 0, ws.zero_end - ws.zero_begin, st) != cudaSuccess) return cuda_status("memset");
#endif
    MGB_TRY(launch_analyze(*plan, (const float2*)d_target_lr, L->target_frames, L->target_piece, L->target_divisions,
                           L->target_slots, ws.spec_part_t, ws.sumsq_part_t, ws.absmax_part_t, st));
    // the level statistics themselves (masks, match RMS, c0, final amplitude coefficient) are computed
    // from these partial sums in the prologue of the next stage's first kernel and recorded in d_state
    return launch_analyze(*plan, (const float2*)d_reference_lr, L->reference_frames, L->reference_piece,
                          L->reference_divisions, L->reference_slots, ws.spec_part_r, ws.sumsq_part_r, ws.absmax_part_r,
                          st);
}

int mgb_match_frequencies(const mgb_plan* plan, const mgb_track_layout* L, const float* d_target_lr,
                          float* d_result_lr, double* d_fir_out, void* d_workspace, mgb_track_state* d_state,
                          void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_target_lr, "d_target_lr"));
    MGB_TRY(check_aligned(d_result_lr, "d_result_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    MGB_TRY(launch_design(*plan, *L, ws, nullptr, d_fir_out, d_state, st));
    return launch_convolve(*plan, *L, (const float2*)d_target_lr, (float2*)d_result_lr, ws, d_state, st);
}

int mgb_correct_levels(const mgb_plan* plan, const mgb_track_layout* L, void* d_workspace, mgb_track_state* d_state,
                       void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    // step 0's per-piece sums and loud lists come out of the convolution kernel's epilogue (gain is
    // still 1 there); each later step is one pass over the loud lists (over the result, for a piece
    // whose list overflowed or at a gain where quiet samples could clip: the result must be unchanged
    // since mgb_match_frequencies) that first derives the previous step's coefficient from that step's
    // sums; a last small kernel closes the chain and writes the scalars __finalize needs.
    for (int step = 1; step < plan->rms_correction_steps; ++step) MGB_TRY(launch_loud_sumsq(*plan, *L, ws, step, d_state, st));
    return launch_correction_final(*plan, *L, ws, d_state, st);
}

int mgb_finalize(const mgb_plan* plan, const mgb_track_layout* L, const float* d_result_lr, float* d_out_limited,
                 float* d_out_no_limiter, float* d_out_normalized, void* d_workspace, mgb_track_state* d_state,
                 void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L != nullptr && d_state != nullptr, MGB_ERR_INVALID, "layout/state is NULL");
    MGB_TRY(check_aligned(d_result_lr, "d_result_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws = carve_workspace(*plan, *L, d_workspace);
    const float2* res = (const float2*)d_result_lr;
    if (d_out_normalized) {
        MGB_TRY(check_aligned(d_out_normalized, "d_out_normalized"));
        MGB_TRY(launch_scale(res, (float2*)d_out_normalized, L->target_frames, &d_state->gain, &d_state->normalize_coef, st));
    }
    if (d_out_no_limiter) {
        MGB_TRY(check_aligned(d_out_no_limiter, "d_out_no_limiter"));
        MGB_TRY(launch_scale(res, (float2*)d_out_no_limiter, L->target_frames, &d_state->gain, nullptr, st));
    }
    if (d_out_limited) {
        MGB_TRY(check_aligned(d_out_limited, "d_out_limited"));
#ifdef MGB_EMULATE
        memset(ws.tickets, 0, ws.limiter_zero_bytes);
#else
        if (cudaMemsetAsync(ws.tickets, 0, ws.limiter_zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
        MGB_TRY(launch_limiter(plan->limiter, res, (float2*)d_out_limited, L->target_frames, &d_state->gain,
                               &d_state->final_amplitude_coef, &d_state->limiter_engaged, ws.tickets,
                               ws.lookback, plan->d_limiter_tables, st));
    }
    return MGB_OK;
}

// standalone limiter workspace: [0,4): peak bits  [16,20): ticket  [256, kLimitHeader): pole tables  [kLimitHeader, ...): look-back words
static const int64_t kLimitHeader = 256 + 32768;

int64_t mgb_limiter_workspace_bytes(const mgb_limiter_params* params, int64_t frames) {
    if (!params) return -1;
    if (frames <= 0) return kLimitHeader;
    return kLimitHeader + limiter_lookback_bytes(*params, frames);
}

static int limit_impl(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
                      void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream, bool gains_only) {
    MGB_REQUIRE(params != nullptr, MGB_ERR_INVALID, "params is NULL");
    MGB_TRY(check_aligned(d_in_lr, "d_in_lr"));
    MGB_TRY(check_aligned(d_out_lr, "d_out_lr"));
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    MGB_REQUIRE(d_engaged != nullptr, MGB_ERR_INVALID, "d_engaged is NULL");
    MGB_REQUIRE(frames > 6, MGB_ERR_INVALID, "limit: the input must be longer than filtfilt's padlen (6)");
    MGB_REQUIRE(limiter_tables_bytes() <= 32768, MGB_ERR_WORKSPACE, "limit: pole tables outgrew the workspace header");
    MGB_REQUIRE(workspace_bytes >= mgb_limiter_workspace_bytes(params, frames), MGB_ERR_WORKSPACE,
                "limit: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
                (long long)mgb_limiter_workspace_bytes(params, frames));
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char* base = (unsigned char*)d_workspace;
    const int64_t zero_bytes = kLimitHeader + limiter_lookback_bytes(*params, frames);
#ifdef MGB_EMULATE
    memset(base, 0, zero_bytes);
#else
    if (cudaMemsetAsync(base, 0, zero_bytes, st) != cudaSuccess) return cuda_status("memset");
#endif
    void* tables = base + 256;
    MGB_TRY(launch_limiter_tables(*params, tables, st));
    float* peak = (float*)base;
    int* ticket = (int*)(base + 16);
    MGB_TRY(launch_absmax((const float2*)d_in_lr, frames, peak, st));
    MGB_TRY(launch_limiter_engaged(peak, nullptr, params->threshold, d_engaged, st));
    return launch_limiter(*params, (const float2*)d_in_lr, (float2*)d_out_lr, frames, nullptr, nullptr, d_engaged, ticket,
                          base + kLimitHeader, tables, st, gains_only);
}

int mgb_limit(const mgb_limiter_params* params, const float* d_in_lr, float* d_out_lr, int64_t frames,
              void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream) {
    return limit_impl(params, d_in_lr, d_out_lr, frames, d_workspace, workspace_bytes, d_engaged, stream, false);
}

int mgb_test_limiter_gains(const mgb_limiter_params* params, const float* d_in_lr, float* d_gains_out, int64_t frames,
                           void* d_workspace, int64_t workspace_bytes, int32_t* d_engaged, void* stream) {
    return limit_impl(params, d_in_lr, d_gains_out, frames, d_workspace, workspace_bytes, d_engaged, stream, true);
}

int mgb_process_host(const mgb_plan* plan, const mgb_track_layout* L, const float* h_target_lr,
                     const float* h_reference_lr, float* h_out_limited, float* h_out_no_limiter,
                     float* h_out_normalized, float* d_target_lr, float* d_reference_lr, float* d_result_lr,
                     float* d_out_lr, void* d_workspace, mgb_track_state* d_state, mgb_track_state* h_state_out,
                     void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(L && h_target_lr && h_reference_lr && d_state, MGB_ERR_INVALID, "NULL argument");
    MGB_REQUIRE(h_out_limited || h_out_no_limiter || h_out_normalized, MGB_ERR_INVALID, "no output requested");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t tbytes = (size_t)L->target_frames * 8, rbytes = (size_t)L->reference_frames * 8;
#ifdef MGB_EMULATE
    memcpy(d_target_lr, h_target_lr, tbytes);
    memcpy(d_reference_lr, h_reference_lr, rbytes);
#else
    if (cudaMemcpyAsync(d_target_lr, h_target_lr, tbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_status("H2D target");
    if (cudaMemcpyAsync(d_reference_lr, h_reference_lr, rbytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return cuda_status("H2D reference");
#endif
    MGB_TRY(mgb_match_levels(plan, L, d_target_lr, d_reference_lr, d_workspace, d_state, stream));
    MGB_TRY(mgb_match_frequencies(plan, L, d_target_lr, d_result_lr, nullptr, d_workspace, d_state, stream));
    MGB_TRY(mgb_correct_levels(plan, L, d_workspace, d_state, stream));
    float* outs[3] = {h_out_limited, h_out_no_limiter, h_out_normalized};
    for (int k = 0; k < 3; ++k) {
        if (!outs[k]) continue;
        MGB_TRY(mgb_finalize(plan, L, d_result_lr, k == 0 ? d_out_lr : nullptr, k == 1 ? d_out_lr : nullptr,
                             k == 2 ? d_out_lr : nullptr, d_workspace, d_state, stream));
#ifdef MGB_EMULATE
        memcpy(outs[k], d_out_lr, tbytes);
#else
        if (cudaMemcpyAsync(outs[k], d_out_lr, tbytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return cuda_status("D2H result");
#endif
    }
#ifdef MGB_EMULATE
    if (h_state_out) memcpy(h_state_out, d_state, sizeof(mgb_track_state));
#else
    if (h_state_out && cudaMemcpyAsync(h_state_out, d_state, sizeof(mgb_track_state), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return cuda_status("D2H state");
    if (cudaStreamSynchronize(st) != cudaSuccess) return cuda_status("stream sync");
#endif
    return MGB_OK;
}

int mgb_convert_f64_to_f32(const double* d_in, float* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_in && d_out && count >= 0, MGB_ERR_INVALID, "convert: bad arguments");
    return launch_convert_f64_f32(d_in, d_out, count, (cudaStream_t)stream);
}
int mgb_convert_f32_to_f64(const float* d_in, double* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_in && d_out && count >= 0, MGB_ERR_INVALID, "convert: bad arguments");
    return launch_convert_f32_f64(d_in, d_out, count, (cudaStream_t)stream);
}

int mgb_pcm_decode(const void* d_pcm, int32_t bits, float* d_out, int64_t count, void* stream) {
    MGB_REQUIRE(d_pcm && d_out && count >= 0, MGB_ERR_INVALID, "pcm_decode: bad arguments");
    return launch_pcm_decode(d_pcm, bits, d_out, count, (cudaStream_t)stream);
}
int mgb_pcm_encode(const float* d_in, int32_t bits, void* d_pcm, int64_t count, void* stream) {
    MGB_REQUIRE(d_pcm && d_in && count >= 0, MGB_ERR_INVALID, "pcm_encode: bad arguments");
    return launch_pcm_encode(d_in, bits, d_pcm, count, (cudaStream_t)stream);
}

int mgb_check_peaks(const float* d_lr, int64_t frames, void* d_scratch16, void* stream) {
    MGB_REQUIRE(d_lr && d_scratch16 && frames > 0, MGB_ERR_INVALID, "check_peaks: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_scratch16, 0, 16);
#else
    if (cudaMemsetAsync(d_scratch16, 0, 16, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_peak_count(d_lr, frames * 2, (float*)d_scratch16, (unsigned long long*)((char*)d_scratch16 + 8), st);
}

int mgb_check_equality(const float* d_a_lr, const float* d_b_lr, int64_t frames, void* d_scratch8, void* stream) {
    MGB_REQUIRE(d_a_lr && d_b_lr && d_scratch8 && frames > 0, MGB_ERR_INVALID, "check_equality: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_scratch8, 0, 8);
#else
    if (cudaMemsetAsync(d_scratch8, 0, 8, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_count_different(d_a_lr, d_b_lr, frames * 2, (unsigned long long*)d_scratch8, st);
}

int mgb_window_energy(const float* d_lr, int64_t frames, int64_t window, int64_t step, int32_t count, double* d_energy,
                      void* stream) {
    MGB_REQUIRE(d_lr && d_energy && window > 0 && step > 0 && count > 0, MGB_ERR_INVALID, "window_energy: bad arguments");
    MGB_REQUIRE((int64_t)(count - 1) * step + window <= frames, MGB_ERR_INVALID,
                "window_energy: %d windows of %lld frames every %lld do not fit in %lld frames", count, (long long)window,
                (long long)step, (long long)frames);
    MGB_REQUIRE(count <= 65535, MGB_ERR_INVALID, "window_energy: too many windows (%d)", count);
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGB_EMULATE
    memset(d_energy, 0, sizeof(double) * count);
#else
    if (cudaMemsetAsync(d_energy, 0, sizeof(double) * count, st) != cudaSuccess) return cuda_status("memset");
#endif
    return launch_window_energy((const float2*)d_lr, window, step, count, d_energy, st);
}

int mgb_preview_piece(const float* d_in_lr, float* d_out_lr, int64_t frames, double clip_to, int64_t fade_frames,
                      void* stream) {
    MGB_REQUIRE(d_in_lr && d_out_lr && frames > 0, MGB_ERR_INVALID, "preview_piece: bad arguments");
    MGB_REQUIRE(fade_frames >= 0 && 2 * fade_frames <= frames, MGB_ERR_INVALID,
                "preview_piece: two fades of %lld frames do not fit in %lld", (long long)fade_frames, (long long)frames);
    return launch_preview_piece((const float2*)d_in_lr, (float2*)d_out_lr, frames, (float)clip_to, fade_frames,
                                (cudaStream_t)stream);
}

int mgb_test_fft(int32_t n, int32_t is_f64, int32_t dir, const void* d_in, void* d_out, int32_t batch,
                 const void* d_twiddles, void* stream) {
    MGB_REQUIRE(d_in && d_out && d_twiddles && batch > 0, MGB_ERR_INVALID, "test_fft: bad arguments");
    return launch_test_fft(n, is_f64, dir, d_in, d_out, batch, d_twiddles, (cudaStream_t)stream);
}

int mgb_test_workspace_regions(const mgb_plan* plan, const mgb_track_layout* layout, int64_t out[16]) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(layout != nullptr && out != nullptr, MGB_ERR_INVALID, "test_workspace_regions: NULL argument");
    const Workspace w = carve_workspace(*plan, *layout, nullptr);  // pointers = byte offsets
    const void* regions[13] = {w.spec_part_t, w.spec_part_r, w.sumsq_part_t, w.sumsq_part_r, w.absmax_part_t,
                               w.absmax_part_r, w.mask_t, w.mask_r, w.h_mid, w.h_side, w.loud_values, w.piece_sums,
                               w.loud_count};
    for (int i = 0; i < 16; ++i) out[i] = 0;
    for (int i = 0; i < 13; ++i) out[i] = (int64_t)reinterpret_cast<uintptr_t>(regions[i]);
    out[13] = w.loud_capacity;
    return MGB_OK;
}

int mgb_test_design_fir(const mgb_plan* plan, const double* d_avg, double* d_fir_out, void* d_workspace, void* stream) {
    MGB_TRY(check_plan(plan));
    MGB_REQUIRE(d_avg && d_fir_out, MGB_ERR_INVALID, "test_design_fir: NULL argument");
    MGB_TRY(check_aligned(d_workspace, "d_workspace"));
    // workspace: [8][stride] doubles then two (2F+1) float2 spectra
    Workspace ws;
    memset(&ws, 0, sizeof(ws));
    ws.design_stride = (design_doubles_per_channel(*plan) + 31) / 32 * 32;
    ws.design = (double*)d_workspace;
    ws.h_mid = (float2*)((unsigned char*)d_workspace + align256(8 * ws.design_stride * 8));
    ws.h_side = ws.h_mid + (2 * plan->fft_size + 1 + 31) / 32 * 32;
    mgb_track_layout L;
    memset(&L, 0, sizeof(L));
    L.target_piece = L.reference_piece = plan->fft_size;
    return launch_design(*plan, L, ws, d_avg, d_fir_out, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
